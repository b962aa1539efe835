// extern "C" boundary (include/visdial_b200.h).  Exceptions stop here: every entry returns an error code and
// leaves the message in a thread-local buffer (vd_last_error).
#include "engine.h"
#include <string.h>
#include <cuda_profiler_api.h>

namespace vd {
void comm_unique_id(void* out);
void comm_init(Engine* e, const void* idbytes, int rank, int world);
void comm_destroy(Engine* e);
struct Corpus;
Corpus* corpus_create(Engine* eng, const vd_corpus_desc* d);
void corpus_destroy(Corpus* c);
void corpus_get_batch(Corpus* c, const int64_t* inds, int n, int decoder_gen, vd_batch* out);
void corpus_read(Corpus* c, const char* name, void* host_dst, int64_t* elems);
void corpus_batch_bytes(Corpus* c, int64_t* bytes, int32_t* launches);
void corpus_region_counts(Corpus* c, const int32_t* counts_host, int64_t numImages);
void test_kernel(Engine* e, const char* name, void* const* ptrs, int n_ptrs, const int64_t* ints, int n_ints, const double* reals,
                 int n_reals);
}  // namespace vd

using vd::Engine;

static thread_local char g_err[1024] = "";

static int fail(int code, const char* msg) {
  snprintf(g_err, sizeof(g_err), "%s", msg);
  return code;
}

#define VD_TRY(body)                                            \
  try {                                                         \
    body;                                                       \
    return VD_OK;                                               \
  } catch (const vd::CudaError& ex) {                           \
    return fail(ex.code, ex.what());                            \
  } catch (const std::exception& ex) {                          \
    return fail(VD_E_CUDA, ex.what());                          \
  } catch (...) {                                               \
    return fail(VD_E_CUDA, "unknown error");                    \
  }

struct vd_engine { Engine* e; };
#define ENG(h) ((h) ? (h)->e : (throw vd::CudaError(VD_E_BADARG, "engine handle is null"), (Engine*)nullptr))
#define NOTNULL(p) VD_REQUIRE((p) != nullptr, VD_E_BADARG, "null output pointer")

extern "C" {

const char* vd_last_error(void) { return g_err; }

int vd_layout_count(const vd_params* p, int32_t* n_segments, int64_t* n_params) {
  VD_TRY({
    vd::Layout l = vd::build_layout(vd::parse_cfg(p));
    if (n_segments) *n_segments = (int32_t)l.segs.size();
    if (n_params) *n_params = l.total;
  })
}

int vd_layout_segment(const vd_params* p, int32_t idx, char* name, int32_t name_cap, int64_t* offset, int64_t* rows,
                      int64_t* cols, int32_t* init_kind, int64_t* fan_in) {
  VD_TRY({
    vd::Layout l = vd::build_layout(vd::parse_cfg(p));
    VD_REQUIRE(idx >= 0 && idx < (int)l.segs.size(), VD_E_BADARG, "segment index out of range");
    const vd::Seg& s = l.segs[idx];
    if (name && name_cap > 0) snprintf(name, name_cap, "%s", s.name.c_str());
    if (offset) *offset = s.off;
    if (rows) *rows = s.rows;
    if (cols) *cols = s.cols;
    if (init_kind) *init_kind = s.init;
    if (fan_in) *fan_in = s.fan_in;
  })
}

int vd_create(const vd_params* p, vd_engine** out) {
  VD_TRY({
    NOTNULL(out);
    *out = nullptr;
    Engine* e = new Engine(p);
    vd_engine* h = new vd_engine;
    h->e = e;
    *out = h;
  })
}

int vd_destroy(vd_engine* h) {
  VD_TRY({
    if (h) { vd::comm_destroy(h->e); delete h->e; delete h; }
  })
}

int vd_num_params(vd_engine* h, int64_t* n) { VD_TRY({ NOTNULL(n); *n = ENG(h)->nparams; }) }
int vd_param_buffers(vd_engine* h, float** W, float** dW) {
  VD_TRY({ Engine* e = ENG(h); if (W) *W = e->W; if (dW) *dW = e->dW; })
}
int vd_optim_buffers(vd_engine* h, float** m, float** v, int64_t* t) {
  VD_TRY({ Engine* e = ENG(h); if (m) *m = e->m; if (v) *v = e->v; if (t) *t = e->adam_t; })
}
int vd_set_optim_state(vd_engine* h, const float* m_host, const float* v_host, int64_t t) {
  VD_TRY({
    Engine* e = ENG(h);
    VD_REQUIRE(m_host && v_host && t >= 0, VD_E_BADARG, "vd_set_optim_state: m / v null or t < 0");
    VD_CUDA_CHECK(cudaSetDevice(e->cfg.gpuid));
    const size_t bytes = (size_t)e->nparams * sizeof(float);
    VD_CUDA_CHECK(cudaMemcpyAsync(e->m, m_host, bytes, cudaMemcpyHostToDevice, e->cx.stream));
    VD_CUDA_CHECK(cudaMemcpyAsync(e->v, v_host, bytes, cudaMemcpyHostToDevice, e->cx.stream));
    VD_CUDA_CHECK(cudaStreamSynchronize(e->cx.stream));
    e->adam_t = t;
  })
}
int vd_set_parameters(vd_engine* h, const float* src, int64_t n) {
  VD_TRY({
    Engine* e = ENG(h);
    VD_REQUIRE(src && n == e->nparams, VD_E_SHAPE, "vd_set_parameters: n must equal vd_num_params");
    e->pool_valid = false;           // before the copy: a failed copy may have written part of the weights
    e->dses.valid = false;
    VD_CUDA_CHECK(cudaSetDevice(e->cfg.gpuid));
    VD_CUDA_CHECK(cudaMemcpyAsync(e->W, src, (size_t)n * sizeof(float), cudaMemcpyHostToDevice, e->cx.stream));
    VD_CUDA_CHECK(cudaStreamSynchronize(e->cx.stream));
  })
}
static void copy_out(Engine* e, float* dst, const float* src, int64_t n) {
  VD_REQUIRE(dst && n == e->nparams, VD_E_SHAPE, "n must equal vd_num_params");
  VD_CUDA_CHECK(cudaSetDevice(e->cfg.gpuid));
  e->join_options_backward();
  // with the overlapped gradient sync some buckets may already be all-reduced: finish the rest, so that what is read is
  // always the complete global sum (never a mixture of local and reduced segments)
  if (src == e->dW && e->world > 1) {
    bool any = false;
    for (char c : e->seg_reduced) any = any || c;
    if (any) e->reduce_remaining();
  }
  VD_CUDA_CHECK(cudaMemcpyAsync(dst, src, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost, e->cx.stream));
  VD_CUDA_CHECK(cudaStreamSynchronize(e->cx.stream));
}
int vd_get_parameters(vd_engine* h, float* dst, int64_t n) { VD_TRY({ Engine* e = ENG(h); copy_out(e, dst, e->W, n); }) }
int vd_get_gradients(vd_engine* h, float* dst, int64_t n) { VD_TRY({ Engine* e = ENG(h); copy_out(e, dst, e->dW, n); }) }
int vd_zero_grad(vd_engine* h) {
  VD_TRY({
    Engine* e = ENG(h);
    VD_CUDA_CHECK(cudaSetDevice(e->cfg.gpuid));
    e->join_options_backward();
    if (e->comm_pending) e->reduce_remaining();          // a reduction still in flight must not race the memset
    VD_CUDA_CHECK(cudaMemsetAsync(e->dW, 0, (size_t)e->nparams * sizeof(float), e->cx.stream));
    e->arm_grad_sync();
  })
}

int vd_set_training(vd_engine* h, int32_t training) {
  VD_TRY({ VD_REQUIRE(training >= 0 && training <= 2, VD_E_BADARG, "training must be 0, 1 or 2"); ENG(h)->training = training; })
}
int vd_set_dropout_seed(vd_engine* h, uint64_t seed, uint64_t iteration) {
  VD_TRY({ Engine* e = ENG(h); e->drop_seed = seed; e->drop_iter = iteration; })
}
int vd_set_option_overlap(vd_engine* h, int32_t on, int32_t reserve_sms) {
  VD_TRY({
    Engine* e = ENG(h);
    e->join_options_backward();
    if (e->opt_fwd_pending) { VD_CUDA_CHECK(cudaStreamSynchronize(e->opt_stream)); e->opt_fwd_pending = false; }
    e->opt_overlap = on != 0;
    if (reserve_sms >= 0) {
      VD_REQUIRE(reserve_sms <= e->cx.sm_count - 16, VD_E_BADARG, "reserve_sms leaves fewer than 16 SMs to the option stream");
      e->opt_reserve_sms = reserve_sms & ~1;
    }
  })
}
int vd_set_deterministic(vd_engine* h, int32_t on) {
  VD_TRY({
    Engine* e = ENG(h);
    VD_REQUIRE(on == 0 || on == 1, VD_E_BADARG, "deterministic must be 0 or 1");
    VD_REQUIRE(on == 0 || e->world == 1, VD_E_STATE, "deterministic mode runs on one GPU (world 1)");
    e->join_options_backward();        // a pending option backward finishes on the routes it was issued with
    e->cx.deterministic = on != 0;
  })
}
int vd_set_math_mode(vd_engine* h, int32_t mode) {
  VD_TRY({
    VD_REQUIRE(mode == VD_MATH_TF32 || mode == VD_MATH_FP32 || mode == VD_MATH_F16, VD_E_BADARG, "unknown math mode");
    Engine* e = ENG(h);
    e->pool_valid = false;           // the pool was encoded on the previous mode's option-LSTM route
    e->dses.valid = false;           // and a dialog session's cache on its routes
    e->math_mode = mode;
  })
}
int vd_set_answer_rules(vd_engine* h, const vd_answer_rules* r) {
  VD_TRY({
    Engine* e = ENG(h);
    if (r) e->set_answer_rules(r->min_words, r->no_repeat_ngram, r->n_banned, r->banned);
    else e->set_answer_rules(0, 0, 0, nullptr);
  })
}

int vd_encoder_forward(vd_engine* h, const vd_batch* b, const float** encOut) {
  VD_TRY({ Engine* e = ENG(h); e->encoder_forward(b); if (encOut) *encOut = e->encOut; })
}
int vd_forward_connect(vd_engine* h) { VD_TRY({ ENG(h)->forward_connect(); }) }
int vd_decoder_forward(vd_engine* h, const vd_batch* b, const float** decOut) {
  VD_TRY({
    (void)b;
    Engine* e = ENG(h);
    e->decoder_forward();
    if (decOut) *decOut = e->cfg.dec == vd::DEC_DISC ? e->scores : e->logp;
  })
}
int vd_set_lazy_decout(vd_engine* h, int32_t on) { VD_TRY({ ENG(h)->want_logp = on == 0; }) }
int vd_criterion_forward(vd_engine* h, const vd_batch* b, float* loss) {
  VD_TRY({ (void)b; NOTNULL(loss); *loss = ENG(h)->criterion_forward(); })
}
int vd_criterion_backward(vd_engine* h, const vd_batch* b) { VD_TRY({ (void)b; ENG(h)->criterion_backward(); }) }
int vd_decoder_backward(vd_engine* h, const vd_batch* b) { VD_TRY({ (void)b; ENG(h)->decoder_backward(); }) }
int vd_backward_connect(vd_engine* h, const float** gradEncOut) {
  VD_TRY({ const float* g = ENG(h)->backward_connect(); if (gradEncOut) *gradEncOut = g; })
}
int vd_encoder_backward(vd_engine* h, const vd_batch* b, const float* gradEncOut) {
  VD_TRY({ (void)b; ENG(h)->encoder_backward(gradEncOut); })
}

int vd_forward_backward(vd_engine* h, const vd_batch* b, int32_t only_forward, float* loss) {
  VD_TRY({
    Engine* e = ENG(h);
    e->encoder_forward(b);
    e->forward_connect();
    const bool saved_want = e->want_logp;
    e->want_logp = false;                 // whole-step call: decOut is not handed out, the gen logits may stay on chip
    try { e->decoder_forward(); } catch (...) { e->want_logp = saved_want; throw; }
    e->want_logp = saved_want;
    float l = e->criterion_forward();
    if (loss) *loss = l;
    if (!only_forward) {
      e->criterion_backward();
      e->decoder_backward();
      const float* g = e->backward_connect();
      e->encoder_backward(g);
    }
  })
}

int vd_forward_backward_dense(vd_engine* h, const vd_batch* b, const int32_t* round_host, const float* relevance_host,
                              float* loss_host) {
  VD_TRY({
    const float l = ENG(h)->forward_backward_dense(b, round_host, relevance_host);
    if (loss_host) *loss_host = l;
  })
}

int vd_forward_backward_dense_gen(vd_engine* h, const vd_batch* b, const int32_t* round_host, const float* relevance_host,
                                  float* loss_host) {
  VD_TRY({
    const float l = ENG(h)->forward_backward_dense_gen(b, round_host, relevance_host);
    if (loss_host) *loss_host = l;
  })
}

int vd_retrieve(vd_engine* h, const vd_batch* b, int32_t use_gt, int32_t* ranks_host) {
  VD_TRY({ ENG(h)->retrieve(b, use_gt, ranks_host); })
}
int vd_compute_ranks(vd_engine* h, const float* scores_dev, int32_t n_rows, const int32_t* gt_dev, int32_t* ranks_dev) {
  VD_TRY({
    Engine* e = ENG(h);
    VD_REQUIRE(scores_dev && ranks_dev && n_rows >= 0, VD_E_BADARG, "null scores / ranks");
    vd::rank_rows(e->cx, scores_dev, gt_dev, ranks_dev, n_rows, e->cfg.K);
  })
}
int vd_gen_option_lhood(vd_engine* h, const vd_batch* b, const float** lhood_dev) {
  VD_TRY({ (void)b; Engine* e = ENG(h); e->gen_option_lhood(); if (lhood_dev) *lhood_dev = e->lhood; })
}

int vd_encoder_rnn_state(vd_engine* h, int32_t level, const float** h_last, const float** c_last) {
  VD_TRY({
    Engine* e = ENG(h);
    VD_REQUIRE(e->have_fwd, VD_E_STATE, "vd_encoder_rnn_state before vd_encoder_forward");
    VD_REQUIRE(level == 0 || level == 1, VD_E_BADARG, "level must be 0 or 1");
    const bool has_layers = e->cfg.rnn_layers;            // the encoders that expose .rnnLayers (gen.lua:31)
    const vd::LstmRun& r = level == 0 ? e->ques1 : e->ques2;
    if (h_last) *h_last = has_layers ? r.h_last() : nullptr;
    if (c_last) *c_last = has_layers ? r.c_last() : nullptr;
  })
}
int vd_gen_decoder_step(vd_engine* h, int32_t rows, const int32_t* tokens_host, const float* const* h_prev,
                        const float* const* c_prev, const float** logp_dev, const float** h_out, const float** c_out) {
  VD_TRY({
    Engine* e = ENG(h);
    e->gen_decoder_step(rows, tokens_host, h_prev, c_prev);
    if (logp_dev) *logp_dev = e->gstep_logp;
    if (h_out) { h_out[0] = e->gstep1.h; h_out[1] = e->gstep2.h; }
    if (c_out) { c_out[0] = e->gstep1.c; c_out[1] = e->gstep2.c; }
  })
}

int vd_gen_beam_search(vd_engine* h, int32_t beam_size, int32_t beam_len, int32_t start_token, int32_t end_token,
                       int32_t* answer_host, int32_t* length_host, double* score_host) {
  VD_TRY({ ENG(h)->gen_beam_search(beam_size, 1, 0.f, beam_len, start_token, end_token, answer_host, length_host, score_host); })
}

int vd_gen_diverse_beam_search(vd_engine* h, int32_t beam_size, int32_t groups, float diversity, int32_t beam_len,
                               int32_t start_token, int32_t end_token, int32_t* answer_host, int32_t* length_host,
                               double* score_host) {
  VD_TRY({
    ENG(h)->gen_beam_search(beam_size, groups, diversity, beam_len, start_token, end_token, answer_host, length_host, score_host);
  })
}

static vd::NBestCfg nbest_cfg(float length_penalty, int32_t nbest, double* norm_host) {
  vd::NBestCfg c;
  c.alpha = length_penalty;
  c.nbest = nbest;
  c.norm_host = norm_host;
  return c;
}
int vd_gen_nbest_beam_search(vd_engine* h, int32_t beam_size, int32_t groups, float diversity, float length_penalty,
                             int32_t nbest, int32_t beam_len, int32_t start_token, int32_t end_token, int32_t* answer_host,
                             int32_t* length_host, double* score_host, double* norm_host) {
  VD_TRY({
    ENG(h)->gen_beam_search(beam_size, groups, diversity, beam_len, start_token, end_token, answer_host, length_host, score_host,
                            nbest_cfg(length_penalty, nbest, norm_host));
  })
}

int vd_gen_sample(vd_engine* h, int32_t beam_len, int32_t start_token, float temperature, uint64_t seed, int64_t row_offset,
                  int32_t* answer_host, float* logp_host) {
  VD_TRY({ ENG(h)->gen_sample(beam_len, start_token, temperature, seed, row_offset, answer_host, logp_host); })
}

int vd_gen_dialog_beam_search(vd_engine* h, const vd_batch* b, int32_t beam_size, int32_t beam_len, int32_t start_token,
                              int32_t end_token, int32_t hist_width, int32_t max_ans_len, int32_t* answer_host,
                              int32_t* length_host, double* score_host, int32_t* hist_host) {
  VD_TRY({ ENG(h)->gen_dialog_beam_search(b, beam_size, 1, 0.f, beam_len, start_token, end_token, hist_width, max_ans_len,
                                          answer_host, length_host, score_host, hist_host); })
}

int vd_gen_dialog_diverse_beam_search(vd_engine* h, const vd_batch* b, int32_t beam_size, int32_t groups, float diversity,
                                      int32_t beam_len, int32_t start_token, int32_t end_token, int32_t hist_width,
                                      int32_t max_ans_len, int32_t* answer_host, int32_t* length_host, double* score_host,
                                      int32_t* hist_host) {
  VD_TRY({ ENG(h)->gen_dialog_beam_search(b, beam_size, groups, diversity, beam_len, start_token, end_token, hist_width,
                                          max_ans_len, answer_host, length_host, score_host, hist_host); })
}

int vd_gen_dialog_nbest_beam_search(vd_engine* h, const vd_batch* b, int32_t beam_size, int32_t groups, float diversity,
                                    float length_penalty, int32_t nbest, int32_t beam_len, int32_t start_token,
                                    int32_t end_token, int32_t hist_width, int32_t max_ans_len, int32_t* answer_host,
                                    int32_t* length_host, double* score_host, double* norm_host, int32_t* hist_host) {
  VD_TRY({ ENG(h)->gen_dialog_beam_search(b, beam_size, groups, diversity, beam_len, start_token, end_token, hist_width,
                                          max_ans_len, answer_host, length_host, score_host, hist_host,
                                          nbest_cfg(length_penalty, nbest, norm_host)); })
}

int vd_gen_dialog_sample(vd_engine* h, const vd_batch* b, int32_t beam_len, int32_t start_token, int32_t end_token,
                         float temperature, uint64_t seed, int64_t row_offset, int32_t hist_width, int32_t max_ans_len,
                         int32_t* answer_host, float* logp_host, int32_t* hist_host) {
  VD_TRY({ ENG(h)->gen_dialog_sample(b, beam_len, start_token, end_token, temperature, seed, row_offset, hist_width, max_ans_len,
                                     answer_host, logp_host, hist_host); })
}

static vd::TruncCfg trunc_cfg(int32_t top_k, float top_p) {
  vd::TruncCfg t;
  t.top_k = top_k;
  t.top_p = top_p;
  return t;
}
int vd_gen_truncated_sample(vd_engine* h, int32_t beam_len, int32_t start_token, float temperature, uint64_t seed,
                            int64_t row_offset, int32_t top_k, float top_p, int32_t* answer_host, float* logp_host) {
  VD_TRY({ ENG(h)->gen_sample(beam_len, start_token, temperature, seed, row_offset, answer_host, logp_host, trunc_cfg(top_k, top_p)); })
}

int vd_gen_dialog_truncated_sample(vd_engine* h, const vd_batch* b, int32_t beam_len, int32_t start_token, int32_t end_token,
                                   float temperature, uint64_t seed, int64_t row_offset, int32_t top_k, float top_p,
                                   int32_t hist_width, int32_t max_ans_len, int32_t* answer_host, float* logp_host,
                                   int32_t* hist_host) {
  VD_TRY({ ENG(h)->gen_dialog_sample(b, beam_len, start_token, end_token, temperature, seed, row_offset, hist_width, max_ans_len,
                                     answer_host, logp_host, hist_host, trunc_cfg(top_k, top_p)); })
}

int vd_answer_pool_encode(vd_engine* h, const int32_t* tokens_host, int64_t m, int32_t width) {
  VD_TRY({ ENG(h)->answer_pool_encode(tokens_host, m, width); })
}
int vd_answer_pool(vd_engine* h, const float** emb_dev, int64_t* m) {
  VD_TRY({
    Engine* e = ENG(h);
    e->check_pool(1);
    if (emb_dev) *emb_dev = (const float*)e->pool_emb.p;
    if (m) *m = e->pool_m;
  })
}
int vd_answer_pool_retrieve(vd_engine* h, const vd_batch* b, int32_t k, int32_t* index_host, float* score_host) {
  VD_TRY({ ENG(h)->answer_pool_retrieve(b, k, index_host, score_host); })
}
int vd_answer_pool_dialog(vd_engine* h, const vd_batch* b, int32_t k, int32_t hist_width, int32_t max_ans_len, int32_t* index_host,
                          float* score_host, int32_t* hist_host) {
  VD_TRY({ ENG(h)->answer_pool_dialog(b, k, hist_width, max_ans_len, index_host, score_host, hist_host); })
}

int vd_dialog_begin(vd_engine* h, const vd_batch* b, int32_t hist_width, int32_t max_ans_len) {
  VD_TRY({ ENG(h)->dialog_begin(b, hist_width, max_ans_len); })
}
int vd_dialog_ask_beam(vd_engine* h, const int32_t* ques, int32_t Tq, int32_t beam_size, int32_t beam_len, int32_t start_token,
                       int32_t end_token, int32_t* answer, int32_t* length, double* score) {
  VD_TRY({
    Engine* e = ENG(h);
    const std::vector<int32_t> s = e->dialog_all_slots();
    e->dialog_ask_beam(s.data(), (int64_t)s.size(), ques, Tq, beam_size, 1, 0.f, beam_len, start_token, end_token, answer, length,
                       score);
  })
}
int vd_dialog_ask_sample(vd_engine* h, const int32_t* ques, int32_t Tq, int32_t beam_len, int32_t start_token, int32_t end_token,
                         float temperature, uint64_t seed, int64_t row_offset, int32_t* answer, float* logp) {
  VD_TRY({
    Engine* e = ENG(h);
    const std::vector<int32_t> s = e->dialog_all_slots();
    e->dialog_ask_sample(s.data(), (int64_t)s.size(), ques, Tq, beam_len, start_token, end_token, temperature, seed, row_offset,
                         answer, logp);
  })
}
int vd_dialog_ask_pool(vd_engine* h, const int32_t* ques, int32_t Tq, int32_t k, int32_t* index, float* score) {
  VD_TRY({
    Engine* e = ENG(h);
    const std::vector<int32_t> s = e->dialog_all_slots();
    e->dialog_ask_pool(s.data(), (int64_t)s.size(), ques, Tq, k, index, score);
  })
}
int vd_dialog_round(vd_engine* h, int32_t* round, int32_t* B) {
  VD_TRY({
    Engine* e = ENG(h);
    const int r = e->dialog_lockstep_round();
    if (round) *round = r;
    if (B) *B = e->dses.C;
  })
}
int vd_dialog_history(vd_engine* h, int32_t* hist_host) {
  VD_TRY({
    Engine* e = ENG(h);
    e->dialog_lockstep_round();
    NOTNULL(hist_host);
    VD_CUDA_CHECK(cudaSetDevice(e->cfg.gpuid));
    const size_t n = (size_t)e->dses.C * e->cfg.R * e->dses.W;
    if (n) VD_CUDA_CHECK(cudaMemcpyAsync(hist_host, e->dses.hist.p, n * sizeof(int32_t), cudaMemcpyDeviceToHost, e->main_stream));
    VD_CUDA_CHECK(cudaStreamSynchronize(e->main_stream));
  })
}
int vd_dialog_encoding(vd_engine* h, const float** encOut_dev) {
  VD_TRY({
    Engine* e = ENG(h);
    VD_REQUIRE(e->dses.open && e->dses.encOut, VD_E_STATE, "no dialog session, or no round asked yet");
    NOTNULL(encOut_dev);
    *encOut_dev = e->dses.encOut;
  })
}
int vd_dialog_rnn_state(vd_engine* h, int32_t level, const float** h_last, const float** c_last) {
  VD_TRY({
    Engine* e = ENG(h);
    VD_REQUIRE(e->dses.open && e->dses.encOut, VD_E_STATE, "no dialog session, or no round asked yet");
    VD_REQUIRE(level == 0 || level == 1, VD_E_BADARG, "level must be 0 or 1");
    const bool has_layers = e->cfg.rnn_layers;
    if (h_last) *h_last = has_layers ? (const float*)e->dses.rnn[2 * level].p : nullptr;
    if (c_last) *c_last = has_layers ? (const float*)e->dses.rnn[2 * level + 1].p : nullptr;
  })
}
int vd_dialog_end(vd_engine* h) { VD_TRY({ ENG(h)->dialog_end(); }) }

int vd_dialog_open(vd_engine* h, int32_t capacity, int32_t Tq, int32_t hist_width, int32_t max_ans_len) {
  VD_TRY({ ENG(h)->dialog_open(capacity, Tq, hist_width, max_ans_len); })
}
int vd_dialog_join(vd_engine* h, const vd_batch* b, const int64_t* draw_base, int32_t* slots) {
  VD_TRY({ ENG(h)->dialog_join(b, draw_base, slots); })
}
int vd_dialog_join_rounds(vd_engine* h, const vd_batch* b, const int32_t* rounds, const int32_t* answers, int32_t Ta,
                          const int64_t* draw_base, const int32_t* slots) {
  VD_TRY({ ENG(h)->dialog_join_rounds(b, rounds, answers, Ta, draw_base, slots); })
}
int vd_dialog_leave(vd_engine* h, const int32_t* slots, int32_t n) { VD_TRY({ ENG(h)->dialog_leave(slots, n); }) }
int vd_dialog_ask_beam_slots(vd_engine* h, const int32_t* slots, int32_t n, const int32_t* ques, int32_t Tq, int32_t beam_size,
                             int32_t beam_len, int32_t start_token, int32_t end_token, int32_t* answer, int32_t* length,
                             double* score) {
  VD_TRY({ ENG(h)->dialog_ask_beam(slots, n, ques, Tq, beam_size, 1, 0.f, beam_len, start_token, end_token, answer, length, score); })
}
int vd_dialog_ask_diverse_slots(vd_engine* h, const int32_t* slots, int32_t n, const int32_t* ques, int32_t Tq, int32_t beam_size,
                                int32_t groups, float diversity, int32_t beam_len, int32_t start_token, int32_t end_token,
                                int32_t* answer, int32_t* length, double* score) {
  VD_TRY({
    ENG(h)->dialog_ask_beam(slots, n, ques, Tq, beam_size, groups, diversity, beam_len, start_token, end_token, answer, length,
                            score);
  })
}
int vd_dialog_ask_nbest_slots(vd_engine* h, const int32_t* slots, int32_t n, const int32_t* ques, int32_t Tq, int32_t beam_size,
                              int32_t groups, float diversity, float length_penalty, int32_t nbest, int32_t beam_len,
                              int32_t start_token, int32_t end_token, int32_t* answer, int32_t* length, double* score,
                              double* norm) {
  VD_TRY({
    ENG(h)->dialog_ask_beam(slots, n, ques, Tq, beam_size, groups, diversity, beam_len, start_token, end_token, answer, length,
                            score, nbest_cfg(length_penalty, nbest, norm));
  })
}
int vd_dialog_ask_sample_slots(vd_engine* h, const int32_t* slots, int32_t n, const int32_t* ques, int32_t Tq, int32_t beam_len,
                               int32_t start_token, int32_t end_token, float temperature, uint64_t seed, int64_t row_offset,
                               int32_t* answer, float* logp) {
  VD_TRY({
    ENG(h)->dialog_ask_sample(slots, n, ques, Tq, beam_len, start_token, end_token, temperature, seed, row_offset, answer, logp);
  })
}
int vd_dialog_ask_truncated_slots(vd_engine* h, const int32_t* slots, int32_t n, const int32_t* ques, int32_t Tq,
                                  int32_t beam_len, int32_t start_token, int32_t end_token, float temperature, uint64_t seed,
                                  int64_t row_offset, int32_t top_k, float top_p, int32_t* answer, float* logp) {
  VD_TRY({
    ENG(h)->dialog_ask_sample(slots, n, ques, Tq, beam_len, start_token, end_token, temperature, seed, row_offset, answer, logp,
                              trunc_cfg(top_k, top_p));
  })
}
int vd_dialog_ask_pool_slots(vd_engine* h, const int32_t* slots, int32_t n, const int32_t* ques, int32_t Tq, int32_t k,
                             int32_t* index, float* score) {
  VD_TRY({ ENG(h)->dialog_ask_pool(slots, n, ques, Tq, k, index, score); })
}
int vd_dialog_slots(vd_engine* h, int32_t* rounds, int32_t* capacity) {
  VD_TRY({
    Engine* e = ENG(h);
    VD_REQUIRE(e->dses.open, VD_E_STATE, "no dialog session");
    if (rounds) std::copy(e->dses.round.begin(), e->dses.round.end(), rounds);
    if (capacity) *capacity = e->dses.C;
  })
}
int vd_dialog_slot_history(vd_engine* h, const int32_t* slots, int32_t n, int32_t* hist_host) {
  VD_TRY({
    Engine* e = ENG(h);
    VD_REQUIRE(e->dses.open, VD_E_STATE, "no dialog session");
    e->dialog_check_slots(slots, n);
    NOTNULL(hist_host);
    VD_CUDA_CHECK(cudaSetDevice(e->cfg.gpuid));
    const size_t rw = (size_t)e->cfg.R * e->dses.W;
    if (rw)
      for (int32_t i = 0; i < n; ++i)
        VD_CUDA_CHECK(cudaMemcpyAsync(hist_host + i * rw, (const int32_t*)e->dses.hist.p + slots[i] * rw, rw * sizeof(int32_t),
                                      cudaMemcpyDeviceToHost, e->main_stream));
    VD_CUDA_CHECK(cudaStreamSynchronize(e->main_stream));
  })
}

int vd_clamp_adam_step(vd_engine* h, float lr) { VD_TRY({ ENG(h)->clamp_adam_step(lr); }) }

int vd_comm_unique_id(void* id_out) { VD_TRY({ NOTNULL(id_out); vd::comm_unique_id(id_out); }) }
int vd_comm_init(vd_engine* h, const void* id, int32_t rank, int32_t world) {
  VD_TRY({
    VD_REQUIRE(id != nullptr || world == 1, VD_E_BADARG, "id is null");
    VD_REQUIRE(world == 1 || !ENG(h)->cx.deterministic, VD_E_STATE, "deterministic mode runs on one GPU (world 1)");
    vd::comm_init(ENG(h), id, rank, world);
  })
}
int vd_comm_allreduce_grads(vd_engine* h) { VD_TRY({ ENG(h)->allreduce_grads(); }) }

int vd_memcpy_d2h(vd_engine* h, void* dst, const void* src, size_t bytes) {
  VD_TRY({
    Engine* e = ENG(h);
    VD_REQUIRE(dst && src, VD_E_BADARG, "null pointer");
    VD_CUDA_CHECK(cudaSetDevice(e->cfg.gpuid));
    VD_CUDA_CHECK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, e->cx.stream));
    VD_CUDA_CHECK(cudaStreamSynchronize(e->cx.stream));
  })
}
int vd_memcpy_h2d(vd_engine* h, void* dst, const void* src, size_t bytes) {
  VD_TRY({
    Engine* e = ENG(h);
    VD_REQUIRE(dst && src, VD_E_BADARG, "null pointer");
    VD_CUDA_CHECK(cudaSetDevice(e->cfg.gpuid));
    VD_CUDA_CHECK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, e->cx.stream));
    VD_CUDA_CHECK(cudaStreamSynchronize(e->cx.stream));
  })
}
int vd_host_alloc(void** ptr, size_t bytes) {
  VD_TRY({ NOTNULL(ptr); *ptr = nullptr; VD_CUDA_CHECK(cudaHostAlloc(ptr, bytes ? bytes : 1, cudaHostAllocDefault)); })
}
int vd_host_free(void* ptr) { VD_TRY({ if (ptr) VD_CUDA_CHECK(cudaFreeHost(ptr)); }) }
int vd_device_alloc(vd_engine* h, void** ptr, size_t bytes) {
  VD_TRY({
    Engine* e = ENG(h);
    NOTNULL(ptr);
    *ptr = nullptr;
    VD_CUDA_CHECK(cudaSetDevice(e->cfg.gpuid));
    VD_CUDA_CHECK(cudaMalloc(ptr, bytes ? bytes : 1));
  })
}
int vd_device_free(vd_engine* h, void* ptr) {
  VD_TRY({ Engine* e = ENG(h); VD_CUDA_CHECK(cudaSetDevice(e->cfg.gpuid)); if (ptr) VD_CUDA_CHECK(cudaFree(ptr)); })
}
int vd_synchronize(vd_engine* h) {
  VD_TRY({
    Engine* e = ENG(h);
    e->join_options_backward();
    VD_CUDA_CHECK(cudaStreamSynchronize(e->cx.stream));
    if (e->opt_fwd_pending) VD_CUDA_CHECK(cudaStreamSynchronize(e->opt_stream));
  })
}
int vd_stream(vd_engine* h, void** s) { VD_TRY({ NOTNULL(s); *s = (void*)ENG(h)->cx.stream; }) }
int vd_timer_start(vd_engine* h) { VD_TRY({ Engine* e = ENG(h); VD_CUDA_CHECK(cudaEventRecord(e->t0, e->cx.stream)); }) }
int vd_timer_stop(vd_engine* h, float* ms) {
  VD_TRY({
    Engine* e = ENG(h);
    NOTNULL(ms);
    VD_CUDA_CHECK(cudaEventRecord(e->t1, e->cx.stream));
    VD_CUDA_CHECK(cudaEventSynchronize(e->t1));
    VD_CUDA_CHECK(cudaEventElapsedTime(ms, e->t0, e->t1));
  })
}
int vd_profile_enable(vd_engine* h, int32_t on) { VD_TRY({ ENG(h)->cx.profiling = on; }) }
int vd_profile_reset(vd_engine* h) {
  VD_TRY({ Engine* e = ENG(h); e->cx.collect(); e->cx.stats.clear(); e->cx.launches = 0; })
}
int vd_launch_count(vd_engine* h, int64_t* n) { VD_TRY({ NOTNULL(n); *n = ENG(h)->cx.launches; }) }
int vd_kernel_stats(vd_engine* h, const char* name, int64_t* launches, double* total_ms, double* total_flops,
                    double* total_bytes) {
  VD_TRY({
    Engine* e = ENG(h);
    VD_REQUIRE(name != nullptr, VD_E_BADARG, "name is null");
    e->cx.collect();
    auto it = e->cx.stats.find(name);
    vd::KStat z;
    const vd::KStat& s = it == e->cx.stats.end() ? z : it->second;
    if (launches) *launches = s.launches;
    if (total_ms) *total_ms = s.ms;
    if (total_flops) *total_flops = s.flops;
    if (total_bytes) *total_bytes = s.bytes;
  })
}
int vd_gemm_tn(vd_engine* h, int32_t M, int32_t N, int32_t K, const float* A, int64_t lda, const float* B, int64_t ldb,
               float* C, int64_t ldc, float beta, const float* bias, int32_t act) {
  VD_TRY({
    Engine* e = ENG(h);
    VD_REQUIRE(A && B && C, VD_E_BADARG, "null operand");
    VD_CUDA_CHECK(cudaSetDevice(e->cfg.gpuid));
    e->gemm_tn(M, N, K, A, lda, nullptr, B, ldb, C, ldc, beta, bias, act);
  })
}
int vd_gemm_atb(vd_engine* h, int32_t M, int32_t N, int64_t K, const float* A, int64_t lda, const float* B, int64_t ldb,
                float* C, int64_t ldc) {
  VD_TRY({
    Engine* e = ENG(h);
    VD_REQUIRE(A && B && C, VD_E_BADARG, "null operand");
    VD_CUDA_CHECK(cudaSetDevice(e->cfg.gpuid));
    e->gemm_atb(M, N, K, A, lda, nullptr, B, ldb, C, ldc);
  })
}
int vd_gemm_atb16(vd_engine* h, int32_t M, int32_t N, int64_t K, const float* A, int64_t lda, const float* B, int64_t ldb,
                  float* C, int64_t ldc, float inv_scale) {
  VD_TRY({
    Engine* e = ENG(h);
    VD_REQUIRE(A && B && C, VD_E_BADARG, "null operand");
    VD_CUDA_CHECK(cudaSetDevice(e->cfg.gpuid));
    __half* A16 = nullptr; __half* B16 = nullptr; float* sc = nullptr;
    VD_CUDA_CHECK(cudaMalloc((void**)&A16, (size_t)K * M * sizeof(__half)));
    VD_CUDA_CHECK(cudaMalloc((void**)&B16, (size_t)K * N * sizeof(__half)));
    VD_CUDA_CHECK(cudaMalloc((void**)&sc, sizeof(float)));
    VD_CUDA_CHECK(cudaMemcpyAsync(sc, &inv_scale, sizeof(float), cudaMemcpyHostToDevice, e->cx.stream));
    cvt_f32_to_f16(e->cx, A16, M, A, lda, K, M);
    cvt_f32_to_f16(e->cx, B16, N, B, ldb, K, N);
    gemm_atb16(e->cx, M, N, K, A16, M, B16, N, C, ldc, sc);
    VD_CUDA_CHECK(cudaStreamSynchronize(e->cx.stream));
    cudaFree(A16); cudaFree(B16); cudaFree(sc);
  })
}
int vd_lstm_step_fwd(vd_engine* h, int64_t R, int32_t H, const float* h_prev, const float* WhT, int64_t ldw, const float* bias,
                     float* gates, int32_t has_xproj, const float* ptable, int64_t ptable_rows, const int32_t* tok,
                     const float* c_prev, float* c_out, float* h_out, const int32_t* mask_ids, int32_t* path) {
  VD_TRY({
    Engine* e = ENG(h);
    NOTNULL(path);
    VD_REQUIRE(R >= 1 && H > 0 && H % 4 == 0 && WhT && bias && gates && c_out && h_out, VD_E_BADARG, "vd_lstm_step_fwd: arguments");
    VD_REQUIRE((has_xproj != 0) != (ptable != nullptr) && (!ptable || (tok && ptable_rows > 0)), VD_E_BADARG,
               "vd_lstm_step_fwd: the x side is either a dense projection (has_xproj) or a table gather (ptable + tok)");
    VD_CUDA_CHECK(cudaSetDevice(e->cfg.gpuid));
    *path = 0;
    // routed as a step of a run without initial state over a gathered (ptable) or dense x side; the backward half of the
    // route is not used here
    const vd::LstmRoute rt = e->route_lstm(R, H, ptable != nullptr, false, WhT, ldw, nullptr);
    VD_REQUIRE(rt.fwd != vd::LstmPath::Opt16, VD_E_BADARG, "vd_lstm_step_fwd: the fp16 option-LSTM steps (lstm16.cu) have no test hook");
    // the CUDA-core route projects gathered inputs inside its x-projection GEMM, never through a table
    VD_REQUIRE(rt.fwd == vd::LstmPath::Tc || !ptable, VD_E_BADARG, "vd_lstm_step_fwd: a table gather runs on the tensor-core route only");
    vd::LstmFwdStep s;
    s.R = R; s.H = H; s.WhT = WhT; s.ldw = ldw; s.bias = bias;
    s.h_prev = h_prev; s.c_prev = c_prev; s.gates = gates; s.mask = mask_ids; s.c_out = c_out; s.h_out = h_out;
    float* pt = nullptr;
    if (rt.fwd == vd::LstmPath::Tc) {
      // the tensor-core steps read the bias from the x-projection (table or dense), where the engine folds it in
      const int64_t n = (ptable ? ptable_rows : R) * 4 * H;
      VD_CUDA_CHECK(cudaMalloc((void**)&pt, (size_t)n * sizeof(float)));
      vd::repeat_rows(e->cx, pt, bias, 1, (int)(n / (4 * H)), 4 * H);           // the bias in every row
      vd::add_inplace(e->cx, ptable ? pt : gates, ptable ? ptable : pt, n);
      if (ptable) { s.ptable = pt; s.tok = tok; }
    }
    if (rt.fwd == vd::LstmPath::Tc) *path = e->lstm_tc_fwd_step(s); else e->lstm_simt_fwd_step(s);
    VD_CUDA_CHECK(cudaStreamSynchronize(e->cx.stream));
    if (pt) cudaFree(pt);
  })
}

int vd_lstm_step_bwd(vd_engine* h, int64_t R, int32_t H, const float* da_next, const float* Wh, const float* gates,
                     const float* c_prev, const float* c_cur, const float* dh_ext, float* dc_carry, const int32_t* mask_ids,
                     float* da, int32_t* path) {
  VD_TRY({
    Engine* e = ENG(h);
    NOTNULL(path);
    VD_REQUIRE(R >= 1 && H > 0 && Wh && gates && c_cur && dc_carry && da, VD_E_BADARG, "vd_lstm_step_bwd: arguments");
    VD_CUDA_CHECK(cudaSetDevice(e->cfg.gpuid));
    *path = 0;
    // routed as a step of a run with a dense x side (the forward half of the route is not used here)
    const vd::LstmRoute rt = e->route_lstm(R, H, false, false, nullptr, H, Wh);
    vd::LstmBwdStep s;
    s.R = R; s.H = H; s.Wh = Wh; s.da_next = da_next; s.dh_ext = dh_ext;
    s.gates = gates; s.c_prev = c_prev; s.c_cur = c_cur; s.mask = mask_ids; s.dc_carry = dc_carry; s.da = da;
    if (rt.bwd == vd::LstmPath::Simt && da_next) VD_CUDA_CHECK(cudaMalloc((void**)&s.dh_rec, (size_t)R * H * sizeof(float)));
    if (rt.bwd == vd::LstmPath::Tc) *path = e->lstm_tc_bwd_step(s); else e->lstm_simt_bwd_step(s);
    VD_CUDA_CHECK(cudaStreamSynchronize(e->cx.stream));
    if (s.dh_rec) cudaFree(s.dh_rec);
  })
}
int vd_lstm16_step_fwd(vd_engine* h, int64_t R, int32_t H, const void* h_prev16, const void* Wh16, const void* ptable16,
                       const int32_t* tok, const float* bias, const float* c_prev, const int32_t* mask_ids, void* gates16,
                       float* c_out, void* h16_out, float* h32_out) {
  VD_TRY({
    Engine* e = ENG(h);
    VD_REQUIRE(h_prev16 && Wh16 && ptable16 && tok && bias && c_out && h16_out, VD_E_BADARG, "vd_lstm16_step_fwd: arguments");
    VD_REQUIRE(vd::lstm16_shape_ok(R, H), VD_E_BADARG, "vd_lstm16_step_fwd: shape");
    VD_CUDA_CHECK(cudaSetDevice(e->cfg.gpuid));
    vd::lstm16_step_fwd(e->cx, R, H, (const __half*)h_prev16, (const __half*)Wh16, (const __half*)ptable16, tok, bias, c_prev,
                        mask_ids, (__half*)gates16, c_out, (__half*)h16_out, h32_out);
    VD_CUDA_CHECK(cudaStreamSynchronize(e->cx.stream));
  })
}
int vd_lstm16_step_bwd(vd_engine* h, int64_t R, int32_t H, const void* da_next16, const void* Whb16, const void* gates16,
                       const float* c_prev, const float* c_cur, float* dc_carry, const int32_t* mask_ids, void* da16) {
  VD_TRY({
    Engine* e = ENG(h);
    VD_REQUIRE(da_next16 && Whb16 && gates16 && c_cur && dc_carry && da16, VD_E_BADARG, "vd_lstm16_step_bwd: arguments");
    VD_REQUIRE(vd::lstm16_shape_ok(R, H), VD_E_BADARG, "vd_lstm16_step_bwd: shape");
    VD_CUDA_CHECK(cudaSetDevice(e->cfg.gpuid));
    vd::lstm16_step_bwd(e->cx, R, H, (const __half*)da_next16, (const __half*)Whb16, (const __half*)gates16, c_prev, c_cur,
                        dc_carry, mask_ids, (__half*)da16);
    VD_CUDA_CHECK(cudaStreamSynchronize(e->cx.stream));
  })
}

int vd_test_kernel(vd_engine* h, const char* name, void* const* ptrs, int32_t n_ptrs, const int64_t* ints, int32_t n_ints,
                   const double* reals, int32_t n_reals) {
  VD_TRY({
    Engine* e = ENG(h);
    VD_CUDA_CHECK(cudaSetDevice(e->cfg.gpuid));
    vd::test_kernel(e, name, ptrs, n_ptrs, ints, n_ints, reals, n_reals);
  })
}

int vd_profiler_range(vd_engine* h, int32_t start) {
  VD_TRY({
    Engine* e = ENG(h);
    VD_CUDA_CHECK(cudaStreamSynchronize(e->cx.stream));
    if (start) VD_CUDA_CHECK(cudaProfilerStart()); else VD_CUDA_CHECK(cudaProfilerStop());
  })
}
int vd_flush_l2(vd_engine* h) {
  VD_TRY({
    Engine* e = ENG(h);
    if (!e->flush_buf) {
      e->flush_n = (int64_t)(192u << 20) / 4;      // 192 MiB > 50 MB L2
      VD_CUDA_CHECK(cudaMalloc((void**)&e->flush_buf, (size_t)e->flush_n * 4));
    }
    vd::fill_l2_flush(e->cx, e->flush_buf, e->flush_n);
  })
}

// ---- dataloader: resident corpus (corpus.cu) ----
struct vd_corpus { vd::Corpus* c; };
#define CORP(h) ((h) ? (h)->c : (throw vd::CudaError(VD_E_BADARG, "corpus handle is null"), (vd::Corpus*)nullptr))

int vd_corpus_create(vd_engine* h, const vd_corpus_desc* d, vd_corpus** out) {
  VD_TRY({
    NOTNULL(out);
    Engine* e = ENG(h);
    VD_CUDA_CHECK(cudaSetDevice(e->cfg.gpuid));
    vd::Corpus* c = vd::corpus_create(e, d);
    *out = new vd_corpus{c};
  })
}
int vd_corpus_destroy(vd_corpus* h) {
  VD_TRY({
    if (h) { vd::corpus_destroy(h->c); delete h; }
  })
}
int vd_corpus_get_batch(vd_corpus* h, const int64_t* inds, int32_t n, int32_t decoder_gen, vd_batch* out) {
  VD_TRY({ vd::corpus_get_batch(CORP(h), inds, n, decoder_gen, out); })
}
int vd_corpus_read(vd_corpus* h, const char* name, void* host_dst, int64_t* elems) {
  VD_TRY({ vd::corpus_read(CORP(h), name, host_dst, elems); })
}
int vd_corpus_region_counts(vd_corpus* h, const int32_t* counts_host, int64_t numImages) {
  VD_TRY({ vd::corpus_region_counts(CORP(h), counts_host, numImages); })
}
int vd_corpus_batch_bytes(vd_corpus* h, int64_t* bytes, int32_t* launches) {
  VD_TRY({ vd::corpus_batch_bytes(CORP(h), bytes, launches); })
}

}  // extern "C"
