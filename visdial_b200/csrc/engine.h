// Engine: owns parameters, activations and the per-batch forward/backward orchestration that
// replaces Model:forwardBackward / Model:retrieveBatch (/root/reference/model.lua:249-430).
#pragma once
#include <functional>
#include <string>
#include <vector>
#include "../../include/visdial_b200.h"
#include "kernels.cuh"

namespace vd {

enum EncKind { ENC_LF_QUES = 0, ENC_LF_QIH = 1, ENC_HREA = 2, ENC_MN_ATT = 3, ENC_LF_QI = 4, ENC_LF_QH = 5, ENC_HRE_QH = 6, ENC_HRE_QIH = 7,
               ENC_MN_QH = 8, ENC_MN_QIH = 9, ENC_LF_ATT = 10 };
enum DecKind { DEC_DISC = 0, DEC_GEN = 1 };

struct Cfg {
  std::string encoder, decoder;
  int enc = 0, dec = 0;
  int V = 0, E = 300, H = 512, L = 2, F = 4096, S = 14, IE = 300, Cm = 512, hops = 1, R = 10, K = 100;
  float dropout = 0.5f;
  int gpuid = 0;
  bool useIm = false, useHist = false, att = false;
  // structure of the encoder graph, derived from its name (encoders/*.lua): late fusion / hierarchical / memory network
  bool fam_lf = false, fam_hre = false, fam_mn = false;
  bool hre_att = false;     // hrea: attention over the history rounds before the dialog LSTM
  bool san = false;         // SAN spatial attention over pool5 (mn-att-*, lf-att-*)
  bool img_in_q = false;    // Linear(fc7) -> MaskTime -> concatenated to the question LSTM input (hre-ques-im-hist, hrea-*)
  bool img_drop = false;    // ... behind Dropout(0.5) (hrea only; commented out in hre-ques-im-hist.lua:45)
  bool mn_qi = false;       // mn-ques-im-hist: tanh(Linear([q | fc7])) replaces q in the memory attention
  bool embdrop = false;     // Dropout(0.5) on the word embeddings (mn-*, lf-att-*)
  bool rnn_layers = false;  // exposes .rnnLayers to the gen decoder's forwardConnect (lf-*, hre*)
};
Cfg parse_cfg(const vd_params* p);

struct Seg {
  std::string name;
  int64_t off = 0, rows = 0, cols = 0;
  int init = 0;
  int64_t fan_in = 0;
};
struct Layout {
  std::vector<Seg> segs;
  int64_t total = 0;
  int find(const std::string& name) const;
};
Layout build_layout(const Cfg& c);

// grow-only bump allocator for activations (reset at every new forward)
struct Arena {
  struct Chunk { char* p; size_t cap; size_t used; };
  std::vector<Chunk> chunks;
  size_t cur = 0;
  void* alloc(size_t bytes);
  template <typename T> T* get(int64_t n) { return reinterpret_cast<T*>(alloc((size_t)n * sizeof(T))); }
  void reset();
  void release();
  // a loop that allocates the same buffers every iteration rewinds to a mark taken before it, so it reuses them instead of
  // growing the arena (stream order keeps the previous iteration's readers ahead of the new writers)
  struct Mark { size_t chunk, used; };
  Mark mark() const { return {cur, cur < chunks.size() ? chunks[cur].used : 0}; }
  void rewind(const Mark& m);
};

// The kernels an nn.SeqLSTM run executes on.  Simt: a GEMM and a pointwise kernel per step on the CUDA cores.  Tc: fused
// wgmma step kernels (lstm_step_fwd_tc / _bwd_tc).  Opt16: VD_MATH_F16 many-row LSTM over embedding-gathered tokens with
// fp16 h / gates / da / table (lstm16.cu).  Pair16: VD_MATH_F16 persistent kernel of two stacked layers (enc_lstm.cu).
enum class LstmPath { Simt, Tc, Opt16, Pair16 };
// Decided once per run by Engine::route_lstm / route_lstm_pair, when the run's forward begins
struct LstmRoute {
  LstmPath fwd = LstmPath::Simt, bwd = LstmPath::Simt;   // the forward and backward step kernels have different predicates
  bool table_grad = false;           // embedding-gathered input: the x-side gradients contract the (V+1, 4H) projected table
  bool wave_fwd = false, wave_bwd = false;   // stacked pair: the two layers run one step apart on three streams
};

// one nn.SeqLSTM execution (forward state kept for BPTT)
struct LstmRun {
  int T = 0; int64_t R = 0; int D = 0, H = 0;
  int wseg = -1;
  const float* x = nullptr;          // dense (T*R, D) or null when rows are gathered from the embedding
  const int32_t* gather = nullptr;   // time-major ids (T*R) for the gather
  const int32_t* mask = nullptr;     // time-major ids (T*R) for maskzero
  const float* h0 = nullptr; const float* c0 = nullptr;
  float* h = nullptr; float* c = nullptr; float* gates = nullptr;
  bool saved = false;
  float* demb_out = nullptr;         // projected-space embedding gradient goes here (overwritten) instead of dW(wordEmbed) +=
  LstmRoute route;
  const float* ptable = nullptr;     // Tc, gathered input: (V+1, 4H) projection table (+ bias)
  // backward run state (lstm_backward_begin / _step / _end)
  float* da = nullptr; float* dc_carry = nullptr; float* dh_rec = nullptr;
  const float* bw_dh_all = nullptr; const float* bw_dh_last = nullptr;
  // fp16 state of Opt16 (`h` and `gates` stay null) and Pair16
  __half *h16 = nullptr, *gates16 = nullptr, *da16 = nullptr, *P16 = nullptr, *Wh16 = nullptr, *Whb16 = nullptr;
  const __half* x16 = nullptr;       // Pair16 layer 2: fp16 copy of x (the h1 sequence)
  float* h32_last = nullptr;         // Opt16: fp32 copy of the last step's h (what the fp32 consumers of the run read)
  float* scale2 = nullptr;           // Opt16: device {s, 1/s}, power-of-two scale of the BPTT (chosen from max|dL/dh_T|)
  const float* h_last() const { return route.fwd == LstmPath::Opt16 ? h32_last : h + (int64_t)(saved ? T - 1 : (T - 1) & 1) * R * H; }
  const float* c_last() const { return c + (int64_t)(saved ? T - 1 : (T - 1) & 1) * R * H; }
};

// Operands of one step on the fp32 routes.  Forward: h_prev null = first step without initial state, c_prev null = zero;
// gates holds the x-projection on entry (null with a table x side when the run keeps no gates) and the activated gates on
// exit; bias is read by Simt only (the Tc kernels take it from the x-projection).  WhT = [4H, ldw] h columns of the
// transposed shadow.  Backward: Wh = [H, 4H] h rows of the weight; da_next null at the last step, where dh_last takes the
// recurrent slot; dc_carry in: dc from step t+1, out: dc for step t-1; dh_rec: Simt scratch (R, H).
struct LstmFwdStep {
  int64_t R = 0, ldw = 0; int H = 0;
  const float *WhT = nullptr, *bias = nullptr, *h_prev = nullptr, *c_prev = nullptr, *ptable = nullptr;
  const int32_t *tok = nullptr, *mask = nullptr;
  float *gates = nullptr, *c_out = nullptr, *h_out = nullptr;
};
struct LstmBwdStep {
  int64_t R = 0; int H = 0;
  const float *Wh = nullptr, *da_next = nullptr, *dh_last = nullptr, *dh_ext = nullptr, *gates = nullptr, *c_prev = nullptr,
              *c_cur = nullptr;
  const int32_t* mask = nullptr;
  float *dc_carry = nullptr, *da = nullptr, *dh_rec = nullptr;
};

struct DevBatch {
  int B = 0, Tq = 0, Th = 0, Ta = 0, To = 0; int64_t N = 0;
  const int32_t* ques = nullptr; const int32_t* hist = nullptr; const float* img = nullptr;
  const int32_t* options = nullptr; const int32_t* answer_ind = nullptr;
  const int32_t* answer_in = nullptr; const int32_t* answer_out = nullptr;
  const int32_t* option_in = nullptr; const int32_t* option_out = nullptr;
};

struct GrowBuf {
  void* p = nullptr; size_t cap = 0;
  void* ensure(size_t bytes);
  void release();
};

struct Engine {
  Cfg cfg;
  Layout lay;
  LaunchCtx cx;
  int64_t nparams = 0;
  float *W = nullptr, *dW = nullptr, *m = nullptr, *v = nullptr, *Wt = nullptr;
  int64_t adam_t = 0;
  int64_t* segtab_dev = nullptr; int nseg2d = 0; int64_t max2d = 0;
  int training = 1;
  uint64_t drop_seed = 1234, drop_iter = 0;
  int math_mode = VD_MATH_TF32;
  bool tcmode() const { return math_mode != VD_MATH_FP32; }   // TF32 and F16 both run the dense contractions on wgmma
  Arena arena;
  GrowBuf stage[9];
  // The image features are 80 % of a host batch (12.8 MB of pool5 at B = 32) and are not needed until the attention stage:
  // they are copied on their own stream into one of two staging buffers while the LSTM chains already run, and the
  // consuming stream waits for the copy at the first use (wait_img).  ev_img_free[k] = last reader of buffer k done.
  GrowBuf stage_img[2];
  cudaStream_t copy_stream = nullptr;
  cudaEvent_t ev_img_ready = nullptr, ev_img_free[2] = {nullptr, nullptr}, ev_copy_fork = nullptr;
  int img_slot = 0;
  bool img_copy_pending = false, img_free_recorded[2] = {false, false};
  void wait_img();                   // cx.stream waits for the asynchronous image copy (no-op once consumed)
  void release_img();                // records "this step's last read of the image staging buffer" on cx.stream
  DevBatch db;
  float* scalars_dev = nullptr;      // [0] loss
  float* flush_buf = nullptr; int64_t flush_n = 0;
  cudaEvent_t t0 = nullptr, t1 = nullptr;
  // side stream for the independent history-LSTM chain (cx.stream is switched while its kernels are issued)
  cudaStream_t main_stream = nullptr, side_stream = nullptr;
  // the streams of one chain's LSTM pair: a = the chain's own stream (layer 1), b = layer 2, c = the contraction between the
  // layers of every step (layer 2's x-projection forward, layer 1's incoming gradient backward)
  struct PairStreams { cudaStream_t a = nullptr, b = nullptr, c = nullptr; };
  PairStreams main_chain, side_chain;
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  bool side_active = false;
  void fork_side();
  void back_to_main();
  void join_side();

  // communicator (NCCL, loaded with dlopen)
  void* nccl_comm = nullptr; int rank = 0, world = 1;

  // ---- forward state ----
  bool have_fwd = false, save_acts = false;
  int32_t *ids_q = nullptr, *ids_h = nullptr, *ids_o = nullptr, *ids_ai = nullptr, *ids_ao = nullptr;
  float *xq = nullptr, *xh = nullptr;
  LstmRun ques1, ques2, hist1, hist2, dialog, opt, dec1, dec2;
  float *encOut = nullptr;
  // lf
  float *join_d = nullptr; int joinK = 0;
  // hrea
  float *img_d = nullptr, *img_e = nullptr, *qi_in = nullptr, *sq = nullptr, *sh = nullptr, *probs = nullptr,
        *att = nullptr, *jt = nullptr, *dial_out = nullptr;
  // mn-att
  float *hAtt = nullptr, *hAtt_d = nullptr, *hAttTr = nullptr, *sum1 = nullptr, *qh2 = nullptr, *t_img = nullptr,
        *img_tr = nullptr, *u_d = nullptr;
  std::vector<float*> img_common, ques_common, sc, pr, u_hop;   // per hop; u_hop[0] = qh2
  // decoder
  float *scores = nullptr, *dscores = nullptr, *row_loss = nullptr, *logp = nullptr, *dlogits = nullptr,
        *lhood = nullptr;
  const float *gen_h0[2] = {nullptr, nullptr}, *gen_c0[2] = {nullptr, nullptr};
  float *gen_dh0[2] = {nullptr, nullptr}, *gen_dc0[2] = {nullptr, nullptr};
  float *dEncFromDec = nullptr;
  // gen decoder, fused vocabulary softmax (tensor-core modes, whole-step entry points): the (rows, V) log-probabilities are
  // never materialised — the projection's epilogue keeps per-slice (max, sum exp) and the target logit, the criterion reads
  // those, the backward recomputes the projection with the softmax gradient in its epilogue.  want_logp = a caller (the
  // module-level vd_decoder_forward) asked for decOut itself.
  bool want_logp = true, fused_vocab_fwd = false;
  float *voc_pm = nullptr, *voc_ps = nullptr, *voc_tl = nullptr, *voc_lse = nullptr;
  int voc_nparts = 0;
  // connect grads handed to the encoder LSTMs (gen.lua:45-60)
  const float *conn_dh_l1 = nullptr, *conn_dc_l1 = nullptr, *conn_dc_l2 = nullptr;

  explicit Engine(const vd_params* p);
  ~Engine();

  // helpers
  const float* Wp(int seg) const { return W + lay.segs[seg].off; }
  const float* Wtp(int seg) const { return Wt + lay.segs[seg].off; }
  float* dWp(int seg) const { return dW + lay.segs[seg].off; }
  int seg(const char* name) const;
  DropCfg dropcfg(float p) const;
  void gemm_tn(int M, int N, int K, const float* A, int64_t lda, const int32_t* gather, const float* B, int64_t ldb,
               float* C, int64_t ldc, float beta, const float* bias, int act);
  void gemm_atb(int M, int N, int64_t K, const float* A, int64_t lda, const int32_t* gather, const float* B, int64_t ldb,
                float* C, int64_t ldc);
  // y = act(x W^T + b) with W = segment `wseg` (out,in), bias = wseg+1
  void linear_fwd(int wseg, const float* x, int64_t rows, float* y, int act);
  // dW += dy^T x ; db += colsum(dy) ; dx (=|+=) dy W
  void linear_bwd(int wseg, const float* x, const float* dy, int64_t rows, float* dx, float beta_dx);
  void refresh_shadows();
  void stage_batch(const vd_batch* b);
  // The route of one SeqLSTM run, the only place where the math mode and the kernels' predicates pick an LSTM's kernels.
  // gathered: rows of the word embedding; WhT / ldw: h columns of the transposed shadow; Wh: h rows of the weight.
  LstmRoute route_lstm(int64_t R, int H, bool gathered, bool has_h0, const float* WhT, int64_t ldw, const float* Wh) const;
  LstmRoute route_lstm(const LstmRun& r) const {
    return route_lstm(r.R, r.H, r.gather != nullptr, r.h0 != nullptr, Wtp(r.wseg) + r.D, r.D + r.H,
                      Wp(r.wseg) + (int64_t)r.D * 4 * r.H);
  }
  // the routes of two stacked runs (layer 2 reads layer 1's h): both layers as one persistent kernel, or the wavefront
  void route_lstm_pair(LstmRun& l1, LstmRun& l2) const;
  // one step on each fp32 route; the Tc steps return the tile width that ran (0: the pointwise kernel)
  void lstm_simt_fwd_step(const LstmFwdStep& s);
  int lstm_tc_fwd_step(const LstmFwdStep& s);
  void lstm_simt_bwd_step(const LstmBwdStep& s);
  int lstm_tc_bwd_step(const LstmBwdStep& s);
  void lstm_forward(LstmRun& r, bool save);          // routes the run, then runs it
  // xproj_by_caller: layer 2 of a pair, whose x-projection lstm_pair_forward (or the persistent kernel) issues per step
  void lstm_forward_begin(LstmRun& r, bool save, bool xproj_by_caller = false);
  void lstm_forward_step(LstmRun& r, int t, bool xproj_by_caller = false);
  void lstm_xproj(const LstmRun& r, int t0, int nt, float* gates);   // gates of steps [t0, t0 + nt) <- x W_x^T (+ bias)
  void lstm_backward_begin(LstmRun& r, const float* dh_all, const float* dh_last, const float* dc_last);
  void lstm_backward_step(LstmRun& r, int t);
  void lstm_backward_end(LstmRun& r, float* dx_out, float* dh0_out, float* dc0_out);
  // two stacked SeqLSTMs, routed by route_lstm_pair.  As a wavefront, layer 2 step t runs (on its own stream) as soon as
  // layer 1 step t is done, and the inter-layer contraction of every step depends on one layer's step t only.
  void lstm_pair_forward(LstmRun& l1, LstmRun& l2, const PairStreams& s);
  void lstm_pair_backward(LstmRun& l1, LstmRun& l2, const float* dh_last2, const float* dc_last2, const float* dh_last1,
                          const float* dc_last1, float* dx1_out, const PairStreams& s);
  // Persistent pair kernels are flag-chained grids that want every SM: two of them must never be co-scheduled (neither
  // could become fully resident), so when the encoder's pairs run as such the two chains run in order on the main stream.
  bool serial_pairs() const { return cfg.useHist && hist1.route.fwd == LstmPath::Pair16; }
  // The disc decoder's option LSTM (disc.lua:4-20) does not depend on the encoder until the final dot product, and its
  // BPTT does not feed the encoder's: both run on their own low-priority stream, concurrently with the encoder's
  // latency-bound chains (which keep priority for SMs as they free up).
  cudaStream_t opt_stream = nullptr;
  cudaEvent_t ev_opt_fork = nullptr, ev_opt_done = nullptr;
  bool opt_overlap = true, opt_fwd_pending = false, opt_bwd_pending = false;
  int opt_reserve_sms = 16;         // SMs the option stream's persistent kernels leave free while they overlap the encoder
  float* opt_demb = nullptr;
  void options_forward_async();
  void options_backward(const float* dfeat);   // the option BPTT from d(h_T) (opt.R, H), on opt_stream when overlapped
  void join_options_backward();      // main stream waits for the option BPTT and folds its embedding gradient in
  // dense fine-tuning step (vd_forward_backward_dense): while dense_round (B, device, 0-based) is set, the option LSTM runs
  // on the K options of round dense_round[b] of each dialog b only
  const int32_t* dense_round = nullptr;
  GrowBuf dense_buf[2];              // the step's rounds and relevance rows, uploaded before the encoder forward
  float forward_backward_dense(const vd_batch* b, const int32_t* round_host, const float* relevance_host);
  std::vector<cudaEvent_t> ev_pool;
  cudaEvent_t pool_event(size_t i);
  void lstm_backward(LstmRun& r, const float* dh_all, const float* dh_last, const float* dc_last, float* dx_out,
                     float* dh0_out, float* dc0_out);

  void encoder_forward(const vd_batch* b);
  void encoder_backward(const float* dEnc);
  // blocks shared by several encoder graphs
  float *qi_join = nullptr, *qi_proj = nullptr;                 // mn-ques-im-hist: [q | fc7] and tanh(Linear(.))
  const float* mn_query_in = nullptr;                           // what enters the memory attention as the query (q3 or qi_proj)
  void mn_block_fwd(const float* qin, const float* h3, float* out);      // MM -> MaskSoftMax -> MM -> fact -> (+q) -> query
  void mn_block_bwd(const float* dout, const float* out, float* dqin, float* dh3);   // dqin / dh3 are overwritten
  void san_block_fwd(const float* u0);                          // SAN hops + out layer -> encOut
  void san_block_bwd(const float* dEnc, float* du0);            // du0 (overwritten) = gradient wrt u0
  void forward_connect();
  void decoder_forward();
  float criterion_forward();
  void criterion_backward();
  void decoder_backward();
  const float* backward_connect();
  void retrieve(const vd_batch* b, int use_gt, int32_t* ranks_host);
  void gen_option_lhood();
  // Model:generateAnswers: one gen-decoder step with explicit state (model.lua:517-526)
  LstmRun gstep1, gstep2;
  float* gstep_logp = nullptr;
  void gen_decoder_step(int64_t rows, const int32_t* tokens_host, const float* const* h_prev, const float* const* c_prev);
  // its core on device-resident tokens, up to the vocabulary projection: gstep_logp holds the LOGITS on return
  void gen_decoder_step_logits(int64_t rows, const int32_t* tok, const float* const* h_prev, const float* const* c_prev);
  // Model:generateAnswers' beam search for every round of the last encoder forward, entirely on the device
  void gen_beam_search(int k, int L, int start_token, int end_token, int32_t* answer_host, int32_t* length_host, double* score_host);
  // its search on n rounds whose start state is row i * stride + off of the last encoder forward; results in the arena
  struct BeamResult { int32_t* ans; int32_t* len; double* score; };     // (n, L), (n), (n)
  BeamResult beam_search_rows(int64_t n, int64_t stride, int64_t off, int k, int L, int start_token, int end_token);
  // the decoder step up to the second LSTM layer (gstep1 / gstep2 hold the new state on return)
  void gen_decoder_step_lstm(int64_t rows, const int32_t* tok, const float* const* h_prev, const float* const* c_prev);
  // Model:generateAnswers' sampling for every round of the last encoder forward, entirely on the device
  void gen_sample(int L, int start_token, float temperature, uint64_t seed, int64_t row_offset, int32_t* answer_host,
                  float* logp_host);
  void check_sample_args(int L, int start_token, float temperature, int64_t row_offset) const;
  // its sampling on n rounds as beam_search_rows takes them; row i draws as global round row_offset + i * stride + off
  struct SampleResult { int32_t* ans; float* logp; };                   // (n, L + 1), (n, L)
  SampleResult sample_rows(int64_t n, int64_t stride, int64_t off, int L, int start_token, float temperature, uint64_t seed,
                           int64_t row_offset);
  // dialogs on the model's own answers (vd_gen_dialog_beam_search / vd_gen_dialog_sample): R rounds of {encoder forward on
  // the engine-owned history, round r's search, the history append} on the device
  struct DialogAnswers {             // where round r's answers are, for the history append
    const int32_t* tokens; int64_t ld;   // row b's answer tokens start at tokens + b * ld
    const int32_t* len;              // beam: hypothesis lengths (the tokens are len - 2 words); null: sampling
    int max_tokens;                  // sampling: the words per row (cut at the first end_token)
    int end_token;
  };
  GrowBuf dialog_hist, dialog_out[4];   // (B, R, W) history; answers, lengths, scores / log-probabilities of all rounds
  void gen_dialog(const vd_batch* b, int W, int max_ans_len, const std::function<DialogAnswers(int)>& search, int32_t* hist_host);
  void gen_dialog_beam_search(const vd_batch* b, int k, int L, int start_token, int end_token, int W, int max_ans_len,
                              int32_t* answer_host, int32_t* length_host, double* score_host, int32_t* hist_host);
  void gen_dialog_sample(const vd_batch* b, int L, int start_token, int end_token, float temperature, uint64_t seed,
                         int64_t row_offset, int W, int max_ans_len, int32_t* answer_host, float* logp_host, int32_t* hist_host);
  void clamp_adam_step(float lr);
  void allreduce_grads();
  // Overlapped gradient sync (world > 1): dW is all-reduced in buckets on `comm_stream` as soon as each bucket's last
  // producer kernel is enqueued — decoder weights at the start of the encoder's backward, the encoder's non-recurrent
  // layers after the attention stage, each LSTM pair after its BPTT, the option LSTM after its stream, the word embedding
  // (the only segment every branch writes) last — instead of one all-reduce after the whole backward.  Armed by
  // vd_zero_grad: a bucket is reduced at most once per zeroed gradient.
  cudaStream_t comm_stream = nullptr;
  cudaEvent_t ev_comm_dep = nullptr, ev_comm_done = nullptr;
  std::vector<char> seg_reduced;
  bool ar_overlap = true, ar_armed = false, comm_pending = false;
  void reduce_range(int64_t off, int64_t count, cudaStream_t producer, cudaEvent_t producer_event);
  void reduce_segments(int first, int last, cudaStream_t producer, cudaEvent_t producer_event = nullptr);
  void reduce_remaining();           // everything not reduced yet, then main_stream waits for the communication stream
  void arm_grad_sync();
};

}  // namespace vd
