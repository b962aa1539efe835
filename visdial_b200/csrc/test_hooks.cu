// vd_test_kernel: the kernels.cuh launchers of pointwise.cu, lstm16.cu's streaming helpers, enc_lstm.cu's persistent
// encoder LSTM pair, gemm_tc.cu's fused vocabulary projections and the engine's two dense contractions, called by name on caller-provided DEVICE buffers on the engine's LaunchCtx, so that grid, shared-memory
// attribute and route are the engine's own; and whole SeqLSTM runs through the engine's own LSTM driver (seq_lstm, seq_lstm_pair).
// The table below is the whole surface: name, pointer / int / real counts, and the call.
//   dropout:  p = reals[0], the site an int; the factors are Engine::dropcfg(p)'s (identity unless training == 1).
//   sampling: SampleCfg from ints (seed, step, row_offset, row_stride) and reals (temperature).
// Pointers may be null where the launcher accepts null (mask ids, gt, inv_scale, ...).
#include "engine.h"

namespace vd {
namespace {

using Fn = void (*)(Engine* e, void* const* P, const int64_t* I, const double* X);
struct Entry {
  const char* name;
  int n_ptrs, n_ints, n_reals;
  Fn fn;
};

#define F(i) (static_cast<float*>(P[i]))
#define CF(i) (static_cast<const float*>(P[i]))
#define I32(i) (static_cast<int32_t*>(P[i]))
#define CI32(i) (static_cast<const int32_t*>(P[i]))
#define H16(i) (static_cast<__half*>(P[i]))
#define CH16(i) (static_cast<const __half*>(P[i]))
#define IN(i) ((int)I[i])
#define DROP(k) e->dropcfg((float)X[k])

// ---- whole SeqLSTM runs: the engine's own route decision and driver on caller buffers.  The run's state lives in the arena
// and is copied out before the arena is rewound to where the call found it.
struct ArenaRewind {
  Arena& a;
  Arena::Mark m;
  ~ArenaRewind() { a.rewind(m); }
};

// an SM budget set for one call, restored however the call ends
struct BudgetRestore {
  LaunchCtx& cx;
  int budget;
  ~BudgetRestore() { cx.sm_budget = budget; }
};

void copy_out(Engine* e, void* dst, const void* src, size_t bytes) {
  if (dst && src) VD_CUDA_CHECK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, e->cx.stream));
}

void route_out(Engine* e, int32_t* dst, const LstmRoute* rt, int n) {
  if (!dst) return;
  int32_t v[10];
  for (int k = 0; k < n; ++k) {
    const int32_t r[5] = {(int32_t)rt[k].fwd, (int32_t)rt[k].bwd, rt[k].table_grad, rt[k].wave_fwd, rt[k].wave_bwd};
    memcpy(v + 5 * k, r, sizeof(r));
  }
  VD_CUDA_CHECK(cudaMemcpyAsync(dst, v, 5 * n * sizeof(int32_t), cudaMemcpyHostToDevice, e->cx.stream));
  VD_CUDA_CHECK(cudaStreamSynchronize(e->cx.stream));
}

// a SeqLSTM on weight segment wseg (bias = wseg + 1), D and H from the segment's (D + H, 4H) shape
LstmRun test_run(Engine* e, int wseg, int T, int64_t R, const float* x, const int32_t* gather, const int32_t* mask) {
  VD_REQUIRE(wseg >= 0 && wseg + 1 < (int)e->lay.segs.size() && e->lay.segs[wseg].init == VD_INIT_LSTM_W, VD_E_BADARG,
             "seq_lstm: wseg is not an LSTM weight segment");
  VD_REQUIRE(T >= 1 && R >= 1 && !(x && gather), VD_E_BADARG, "seq_lstm: T, R, or both x and gather");
  const Seg& s = e->lay.segs[wseg];
  LstmRun r;
  r.T = T; r.R = R; r.H = (int)(s.cols / 4); r.D = (int)(s.rows - s.cols / 4); r.wseg = wseg;
  r.x = x; r.gather = gather; r.mask = mask;
  return r;
}

void seq_lstm_hook(Engine* e, void* const* P, const int64_t* I) {
  e->refresh_shadows();
  ArenaRewind rw{e->arena, e->arena.mark()};
  const bool train = I[3] != 0;
  VD_REQUIRE(P[0] || P[1], VD_E_BADARG, "seq_lstm: x or gather");
  VD_REQUIRE(train || !(P[5] || P[6] || P[7] || P[10] || P[11] || P[12] || P[13] || P[14] || P[15] || P[16]), VD_E_BADARG,
             "seq_lstm: a forward-only run has no saved gates and no gradients");
  LstmRun r = test_run(e, IN(0), IN(1), I[2], CF(0), CI32(1), CI32(2));
  r.h0 = CF(3); r.c0 = CF(4);
  r.demb_out = F(15);
  e->lstm_forward(r, train);
  if (train) e->lstm_backward(r, CF(5), CF(6), CF(7), F(12), F(13), F(14));
  const bool f16 = r.route.fwd == LstmPath::Opt16;
  const size_t RH = (size_t)r.R * r.H, TRH = (size_t)r.T * RH, el = f16 ? sizeof(__half) : sizeof(float);
  if (train) {
    copy_out(e, P[8], f16 ? (const void*)r.h16 : r.h, TRH * el);
    copy_out(e, P[9], r.c, TRH * sizeof(float));
    copy_out(e, P[10], f16 ? (const void*)r.gates16 : r.gates, 4 * TRH * el);
    copy_out(e, P[11], f16 ? (const void*)r.da16 : r.da, 4 * TRH * el);
    copy_out(e, P[16], r.scale2, 2 * sizeof(float));
  } else {
    copy_out(e, P[8], r.h_last(), RH * sizeof(float));
    copy_out(e, P[9], r.c_last(), RH * sizeof(float));
  }
  route_out(e, I32(17), &r.route, 1);
  VD_CUDA_CHECK(cudaStreamSynchronize(e->cx.stream));
}

void seq_lstm_pair_hook(Engine* e, void* const* P, const int64_t* I) {
  e->refresh_shadows();
  ArenaRewind rw{e->arena, e->arena.mark()};
  VD_REQUIRE(P[0], VD_E_BADARG, "seq_lstm_pair: x");
  LstmRun l[2] = {test_run(e, IN(0), IN(2), I[3], CF(0), nullptr, CI32(1)), test_run(e, IN(1), IN(2), I[3], nullptr, nullptr, CI32(1))};
  VD_REQUIRE(l[1].D == l[0].H, VD_E_BADARG, "seq_lstm_pair: layer 2's input is layer 1's h");
  e->route_lstm_pair(l[0], l[1]);
  e->lstm_pair_forward(l[0], l[1], e->main_chain);
  e->lstm_pair_backward(l[0], l[1], CF(2), CF(3), CF(4), CF(5), F(10), e->main_chain);
  const size_t TRH = (size_t)l[0].T * l[0].R * l[0].H * sizeof(float);
  copy_out(e, P[6], l[0].h, TRH);
  copy_out(e, P[7], l[0].c, TRH);
  copy_out(e, P[8], l[1].h, TRH);
  copy_out(e, P[9], l[1].c, TRH);
  const LstmRoute rt[2] = {l[0].route, l[1].route};
  route_out(e, I32(11), rt, 2);
  VD_CUDA_CHECK(cudaStreamSynchronize(e->cx.stream));
}

// the answer rules of a *_rules hook: P = {hist, banned}, I = {step, ld, end_token, min_words, no_repeat_ngram, n_banned}
AnswerRules hook_rules(void* const* P, const int64_t* I) {
  AnswerRules a;
  a.hist = static_cast<const int32_t*>(P[0]); a.banned = static_cast<const int32_t*>(P[1]);
  a.step = (int32_t)I[0]; a.ld = I[1]; a.end_token = (int32_t)I[2];
  a.min_words = (int32_t)I[3]; a.no_repeat_ngram = (int32_t)I[4]; a.n_banned = (int32_t)I[5];
  return a;
}

const Entry TABLE[] = {
    // ---- history attention: (ptrs), ints B, R, H
    {"mn_attention_fwd", 4, 3, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) { mn_attention_fwd(e->cx, CF(0), CF(1), F(2), F(3), IN(0), IN(1), IN(2)); }},
    {"mn_attention_bwd", 6, 3, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       mn_attention_bwd(e->cx, CF(0), CF(1), CF(2), CF(3), F(4), F(5), IN(0), IN(1), IN(2));
     }},
    {"hrea_attention_fwd", 5, 3, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       hrea_attention_fwd(e->cx, CF(0), CF(1), CF(2), F(3), F(4), IN(0), IN(1), IN(2));
     }},
    {"hrea_attention_bwd", 8, 3, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       hrea_attention_bwd(e->cx, CF(0), CF(1), CF(2), CF(3), CF(4), F(5), F(6), F(7), IN(0), IN(1), IN(2));
     }},
    // round-range forms (a dialog session's [r, r+1)): ints B, R, H, r0, r1, fact pitch
    {"mn_attention_rows_fwd", 4, 6, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       mn_attention_rows_fwd(e->cx, CF(0), CF(1), I[5], F(2), F(3), IN(0), IN(1), IN(2), IN(3), IN(4));
     }},
    {"hrea_attention_rows_fwd", 5, 6, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       hrea_attention_rows_fwd(e->cx, CF(0), CF(1), CF(2), I[5], F(3), F(4), IN(0), IN(1), IN(2), IN(3), IN(4));
     }},
    // facts, shc (or null), h3, sh (or null); ints B, R, H, r
    {"dialog_cache_write", 4, 4, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       dialog_cache_write(e->cx, F(0), F(1), CF(2), CF(3), I[0], IN(1), IN(2), IN(3));
     }},
    // per-row forms (a dialog pool's ask): ptrs as above, then slot, round (device, n); ints n, R, H, fact pitch
    {"mn_attention_slots_fwd", 6, 4, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       mn_attention_rows_fwd(e->cx, CF(0), CF(1), I[3], F(2), F(3), IN(0), IN(1), IN(2), 0, 1, CI32(4), CI32(5));
     }},
    {"hrea_attention_slots_fwd", 7, 4, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       hrea_attention_rows_fwd(e->cx, CF(0), CF(1), CF(2), I[3], F(3), F(4), IN(0), IN(1), IN(2), 0, 1, CI32(5), CI32(6));
     }},
    // facts, shc, h3, sh, slot, round, st_h, st_c, hn, cn (each pair may be null); ints n, R, H
    {"dialog_cache_write_slots", 10, 3, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       dialog_cache_write(e->cx, F(0), F(1), CF(2), CF(3), I[0], IN(1), IN(2), 0, CI32(4), CI32(5), F(6), F(7), CF(8), CF(9));
     }},
    // slot, round, q, ques, ids_q, hist, ids_h, img, img_out, h, c, h_out, c_out; ints n, R, Tq, W, img_cols, H
    {"dialog_gather", 13, 6, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       DialogGather g;
       g.n = I[0]; g.R = IN(1); g.slot = CI32(0); g.round = CI32(1); g.q = CI32(2); g.Tq = IN(2); g.ques = I32(3); g.ids_q = I32(4);
       g.hist = CI32(5); g.W = IN(3); g.ids_h = I32(6); g.img = CF(7); g.img_cols = I[4]; g.img_out = F(8);
       g.h = CF(9); g.c = CF(10); g.H = IN(5); g.h_out = F(11); g.c_out = F(12);
       dialog_gather(e->cx, g);
     }},
    // dst, src, slot; ints n, cols
    {"scatter_rows", 3, 2, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) { scatter_rows(e->cx, F(0), CF(1), CI32(2), I[0], I[1]); }},
    // hist, src, ans, ans_len (or null), slot, round (or null); ints B, R, W, r, src_w, ans_ld, ans_max, end_token,
    // max_ans_len, concat
    {"hist_append_slots", 6, 10, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       hist_append(e->cx, I32(0), I[0], IN(1), IN(2), IN(3), CI32(1), IN(4), CI32(2), I[5], CI32(3), IN(6), IN(7), IN(8), I[9] != 0,
                   CI32(4), CI32(5));
     }},
    // hist, slot, rounds, row0, q, ans; ints n, R, W, src_w, Ta, end_token, max_ans_len, concat
    {"hist_prefill", 6, 8, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       hist_prefill(e->cx, I32(0), I[0], IN(1), IN(2), CI32(1), CI32(2), CI32(3), CI32(4), IN(3), CI32(5), IN(4), IN(5), IN(6),
                    I[7] != 0);
     }},
    // ---- SAN: ints as the launcher's, the dropout site last; reals p
    {"san_expand_dropout", 2, 5, 1,
     [](Engine* e, void* const* P, const int64_t* I, const double* X) {
       san_expand_dropout(e->cx, F(0), CF(1), IN(0), IN(1), IN(2), IN(3), DROP(0), (uint32_t)I[4]);
     }},
    {"san_score_fwd", 5, 4, 1,
     [](Engine* e, void* const* P, const int64_t* I, const double* X) {
       san_score_fwd(e->cx, CF(0), CF(1), CF(2), CF(3), F(4), I[0], IN(1), IN(2), DROP(0), (uint32_t)I[3]);
     }},
    {"san_softmax_att_fwd", 5, 3, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       san_softmax_att_fwd(e->cx, CF(0), F(1), CF(2), CF(3), F(4), I[0], IN(1), IN(2));
     }},
    {"san_att_bwd", 5, 3, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       san_att_bwd(e->cx, CF(0), CF(1), CF(2), F(3), F(4), I[0], IN(1), IN(2));
     }},
    {"san_score_bwd", 8, 4, 1,
     [](Engine* e, void* const* P, const int64_t* I, const double* X) {
       san_score_bwd(e->cx, CF(0), CF(1), CF(2), CF(3), F(4), F(5), F(6), F(7), I[0], IN(1), IN(2), DROP(0), (uint32_t)I[3]);
     }},
    {"san_collapse_bwd", 3, 5, 1,
     [](Engine* e, void* const* P, const int64_t* I, const double* X) {
       san_collapse_bwd(e->cx, CF(0), CF(1), F(2), IN(0), IN(1), IN(2), IN(3), DROP(0), (uint32_t)I[4]);
     }},
    // masked SAN (region features, DESIGN §26): the pointer after the unmasked entry's is the count array; ints as the
    // unmasked entry's, then R (rows per count; san_collapse_bwd's counts are per dialog)
    {"san_score_fwd_masked", 6, 5, 1,
     [](Engine* e, void* const* P, const int64_t* I, const double* X) {
       san_score_fwd(e->cx, CF(0), CF(1), CF(2), CF(3), F(4), I[0], IN(1), IN(2), DROP(0), (uint32_t)I[3], CI32(5), IN(4));
     }},
    {"san_softmax_att_fwd_masked", 6, 4, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       san_softmax_att_fwd(e->cx, CF(0), F(1), CF(2), CF(3), F(4), I[0], IN(1), IN(2), CI32(5), IN(3));
     }},
    {"san_att_bwd_masked", 6, 4, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       san_att_bwd(e->cx, CF(0), CF(1), CF(2), F(3), F(4), I[0], IN(1), IN(2), CI32(5), IN(3));
     }},
    {"san_score_bwd_masked", 9, 5, 1,
     [](Engine* e, void* const* P, const int64_t* I, const double* X) {
       san_score_bwd(e->cx, CF(0), CF(1), CF(2), CF(3), F(4), F(5), F(6), F(7), I[0], IN(1), IN(2), DROP(0), (uint32_t)I[3],
                     CI32(8), IN(4));
     }},
    {"san_collapse_bwd_masked", 4, 5, 1,
     [](Engine* e, void* const* P, const int64_t* I, const double* X) {
       san_collapse_bwd(e->cx, CF(0), CF(1), F(2), IN(0), IN(1), IN(2), IN(3), DROP(0), (uint32_t)I[4], CI32(3));
     }},
    // ---- option scores, criteria, ranks
    {"disc_scores_fwd", 3, 3, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) { disc_scores_fwd(e->cx, CF(0), CF(1), F(2), I[0], IN(1), IN(2)); }},
    {"disc_scores_bwd", 5, 3, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       disc_scores_bwd(e->cx, CF(0), CF(1), CF(2), F(3), F(4), I[0], IN(1), IN(2));
     }},
    {"xent_fwd", 3, 2, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) { xent_fwd(e->cx, CF(0), CI32(1), F(2), I[0], IN(1)); }},
    {"xent_bwd", 3, 2, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) { xent_bwd(e->cx, CF(0), CI32(1), F(2), I[0], IN(1)); }},
    {"soft_xent", 4, 2, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) { soft_xent(e->cx, CF(0), CF(1), F(2), F(3), I[0], IN(1)); }},
    {"reduce_sum", 2, 1, 1,
     [](Engine* e, void* const* P, const int64_t* I, const double* X) { reduce_sum(e->cx, CF(0), F(1), I[0], (float)X[0]); }},
    {"rank_rows", 3, 2, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) { rank_rows(e->cx, CF(0), CI32(1), I32(2), I[0], IN(1)); }},
    // ---- vocabulary rows: ints rows, V (, ...)
    {"logsoftmax_rows", 2, 2, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) { logsoftmax_rows(e->cx, F(0), CI32(1), I[0], IN(1)); }},
    {"lhood_accumulate", 4, 2, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) { lhood_accumulate(e->cx, CF(0), CI32(1), CI32(2), F(3), I[0], IN(1)); }},
    {"nll_fwd", 4, 2, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) { nll_fwd(e->cx, CF(0), CI32(1), CI32(2), F(3), I[0], IN(1)); }},
    {"nll_bwd", 4, 2, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) { nll_bwd(e->cx, CF(0), CI32(1), CI32(2), F(3), I[0], IN(1)); }},
    // writes vocab_lse_nparts(ints[0]) into the device int32 at ptrs[0]
    {"vocab_lse_nparts", 1, 1, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       const int32_t n = vocab_lse_nparts(IN(0));
       VD_CUDA_CHECK(cudaMemcpyAsync(P[0], &n, sizeof(n), cudaMemcpyHostToDevice, e->cx.stream));
       VD_CUDA_CHECK(cudaStreamSynchronize(e->cx.stream));
     }},
    // ptrs part_max, part_sum, tgt_logit, tgt, row_ids, lse, out; ints nparts, accumulate, rows; reals sign
    {"vocab_lse_finish", 7, 3, 1,
     [](Engine* e, void* const* P, const int64_t* I, const double* X) {
       vocab_lse_finish(e->cx, CF(0), CF(1), IN(0), CF(2), CI32(3), CI32(4), F(5), F(6), (float)X[0], IN(1), I[2]);
     }},
    {"logsoftmax_topk_rows", 4, 3, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       logsoftmax_topk_rows(e->cx, CF(0), CI32(1), I[0], IN(1), IN(2), F(2), I32(3));
     }},
    // the beam-search merge of one step (DESIGN §22).  ptrs topv, topi, scores_in, scores_out, beams_in, beams_out, tokens,
    // parent, ans, ans_len, ans_score, pick_ans, pick_len, pick_score (the three pick pointers all null or none); ints N, stp,
    // k, G, L, end_token; reals diversity
    {"beam_merge", 14, 6, 1,
     [](Engine* e, void* const* P, const int64_t* I, const double* X) {
       BeamLists b;
       b.ans = I32(8); b.len = I32(9); b.score = static_cast<double*>(P[10]);
       beam_merge(e->cx, I[0], IN(1), IN(2), IN(3), (float)X[0], IN(4), IN(5), CF(0), CI32(1), static_cast<const double*>(P[2]),
                  static_cast<double*>(P[3]), CI32(4), I32(5), I32(6), I32(7), b, I32(11), I32(12), static_cast<double*>(P[13]));
     }},
    // as beam_merge with n-best lists (DESIGN §24): ans / ans_len / ans_score are the list slots (N, G, n, ...), and seven
    // more ptrs: lp (L, or null), norm, ord, out_ans, out_len, out_score, out_norm (the last five null for n = 1); a seventh
    // int n
    {"beam_merge_nbest", 21, 7, 1,
     [](Engine* e, void* const* P, const int64_t* I, const double* X) {
       BeamLists b;
       b.nbest = IN(6);
       b.ans = I32(8); b.len = I32(9); b.score = static_cast<double*>(P[10]);
       b.lp = static_cast<const double*>(P[14]); b.norm = static_cast<double*>(P[15]); b.ord = I32(16);
       b.out_ans = I32(17); b.out_len = I32(18); b.out_score = static_cast<double*>(P[19]); b.out_norm = static_cast<double*>(P[20]);
       beam_merge(e->cx, I[0], IN(1), IN(2), IN(3), (float)X[0], IN(4), IN(5), CF(0), CI32(1), static_cast<const double*>(P[2]),
                  static_cast<double*>(P[3]), CI32(4), I32(5), I32(6), I32(7), b, I32(11), I32(12), static_cast<double*>(P[13]));
     }},
    // ptrs logits, tokens, answer, logp; ints rows, V, L, seed, step, row_offset, row_stride; reals temperature
    {"logsoftmax_sample_rows", 4, 7, 1,
     [](Engine* e, void* const* P, const int64_t* I, const double* X) {
       SampleCfg s;
       s.seed_lo = (uint32_t)(uint64_t)I[3]; s.seed_hi = (uint32_t)((uint64_t)I[3] >> 32); s.step = (uint32_t)I[4];
       s.temperature = (float)X[0]; s.row_offset = I[5]; s.row_stride = I[6];
       logsoftmax_sample_rows(e->cx, CF(0), I[0], IN(1), s, IN(2), I32(1), I32(2), F(3));
     }},
    // as logsoftmax_sample_rows, and a fifth pointer: the per-row global rounds (SampleCfg::row_round)
    {"logsoftmax_sample_rows_drawn", 5, 7, 1,
     [](Engine* e, void* const* P, const int64_t* I, const double* X) {
       SampleCfg s;
       s.seed_lo = (uint32_t)(uint64_t)I[3]; s.seed_hi = (uint32_t)((uint64_t)I[3] >> 32); s.step = (uint32_t)I[4];
       s.temperature = (float)X[0]; s.row_offset = I[5]; s.row_stride = I[6];
       s.row_round = static_cast<const int64_t*>(P[4]);
       logsoftmax_sample_rows(e->cx, CF(0), I[0], IN(1), s, IN(2), I32(1), I32(2), F(3));
     }},
    // as logsoftmax_sample_rows, a fifth pointer (the per-row global rounds, or null: the affine rule), an eighth int top_k
    // and a second real top_p (DESIGN §23)
    {"truncated_sample_rows", 5, 8, 2,
     [](Engine* e, void* const* P, const int64_t* I, const double* X) {
       SampleCfg s;
       s.seed_lo = (uint32_t)(uint64_t)I[3]; s.seed_hi = (uint32_t)((uint64_t)I[3] >> 32); s.step = (uint32_t)I[4];
       s.temperature = (float)X[0]; s.row_offset = I[5]; s.row_stride = I[6];
       s.row_round = static_cast<const int64_t*>(P[4]);
       TruncCfg t;
       t.top_k = IN(7); t.top_p = (float)X[1];
       truncated_sample_rows(e->cx, CF(0), I[0], IN(1), s, t, IN(2), I32(1), I32(2), F(3));
     }},
    // ---- the answer rules (DESIGN §25) on the kernels above: each takes its hook's arguments plus the row histories hist
    // (row pitch ld) and the banned ids (device, or null), and the ints ld, end_token, min_words, no_repeat_ngram, n_banned
    // (the rules' step is the hook's step).  ptrs logits, mask_ids, topv, topi, hist, banned; ints rows, V, k, step, then
    // the five
    {"logsoftmax_topk_rows_rules", 6, 9, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       const AnswerRules ar = hook_rules(P + 4, I + 3);
       logsoftmax_topk_rows(e->cx, CF(0), CI32(1), I[0], IN(1), IN(2), F(2), I32(3), &ar);
     }},
    // beam_merge_nbest's arguments; -inf top-k entries are no candidates
    {"beam_merge_rules", 21, 7, 1,
     [](Engine* e, void* const* P, const int64_t* I, const double* X) {
       BeamLists b;
       b.nbest = IN(6);
       b.ans = I32(8); b.len = I32(9); b.score = static_cast<double*>(P[10]);
       b.lp = static_cast<const double*>(P[14]); b.norm = static_cast<double*>(P[15]); b.ord = I32(16);
       b.out_ans = I32(17); b.out_len = I32(18); b.out_score = static_cast<double*>(P[19]); b.out_norm = static_cast<double*>(P[20]);
       beam_merge(e->cx, I[0], IN(1), IN(2), IN(3), (float)X[0], IN(4), IN(5), CF(0), CI32(1), static_cast<const double*>(P[2]),
                  static_cast<double*>(P[3]), CI32(4), I32(5), I32(6), I32(7), b, I32(11), I32(12), static_cast<double*>(P[13]), true);
     }},
    // logsoftmax_sample_rows_drawn's arguments (the fifth pointer may be null: the affine rule), then hist, banned; the
    // seven ints, then the five
    {"logsoftmax_sample_rows_rules", 7, 12, 1,
     [](Engine* e, void* const* P, const int64_t* I, const double* X) {
       SampleCfg s;
       s.seed_lo = (uint32_t)(uint64_t)I[3]; s.seed_hi = (uint32_t)((uint64_t)I[3] >> 32); s.step = (uint32_t)I[4];
       s.temperature = (float)X[0]; s.row_offset = I[5]; s.row_stride = I[6];
       s.row_round = static_cast<const int64_t*>(P[4]);
       AnswerRules ar = hook_rules(P + 5, I + 6);
       ar.step = IN(4);
       logsoftmax_sample_rows(e->cx, CF(0), I[0], IN(1), s, IN(2), I32(1), I32(2), F(3), &ar);
     }},
    // truncated_sample_rows' arguments, then hist, banned; its eight ints, then the five
    {"truncated_sample_rows_rules", 7, 13, 2,
     [](Engine* e, void* const* P, const int64_t* I, const double* X) {
       SampleCfg s;
       s.seed_lo = (uint32_t)(uint64_t)I[3]; s.seed_hi = (uint32_t)((uint64_t)I[3] >> 32); s.step = (uint32_t)I[4];
       s.temperature = (float)X[0]; s.row_offset = I[5]; s.row_stride = I[6];
       s.row_round = static_cast<const int64_t*>(P[4]);
       TruncCfg t;
       t.top_k = IN(7); t.top_p = (float)X[1];
       AnswerRules ar = hook_rules(P + 5, I + 7);
       ar.step = IN(4);
       truncated_sample_rows(e->cx, CF(0), I[0], IN(1), s, t, IN(2), I32(1), I32(2), F(3), &ar);
     }},
    // ptrs logits, lse, tgt, mask_ids, scale, dlogits (may alias logits); ints rows, V
    {"nll_bwd_scaled", 6, 2, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       nll_bwd_scaled(e->cx, CF(0), CF(1), CI32(2), CI32(3), CF(4), F(5), I[0], IN(1));
     }},
    {"scale_copy", 2, 1, 1,
     [](Engine* e, void* const* P, const int64_t* I, const double* X) { scale_copy(e->cx, F(0), CF(1), I[0], (float)X[0]); }},
    // ---- fused vocabulary projections (gemm_tc.cu): a shape vocab_tc_ok refuses comes back as VD_E_SHAPE, nothing launched.
    // ptrs A, B, bias, tgt, part_max, part_sum, tgt_logit; ints M, N, K, lda, ldb
    {"vocab_lse_tc", 7, 5, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       VD_REQUIRE(vocab_lse_tc(e->cx, IN(0), IN(1), IN(2), CF(0), I[3], CF(1), I[4], CF(2), CI32(3), F(4), F(5), F(6)), VD_E_SHAPE,
                  "vocab_lse_tc: shape refused");
     }},
    // ptrs A, B, bias, tgt, row_ids, lse, C, row_scale (null: unscaled); ints M, N, K, lda, ldb, ldc
    {"vocab_dlogits_tc", 8, 6, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       VD_REQUIRE(vocab_dlogits_tc(e->cx, IN(0), IN(1), IN(2), CF(0), I[3], CF(1), I[4], CF(2), CI32(3), CI32(4), CF(5), F(6), I[5],
                                   CF(7)),
                  VD_E_SHAPE, "vocab_dlogits_tc: shape refused");
     }},
    // ptrs A, B, bias, part_max, part_sum, part_key, part_cls, part_x; ints M, N, K, lda, ldb, seed, step, row_offset, row_stride;
    // reals temperature
    {"vocab_sample_tc", 8, 9, 1,
     [](Engine* e, void* const* P, const int64_t* I, const double* X) {
       SampleCfg s;
       s.seed_lo = (uint32_t)(uint64_t)I[5]; s.seed_hi = (uint32_t)((uint64_t)I[5] >> 32); s.step = (uint32_t)I[6];
       s.temperature = (float)X[0]; s.row_offset = I[7]; s.row_stride = I[8];
       VD_REQUIRE(vocab_sample_tc(e->cx, IN(0), IN(1), IN(2), CF(0), I[3], CF(1), I[4], CF(2), s, F(3), F(4), F(5), I32(6), F(7)),
                  VD_E_SHAPE, "vocab_sample_tc: shape refused");
     }},
    // as vocab_sample_tc, and a ninth pointer: the per-row global rounds (SampleCfg::row_round)
    {"vocab_sample_tc_drawn", 9, 9, 1,
     [](Engine* e, void* const* P, const int64_t* I, const double* X) {
       SampleCfg s;
       s.seed_lo = (uint32_t)(uint64_t)I[5]; s.seed_hi = (uint32_t)((uint64_t)I[5] >> 32); s.step = (uint32_t)I[6];
       s.temperature = (float)X[0]; s.row_offset = I[7]; s.row_stride = I[8];
       s.row_round = static_cast<const int64_t*>(P[8]);
       VD_REQUIRE(vocab_sample_tc(e->cx, IN(0), IN(1), IN(2), CF(0), I[3], CF(1), I[4], CF(2), s, F(3), F(4), F(5), I32(6), F(7)),
                  VD_E_SHAPE, "vocab_sample_tc: shape refused");
     }},
    // ptrs part_max, part_sum, part_key, part_cls, part_x, tokens, answer, logp (may be null); ints nparts, rows, step, L
    {"vocab_sample_finish", 8, 4, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       vocab_sample_finish(e->cx, CF(0), CF(1), CF(2), CI32(3), CF(4), IN(0), I[1], IN(2), IN(3), I32(5), I32(6), F(7));
     }},
    // ---- embedding and token grouping
    {"embed_rows", 3, 3, 1,
     [](Engine* e, void* const* P, const int64_t* I, const double* X) {
       embed_rows(e->cx, F(0), CF(1), CI32(2), I[0], IN(1), DROP(0), (uint32_t)I[2]);
     }},
    {"embed_scatter_add", 3, 4, 1,
     [](Engine* e, void* const* P, const int64_t* I, const double* X) {
       embed_scatter_add(e->cx, F(0), CF(1), I[0], CI32(2), I[1], IN(2), DROP(0), (uint32_t)I[3], e->cfg.V + 1);
     }},
    // ptrs ids, scratch (3 nv int32), perm, sorted_tok; ints n, nv
    {"group_rows_by_token", 4, 2, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       group_rows_by_token(e->cx, CI32(0), I[0], IN(1), I32(1), I32(2), I32(3));
     }},
    {"segsum_rows", 4, 3, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       segsum_rows(e->cx, CF(0), I[0], CI32(1), CI32(2), I[1], F(3), IN(2));
     }},
    {"cvt_f32_to_f16", 2, 4, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) { cvt_f32_to_f16(e->cx, H16(0), I[0], CF(1), I[1], I[2], IN(3)); }},
    {"pick_grad_scale", 3, 1, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       pick_grad_scale(e->cx, CF(0), I[0], static_cast<uint32_t*>(P[1]), F(2));
     }},
    // ptrs A16, B16, C, inv_scale; ints M, N, K, lda, ldb, ldc, CTAs (0 = the engine's), launches, streams (1 or 2: launch i
    // goes to stream i % streams, the second one a fresh stream that starts after and ends before the engine's)
    {"gemm_atb16", 4, 9, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       VD_REQUIRE(I[8] == 1 || I[8] == 2, VD_E_BADARG, "gemm_atb16: streams");
       LaunchCtx cs[2];
       for (LaunchCtx& c : cs) {
         c.sm_count = e->cx.sm_count; c.sm_budget = IN(6); c.stream = e->cx.stream;
         c.deterministic = e->cx.deterministic; c.scratch = e->cx.scratch;
       }
       cudaEvent_t ev = nullptr;
       if (I[8] == 2) {
         VD_CUDA_CHECK(cudaStreamCreateWithFlags(&cs[1].stream, cudaStreamNonBlocking));
         VD_CUDA_CHECK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
         VD_CUDA_CHECK(cudaEventRecord(ev, cs[0].stream));
         VD_CUDA_CHECK(cudaStreamWaitEvent(cs[1].stream, ev, 0));
       }
       for (int64_t i = 0; i < I[7]; ++i)
         gemm_atb16(cs[i % I[8]], IN(0), IN(1), I[2], CH16(0), I[3], CH16(1), I[4], F(2), I[5], CF(3));
       if (I[8] == 2) {
         VD_CUDA_CHECK(cudaEventRecord(ev, cs[1].stream));
         VD_CUDA_CHECK(cudaStreamWaitEvent(cs[0].stream, ev, 0));
         VD_CUDA_CHECK(cudaStreamSynchronize(cs[1].stream));
         VD_CUDA_CHECK(cudaEventDestroy(ev));
         VD_CUDA_CHECK(cudaStreamDestroy(cs[1].stream));
       }
     }},
    // ---- the dense contractions as the engine routes them in its current math mode (Engine::gemm_tn / gemm_atb: the
    // tensor-core kernel where gemm_tn_tc / gemm_atb_tc take the shape, the CUDA-core one otherwise).
    // ptrs A, gather (or null), B, C, bias (or null); ints M, N, K, lda, ldb, ldc, act; reals beta
    {"gemm_tn", 5, 7, 1,
     [](Engine* e, void* const* P, const int64_t* I, const double* X) {
       e->gemm_tn(IN(0), IN(1), IN(2), CF(0), I[3], CI32(1), CF(2), I[4], F(3), I[5], (float)X[0], CF(4), IN(6));
     }},
    // ptrs A, gather (or null), B, C; ints M, N, K, lda, ldb, ldc, SM budget (0: the engine's own, as it stands), which holds
    // for this call only
    {"gemm_atb", 4, 7, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       BudgetRestore br{e->cx, e->cx.sm_budget};
       if (I[6] > 0) e->cx.sm_budget = IN(6);
       e->gemm_atb(IN(0), IN(1), I[2], CF(0), I[3], CI32(1), CF(2), I[4], F(3), I[5]);
     }},
    // ---- the fp16 option-LSTM BPTT (lstm16.cu, k_lstm16_bptt) over steps T - 2 .. 0 in waves of clusters.  ptrs da16 (T slices
    // of (R, 4H); slice T - 1 is the input), Whb16 (H, 4H), gates16 (T slices of (R, 4H)), c (T slices of (R, H)), c0 (R, H) or
    // null, mask ids (T slices of R) or null, dc_carry (R, H, in and out), plan (3 int64: cluster size, row blocks per launch,
    // launches; may be null).  ints R, H, T, SM budget (0: all SMs)
    {"lstm16_bptt", 8, 4, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       LaunchCtx cx;
       cx.sm_count = e->cx.sm_count; cx.sm_budget = IN(3); cx.stream = e->cx.stream;
       lstm16_bptt(cx, I[0], IN(1), IN(2), H16(0), CH16(1), CH16(2), CF(3), CF(4), CI32(5), F(6));
       if (P[7]) {
         const Bptt16Plan pl = lstm16_bptt_plan(cx, I[0], IN(1));
         const int64_t v[3] = {pl.csize, pl.clusters, pl.waves};
         VD_CUDA_CHECK(cudaMemcpyAsync(P[7], v, sizeof(v), cudaMemcpyHostToDevice, e->cx.stream));
         VD_CUDA_CHECK(cudaStreamSynchronize(e->cx.stream));
       }
     }},
    {"segsum_rows16", 5, 3, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       segsum_rows16(e->cx, static_cast<const __half*>(P[0]), I[0], CI32(1), CI32(2), I[1], F(3), IN(2), CF(4));
     }},
    // ---- persistent encoder LSTM pair (enc_lstm.cu), ints T, R, H.  forward ptrs W1h16, W2cat16, bias2, mask, gates1, c1, h1,
    // h1_16, gates2, c2, h2, h2_16, flags;  backward ptrs B1cat16, Whb2_16, mask, gates1, c1, gates2, c2, dh_last1, dc_last1,
    // dh_last2, dc_last2, da1, da1_16, da2, da2_16, flags, dh1, dh2, scale (null dh1 / dh2 = the unit split at any H)
    {"enc_pair_forward", 13, 3, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       enc_pair_forward(e->cx, IN(0), I[1], IN(2), CH16(0), CH16(1), CF(2), CI32(3), F(4), F(5), F(6), H16(7), F(8), F(9), F(10),
                        H16(11), I32(12));
     }},
    {"enc_pair_backward", 19, 3, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       enc_pair_backward(e->cx, IN(0), I[1], IN(2), CH16(0), CH16(1), CI32(2), CF(3), CF(4), CF(5), CF(6), CF(7), CF(8), CF(9), CF(10),
                         F(11), H16(12), F(13), H16(14), I32(15), F(16), F(17), F(18));
     }},
    // writes enc_pair_bwd_flag_ints(T, R, H) into the device int64 at ptrs[0]
    {"enc_pair_bwd_flag_ints", 1, 3, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       const int64_t n = enc_pair_bwd_flag_ints(IN(0), I[1], IN(2));
       VD_CUDA_CHECK(cudaMemcpyAsync(P[0], &n, sizeof(n), cudaMemcpyHostToDevice, e->cx.stream));
       VD_CUDA_CHECK(cudaStreamSynchronize(e->cx.stream));
     }},
    // ---- whole SeqLSTM runs (Engine::lstm_forward / lstm_backward, routed by route_lstm) on weight segment wseg.  ptrs x (T R, D)
    // or null, gather ids (T R) or null, mask ids (T R), h0, c0, dh_all (T R, H), dh_last, dc_last (R, H); outputs h, c, gates, da,
    // dx, dh0, dc0, demb_out ((V+1, E), overwritten; null: the embedding gradient goes to dW), scale, info; any of them may be
    // null.  ints wseg, T, R, train.  train = 1: a saved run and its BPTT, h / c / gates / da of all T steps (Opt16: its fp16 h,
    // gates and da, da times s; scale {s, 1/s}); train = 0: a run without saved state, h / c of the last step.  info int32
    // {fwd path, bwd path, table_grad, wave_fwd, wave_bwd} (LstmPath values).  Weight and bias gradients accumulate into dW.
    {"seq_lstm", 18, 4, 0, [](Engine* e, void* const* P, const int64_t* I, const double*) { seq_lstm_hook(e, P, I); }},
    // two stacked runs routed by route_lstm_pair on the main chain's streams, forward and BPTT.  ptrs x (T R, D1), mask,
    // dh_last2, dc_last2, dh_last1, dc_last1 (each may be null); outputs h1, c1, h2, c2 (T R, H), dx1 (T R, D1), info (two
    // layers' five ints as seq_lstm's).  ints wseg1, wseg2, T, R
    {"seq_lstm_pair", 12, 4, 0, [](Engine* e, void* const* P, const int64_t* I, const double*) { seq_lstm_pair_hook(e, P, I); }},
    // ---- answer-pool top-k (DESIGN §18), routed as the engine routes it: ptrs Q, E, topv, topi; ints rows, ldq, m, H, k
    {"answer_pool_topk", 4, 5, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       e->pool_topk(CF(0), I[1], I[0], CF(1), I[2], IN(3), IN(4), F(2), I32(3));
     }},
    // ---- the gen dense step's d-logit budget in bytes (ints[0] <= 0: the default, Engine::kDenseGenChunkBytes)
    {"dense_gen_chunk_bytes", 0, 1, 0,
     [](Engine* e, void* const*, const int64_t* I, const double*) {
       e->dense_gen_chunk_bytes = I[0] > 0 ? I[0] : Engine::kDenseGenChunkBytes;
     }},
    // the (B, numOptions) scores of the last dense step into the device floats at ptrs[0]; ints B * numOptions
    {"dense_scores", 1, 1, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       VD_REQUIRE(e->scores && I[0] > 0, VD_E_STATE, "dense_scores: no step has run");
       VD_CUDA_CHECK(cudaMemcpyAsync(P[0], e->scores, (size_t)I[0] * sizeof(float), cudaMemcpyDeviceToDevice, e->cx.stream));
     }},
    // ---- small helpers
    {"colsum_add", 2, 3, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) { colsum_add(e->cx, F(0), CF(1), I[0], IN(1), I[2]); }},
    {"rowdot_fwd", 4, 2, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) { rowdot_fwd(e->cx, F(0), CF(1), CF(2), CF(3), I[0], IN(1)); }},
    // ptrs ds, x, w, dx, dw, db; ints accumulate_dx, rows, H
    {"rowdot_bwd", 6, 3, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       rowdot_bwd(e->cx, CF(0), CF(1), CF(2), F(3), IN(0), F(4), F(5), I[1], IN(2));
     }},
    {"repeat_rows", 2, 4, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) { repeat_rows(e->cx, F(0), CF(1), I[0], IN(1), I[2], I[3]); }},
    {"sum_repeated_rows", 2, 3, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) { sum_repeated_rows(e->cx, F(0), CF(1), I[0], IN(1), I[2]); }},
    {"masktime_concat_fwd", 4, 4, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       masktime_concat_fwd(e->cx, F(0), CF(1), CF(2), CI32(3), IN(0), I[1], IN(2), IN(3));
     }},
    // ptrs dx, ids_tm, dimg; ints ldx, off, T, N, I
    {"masktime_bwd", 3, 5, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       masktime_bwd(e->cx, CF(0), I[0], IN(1), CI32(1), F(2), IN(2), I[3], IN(4));
     }},
    {"transpose_ids", 2, 2, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) { transpose_ids(e->cx, CI32(0), I32(1), I[0], IN(1)); }},
    {"transpose_ids_rounds", 3, 4, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       transpose_ids_rounds(e->cx, CI32(0), CI32(1), I32(2), I[0], IN(1), IN(2), IN(3));
     }},
    {"gather_round_rows", 3, 3, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) { gather_round_rows(e->cx, CF(0), CI32(1), F(2), I[0], IN(1), IN(2)); }},
    {"scatter_round_rows", 3, 3, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) { scatter_round_rows(e->cx, CF(0), CI32(1), F(2), I[0], IN(1), IN(2)); }},
    // ptrs W, dW, m, v; ints n; reals step, beta1, beta2, eps, grad_scale
    {"clamp_adam", 4, 1, 5,
     [](Engine* e, void* const* P, const int64_t* I, const double* X) {
       clamp_adam(e->cx, F(0), F(1), F(2), F(3), I[0], (float)X[0], (float)X[1], (float)X[2], (float)X[3], (float)X[4]);
     }},
};

#undef F
#undef CF
#undef I32
#undef CI32
#undef H16
#undef CH16
#undef IN
#undef DROP

}  // namespace

void test_kernel(Engine* e, const char* name, void* const* ptrs, int n_ptrs, const int64_t* ints, int n_ints, const double* reals,
                 int n_reals) {
  VD_REQUIRE(name != nullptr, VD_E_BADARG, "vd_test_kernel: name is null");
  for (const Entry& t : TABLE) {
    if (strcmp(t.name, name) != 0) continue;
    VD_REQUIRE(n_ptrs == t.n_ptrs && n_ints == t.n_ints && n_reals == t.n_reals, VD_E_BADARG, "vd_test_kernel: argument counts");
    VD_REQUIRE((n_ptrs == 0 || ptrs) && (n_ints == 0 || ints) && (n_reals == 0 || reals), VD_E_BADARG,
               "vd_test_kernel: null argument array");
    const Arena::Mark mk = e->arena.mark();
    t.fn(e, ptrs, ints, reals);
    VD_CUDA_CHECK(cudaStreamSynchronize(e->cx.stream));
    if (e->cx.deterministic) e->arena.rewind(mk);   // the deterministic routes' partial sums
    return;
  }
  throw CudaError(VD_E_BADARG, std::string("vd_test_kernel: unknown kernel ") + name);
}

}  // namespace vd
