// vd_test_kernel: the kernels.cuh launchers of pointwise.cu and lstm16.cu's streaming helpers, called by name on
// caller-provided DEVICE buffers on the engine's LaunchCtx, so that grid, shared-memory attribute and route are the
// engine's own.  The table below is the whole surface: name, pointer / int / real counts, and the call.
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
#define IN(i) ((int)I[i])
#define DROP(k) e->dropcfg((float)X[k])

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
    // ptrs logits, tokens, answer, logp; ints rows, V, L, seed, step, row_offset, row_stride; reals temperature
    {"logsoftmax_sample_rows", 4, 7, 1,
     [](Engine* e, void* const* P, const int64_t* I, const double* X) {
       SampleCfg s;
       s.seed_lo = (uint32_t)(uint64_t)I[3]; s.seed_hi = (uint32_t)((uint64_t)I[3] >> 32); s.step = (uint32_t)I[4];
       s.temperature = (float)X[0]; s.row_offset = I[5]; s.row_stride = I[6];
       logsoftmax_sample_rows(e->cx, CF(0), I[0], IN(1), s, IN(2), I32(1), I32(2), F(3));
     }},
    // ---- embedding and token grouping
    {"embed_rows", 3, 3, 1,
     [](Engine* e, void* const* P, const int64_t* I, const double* X) {
       embed_rows(e->cx, F(0), CF(1), CI32(2), I[0], IN(1), DROP(0), (uint32_t)I[2]);
     }},
    {"embed_scatter_add", 3, 4, 1,
     [](Engine* e, void* const* P, const int64_t* I, const double* X) {
       embed_scatter_add(e->cx, F(0), CF(1), I[0], CI32(2), I[1], IN(2), DROP(0), (uint32_t)I[3]);
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
    {"segsum_rows16", 5, 3, 0,
     [](Engine* e, void* const* P, const int64_t* I, const double*) {
       segsum_rows16(e->cx, static_cast<const __half*>(P[0]), I[0], CI32(1), CI32(2), I[1], F(3), IN(2), CF(4));
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
    t.fn(e, ptrs, ints, reals);
    VD_CUDA_CHECK(cudaStreamSynchronize(e->cx.stream));
    return;
  }
  throw CudaError(VD_E_BADARG, std::string("vd_test_kernel: unknown kernel ") + name);
}

}  // namespace vd
