// Kernel launchers of the visdial_b200 engine.  Every launcher cites the reference site it replaces
// (paths relative to /root/reference).  All tensors fp32 row-major; ids int32 (0 = pad).
#pragma once
#include <algorithm>
#include <cuda_fp16.h>
#include "common.cuh"

namespace vd {

// ---- dense contractions -----------------------------------------------------------------------
// C[m,n] = act(beta*C + bias[n] + sum_k A[row(m),k] B[n,k]).  act: 0 none, 1 tanh.
// Replaces nn.Linear / the SeqLSTM addmm pair [upstream]; fp32 CUDA-core version.
void gemm_tn_simt(LaunchCtx& cx, int M, int N, int K, const float* A, int64_t lda, const int32_t* a_gather,
                  const float* B, int64_t ldb, float* C, int64_t ldc, float beta, const float* bias, int act);
// C[m,n] += sum_k A[row(k),m] B[k,n]   (accGradParameters of Linear / SeqLSTM)
void gemm_atb_simt(LaunchCtx& cx, int M, int N, int64_t K, const float* A, int64_t lda, const int32_t* a_gather,
                   const float* B, int64_t ldb, float* C, int64_t ldc);
// wgmma / TMA versions (gemm_tc.cu); return false when the shape is not taken.
bool gemm_tn_tc(LaunchCtx& cx, int M, int N, int K, const float* A, int64_t lda, const int32_t* a_gather,
                const float* B, int64_t ldb, float* C, int64_t ldc, float beta, const float* bias, int act);
bool gemm_atb_tc(LaunchCtx& cx, int M, int N, int64_t K, const float* A, int64_t lda, const int32_t* a_gather,
                 const float* B, int64_t ldb, float* C, int64_t ldc);

// fused vocabulary softmax (gemm_tc.cu, pointwise.cu): the (rows, V) logits of decoders/gen.lua:21-24 never reach HBM
int vocab_lse_nparts(int N);
bool vocab_tc_ok(int M, int N, int K, const float* A, int64_t lda, const float* B, int64_t ldb);   // both halves take exactly this
bool vocab_lse_tc(LaunchCtx& cx, int M, int N, int K, const float* A, int64_t lda, const float* B, int64_t ldb, const float* bias,
                  const int32_t* tgt, float* part_max, float* part_sum, float* tgt_logit);
bool vocab_dlogits_tc(LaunchCtx& cx, int M, int N, int K, const float* A, int64_t lda, const float* B, int64_t ldb, const float* bias,
                      const int32_t* tgt, const int32_t* row_ids, const float* lse, float* C, int64_t ldc);
// lse[r] from the partials; then  out[r] (+)= keep ? sign * (tgt_logit[r] - lse[r]) : 0   (keep: row id != 0 and target > 0)
void vocab_lse_finish(LaunchCtx& cx, const float* part_max, const float* part_sum, int nparts, const float* tgt_logit,
                      const int32_t* tgt, const int32_t* row_ids, float* lse, float* out, float sign, int accumulate, int64_t rows);
// sampling (Engine::gen_sample, rule in common.cuh): the projection with the Gumbel-max draw in its epilogue (same shapes as
// vocab_lse_tc), then the reduction of the slices — lse as vocab_lse_finish forms it, the winner by (key desc, class asc) —
// which writes what every sampling route writes for step smp.step (1-based): tokens[r] = class + 1 (the next step's
// input), answer[r * (L + 1) + step] = the same, logp[r * L + step - 1] = x_tok - lse (logp may be null)
bool vocab_sample_tc(LaunchCtx& cx, int M, int N, int K, const float* A, int64_t lda, const float* B, int64_t ldb, const float* bias,
                     const SampleCfg& smp, float* part_max, float* part_sum, float* part_key, int32_t* part_cls, float* part_x);
void vocab_sample_finish(LaunchCtx& cx, const float* part_max, const float* part_sum, const float* part_key, const int32_t* part_cls,
                         const float* part_x, int nparts, int64_t rows, int step, int L, int32_t* tokens, int32_t* answer, float* logp);

// ---- ids / embedding ---------------------------------------------------------------------------
// (rows,T) batch-major -> (T,rows) time-major: the `view(-1,T):t()` of model.lua:256,276,308.
void transpose_ids(LaunchCtx& cx, const int32_t* src, int32_t* dst, int64_t rows, int T);
// dense fine-tuning (Engine::forward_backward_dense): one selected round per dialog, round[b] in [0, R).
// transpose_ids over the K option rows of round round[b] of each dialog b: src (B*R*K, T) -> dst (T, B*K)
void transpose_ids_rounds(LaunchCtx& cx, const int32_t* src, const int32_t* round, int32_t* dst, int64_t B, int R, int K, int T);
// dst (B,H) <- rows b*R + round[b] of src (B*R,H);  and back: a zeroed (B*R,H) dst with src's rows at b*R + round[b]
void gather_round_rows(LaunchCtx& cx, const float* src, const int32_t* round, float* dst, int64_t B, int R, int H);
void scatter_round_rows(LaunchCtx& cx, const float* src, const int32_t* round, float* dst, int64_t B, int R, int H);
// nn.LookupTableMaskZero forward (+ the nn.Dropout that follows it in mn-att-ques-im-hist.lua:24-25)
void embed_rows(LaunchCtx& cx, float* out, const float* emb, const int32_t* ids, int64_t rows, int E,
                DropCfg d, uint32_t site);
// LookupTable accGradParameters: demb[ids[r],:] += dx[r,0:E] * dropfactor; pad rows privatised per block.
void embed_scatter_add(LaunchCtx& cx, float* demb, const float* dx, int64_t ldx, const int32_t* ids,
                       int64_t rows, int E, DropCfg d, uint32_t site);

// ---- SeqLSTM pointwise halves (the GEMM halves are gemm_tn) --------------------------------------
// gates (R,4H) holds pre-activations without bias on entry, activated [i f o g] on exit.
void lstm_pointwise_fwd(LaunchCtx& cx, float* gates, const float* bias, const float* c_prev,
                        const int32_t* mask_ids, float* c_out, float* h_out, int64_t R, int H);
// first step of a sequence without initial state: no recurrent term, the pre-activation is the x-projection
// (in `gates`, or gathered from `ptable[tok]`), bias optional
void lstm_first_step_fwd(LaunchCtx& cx, float* gates, const float* ptable, const int32_t* tok, const float* bias,
                         const float* c_prev, const int32_t* mask_ids, float* c_out, float* h_out, int64_t R, int H);
// da (R,4H) out; dc_carry (R,H) in: dc from step t+1, out: dc for step t-1.
void lstm_pointwise_bwd(LaunchCtx& cx, const float* gates, const float* c_prev, const float* c,
                        const float* dh_rec, const float* dh_ext, const float* dc_ext, float* dc_carry,
                        const int32_t* mask_ids, float* da, int64_t R, int H);

// ---- small helpers -----------------------------------------------------------------------------
void colsum_add(LaunchCtx& cx, float* out, const float* X, int64_t rows, int cols, int64_t ldx);
void dropout_apply(LaunchCtx& cx, float* out, const float* in, int64_t n, DropCfg d, uint32_t site);
void tanh_bwd(LaunchCtx& cx, float* dpre, const float* dy, const float* y, int64_t n);
void add_inplace(LaunchCtx& cx, float* a, const float* b, int64_t n);
void add_out(LaunchCtx& cx, float* out, const float* a, const float* b, int64_t n);
void copy_cols(LaunchCtx& cx, float* dst, int64_t ldd, const float* src, int64_t lds, int64_t rows, int cols);
// model.lua:267-269: dst row n <- src row n / R; src rows lds apart (lds < 0: cols, contiguous)
void repeat_rows(LaunchCtx& cx, float* dst, const float* src, int64_t B, int R, int64_t cols, int64_t lds = -1);
void sum_repeated_rows(LaunchCtx& cx, float* dst, const float* src, int64_t B, int R, int64_t cols);
void transpose_segments(LaunchCtx& cx, const float* W, float* Wt, const int64_t* seg_table_dev, int nseg,
                        int64_t max_elems);
// out[r] = x[r,:].w + b  (nn.Linear(H,1)); bwd: dx[r,:] (+)= ds[r] w, dw += sum ds[r] x[r,:], db += sum ds
void rowdot_fwd(LaunchCtx& cx, float* out, const float* x, const float* w, const float* b, int64_t rows, int H);
void rowdot_bwd(LaunchCtx& cx, const float* ds, const float* x, const float* w, float* dx, int accumulate_dx,
                float* dw, float* db, int64_t rows, int H);

// ---- attention over history ----------------------------------------------------------------------
// mn-att-ques-im-hist.lua:48-62 + MaskSoftMax.lua (mask j>i generated in-kernel, model.lua:281-288)
void mn_attention_fwd(LaunchCtx& cx, const float* q, const float* h, float* probs, float* hAtt, int B, int R, int H);
void mn_attention_bwd(LaunchCtx& cx, const float* q, const float* h, const float* probs, const float* dhAtt,
                      float* dq, float* dh, int B, int R, int H);
// hrea-ques-im-hist.lua:89-129 + MaskFuture.lua + ReplaceZero.lua
void hrea_attention_fwd(LaunchCtx& cx, const float* sq, const float* sh, const float* Hs, float* probs, float* att,
                        int B, int R, int H);
void hrea_attention_bwd(LaunchCtx& cx, const float* sq, const float* sh, const float* Hs, const float* probs,
                        const float* datt, float* dsq, float* dsh, float* dHs, int B, int R, int H);
// MaskTime.lua:12-28 + JoinTable(-1) (hrea-ques-im-hist.lua:52-55,67-69)
void masktime_concat_fwd(LaunchCtx& cx, float* out, const float* wemb, const float* img, const int32_t* ids_tm,
                         int T, int64_t N, int E, int I);
void masktime_bwd(LaunchCtx& cx, const float* dx, int64_t ldx, int off, const int32_t* ids_tm, float* dimg,
                  int T, int64_t N, int I);

// ---- SAN spatial attention (mn-att-ques-im-hist.lua:67-106) ---------------------------------------
void san_expand_dropout(LaunchCtx& cx, float* img_tr, const float* t, int B, int R, int P, int H, DropCfg d, uint32_t site);
void san_score_fwd(LaunchCtx& cx, const float* img_common, const float* ques_common, const float* w, const float* b,
                   float* s, int64_t N, int P, int Cm, DropCfg d, uint32_t site);
void san_softmax_att_fwd(LaunchCtx& cx, const float* s, float* p, const float* img_tr, const float* u_in, float* u_out,
                         int64_t N, int P, int H);
void san_att_bwd(LaunchCtx& cx, const float* du, const float* p, const float* img_tr, float* ds, float* dimg_tr,
                 int64_t N, int P, int H);
void san_score_bwd(LaunchCtx& cx, const float* ds, const float* img_common, const float* ques_common, const float* w,
                   float* d_img_common, float* d_ques_common, float* dw, float* db, int64_t N, int P, int Cm,
                   DropCfg d, uint32_t site);
void san_collapse_bwd(LaunchCtx& cx, const float* dimg_tr, const float* t, float* dt_pre, int B, int R, int P, int H,
                      DropCfg d, uint32_t site);

// ---- decoders / criterions / ranks ---------------------------------------------------------------
// disc.lua:22-29  scores[n,k] = feat[n,k,:] . encOut[n,:]
void disc_scores_fwd(LaunchCtx& cx, const float* feat, const float* encOut, float* scores, int64_t N, int K, int H);
void disc_scores_bwd(LaunchCtx& cx, const float* dscores, const float* feat, const float* encOut, float* dfeat,
                     float* dencOut, int64_t N, int K, int H);
// nn.CrossEntropyCriterion (model.lua:38,330,334): mean over rows; writes loss[0] and dscores
void xent_fwd(LaunchCtx& cx, const float* scores, const int32_t* gt, float* row_loss, int64_t N, int K);
void xent_bwd(LaunchCtx& cx, const float* scores, const int32_t* gt, float* dscores, int64_t N, int K);
// soft-target cross-entropy over rows with relevance rel >= 0 (positive row sums): p = rel / sum(rel),
// row_loss[n] = lse(s_n) - sum_k p_k s_nk,  dscores = (softmax(s_n) - p_n) / N
void soft_xent(LaunchCtx& cx, const float* scores, const float* rel, float* row_loss, float* dscores, int64_t N, int K);
void reduce_sum(LaunchCtx& cx, const float* x, float* out, int64_t n, float scale);
// utils.computeRanks (utils.lua:106-128); tie rule: lower index wins
void rank_rows(LaunchCtx& cx, const float* scores, const int32_t* gt, int32_t* ranks, int64_t N, int K);
// gen.lua:23-24: rows with mask id 0 are zeroed (MaskZero), others log_softmax in place
void logsoftmax_rows(LaunchCtx& cx, float* logits, const int32_t* mask_ids, int64_t rows, int V);
// model.lua:33-36 criterion: row_loss[r] = -logp[r,tgt-1] for kept rows; dlogits = exp(logp) - onehot
void nll_fwd(LaunchCtx& cx, const float* logp, const int32_t* tgt, const int32_t* mask_ids, float* row_loss, int64_t rows, int V);
void nll_bwd(LaunchCtx& cx, const float* logp, const int32_t* tgt, const int32_t* mask_ids, float* dlogits, int64_t rows, int V);
// utils.computeLhood (utils.lua:86-102) from raw logits: lh[r] += logits[r,tgt-1] - logsumexp(logits[r,:])
void lhood_accumulate(LaunchCtx& cx, const float* logits, const int32_t* tgt, const int32_t* mask_ids, float* lh,
                      int64_t rows, int V);

// beam search on the device (model.lua:510-570): state shuffle by parent index
void beam_gather(LaunchCtx& cx, float* dst, const float* out_prev, const float* in_prev, const int32_t* parent, int64_t rows, int H);
// the k <= 32 best log-probabilities per row and their classes (value desc, class asc), never writing the log-probabilities:
// lse from the same row_lse as logsoftmax_rows, so the values are logsoftmax_rows' bits
void logsoftmax_topk_rows(LaunchCtx& cx, const float* logits, const int32_t* mask_ids, int64_t rows, int V, int k, float* topv,
                          int32_t* topi);
// the whole search on the device (Engine::gen_beam_search): beams (rows, L) = <start> then pads, tokens = <start>, scores = 0
void beam_init(LaunchCtx& cx, int64_t rows, int L, int start_token, int32_t* beams, int32_t* tokens, double* scores);
// the candidate merge of step stp for N rounds of k hypotheses (model.lua:529-569): next beams / scores / tokens / parents,
// and each round's best finished hypothesis (ans (N, L), ans_len (N) = 0 while there is none, ans_score (N))
void beam_merge(LaunchCtx& cx, int64_t N, int stp, int k, int L, int end_token, const float* topv, const int32_t* topi,
                const double* scores_in, double* scores_out, const int32_t* beams_in, int32_t* beams_out, int32_t* tokens,
                int32_t* parent, int32_t* ans, int32_t* ans_len, double* ans_score);
// the sampling step from materialised logits, one block per row: lse from the same row_lse as logsoftmax_rows (so logp is
// the bits it would give), the Gumbel-max draw of common.cuh; writes as vocab_sample_finish
void logsoftmax_sample_rows(LaunchCtx& cx, const float* logits, int64_t rows, int V, const SampleCfg& smp, int L, int32_t* tokens,
                            int32_t* answer, float* logp);
// the dialog loop's history (Engine::gen_dialog), one CTA per dialog b of hist (B, R, W), right-aligned rows.
// r < 0: row 0 <- row b*R of src (B*R, src_w), right-aligned into W >= src_w; rows 1.. <- pads.
// r >= 0: row r+1 <- round r's write (DESIGN §17): Q = the words of question row b*R + r of src (B*R, src_w), A = the first
// max_ans_len non-pad words of ans + b*ans_ld before the first end_token, of ans_len[b] - 2 words (ans_len null: ans_max);
// an empty Q empties A.  Per-round: Q ++ A; concat: row r ++ <END> ++ Q ++ A; the rightmost W words.  An empty row r leaves
// row r+1 empty (rightAlign's break, utils.lua:20-22).
void hist_append(LaunchCtx& cx, int32_t* hist, int64_t B, int R, int W, int r, const int32_t* src, int src_w, const int32_t* ans,
                 int64_t ans_ld, const int32_t* ans_len, int ans_max, int end_token, int max_ans_len, bool concat);

// ---- optimiser (model.lua:96-99, optim_updates.lua:62-91) ------------------------------------------
void clamp_adam(LaunchCtx& cx, float* W, float* dW, float* m, float* v, int64_t n, float step, float beta1,
                float beta2, float eps, float grad_scale);
void fill_l2_flush(LaunchCtx& cx, float* buf, int64_t n);
// counting sort of rows by token id (perm = row indices grouped by token, sorted_tok = their ids) and the
// segmented row sum out[tok,:] += sum_{rows with that token} X[row,:]   (LookupTable accGradParameters in
// projected space: the embedding gradient of the option LSTM without a 640k x 300 x 2048 contraction)
void group_rows_by_token(LaunchCtx& cx, const int32_t* ids, int64_t n, int nv, int32_t* scratch3nv, int32_t* perm,
                         int32_t* sorted_tok);
void segsum_rows(LaunchCtx& cx, const float* X, int64_t ldx, const int32_t* perm, const int32_t* sorted_tok, int64_t n,
                 float* out, int ncols);

}  // namespace vd

namespace vd {
// fused SeqLSTM steps on the tensor cores (gemm_tc.cu); return false when the shape is not taken.  The *_ok predicates
// are the weight / width conditions of those decisions, for the engine to route with; *tile receives the tile width.
bool lstm_step_fwd_tc_ok(int H, const float* WtS_h, int64_t ldw);
bool lstm_step_bwd_tc_ok(int H, const float* Wh);
bool lstm_step_fwd_tc(LaunchCtx& cx, int64_t R, int H, const float* h_prev, const float* WtS_h, int64_t ldw, const float* bias,
                      float* gates, int has_xproj, const float* ptable, const int32_t* tok, const float* c_prev, float* c_out,
                      float* h_out, const int32_t* mask_ids, int* tile = nullptr);
bool lstm_step_bwd_tc(LaunchCtx& cx, int64_t R, int H, const float* da_next, const float* Wh, const float* gsave,
                      const float* c_prev, const float* c_cur, const float* dh_ext, float* dc_carry, const int32_t* mask_ids,
                      float* da, int* tile = nullptr);
}  // namespace vd

namespace vd {
// VD_MATH_F16 (lstm16.cu): SeqLSTM over many rows with fp16 operands / fp16 saved state, fp32 accumulation and cell state
bool lstm16_shape_ok(int64_t R, int H);
void lstm16_step_fwd(LaunchCtx& cx, int64_t R, int H, const __half* h_prev16, const __half* Wh16, const __half* ptable16,
                     const int32_t* tok, const float* bias, const float* c_prev, const int32_t* mask_ids, __half* gates16,
                     float* c_out, __half* h16_out, float* h32_out);
void lstm16_step_bwd(LaunchCtx& cx, int64_t R, int H, const __half* da_next16, const __half* Whb16, const __half* gates16,
                     const float* c_prev, const float* c_cur, float* dc_carry, const int32_t* mask_ids, __half* da16);
void lstm16_first_step(LaunchCtx& cx, int64_t R, int H, const __half* ptable16, const int32_t* tok, const float* bias,
                       const float* c_prev, const int32_t* mask_ids, __half* gates16, float* c_out, __half* h16_out, float* h32_out);
void lstm16_bwd_last(LaunchCtx& cx, int64_t R, int H, const __half* gates16, const float* c_prev, const float* c_cur,
                     const float* dh_last, const float* scale, const int32_t* mask_ids, float* dc_carry, __half* da16);
// round to nearest even, saturating: |x| > 65504 (inf included) becomes +-65504, NaN stays NaN (cvt.rn.satfinite)
void cvt_f32_to_f16(LaunchCtx& cx, __half* dst, int64_t ldd, const float* src, int64_t lds, int64_t rows, int cols);
// scale2 = {s, 1/s}: the power of two s = 2^clamp(10 - e, -60, 60) with max|x| = f 2^e, f in [1/2, 1), so max|x| s lies
// in [2^9, 2^10); s = 1 when max|x| is 0 or infinite.  NaN elements do not take part in the maximum (fmaxf).
void pick_grad_scale(LaunchCtx& cx, const float* x, int64_t n, uint32_t* bits, float* scale2);
void segsum_rows16(LaunchCtx& cx, const __half* X, int64_t ldx, const int32_t* perm, const int32_t* sorted_tok, int64_t n,
                   float* out, int ncols, const float* inv_scale);
void gemm_atb16(LaunchCtx& cx, int M, int N, int64_t K, const __half* A, int64_t lda, const __half* B, int64_t ldb, float* C,
                int64_t ldc, const float* inv_scale);
// persistent two-layer SeqLSTM of the few-row encoder LSTMs (enc_lstm.cu): one launch for both layers and all T steps
bool enc_pair_shape_ok(int64_t R, int H, int sm_count);
void enc_pair_forward(LaunchCtx& cx, int T, int64_t R, int H, const __half* W1h16, const __half* W2cat16, const float* bias2,
                      const int32_t* mask, float* gates1, float* c1, float* h1, __half* h1_16, float* gates2, float* c2, float* h2,
                      __half* h2_16, int* flags);
void enc_pair_backward(LaunchCtx& cx, int T, int64_t R, int H, const __half* B1cat16, const __half* Whb2_16, const int32_t* mask,
                       const float* gates1, const float* c1, const float* gates2, const float* c2, const float* dh_last1,
                       const float* dc_last1, const float* dh_last2, const float* dc_last2, float* da1, __half* da1_16, float* da2,
                       __half* da2_16, int* flags, float* dh1, float* dh2);
int64_t enc_pair_bwd_flag_ints(int T, int64_t R, int H);
bool enc_pair_gate_split(int H);
}  // namespace vd
