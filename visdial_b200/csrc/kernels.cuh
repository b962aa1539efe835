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
                      const int32_t* tgt, const int32_t* row_ids, const float* lse, float* C, int64_t ldc,
                      const float* row_scale = nullptr);   // row_scale: C[m,:] *= row_scale[m] (null: today's epilogue)
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
// LookupTable accGradParameters: demb[ids[r],:] += dx[r,0:E] * dropfactor; pad rows privatised per block.  Deterministic
// mode: group_rows_by_token's stable sort of the ids (in [0, nv)) and a segmented sum in row order, without atomics.
void embed_scatter_add(LaunchCtx& cx, float* demb, const float* dx, int64_t ldx, const int32_t* ids,
                       int64_t rows, int E, DropCfg d, uint32_t site, int nv);

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
// rounds [r0, r1) only (a dialog session: [r, r+1)): q / hAtt (B*(r1-r0), H), the facts of dialog b rows 0..r1-1 of
// h + b*hpitch, probs (B, r1-r0, R); row r of the full form's output, bit for bit.  slot / round (device, B; a dialog
// pool's ask): row b alone at round round[b] over the facts of dialog slot[b] (h + slot[b]*hpitch), probs (B, 1, R); r0, r1
// are not read
void mn_attention_rows_fwd(LaunchCtx& cx, const float* q, const float* h, int64_t hpitch, float* probs, float* hAtt, int B,
                           int R, int H, int r0, int r1, const int32_t* slot = nullptr, const int32_t* round = nullptr);
void mn_attention_bwd(LaunchCtx& cx, const float* q, const float* h, const float* probs, const float* dhAtt,
                      float* dq, float* dh, int B, int R, int H);
// hrea-ques-im-hist.lua:89-129 + MaskFuture.lua + ReplaceZero.lua
void hrea_attention_fwd(LaunchCtx& cx, const float* sq, const float* sh, const float* Hs, float* probs, float* att,
                        int B, int R, int H);
// rounds [r0, r1) as mn_attention_rows_fwd: sq / att rows B*(r1-r0), sh (B, R), Hs rows of dialog b at Hs + b*hpitch;
// slot / round as there (sh then has a row per dialog, read at slot[b])
void hrea_attention_rows_fwd(LaunchCtx& cx, const float* sq, const float* sh, const float* Hs, int64_t hpitch, float* probs,
                             float* att, int B, int R, int H, int r0, int r1, const int32_t* slot = nullptr,
                             const int32_t* round = nullptr);
// a dialog session's cache write, one launch for every piece given (each destination null with its source):
//   h3 (B, H) -> facts (dialogs, R, H) at row (slot[b], round[b]); sh (B) -> shc (dialogs, R) at the same place;
//   hn / cn (B, H) -> st_h / st_c (dialogs, H) at row slot[b] (the dialog LSTM's carried state).
// slot null: dialog b; round null: round r.
void dialog_cache_write(LaunchCtx& cx, float* facts, float* shc, const float* h3, const float* sh, int64_t B, int R, int H, int r,
                        const int32_t* slot = nullptr, const int32_t* round = nullptr, float* st_h = nullptr, float* st_c = nullptr,
                        const float* hn = nullptr, const float* cn = nullptr);
// A dialog pool's ask gather, one launch: asked row b is conversation slot[b] at its round round[b] (device, n).
//   q (n, Tq) right-aligned questions -> the question cache ques (slots, R, Tq) at (slot, round), and ids_q (Tq, n);
//   the history cache hist (slots, R, W) at (slot, round) -> ids_h (W, n) (ids_h null: no history);
//   img (slots, img_cols) -> img_out (n, img_cols) (img_out null: no image product);
//   the dialog-LSTM state h / c (slots, H) -> h_out / c_out (n, H), zeros where round is 0 (h_out null: none).
struct DialogGather {
  int64_t n = 0; int R = 0;
  const int32_t *slot = nullptr, *round = nullptr;
  const int32_t* q = nullptr; int Tq = 0; int32_t *ques = nullptr, *ids_q = nullptr;
  const int32_t* hist = nullptr; int W = 0; int32_t* ids_h = nullptr;
  const float* img = nullptr; int64_t img_cols = 0; float* img_out = nullptr;
  const float *h = nullptr, *c = nullptr; int H = 0; float *h_out = nullptr, *c_out = nullptr;
};
void dialog_gather(LaunchCtx& cx, const DialogGather& g);
// dst row slot[i] <- src row i (n, cols): a join's image products into the joined slots
void scatter_rows(LaunchCtx& cx, float* dst, const float* src, const int32_t* slot, int64_t n, int64_t cols);
void hrea_attention_bwd(LaunchCtx& cx, const float* sq, const float* sh, const float* Hs, const float* probs,
                        const float* datt, float* dsq, float* dsh, float* dHs, int B, int R, int H);
// MaskTime.lua:12-28 + JoinTable(-1) (hrea-ques-im-hist.lua:52-55,67-69)
void masktime_concat_fwd(LaunchCtx& cx, float* out, const float* wemb, const float* img, const int32_t* ids_tm,
                         int T, int64_t N, int E, int I);
void masktime_bwd(LaunchCtx& cx, const float* dx, int64_t ldx, int off, const int32_t* ids_tm, float* dimg,
                  int T, int64_t N, int I);

// ---- SAN spatial attention (mn-att-ques-im-hist.lua:67-106) ---------------------------------------
// cnt (region features, DESIGN §26): null = every position attended; else (N / R) per-dialog counts c in [1, P], row n
// attends over positions 0 .. cnt[n / R] - 1 and the pad positions' outputs are zeros (san_collapse_bwd: cnt (B)).
void san_expand_dropout(LaunchCtx& cx, float* img_tr, const float* t, int B, int R, int P, int H, DropCfg d, uint32_t site);
void san_score_fwd(LaunchCtx& cx, const float* img_common, const float* ques_common, const float* w, const float* b,
                   float* s, int64_t N, int P, int Cm, DropCfg d, uint32_t site, const int32_t* cnt = nullptr, int R = 1);
void san_softmax_att_fwd(LaunchCtx& cx, const float* s, float* p, const float* img_tr, const float* u_in, float* u_out,
                         int64_t N, int P, int H, const int32_t* cnt = nullptr, int R = 1);
void san_att_bwd(LaunchCtx& cx, const float* du, const float* p, const float* img_tr, float* ds, float* dimg_tr,
                 int64_t N, int P, int H, const int32_t* cnt = nullptr, int R = 1);
void san_score_bwd(LaunchCtx& cx, const float* ds, const float* img_common, const float* ques_common, const float* w,
                   float* d_img_common, float* d_ques_common, float* dw, float* db, int64_t N, int P, int Cm,
                   DropCfg d, uint32_t site, const int32_t* cnt = nullptr, int R = 1);
void san_collapse_bwd(LaunchCtx& cx, const float* dimg_tr, const float* t, float* dt_pre, int B, int R, int P, int H,
                      DropCfg d, uint32_t site, const int32_t* cnt = nullptr);

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
// (lse, when not null, receives logsumexp(logits[r,:]) of the kept rows)
void lhood_accumulate(LaunchCtx& cx, const float* logits, const int32_t* tgt, const int32_t* mask_ids, float* lh,
                      int64_t rows, int V, float* lse = nullptr);
// nll_bwd on raw logits with a per-row factor: dlogits[r,:] = keep ? scale[r] * (exp(logits[r,:] - lse[r]) - onehot) : 0
// (the dense gen step's rows route; dlogits may alias logits)
void nll_bwd_scaled(LaunchCtx& cx, const float* logits, const float* lse, const int32_t* tgt, const int32_t* mask_ids,
                    const float* scale, float* dlogits, int64_t rows, int V);
// dst[i] = alpha * src[i]
void scale_copy(LaunchCtx& cx, float* dst, const float* src, int64_t n, float alpha);

// beam search on the device (model.lua:510-570): state shuffle by parent index
void beam_gather(LaunchCtx& cx, float* dst, const float* out_prev, const float* in_prev, const int32_t* parent, int64_t rows, int H);
// the k <= 32 best log-probabilities per row and their classes (value desc, class asc), never writing the log-probabilities:
// lse from the same row_lse as logsoftmax_rows, so the values are logsoftmax_rows' bits
// ar (DESIGN §25): the answer rules' barred classes take no part; entries past a row's allowed count are (-inf, -1)
void logsoftmax_topk_rows(LaunchCtx& cx, const float* logits, const int32_t* mask_ids, int64_t rows, int V, int k, float* topv,
                          int32_t* topi, const AnswerRules* ar = nullptr);
// the whole search on the device (Engine::gen_beam_search): beams (rows, L) = <start> then pads, tokens = <start>, scores = 0
void beam_init(LaunchCtx& cx, int64_t rows, int L, int start_token, int32_t* beams, int32_t* tokens, double* scores);
// Each group's list of its n best finished hypotheses (DESIGN §24), ordered by (norm desc, step asc, candidate asc), norm =
// score / lp(length - 1).  The merge keeps the entries in slots: ans (N, G, n, L), len (N, G, n) (0: never filled; slots
// fill in order 0, 1, ..), score (N, G, n), norm (N, G, n), and ord (N, G, n) the slot at each list position.  At the last
// step it writes the lists in order to out_* (N, G, n, ...).  n = 1: the slot is the list, ord and out_* are null.
struct BeamLists {
  int nbest = 1;
  const double* lp = nullptr;     // lp[l], l = 0 .. L-1, or null: every lp is 1 (length penalty 0)
  int32_t* ans = nullptr; int32_t* len = nullptr; double* score = nullptr;
  double* norm = nullptr;         // null (only with lp null): the norm is the score
  int32_t* ord = nullptr;
  int32_t* out_ans = nullptr; int32_t* out_len = nullptr; double* out_score = nullptr; double* out_norm = nullptr;
};
// the candidate merge of step stp for N rounds of k hypotheses in G groups of k / G (model.lua:529-569; diverse beam search
// with Hamming diversity lam for G > 1, DESIGN §22): next beams / scores / tokens / parents, and each group's list of
// finished hypotheses (DESIGN §24; n = 1, lp null: its best finished hypothesis, len 0 while there is none).  pick_* (N, L),
// (N), (N) or all null: at the last step (stp == L - 1), the best of each round's G list heads by (norm desc, group asc)
void beam_merge(LaunchCtx& cx, int64_t N, int stp, int k, int G, float lam, int L, int end_token, const float* topv,
                const int32_t* topi, const double* scores_in, double* scores_out, const int32_t* beams_in, int32_t* beams_out,
                int32_t* tokens, int32_t* parent, const BeamLists& lists, int32_t* pick_ans, int32_t* pick_len,
                double* pick_score, bool skip_empty = false);   // skip_empty: -inf entries are no candidates (DESIGN §25)
// the sampling step from materialised logits, one block per row: lse from the same row_lse as logsoftmax_rows (so logp is
// the bits it would give), the Gumbel-max draw of common.cuh; writes as vocab_sample_finish
// ar (DESIGN §25): the answer rules' barred classes take no part in the draw
void logsoftmax_sample_rows(LaunchCtx& cx, const float* logits, int64_t rows, int V, const SampleCfg& smp, int L, int32_t* tokens,
                            int32_t* answer, float* logp, const AnswerRules* ar = nullptr);
// its truncated form (common.cuh's TruncCfg rule, DESIGN §23): the same draw over the top-k / top-p prefix of each row, logp
// still logsoftmax_rows' bits.  V <= TRUNC_MAX_V (the row is staged in shared memory); VD_E_BADARG otherwise, or for
// top_k < 0 or top_p outside (0, 1].
void truncated_sample_rows(LaunchCtx& cx, const float* logits, int64_t rows, int V, const SampleCfg& smp, const TruncCfg& tr,
                           int L, int32_t* tokens, int32_t* answer, float* logp, const AnswerRules* ar = nullptr);
// the dialog loop's history (Engine::gen_dialog), one CTA per dialog b of hist (B, R, W), right-aligned rows.
// r < 0: row 0 <- row b*R of src (B*R, src_w), right-aligned into W >= src_w; rows 1.. <- pads.
// r >= 0: row r+1 <- round r's write (DESIGN §17): Q = the words of question row b*R + r of src (B*R, src_w), A = the first
// max_ans_len non-pad words of ans + b*ans_ld before the first end_token, of ans_len[b] - 2 words (ans_len null: ans_max);
// an empty Q empties A.  Per-round: Q ++ A; concat: row r ++ <END> ++ Q ++ A; the rightmost W words.  An empty row r leaves
// row r+1 empty (rightAlign's break, utils.lua:20-22).
// slot (device, B; a dialog pool): CTA b writes dialog slot[b] of hist (and reads its question row slot[b]*R + round);
// r < 0 (a join) still reads src row b*R.  round (device, B): CTA b appends at round round[b] (r is then any value >= 0),
// and writes nothing at round R-1.
void hist_append(LaunchCtx& cx, int32_t* hist, int64_t B, int R, int W, int r, const int32_t* src, int src_w, const int32_t* ans,
                 int64_t ans_ld, const int32_t* ans_len, int ans_max, int end_token, int max_ans_len, bool concat,
                 const int32_t* slot = nullptr, const int32_t* round = nullptr);
// a dialog pool's resume (Engine::dialog_join_rounds): CTA i writes rows 1..rounds[i] of dialog slot[i] of hist, in order,
// by hist_append's rule from row 0 on.  Round j's question is row row0[j] + i of q (rows, src_w) (rows packed time-major,
// round j's a prefix block of the dialogs still going); its answer is row (i, j) of ans (n, R, Ta), left-aligned, pads not
// words, cut at end_token (hist_append's ans_len-null form).
void hist_prefill(LaunchCtx& cx, int32_t* hist, int64_t n, int R, int W, const int32_t* slot, const int32_t* rounds,
                  const int32_t* row0, const int32_t* q, int src_w, const int32_t* ans, int Ta, int end_token, int max_ans_len,
                  bool concat);

// ---- optimiser (model.lua:96-99, optim_updates.lua:62-91) ------------------------------------------
void clamp_adam(LaunchCtx& cx, float* W, float* dW, float* m, float* v, int64_t n, float step, float beta1,
                float beta2, float eps, float grad_scale);
void fill_l2_flush(LaunchCtx& cx, float* buf, int64_t n);
// deterministic mode (DESIGN §27): C[m, n] (row pitch ldc) += the sum over s = 0 .. S-1, in that order, of ws[s][m][n]
// (S slots of M x N, row pitch N) — the second pass of every reduction whose partial sums the first pass wrote to slots
void slot_reduce(LaunchCtx& cx, float* C, int64_t ldc, const float* ws, int S, int64_t M, int N);
// counting sort of rows by token id (perm = row indices grouped by token, sorted_tok = their ids) and the
// segmented row sum out[tok,:] += sum_{rows with that token} X[row,:]   (LookupTable accGradParameters in
// projected space: the embedding gradient of the option LSTM without a 640k x 300 x 2048 contraction).
// Deterministic mode: the sort is stable (a token's rows in index order) and the sum adds each token's rows in that order.
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
// one BPTT step t < T - 1 (k_lstm16_bptt over one step): dc_carry is read and overwritten in place
void lstm16_step_bwd(LaunchCtx& cx, int64_t R, int H, const __half* da_next16, const __half* Whb16, const __half* gates16,
                     const float* c_prev, const float* c_cur, float* dc_carry, const int32_t* mask_ids, __half* da16);
// BPTT steps T - 2 .. 0 of a saved run (da16: T slices of (R, 4H), slice T - 1 written by lstm16_bwd_last; gates16 likewise;
// c: T slices of (R, H); c0 the initial cell state or null; mask: T slices of R ids or null), in waves of clusters that each
// run one 128-row block through every step with the dc carry on chip
void lstm16_bptt(LaunchCtx& cx, int64_t R, int H, int T, __half* da16, const __half* Whb16, const __half* gates16, const float* c,
                 const float* c0, const int32_t* mask, float* dc_carry);
// its launch plan: clusters of csize = H / 128 CTAs, one per row block; `clusters` row blocks per launch (the last launch may
// take fewer), `waves` launches
struct Bptt16Plan { int csize, clusters, waves; };
Bptt16Plan lstm16_bptt_plan(LaunchCtx& cx, int64_t R, int H);
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
void segsum_rows16_det(LaunchCtx& cx, const __half* X, int64_t ldx, const int32_t* perm, const int32_t* sorted_tok, int64_t n,
                       float* out, int ncols, const float* inv_scale);   // segsum_rows16's deterministic route (pointwise.cu)
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
                       __half* da2_16, int* flags, float* dh1, float* dh2, float* scale);
int64_t enc_pair_bwd_flag_ints(int T, int64_t R, int H);
bool enc_pair_gate_split(int H);
}  // namespace vd

namespace vd {
// answer-pool retrieval (DESIGN §18; answer_pool.cu, gemm_tc.cu): per query row of Q (rows, H; row pitch ldq) the k <= 32 best
// rows of the pool embeddings E (m, H) by (score desc, index asc), score = Q[r] . E[j], never writing the (rows, m) scores.
// A route writes partial lists part_v / part_i (rows, slots, k), best first, (-inf, -1) = empty; pool_topk_merge reduces them.
struct PoolTcGeom { int num_n = 0; int64_t tiles = 0; int grid = 0, slots = 0; };
bool pool_tc_ok(int H, const float* Q, int64_t ldq, const float* E);          // the shapes the tensor-core route takes
PoolTcGeom pool_topk_tc_geom(const LaunchCtx& cx, int64_t rows, int64_t m);
void pool_topk_tc(LaunchCtx& cx, const PoolTcGeom& g, const float* Q, int64_t ldq, int64_t rows, const float* E, int64_t m, int H,
                  int k, float* part_v, int32_t* part_i);
int pool_topk_simt_slots(const LaunchCtx& cx, int64_t rows, int64_t m);
void pool_topk_simt(LaunchCtx& cx, int slots, const float* Q, int64_t ldq, int64_t rows, const float* E, int64_t m, int H, int k,
                    float* part_v, int32_t* part_i);
// tc_grid > 0: lists of the tensor-core route (geometry tc_num_n / tc_grid), of which only the walked ones are read
void pool_topk_merge(LaunchCtx& cx, const float* part_v, const int32_t* part_i, int64_t rows, int slots, int k, int tc_num_n,
                     int tc_grid, float* topv, int32_t* topi);
// out (n, w) <- pool_tok rows idx[b * idx_ld]
void gather_pool_rows(LaunchCtx& cx, const int32_t* pool_tok, int w, const int32_t* idx, int64_t idx_ld, int64_t n, int32_t* out);
}  // namespace vd
