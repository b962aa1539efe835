/*
 * visdial_b200 — C ABI of the H100-native Visual Dialog encoder/decoder engine.
 *
 * This is the drop-in boundary for the reference's per-batch hot path.  Every entry point cites
 * the reference interface it replaces (paths relative to /root/reference).  Host languages bind it
 * directly: LuaJIT `ffi.cdef` (see INTEGRATION.md and lua/), Python ctypes (visdial_b200/_lib.py).
 *
 * Conventions
 *  - every call returns int: 0 = ok, <0 = error class (VD_E_*); message via vd_last_error().
 *    No exceptions cross the ABI, nothing calls exit().  (The reference's error()/assert kill the
 *    CLI: model.lua:436, weight-init.lua:46; the Lua shim turns rc != 0 into error(msg).)
 *  - all tensors fp32; token / class ids int32, 1-based with 0 = pad, exactly as the reference
 *    dataloader emits them (dataloader.lua:143-321; on GPU the reference stores them as fp32).
 *  - batch tensors are passed BATCH-MAJOR as the dataloader hands them to Model:forwardBackward
 *    (model.lua:255-311 only re-views them time-major; the engine does that indexing itself).
 *  - one engine <-> one device <-> one non-default stream; an engine is single-caller.
 *  - pointers returned by the engine (parameters, outputs) are DEVICE pointers that stay valid for
 *    the engine's lifetime (outputs: until the next call that produces the same output).
 */
#ifndef VISDIAL_B200_H
#define VISDIAL_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VD_OK 0
#define VD_E_BADARG (-1)   /* null pointer, unknown encoder/decoder name, bad flag            */
#define VD_E_SHAPE (-2)    /* batch sizes inconsistent with params                             */
#define VD_E_CUDA (-3)     /* CUDA runtime / launch failure                                    */
#define VD_E_COMM (-4)     /* NCCL failure                                                     */
#define VD_E_OOM (-5)      /* device allocation failed                                         */
#define VD_E_STATE (-6)    /* call order violated (backward before forward, ...)               */

typedef struct vd_engine vd_engine;

/* modelParams (opts.lua:6-40, train.lua:55-59, evaluate.lua:72-75).  Field names are the
 * reference's.  useHistory / useIm / concatHistory are derived from `encoder` by substring match
 * exactly as opts.lua:55-59 does. */
typedef struct vd_params {
  const char* encoder;          /* 'lf-ques' | 'lf-ques-im-hist' | 'hrea-ques-im-hist' | 'mn-att-ques-im-hist' */
  const char* decoder;          /* 'disc' | 'gen' */
  int32_t vocabSize;            /* V, incl. <START>=V-1 and <END>=V; the embedding has V+1 rows */
  int32_t embedSize;            /* 300 */
  int32_t rnnHiddenSize;        /* 512 */
  int32_t numLayers;            /* 2 (the only value the configured graphs are built for) */
  int32_t imgFeatureSize;       /* 4096 (fc7) or 512 (pool5 channels) */
  int32_t imgSpatialSize;       /* 14 */
  int32_t imgEmbedSize;         /* 300 */
  int32_t commonEmbeddingSize;  /* 512 */
  int32_t numAttentionLayers;   /* 1 */
  int32_t maxQuesCount;         /* 10 rounds */
  int32_t numOptions;           /* 100 */
  float dropout;                /* 0.5; used by the LF graphs, MN/att/HREA hard-code 0.5 */
  int32_t gpuid;                /* CUDA device ordinal */
} vd_params;

/* A batch as produced by dataloader:getTrainBatch / getTestBatch (dataloader.lua:324-478),
 * Appendix A of SURVEY.md.  Unused pointers may be NULL.  N = B * maxQuesCount. */
typedef struct vd_batch {
  int32_t B;                    /* dialogs ("threads") in this batch */
  int32_t Tq, Th, Ta, To;       /* trimmed question / history / answer(+1) / option widths */
  const int32_t* ques_fwd;      /* (B,10,Tq) right-aligned */
  const int32_t* hist;          /* (B,10,Th) right-aligned */
  const float* img_feat;        /* (B,F) fc7 or (B,S,S,C) NHWC pool5 — one row per dialog */
  const int32_t* options;       /* disc: (N,100,To) left-aligned raw option tokens */
  const int32_t* answer_ind;    /* (N) 1-based ground-truth option */
  const int32_t* answer_in;     /* gen: (B,10,Ta) <START> a.. 0.. */
  const int32_t* answer_out;    /* gen: (B,10,Ta) a.. <END> 0.. */
  const int32_t* option_in;     /* gen eval: (B,10,100,To) */
  const int32_t* option_out;    /* gen eval: (B,10,100,To) */
  int32_t on_device;            /* 0: host pointers (staged + copied H2D by the engine), 1: device */
} vd_batch;

/* ---- parameter layout: host-only, needs no GPU --------------------------------------------- */
/* Replaces nn.Module:getParameters() flattening (model.lua:55).  Segment order = DESIGN.md §3. */
#define VD_INIT_EMBED 0       /* N(0,1)                       [upstream nn.LookupTable]            */
#define VD_INIT_LINEAR_W 1    /* U(-1/sqrt(in), 1/sqrt(in))   [upstream nn.Linear]                 */
#define VD_INIT_LINEAR_B 2    /* U(-1/sqrt(in), 1/sqrt(in))                                        */
#define VD_INIT_LSTM_W 3      /* N(0, 1/sqrt(D+H))            [upstream rnn.SeqLSTM]               */
#define VD_INIT_LSTM_B 4      /* 0, forget block (cols H..2H) = 1                                  */
int vd_layout_count(const vd_params* p, int32_t* n_segments, int64_t* n_params);
int vd_layout_segment(const vd_params* p, int32_t idx, char* name, int32_t name_cap,
                      int64_t* offset, int64_t* rows, int64_t* cols, int32_t* init_kind,
                      int64_t* fan_in);

/* ---- lifetime ------------------------------------------------------------------------------ */
/* encoder.model(params) + decoder.model(params, enc) + nn.Sequential wrapper + :cuda()
 * (model.lua:19-55). */
int vd_create(const vd_params* p, vd_engine** out);
int vd_destroy(vd_engine* e);
const char* vd_last_error(void);

/* ---- parameters (wrapperW / wrapperdW, model.lua:55) --------------------------------------- */
int vd_num_params(vd_engine* e, int64_t* n);
int vd_param_buffers(vd_engine* e, float** W_dev, float** dW_dev);
int vd_optim_buffers(vd_engine* e, float** m_dev, float** v_dev, int64_t* t);
/* restore Adam's state table (optims.m / .v / .t of model_utils/optim_updates.lua:67-84) from HOST vectors of
 * vd_num_params floats — resuming from a checkpoint written by train.lua:99-102 */
int vd_set_optim_state(vd_engine* e, const float* m_host, const float* v_host, int64_t t);
int vd_set_parameters(vd_engine* e, const float* host_src, int64_t n);   /* wrapperW:copy(modelW), evaluate.lua:91 */
int vd_get_parameters(vd_engine* e, float* host_dst, int64_t n);
int vd_get_gradients(vd_engine* e, float* host_dst, int64_t n);
int vd_zero_grad(vd_engine* e);                                          /* wrapper:zeroGradParameters(), model.lua:68 */

/* ---- modes ---------------------------------------------------------------------------------- */
int vd_set_training(vd_engine* e, int32_t training);   /* wrapper:training()/:evaluate(), model.lua:57,111 */
/* Dropout masks are a pure function philox4x32-10(seed; site, iteration, element index)
 * (DESIGN.md §5) so that the oracle can be given identical masks. */
int vd_set_dropout_seed(vd_engine* e, uint64_t seed, uint64_t iteration);
#define VD_MATH_TF32 0        /* dense contractions on wgmma tensor cores, TF32 operands, fp32 accumulate */
#define VD_MATH_FP32 1        /* same contractions on CUDA cores in fp32 (verification mode) */
#define VD_MATH_F16 2         /* TF32 mode + the many-row option LSTM (disc.lua:4-20) with fp16 operands and fp16 saved state
                                 (h, gates, da, x-projection table), fp32 accumulation, fp32 cell state and gradients */
int vd_set_math_mode(vd_engine* e, int32_t mode);
/* gen decoder: on = 1 lets vd_decoder_forward keep the (rows, vocabSize) log-probabilities on chip when the caller only
 * passes decOut on to the criterion (decoder:forward -> criterion:forward, model.lua:313-314): decOut_dev is then NULL, the
 * projection's epilogue keeps the softmax statistics and the target log-probability, and vd_criterion_backward recomputes the
 * projection with the softmax gradient fused in.  Default 0: decOut is materialised (LogSoftMax output, gen.lua:23-24).
 * vd_forward_backward and vd_retrieve never hand decOut out and always take the fused route in the tensor-core modes. */
int vd_set_lazy_decout(vd_engine* e, int32_t on);
/* Scheduling knob (results are identical either way).  on = 1 (default): the disc decoder's option LSTM (disc.lua:4-20),
 * which does not depend on the encoder until the final dot product, runs on its own stream concurrently with the
 * encoder's forward and backward, its persistent kernels leaving `reserve_sms` SMs (default 16, < 0 keeps the current
 * value) to the encoder's chains.  on = 0: the reference's order (encoder, then decoder) on one timeline — used by
 * bench.py to time the option-LSTM step kernel alone for the roofline. */
int vd_set_option_overlap(vd_engine* e, int32_t on, int32_t reserve_sms);

/* ---- fine-grained module protocol (what Model:forwardBackward calls, model.lua:297-337) ----- */
int vd_encoder_forward(vd_engine* e, const vd_batch* b, const float** encOut_dev);       /* encoder:forward(inputs), :297 */
int vd_forward_connect(vd_engine* e);                                                    /* decoders/gen.lua:30-42; no-op for disc (disc.lua:35) */
int vd_decoder_forward(vd_engine* e, const vd_batch* b, const float** decOut_dev);       /* decoder:forward, :313 / :329 */
int vd_criterion_forward(vd_engine* e, const vd_batch* b, float* loss_host);             /* criterion:forward, :314 / :330 */
int vd_criterion_backward(vd_engine* e, const vd_batch* b);                              /* criterion:backward, :318 / :334 */
int vd_decoder_backward(vd_engine* e, const vd_batch* b);                                /* decoder:backward, :319 / :335 */
int vd_backward_connect(vd_engine* e, const float** gradEncOut_dev);                     /* gen.lua:45-60; disc: t[2] of :335 */
int vd_encoder_backward(vd_engine* e, const vd_batch* b, const float* gradEncOut_dev);   /* encoder:backward, :323 / :337 */

/* ---- fused fast paths ----------------------------------------------------------------------- */
int vd_forward_backward(vd_engine* e, const vd_batch* b, int32_t only_forward, float* loss_host);  /* Model:forwardBackward, model.lua:249-342 */
/* One training step on dense relevance targets (disc decoder only).  b: a disc training batch exactly as for
 * vd_forward_backward; round_host (B) 0-based annotated round of each dialog; relevance_host (B, numOptions) >= 0 with a
 * positive sum per row.  loss = mean over the B rows of  lse(s_b) - sum_k p_bk s_bk,  p_b = relevance_b / sum(relevance_b),
 * s_b = the disc scores of round round_host[b] of dialog b.  Gradients accumulate into dW as vd_forward_backward's do.
 * The encoder runs over all rounds (same dropout masks as vd_forward_backward); the option LSTM only over the B selected
 * rounds' options.  VD_E_STATE for a gen engine; VD_E_BADARG for a null pointer, a round outside [0, maxQuesCount) or a
 * negative, non-finite or zero-sum relevance row. */
int vd_forward_backward_dense(vd_engine* e, const vd_batch* b, const int32_t* round_host, const float* relevance_host,
                              float* loss_host);
/* Model:retrieveBatch (model.lua:344-430).  use_gt != 0: ranks_host is (N) = rank of the ground
 * truth; else (N,100) = rank of every option.  Ranks are 1-based; ties: lower index wins. */
int vd_retrieve(vd_engine* e, const vd_batch* b, int32_t use_gt, int32_t* ranks_host);
/* utils.computeRanks (utils.lua:106-128) on device scores (n_rows,100). */
int vd_compute_ranks(vd_engine* e, const float* scores_dev, int32_t n_rows,
                     const int32_t* gt_dev_or_null, int32_t* ranks_dev);
/* utils.computeLhood (utils.lua:86-102) fused with the gen decoder: log-likelihood (N,100) of
 * every candidate answer, never materialising the (T,N,V) log-probs. */
int vd_gen_option_lhood(vd_engine* e, const vd_batch* b, const float** lhood_dev);
/* Model:generateAnswers (model.lua:432-613): the pieces its beam search / sampling loop drives on the device.
 *  vd_encoder_rnn_state: enc.rnnLayers[level].output[Tq] / .cell[Tq] of the last vd_encoder_forward, (N,H) device
 *    pointers, level = 0 | 1 (model.lua:480-483); both NULL for encoders without .rnnLayers (mn-att, :491-501).
 *  vd_gen_decoder_step: decoder:forward(tokens) for ONE time step on `rows` independent rows with
 *    .userPrevOutput / .userPrevCell = h_prev[l] / c_prev[l] (l = 0, 1; (rows,H) device pointers, NULL = zeros)
 *    (model.lua:517-526, gen.lua:3-27).  tokens: HOST int32 (rows).  Returns device pointers, valid until the next
 *    vd_encoder_forward: log-probabilities (rows,V) (all-zero row for a pad token, MaskZero) and the new state. */
int vd_encoder_rnn_state(vd_engine* e, int32_t level, const float** h_last_dev, const float** c_last_dev);
int vd_gen_decoder_step(vd_engine* e, int32_t rows, const int32_t* tokens_host, const float* const* h_prev,
                        const float* const* c_prev, const float** logp_dev, const float** h_out, const float** c_out);
/* Model:generateAnswers' beam search (model.lua:472-579) for EVERY round of every dialog of the last vd_encoder_forward
 * (N = B * maxQuesCount searches, N * beam_size hypotheses per step), entirely on the device: the decoder steps, the top-k,
 * the candidate merge with all of the reference's quirks, and the best finished hypothesis.  One synchronisation, at the end.
 * answer_host (N, beam_len) int32: the best finished beam (position 0 = start_token, zero-padded), length_host (N): its
 * length (0 = no hypothesis reached end_token; the reference indexes nil there, :575), score_host (N) fp64: its score.
 * VD_E_STATE for a disc engine or before any vd_encoder_forward; VD_E_BADARG unless 1 <= beam_size <= min(32, vocabSize)
 * and beam_len >= 2. */
int vd_gen_beam_search(vd_engine* e, int32_t beam_size, int32_t beam_len, int32_t start_token, int32_t end_token,
                       int32_t* answer_host, int32_t* length_host, double* score_host);
/* Model:generateAnswers' sampling (model.lua:581-602, sampleWords = 1) for EVERY round of the last vd_encoder_forward (N =
 * B * maxQuesCount rows), entirely on the device, the decoder fed its own samples (gen.lua:63-68).  One synchronisation, at
 * the end.  Draw rule (Gumbel-max over x / temperature, counter-based Philox; see DESIGN §14): the token of step t of row r
 * depends only on (seed, row_offset + r, t, the logits), so rounds sampled in different calls or on different ranks draw
 * the same tokens when row_offset is the global index of the call's first round.
 * answer_host (N, beam_len + 1) int32: column 0 = start_token, columns 1..beam_len the samples.  logp_host (N, beam_len) or
 * NULL: each sampled token's log-probability under the un-tempered LogSoftMax output (decOut).
 * VD_E_STATE for a disc engine or before any vd_encoder_forward; VD_E_BADARG unless beam_len >= 1, temperature is finite and
 * > 0, row_offset >= 0, 1 <= start_token <= vocabSize and answer_host != NULL. */
int vd_gen_sample(vd_engine* e, int32_t beam_len, int32_t start_token, float temperature, uint64_t seed, int64_t row_offset,
                  int32_t* answer_host, float* logp_host);
/* Dialogs on the model's own answers (DESIGN §17): for every dialog of batch b (gen, history encoders), round by round
 * r = 0 .. maxQuesCount-1, the encoder forward in eval mode on a history whose rows 0..r hold the batch's caption row, the
 * batch's questions and the answers the call generated for the earlier rounds, then vd_gen_beam_search's search (or
 * vd_gen_sample's draw) on round r's rows only, then round r's write into history row r+1 by dataloader.lua:202-278's rule:
 * Q ++ A right-aligned, or for the concatenated history of the late-fusion encoders row r ++ <END> ++ Q ++ A.  A = the
 * non-pad words between <START> and <END> of the best finished hypothesis (empty when none finished), or the samples before
 * the first end_token, cut to their first max_ans_len words; a question of pads only writes no Q and no A.  History rows
 * are hist_width wide and keep their rightmost hist_width words.  The whole loop is enqueued on the device: one
 * synchronisation, at the end.
 * Outputs are those of vd_gen_beam_search / vd_gen_sample for the N = B * maxQuesCount rounds of the batch; sampled round r
 * of dialog b draws as global round row_offset + b * maxQuesCount + r.  hist_host: NULL or (B, maxQuesCount, hist_width)
 * int32, the history rows the encoder read.
 * VD_E_STATE for a disc engine or an encoder without history; VD_E_BADARG for the arguments vd_gen_beam_search /
 * vd_gen_sample refuse, hist_width < b->Th or max_ans_len < 1 (and end_token outside [1, vocabSize] when sampling). */
int vd_gen_dialog_beam_search(vd_engine* e, const vd_batch* b, int32_t beam_size, int32_t beam_len, int32_t start_token,
                              int32_t end_token, int32_t hist_width, int32_t max_ans_len, int32_t* answer_host,
                              int32_t* length_host, double* score_host, int32_t* hist_host);
int vd_gen_dialog_sample(vd_engine* e, const vd_batch* b, int32_t beam_len, int32_t start_token, int32_t end_token,
                         float temperature, uint64_t seed, int64_t row_offset, int32_t hist_width, int32_t max_ans_len,
                         int32_t* answer_host, float* logp_host, int32_t* hist_host);

/* ---- optimiser step (model.lua:96-105 + optim_updates.lua:62-91) ---------------------------- */
/* all-reduce(SUM)/world of dW when a communicator is attached, then clamp(-5,5), then adam.
 * The LR decay (model.lua:102-105) stays with the caller, as in the reference. */
int vd_clamp_adam_step(vd_engine* e, float learning_rate);

/* ---- data-parallel communicator (no reference counterpart: train.lua is single-GPU) -------- */
#define VD_COMM_ID_BYTES 128
int vd_comm_unique_id(void* id_out);                        /* rank 0; broadcast the bytes out of band */
int vd_comm_init(vd_engine* e, const void* id, int32_t rank, int32_t world);
int vd_comm_allreduce_grads(vd_engine* e);                  /* exposed for tests; vd_clamp_adam_step calls it */

/* ---- plumbing -------------------------------------------------------------------------------- */
int vd_memcpy_d2h(vd_engine* e, void* host_dst, const void* dev_src, size_t bytes);
int vd_memcpy_h2d(vd_engine* e, void* dev_dst, const void* host_src, size_t bytes);
/* pinned host memory for batch buffers (the H2D copy of a batch is only asynchronous from pinned memory) */
int vd_host_alloc(void** ptr, size_t bytes);
int vd_host_free(void* ptr);
/* device memory for callers that keep batches resident in HBM (vd_batch.on_device = 1) */
int vd_device_alloc(vd_engine* e, void** ptr, size_t bytes);
int vd_device_free(vd_engine* e, void* ptr);
int vd_synchronize(vd_engine* e);
int vd_stream(vd_engine* e, void** cuda_stream);
/* device-side timing on the engine's stream (CUDA events) */
int vd_timer_start(vd_engine* e);
int vd_timer_stop(vd_engine* e, float* ms);
/* launch accounting: every kernel the engine launches is counted; kernels of class `name`
 * ("lstm_step", "gemm", ...) are additionally bracketed by events when profiling is on.  With profiling 1 every launch
 * is also counted under its launch-site name ("k_segsum_rows", "rank_rows", ...; launches only, no time). */
int vd_profile_enable(vd_engine* e, int32_t on);
int vd_profile_reset(vd_engine* e);
int vd_launch_count(vd_engine* e, int64_t* n_launches);
int vd_kernel_stats(vd_engine* e, const char* name, int64_t* launches, double* total_ms,
                    double* total_flops, double* total_bytes);
/* test hooks: the engine's two dense-contraction primitives on caller-provided DEVICE buffers, routed exactly as
 * the engine routes them (math mode).  tn: C[m,n] = act(beta*C + bias[n] + sum_k A[m,k] B[n,k]);
 * atb: C[m,n] += sum_k A[k,m] B[k,n]. */
int vd_gemm_tn(vd_engine* e, int32_t M, int32_t N, int32_t K, const float* A, int64_t lda, const float* B, int64_t ldb,
               float* C, int64_t ldc, float beta, const float* bias, int32_t act);
int vd_gemm_atb(vd_engine* e, int32_t M, int32_t N, int64_t K, const float* A, int64_t lda, const float* B, int64_t ldb,
                float* C, int64_t ldc);
/* test hook of the VD_MATH_F16 weight-gradient primitive: A (K x M) and B (K x N) fp32 DEVICE buffers are rounded to
 * fp16, then C[m,n] += inv_scale * sum_k A[k,m] B[k,n] on f16 wgmma (both operands MN-major). */
int vd_gemm_atb16(vd_engine* e, int32_t M, int32_t N, int64_t K, const float* A, int64_t lda, const float* B, int64_t ldb,
                  float* C, int64_t ldc, float inv_scale);
/* test hooks of one SeqLSTM time step on caller-provided DEVICE buffers (fp32, row-major), routed exactly as the engine
 * routes a step in its math mode: the fused tensor-core step kernel when it takes the shape, otherwise the recurrent GEMM
 * and the pointwise kernel.  *path receives the tile width of the fused kernel that ran, or 0 for CUDA cores.
 * fwd: z[r] = bias + (has_xproj ? gates[r] : ptable[tok[r]]) + h_prev[r] WhT^T      (h_prev NULL: no recurrent term)
 *      gates <- [sigmoid(z_i) sigmoid(z_f) sigmoid(z_o) tanh(z_g)],  c_out = f c_prev + i g,  h_out = o tanh(c_out);
 *      WhT (4H, ldw) = the h columns of the transposed weight; ptable (ptable_rows, 4H) is a gathered x-projection, which
 *      only the tensor-core route takes; c_prev NULL = zeros; rows whose mask id is 0 are all zero.
 * bwd: dh = da_next[r] Wh^T + dh_ext[r],  d = dc_carry + dh o (1 - tanh^2 c_cur),
 *      da <- [d g i(1-i)  d c_prev f(1-f)  dh tanh(c_cur) o(1-o)  d i(1-g^2)],  dc_carry <- d f;
 *      Wh (H, 4H) = the h rows of the weight; da_next / dh_ext / c_prev NULL = zeros; masked rows all zero.
 * The fp16 option-LSTM steps of VD_MATH_F16 are not reachable through these hooks (an error). */
int vd_lstm_step_fwd(vd_engine* e, int64_t R, int32_t H, const float* h_prev, const float* WhT, int64_t ldw, const float* bias,
                     float* gates, int32_t has_xproj, const float* ptable, int64_t ptable_rows, const int32_t* tok,
                     const float* c_prev, float* c_out, float* h_out, const int32_t* mask_ids, int32_t* path);
int vd_lstm_step_bwd(vd_engine* e, int64_t R, int32_t H, const float* da_next, const float* Wh, const float* gates,
                     const float* c_prev, const float* c_cur, const float* dh_ext, float* dc_carry, const int32_t* mask_ids,
                     float* da, int32_t* path);
/* test hooks of the VD_MATH_F16 option-LSTM step kernels (lstm16.cu) on caller-provided DEVICE buffers, row-major; "16"
 * buffers hold IEEE binary16, the others fp32.  Shapes as the engine routes them there: H % 256 == 0, H <= 512, R >= 1024.
 * fwd: z[r] = bias + ptable16[tok[r]] + h_prev16[r] Wh16^T   (Wh16 (4H, H), ptable16 (V, 4H) without bias, whose row 0 =
 *      the pad token's = zeros), gates16 (R, 4H) <- [sigmoid(z_i) sigmoid(z_f) sigmoid(z_o) tanh(z_g)] unless NULL,
 *      c_out = f c_prev + i g (c_prev NULL = zeros), h16_out = o tanh(c_out), h32_out (NULL or fp32) = the same h;
 *      rows whose mask id is 0 are all zero.
 * bwd: dh = da_next16[r] Whb16^T (Whb16 (H, 4H)), d = dc_carry + dh o (1 - tanh^2 c_cur),
 *      da16 <- [d g i(1-i)  d c_prev f(1-f)  dh tanh(c_cur) o(1-o)  d i(1-g^2)], dc_carry <- d f; c_prev NULL = zeros. */
int vd_lstm16_step_fwd(vd_engine* e, int64_t R, int32_t H, const void* h_prev16, const void* Wh16, const void* ptable16,
                       const int32_t* tok, const float* bias, const float* c_prev, const int32_t* mask_ids, void* gates16,
                       float* c_out, void* h16_out, float* h32_out);
int vd_lstm16_step_bwd(vd_engine* e, int64_t R, int32_t H, const void* da_next16, const void* Whb16, const void* gates16,
                       const float* c_prev, const float* c_cur, float* dc_carry, const int32_t* mask_ids, void* da16);
/* test hook of the engine's pointwise, attention, criterion and decoding kernels: calls the launcher `name` (the table in
 * visdial_b200/csrc/test_hooks.cu lists each one's pointer / int / real arguments) on caller-provided DEVICE buffers, on the
 * engine's stream, then synchronises.  Dropout factors are the engine's own for the seed and iteration of
 * vd_set_dropout_seed (identity unless training mode 1).  VD_E_BADARG for an unknown name or wrong argument counts; a
 * launcher's refusal comes back as its error code. */
int vd_test_kernel(vd_engine* e, const char* name, void* const* ptrs, int32_t n_ptrs, const int64_t* ints, int32_t n_ints,
                   const double* reals, int32_t n_reals);
/* cudaProfilerStart / cudaProfilerStop (ncu --profile-from-start off) */
int vd_profiler_range(vd_engine* e, int32_t start);
/* flush L2 by writing a scratch buffer larger than L2 (bench hygiene) */
int vd_flush_l2(vd_engine* e);

/* ---- dataloader: HBM-resident corpus and on-device batch assembly --------------------------------
 * Replaces dataloader:initialize's tensor preparation and the per-batch indexing
 * (dataloader.lua:143-321 prepareDataset / processAnswers / processHistory / processOptions,
 * utils.lua:6-45 rightAlign, dataloader.lua:324-478 getTrainBatch / getTestBatch / getIndexData /
 * getIndexOption).  The raw arrays are the datasets of visdial_data.h5 for ONE split exactly as
 * data/prepro.py:105-183 writes them (the HDF5 read itself stays with the host language); they are
 * uploaded once, prepared on the device, and every later batch is gathered + trimmed on the device:
 * per batch only the dialog indices cross PCIe.  All ids int32, 1-based with 0 = pad. */
typedef struct vd_corpus vd_corpus;

typedef struct vd_corpus_desc {
  int32_t numThreads;           /* dialogs in the split: ques:size(1)                      (dataloader.lua:94-105) */
  int32_t numRounds;            /* ques:size(2) = maxQuesCount                             (:122)  */
  int32_t maxQuesLen;           /* ques:size(3)                                            (:124)  */
  int32_t maxAnsLen;            /* ans:size(3) = opt_list:size(2)                          (:126)  */
  int32_t maxCapLen;            /* cap:size(2); must be >= maxQuesLen + maxAnsLen when useHistory (:236) */
  int32_t numOptions;           /* opt:size(3)                                             (:112)  */
  int32_t numOptList;           /* opt_list:size(1)                                                */
  int32_t numImages;            /* images:size(1)                                                  */
  int32_t useHistory;           /* opt.useHistory / concatHistory / useIm                  (:139-141) */
  int32_t concatHistory;
  int32_t useIm;
  int32_t maxHistoryLen;        /* opt.maxHistoryLen (60) — overwritten by min(R*(Lq+La),300) when concatHistory (:142,:217) */
  int32_t imgNorm;              /* 1: L2-normalise over dim 2 at load                      (:64-68) */
  int32_t imgAtt;               /* 1: images are (N,C,S,S) and are stored (N,S,S,C)        (:70-72) */
  int32_t imgChannels;          /* C (pool5 512) or F (fc7 4096)                                   */
  int32_t imgSpatial;           /* S (14); ignored unless imgAtt                                   */
  int32_t startToken, endToken; /* word2ind['<START>'], word2ind['<END>']                  (:17-22) */
  const int32_t* ques;          /* (n,R,Lq) left-aligned  'ques_<split>'                           */
  const int32_t* ques_len;      /* (n,R)                  'ques_length_<split>'                    */
  const int32_t* ans;           /* (n,R,La)               'ans_<split>'                            */
  const int32_t* ans_len;       /* (n,R)                  'ans_length_<split>'                     */
  const int32_t* cap;           /* (n,Lc)                 'cap_<split>'        (NULL unless useHistory) */
  const int32_t* cap_len;       /* (n)                    'cap_length_<split>'                     */
  const int32_t* opt;           /* (n,R,K) 1-based rows of opt_list  'opt_<split>'                 */
  const int32_t* opt_list;      /* (m,La)                 'opt_list_<split>'                       */
  const int32_t* opt_len;       /* (m)                    'opt_length_<split>'                     */
  const int32_t* ans_index;     /* (n,R) 1-based gt option 'ans_index_<split>' (NULL for test)     */
  const int32_t* img_pos;       /* (n) 0-based row of images as stored ('img_pos_<split>'; the +1 of :76-77 is Lua indexing) */
  const int32_t* num_rounds;    /* (n)                    'num_rounds_<split>' (may be NULL)       */
  const float* images;          /* (N,F) or (N,C,S,S) fp32 'images_<split>' of the image h5 (NULL unless useIm) */
} vd_corpus_desc;

/* dataloader:initialize tensors -> HBM + dataloader:prepareDataset on the device.  Host pointers. */
int vd_corpus_create(vd_engine* e, const vd_corpus_desc* d, vd_corpus** out);
int vd_corpus_destroy(vd_corpus* c);
/* Assemble the batch of dialogs `inds` (HOST array of n 0-based dialog indices = Lua's inds - 1) on the engine's stream.
 *   decoder_gen = 0: getIndexData + getIndexOption('disc')  -> ques_fwd, hist, img_feat, answer_in/out, answer_ind, options
 *   decoder_gen = 1: getIndexData only (getTrainBatch, gen)  -> ... without options
 *   decoder_gen = 2: getIndexData + getIndexOption('gen')   -> ... plus option_in / option_out (getTestBatch, gen)
 * `out` receives DEVICE pointers (on_device = 1) into corpus-owned buffers that stay valid until the second-next
 * vd_corpus_get_batch on this corpus (two buffer sets, alternating). */
int vd_corpus_get_batch(vd_corpus* c, const int64_t* inds, int32_t n, int32_t decoder_gen, vd_batch* out);
/* Read one PREPARED tensor back to the host (parity tests): name in {"ques_fwd","hist","hist_len","ans_in","ans_out",
 * "opt_in","opt_out","img_fv"}; *elems receives the element count (call with host_dst = NULL to size). */
int vd_corpus_read(vd_corpus* c, const char* name, void* host_dst, int64_t* elems);
/* bytes the last vd_corpus_get_batch read + wrote in HBM (algorithmic) and the number of kernels it launched */
int vd_corpus_batch_bytes(vd_corpus* c, int64_t* bytes, int32_t* launches);

#ifdef __cplusplus
}
#endif
#endif /* VISDIAL_B200_H */
