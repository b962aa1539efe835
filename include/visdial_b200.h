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
  int32_t imgRegions;           /* 0: img_feat is the imgSpatialSize^2 grid; P > 0: P detector region rows of imgFeatureSize
                                   channels per image (DESIGN §26), att encoders only */
} vd_params;

/* A batch as produced by dataloader:getTrainBatch / getTestBatch (dataloader.lua:324-478),
 * Appendix A of SURVEY.md.  Unused pointers may be NULL.  N = B * maxQuesCount. */
typedef struct vd_batch {
  int32_t B;                    /* dialogs ("threads") in this batch */
  int32_t Tq, Th, Ta, To;       /* trimmed question / history / answer(+1) / option widths */
  const int32_t* ques_fwd;      /* (B,10,Tq) right-aligned */
  const int32_t* hist;          /* (B,10,Th) right-aligned */
  const float* img_feat;        /* (B,F) fc7, (B,S,S,C) NHWC pool5 or (B,P,C) regions — one row per dialog */
  const int32_t* options;       /* disc: (N,100,To) left-aligned raw option tokens */
  const int32_t* answer_ind;    /* (N) 1-based ground-truth option */
  const int32_t* answer_in;     /* gen: (B,10,Ta) <START> a.. 0.. */
  const int32_t* answer_out;    /* gen: (B,10,Ta) a.. <END> 0.. */
  const int32_t* option_in;     /* gen eval: (B,10,100,To) */
  const int32_t* option_out;    /* gen eval: (B,10,100,To) */
  int32_t on_device;            /* 0: host pointers (staged + copied H2D by the engine), 1: device */
  const int32_t* img_count;     /* (B) regions present per dialog's image, each in [1, imgRegions] (checked when staged from
                                   the host; a precondition for device batches); NULL = all present.  Region engines only:
                                   the SAN attends over rows 0 .. count-1 and the rest never affect a result (DESIGN §26) */
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
/* Answer rules (DESIGN §25): classes barred from every token choice of a gen model's answering calls, beam search (plain,
 * diverse, n-best) and sampling (plain, truncated), for whole splits, dialogs and dialog asks alike, until changed.  At step
 * t the answer so far has t - 1 words w[1 .. t-1] (the row's own earlier tokens; a beam's pads are 0):
 *  - min_words m >= 0: end_token is barred while t <= m, so every finished answer has at least m words;
 *  - no_repeat_ngram n >= 0 (0 = off): a word is barred if it would complete an n-gram already in w (a window holding a pad
 *    matches nothing, <START> is in no n-gram, end_token is never barred by this rule); n = 1 bars every word already used;
 *  - banned: n_banned <= 1024 ids in [1, vocabSize], never chosen.
 * If a row's barred set would cover every class, end_token is allowed.  Scores and log-probabilities stay the unconstrained
 * LogSoftMax's.  A beam row with fewer allowed classes than the beam lists what it has; sampling draws from the allowed
 * classes with the same keys, so a draw is unchanged whenever its unconstrained token is allowed.  Active rules send
 * sampling through the materialised-logits route in every math mode.  vd_gen_sample and vd_gen_truncated_sample take no
 * end_token: their <END> is vocabSize (the dataloader's).
 * r = NULL turns the rules off (the default: every call is then exactly what it is without them).  Refused with VD_E_BADARG,
 * keeping the old rules: a negative count, n_banned > 1024, banned NULL with n_banned > 0, an id outside [1, vocabSize], or
 * active rules with vocabSize > 49152 (a row's barred set is a bit mask in shared memory).  While active, an answering call
 * is refused with VD_E_BADARG, before any state changes, when its end_token is banned, or when min_words > beam_len - 2
 * (beam search) / beam_len - 1 (sampling).  Disc retrieval, training, evaluation and vd_gen_decoder_step ignore them. */
typedef struct vd_answer_rules {
  int32_t min_words;
  int32_t no_repeat_ngram;
  int32_t n_banned;
  const int32_t* banned; /* HOST, n_banned ids; copied by the call */
} vd_answer_rules;
int vd_set_answer_rules(vd_engine* e, const vd_answer_rules* r);
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
/* Deterministic training (DESIGN §27).  on = 1: every output of a training step (vd_forward_backward, _dense, _dense_gen and
 * the fine-grained backward calls: the loss and dW; W, m and v after vd_clamp_adam_step) is a function of the parameters,
 * math mode, W, optimiser state, batch and dropout seed / iteration only — bit for bit the same on every run, whatever the
 * GPU's SM count, vd_set_option_overlap's setting or the streams' timing.  The gradient reductions then take routes without
 * float atomics (partial sums in fixed slots, added in a fixed order), at some cost in speed.  Default 0: the atomic routes.
 * May be set between steps.  VD_E_BADARG unless on is 0 or 1; VD_E_STATE for on = 1 on an engine with a communicator of
 * world > 1 (vd_comm_init with world > 1 is likewise refused on a deterministic engine). */
int vd_set_deterministic(vd_engine* e, int32_t on);

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
/* The same step for the gen decoder (DESIGN §16).  b: a gen batch carrying option_in / option_out (vd_corpus_get_batch
 * mode 2), To its option width; round_host and relevance_host as above.  s_bk = the log-likelihood of option k of round
 * round_host[b] under the teacher-forced gen decoder started from that round's state, exactly what vd_gen_option_lhood
 * gives for that row (sum over t of keep * (x_t[tgt_t] - lse_t), keep = input token != 0 and target > 0); the loss is the
 * soft-target cross-entropy above.  The encoder runs over all rounds (same dropout masks as vd_forward_backward); the
 * decoder only over the B*numOptions selected option rows, and the encoder receives gradient through the annotated
 * rounds' initial decoder state only.  Gradients accumulate into dW as vd_forward_backward's do (world > 1: vd_zero_grad
 * between backward passes).  VD_E_STATE for a disc engine; VD_E_SHAPE for a batch without option_in / option_out;
 * VD_E_BADARG as vd_forward_backward_dense.  The engine stays usable after any refusal. */
int vd_forward_backward_dense_gen(vd_engine* e, const vd_batch* b, const int32_t* round_host, const float* relevance_host,
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
 *    (model.lua:517-526, gen.lua:3-27).  tokens: HOST int32 (rows).  Callable after vd_encoder_forward or a
 *    vd_dialog_ask_* (DESIGN §19).  Returns device pointers, valid until the next vd_encoder_forward: log-probabilities (rows,V) (all-zero row for a pad token, MaskZero) and the new state. */
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
/* Diverse beam search (Vijayakumar et al., arXiv:1610.02424; DESIGN §22): vd_gen_beam_search's search with its beam_size
 * = k columns split into `groups` G groups of w = k / G, group g owning columns [g*w, (g+1)*w).  Each step fills the
 * groups in order; a candidate of group g is penalised by diversity * (the number of columns of groups < g filled at this
 * step with its token) (Hamming diversity; unfilled columns and finished hypotheses do not count, so end_token never
 * is).  Each explored column of group g takes its w best classes under the penalty; <END> candidates compete for the
 * group's best finished hypothesis by their unpenalised score, the others fill the group's columns by their penalised
 * score, and a column stores the unpenalised score, so every reported score is a log-probability.  At step 1 only each
 * group's first column is explored.  G = 1 is vd_gen_beam_search bit for bit; diversity 0 makes every group a search of
 * width w.  The decoder work is that of vd_gen_beam_search at beam_size k.
 * answer_host (N, G, beam_len), length_host (N, G), score_host (N, G): each group's best finished hypothesis as
 * vd_gen_beam_search's (length 0: none).  A round's pick (what a dialog's history takes) is the best of its G by (score
 * desc, group asc) among groups of length > 0.
 * Refusals as vd_gen_beam_search's, and VD_E_BADARG unless groups >= 1 divides beam_size and diversity is finite and >= 0. */
int vd_gen_diverse_beam_search(vd_engine* e, int32_t beam_size, int32_t groups, float diversity, int32_t beam_len,
                               int32_t start_token, int32_t end_token, int32_t* answer_host, int32_t* length_host,
                               double* score_host);
/* n-best lists with length normalisation (DESIGN §24): vd_gen_diverse_beam_search's search (groups = 1: vd_gen_beam_search's)
 * with each group keeping its nbest best finished hypotheses instead of one.  A finished hypothesis of `length` tokens
 * (<START> .. <END>) has l = length - 1 generated tokens and norm = score / lp(l), lp(l) = ((5 + l) / 6)^length_penalty
 * (GNMT, Wu et al., arXiv:1609.08144), lp computed in fp64 with the host's pow and the division in IEEE fp64; score stays
 * the summed log-probability.  A group's list holds its n best of all the <END> candidates the search met, by (norm desc,
 * step asc, candidate asc).  Live beams, their scores and the decoder work are those of the search without lists.  A
 * round's pick (what a dialog's history takes) is the best list head by (norm desc, group asc) among groups that finished
 * a hypothesis.  nbest = 1 and length_penalty = 0 is vd_gen_diverse_beam_search bit for bit.
 * answer_host (N, G, nbest, beam_len), length_host (N, G, nbest) (0: an entry never filled), score_host (N, G, nbest) and
 * norm_host (N, G, nbest) or NULL, each list best first.
 * Refusals as vd_gen_diverse_beam_search's, and VD_E_BADARG unless 1 <= nbest <= 32 and length_penalty is finite and
 * >= 0. */
int vd_gen_nbest_beam_search(vd_engine* e, int32_t beam_size, int32_t groups, float diversity, float length_penalty,
                             int32_t nbest, int32_t beam_len, int32_t start_token, int32_t end_token, int32_t* answer_host,
                             int32_t* length_host, double* score_host, double* norm_host);
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
/* vd_gen_dialog_beam_search's loop with vd_gen_diverse_beam_search's search: round r's history row takes the round's
 * pick.  Outputs (N, G, beam_len), (N, G), (N, G) for the N = B * maxQuesCount rounds; hist_host and refusals as
 * vd_gen_dialog_beam_search's and vd_gen_diverse_beam_search's. */
int vd_gen_dialog_diverse_beam_search(vd_engine* e, const vd_batch* b, int32_t beam_size, int32_t groups, float diversity,
                                      int32_t beam_len, int32_t start_token, int32_t end_token, int32_t hist_width,
                                      int32_t max_ans_len, int32_t* answer_host, int32_t* length_host, double* score_host,
                                      int32_t* hist_host);
/* vd_gen_dialog_beam_search's loop with vd_gen_nbest_beam_search's search: round r's history row takes the round's pick.
 * Outputs (N, G, nbest, beam_len), (N, G, nbest) three times for the N = B * maxQuesCount rounds; hist_host and refusals as
 * vd_gen_dialog_beam_search's and vd_gen_nbest_beam_search's. */
int vd_gen_dialog_nbest_beam_search(vd_engine* e, const vd_batch* b, int32_t beam_size, int32_t groups, float diversity,
                                    float length_penalty, int32_t nbest, int32_t beam_len, int32_t start_token,
                                    int32_t end_token, int32_t hist_width, int32_t max_ans_len, int32_t* answer_host,
                                    int32_t* length_host, double* score_host, double* norm_host, int32_t* hist_host);
/* Truncated sampling (DESIGN §23): vd_gen_sample / vd_gen_dialog_sample with the draw restricted, at every step of every
 * row, to a prefix of the classes in the order (y desc, class asc), y = logit / temperature: the first top_k of them
 * (top_k = 0: all), then of those the shortest prefix holding top_p of their softmax mass (top_p = 1: all), measured in
 * integer masses rint(exp(y - max y) 2^32) so that the boundary does not depend on summation order.  The token is the
 * Gumbel-max argmax of vd_gen_sample's keys over the prefix: an exact draw from the renormalised truncated softmax, equal
 * to vd_gen_sample's token whenever that token is in the prefix.  logp stays the un-tempered, untruncated LogSoftMax's.
 * Truncation is active when 1 <= top_k < vocabSize or top_p < 1; inactive, the calls are vd_gen_sample /
 * vd_gen_dialog_sample bit for bit.  Outputs as theirs.
 * Refusals, before any state changes: those of vd_gen_sample / vd_gen_dialog_sample, and VD_E_BADARG for top_k < 0, top_p
 * outside (0, 1] or not finite, and active truncation with vocabSize > 49152 (a row is staged in shared memory). */
int vd_gen_truncated_sample(vd_engine* e, int32_t beam_len, int32_t start_token, float temperature, uint64_t seed,
                            int64_t row_offset, int32_t top_k, float top_p, int32_t* answer_host, float* logp_host);
int vd_gen_dialog_truncated_sample(vd_engine* e, const vd_batch* b, int32_t beam_len, int32_t start_token, int32_t end_token,
                                   float temperature, uint64_t seed, int64_t row_offset, int32_t top_k, float top_p,
                                   int32_t hist_width, int32_t max_ans_len, int32_t* answer_host, float* logp_host,
                                   int32_t* hist_host);

/* ---- answer-pool retrieval: disc models answer (DESIGN §18) --------------------------------------------------------
 * A disc model answers a question by retrieval: it scores every answer of the split's answer pool (opt_list_<split>, every
 * distinct candidate answer of the split) with disc.lua:22-29's dot product and takes the best.
 *  vd_answer_pool_encode: tokens_host (m, width) int32 HOST, the pool's token rows as opt_list stores them (left-aligned,
 *    zero-padded; width = the corpus's maxAnsLen gives each answer the encoding the disc decoder computes for it in any
 *    batch).  Runs opt.lstm (no maskzero, disc.lua:4-20) forward-only over every row in the current math mode and keeps
 *    h_T, (m, rnnHiddenSize) fp32, replacing any earlier pool.  VD_E_STATE for a gen engine; VD_E_BADARG for m < 1,
 *    width < 1 or a token outside [0, vocabSize].
 *  vd_answer_pool: the pool embeddings (m, rnnHiddenSize) as a DEVICE pointer, valid until the next encode.
 *  vd_answer_pool_retrieve: the encoder forward in eval mode on batch b (its options, if any, are not read), then per round
 *    n of the N = B * maxQuesCount rounds the k best pool rows by (score desc, pool index asc), score = encOut[n] . e_j:
 *    index_host (N, k) 0-based pool rows, score_host (N, k) fp32.  One synchronisation, at the end.  1 <= k <= min(32, m).
 *  vd_answer_pool_dialog: vd_gen_dialog_*'s loop (history rule, widths, hist_host and their refusals) with this retrieval
 *    as round r's search; the top-1 pool row's non-pad words (before any <END> = vocabSize) are round r's answer.
 *    Outputs as vd_answer_pool_retrieve's for all N rounds.  VD_E_STATE for an encoder without history.
 * The pool belongs to the weights and the math mode it was encoded with: vd_set_parameters, vd_clamp_adam_step and
 * vd_set_math_mode drop it, and a retrieval without a current pool is refused (VD_E_STATE), as it is on a gen engine.
 * Writes a caller makes to the weights through vd_param_buffers do not drop it: re-encode after them. */
int vd_answer_pool_encode(vd_engine* e, const int32_t* tokens_host, int64_t m, int32_t width);
int vd_answer_pool(vd_engine* e, const float** emb_dev, int64_t* m);
int vd_answer_pool_retrieve(vd_engine* e, const vd_batch* b, int32_t k, int32_t* index_host, float* score_host);
int vd_answer_pool_dialog(vd_engine* e, const vd_batch* b, int32_t k, int32_t hist_width, int32_t max_ans_len,
                          int32_t* index_host, float* score_host, int32_t* hist_host);

/* ---- dialog sessions: questions asked one round at a time (DESIGN §19) ---------------------- */
/* A session holds the B dialogs of batch b on the engine (one session per engine; a new begin replaces it).  It takes b's
 * image rows and round-0 history row (the caption) and ignores its questions, answers and options.  Each ask supplies one
 * question row per dialog for the next round r: ques (B, Tq) int32 HOST, right-aligned and zero-padded as ques_fwd, with
 * 1 <= Tq <= b's Tq.  The ask encodes round r's B rows in eval mode over the session's cached history facts, image
 * products and dialog-LSTM state, answers them, and appends Q_r and the answer to the history by vd_gen_dialog_*'s rule
 * (hist_width, max_ans_len, pad questions and concatenated history as there).  Fed the batch's own questions, a session
 * gives vd_gen_dialog_beam_search's / vd_gen_dialog_sample's / vd_answer_pool_dialog's round-r results.  Encoders without
 * history (lf-ques, lf-ques-im) encode just the question (and image); hist_width and max_ans_len are not read for them.
 *  vd_dialog_ask_beam: vd_gen_beam_search's search on the B rows: answer (B, beam_len), length (B), score (B).
 *  vd_dialog_ask_sample: vd_gen_sample's draw: answer (B, beam_len + 1), logp (B, beam_len) or NULL; row b draws as global
 *    round row_offset + b * maxQuesCount + r, as vd_gen_dialog_sample's round r.
 *  vd_dialog_ask_pool: vd_answer_pool_retrieve's top-k (disc, current pool): index (B, k), score (B, k).
 *  vd_dialog_round: the next round to be asked and B.  vd_dialog_history: the (B, maxQuesCount, hist_width) rows.
 *  vd_dialog_encoding: the last ask's encoder output (B, rnnHiddenSize), a DEVICE pointer valid until the next ask.
 *  vd_dialog_rnn_state: vd_encoder_rnn_state for the last ask: question-LSTM layer `level`'s h and c at Tq, (B, H)
 *    DEVICE pointers valid until the next ask, NULL for encoders without .rnnLayers.  With vd_dialog_encoding it is the
 *    decoder start state the ask's answerer used.
 * Each ask ends in one synchronisation.  Session state lives outside the activation arena, so any other engine call
 * between two asks leaves it intact; begin and each ask end the last vd_encoder_forward (as a new forward would).
 * hist_width must hold the batch's round-0 row and a whole question row (hist_width >= its Th and Tq), as
 * vd_gen_dialog_*'s history append needs.
 * Refusals, before any state changes: VD_E_STATE for no session, a full one (maxQuesCount asks done), weights or math
 * mode changed since begin (vd_set_parameters, vd_clamp_adam_step, vd_set_math_mode), an answerer the decoder lacks,
 * or a stale pool; VD_E_SHAPE / VD_E_BADARG for widths, B, and tokens outside [0, vocabSize]. */
int vd_dialog_begin(vd_engine* e, const vd_batch* b, int32_t hist_width, int32_t max_ans_len);
int vd_dialog_ask_beam(vd_engine* e, const int32_t* ques, int32_t Tq, int32_t beam_size, int32_t beam_len, int32_t start_token,
                       int32_t end_token, int32_t* answer, int32_t* length, double* score);
int vd_dialog_ask_sample(vd_engine* e, const int32_t* ques, int32_t Tq, int32_t beam_len, int32_t start_token, int32_t end_token,
                         float temperature, uint64_t seed, int64_t row_offset, int32_t* answer, float* logp);
int vd_dialog_ask_pool(vd_engine* e, const int32_t* ques, int32_t Tq, int32_t k, int32_t* index, float* score);
int vd_dialog_round(vd_engine* e, int32_t* round, int32_t* B);
int vd_dialog_history(vd_engine* e, int32_t* hist_host);
int vd_dialog_encoding(vd_engine* e, const float** encOut_dev);
int vd_dialog_rnn_state(vd_engine* e, int32_t level, const float** h_last, const float** c_last);
int vd_dialog_end(vd_engine* e);

/* ---- dialog pools: many conversations, each at its own round (DESIGN §20) --------------------- */
/* A session has a capacity of C slots (vd_dialog_begin's is C = B, all joined at once).  A slot is free or holds one
 * conversation with its own round r_s in [0, maxQuesCount] and its own cached state (history rows, asked questions,
 * facts, image products, dialog-LSTM state, draw base).  Conversations join, are asked and leave independently; fed the
 * same questions, a conversation's answers do not depend on its slot, on when it joined or on which other conversations
 * share its asks (in VD_MATH_FP32 bit for bit).
 *  vd_dialog_open: a pool of `capacity` free slots with question width Tq and hist_width / max_ans_len as
 *    vd_dialog_begin's (hist_width >= Tq); replaces any session.
 *  vd_dialog_join: batch b's B dialogs (image rows and round-0 history row, as vd_dialog_begin reads them) into the B
 *    lowest free slots, their ids into slots (B), each at round 0.  draw_base (B) or NULL (all 0): the global round a
 *    conversation's round 0 draws as in sampling asks.  Fewer than B free slots: VD_E_STATE, nothing joined.
 *  vd_dialog_leave: frees n slots; a freed slot's cache is never read again and a later join may reuse it.
 *  vd_dialog_ask_*_slots: one row per asked slot, slots (n) distinct and occupied, ques (n, Tq) HOST as vd_dialog_ask_*'s.
 *    Row i is encoded at round r of slot slots[i] over that slot's cache, answered as vd_dialog_ask_* answers, appended to
 *    the slot's history, and the slot's round advances.  Results are in row order.  Sampling: row i draws as global round
 *    row_offset + draw_base[slot] + r.  vd_dialog_encoding / vd_dialog_rnn_state then have n rows in row order.
 *  vd_dialog_slots: rounds (capacity) HOST or NULL: each slot's next round, -1 when free; and the capacity.
 *  vd_dialog_slot_history: the (n, maxQuesCount, hist_width) history rows of n distinct occupied slots.
 * vd_dialog_ask_* / vd_dialog_round / vd_dialog_history are the all-slots case: an ask of slots 0..C-1, and the round and
 * rows when every slot is occupied at one round (else VD_E_STATE), as a vd_dialog_begin session is until its first leave.
 * Refusals, before any state changes: VD_E_STATE for no session, stale weights or math mode (vd_set_parameters,
 * vd_clamp_adam_step and vd_set_math_mode invalidate the whole pool until it is reopened), a free slot asked or left, a
 * conversation that has had maxQuesCount asks, a join beyond capacity, an answerer the decoder lacks, a stale pool;
 * VD_E_BADARG for n < 1, slot ids outside [0, capacity) or named twice, tokens and search arguments; VD_E_SHAPE for a
 * question width outside [1, Tq]. */
int vd_dialog_open(vd_engine* e, int32_t capacity, int32_t Tq, int32_t hist_width, int32_t max_ans_len);
int vd_dialog_join(vd_engine* e, const vd_batch* b, const int64_t* draw_base, int32_t* slots);
int vd_dialog_leave(vd_engine* e, const int32_t* slots, int32_t n);
int vd_dialog_ask_beam_slots(vd_engine* e, const int32_t* slots, int32_t n, const int32_t* ques, int32_t Tq, int32_t beam_size,
                             int32_t beam_len, int32_t start_token, int32_t end_token, int32_t* answer, int32_t* length,
                             double* score);
int vd_dialog_ask_sample_slots(vd_engine* e, const int32_t* slots, int32_t n, const int32_t* ques, int32_t Tq, int32_t beam_len,
                               int32_t start_token, int32_t end_token, float temperature, uint64_t seed, int64_t row_offset,
                               int32_t* answer, float* logp);
int vd_dialog_ask_pool_slots(vd_engine* e, const int32_t* slots, int32_t n, const int32_t* ques, int32_t Tq, int32_t k,
                             int32_t* index, float* score);
/* vd_dialog_ask_beam_slots with vd_gen_diverse_beam_search's search (DESIGN §22): answer (n, G, beam_len), length (n, G),
 * score (n, G) in row order; each slot's history takes its row's pick.  A vd_dialog_begin session is the pool of slots
 * 0..B-1.  Refusals, before any state changes, as vd_dialog_ask_beam_slots' and vd_gen_diverse_beam_search's. */
int vd_dialog_ask_diverse_slots(vd_engine* e, const int32_t* slots, int32_t n, const int32_t* ques, int32_t Tq, int32_t beam_size,
                                int32_t groups, float diversity, int32_t beam_len, int32_t start_token, int32_t end_token,
                                int32_t* answer, int32_t* length, double* score);
/* vd_dialog_ask_beam_slots with vd_gen_nbest_beam_search's search (DESIGN §24): answer (n, G, nbest, beam_len), length,
 * score and norm (n, G, nbest) (norm may be NULL) in row order; each slot's history takes its row's pick.  A
 * vd_dialog_begin session is the pool of slots 0..B-1.  Refusals, before any state changes, as vd_dialog_ask_beam_slots'
 * and vd_gen_nbest_beam_search's. */
int vd_dialog_ask_nbest_slots(vd_engine* e, const int32_t* slots, int32_t n, const int32_t* ques, int32_t Tq, int32_t beam_size,
                              int32_t groups, float diversity, float length_penalty, int32_t nbest, int32_t beam_len,
                              int32_t start_token, int32_t end_token, int32_t* answer, int32_t* length, double* score,
                              double* norm);
/* vd_dialog_ask_sample_slots with vd_gen_truncated_sample's draw (DESIGN §23): answer (n, beam_len + 1), logp (n, beam_len)
 * or NULL in row order.  A vd_dialog_begin session is the pool of slots 0..B-1.  Refusals, before any state changes, as
 * vd_dialog_ask_sample_slots' and vd_gen_truncated_sample's. */
int vd_dialog_ask_truncated_slots(vd_engine* e, const int32_t* slots, int32_t n, const int32_t* ques, int32_t Tq,
                                  int32_t beam_len, int32_t start_token, int32_t end_token, float temperature, uint64_t seed,
                                  int64_t row_offset, int32_t top_k, float top_p, int32_t* answer, float* logp);
int vd_dialog_slots(vd_engine* e, int32_t* rounds, int32_t* capacity);
int vd_dialog_slot_history(vd_engine* e, const int32_t* slots, int32_t n, int32_t* hist);

/* ---- resuming conversations in a dialog pool (DESIGN §21) ------------------------------------ */
/* vd_dialog_join_rounds: batch b's B dialogs join the open pool in the free slots slots[i] (HOST, an input: a reopened
 * pool puts each conversation back in its own slot), at rounds[i] in [0, maxQuesCount-1] (HOST), with the rounds
 * 0..rounds[i]-1 they already had: the image row and round-0 history row as vd_dialog_join reads them; questions 0..r-1
 * from b->ques_fwd, right-aligned into the pool's width as asks do; answers (B, maxQuesCount, Ta) HOST word ids, row j
 * the answer to question j, left-aligned and zero-padded (zeros are not words; <END> = vocabSize ends one).  draw_base as
 * vd_dialog_join's, or NULL.  Afterwards a slot's history rows 0..r, question cache, facts and sh of rounds < r, dialog-LSTM
 * (h, c) after round r-1, round (r) and draw base are those of a conversation that joined at round 0 and was asked
 * q_0..q_{r-1} with the pool's answers replaced by a_0..a_{r-1} (in VD_MATH_FP32 bit for bit); round r's fact comes with
 * the next ask.  One encoder pass over the sum of the rounds' rows, one synchronisation.  lf-ques / lf-ques-im: only the
 * questions and the round are set, and answers may be NULL.
 * Refusals, before any state changes: VD_E_STATE for no pool, a stale pool or an occupied target slot; VD_E_BADARG for a
 * round outside [0, maxQuesCount-1], a slot outside [0, capacity) or named twice, Ta < 1, answer or question tokens
 * outside [0, vocabSize], null answers for a history encoder, hist_width < b->Th; VD_E_SHAPE for b->Tq above the pool's
 * question width. */
int vd_dialog_join_rounds(vd_engine* e, const vd_batch* b, const int32_t* rounds, const int32_t* answers, int32_t Ta,
                          const int64_t* draw_base, const int32_t* slots);

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
/* test hook of the engine's pointwise, attention, criterion, decoding and encoder-pair LSTM kernels and of its fused
 * vocabulary projections (the softmax-statistics, d-logit and sampling epilogues of the tensor-core GEMM): calls the launcher
 * `name` (the table in visdial_b200/csrc/test_hooks.cu lists each one's pointer / int / real arguments) on caller-provided
 * DEVICE buffers, on the
 * engine's stream, then synchronises.  Dropout factors are the engine's own for the seed and iteration of
 * vd_set_dropout_seed (identity unless training mode 1).  VD_E_BADARG for an unknown name or wrong argument counts; a
 * launcher's refusal comes back as its error code; a fused vocabulary projection refuses a shape with VD_E_SHAPE and launches
 * nothing.  Two entries reach the gen dense step rather than a kernel:
 * "dense_gen_chunk_bytes" sets its d-logit budget, "dense_scores" copies out the last dense step's (B, numOptions) scores. */
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
  int32_t imgAtt;               /* 1: images are (N,C,S,S) and are stored (N,S,S,C)        (:70-72);
                                   2: region features (N,P,C), stored as given (DESIGN §26) */
  int32_t imgChannels;          /* C (pool5 512) or F (fc7 4096)                                   */
  int32_t imgSpatial;           /* S (14) for imgAtt 1, P (regions per image) for imgAtt 2; ignored unless imgAtt */
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
  const float* images;          /* (N,F), (N,C,S,S) or (N,P,C) fp32 'images_<split>' of the image h5 (NULL unless useIm) */
} vd_corpus_desc;

/* dataloader:initialize tensors -> HBM + dataloader:prepareDataset on the device.  Host pointers. */
int vd_corpus_create(vd_engine* e, const vd_corpus_desc* d, vd_corpus** out);
/* vd_corpus_create with a limit: imgDeviceBytes is the most prepared image feature bytes (numImages x row x 4) the corpus
 * keeps on the device, 0 = no limit (vd_corpus_create).  A split over it keeps them in one pinned host allocation
 * (DESIGN §29), and each batch's rows are copied to the device by the copy engines; the batches are bit for bit the same.
 * VD_E_OOM when the pinned allocation fails. */
int vd_corpus_create_limited(vd_engine* e, const vd_corpus_desc* d, int64_t imgDeviceBytes, vd_corpus** out);
int vd_corpus_destroy(vd_corpus* c);
/* Assemble the batch of dialogs `inds` (HOST array of n 0-based dialog indices = Lua's inds - 1) on the engine's stream.
 *   decoder_gen = 0: getIndexData + getIndexOption('disc')  -> ques_fwd, hist, img_feat, answer_in/out, answer_ind, options
 *   decoder_gen = 1: getIndexData only (getTrainBatch, gen)  -> ... without options
 *   decoder_gen = 2: getIndexData + getIndexOption('gen')   -> ... plus option_in / option_out (getTestBatch, gen)
 * `out` receives DEVICE pointers (on_device = 1) into corpus-owned buffers that stay valid until the second-next
 * vd_corpus_get_batch on this corpus (two buffer sets, alternating). */
int vd_corpus_get_batch(vd_corpus* c, const int64_t* inds, int32_t n, int32_t decoder_gen, vd_batch* out);
/* Start copying the image rows of dialogs `inds` (HOST array of n 0-based indices) from a host-placed corpus's pinned
 * features into a landing buffer outside the two buffer sets, on the corpus's copy stream, behind the work already on the
 * engine's stream; returns without waiting.  The next vd_corpus_get_batch takes those rows when it is given the same n
 * indices in the same order, and copies its rows itself otherwise; either way it ends the prefetch.  Batches keep their
 * lifetime (until the second-next vd_corpus_get_batch).  Does nothing on a corpus whose features are on the device.
 * VD_E_SHAPE for n < 1 or an index out of range. */
int vd_corpus_prefetch(vd_corpus* c, const int64_t* inds, int32_t n);
/* Where the prepared image features are: *on_host = 1 in pinned host memory, 0 on the device; *bytes = their size
 * (0 without images).  Either pointer may be NULL. */
int vd_corpus_image_memory(vd_corpus* c, int32_t* on_host, int64_t* bytes);
/* Read one PREPARED tensor back to the host (parity tests): name in {"ques_fwd","hist","hist_len","ans_in","ans_out",
 * "opt_in","opt_out","img_fv"}, or "opt_list": the raw (numOptList, maxAnsLen) answer pool as uploaded, which the host no
 * longer keeps (the pool vd_answer_pool_encode takes); *elems receives the element count (call with host_dst = NULL to size). */
int vd_corpus_read(vd_corpus* c, const char* name, void* host_dst, int64_t* elems);
/* Region corpora (imgAtt = 2): counts_host (numImages) = 'num_boxes_<split>', each image's region count in [1, P].  Checks
 * every count (VD_E_BADARG, corpus unchanged, if one is outside), uploads them and zeroes every pad row (rows >= count) of
 * the resident features (on the host for a host-placed corpus, with the same +0.0f values).  Later batches carry img_count[b] = counts[img_pos[inds[b]]], gathered on the device.  Without
 * this call every region is present.  Once per corpus: the pad rows are zeroed in place, so a second call is VD_E_STATE,
 * as is a corpus without region features. */
int vd_corpus_region_counts(vd_corpus* c, const int32_t* counts_host, int64_t numImages);
/* bytes the last vd_corpus_get_batch read + wrote in HBM (algorithmic) and the number of kernels it launched */
int vd_corpus_batch_bytes(vd_corpus* c, int64_t* bytes, int32_t* launches);

#ifdef __cplusplus
}
#endif
#endif /* VISDIAL_B200_H */
