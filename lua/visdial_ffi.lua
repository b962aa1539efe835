-- LuaJIT-FFI binding of libvisdial_b200.so (include/visdial_b200.h).
-- AUTHORED, NOT EXECUTED: this image has no lua/luajit/th (SURVEY.md, container facts).  The same C ABI is
-- exercised call-for-call by visdial_b200/_lib.py (ctypes), which is what the tests drive.
local ffi = require 'ffi'

ffi.cdef[[
typedef struct vd_engine vd_engine;
typedef struct vd_params {
  const char* encoder; const char* decoder;
  int32_t vocabSize, embedSize, rnnHiddenSize, numLayers, imgFeatureSize, imgSpatialSize, imgEmbedSize,
          commonEmbeddingSize, numAttentionLayers, maxQuesCount, numOptions;
  float dropout; int32_t gpuid;
  int32_t imgRegions;            /* 0: the S x S grid; P > 0: P region rows per image (att encoders) */
} vd_params;
typedef struct vd_batch {
  int32_t B, Tq, Th, Ta, To;
  const int32_t* ques_fwd; const int32_t* hist; const float* img_feat; const int32_t* options;
  const int32_t* answer_ind; const int32_t* answer_in; const int32_t* answer_out;
  const int32_t* option_in; const int32_t* option_out; int32_t on_device;
  const int32_t* img_count;      /* (B) region counts in [1, imgRegions], NULL = every region present */
} vd_batch;
const char* vd_last_error(void);
int vd_create(const vd_params* p, vd_engine** out);
int vd_destroy(vd_engine* e);
int vd_num_params(vd_engine* e, int64_t* n);
int vd_param_buffers(vd_engine* e, float** W_dev, float** dW_dev);
int vd_set_parameters(vd_engine* e, const float* host_src, int64_t n);
int vd_get_parameters(vd_engine* e, float* host_dst, int64_t n);
int vd_zero_grad(vd_engine* e);
int vd_set_training(vd_engine* e, int32_t training);
int vd_set_dropout_seed(vd_engine* e, uint64_t seed, uint64_t iteration);
int vd_set_deterministic(vd_engine* e, int32_t on);   /* 1: training steps repeat bit for bit (DESIGN §27); one GPU */
int vd_encoder_forward(vd_engine* e, const vd_batch* b, const float** encOut_dev);
int vd_forward_connect(vd_engine* e);
int vd_decoder_forward(vd_engine* e, const vd_batch* b, const float** decOut_dev);
int vd_criterion_forward(vd_engine* e, const vd_batch* b, float* loss_host);
int vd_criterion_backward(vd_engine* e, const vd_batch* b);
int vd_decoder_backward(vd_engine* e, const vd_batch* b);
int vd_backward_connect(vd_engine* e, const float** gradEncOut_dev);
int vd_encoder_backward(vd_engine* e, const vd_batch* b, const float* gradEncOut_dev);
int vd_forward_backward(vd_engine* e, const vd_batch* b, int32_t only_forward, float* loss_host);
int vd_forward_backward_dense(vd_engine* e, const vd_batch* b, const int32_t* round_host, const float* relevance_host,
                              float* loss_host);
int vd_forward_backward_dense_gen(vd_engine* e, const vd_batch* b, const int32_t* round_host, const float* relevance_host,
                                  float* loss_host);
int vd_retrieve(vd_engine* e, const vd_batch* b, int32_t use_gt, int32_t* ranks_host);
int vd_gen_beam_search(vd_engine* e, int32_t beam_size, int32_t beam_len, int32_t start_token, int32_t end_token,
                       int32_t* answer_host, int32_t* length_host, double* score_host);
int vd_gen_diverse_beam_search(vd_engine* e, int32_t beam_size, int32_t groups, float diversity, int32_t beam_len,
                               int32_t start_token, int32_t end_token, int32_t* answer_host, int32_t* length_host,
                               double* score_host);
int vd_gen_nbest_beam_search(vd_engine* e, int32_t beam_size, int32_t groups, float diversity, float length_penalty,
                             int32_t nbest, int32_t beam_len, int32_t start_token, int32_t end_token, int32_t* answer_host,
                             int32_t* length_host, double* score_host, double* norm_host);
int vd_gen_sample(vd_engine* e, int32_t beam_len, int32_t start_token, float temperature, uint64_t seed, int64_t row_offset,
                  int32_t* answer_host, float* logp_host);
int vd_gen_dialog_beam_search(vd_engine* e, const vd_batch* b, int32_t beam_size, int32_t beam_len, int32_t start_token,
                              int32_t end_token, int32_t hist_width, int32_t max_ans_len, int32_t* answer_host,
                              int32_t* length_host, double* score_host, int32_t* hist_host);
int vd_gen_dialog_sample(vd_engine* e, const vd_batch* b, int32_t beam_len, int32_t start_token, int32_t end_token,
                         float temperature, uint64_t seed, int64_t row_offset, int32_t hist_width, int32_t max_ans_len,
                         int32_t* answer_host, float* logp_host, int32_t* hist_host);
int vd_gen_dialog_diverse_beam_search(vd_engine* e, const vd_batch* b, int32_t beam_size, int32_t groups, float diversity,
                                      int32_t beam_len, int32_t start_token, int32_t end_token, int32_t hist_width,
                                      int32_t max_ans_len, int32_t* answer_host, int32_t* length_host, double* score_host,
                                      int32_t* hist_host);
int vd_gen_dialog_nbest_beam_search(vd_engine* e, const vd_batch* b, int32_t beam_size, int32_t groups, float diversity,
                                    float length_penalty, int32_t nbest, int32_t beam_len, int32_t start_token,
                                    int32_t end_token, int32_t hist_width, int32_t max_ans_len, int32_t* answer_host,
                                    int32_t* length_host, double* score_host, double* norm_host, int32_t* hist_host);
typedef struct vd_answer_rules {
  int32_t min_words; int32_t no_repeat_ngram; int32_t n_banned; const int32_t* banned;
} vd_answer_rules;
int vd_set_answer_rules(vd_engine* e, const vd_answer_rules* r);
int vd_gen_truncated_sample(vd_engine* e, int32_t beam_len, int32_t start_token, float temperature, uint64_t seed,
                            int64_t row_offset, int32_t top_k, float top_p, int32_t* answer_host, float* logp_host);
int vd_gen_dialog_truncated_sample(vd_engine* e, const vd_batch* b, int32_t beam_len, int32_t start_token, int32_t end_token,
                                   float temperature, uint64_t seed, int64_t row_offset, int32_t top_k, float top_p,
                                   int32_t hist_width, int32_t max_ans_len, int32_t* answer_host, float* logp_host,
                                   int32_t* hist_host);
int vd_answer_pool_encode(vd_engine* e, const int32_t* tokens_host, int64_t m, int32_t width);
int vd_answer_pool(vd_engine* e, const float** emb_dev, int64_t* m);
int vd_answer_pool_retrieve(vd_engine* e, const vd_batch* b, int32_t k, int32_t* index_host, float* score_host);
int vd_answer_pool_dialog(vd_engine* e, const vd_batch* b, int32_t k, int32_t hist_width, int32_t max_ans_len,
                          int32_t* index_host, float* score_host, int32_t* hist_host);
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
int vd_dialog_ask_diverse_slots(vd_engine* e, const int32_t* slots, int32_t n, const int32_t* ques, int32_t Tq, int32_t beam_size,
                                int32_t groups, float diversity, int32_t beam_len, int32_t start_token, int32_t end_token,
                                int32_t* answer, int32_t* length, double* score);
int vd_dialog_ask_nbest_slots(vd_engine* e, const int32_t* slots, int32_t n, const int32_t* ques, int32_t Tq, int32_t beam_size,
                              int32_t groups, float diversity, float length_penalty, int32_t nbest, int32_t beam_len,
                              int32_t start_token, int32_t end_token, int32_t* answer, int32_t* length, double* score,
                              double* norm);
int vd_dialog_ask_truncated_slots(vd_engine* e, const int32_t* slots, int32_t n, const int32_t* ques, int32_t Tq,
                                  int32_t beam_len, int32_t start_token, int32_t end_token, float temperature, uint64_t seed,
                                  int64_t row_offset, int32_t top_k, float top_p, int32_t* answer, float* logp);
int vd_dialog_slots(vd_engine* e, int32_t* rounds, int32_t* capacity);
int vd_dialog_slot_history(vd_engine* e, const int32_t* slots, int32_t n, int32_t* hist);
int vd_dialog_join_rounds(vd_engine* e, const vd_batch* b, const int32_t* rounds, const int32_t* answers, int32_t Ta,
                          const int64_t* draw_base, const int32_t* slots);
int vd_clamp_adam_step(vd_engine* e, float learning_rate);
int vd_comm_unique_id(void* id_out);
int vd_comm_init(vd_engine* e, const void* id, int32_t rank, int32_t world);
int vd_memcpy_d2h(vd_engine* e, void* host_dst, const void* dev_src, size_t bytes);
int vd_synchronize(vd_engine* e);
/* dataloader on the device (dataloader.lua:143-478) */
typedef struct vd_corpus vd_corpus;
typedef struct vd_corpus_desc {
  int32_t numThreads, numRounds, maxQuesLen, maxAnsLen, maxCapLen, numOptions, numOptList, numImages;
  int32_t useHistory, concatHistory, useIm, maxHistoryLen, imgNorm, imgAtt, imgChannels, imgSpatial;
  int32_t startToken, endToken;
  const int32_t *ques, *ques_len, *ans, *ans_len, *cap, *cap_len, *opt, *opt_list, *opt_len, *ans_index, *img_pos, *num_rounds;
  const float* images;
} vd_corpus_desc;
int vd_corpus_create(vd_engine* e, const vd_corpus_desc* d, vd_corpus** out);
int vd_corpus_destroy(vd_corpus* c);
int vd_corpus_get_batch(vd_corpus* c, const int64_t* inds, int32_t n, int32_t decoder_gen, vd_batch* out);
]]

local M = {}
M.C = ffi.load('visdial_b200')   -- libvisdial_b200.so on package.cpath / LD_LIBRARY_PATH

-- rc ~= 0 becomes a Lua error, like the reference's error()/assert (model.lua:436, weight-init.lua:46)
function M.check(rc)
  if rc ~= 0 then error(string.format('visdial_b200 error %d: %s', rc, ffi.string(M.C.vd_last_error()))) end
end

-- modelParams table (opts.lua:6-40 + train.lua:55-59) -> vd_params
function M.params(p)
  local c = ffi.new('vd_params')
  M._enc, M._dec = p.encoder, p.decoder          -- keep the strings alive
  c.encoder, c.decoder = p.encoder, p.decoder
  c.vocabSize = p.vocabSize; c.embedSize = p.embedSize; c.rnnHiddenSize = p.rnnHiddenSize
  c.numLayers = p.numLayers; c.imgFeatureSize = p.imgFeatureSize; c.imgSpatialSize = p.imgSpatialSize or 14
  c.imgEmbedSize = p.imgEmbedSize; c.commonEmbeddingSize = p.commonEmbeddingSize or 512
  c.numAttentionLayers = p.numAttentionLayers or 1; c.maxQuesCount = p.maxQuesCount or 10
  c.numOptions = p.numOptions or 100; c.dropout = p.dropout or 0.5; c.gpuid = p.gpuid
  return c
end

-- dataloader batch table (dataloader.lua:324-478) -> vd_batch.  Ids are IntTensors on the host
-- (`:int():contiguous()`); the engine stages them to the device itself.  The converted tensors are temporaries: only
-- their data pointers go into the struct, so they are ANCHORED in the returned table (`keep`) — otherwise LuaJIT may
-- collect them before vd_encoder_forward has copied them (any ffi.new in between can trigger a GC cycle).  The caller
-- holds the returned table until the step's last call that reads the batch (criterion / backward) has returned.
function M.batch(b)
  local c = ffi.new('vd_batch')
  local keep = {}
  local function ip(t)
    if not t then return nil end
    local ti = t:int():contiguous()
    keep[#keep + 1] = ti
    return ffi.cast('const int32_t*', ti:data())
  end
  c.B = b.ques_fwd:size(1); c.Tq = b.ques_fwd:size(3)
  c.ques_fwd = ip(b.ques_fwd)
  if b.hist then c.Th = b.hist:size(3); c.hist = ip(b.hist) end
  if b.img_feat then
    local tf = b.img_feat:float():contiguous()
    keep[#keep + 1] = tf
    c.img_feat = ffi.cast('const float*', tf:data())
  end
  if b.options then c.To = b.options:size(3); c.options = ip(b.options) end
  if b.answer_ind then c.answer_ind = ip(b.answer_ind) end
  if b.answer_in then c.Ta = b.answer_in:size(3); c.answer_in = ip(b.answer_in); c.answer_out = ip(b.answer_out) end
  if b.option_in then c.To = b.option_in:size(4); c.option_in = ip(b.option_in); c.option_out = ip(b.option_out) end
  c.on_device = 0
  return {c = c, keep = keep}
end

return M
