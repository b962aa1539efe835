// Engine orchestration: replaces Model:forwardBackward / retrieveBatch (/root/reference/model.lua:249-430)
// and the nn graphs of encoders/*.lua + decoders/*.lua for the four configured encoders.
#include "engine.h"
#include <string.h>
#include <math.h>
#include <cmath>
#include <algorithm>

namespace vd {

// ------------------------------------------------------------------------------------------------
// config + parameter layout (DESIGN.md §3)
// ------------------------------------------------------------------------------------------------
Cfg parse_cfg(const vd_params* p) {
  VD_REQUIRE(p && p->encoder && p->decoder, VD_E_BADARG, "params / encoder / decoder is null");
  Cfg c;
  c.encoder = p->encoder; c.decoder = p->decoder;
  struct { const char* name; int enc; } known[] = {
      {"lf-ques", ENC_LF_QUES}, {"lf-ques-im-hist", ENC_LF_QIH}, {"hrea-ques-im-hist", ENC_HREA}, {"mn-att-ques-im-hist", ENC_MN_ATT},
      {"lf-ques-im", ENC_LF_QI}, {"lf-ques-hist", ENC_LF_QH}, {"hre-ques-hist", ENC_HRE_QH}, {"hre-ques-im-hist", ENC_HRE_QIH},
      {"mn-ques-hist", ENC_MN_QH}, {"mn-ques-im-hist", ENC_MN_QIH}, {"lf-att-ques-im-hist", ENC_LF_ATT}};
  c.enc = -1;
  for (auto& k : known)
    if (c.encoder == k.name) c.enc = k.enc;
  VD_REQUIRE(c.enc >= 0, VD_E_BADARG, "unknown encoder (one of the eleven names of encoders/*.lua)");
  if (c.decoder == "disc") c.dec = DEC_DISC;
  else if (c.decoder == "gen") c.dec = DEC_GEN;
  else VD_REQUIRE(false, VD_E_BADARG, "unknown decoder (disc | gen)");
  c.V = p->vocabSize; c.E = p->embedSize; c.H = p->rnnHiddenSize; c.L = p->numLayers; c.F = p->imgFeatureSize;
  c.S = p->imgSpatialSize; c.IE = p->imgEmbedSize; c.Cm = p->commonEmbeddingSize; c.hops = p->numAttentionLayers;
  c.regions = p->imgRegions;
  c.R = p->maxQuesCount; c.K = p->numOptions; c.dropout = p->dropout; c.gpuid = p->gpuid;
  // opts.lua:55-59,62
  c.useHist = c.encoder.find("hist") != std::string::npos;
  c.useIm = c.encoder.find("im") != std::string::npos;
  c.att = c.encoder.find("att") != std::string::npos;
  c.fam_lf = c.encoder.compare(0, 3, "lf-") == 0;
  c.fam_hre = c.encoder.compare(0, 3, "hre") == 0;
  c.fam_mn = c.encoder.compare(0, 3, "mn-") == 0;
  c.hre_att = c.enc == ENC_HREA;
  c.san = c.att;
  c.img_in_q = c.fam_hre && c.useIm;
  c.img_drop = c.enc == ENC_HREA;
  c.mn_qi = c.enc == ENC_MN_QIH;
  c.embdrop = c.fam_mn || c.enc == ENC_LF_ATT;
  c.rnn_layers = (c.fam_lf && !c.att) || c.fam_hre;
  VD_REQUIRE(c.regions >= 0 && c.regions <= 4096, VD_E_BADARG, "imgRegions must be in [0, 4096]");
  VD_REQUIRE(c.regions == 0 || c.att, VD_E_BADARG, "region features (imgRegions > 0) are for the att encoders only");
  c.P = c.regions > 0 ? c.regions : c.S * c.S;
  // k_san_att_bwd stages a dialog round's du, p and dp rows in (H + 2P + 33) floats of shared memory (48 KB without opt-in)
  VD_REQUIRE(!c.san || (int64_t)c.H + 2 * (int64_t)c.P + 33 <= 12288, VD_E_BADARG,
             "attention positions too many for rnnHiddenSize: rnnHiddenSize + 2 * positions must be <= 12255");
  if (c.enc == ENC_LF_ATT) c.hops = 1;           // hard-wired upstream: lf-att-ques-im-hist.lua:49 does not read params.numAttentionLayers
  VD_REQUIRE(c.V > 2 && c.E > 0 && c.H > 0, VD_E_BADARG, "vocabSize / embedSize / rnnHiddenSize must be positive");
  VD_REQUIRE(c.L == 2, VD_E_BADARG, "numLayers must be 2");
  VD_REQUIRE(c.E % 4 == 0 && c.H % 32 == 0 && c.IE % 4 == 0 && c.Cm % 4 == 0 && c.F % 4 == 0, VD_E_BADARG,
             "embedSize/imgEmbedSize/commonEmbeddingSize/imgFeatureSize must be multiples of 4, rnnHiddenSize of 32");
  VD_REQUIRE(c.R >= 1 && c.R <= 32 && c.K >= 1 && c.K <= 1024 && c.hops >= 1, VD_E_BADARG, "maxQuesCount/numOptions/numAttentionLayers out of range");
  VD_REQUIRE(c.dropout >= 0.f && c.dropout < 1.f, VD_E_BADARG, "dropout must be in [0,1)");
  return c;
}

int Layout::find(const std::string& name) const {
  for (size_t i = 0; i < segs.size(); ++i)
    if (segs[i].name == name) return (int)i;
  return -1;
}

static void add_seg(Layout& l, const std::string& name, int64_t rows, int64_t cols, int init, int64_t fan_in) {
  Seg s; s.name = name; s.rows = rows; s.cols = cols; s.init = init; s.fan_in = fan_in; s.off = l.total;
  l.segs.push_back(s);
  l.total += (rows * cols + 31) / 32 * 32;       // every segment starts 128-byte aligned
}
static void add_lstm(Layout& l, const std::string& n, int D, int H) {
  add_seg(l, n + ".weight", D + H, 4 * H, VD_INIT_LSTM_W, D + H);
  add_seg(l, n + ".bias", 1, 4 * H, VD_INIT_LSTM_B, D + H);
}
static void add_linear(Layout& l, const std::string& n, int out, int in) {
  add_seg(l, n + ".weight", out, in, VD_INIT_LINEAR_W, in);
  add_seg(l, n + ".bias", 1, out, VD_INIT_LINEAR_B, in);
}

Layout build_layout(const Cfg& c) {
  Layout l;
  add_seg(l, "wordEmbed.weight", c.V + 1, c.E, VD_INIT_EMBED, 0);
  auto add_san = [&]() {
    add_linear(l, "san.img", c.H, c.F);
    for (int h = 1; h <= c.hops; ++h) {
      std::string p = "san.hop" + std::to_string(h) + ".";
      add_linear(l, p + "img_common", c.Cm, c.H);
      add_linear(l, p + "ques_common", c.Cm, c.H);
      add_linear(l, p + "score", 1, c.Cm);
    }
    add_linear(l, "san.out", c.H, c.H);
  };
  if (c.fam_lf && !c.san) {
    // lf-ques / lf-ques-im / lf-ques-hist / lf-ques-im-hist: fusion over [q | img | h]
    add_lstm(l, "ques.lstm1", c.E, c.H); add_lstm(l, "ques.lstm2", c.H, c.H);
    if (c.useHist) { add_lstm(l, "hist.lstm1", c.E, c.H); add_lstm(l, "hist.lstm2", c.H, c.H); }
    add_linear(l, "fusion", c.H, c.H + (c.useIm ? c.F : 0) + (c.useHist ? c.H : 0));
  } else if (c.fam_hre) {
    if (c.img_in_q) add_linear(l, "img.embed", c.IE, c.F);
    add_lstm(l, "hist.lstm1", c.E, c.H); add_lstm(l, "hist.lstm2", c.H, c.H);
    add_lstm(l, "ques.lstm1", c.E + (c.img_in_q ? c.IE : 0), c.H); add_lstm(l, "ques.lstm2", c.H, c.H);
    if (c.hre_att) { add_linear(l, "att.q", 1, c.H); add_linear(l, "att.h", 1, c.H); }
    add_lstm(l, "dialog.lstm", 2 * c.H, c.H);
  } else {
    // mn-* and lf-att-ques-im-hist: history then question LSTMs, then the attention blocks
    add_lstm(l, "hist.lstm1", c.E, c.H); add_lstm(l, "hist.lstm2", c.H, c.H);
    add_lstm(l, "ques.lstm1", c.E, c.H); add_lstm(l, "ques.lstm2", c.H, c.H);
    if (c.fam_lf) add_linear(l, "fusion", c.H, 2 * c.H);                   // lf-att: tanh(Linear([q | h]))
    if (c.mn_qi) add_linear(l, "mn.qi", c.H, c.H + c.F);                   // mn-ques-im-hist: tanh(Linear([q | fc7]))
    if (c.fam_mn) { add_linear(l, "mn.fact", c.H, c.H); add_linear(l, "mn.query", c.H, c.H); }
    if (c.san) add_san();
  }
  if (c.dec == DEC_DISC) {
    add_lstm(l, "opt.lstm", c.E, c.H);
  } else {
    add_lstm(l, "dec.lstm1", c.E, c.H); add_lstm(l, "dec.lstm2", c.H, c.H);
    add_linear(l, "dec.out", c.V, c.H);
  }
  return l;
}

// ------------------------------------------------------------------------------------------------
// memory
// ------------------------------------------------------------------------------------------------
void* Arena::alloc(size_t bytes) {
  bytes = (bytes + 255) & ~(size_t)255;
  if (bytes == 0) bytes = 256;
  while (cur < chunks.size()) {
    Chunk& c = chunks[cur];
    if (c.used + bytes <= c.cap) { void* p = c.p + c.used; c.used += bytes; return p; }
    ++cur;
  }
  Chunk c; c.cap = std::max<size_t>(bytes, (size_t)256 << 20); c.used = bytes;
  VD_CUDA_CHECK(cudaMalloc((void**)&c.p, c.cap));
  chunks.push_back(c);
  cur = chunks.size() - 1;
  return c.p;
}
void Arena::reset() { for (auto& c : chunks) c.used = 0; cur = 0; }
void Arena::release() { for (auto& c : chunks) cudaFree(c.p); chunks.clear(); cur = 0; }
void Arena::rewind(const Mark& m) {
  for (size_t i = m.chunk; i < chunks.size(); ++i) chunks[i].used = i == m.chunk ? m.used : 0;   // chunks past `cur` are unused
  cur = m.chunk;
}

void* GrowBuf::ensure(size_t bytes) {
  if (bytes > cap) {
    if (p) cudaFree(p);
    p = nullptr; cap = 0;
    VD_CUDA_CHECK(cudaMalloc(&p, bytes));
    cap = bytes;
  }
  return p;
}
void GrowBuf::release() { if (p) cudaFree(p); p = nullptr; cap = 0; }

// ------------------------------------------------------------------------------------------------
Engine::Engine(const vd_params* p) {
  cfg = parse_cfg(p);
  lay = build_layout(cfg);
  nparams = lay.total;
  int ndev = 0;
  VD_CUDA_CHECK(cudaGetDeviceCount(&ndev));
  VD_REQUIRE(cfg.gpuid >= 0 && cfg.gpuid < ndev, VD_E_BADARG, "gpuid out of range");
  VD_CUDA_CHECK(cudaSetDevice(cfg.gpuid));
  cudaDeviceProp prop;
  VD_CUDA_CHECK(cudaGetDeviceProperties(&prop, cfg.gpuid));
  VD_REQUIRE(prop.major == 9 && prop.minor == 0, VD_E_CUDA, "visdial_b200 is built for sm_90a (H100) only");
  cx.sm_count = prop.multiProcessorCount;
  cx.scratch = [this](size_t bytes) { return arena.alloc(bytes); };
  // the encoder's chains of small dependent kernels get the highest priority, the option LSTM's SM-filling launches
  // the lowest: a freed SM goes to the latency-bound chain first
  int prio_lo = 0, prio_hi = 0;
  VD_CUDA_CHECK(cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));
  VD_CUDA_CHECK(cudaStreamCreateWithPriority(&cx.stream, cudaStreamNonBlocking, prio_hi));
  main_stream = cx.stream;
  VD_CUDA_CHECK(cudaStreamCreateWithPriority(&side_stream, cudaStreamNonBlocking, prio_hi));
  main_chain.a = main_stream; side_chain.a = side_stream;
  for (cudaStream_t* s : {&main_chain.b, &side_chain.b, &main_chain.c, &side_chain.c})
    VD_CUDA_CHECK(cudaStreamCreateWithPriority(s, cudaStreamNonBlocking, prio_hi));
  VD_CUDA_CHECK(cudaStreamCreateWithPriority(&opt_stream, cudaStreamNonBlocking, prio_lo));
  VD_CUDA_CHECK(cudaEventCreateWithFlags(&ev_fork, cudaEventDisableTiming));
  VD_CUDA_CHECK(cudaEventCreateWithFlags(&ev_join, cudaEventDisableTiming));
  VD_CUDA_CHECK(cudaEventCreateWithFlags(&ev_opt_fork, cudaEventDisableTiming));
  VD_CUDA_CHECK(cudaEventCreateWithFlags(&ev_opt_done, cudaEventDisableTiming));
  size_t bytes = (size_t)nparams * sizeof(float);
  VD_CUDA_CHECK(cudaMalloc((void**)&W, bytes));
  VD_CUDA_CHECK(cudaMalloc((void**)&dW, bytes));
  VD_CUDA_CHECK(cudaMalloc((void**)&m, bytes));
  VD_CUDA_CHECK(cudaMalloc((void**)&v, bytes));
  VD_CUDA_CHECK(cudaMalloc((void**)&Wt, bytes));
  VD_CUDA_CHECK(cudaMemsetAsync(W, 0, bytes, cx.stream));
  VD_CUDA_CHECK(cudaMemsetAsync(dW, 0, bytes, cx.stream));
  VD_CUDA_CHECK(cudaMemsetAsync(m, 0, bytes, cx.stream));
  VD_CUDA_CHECK(cudaMemsetAsync(v, 0, bytes, cx.stream));
  VD_CUDA_CHECK(cudaMemsetAsync(Wt, 0, bytes, cx.stream));
  VD_CUDA_CHECK(cudaMalloc((void**)&scalars_dev, 64 * sizeof(float)));
  // table of 2-D weight segments that get a transposed shadow copy
  std::vector<int64_t> tab;
  for (auto& s : lay.segs) {
    if (s.init == VD_INIT_LSTM_W || s.init == VD_INIT_LINEAR_W) {
      tab.push_back(s.off); tab.push_back(s.rows); tab.push_back(s.cols);
      max2d = std::max(max2d, s.rows * s.cols);
    }
  }
  nseg2d = (int)tab.size() / 3;
  VD_CUDA_CHECK(cudaMalloc((void**)&segtab_dev, tab.size() * sizeof(int64_t)));
  VD_CUDA_CHECK(cudaMemcpyAsync(segtab_dev, tab.data(), tab.size() * sizeof(int64_t), cudaMemcpyHostToDevice, cx.stream));
  VD_CUDA_CHECK(cudaStreamSynchronize(cx.stream));
  VD_CUDA_CHECK(cudaEventCreate(&t0));
  VD_CUDA_CHECK(cudaEventCreate(&t1));
}

Engine::~Engine() {
  cudaSetDevice(cfg.gpuid);
  cudaStreamSynchronize(cx.stream);
  if (opt_stream) cudaStreamSynchronize(opt_stream);
  arena.release();
  for (auto& g : stage) g.release();
  for (auto& g : dense_buf) g.release();
  dialog_hist.release();
  beam_lp.release();
  rules_banned.release();
  for (auto& g : dialog_out) g.release();
  if (copy_stream) {
    cudaStreamSynchronize(copy_stream); cudaStreamDestroy(copy_stream);
    cudaEventDestroy(ev_img_ready); cudaEventDestroy(ev_copy_fork);
    for (auto ev : ev_img_free) cudaEventDestroy(ev);
  }
  for (auto& g : stage_img) g.release();
  cudaFree(W); cudaFree(dW); cudaFree(m); cudaFree(v); cudaFree(Wt); cudaFree(scalars_dev); cudaFree(segtab_dev);
  if (flush_buf) cudaFree(flush_buf);
  cx.collect();
  for (auto e : cx.free_events) cudaEventDestroy(e);
  if (t0) cudaEventDestroy(t0);
  if (t1) cudaEventDestroy(t1);
  if (ev_fork) cudaEventDestroy(ev_fork);
  if (ev_join) cudaEventDestroy(ev_join);
  if (side_stream) { cudaStreamSynchronize(side_stream); cudaStreamDestroy(side_stream); }
  for (cudaStream_t s : {main_chain.b, side_chain.b, main_chain.c, side_chain.c})
    if (s) { cudaStreamSynchronize(s); cudaStreamDestroy(s); }
  if (opt_stream) { cudaStreamSynchronize(opt_stream); cudaStreamDestroy(opt_stream); }
  if (ev_opt_fork) cudaEventDestroy(ev_opt_fork);
  if (ev_opt_done) cudaEventDestroy(ev_opt_done);
  for (auto e : ev_pool) cudaEventDestroy(e);
  cudaStreamDestroy(main_stream);
}

int Engine::seg(const char* name) const {
  int i = lay.find(name);
  VD_REQUIRE(i >= 0, VD_E_STATE, name);
  return i;
}

DropCfg Engine::dropcfg(float p) const {
  DropCfg d;
  d.seed_lo = (uint32_t)drop_seed; d.seed_hi = (uint32_t)(drop_seed >> 32); d.iter = (uint32_t)drop_iter;
  if (training == 1 && p > 0.f) {
    double t = (double)p * 4294967296.0;
    d.thresh = (uint32_t)std::min(t, 4294967295.0);
    d.scale = 1.f / (1.f - p);
  } else { d.thresh = 0; d.scale = 1.f; }
  return d;
}

void Engine::gemm_tn(int M, int N, int K, const float* A, int64_t lda, const int32_t* gather, const float* B, int64_t ldb,
                     float* C, int64_t ldc, float beta, const float* bias, int act) {
  LaunchCtx::Scope sc(&cx, "gemm", 2.0 * M * N * K, 4.0 * ((double)M * K + (double)N * K + (double)M * N));
  if (tcmode() && gemm_tn_tc(cx, M, N, K, A, lda, gather, B, ldb, C, ldc, beta, bias, act)) return;
  gemm_tn_simt(cx, M, N, K, A, lda, gather, B, ldb, C, ldc, beta, bias, act);
}
void Engine::gemm_atb(int M, int N, int64_t K, const float* A, int64_t lda, const int32_t* gather, const float* B,
                      int64_t ldb, float* C, int64_t ldc) {
  LaunchCtx::Scope sc(&cx, "gemm_wgrad", 2.0 * M * N * K, 4.0 * ((double)M * K + (double)N * K + (double)M * N));
  if (tcmode() && gemm_atb_tc(cx, M, N, K, A, lda, gather, B, ldb, C, ldc)) return;
  gemm_atb_simt(cx, M, N, K, A, lda, gather, B, ldb, C, ldc);
}

void Engine::linear_fwd(int wseg, const float* x, int64_t rows, float* y, int act) {
  const Seg& s = lay.segs[wseg];
  gemm_tn((int)rows, (int)s.rows, (int)s.cols, x, s.cols, nullptr, Wp(wseg), s.cols, y, s.rows, 0.f, Wp(wseg + 1), act);
}
void Engine::linear_bwd(int wseg, const float* x, const float* dy, int64_t rows, float* dx, float beta_dx) {
  const Seg& s = lay.segs[wseg];
  int out = (int)s.rows, in = (int)s.cols;
  gemm_atb(out, in, rows, dy, out, nullptr, x, in, dWp(wseg), in);
  colsum_add(cx, dWp(wseg + 1), dy, rows, out, out);
  if (dx) gemm_tn((int)rows, in, out, dy, out, nullptr, Wtp(wseg), out, dx, in, beta_dx, nullptr, 0);
}

void Engine::refresh_shadows() {
  // LookupTableMaskZero.updateOutput zeroes the pad row at every forward [upstream rnn]
  VD_CUDA_CHECK(cudaMemsetAsync(W, 0, (size_t)cfg.E * sizeof(float), cx.stream));
  transpose_segments(cx, W, Wt, segtab_dev, nseg2d, max2d);
}

void Engine::stage_batch(const vd_batch* b) {
  VD_REQUIRE(b != nullptr, VD_E_BADARG, "batch is null");
  VD_REQUIRE(b->B > 0, VD_E_SHAPE, "batch B must be > 0");
  db = DevBatch();
  db.B = b->B; db.N = (int64_t)b->B * cfg.R;
  db.Tq = b->Tq; db.Th = b->Th; db.Ta = b->Ta; db.To = b->To;
  VD_REQUIRE(b->ques_fwd && b->Tq > 0, VD_E_SHAPE, "ques_fwd / Tq missing");
  if (cfg.useHist) VD_REQUIRE(b->hist && b->Th > 0, VD_E_SHAPE, "encoder uses history: hist / Th missing");
  if (cfg.useIm) VD_REQUIRE(b->img_feat, VD_E_SHAPE, "encoder uses the image: img_feat missing");
  int64_t img_elems = cfg.att ? (int64_t)b->B * cfg.P * cfg.F : (int64_t)b->B * cfg.F;
  if (b->img_count) {
    VD_REQUIRE(cfg.regions > 0, VD_E_BADARG, "img_count is for region engines (imgRegions > 0) only");
    if (b->on_device) {
      db.img_count = b->img_count;             // [1, P] is the caller's precondition (a corpus checked its counts)
    } else {
      for (int i = 0; i < b->B; ++i)
        VD_REQUIRE(b->img_count[i] >= 1 && b->img_count[i] <= cfg.P, VD_E_BADARG, "img_count outside [1, imgRegions]");
      int32_t* d = (int32_t*)stage_cnt.ensure((size_t)b->B * sizeof(int32_t));
      VD_CUDA_CHECK(cudaMemcpyAsync(d, b->img_count, (size_t)b->B * sizeof(int32_t), cudaMemcpyHostToDevice, cx.stream));
      db.img_count = d;
    }
  }
  struct Item { const void* src; size_t bytes; const void** dst; } items[9] = {
      {b->ques_fwd, (size_t)db.N * b->Tq * 4, (const void**)&db.ques},
      {cfg.useHist ? b->hist : nullptr, (size_t)db.N * b->Th * 4, (const void**)&db.hist},
      {cfg.useIm ? b->img_feat : nullptr, (size_t)img_elems * 4, (const void**)&db.img},
      {b->options, (size_t)db.N * cfg.K * b->To * 4, (const void**)&db.options},
      {b->answer_ind, (size_t)db.N * 4, (const void**)&db.answer_ind},
      {b->answer_in, (size_t)db.N * b->Ta * 4, (const void**)&db.answer_in},
      {b->answer_out, (size_t)db.N * b->Ta * 4, (const void**)&db.answer_out},
      {b->option_in, (size_t)db.N * cfg.K * b->To * 4, (const void**)&db.option_in},
      {b->option_out, (size_t)db.N * cfg.K * b->To * 4, (const void**)&db.option_out}};
  img_copy_pending = false;
  for (int i = 0; i < 9; ++i) {
    if (!items[i].src || items[i].bytes == 0) { *items[i].dst = nullptr; continue; }
    if (b->on_device) { *items[i].dst = items[i].src; continue; }
    if (i == 2 && items[i].bytes >= ((size_t)1 << 20)) {
      // image features: asynchronous copy on the copy stream into the staging buffer the previous step is not using
      if (!copy_stream) {
        VD_CUDA_CHECK(cudaStreamCreateWithFlags(&copy_stream, cudaStreamNonBlocking));
        VD_CUDA_CHECK(cudaEventCreateWithFlags(&ev_img_ready, cudaEventDisableTiming));
        VD_CUDA_CHECK(cudaEventCreateWithFlags(&ev_copy_fork, cudaEventDisableTiming));
        for (int k = 0; k < 2; ++k) VD_CUDA_CHECK(cudaEventCreateWithFlags(&ev_img_free[k], cudaEventDisableTiming));
      }
      img_slot ^= 1;
      if (items[i].bytes > stage_img[img_slot].cap) VD_CUDA_CHECK(cudaStreamSynchronize(copy_stream));   // growing frees the old block
      void* d = stage_img[img_slot].ensure(items[i].bytes);
      VD_CUDA_CHECK(cudaEventRecord(ev_copy_fork, cx.stream));                  // stream order behind whatever freed / allocated before
      VD_CUDA_CHECK(cudaStreamWaitEvent(copy_stream, ev_copy_fork, 0));
      if (img_free_recorded[img_slot]) VD_CUDA_CHECK(cudaStreamWaitEvent(copy_stream, ev_img_free[img_slot], 0));
      VD_CUDA_CHECK(cudaMemcpyAsync(d, items[i].src, items[i].bytes, cudaMemcpyHostToDevice, copy_stream));
      VD_CUDA_CHECK(cudaEventRecord(ev_img_ready, copy_stream));
      img_copy_pending = true;
      *items[i].dst = d;
      continue;
    }
    void* d = stage[i].ensure(items[i].bytes);
    VD_CUDA_CHECK(cudaMemcpyAsync(d, items[i].src, items[i].bytes, cudaMemcpyHostToDevice, cx.stream));
    *items[i].dst = d;
  }
}

void Engine::wait_img() {
  if (!img_copy_pending) return;
  VD_CUDA_CHECK(cudaStreamWaitEvent(cx.stream, ev_img_ready, 0));
  if (cx.stream != main_stream) VD_CUDA_CHECK(cudaStreamWaitEvent(main_stream, ev_img_ready, 0));   // later readers live on the main stream
  img_copy_pending = false;
}
void Engine::release_img() {
  if (!copy_stream || !db.img || db.img != stage_img[img_slot].p) return;
  VD_CUDA_CHECK(cudaEventRecord(ev_img_free[img_slot], cx.stream));
  img_free_recorded[img_slot] = true;
}

// ------------------------------------------------------------------------------------------------
// nn.SeqLSTM [upstream rnn], SURVEY.md Appendix C.  Forward: one batched x-projection (or per step in
// the non-saving mode) + per step {recurrent GEMM, pointwise}.
// ------------------------------------------------------------------------------------------------
// Wavefront over two stacked layers: layer-2 step t only needs layer-1 step t, so the two recurrences run one step
// apart on two streams instead of back to back (the per-step kernels of these 320-row LSTMs are latency-bound), with
// the contraction between the layers on a third stream.  Below this many rows the per-step contractions leave the
// tensor-core path (M < 64) and the wavefront only adds launches and event traffic.
constexpr int64_t kWavefrontMinRows = 64;

LstmRoute Engine::route_lstm(int64_t R, int H, bool gathered, bool has_h0, const float* WhT, int64_t ldw, const float* Wh) const {
  LstmRoute rt;
  // VD_MATH_F16: a many-row LSTM over embedding-gathered tokens (the option LSTM) keeps h, the activated gates, da and
  // the projection table in fp16 and runs f16 contractions (lstm16.cu); c, the accumulators and h_T stay fp32
  if (math_mode == VD_MATH_F16 && gathered && !has_h0 && lstm16_shape_ok(R, H)) {
    rt.fwd = rt.bwd = LstmPath::Opt16;
  } else {
    rt.fwd = tcmode() && lstm_step_fwd_tc_ok(H, WhT, ldw) ? LstmPath::Tc : LstmPath::Simt;
    rt.bwd = tcmode() && lstm_step_bwd_tc_ok(H, Wh) ? LstmPath::Tc : LstmPath::Simt;
  }
  rt.table_grad = gathered && tcmode();
  return rt;
}

void Engine::route_lstm_pair(LstmRun& l1, LstmRun& l2) const {
  // VD_MATH_F16: both layers and all time steps in ONE persistent launch (enc_lstm.cu) — weight slices stationary in
  // shared memory, steps chained through global flags — instead of 3 launches per time step on three streams.  The
  // kernel takes a dense layer-1 input, no initial state, and one row count, length and mask for both layers.
  if (math_mode == VD_MATH_F16 && !l1.h0 && !l1.c0 && !l2.h0 && !l2.c0 && !l1.gather && l1.x && l1.H == l2.H &&
      l2.D == l1.H && l1.R == l2.R && l1.T == l2.T && l1.mask == l2.mask && enc_pair_shape_ok(l1.R, l1.H, cx.sm_count)) {
    l1.route = l2.route = LstmRoute();
    l1.route.fwd = l1.route.bwd = l2.route.fwd = l2.route.bwd = LstmPath::Pair16;
    return;
  }
  l1.route = route_lstm(l1);
  l2.route = route_lstm(l2);
  // in the wavefront layer 2 projects its input per step, which the tensor-core step path takes (a batched projection
  // would read h1 before it exists)
  l1.route.wave_fwd = l2.route.wave_fwd = l2.route.fwd == LstmPath::Tc && l2.R >= kWavefrontMinRows;
  l1.route.wave_bwd = l2.route.wave_bwd = l1.route.bwd == LstmPath::Tc && l2.route.bwd == LstmPath::Tc && l2.R >= kWavefrontMinRows;
}

void Engine::lstm_simt_fwd_step(const LstmFwdStep& s) {
  const int G = 4 * s.H;
  if (s.h_prev) gemm_tn((int)s.R, G, s.H, s.h_prev, s.H, nullptr, s.WhT, s.ldw, s.gates, G, 1.f, nullptr, 0);
  lstm_pointwise_fwd(cx, s.gates, s.bias, s.c_prev, s.mask, s.c_out, s.h_out, s.R, s.H);
}

int Engine::lstm_tc_fwd_step(const LstmFwdStep& s) {
  if (!s.h_prev) {      // no recurrent term: a plain streaming kernel (the x-projection already has the bias)
    lstm_first_step_fwd(cx, s.gates, s.ptable, s.tok, nullptr, s.c_prev, s.mask, s.c_out, s.h_out, s.R, s.H);
    return 0;
  }
  int tile = 0;
  const bool ok = lstm_step_fwd_tc(cx, s.R, s.H, s.h_prev, s.WhT, s.ldw, nullptr, s.gates, s.ptable == nullptr, s.ptable, s.tok,
                                   s.c_prev, s.c_out, s.h_out, s.mask, &tile);
  VD_REQUIRE(ok, VD_E_STATE, "lstm_step_fwd_tc refused a shape the engine routed to it");
  return tile;
}

void Engine::lstm_simt_bwd_step(const LstmBwdStep& s) {
  const int G = 4 * s.H;
  if (s.da_next) gemm_tn((int)s.R, s.H, G, s.da_next, G, nullptr, s.Wh, G, s.dh_rec, s.H, 0.f, nullptr, 0);
  lstm_pointwise_bwd(cx, s.gates, s.c_prev, s.c_cur, s.da_next ? s.dh_rec : s.dh_last, s.dh_ext, nullptr, s.dc_carry, s.mask, s.da,
                     s.R, s.H);
}

int Engine::lstm_tc_bwd_step(const LstmBwdStep& s) {
  if (!s.da_next) { lstm_simt_bwd_step(s); return 0; }    // last step: no recurrent gradient yet, the pointwise kernel alone
  // one fused kernel: dh_rec = da_{t+1} Wh^T on wgmma, backward pointwise in the epilogue
  int tile = 0;
  const bool ok = lstm_step_bwd_tc(cx, s.R, s.H, s.da_next, s.Wh, s.gates, s.c_prev, s.c_cur, s.dh_ext, s.dc_carry, s.mask,
                                   s.da, &tile);
  VD_REQUIRE(ok, VD_E_STATE, "lstm_step_bwd_tc refused a shape the engine routed to it");
  return tile;
}

// gates of steps [t0, t0 + nt) <- x W_x^T; the Tc and Pair16 step kernels take the bias from here
void Engine::lstm_xproj(const LstmRun& r, int t0, int nt, float* gates) {
  const int64_t off = (int64_t)t0 * r.R;
  gemm_tn((int)(nt * r.R), 4 * r.H, r.D, r.x ? r.x + off * r.D : Wp(0), r.x ? r.D : cfg.E, r.gather ? r.gather + off : nullptr,
          Wtp(r.wseg), r.D + r.H, gates, 4 * r.H, 0.f, r.route.fwd == LstmPath::Simt ? nullptr : Wp(r.wseg + 1), 0);
}

void Engine::lstm_forward_begin(LstmRun& r, bool save, bool xproj_by_caller) {
  const Seg& ws = lay.segs[r.wseg];
  VD_REQUIRE(ws.rows == r.D + r.H && ws.cols == 4 * r.H, VD_E_STATE, "lstm weight shape");
  VD_REQUIRE(!r.gather || r.D == cfg.E, VD_E_STATE, "gathered LSTM input must be the word embedding");
  const int H = r.H, D = r.D, G = 4 * r.H;
  const int64_t R = r.R;
  const float* WtS = Wtp(r.wseg);          // [4H, D+H]
  r.saved = save;
  r.ptable = nullptr;
  if (r.route.fwd == LstmPath::Opt16) {
    float* pt = arena.get<float>((int64_t)(cfg.V + 1) * G);
    gemm_tn(cfg.V + 1, G, D, Wp(0), cfg.E, nullptr, WtS, D + H, pt, G, 0.f, nullptr, 0);     // bias stays fp32, added per step
    r.P16 = arena.get<__half>((int64_t)(cfg.V + 1) * G);
    cvt_f32_to_f16(cx, r.P16, G, pt, G, cfg.V + 1, G);
    r.Wh16 = arena.get<__half>((int64_t)G * H);
    cvt_f32_to_f16(cx, r.Wh16, H, WtS + D, D + H, G, H);                                    // [4H, H]: B operand of the forward step
    r.Whb16 = nullptr;
    if (save) {
      r.Whb16 = arena.get<__half>((int64_t)H * G);
      cvt_f32_to_f16(cx, r.Whb16, G, Wp(r.wseg) + (int64_t)D * G, G, H, G);                 // [H, 4H]: B operand of the backward step
    }
    const int64_t slots = save ? r.T : 2;
    r.h16 = arena.get<__half>(slots * R * H);
    r.c = arena.get<float>(slots * R * H);
    r.gates16 = save ? arena.get<__half>((int64_t)r.T * R * G) : nullptr;
    r.h32_last = arena.get<float>(R * H);
    r.h = nullptr; r.gates = nullptr;
    return;
  }
  // Tensor-core path: the x-projection of an embedding-gathered input becomes a (V+1, 4H) projection table
  // computed once per forward (E Wx^T: the 300-wide half of every step's contraction collapses into a
  // gather in the step epilogue); a dense input keeps the batched x-projection.  Each step is then ONE fused
  // kernel: recurrent wgmma GEMM + SeqLSTM pointwise epilogue.  The bias is folded into the x-projection (table or
  // GEMM epilogue), so the per-step kernel reads one array less.
  if (r.route.fwd == LstmPath::Tc && r.gather) {
    float* pt = arena.get<float>((int64_t)(cfg.V + 1) * G);
    gemm_tn(cfg.V + 1, G, D, Wp(0), cfg.E, nullptr, WtS, D + H, pt, G, 0.f, Wp(r.wseg + 1), 0);
    r.ptable = pt;
  }
  const int64_t slots = save ? r.T : 2;
  r.h = arena.get<float>(slots * R * H);
  r.c = arena.get<float>(slots * R * H);
  r.gates = arena.get<float>((save ? r.T : 1) * R * G);
  if (save && !r.ptable && !xproj_by_caller) lstm_xproj(r, 0, r.T, r.gates);
}

void Engine::lstm_forward_step(LstmRun& r, int t, bool xproj_by_caller) {
  const int H = r.H, G = 4 * r.H;
  const int64_t R = r.R, RH = R * H;
  const int64_t slot = r.saved ? t : (t & 1), pslot = r.saved ? t - 1 : ((t - 1) & 1);
  const float* bias = Wp(r.wseg + 1);
  const float* cp = t > 0 ? r.c + pslot * RH : r.c0;
  const int32_t* mk = r.mask ? r.mask + (int64_t)t * R : nullptr;
  if (r.route.fwd == LstmPath::Opt16) {
    __half* g16 = r.saved ? r.gates16 + (int64_t)t * R * G : nullptr;
    const int32_t* tok = r.gather + (int64_t)t * R;
    float* h32 = t == r.T - 1 ? r.h32_last : nullptr;
    if (t == 0) {       // no recurrent term: a streaming kernel, accounted outside the roofline class
      LaunchCtx::Scope sc(&cx, "lstm_step_first", 0.0, R * (2.0 * G + 2.0 * G + 6.0 * H));
      lstm16_first_step(cx, R, H, r.P16, tok, bias, cp, mk, g16, r.c + slot * RH, r.h16 + slot * RH, h32);
    } else {
      // algorithmic HBM bytes: fp16 gates out, fp32 c in + out, fp16 h in + out (the fp16 table gather is L2-resident: not counted)
      LaunchCtx::Scope sc(&cx, "lstm_step", 2.0 * R * G * H, R * (2.0 * G + 4.0 * H + 4.0 * H + 2.0 * H + 2.0 * H));
      lstm16_step_fwd(cx, R, H, r.h16 + pslot * RH, r.Wh16, r.P16, tok, bias, cp, mk, g16, r.c + slot * RH, r.h16 + slot * RH, h32);
    }
    return;
  }
  LstmFwdStep s;
  s.R = R; s.H = H; s.WhT = Wtp(r.wseg) + r.D; s.ldw = r.D + H; s.bias = bias; s.c_prev = cp; s.mask = mk;
  s.h_prev = t > 0 ? r.h + pslot * RH : r.h0;
  s.gates = r.saved ? r.gates + (int64_t)t * R * G : r.ptable ? nullptr : r.gates;    // a table-fed step that is not saved keeps no gates
  if (r.ptable) { s.ptable = r.ptable; s.tok = r.gather + (int64_t)t * R; }
  s.c_out = r.c + slot * RH; s.h_out = r.h + slot * RH;
  const bool tc = r.route.fwd == LstmPath::Tc;
  const bool x_per_step = !r.ptable && (!r.saved || xproj_by_caller);
  // the big (option-LSTM) launches run alone on the GPU: they are the roofline kernel class; the 320-row encoder
  // steps overlap on 4 streams and are accounted separately
  // EXECUTED work only: a gathered x-projection is a table lookup, and a first step without initial state has no
  // recurrent contraction at all (it is a streaming kernel, kept out of the roofline class)
  const bool first_no_rec = tc && !s.h_prev;
  LaunchCtx::Scope sc(&cx, first_no_rec ? "lstm_step_first" : (R >= 4096 ? "lstm_step" : "lstm_step_small"),
                      first_no_rec ? 0.0 : 2.0 * R * G * (H + (x_per_step ? r.D : 0)), 4.0 * R * (G + 4.0 * H));
  if (x_per_step && !r.saved) lstm_xproj(r, t, 1, s.gates);
  if (tc) lstm_tc_fwd_step(s); else lstm_simt_fwd_step(s);
}

void Engine::lstm_forward(LstmRun& r, bool save) {
  r.route = route_lstm(r);
  lstm_forward_begin(r, save);
  for (int t = 0; t < r.T; ++t) lstm_forward_step(r, t);
}

cudaEvent_t Engine::pool_event(size_t i) {
  while (ev_pool.size() <= i) {
    cudaEvent_t e;
    VD_CUDA_CHECK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    ev_pool.push_back(e);
  }
  return ev_pool[i];
}

void Engine::lstm_pair_forward(LstmRun& l1, LstmRun& l2, const PairStreams& s) {
  cx.stream = s.a;
  if (l1.route.fwd == LstmPath::Pair16) {
    const int H = l1.H, G = 4 * H, T = l1.T;
    const int64_t R = l1.R;
    lstm_forward_begin(l1, true);               // h / c / gates of layer 1; gates1 <- x-projection + bias (batched GEMM)
    l2.x = l1.h;
    lstm_forward_begin(l2, true, true);         // the kernel's projection CTAs compute layer 2's x-projection per step
    l1.h16 = arena.get<__half>((int64_t)T * R * H);
    l2.h16 = arena.get<__half>((int64_t)T * R * H);
    l2.x16 = l1.h16;
    __half* W1h = arena.get<__half>((int64_t)G * H);
    __half* W2c = arena.get<__half>((int64_t)G * 2 * H);
    cvt_f32_to_f16(cx, W1h, H, Wtp(l1.wseg) + l1.D, l1.D + H, G, H);                   // [4H, H]   recurrent block of layer 1
    cvt_f32_to_f16(cx, W2c, 2 * H, Wtp(l2.wseg), 2 * H, G, 2 * H);                     // [4H, 2H]  [Wx2 | Wh2] of layer 2
    int* flags = arena.get<int>(3 * (int64_t)cdiv(R, 128) * T);
    LaunchCtx::Scope sc2(&cx, "enc_pair_fwd", 2.0 * T * R * G * 3.0 * H, 4.0 * T * R * (2.0 * G + 2.0 * G + 6.0 * H));
    enc_pair_forward(cx, T, R, H, W1h, W2c, Wp(l2.wseg + 1), l1.mask, l1.gates, l1.c, l1.h, l1.h16, l2.gates, l2.c, l2.h, l2.h16, flags);
    return;
  }
  if (!l1.route.wave_fwd) {
    lstm_forward_begin(l1, true);
    for (int t = 0; t < l1.T; ++t) lstm_forward_step(l1, t);
    l2.x = l1.h;
    lstm_forward_begin(l2, true);
    for (int t = 0; t < l2.T; ++t) lstm_forward_step(l2, t);
    return;
  }
  lstm_forward_begin(l1, true);
  l2.x = l1.h;
  cudaEvent_t e0 = pool_event(0);
  VD_CUDA_CHECK(cudaEventRecord(e0, s.a));
  VD_CUDA_CHECK(cudaStreamWaitEvent(s.b, e0, 0));
  cx.stream = s.b;
  lstm_forward_begin(l2, true, true);
  for (int t = 0; t < l1.T; ++t) {
    cx.stream = s.a;
    lstm_forward_step(l1, t);
    cudaEvent_t e = pool_event(1 + t);
    VD_CUDA_CHECK(cudaEventRecord(e, s.a));
    // layer 2's x-projection of step t needs h1_t only: on its own stream it runs beside layer 2's step t-1, so
    // each of the three chains advances by ONE kernel per time step
    VD_CUDA_CHECK(cudaStreamWaitEvent(s.c, e, 0));
    if (t == 0) VD_CUDA_CHECK(cudaStreamWaitEvent(s.c, e0, 0));
    cx.stream = s.c;
    lstm_xproj(l2, t, 1, l2.gates + (int64_t)t * l2.R * 4 * l2.H);
    cudaEvent_t ex = pool_event(1 + l1.T + t);
    VD_CUDA_CHECK(cudaEventRecord(ex, s.c));
    VD_CUDA_CHECK(cudaStreamWaitEvent(s.b, ex, 0));
    cx.stream = s.b;
    lstm_forward_step(l2, t, true);
  }
  VD_CUDA_CHECK(cudaEventRecord(e0, s.b));
  VD_CUDA_CHECK(cudaStreamWaitEvent(s.a, e0, 0));
  cx.stream = s.a;
}

void Engine::lstm_backward_begin(LstmRun& r, const float* dh_all, const float* dh_last, const float* dc_last) {
  VD_REQUIRE(r.saved, VD_E_STATE, "lstm_backward needs a forward run in training mode");
  const int H = r.H, G = 4 * r.H;
  const int64_t R = r.R, TR = (int64_t)r.T * R;
  r.dc_carry = arena.get<float>(R * H);
  r.bw_dh_all = dh_all; r.bw_dh_last = dh_last;
  if (r.route.bwd == LstmPath::Opt16) {
    VD_REQUIRE(dh_last && !dh_all && !dc_last, VD_E_STATE, "fp16 BPTT takes its gradient from the last step only");
    r.da16 = arena.get<__half>(TR * G);
    r.scale2 = arena.get<float>(4);
    pick_grad_scale(cx, dh_last, R * H, reinterpret_cast<uint32_t*>(r.scale2 + 2), r.scale2);
    return;
  }
  r.da = arena.get<float>(TR * G);
  r.dh_rec = arena.get<float>(R * H);
  if (dc_last)
    VD_CUDA_CHECK(cudaMemcpyAsync(r.dc_carry, dc_last, (size_t)R * H * sizeof(float), cudaMemcpyDeviceToDevice, cx.stream));
  else
    VD_CUDA_CHECK(cudaMemsetAsync(r.dc_carry, 0, (size_t)R * H * sizeof(float), cx.stream));
}

void Engine::lstm_backward_step(LstmRun& r, int t) {
  const int H = r.H, G = 4 * r.H;
  const int64_t R = r.R, RH = R * H, RG = R * G;
  const bool last = t == r.T - 1;
  const float* cp = t > 0 ? r.c + (t - 1) * RH : r.c0;
  const int32_t* mk = r.mask ? r.mask + (int64_t)t * R : nullptr;
  if (r.route.bwd == LstmPath::Opt16) {
    const __half* g16 = r.gates16 + t * RG;
    __half* da16_t = r.da16 + t * RG;
    // steps T - 2 .. 0 run in lstm_backward, all in one lstm16_bptt call
    VD_REQUIRE(last, VD_E_STATE, "fp16 BPTT: lstm_backward runs the steps before the last one");
    LaunchCtx::Scope sc(&cx, "lstm_step_bwd_last", 0.0, R * (2.0 * G + 2.0 * G + 16.0 * H));
    lstm16_bwd_last(cx, R, H, g16, cp, r.c + t * RH, r.bw_dh_last, r.scale2, mk, r.dc_carry, da16_t);
    return;
  }
  LstmBwdStep s;
  s.R = R; s.H = H; s.Wh = Wp(r.wseg) + (int64_t)r.D * G; s.dc_carry = r.dc_carry; s.dh_rec = r.dh_rec; s.mask = mk;
  s.da_next = last ? nullptr : r.da + (t + 1) * RG; s.dh_last = last ? r.bw_dh_last : nullptr;
  s.dh_ext = r.bw_dh_all ? r.bw_dh_all + t * RH : nullptr;
  s.gates = r.gates + t * RG; s.c_prev = cp; s.c_cur = r.c + t * RH; s.da = r.da + t * RG;
  const bool tc = r.route.bwd == LstmPath::Tc;
  LaunchCtx::Scope sc(&cx, (last && tc) ? "lstm_step_bwd_last" : (R >= 4096 ? "lstm_step_bwd" : "lstm_step_bwd_small"),
                      last ? 0.0 : 2.0 * R * G * H, 4.0 * R * (2.0 * G + 5.0 * H));
  if (tc) lstm_tc_bwd_step(s); else lstm_simt_bwd_step(s);
}

void Engine::lstm_backward_end(LstmRun& r, float* dx_out, float* dh0_out, float* dc0_out) {
  const int H = r.H, D = r.D, G = 4 * r.H;
  const int64_t R = r.R, TR = (int64_t)r.T * R;
  const float* Ws = Wp(r.wseg);
  float* dWs = dWp(r.wseg);
  const bool opt16 = r.route.bwd == LstmPath::Opt16;
  if (opt16) VD_REQUIRE(!dh0_out && !dc0_out && !dx_out && !r.h0, VD_E_STATE, "fp16 BPTT: no initial-state / input gradients");
  if (dh0_out) gemm_tn((int)R, H, G, r.da, G, nullptr, Ws + (int64_t)D * G, G, dh0_out, H, 0.f, nullptr, 0);
  if (dc0_out) VD_CUDA_CHECK(cudaMemcpyAsync(dc0_out, r.dc_carry, (size_t)R * H * sizeof(float), cudaMemcpyDeviceToDevice, cx.stream));
  // accGradParameters.  The fp16 routes' kernels left fp16 copies of h and da — the operands of the recurrence itself —
  // so the weight gradients contract those on the fp16 tensor-core path (fp32 accumulation) instead of the TF32 one.  The
  // persistent pair's shape check (enc_pair_shape_ok) already guarantees H % 64 == 0.
  const bool wgrad16 = opt16 || (r.route.bwd == LstmPath::Pair16 && TR - R >= 256);
  if (r.T > 1) {
    if (wgrad16) {
      LaunchCtx::Scope sc(&cx, "gemm_wgrad", 2.0 * H * G * (double)(TR - R), 2.0 * (double)(TR - R) * (H + G));
      // stream-K: a CTA whose SM is still busy with another stream's kernel starts late and claims less work, so the
      // weight gradient is sized to the whole GPU even under the option stream's overlap budget
      const int budget = cx.sm_budget;
      cx.sm_budget = 0;
      gemm_atb16(cx, H, G, TR - R, r.h16, H, r.da16 + R * G, G, dWs + (int64_t)D * G, G, r.scale2 + 1);
      cx.sm_budget = budget;
    } else gemm_atb(H, G, TR - R, r.h, H, nullptr, r.da + R * G, G, dWs + (int64_t)D * G, G);
  }
  if (r.h0) gemm_atb(H, G, R, r.h0, H, nullptr, r.da, G, dWs + (int64_t)D * G, G);
  if (r.route.table_grad) {
    // Embedding-gathered input: every x_t is a row of the (V+1, E) table, so the three x-side gradients collapse
    // onto the table.  dP[v] = sum of da over the rows whose token is v (counting sort + balanced segmented sum,
    // HBM-bound) and then  dWx += E^T dP,  db += colsum(dP),  dEmb += dP Wx^T  are (V+1)-row contractions instead
    // of T*R-row ones (2 x 786 GFLOP -> 2 x 12 GFLOP for the 100 x 20-token option LSTM).
    VD_REQUIRE(dx_out == nullptr, VD_E_STATE, "projected-space embedding gradient: caller must not ask for dx");
    const int V1 = cfg.V + 1;
    float* dP = arena.get<float>((int64_t)V1 * G);
    VD_CUDA_CHECK(cudaMemsetAsync(dP, 0, (size_t)V1 * G * sizeof(float), cx.stream));
    int32_t* scratch = arena.get<int32_t>(3 * (int64_t)V1);
    int32_t* perm = arena.get<int32_t>(TR);
    int32_t* stok = arena.get<int32_t>(TR);
    {
      LaunchCtx::Scope sc(&cx, "embed_grad_segsum", 0.0, (opt16 ? 2.0 : 4.0) * TR * G);
      group_rows_by_token(cx, r.gather, TR, V1, scratch, perm, stok);
      if (opt16) segsum_rows16(cx, r.da16, G, perm, stok, TR, dP, G, r.scale2 + 1);
      else segsum_rows(cx, r.da, G, perm, stok, TR, dP, G);
    }
    gemm_atb(D, G, V1, Wp(0), cfg.E, nullptr, dP, G, dWs, G);
    colsum_add(cx, dWp(r.wseg + 1), dP, V1, G, G);
    if (r.demb_out) gemm_tn(V1, D, G, dP, G, nullptr, Ws, G, r.demb_out, cfg.E, 0.f, nullptr, 0);   // folded in by the caller
    else gemm_tn(V1, D, G, dP, G, nullptr, Ws, G, dWp(0), cfg.E, 1.f, nullptr, 0);
    return;
  }
  if (wgrad16 && r.x16) {            // layer 2 of the pair: x = h1, D = H
    LaunchCtx::Scope sc(&cx, "gemm_wgrad", 2.0 * D * G * (double)TR, 2.0 * (double)TR * (D + G));
    gemm_atb16(cx, D, G, TR, r.x16, D, r.da16, G, dWs, G, r.scale2 + 1);
  } else gemm_atb(D, G, TR, r.x ? r.x : Wp(0), r.x ? D : cfg.E, r.gather, r.da, G, dWs, G);
  colsum_add(cx, dWp(r.wseg + 1), r.da, TR, G, G);
  if (dx_out) gemm_tn((int)TR, D, G, r.da, G, nullptr, Ws, G, dx_out, D, 0.f, nullptr, 0);
}

void Engine::lstm_backward(LstmRun& r, const float* dh_all, const float* dh_last, const float* dc_last, float* dx_out,
                           float* dh0_out, float* dc0_out) {
  lstm_backward_begin(r, dh_all, dh_last, dc_last);
  if (r.route.bwd == LstmPath::Opt16) {
    lstm_backward_step(r, r.T - 1);
    if (r.T > 1) {
      // every 128-row block runs steps T - 2 .. 0 in one launch, with its dc carry on chip: per row and step the HBM bytes
      // are the fp16 gates in and da out and the fp32 c_{t-1} and c_t in (12 KB at H = 512), plus the carry in and out once
      // (the block's da_{t+1} is read back from L2, where the cluster wrote it the step before)
      const int H = r.H, G = 4 * r.H, S = r.T - 1;
      const double R = (double)r.R;
      LaunchCtx::Scope sc(&cx, "lstm_step_bwd", S * 2.0 * R * G * H, S * R * (2.0 * G + 2.0 * G + 8.0 * H) + R * 8.0 * H);
      lstm16_bptt(cx, r.R, H, r.T, r.da16, r.Whb16, r.gates16, r.c, r.c0, r.mask, r.dc_carry);
    }
  } else {
    for (int t = r.T - 1; t >= 0; --t) lstm_backward_step(r, t);
  }
  lstm_backward_end(r, dx_out, dh0_out, dc0_out);
}

// BPTT wavefront of two stacked layers: layer-1 step t needs d(h1_t) = da2_t Wx2^T, produced per step on stream c,
// so the two recurrences again run one step apart (layer 2 on b, layer 1 on a).
void Engine::lstm_pair_backward(LstmRun& l1, LstmRun& l2, const float* dh_last2, const float* dc_last2, const float* dh_last1,
                                const float* dc_last1, float* dx1_out, const PairStreams& s) {
  const int H = l2.H, G = 4 * l2.H;
  const int64_t R = l2.R;
  cx.stream = s.a;
  if (l1.route.bwd == LstmPath::Pair16) {
    // one launch for both layers and all time steps (enc_lstm.cu::k_enc_pair_bwd); the weight / input gradients follow
    // as batched contractions over all T*R rows
    const int T = l2.T;
    const int64_t TR = (int64_t)T * R;
    l1.da = arena.get<float>(TR * G); l2.da = arena.get<float>(TR * G);
    l1.da16 = arena.get<__half>(TR * G); l2.da16 = arena.get<__half>(TR * G);
    __half* Whb2 = arena.get<__half>((int64_t)H * G);
    __half* B1cat = arena.get<__half>((int64_t)H * 2 * G);
    cvt_f32_to_f16(cx, Whb2, G, Wp(l2.wseg) + (int64_t)l2.D * G, G, H, G);                 // Wh2: rows D2.. of (D2+H, 4H)
    cvt_f32_to_f16(cx, B1cat, 2 * G, Wp(l2.wseg), G, H, G);                                 // [Wx2 | ...]: rows 0..H-1 of layer 2
    cvt_f32_to_f16(cx, B1cat + G, 2 * G, Wp(l1.wseg) + (int64_t)l1.D * G, G, H, G);         // [... | Wh1]
    int* flags = arena.get<int>(enc_pair_bwd_flag_ints(T, R, H));
    float* dh1 = nullptr; float* dh2 = nullptr;
    // the gate split sums its partial products with float atomics: deterministic mode takes the unit split
    if (enc_pair_gate_split(H) && !cx.deterministic) { dh1 = arena.get<float>(TR * H); dh2 = arena.get<float>(TR * H); }
    l1.scale2 = l2.scale2 = arena.get<float>(2);       // da16 of both layers = fp16(s da); the weight gradients take 1/s
    {
      LaunchCtx::Scope sc2(&cx, "enc_pair_bwd", 2.0 * T * R * (double)H * 3.0 * G, 4.0 * T * R * (4.0 * G + 4.0 * H));
      enc_pair_backward(cx, T, R, H, B1cat, Whb2, l1.mask, l1.gates, l1.c, l2.gates, l2.c, dh_last1, dc_last1, dh_last2, dc_last2,
                        l1.da, l1.da16, l2.da, l2.da16, flags, dh1, dh2, l1.scale2);
    }
    lstm_backward_end(l2, nullptr, nullptr, nullptr);
    lstm_backward_end(l1, dx1_out, nullptr, nullptr);
    return;
  }
  float* dx2 = arena.get<float>((int64_t)l2.T * R * l2.D);      // = gradient wrt layer-1 outputs, all steps
  if (!l1.route.wave_bwd) {
    lstm_backward(l2, nullptr, dh_last2, dc_last2, dx2, nullptr, nullptr);
    lstm_backward(l1, dx2, dh_last1, dc_last1, dx1_out, nullptr, nullptr);
    return;
  }
  const float* Wx2 = Wp(l2.wseg);            // rows 0..D2 of (D2+H, 4H): [N = D2, K = 4H]
  cudaEvent_t e0 = pool_event(0);
  VD_CUDA_CHECK(cudaEventRecord(e0, s.a));
  VD_CUDA_CHECK(cudaStreamWaitEvent(s.b, e0, 0));
  cx.stream = s.b;
  lstm_backward_begin(l2, nullptr, dh_last2, dc_last2);
  cx.stream = s.a;
  lstm_backward_begin(l1, dx2, dh_last1, dc_last1);
  for (int t = l2.T - 1; t >= 0; --t) {
    cx.stream = s.b;
    lstm_backward_step(l2, t);
    // d(h1_t) = da2_t Wx2 needs layer 2's step t only: on its own stream it runs beside layer 2's step t-1
    cudaEvent_t e = pool_event(1 + t);
    VD_CUDA_CHECK(cudaEventRecord(e, s.b));
    VD_CUDA_CHECK(cudaStreamWaitEvent(s.c, e, 0));
    cx.stream = s.c;
    gemm_tn((int)R, l2.D, G, l2.da + (int64_t)t * R * G, G, nullptr, Wx2, G, dx2 + (int64_t)t * R * l2.D, l2.D, 0.f, nullptr, 0);
    cudaEvent_t ex = pool_event(1 + l2.T + t);
    VD_CUDA_CHECK(cudaEventRecord(ex, s.c));
    VD_CUDA_CHECK(cudaStreamWaitEvent(s.a, ex, 0));
    cx.stream = s.a;
    lstm_backward_step(l1, t);
  }
  cx.stream = s.b;
  lstm_backward_end(l2, nullptr, nullptr, nullptr);       // weight gradients of layer 2 (its dx was produced per step)
  VD_CUDA_CHECK(cudaEventRecord(e0, s.b));
  cx.stream = s.a;
  lstm_backward_end(l1, dx1_out, nullptr, nullptr);
  VD_CUDA_CHECK(cudaStreamWaitEvent(s.a, e0, 0));
}

// ------------------------------------------------------------------------------------------------
// encoders
// ------------------------------------------------------------------------------------------------
static LstmRun make_run(int T, int64_t R, int D, int H, int wseg, const float* x, const int32_t* gather, const int32_t* mask) {
  LstmRun r; r.T = T; r.R = R; r.D = D; r.H = H; r.wseg = wseg; r.x = x; r.gather = gather; r.mask = mask;
  return r;
}

// ---- blocks shared by several encoder graphs -----------------------------------------------------------------------
// memory network over the history facts (mn-*.lua): MM -> MaskSoftMax (causal) -> MM -> Dropout -> Linear -> Tanh, residual query, Linear -> Tanh
// Rounds [r0, r1) of B dialogs: qin / out have B*(r1-r0) rows, the facts of dialog b are rows 0..r1-1 of facts + b*fpitch
// (the full forward: [0, R) over hist2's h_T; a dialog session: [r, r+1) over its cached facts)
void Engine::mn_block_fwd(const float* qin, const float* facts, int64_t fpitch, float* out, int B, int r0, int r1,
                          const int32_t* slot, const int32_t* round) {
  const int H = cfg.H, R = cfg.R;
  const int64_t N = (int64_t)B * (r1 - r0);
  const DropCfg d05 = dropcfg(0.5f);
  probs = arena.get<float>(N * R);
  hAtt = arena.get<float>(N * H);
  mn_attention_rows_fwd(cx, qin, facts, fpitch, probs, hAtt, B, R, H, r0, r1, slot, round);
  hAtt_d = arena.get<float>(N * H);
  dropout_apply(cx, hAtt_d, hAtt, N * H, d05, SITE_HATT);
  hAttTr = arena.get<float>(N * H);
  linear_fwd(seg("mn.fact.weight"), hAtt_d, N, hAttTr, 1);
  sum1 = arena.get<float>(N * H);
  add_out(cx, sum1, hAttTr, qin, N * H);
  linear_fwd(seg("mn.query.weight"), sum1, N, out, 1);
}
// dout = gradient wrt `out` (post-tanh); dqin / dh3 receive the gradients wrt the query input and the facts
void Engine::mn_block_bwd(const float* dout, const float* out, float* dqin, float* dh3) {
  const int H = cfg.H, R = cfg.R, B = db.B;
  const int64_t N = db.N;
  const DropCfg d05 = dropcfg(0.5f);
  float* dpre = arena.get<float>(N * H);
  tanh_bwd(cx, dpre, dout, out, N * H);
  float* dsum1 = arena.get<float>(N * H);
  linear_bwd(seg("mn.query.weight"), sum1, dpre, N, dsum1, 0.f);
  tanh_bwd(cx, dpre, dsum1, hAttTr, N * H);
  float* dhAtt = arena.get<float>(N * H);
  linear_bwd(seg("mn.fact.weight"), hAtt_d, dpre, N, dhAtt, 0.f);
  dropout_apply(cx, dhAtt, dhAtt, N * H, d05, SITE_HATT);
  mn_attention_bwd(cx, mn_query_in, hist2.h_last(), probs, dhAtt, dqin, dh3, B, R, H);
  add_inplace(cx, dqin, dsum1, N * H);
}
// SAN (mn-att-ques-im-hist.lua:67-106, lf-att-ques-im-hist.lua:43-86): tanh(Linear(img)) is computed once per dialog; Dropout then
// acts on the repeated tensor; hops of {img_common + ques_common -> tanh -> dropout -> score -> softmax -> weighted sum + u}
void Engine::san_image(const float* pool5, int64_t B, float* t) {
  wait_img();
  linear_fwd(seg("san.img.weight"), pool5, B * cfg.P, t, 1);
}
// Region engines (DESIGN §26): san_cnt holds the B dialogs' counts (null: all present); the GEMMs run over all P rows, the
// attention kernels skip the pad rows and give them zero probability and zero gradients.
void Engine::san_block_fwd(const float* u0, const float* timg, int B, int nr, float* out) {
  const int H = cfg.H;
  const int64_t N = (int64_t)B * nr;
  const int P = cfg.P, Cm = cfg.Cm;
  const DropCfg d05 = dropcfg(0.5f);
  t_img = const_cast<float*>(timg);
  img_tr = arena.get<float>(N * P * H);
  san_expand_dropout(cx, img_tr, t_img, B, nr, P, H, d05, SITE_IMG_TR);
  img_common.assign(cfg.hops, nullptr); ques_common.assign(cfg.hops, nullptr);
  sc.assign(cfg.hops, nullptr); pr.assign(cfg.hops, nullptr); u_hop.assign(cfg.hops + 1, nullptr);
  u_hop[0] = const_cast<float*>(u0);
  for (int hop = 0; hop < cfg.hops; ++hop) {
    std::string pre = "san.hop" + std::to_string(hop + 1) + ".";
    int w_ic = seg((pre + "img_common.weight").c_str()), w_qc = seg((pre + "ques_common.weight").c_str()),
        w_s = seg((pre + "score.weight").c_str());
    img_common[hop] = arena.get<float>(N * P * Cm);
    linear_fwd(w_ic, img_tr, N * P, img_common[hop], 0);
    ques_common[hop] = arena.get<float>(N * Cm);
    linear_fwd(w_qc, u_hop[hop], N, ques_common[hop], 0);
    sc[hop] = arena.get<float>(N * P);
    san_score_fwd(cx, img_common[hop], ques_common[hop], Wp(w_s), Wp(w_s + 1), sc[hop], N, P, Cm, d05, SITE_HOP0 + hop, san_cnt,
                  nr);
    pr[hop] = arena.get<float>(N * P);
    u_hop[hop + 1] = arena.get<float>(N * H);
    san_softmax_att_fwd(cx, sc[hop], pr[hop], img_tr, u_hop[hop], u_hop[hop + 1], N, P, H, san_cnt, nr);
  }
  u_d = arena.get<float>(N * H);
  dropout_apply(cx, u_d, u_hop[cfg.hops], N * H, d05, SITE_U_OUT);
  linear_fwd(seg("san.out.weight"), u_d, N, out, 1);
}
void Engine::san_block_bwd(const float* dEnc, float* du) {
  const int H = cfg.H, R = cfg.R, B = db.B;
  const int64_t N = db.N;
  const int P = cfg.P, Cm = cfg.Cm;
  const DropCfg d05 = dropcfg(0.5f);
  float* dpre = arena.get<float>(N * H);
  tanh_bwd(cx, dpre, dEnc, encOut, N * H);
  linear_bwd(seg("san.out.weight"), u_d, dpre, N, du, 0.f);
  dropout_apply(cx, du, du, N * H, d05, SITE_U_OUT);
  float* dimg_tr = arena.get<float>(N * P * H);
  float* ds = arena.get<float>(N * P);
  float* dic = arena.get<float>(N * P * Cm);
  float* dqc = arena.get<float>(N * Cm);
  for (int hop = cfg.hops - 1; hop >= 0; --hop) {
    std::string pre = "san.hop" + std::to_string(hop + 1) + ".";
    int w_ic = seg((pre + "img_common.weight").c_str()), w_qc = seg((pre + "ques_common.weight").c_str()),
        w_s = seg((pre + "score.weight").c_str());
    if (hop == cfg.hops - 1) {
      san_att_bwd(cx, du, pr[hop], img_tr, ds, dimg_tr, N, P, H, san_cnt, R);
    } else {
      float* tmp = arena.get<float>(N * P * H);
      san_att_bwd(cx, du, pr[hop], img_tr, ds, tmp, N, P, H, san_cnt, R);
      add_inplace(cx, dimg_tr, tmp, N * P * H);
    }
    san_score_bwd(cx, ds, img_common[hop], ques_common[hop], Wp(w_s), dic, dqc, dWp(w_s), dWp(w_s + 1), N, P, Cm, d05,
                  SITE_HOP0 + hop, san_cnt, R);
    linear_bwd(w_ic, img_tr, dic, N * P, dimg_tr, 1.f);
    linear_bwd(w_qc, u_hop[hop], dqc, N, du, 1.f);          // du now = grad wrt u_hop[hop]
  }
  float* dt_pre = arena.get<float>((int64_t)B * P * H);
  san_collapse_bwd(cx, dimg_tr, t_img, dt_pre, B, R, P, H, d05, SITE_IMG_TR, san_cnt);
  linear_bwd(seg("san.img.weight"), db.img, dt_pre, (int64_t)B * P, nullptr, 0.f);
  release_img();                                   // last reader of this step's image staging buffer
}

// late fusion (lf-ques.lua:29-33 / lf-ques-im.lua / lf-ques-hist.lua / lf-ques-im-hist.lua:49-59): JoinTable [q | img | h] ->
// Dropout -> Linear -> Tanh.  lf-att-ques-im-hist.lua:41: Tanh(Linear([q | h])) with no dropout, then the SAN block on pool5.
// q3 / h3 / out: B*nr rows (nr rounds per dialog); fc7: B rows, repeated per round (model.lua:267-269); timg: the SAN's
// tanh(Linear(pool5)) of the B dialogs (san_image)
void Engine::lf_block_fwd(const float* q3, const float* fc7, const float* timg, const float* h3, int B, int nr, float* out) {
  const int H = cfg.H;
  const int64_t N = (int64_t)B * nr;
  const bool use_fc7 = cfg.useIm && !cfg.san;
  joinK = H + (use_fc7 ? cfg.F : 0) + (cfg.useHist ? H : 0);
  join_d = arena.get<float>(N * joinK);
  copy_cols(cx, join_d, joinK, q3, H, N, H);
  if (use_fc7) {
    float* tmp = arena.get<float>(N * cfg.F);
    wait_img();
    repeat_rows(cx, tmp, fc7, B, nr, cfg.F);
    copy_cols(cx, join_d + H, joinK, tmp, cfg.F, N, cfg.F);
  }
  if (cfg.useHist) copy_cols(cx, join_d + H + (use_fc7 ? cfg.F : 0), joinK, h3, H, N, H);
  if (!cfg.san) {
    dropout_apply(cx, join_d, join_d, N * joinK, dropcfg(cfg.dropout), SITE_FUSION);
    linear_fwd(seg("fusion.weight"), join_d, N, out, 1);
  } else {
    qh2 = arena.get<float>(N * H);
    linear_fwd(seg("fusion.weight"), join_d, N, qh2, 1);
    san_block_fwd(qh2, timg, B, nr, out);
  }
}

// hre / hrea: the dialog LSTM's input rows j (B*(r1-r0), 2H) of rounds [r0, r1).  hrea-ques-im-hist.lua:89-129: attention
// of the round's sq over the scores sh (B, R) and facts (dialog b at facts + b*fpitch) of rounds <= it, then [att | q];
// hre-ques-*.lua: [q | h]
void Engine::hre_join_fwd(const float* q3, const float* facts, const float* sq_, const float* sh_, int64_t fpitch, int B, int r0,
                          int r1, float* j, const int32_t* slot, const int32_t* round) {
  const int H = cfg.H, R = cfg.R;
  const int64_t N = (int64_t)B * (r1 - r0);
  if (cfg.hre_att) {
    probs = arena.get<float>(N * R);
    att = arena.get<float>(N * H);
    hrea_attention_rows_fwd(cx, sq_, sh_, facts, fpitch, probs, att, B, R, H, r0, r1, slot, round);
    copy_cols(cx, j, 2 * H, att, H, N, H);
    copy_cols(cx, j + H, 2 * H, q3, H, N, H);
  } else {
    copy_cols(cx, j, 2 * H, q3, H, N, H);              // nr == 1 or the full forward: the facts are h3's own rows
    copy_cols(cx, j + H, 2 * H, facts, H, N, H);
  }
}

// the dialog-level LSTM over nr rounds of B dialogs from (h0, c0) (null: the first round), rows j (B*nr, 2H) in dialog-major
// order.  View(-1,10,2H), Transpose(1,2): row (r,b) <- row (b,r), a strided 2-D copy per round; out (B*nr, H) dialog-major.
// The run (`dialog`) keeps its last h and c, which a dialog session carries to the next round.
void Engine::hre_dialog_fwd(const float* j, int B, int nr, const float* h0, const float* c0, float* out) {
  const int H = cfg.H;
  const int64_t N = (int64_t)B * nr;
  jt = arena.get<float>(N * 2 * H);
  for (int rr = 0; rr < nr; ++rr)
    copy_cols(cx, jt + (int64_t)rr * B * 2 * H, 2 * H, j + (int64_t)rr * 2 * H, (int64_t)nr * 2 * H, B, 2 * H);
  dialog = make_run(nr, B, 2 * H, H, seg("dialog.lstm.weight"), jt, nullptr, nullptr);
  dialog.h0 = h0; dialog.c0 = c0;
  dialog.route = route_lstm(dialog);
  lstm_forward_begin(dialog, true);
  for (int t = 0; t < nr; ++t) lstm_forward_step(dialog, t);
  for (int rr = 0; rr < nr; ++rr)
    copy_cols(cx, out + (int64_t)rr * H, (int64_t)nr * H, dialog.h + (int64_t)rr * B * H, H, B, H);
}

// mn-ques-hist.lua / mn-ques-im-hist.lua / mn-att-ques-im-hist.lua:48-106 on rounds [r0, r1): q3 / out B*(r1-r0) rows, img
// the B dialogs' fc7 (mn-ques-im-hist), timg as lf_block_fwd's, facts as mn_block_fwd takes them
void Engine::mn_family_fwd(const float* q3, const float* img, const float* timg, const float* facts, int64_t fpitch, int B, int r0,
                           int r1, float* out, const int32_t* slot, const int32_t* round) {
  const int H = cfg.H, nr = r1 - r0;
  const int64_t N = (int64_t)B * nr;
  mn_query_in = q3;
  if (cfg.mn_qi) {                                    // mn-ques-im-hist.lua: qi_proj = Tanh(Linear([q | fc7]))
    qi_join = arena.get<float>(N * (H + cfg.F));
    copy_cols(cx, qi_join, H + cfg.F, q3, H, N, H);
    float* tmp = arena.get<float>(N * cfg.F);
    wait_img();
    repeat_rows(cx, tmp, img, B, nr, cfg.F);
    copy_cols(cx, qi_join + H, H + cfg.F, tmp, cfg.F, N, cfg.F);
    qi_proj = arena.get<float>(N * H);
    linear_fwd(seg("mn.qi.weight"), qi_join, N, qi_proj, 1);
    mn_query_in = qi_proj;
  }
  if (cfg.san) {
    qh2 = arena.get<float>(N * H);
    mn_block_fwd(mn_query_in, facts, fpitch, qh2, B, r0, r1, slot, round);
    san_block_fwd(qh2, timg, B, nr, out);
  } else {
    mn_block_fwd(mn_query_in, facts, fpitch, out, B, r0, r1, slot, round);
  }
}

void Engine::quiesce() {
  VD_CUDA_CHECK(cudaSetDevice(cfg.gpuid));
  if (side_active) { cudaStreamSynchronize(side_stream); side_active = false; }   // only after an aborted call
  cx.stream = main_stream;
  if (opt_fwd_pending || opt_bwd_pending) {       // a previous call sequence was abandoned half-way: drain before reuse
    VD_CUDA_CHECK(cudaStreamSynchronize(opt_stream));
    opt_fwd_pending = opt_bwd_pending = false;
  }
  opt_demb = nullptr; opt_dx = nullptr;          // an abandoned step's option gradients are not folded in later
  arena.reset();
  have_fwd = false;
}

// The question and history LSTM pairs over `rows` rows of time-major ids ids_q (Tq, rows) / ids_h (Th, rows).  img_rows
// (rows, IE): the image embedding MaskTime joins to the question LSTM's input (img_in_q), else null.
void Engine::encoder_lstms(int64_t rows, int Tq, int Th, const float* img_rows, bool ques_pair) {
  const int E = cfg.E, H = cfg.H;
  const int64_t N = rows;
  const DropCfg d05 = dropcfg(0.5f), dnone = dropcfg(0.f);
  const bool embdrop = cfg.embdrop;                        // mn-*.lua / lf-att-*.lua: Dropout(0.5) on both embeddings
  // history branch
  if (cfg.useHist) {
    fork_side();
    xh = arena.get<float>(N * Th * E);
    embed_rows(cx, xh, Wp(0), ids_h, N * Th, E, embdrop ? d05 : dnone, SITE_HEMBED);
    hist1 = make_run(Th, N, E, H, seg("hist.lstm1.weight"), xh, nullptr, ids_h);
    hist2 = make_run(Th, N, H, H, seg("hist.lstm2.weight"), nullptr, nullptr, ids_h);
    route_lstm_pair(hist1, hist2);
    // The 2nd layer consumes every step of the 1st, so encoder LSTMs always keep all steps (T*N*H is small).
    // The history and question LSTM chains are independent until the fusion/attention stage: the history chain runs
    // on the side stream (its tiny per-step kernels are latency-bound; overlapping the two chains hides half of it).
    if (serial_pairs()) { join_side(); lstm_pair_forward(hist1, hist2, main_chain); }
    else { lstm_pair_forward(hist1, hist2, side_chain); back_to_main(); }
  }
  if (!ques_pair) { join_side(); return; }
  // question branch
  xq = arena.get<float>(N * Tq * E);
  embed_rows(cx, xq, Wp(0), ids_q, N * Tq, E, embdrop ? d05 : dnone, SITE_QEMBED);
  if (img_rows) {
    // hre(a)-ques-im-hist.lua:41-55: MaskTime, JoinTable(-1)
    qi_in = arena.get<float>(N * Tq * (E + cfg.IE));
    masktime_concat_fwd(cx, qi_in, xq, img_rows, ids_q, Tq, N, E, cfg.IE);
    ques1 = make_run(Tq, N, E + cfg.IE, H, seg("ques.lstm1.weight"), qi_in, nullptr, ids_q);
  } else {
    ques1 = make_run(Tq, N, E, H, seg("ques.lstm1.weight"), xq, nullptr, ids_q);
  }
  ques2 = make_run(Tq, N, H, H, seg("ques.lstm2.weight"), nullptr, nullptr, ids_q);
  route_lstm_pair(ques1, ques2);
  lstm_pair_forward(ques1, ques2, main_chain);
  join_side();
}

void Engine::encoder_forward(const vd_batch* b) {
  quiesce();
  stage_batch(b);
  save_acts = training != 0;
  refresh_shadows();
  if (opt_overlap && cfg.dec == DEC_DISC && db.options && db.To > 0) options_forward_async();
  conn_dh_l1 = conn_dc_l1 = conn_dc_l2 = nullptr;
  gen_h0[0] = gen_h0[1] = gen_c0[0] = gen_c0[1] = nullptr;
  const int H = cfg.H, R = cfg.R;
  const int64_t N = db.N;
  const int B = db.B;
  const DropCfg d05 = dropcfg(0.5f);
  // time-major ids: the view(-1,T):t() of model.lua:255-257,274-278
  ids_q = arena.get<int32_t>(N * db.Tq);
  transpose_ids(cx, db.ques, ids_q, N, db.Tq);
  if (cfg.useHist) {
    ids_h = arena.get<int32_t>(N * db.Th);
    transpose_ids(cx, db.hist, ids_h, N, db.Th);
  }
  const float* img_rows = nullptr;
  if (cfg.img_in_q) {
    // hre(a)-ques-im-hist.lua:41-55: [Dropout(0.5) ->] Linear(F,IE) on the 10x repeated fc7
    img_d = arena.get<float>(N * cfg.F);
    wait_img();
    repeat_rows(cx, img_d, db.img, B, R, cfg.F);
    if (cfg.img_drop) dropout_apply(cx, img_d, img_d, N * cfg.F, d05, SITE_IMG_FC7);
    img_e = arena.get<float>(N * cfg.IE);
    linear_fwd(seg("img.embed.weight"), img_d, N, img_e, 0);
    img_rows = img_e;
  }
  encoder_lstms(N, db.Tq, db.Th, img_rows);
  const float* q3 = ques2.h_last();
  const float* h3 = cfg.useHist ? hist2.h_last() : nullptr;
  encOut = arena.get<float>(N * H);

  const float* timg = nullptr;
  if (cfg.san) {
    float* t = arena.get<float>((int64_t)B * cfg.P * H);
    san_image(db.img, B, t);
    timg = t;
    san_cnt = db.img_count;
  }
  if (cfg.fam_lf) {
    lf_block_fwd(q3, db.img, timg, h3, B, R, encOut);
  } else if (cfg.fam_hre) {
    float* j = arena.get<float>(N * 2 * H);
    if (cfg.hre_att) {
      sq = arena.get<float>(N); sh = arena.get<float>(N);
      int sq_w = seg("att.q.weight"), sh_w = seg("att.h.weight");
      rowdot_fwd(cx, sq, q3, Wp(sq_w), Wp(sq_w + 1), N, H);
      rowdot_fwd(cx, sh, h3, Wp(sh_w), Wp(sh_w + 1), N, H);
    }
    hre_join_fwd(q3, h3, sq, sh, (int64_t)R * H, B, 0, R, j);
    hre_dialog_fwd(j, B, R, nullptr, nullptr, encOut);
  } else {
    mn_family_fwd(q3, db.img, timg, h3, (int64_t)R * H, B, 0, R, encOut);
  }
  wait_img();                // (an encoder that never reads the image still has to retire the copy before the buffer is reused)
  release_img();             // forward-only callers never reach the backward's release; a later one simply overrides this
  have_fwd = true;
}

void Engine::encoder_backward(const float* dEnc) {
  VD_REQUIRE(have_fwd && save_acts, VD_E_STATE, "encoder_backward: no training-mode forward to back-propagate");
  VD_REQUIRE(dEnc != nullptr, VD_E_BADARG, "gradEncOut is null");
  const int E = cfg.E, H = cfg.H, R = cfg.R;
  const int64_t N = db.N;
  const int B = db.B;
  const DropCfg d05 = dropcfg(0.5f), dp = dropcfg(cfg.dropout), dnone = dropcfg(0.f);
  float* dq3 = arena.get<float>(N * H);
  float* dh3 = cfg.useHist ? arena.get<float>(N * H) : nullptr;
  float* dpre = arena.get<float>(N * H);
  // gradient sync, bucket 0: the decoder's own weights are final once decoder_backward is enqueued (gen: dec.lstm1/2 +
  // dec.out, 20 MB at V = 10k; disc without the option stream: opt.lstm) — their all-reduce overlaps the whole encoder BPTT
  if (cfg.dec == DEC_GEN) reduce_segments(seg("dec.lstm1.weight"), (int)lay.segs.size() - 1, main_stream);
  else if (!opt_bwd_pending) reduce_segments(seg("opt.lstm.weight"), (int)lay.segs.size() - 1, main_stream);

  if (cfg.fam_lf) {
    const bool fc7 = cfg.useIm && !cfg.san;
    float* dj = arena.get<float>(N * joinK);
    if (!cfg.san) {
      tanh_bwd(cx, dpre, dEnc, encOut, N * H);
      linear_bwd(seg("fusion.weight"), join_d, dpre, N, dj, 0.f);
      dropout_apply(cx, dj, dj, N * joinK, dp, SITE_FUSION);
    } else {
      float* dqh = arena.get<float>(N * H);
      san_block_bwd(dEnc, dqh);
      tanh_bwd(cx, dpre, dqh, qh2, N * H);
      linear_bwd(seg("fusion.weight"), join_d, dpre, N, dj, 0.f);
    }
    copy_cols(cx, dq3, H, dj, joinK, N, H);
    if (cfg.useHist) copy_cols(cx, dh3, H, dj + H + (fc7 ? cfg.F : 0), joinK, N, H);
  } else if (cfg.fam_hre) {
    const float* q3 = ques2.h_last();
    const float* h3 = hist2.h_last();
    // un-permute the gradient (n = b*R + r) -> (r,b), BPTT over rounds
    float* dd = arena.get<float>(N * H);
    for (int rr = 0; rr < R; ++rr)
      copy_cols(cx, dd + (int64_t)rr * B * H, H, dEnc + (int64_t)rr * H, (int64_t)R * H, B, H);
    float* djt = arena.get<float>(N * 2 * H);
    lstm_backward(dialog, dd, nullptr, nullptr, djt, nullptr, nullptr);
    float* dj = arena.get<float>(N * 2 * H);
    for (int rr = 0; rr < R; ++rr)
      copy_cols(cx, dj + (int64_t)rr * 2 * H, (int64_t)R * 2 * H, djt + (int64_t)rr * B * 2 * H, 2 * H, B, 2 * H);
    if (cfg.hre_att) {
      float* datt = arena.get<float>(N * H);
      copy_cols(cx, datt, H, dj, 2 * H, N, H);
      copy_cols(cx, dq3, H, dj + H, 2 * H, N, H);
      float* dsq = arena.get<float>(N); float* dsh = arena.get<float>(N);
      hrea_attention_bwd(cx, sq, sh, h3, probs, datt, dsq, dsh, dh3, B, R, H);
      int sq_w = seg("att.q.weight"), sh_w = seg("att.h.weight");
      rowdot_bwd(cx, dsq, q3, Wp(sq_w), dq3, 1, dWp(sq_w), dWp(sq_w + 1), N, H);
      rowdot_bwd(cx, dsh, h3, Wp(sh_w), dh3, 1, dWp(sh_w), dWp(sh_w + 1), N, H);
    } else {
      copy_cols(cx, dq3, H, dj, 2 * H, N, H);
      copy_cols(cx, dh3, H, dj + H, 2 * H, N, H);
    }
  } else {
    // memory-network family: [SAN ->] memory block -> [qi projection]
    float* dqin = cfg.mn_qi ? arena.get<float>(N * H) : dq3;
    if (cfg.san) {
      float* du = arena.get<float>(N * H);
      san_block_bwd(dEnc, du);
      mn_block_bwd(du, qh2, dqin, dh3);
    } else {
      mn_block_bwd(dEnc, encOut, dqin, dh3);
    }
    if (cfg.mn_qi) {
      tanh_bwd(cx, dpre, dqin, qi_proj, N * H);
      float* dqj = arena.get<float>(N * (H + cfg.F));
      linear_bwd(seg("mn.qi.weight"), qi_join, dpre, N, dqj, 0.f);
      copy_cols(cx, dq3, H, dqj, H + cfg.F, N, H);
    }
    // gradient sync, bucket 1: every non-recurrent layer of the encoder is final here, before the LSTM BPTTs start
    if (cfg.san) reduce_segments(seg(cfg.mn_qi ? "mn.qi.weight" : "mn.fact.weight"), seg("san.out.weight") + 1, main_stream);
  }

  // question LSTMs (+ gradients handed back by the gen decoder, gen.lua:45-60); the history chain's BPTT runs
  // concurrently on the side stream (disjoint weight segments; the shared embedding gradient is atomics-only).  Deterministic
  // mode: the history's embedding gradient is added after the join, behind the question's (its route adds without atomics)
  const bool embdrop = cfg.embdrop;
  const float* hist_dx = nullptr;
  if (cfg.useHist) {
    if (serial_pairs()) join_side(); else fork_side();
    const PairStreams& hs = serial_pairs() ? main_chain : side_chain;
    float* dx1 = arena.get<float>(N * db.Th * E);
    lstm_pair_backward(hist1, hist2, dh3, nullptr, nullptr, nullptr, dx1, hs);
    reduce_segments(seg("hist.lstm1.weight"), seg("hist.lstm2.weight") + 1, hs.a);              // bucket 2
    if (cx.deterministic) hist_dx = dx1;
    else embed_scatter_add(cx, dWp(0), dx1, E, ids_h, N * db.Th, E, embdrop ? d05 : dnone, SITE_HEMBED, cfg.V + 1);
    back_to_main();
  }
  {
    int D1 = ques1.D;
    float* dx1 = arena.get<float>(N * db.Tq * D1);
    lstm_pair_backward(ques1, ques2, dq3, conn_dc_l2, conn_dh_l1, conn_dc_l1, dx1, main_chain);
    reduce_segments(seg("ques.lstm1.weight"), seg("ques.lstm2.weight") + 1, main_stream);       // bucket 3
    embed_scatter_add(cx, dWp(0), dx1, D1, ids_q, N * db.Tq, E, embdrop ? d05 : dnone, SITE_QEMBED, cfg.V + 1);
    if (cfg.img_in_q) {
      float* die = arena.get<float>(N * cfg.IE);
      masktime_bwd(cx, dx1, D1, E, ids_q, die, db.Tq, N, cfg.IE);
      linear_bwd(seg("img.embed.weight"), img_d, die, N, nullptr, 0.f);
    }
  }
  join_side();
  if (hist_dx) embed_scatter_add(cx, dWp(0), hist_dx, E, ids_h, N * db.Th, E, embdrop ? d05 : dnone, SITE_HEMBED, cfg.V + 1);
  // what is left — the option LSTM's weights (final when the option stream ends, i.e. now), the word embedding, which every
  // branch writes, and the small layers not covered above — goes in clamp_adam_step
  // (opt.lstm, final at the same moment, goes out with the embedding in the grouped launch of reduce_remaining)
  join_options_backward();
}

void Engine::fork_side() {
  if (!side_active) {
    VD_CUDA_CHECK(cudaEventRecord(ev_fork, main_stream));
    VD_CUDA_CHECK(cudaStreamWaitEvent(side_stream, ev_fork, 0));
    side_active = true;
  }
  cx.stream = side_stream;
}
void Engine::back_to_main() { cx.stream = main_stream; }
void Engine::join_side() {
  cx.stream = main_stream;
  if (side_active) {
    VD_CUDA_CHECK(cudaEventRecord(ev_join, side_stream));
    VD_CUDA_CHECK(cudaStreamWaitEvent(main_stream, ev_join, 0));
    side_active = false;
  }
}

// ------------------------------------------------------------------------------------------------
// decoders + criterions
// ------------------------------------------------------------------------------------------------
void Engine::forward_connect() {
  // decoders/gen.lua:30-42; decoders/disc.lua:35 is a no-op
  if (cfg.dec != DEC_GEN) return;
  VD_REQUIRE(have_fwd, VD_E_STATE, "forward_connect before encoder_forward");
  gen_h0[0] = gen_h0[1] = gen_c0[0] = gen_c0[1] = nullptr;
  if (cfg.rnn_layers) {                              // encoders with .rnnLayers
    gen_h0[0] = ques1.h_last(); gen_c0[0] = ques1.c_last();
    gen_c0[1] = ques2.c_last();
  }
  gen_h0[1] = encOut;
}

// disc.lua:4-20: the option LSTM over all N*100 candidate answers.  Depends only on the batch and the weights, so it
// is enqueued on opt_stream before the encoder's kernels and meets the encoder output at disc_scores_fwd.
void Engine::options_forward_async() {
  const int64_t Ro = (dense_round ? db.B : db.N) * cfg.K;
  cudaStream_t s = opt_overlap ? opt_stream : main_stream;
  if (opt_overlap) {
    VD_CUDA_CHECK(cudaEventRecord(ev_opt_fork, main_stream));          // batch staged, shadows refreshed
    VD_CUDA_CHECK(cudaStreamWaitEvent(opt_stream, ev_opt_fork, 0));
  }
  cudaStream_t prev = cx.stream;
  cx.stream = s;
  // leave SMs to the encoder's concurrent chains; with the persistent encoder forward (VD_MATH_F16) nothing latency-bound
  // runs beside the option stream's forward: no reserve
  if (opt_overlap) cx.sm_budget = cx.sm_count - (math_mode == VD_MATH_F16 ? 0 : opt_reserve_sms);
  ids_o = arena.get<int32_t>(Ro * db.To);
  if (dense_round) transpose_ids_rounds(cx, db.options, dense_round, ids_o, db.B, cfg.R, cfg.K, db.To);
  else transpose_ids(cx, db.options, ids_o, Ro, db.To);
  opt = make_run(db.To, Ro, cfg.E, cfg.H, seg("opt.lstm.weight"), nullptr, ids_o, nullptr);   // disc.lua:4-5: no maskzero
  lstm_forward(opt, save_acts);
  VD_CUDA_CHECK(cudaEventRecord(ev_opt_done, s));
  cx.stream = prev;
  cx.sm_budget = 0;
  opt_fwd_pending = true;
}

void Engine::join_options_backward() {
  if (!opt_bwd_pending && !opt_demb && !opt_dx) return;
  cudaStream_t prev = cx.stream;
  cx.stream = main_stream;
  if (opt_bwd_pending) VD_CUDA_CHECK(cudaStreamWaitEvent(main_stream, ev_opt_done, 0));
  opt_bwd_pending = false;
  if (opt_demb) add_inplace(cx, dWp(0), opt_demb, (int64_t)(cfg.V + 1) * cfg.E);
  if (opt_dx) embed_scatter_add(cx, dWp(0), opt_dx, cfg.E, ids_o, opt.R * db.To, cfg.E, dropcfg(0.f), 0, cfg.V + 1);
  opt_demb = nullptr; opt_dx = nullptr;
  cx.stream = prev;
}

void Engine::decoder_forward() {
  VD_REQUIRE(have_fwd, VD_E_STATE, "decoder_forward before encoder_forward");
  const int E = cfg.E, H = cfg.H, K = cfg.K;
  const int64_t N = db.N;
  if (cfg.dec == DEC_DISC) {
    VD_REQUIRE(db.options && db.To > 0, VD_E_SHAPE, "disc decoder: options / To missing");
    if (!opt_fwd_pending) options_forward_async();          // normally started by encoder_forward already
    VD_CUDA_CHECK(cudaStreamWaitEvent(main_stream, ev_opt_done, 0));
    opt_fwd_pending = false;
    cx.stream = main_stream;
    scores = arena.get<float>(N * K);
    disc_scores_fwd(cx, opt.h_last(), encOut, scores, N, K, H);
  } else {
    VD_REQUIRE(db.answer_in && db.Ta > 0, VD_E_SHAPE, "gen decoder: answer_in / Ta missing");
    forward_connect();
    ids_ai = arena.get<int32_t>(N * db.Ta);
    transpose_ids(cx, db.answer_in, ids_ai, N, db.Ta);
    float* xa = arena.get<float>(N * db.Ta * E);
    embed_rows(cx, xa, Wp(0), ids_ai, N * db.Ta, E, dropcfg(0.f), 0);
    dec1 = make_run(db.Ta, N, E, H, seg("dec.lstm1.weight"), xa, nullptr, ids_ai);
    dec1.h0 = gen_h0[0]; dec1.c0 = gen_c0[0];
    lstm_forward(dec1, true);
    dec2 = make_run(db.Ta, N, H, H, seg("dec.lstm2.weight"), dec1.h, nullptr, ids_ai);
    dec2.h0 = gen_h0[1]; dec2.c0 = gen_c0[1];
    lstm_forward(dec2, true);
    fused_vocab_fwd = false;
    const int64_t rows = N * db.Ta;
    const int wo = seg("dec.out.weight");
    if (!want_logp && tcmode() && db.answer_out) {
      // whole-step entry point: nobody reads decOut, only the criterion does — keep the logits on chip
      ids_ao = arena.get<int32_t>(rows);
      transpose_ids(cx, db.answer_out, ids_ao, N, db.Ta);
      voc_nparts = vocab_lse_nparts(cfg.V);
      voc_pm = arena.get<float>(rows * voc_nparts); voc_ps = arena.get<float>(rows * voc_nparts);
      voc_tl = arena.get<float>(rows); voc_lse = arena.get<float>(rows);
      LaunchCtx::Scope sc(&cx, "vocab_lse", 2.0 * rows * cfg.V * H, 4.0 * (rows * (double)H + (double)cfg.V * H + 2.0 * rows * voc_nparts));
      fused_vocab_fwd = vocab_lse_tc(cx, (int)rows, cfg.V, H, dec2.h, H, Wp(wo), H, Wp(wo + 1), ids_ao, voc_pm, voc_ps, voc_tl);
    }
    if (!fused_vocab_fwd) {
      logp = arena.get<float>(rows * cfg.V);
      linear_fwd(wo, dec2.h, rows, logp, 0);
      logsoftmax_rows(cx, logp, ids_ai, rows, cfg.V);            // gen.lua:23-24 (MaskZero)
    } else {
      logp = nullptr;
    }
  }
}

float Engine::criterion_forward() {
  const int64_t N = db.N;
  if (cfg.dec == DEC_DISC) {
    VD_REQUIRE(scores && db.answer_ind, VD_E_STATE, "criterion: decoder_forward / answer_ind missing");
    row_loss = arena.get<float>(N);
    xent_fwd(cx, scores, db.answer_ind, row_loss, N, cfg.K);
    reduce_sum(cx, row_loss, scalars_dev, N, 1.f / (float)N);        // CrossEntropyCriterion: mean
  } else {
    VD_REQUIRE((logp || fused_vocab_fwd) && db.answer_out, VD_E_STATE, "criterion: decoder_forward / answer_out missing");
    row_loss = arena.get<float>(N * db.Ta);
    if (fused_vocab_fwd) {
      vocab_lse_finish(cx, voc_pm, voc_ps, voc_nparts, voc_tl, ids_ao, ids_ai, voc_lse, row_loss, -1.f, 0, N * db.Ta);
    } else {
      ids_ao = arena.get<int32_t>(N * db.Ta);
      transpose_ids(cx, db.answer_out, ids_ao, N, db.Ta);
      nll_fwd(cx, logp, ids_ao, ids_ai, row_loss, N * db.Ta, cfg.V);
    }
    reduce_sum(cx, row_loss, scalars_dev, N * db.Ta, 1.f);            // ClassNLL sizeAverage=false
  }
  float loss = 0.f;
  VD_CUDA_CHECK(cudaMemcpyAsync(&loss, scalars_dev, sizeof(float), cudaMemcpyDeviceToHost, cx.stream));
  VD_CUDA_CHECK(cudaStreamSynchronize(cx.stream));                    // the reference reads curLoss here too (model.lua:330)
  return loss;
}

void Engine::criterion_backward() {
  const int64_t N = db.N;
  if (cfg.dec == DEC_DISC) {
    VD_REQUIRE(scores && db.answer_ind, VD_E_STATE, "criterion_backward: decoder_forward / answer_ind missing");
    dscores = arena.get<float>(N * cfg.K);
    xent_bwd(cx, scores, db.answer_ind, dscores, N, cfg.K);
  } else {
    VD_REQUIRE((logp || fused_vocab_fwd) && ids_ao, VD_E_STATE, "criterion_backward before criterion_forward");
    dlogits = arena.get<float>(N * db.Ta * cfg.V);
    if (fused_vocab_fwd) {
      const int wo = seg("dec.out.weight");
      LaunchCtx::Scope sc(&cx, "vocab_dlogits", 2.0 * N * db.Ta * cfg.V * cfg.H, 4.0 * N * db.Ta * (double)cfg.V);
      bool ok = vocab_dlogits_tc(cx, (int)(N * db.Ta), cfg.V, cfg.H, dec2.h, cfg.H, Wp(wo), cfg.H, Wp(wo + 1), ids_ao, ids_ai, voc_lse,
                                 dlogits, cfg.V);
      VD_REQUIRE(ok, VD_E_STATE, "vocab_dlogits_tc refused a shape vocab_lse_tc took");
    } else {
      nll_bwd(cx, logp, ids_ao, ids_ai, dlogits, N * db.Ta, cfg.V);
    }
  }
}

void Engine::decoder_backward() {
  VD_REQUIRE(save_acts, VD_E_STATE, "decoder_backward needs a training-mode forward");
  if (world > 1)
    for (char c : seg_reduced)
      VD_REQUIRE(!c, VD_E_STATE, "world > 1: vd_zero_grad is required between backward passes (gradients already all-reduced)");
  const int E = cfg.E, H = cfg.H, K = cfg.K;
  const int64_t N = db.N;
  dEncFromDec = arena.get<float>(N * H);
  if (cfg.dec == DEC_DISC) {
    VD_REQUIRE(dscores, VD_E_STATE, "decoder_backward before criterion_backward");
    const int64_t Ro = N * K;
    float* dfeat = arena.get<float>(Ro * H);
    disc_scores_bwd(cx, dscores, opt.h_last(), encOut, dfeat, dEncFromDec, N, K, H);
    options_backward(dfeat);
  } else {
    VD_REQUIRE(dlogits, VD_E_STATE, "decoder_backward before criterion_backward");
    float* do2 = arena.get<float>(N * db.Ta * H);
    linear_bwd(seg("dec.out.weight"), dec2.h, dlogits, N * db.Ta, do2, 0.f);
    for (int l = 0; l < 2; ++l) { gen_dh0[l] = arena.get<float>(N * H); gen_dc0[l] = arena.get<float>(N * H); }
    float* dx2 = arena.get<float>(N * db.Ta * H);
    lstm_backward(dec2, do2, nullptr, nullptr, dx2, gen_dh0[1], gen_dc0[1]);
    float* dx1 = arena.get<float>(N * db.Ta * E);
    lstm_backward(dec1, dx2, nullptr, nullptr, dx1, gen_dh0[0], gen_dc0[0]);
    embed_scatter_add(cx, dWp(0), dx1, E, ids_ai, N * db.Ta, E, dropcfg(0.f), 0, cfg.V + 1);
  }
}

void Engine::options_backward(const float* dfeat) {
  const int E = cfg.E;
  // The option BPTT feeds only opt.lstm's weights and the word embedding: it runs on opt_stream while the caller
  // goes on to the encoder's backward; join_options_backward() (encoder_backward / any gradient consumer) waits.
  cudaStream_t prev = cx.stream;
  if (opt_overlap) {
    VD_CUDA_CHECK(cudaEventRecord(ev_opt_fork, cx.stream));
    VD_CUDA_CHECK(cudaStreamWaitEvent(opt_stream, ev_opt_fork, 0));
    cx.stream = opt_stream;
    cx.sm_budget = cx.sm_count - opt_reserve_sms;
  }
  // Deterministic mode: with or without the overlap, the option LSTM's embedding gradient is added to dW(wordEmbed) in
  // join_options_backward, after the encoder's (its routes add without atomics)
  if (opt.route.table_grad) {
    // embedding gradient in projected space; written to a private (V+1,E) buffer when overlapped, because the
    // encoder's embedding gradients accumulate into dW(wordEmbed) with atomics at the same time
    opt.demb_out = opt_overlap || cx.deterministic ? (opt_demb = arena.get<float>((int64_t)(cfg.V + 1) * E)) : nullptr;
    lstm_backward(opt, nullptr, dfeat, nullptr, nullptr, nullptr, nullptr);
  } else {
    float* dx = arena.get<float>(opt.R * db.To * E);
    lstm_backward(opt, nullptr, dfeat, nullptr, dx, nullptr, nullptr);
    if (cx.deterministic) opt_dx = dx;
    else embed_scatter_add(cx, dWp(0), dx, E, ids_o, opt.R * db.To, E, dropcfg(0.f), 0, cfg.V + 1);   // atomics: safe next to the encoder's
  }
  if (opt_overlap) {
    VD_CUDA_CHECK(cudaEventRecord(ev_opt_done, opt_stream));
    cx.stream = prev;
    cx.sm_budget = 0;
    opt_bwd_pending = true;
  }
}

void Engine::dense_targets(const vd_batch* b, const int32_t* round_host, const float* relevance_host, int32_t** rd_out,
                           float** rel_out) {
  VD_REQUIRE(b && round_host && relevance_host, VD_E_BADARG, "batch / rounds / relevance is null");
  VD_REQUIRE(b->B > 0, VD_E_SHAPE, "batch B must be > 0");
  const int B = b->B, R = cfg.R, K = cfg.K;
  for (int i = 0; i < B; ++i) {
    VD_REQUIRE(round_host[i] >= 0 && round_host[i] < R, VD_E_BADARG, "round outside [0, maxQuesCount)");
    double sum = 0.0;
    for (int k = 0; k < K; ++k) {
      const float r = relevance_host[(int64_t)i * K + k];
      VD_REQUIRE(std::isfinite(r) && r >= 0.f, VD_E_BADARG, "relevance must be finite and >= 0");
      sum += r;
    }
    VD_REQUIRE(sum > 0.0, VD_E_BADARG, "a relevance row sums to 0");
  }
  VD_CUDA_CHECK(cudaSetDevice(cfg.gpuid));
  if (opt_fwd_pending || opt_bwd_pending) {       // as encoder_forward: nothing of an abandoned call may still read these
    VD_CUDA_CHECK(cudaStreamSynchronize(opt_stream));
    opt_fwd_pending = opt_bwd_pending = false;
  }
  int32_t* rd = static_cast<int32_t*>(dense_buf[0].ensure((size_t)B * sizeof(int32_t)));
  float* rel = static_cast<float*>(dense_buf[1].ensure((size_t)B * K * sizeof(float)));
  VD_CUDA_CHECK(cudaMemcpyAsync(rd, round_host, (size_t)B * sizeof(int32_t), cudaMemcpyHostToDevice, main_stream));
  VD_CUDA_CHECK(cudaMemcpyAsync(rel, relevance_host, (size_t)B * K * sizeof(float), cudaMemcpyHostToDevice, main_stream));
  *rd_out = rd;
  *rel_out = rel;
}

float Engine::dense_loss(const float* sc, const float* rel, int B) {
  const int K = cfg.K;
  row_loss = arena.get<float>(B);
  dscores = arena.get<float>((int64_t)B * K);
  soft_xent(cx, sc, rel, row_loss, dscores, B, K);
  reduce_sum(cx, row_loss, scalars_dev, B, 1.f / (float)B);
  float loss = 0.f;
  VD_CUDA_CHECK(cudaMemcpyAsync(&loss, scalars_dev, sizeof(float), cudaMemcpyDeviceToHost, cx.stream));
  VD_CUDA_CHECK(cudaStreamSynchronize(cx.stream));                    // read where vd_forward_backward reads its loss
  return loss;
}

// vd_forward_backward_dense: the encoder over all N rounds as in vd_forward_backward (same dropout sites and masks), the
// disc decoder on the one annotated round per dialog only (B*K option rows instead of N*K), the soft-target cross-entropy
// against the relevance rows, and the encoder backward from a dEnc that is zero on every unselected round.
float Engine::forward_backward_dense(const vd_batch* b, const int32_t* round_host, const float* relevance_host) {
  VD_REQUIRE(cfg.dec == DEC_DISC, VD_E_STATE, "dense fine-tuning runs the disc decoder only");
  int32_t* rd = nullptr; float* rel = nullptr;
  dense_targets(b, round_host, relevance_host, &rd, &rel);
  const int B = b->B, R = cfg.R, K = cfg.K, H = cfg.H;
  struct Reset { const int32_t*& p; ~Reset() { p = nullptr; } } reset{dense_round};
  dense_round = rd;
  encoder_forward(b);                             // starts the option LSTM on the selected rows (options_forward_async)
  VD_REQUIRE(db.options && db.To > 0, VD_E_SHAPE, "disc decoder: options / To missing");
  VD_REQUIRE(save_acts, VD_E_STATE, "the dense step needs a training-mode forward");
  if (world > 1)
    for (char c : seg_reduced)
      VD_REQUIRE(!c, VD_E_STATE, "world > 1: vd_zero_grad is required between backward passes (gradients already all-reduced)");
  if (!opt_fwd_pending) options_forward_async();
  VD_CUDA_CHECK(cudaStreamWaitEvent(main_stream, ev_opt_done, 0));
  opt_fwd_pending = false;
  cx.stream = main_stream;
  float* enc_sel = arena.get<float>((int64_t)B * H);
  gather_round_rows(cx, encOut, rd, enc_sel, B, R, H);
  scores = arena.get<float>((int64_t)B * K);
  disc_scores_fwd(cx, opt.h_last(), enc_sel, scores, B, K, H);
  const float loss = dense_loss(scores, rel, B);
  float* dfeat = arena.get<float>((int64_t)B * K * H);
  float* denc_sel = arena.get<float>((int64_t)B * H);
  disc_scores_bwd(cx, dscores, opt.h_last(), enc_sel, dfeat, denc_sel, B, K, H);
  options_backward(dfeat);
  dEncFromDec = arena.get<float>(db.N * H);
  scatter_round_rows(cx, denc_sel, rd, dEncFromDec, B, R, H);
  encoder_backward(dEncFromDec);
  return loss;
}

// vd_forward_backward_dense_gen (DESIGN §16): the encoder over all N rounds as in vd_forward_backward; the gen decoder,
// teacher-forced, over the K candidate answers of the annotated round of each dialog only (B*K rows), started from that
// round's forward_connect() state; the scores s_bk = sum_t keep (x_t[tgt_t] - lse_t) as gen_option_lhood forms them; the
// soft-target cross-entropy; and the backward with d-logits  -g_bk keep (softmax(x_t) - onehot(tgt_t)),  g = dscores.
float Engine::forward_backward_dense_gen(const vd_batch* b, const int32_t* round_host, const float* relevance_host) {
  VD_REQUIRE(cfg.dec == DEC_GEN, VD_E_STATE, "the gen dense step runs the gen decoder only");
  int32_t* rd = nullptr; float* rel = nullptr;
  dense_targets(b, round_host, relevance_host, &rd, &rel);
  VD_REQUIRE(b->option_in && b->option_out && b->To > 0, VD_E_SHAPE, "gen dense step: option_in / option_out / To missing");
  encoder_forward(b);
  VD_REQUIRE(save_acts, VD_E_STATE, "the dense step needs a training-mode forward");
  if (world > 1)
    for (char c : seg_reduced)
      VD_REQUIRE(!c, VD_E_STATE, "world > 1: vd_zero_grad is required between backward passes (gradients already all-reduced)");
  cx.stream = main_stream;
  forward_connect();
  const int B = b->B, R = cfg.R, K = cfg.K, E = cfg.E, H = cfg.H, V = cfg.V, To = db.To;
  const int64_t Ro = (int64_t)B * K, TR = (int64_t)To * Ro;
  // the annotated rounds' option tokens, time-major (To, B*K) as the disc options are taken
  int32_t* oi = arena.get<int32_t>(TR);
  int32_t* oo = arena.get<int32_t>(TR);
  transpose_ids_rounds(cx, db.option_in, rd, oi, B, R, K, To);
  transpose_ids_rounds(cx, db.option_out, rd, oo, B, R, K, To);
  // initial state: row b*K + k <- round rd[b] of dialog b (null layer-1 state stays null: encoders without .rnnLayers)
  const float* st0[4] = {gen_h0[0], gen_h0[1], gen_c0[0], gen_c0[1]};
  const float* st[4] = {nullptr, nullptr, nullptr, nullptr};
  float* sel = arena.get<float>((int64_t)B * H);
  for (int i = 0; i < 4; ++i) {
    if (!st0[i]) continue;
    float* t = arena.get<float>(Ro * H);
    gather_round_rows(cx, st0[i], rd, sel, B, R, H);
    repeat_rows(cx, t, sel, B, K, H);
    st[i] = t;
  }
  // decoders/gen.lua:3-27 over the selected options, activations saved (decoder_forward's kernels)
  float* xo = arena.get<float>(TR * E);
  embed_rows(cx, xo, Wp(0), oi, TR, E, dropcfg(0.f), 0);
  LstmRun l1 = make_run(To, Ro, E, H, seg("dec.lstm1.weight"), xo, nullptr, oi);
  l1.h0 = st[0]; l1.c0 = st[2];
  lstm_forward(l1, true);
  LstmRun l2 = make_run(To, Ro, H, H, seg("dec.lstm2.weight"), l1.h, nullptr, oi);
  l2.h0 = st[1]; l2.c0 = st[3];
  lstm_forward(l2, true);
  // per-step vocabulary statistics on gen_option_lhood's two routes; lse (To, B*K) is kept for the backward
  const int wo = seg("dec.out.weight");
  float* lse = arena.get<float>(TR);
  scores = arena.get<float>(Ro);
  VD_CUDA_CHECK(cudaMemsetAsync(scores, 0, (size_t)Ro * sizeof(float), cx.stream));
  bool fused = tcmode();
  for (int t = 0; t < To && fused; ++t) fused = vocab_tc_ok((int)Ro, V, H, l2.h + (int64_t)t * Ro * H, H, Wp(wo), H);
  if (fused) {
    const int nparts = vocab_lse_nparts(V);
    float* pm = arena.get<float>(Ro * nparts);
    float* ps = arena.get<float>(Ro * nparts);
    float* tl = arena.get<float>(Ro);
    for (int t = 0; t < To; ++t) {
      const int64_t o = (int64_t)t * Ro;
      {
        LaunchCtx::Scope sc(&cx, "vocab_lse", 2.0 * Ro * V * H, 4.0 * (Ro * (double)H + (double)V * H + 2.0 * Ro * nparts));
        const bool ok = vocab_lse_tc(cx, (int)Ro, V, H, l2.h + o * H, H, Wp(wo), H, Wp(wo + 1), oo + o, pm, ps, tl);
        VD_REQUIRE(ok, VD_E_STATE, "vocab_lse_tc refused a shape vocab_tc_ok took");
      }
      vocab_lse_finish(cx, pm, ps, nparts, tl, oo + o, oi + o, lse + o, scores, 1.f, 1, Ro);
    }
  } else {
    float* logits = arena.get<float>(Ro * V);
    for (int t = 0; t < To; ++t) {
      const int64_t o = (int64_t)t * Ro;
      linear_fwd(wo, l2.h + o * H, Ro, logits, 0);
      LaunchCtx::Scope sc(&cx, "vocab_lse_rows", 0.0, 4.0 * Ro * (double)V);
      lhood_accumulate(cx, logits, oo + o, oi + o, scores, Ro, V, lse + o);
    }
  }
  const float loss = dense_loss(scores, rel, B);
  float* nscale = arena.get<float>(Ro);
  scale_copy(cx, nscale, dscores, Ro, -1.f);        // d loss / d s_bk = g_bk; s_bk enters the logits with sign -1
  // d-logits a chunk of time steps at a time: at most dense_gen_chunk_bytes of them live (never (To*B*K, V)); per chunk,
  // dec.out's dW / db accumulate and the chunk's rows of dh2 (the gradient at layer 2's outputs) are written
  float* dh2 = arena.get<float>(TR * H);
  const int64_t step_bytes = Ro * V * (int64_t)sizeof(float);
  const int per_chunk = (int)std::max<int64_t>(1, std::min<int64_t>(To, dense_gen_chunk_bytes / step_bytes));
  const Arena::Mark mk = arena.mark();
  for (int t0 = 0; t0 < To; t0 += per_chunk) {
    const int nt = std::min(per_chunk, To - t0);
    arena.rewind(mk);
    float* dl = arena.get<float>((int64_t)nt * Ro * V);
    for (int t = t0; t < t0 + nt; ++t) {
      const int64_t o = (int64_t)t * Ro;
      float* dlt = dl + (int64_t)(t - t0) * Ro * V;
      if (fused) {
        LaunchCtx::Scope sc(&cx, "vocab_dlogits", 2.0 * Ro * V * H, 4.0 * Ro * (double)V);
        const bool ok = vocab_dlogits_tc(cx, (int)Ro, V, H, l2.h + o * H, H, Wp(wo), H, Wp(wo + 1), oo + o, oi + o, lse + o, dlt, V,
                                         nscale);
        VD_REQUIRE(ok, VD_E_STATE, "vocab_dlogits_tc refused a shape vocab_lse_tc took");
      } else {
        linear_fwd(wo, l2.h + o * H, Ro, dlt, 0);
        LaunchCtx::Scope sc(&cx, "vocab_dlogits_rows", 0.0, 8.0 * Ro * (double)V);
        nll_bwd_scaled(cx, dlt, lse + o, oo + o, oi + o, nscale, dlt, Ro, V);
      }
    }
    linear_bwd(wo, l2.h + (int64_t)t0 * Ro * H, dl, (int64_t)nt * Ro, dh2 + (int64_t)t0 * Ro * H, 0.f);
  }
  arena.rewind(mk);
  // BPTT through both layers, then the embedding gradient of option_in (decoder_backward's kernels)
  float* dst[4] = {nullptr, nullptr, nullptr, nullptr};      // d(h0, c0) per option row, for the initial states that exist
  for (int i = 0; i < 4; ++i) if (st[i]) dst[i] = arena.get<float>(Ro * H);
  float* dx2 = arena.get<float>(TR * H);
  lstm_backward(l2, dh2, nullptr, nullptr, dx2, dst[1], dst[3]);
  float* dx1 = arena.get<float>(TR * E);
  lstm_backward(l1, dx2, nullptr, nullptr, dx1, dst[0], dst[2]);
  embed_scatter_add(cx, dWp(0), dx1, E, oi, TR, E, dropcfg(0.f), 0, cfg.V + 1);
  // the K options' initial-state gradients summed per dialog (fixed k order, no atomics), onto the annotated round
  float** gout[4] = {&gen_dh0[0], &gen_dh0[1], &gen_dc0[0], &gen_dc0[1]};
  for (int i = 0; i < 4; ++i) {
    *gout[i] = nullptr;
    if (!dst[i]) continue;
    *gout[i] = arena.get<float>(db.N * H);
    {
      LaunchCtx::Scope sc(&cx, "dense_state_sum", (double)Ro * H, 4.0 * (Ro + B) * (double)H);
      sum_repeated_rows(cx, sel, dst[i], B, K, H);
    }
    scatter_round_rows(cx, sel, rd, *gout[i], B, R, H);
  }
  encoder_backward(backward_connect());
  return loss;
}

const float* Engine::backward_connect() {
  // decoders/gen.lua:45-60
  if (cfg.dec == DEC_DISC) return dEncFromDec;     // t[2] of model.lua:335
  conn_dh_l1 = conn_dc_l1 = conn_dc_l2 = nullptr;
  if (cfg.rnn_layers) {
    conn_dc_l1 = gen_dc0[0]; conn_dc_l2 = gen_dc0[1];
    conn_dh_l1 = gen_dh0[0];
  }
  return gen_dh0[1];
}

// Model:retrieveBatch (model.lua:344-430)
void Engine::retrieve(const vd_batch* b, int use_gt, int32_t* ranks_host) {
  VD_REQUIRE(ranks_host != nullptr, VD_E_BADARG, "ranks_host is null");
  int saved_training = training;
  training = 0;
  try {
    encoder_forward(b);
    const int64_t N = db.N;
    const float* sc_dev = nullptr;
    if (cfg.dec == DEC_DISC) { decoder_forward(); sc_dev = scores; }
    else { gen_option_lhood(); sc_dev = lhood; }
    if (use_gt) VD_REQUIRE(db.answer_ind, VD_E_SHAPE, "use_gt needs answer_ind");
    int64_t nout = use_gt ? N : N * cfg.K;
    int32_t* ranks = arena.get<int32_t>(nout);
    rank_rows(cx, sc_dev, use_gt ? db.answer_ind : nullptr, ranks, N, cfg.K);
    VD_CUDA_CHECK(cudaMemcpyAsync(ranks_host, ranks, (size_t)nout * sizeof(int32_t), cudaMemcpyDeviceToHost, cx.stream));
    VD_CUDA_CHECK(cudaStreamSynchronize(cx.stream));
  } catch (...) { training = saved_training; throw; }
  training = saved_training;
}

// gen retrieval: the 100-iteration option loop of model.lua:405-415 batched over (N*100) rows, log-likelihood
// accumulated per time step without materialising (T,N*100,V) log-probs.
void Engine::gen_option_lhood() {
  VD_REQUIRE(cfg.dec == DEC_GEN, VD_E_STATE, "gen_option_lhood needs the gen decoder");
  VD_REQUIRE(have_fwd && db.option_in && db.option_out && db.To > 0, VD_E_SHAPE, "option_in / option_out / To missing");
  const int E = cfg.E, H = cfg.H, K = cfg.K, V = cfg.V;
  const int64_t N = db.N, Ro = N * K;
  forward_connect();
  int32_t* oi = arena.get<int32_t>(Ro * db.To);
  int32_t* oo = arena.get<int32_t>(Ro * db.To);
  transpose_ids(cx, db.option_in, oi, Ro, db.To);
  transpose_ids(cx, db.option_out, oo, Ro, db.To);
  // (h0,c0) repeated over the K options of a round: row (n,k) <- row n
  const float* h0[2] = {nullptr, nullptr}; const float* c0[2] = {nullptr, nullptr};
  for (int l = 0; l < 2; ++l) {
    if (gen_h0[l]) { float* t = arena.get<float>(Ro * H); repeat_rows(cx, t, gen_h0[l], N, K, H); h0[l] = t; }
    if (gen_c0[l]) { float* t = arena.get<float>(Ro * H); repeat_rows(cx, t, gen_c0[l], N, K, H); c0[l] = t; }
  }
  LstmRun l1 = make_run(db.To, Ro, E, H, seg("dec.lstm1.weight"), nullptr, oi, oi);
  l1.h0 = h0[0]; l1.c0 = c0[0];
  lstm_forward(l1, true);
  LstmRun l2 = make_run(db.To, Ro, H, H, seg("dec.lstm2.weight"), l1.h, nullptr, oi);
  l2.h0 = h0[1]; l2.c0 = c0[1];
  lstm_forward(l2, true);
  lhood = arena.get<float>(Ro);
  VD_CUDA_CHECK(cudaMemsetAsync(lhood, 0, (size_t)Ro * sizeof(float), cx.stream));
  int wo = seg("dec.out.weight");
  // utils.computeLhood per time step.  Tensor-core modes: the vocabulary projection keeps its (N*100, V) logits on chip and
  // writes (max, sum exp) partials + the target logit only (20 MB per step instead of 1.28 GB written and read back)
  const int nparts = vocab_lse_nparts(V);
  float *pm = nullptr, *ps = nullptr, *tl = nullptr, *logits = nullptr;
  bool fused = tcmode() && Ro >= 64 && V >= 256;
  if (fused) { pm = arena.get<float>(Ro * nparts); ps = arena.get<float>(Ro * nparts); tl = arena.get<float>(Ro); }
  for (int t = 0; t < db.To; ++t) {
    const float* ht = l2.h + (int64_t)t * Ro * H;
    if (fused) {
      LaunchCtx::Scope sc(&cx, "vocab_lse", 2.0 * Ro * V * H, 4.0 * (Ro * (double)H + (double)V * H + 2.0 * Ro * nparts));
      fused = vocab_lse_tc(cx, (int)Ro, V, H, ht, H, Wp(wo), H, Wp(wo + 1), oo + (int64_t)t * Ro, pm, ps, tl);
      VD_REQUIRE(fused || t == 0, VD_E_STATE, "vocab_lse_tc changed its mind between time steps");
    }
    if (fused) {
      vocab_lse_finish(cx, pm, ps, nparts, tl, oo + (int64_t)t * Ro, oi + (int64_t)t * Ro, nullptr, lhood, 1.f, 1, Ro);
    } else {
      if (!logits) logits = arena.get<float>(Ro * V);
      linear_fwd(wo, ht, Ro, logits, 0);
      lhood_accumulate(cx, logits, oo + (int64_t)t * Ro, oi + (int64_t)t * Ro, lhood, Ro, V);
    }
  }
}

// Model:generateAnswers' inner decoder call (model.lua:517-526): decoders/gen.lua:3-27 for ONE time step on `rows`
// independent rows with explicit previous state.  Same kernels, in the same order, as decoder_forward's gen branch with
// Ta = 1 (dense embedded input, maskzero on the token, MaskZero'd Linear + LogSoftMax).
void Engine::gen_decoder_step(int64_t rows, const int32_t* tokens_host, const float* const* h_prev, const float* const* c_prev) {
  VD_REQUIRE(cfg.dec == DEC_GEN, VD_E_STATE, "gen_decoder_step needs the gen decoder");
  // the step reads only its explicit state and the weights' transposed shadow, which an encoder forward and a dialog ask
  // both refresh: after an ask it replays the ask's search from vd_dialog_encoding / vd_dialog_rnn_state
  VD_REQUIRE(have_fwd || dses.encOut, VD_E_STATE, "gen_decoder_step before encoder_forward or a dialog ask");
  VD_REQUIRE(rows > 0 && tokens_host != nullptr, VD_E_BADARG, "rows / tokens");
  VD_CUDA_CHECK(cudaSetDevice(cfg.gpuid));
  cx.stream = main_stream;
  int32_t* tok = arena.get<int32_t>(rows);
  VD_CUDA_CHECK(cudaMemcpyAsync(tok, tokens_host, (size_t)rows * sizeof(int32_t), cudaMemcpyHostToDevice, cx.stream));
  VD_CUDA_CHECK(cudaStreamSynchronize(cx.stream));               // tokens_host may be a temporary of the caller
  gen_decoder_step_logits(rows, tok, h_prev, c_prev);
  logsoftmax_rows(cx, gstep_logp, tok, rows, cfg.V);            // gen.lua:23-24 (MaskZero)
}

void Engine::gen_decoder_step_logits(int64_t rows, const int32_t* tok, const float* const* h_prev, const float* const* c_prev) {
  gen_decoder_step_lstm(rows, tok, h_prev, c_prev);
  gstep_logp = arena.get<float>(rows * cfg.V);
  linear_fwd(seg("dec.out.weight"), gstep2.h, rows, gstep_logp, 0);
}

void Engine::gen_decoder_step_lstm(int64_t rows, const int32_t* tok, const float* const* h_prev, const float* const* c_prev) {
  const int E = cfg.E, H = cfg.H;
  float* xa = arena.get<float>(rows * E);
  embed_rows(cx, xa, Wp(0), tok, rows, E, dropcfg(0.f), 0);
  gstep1 = make_run(1, rows, E, H, seg("dec.lstm1.weight"), xa, nullptr, tok);
  gstep1.h0 = h_prev ? h_prev[0] : nullptr; gstep1.c0 = c_prev ? c_prev[0] : nullptr;
  lstm_forward(gstep1, true);
  gstep2 = make_run(1, rows, H, H, seg("dec.lstm2.weight"), gstep1.h, nullptr, tok);
  gstep2.h0 = h_prev ? h_prev[1] : nullptr; gstep2.c0 = c_prev ? c_prev[1] : nullptr;
  lstm_forward(gstep2, true);
}

// Model:generateAnswers' beam search (model.lua:472-579) for all N rounds of the last encoder forward at once; with G > 1
// groups, diverse beam search (DESIGN §22); with nc, n-best lists (DESIGN §24).
void Engine::gen_beam_search(int k, int G, float lam, int L, int start_token, int end_token, int32_t* answer_host,
                             int32_t* length_host, double* score_host, const NBestCfg& nc) {
  VD_REQUIRE(cfg.dec == DEC_GEN && have_fwd, VD_E_STATE, "gen_beam_search needs the gen decoder after encoder_forward");
  check_beam_args(k, G, lam, L, nc);
  check_rules(L, end_token, true);
  VD_REQUIRE(answer_host && length_host && score_host, VD_E_BADARG, "null output pointer");
  VD_CUDA_CHECK(cudaSetDevice(cfg.gpuid));
  cx.stream = main_stream;
  const int64_t NG = db.N * G * nc.nbest;
  const double* lp = length_penalty_table(nc.alpha, L);
  const BeamResult res = beam_search_rows(db.N, 1, 0, k, G, lam, L, start_token, end_token, nc.nbest, lp);
  VD_CUDA_CHECK(cudaMemcpyAsync(answer_host, res.gans, (size_t)NG * L * sizeof(int32_t), cudaMemcpyDeviceToHost, cx.stream));
  VD_CUDA_CHECK(cudaMemcpyAsync(length_host, res.glen, (size_t)NG * sizeof(int32_t), cudaMemcpyDeviceToHost, cx.stream));
  VD_CUDA_CHECK(cudaMemcpyAsync(score_host, res.gscore, (size_t)NG * sizeof(double), cudaMemcpyDeviceToHost, cx.stream));
  if (nc.norm_host)
    VD_CUDA_CHECK(cudaMemcpyAsync(nc.norm_host, res.gnorm, (size_t)NG * sizeof(double), cudaMemcpyDeviceToHost, cx.stream));
  VD_CUDA_CHECK(cudaStreamSynchronize(cx.stream));
}

void Engine::set_answer_rules(int32_t min_words, int32_t no_repeat_ngram, int32_t n_banned, const int32_t* banned_host) {
  VD_REQUIRE(min_words >= 0 && no_repeat_ngram >= 0 && n_banned >= 0, VD_E_BADARG, "answer rules: counts must be >= 0");
  VD_REQUIRE(n_banned <= 1024, VD_E_BADARG, "answer rules: at most 1024 banned ids");
  VD_REQUIRE(banned_host || n_banned == 0, VD_E_BADARG, "answer rules: null banned ids");
  for (int i = 0; i < n_banned; ++i)
    VD_REQUIRE(banned_host[i] >= 1 && banned_host[i] <= cfg.V, VD_E_BADARG, "answer rules: a banned id outside [1, vocabSize]");
  const bool active = rules_active(min_words, no_repeat_ngram, n_banned);
  VD_REQUIRE(!active || cfg.V <= TRUNC_MAX_V, VD_E_BADARG, "answer rules keep a row's barred set in shared memory: vocabSize <= 49152");
  if (n_banned > 0) {
    VD_CUDA_CHECK(cudaSetDevice(cfg.gpuid));
    int32_t* d = (int32_t*)rules_banned.ensure((size_t)n_banned * sizeof(int32_t));
    VD_CUDA_CHECK(cudaMemcpy(d, banned_host, (size_t)n_banned * sizeof(int32_t), cudaMemcpyHostToDevice));
  }
  rules.min_words = min_words;
  rules.no_repeat_ngram = no_repeat_ngram;
  rules.banned.assign(banned_host, banned_host + n_banned);
  rules.active = active;
}

void Engine::check_rules(int L, int end_token, bool beam) const {
  if (!rules.active) return;
  VD_REQUIRE(end_token >= 1 && end_token <= cfg.V, VD_E_BADARG, "answer rules: end_token in [1, vocabSize]");
  for (int32_t b : rules.banned) VD_REQUIRE(b != end_token, VD_E_BADARG, "answer rules: end_token is banned");
  VD_REQUIRE(rules.min_words <= (beam ? L - 2 : L - 1), VD_E_BADARG,
             beam ? "answer rules: min_words > beam_len - 2 (no answer could finish)" : "answer rules: min_words > beam_len - 1");
}

AnswerRules Engine::answer_rules(int end_token, int step, const int32_t* hist, int64_t ld) const {
  AnswerRules a;
  a.min_words = rules.min_words; a.no_repeat_ngram = rules.no_repeat_ngram; a.n_banned = (int32_t)rules.banned.size();
  a.banned = a.n_banned ? (const int32_t*)rules_banned.p : nullptr;
  a.end_token = end_token; a.step = step; a.hist = hist; a.ld = ld;
  return a;
}

void Engine::check_beam_args(int k, int G, float lam, int L, const NBestCfg& nc) const {
  VD_REQUIRE(nc.nbest >= 1 && nc.nbest <= 32, VD_E_BADARG, "nbest in [1, 32]");
  VD_REQUIRE(std::isfinite(nc.alpha) && nc.alpha >= 0.f, VD_E_BADARG, "length_penalty finite and >= 0");
  VD_REQUIRE(k >= 1 && k <= 32 && k <= cfg.V && L >= 2, VD_E_BADARG, "beam_size in [1, min(32, vocabSize)], beam_len >= 2");
  VD_REQUIRE(G >= 1 && k % G == 0, VD_E_BADARG, "groups >= 1 and a divisor of beam_size");
  VD_REQUIRE(std::isfinite(lam) && lam >= 0.f, VD_E_BADARG, "diversity finite and >= 0");
}

// lp(l) = ((5 + l) / 6)^alpha (Wu et al., arXiv:1609.08144) for l = 0 .. L-1, in fp64 with the C library's pow, so that a
// host twin calling the same pow gets the same bits; the device never calls pow.  The copy is from pageable memory: it
// has left `t` when cudaMemcpyAsync returns.  alpha 0: null, every lp is exactly 1.
const double* Engine::length_penalty_table(float alpha, int L) {
  if (alpha == 0.f) return nullptr;
  std::vector<double> t(L);
  for (int l = 0; l < L; ++l) t[l] = std::pow((5.0 + l) / 6.0, (double)alpha);
  double* d = (double*)beam_lp.ensure((size_t)L * sizeof(double));
  VD_CUDA_CHECK(cudaMemcpyAsync(d, t.data(), (size_t)L * sizeof(double), cudaMemcpyHostToDevice, cx.stream));
  return d;
}

// The search itself, enqueued on cx.stream, for n rounds whose start state is row i * stride + off of the last encoder
// forward (i < n; stride 1, off 0: every round): row i*k + j is hypothesis j of round i.  Every step runs on device-resident
// tokens and parents: the state gather, the decoder step of gen_decoder_step_logits, the fused log-softmax + top-k and the
// candidate merge, which writes the next step's tokens and parents.  The merge fills G groups of k / G columns in order,
// penalising the tokens earlier groups chose (DESIGN §22); its top-k input is the same k per row at any G.  Returns each
// group's list of its nbest best finished hypotheses by norm (lp: the length-penalty table, DESIGN §24) and each round's
// pick in the arena, valid until the next encoder forward.
Engine::BeamResult Engine::beam_search_rows(int64_t n, int64_t stride, int64_t off, int k, int G, float lam, int L,
                                            int start_token, int end_token, int nbest, const double* lp) {
  forward_connect();
  const int H = cfg.H;
  const int64_t N = n, rows = N * k;
  // allocated once per call.  Two sets of fed states {h1, h2, c1, c2}: the gather of step s reads the set step s-1 was
  // fed (a column that got no candidate keeps it) and writes the other; beams / scores ping-pong because the merge fills
  // columns from the pre-merge beams.
  float* st[2][4];
  for (auto& s : st)
    for (auto& p : s) p = arena.get<float>(rows * H);
  int32_t* beams[2] = {arena.get<int32_t>(rows * L), arena.get<int32_t>(rows * L)};
  double* scores[2] = {arena.get<double>(rows), arena.get<double>(rows)};
  int32_t* tok = arena.get<int32_t>(rows);
  int32_t* parent = arena.get<int32_t>(rows);
  float* tv = arena.get<float>(rows * k);
  int32_t* ti = arena.get<int32_t>(rows * k);
  // the lists' slots (a slot's tokens past its length stay 0); the norms and the order are read only where filled
  const int64_t NL = N * G * nbest;
  BeamLists lists;
  lists.nbest = nbest;
  lists.lp = lp;
  lists.ans = arena.get<int32_t>(NL * L);
  lists.len = arena.get<int32_t>(NL);
  lists.score = arena.get<double>(NL);
  VD_CUDA_CHECK(cudaMemsetAsync(lists.ans, 0, (size_t)NL * L * sizeof(int32_t), cx.stream));
  VD_CUDA_CHECK(cudaMemsetAsync(lists.len, 0, (size_t)NL * sizeof(int32_t), cx.stream));
  VD_CUDA_CHECK(cudaMemsetAsync(lists.score, 0, (size_t)NL * sizeof(double), cx.stream));
  if (lp || nbest > 1) lists.norm = arena.get<double>(NL);
  BeamResult res = {lists.ans, lists.len, lists.score, lists.ans, lists.len, lists.score, lists.norm ? lists.norm : lists.score};
  if (nbest > 1) {                                 // the last step's merge writes the lists in order
    lists.ord = arena.get<int32_t>(NL);
    res.gans = lists.out_ans = arena.get<int32_t>(NL * L);
    res.glen = lists.out_len = arena.get<int32_t>(NL);
    res.gscore = lists.out_score = arena.get<double>(NL);
    res.gnorm = lists.out_norm = arena.get<double>(NL);
  }
  // G > 1 or nbest > 1: the last step's merge also writes each round's pick
  const bool pick = G > 1 || nbest > 1;
  if (pick) { res.ans = arena.get<int32_t>(N * L); res.len = arena.get<int32_t>(N); res.score = arena.get<double>(N); }
  int32_t* pick_ans = pick ? res.ans : nullptr;
  // model.lua:478-503: h = {layer-1 h at Tq, encOut}, c = {layer-1 c, layer-2 c}, each round's row repeated k times.  Encoders
  // without .rnnLayers feed explicit zero rows, not "no initial state": the first step's kernels differ between the two.
  const float* init[4] = {gen_h0[0], gen_h0[1], gen_c0[0], gen_c0[1]};
  for (int i = 0; i < 4; ++i) {
    if (init[i]) repeat_rows(cx, st[0][i], init[i] + off * H, N, k, H, stride * H);
    else VD_CUDA_CHECK(cudaMemsetAsync(st[0][i], 0, (size_t)rows * H * sizeof(float), cx.stream));
  }
  beam_init(cx, rows, L, start_token, beams[0], tok, scores[0]);
  const Arena::Mark step_mark = arena.mark();
  for (int stp = 1; stp < L; ++stp) {
    float* const* fed = st[(stp - 1) & 1];
    if (stp > 1) {
      const float* out[4] = {gstep1.h, gstep2.h, gstep1.c, gstep2.c};
      for (int i = 0; i < 4; ++i) beam_gather(cx, fed[i], out[i], st[stp & 1][i], parent, rows, H);
    }
    arena.rewind(step_mark);                       // every step's decoder buffers land where the last step's were
    const float* h[2] = {fed[0], fed[1]};
    const float* c[2] = {fed[2], fed[3]};
    gen_decoder_step_logits(rows, tok, h, c);
    const int a = (stp - 1) & 1;
    // the answer rules read each row's pre-merge beam: positions 1 .. stp-1 are its words so far
    const AnswerRules ar = answer_rules(end_token, stp, beams[a], L);
    logsoftmax_topk_rows(cx, gstep_logp, tok, rows, cfg.V, k, tv, ti, rules.active ? &ar : nullptr);
    // the top-k lists, the scores and beams in and out
    LaunchCtx::Scope sc(&cx, "beam_merge", 0.0, 8.0 * rows * k + 16.0 * rows + 8.0 * rows * (stp + 1));
    beam_merge(cx, N, stp, k, G, lam, L, end_token, tv, ti, scores[a], scores[a ^ 1], beams[a], beams[a ^ 1], tok, parent, lists,
               pick_ans, pick_ans ? res.len : nullptr, pick_ans ? res.score : nullptr, rules.active);
  }
  return res;
}

// Model:generateAnswers' sampling (model.lua:581-602) for all N rounds of the last encoder forward at once, on the device.
void Engine::gen_sample(int L, int start_token, float temperature, uint64_t seed, int64_t row_offset, int32_t* answer_host,
                        float* logp_host, const TruncCfg& tr) {
  VD_REQUIRE(cfg.dec == DEC_GEN && have_fwd, VD_E_STATE, "gen_sample needs the gen decoder after encoder_forward");
  check_sample_args(L, start_token, temperature, row_offset, tr);
  check_rules(L, cfg.V, false);                    // no end_token argument: <END> is vocabSize, the dataloader's
  VD_REQUIRE(answer_host, VD_E_BADARG, "null answer pointer");
  VD_CUDA_CHECK(cudaSetDevice(cfg.gpuid));
  cx.stream = main_stream;
  const int64_t N = db.N;
  const SampleResult res = sample_rows(N, 1, 0, L, start_token, temperature, seed, row_offset, -1, 0, nullptr, tr);
  VD_CUDA_CHECK(cudaMemcpyAsync(answer_host, res.ans, (size_t)N * (L + 1) * sizeof(int32_t), cudaMemcpyDeviceToHost, cx.stream));
  if (logp_host)
    VD_CUDA_CHECK(cudaMemcpyAsync(logp_host, res.logp, (size_t)N * L * sizeof(float), cudaMemcpyDeviceToHost, cx.stream));
  VD_CUDA_CHECK(cudaStreamSynchronize(cx.stream));
}

void Engine::check_sample_args(int L, int start_token, float temperature, int64_t row_offset, const TruncCfg& tr) const {
  VD_REQUIRE(L >= 1 && std::isfinite(temperature) && temperature > 0.f && row_offset >= 0 && start_token >= 1 &&
             start_token <= cfg.V, VD_E_BADARG, "beam_len >= 1, finite temperature > 0, row_offset >= 0, start_token in [1, V]");
  VD_REQUIRE(tr.top_k >= 0 && std::isfinite(tr.top_p) && tr.top_p > 0.f && tr.top_p <= 1.f, VD_E_BADARG,
             "top_k >= 0, top_p in (0, 1]");
  VD_REQUIRE(!trunc_active(tr, cfg.V) || cfg.V <= TRUNC_MAX_V, VD_E_BADARG,
             "truncated sampling stages a vocabulary row in shared memory: vocabSize <= 49152");
}

// The sampling itself, enqueued on cx.stream, for n rounds whose start state is row i * stride + off of the last encoder
// forward; search row i draws as global round row_offset + i * stride + off.  Every step runs the decoder step of
// gen_decoder_step_logits on the device-resident tokens, then draws with the Gumbel-max rule of common.cuh: fused into the
// vocabulary projection's epilogue (tensor-core modes, vocab_tc_ok's shapes) or from materialised logits
// (k_logsoftmax_sample_rows).  The draw writes the next step's tokens, so nothing waits for the host.  Returns the answers
// (n, L + 1) and log-probabilities (n, L) in the arena, valid until the next encoder forward.
Engine::SampleResult Engine::sample_rows(int64_t n, int64_t stride, int64_t off, int L, int start_token, float temperature,
                                         uint64_t seed, int64_t row_offset, int64_t draw_stride, int64_t draw_off,
                                         const int64_t* draw_rounds, const TruncCfg& tr, int end_token) {
  forward_connect();
  const int H = cfg.H, V = cfg.V;
  const int64_t N = n;
  const int wo = seg("dec.out.weight");
  // allocated once per call
  float* zero = arena.get<float>(N * H);
  int32_t* tok = arena.get<int32_t>(N);
  int32_t* ans = arena.get<int32_t>(N * (L + 1));
  float* lp = arena.get<float>(N * L);
  double* unused_scores = arena.get<double>(N);
  const int nparts = vocab_lse_nparts(V);
  float *pm = nullptr, *ps = nullptr, *pk = nullptr, *px = nullptr;
  int32_t* pc = nullptr;
  // active truncation needs each row's boundaries before its draw, and active answer rules its barred set, which the fused
  // epilogue cannot have: the rows route
  const bool trunc = trunc_active(tr, V), rows_route = trunc || rules.active;
  if (tcmode() && !rows_route) {
    pm = arena.get<float>(N * nparts); ps = arena.get<float>(N * nparts); pk = arena.get<float>(N * nparts);
    px = arena.get<float>(N * nparts); pc = arena.get<int32_t>(N * nparts);
  }
  VD_CUDA_CHECK(cudaMemsetAsync(zero, 0, (size_t)N * H * sizeof(float), cx.stream));
  beam_init(cx, N, L + 1, start_token, ans, tok, unused_scores);       // answer column 0 = <START>, tokens = <START>
  // h = {layer-1 h at Tq, encOut}, c = {layer-1 c, layer-2 c} (gen.lua:30-42); encoders without .rnnLayers feed explicit zero
  // rows, not "no initial state", as gen_beam_search does
  const float* h[2] = {gen_h0[0] ? gen_h0[0] : zero, gen_h0[1]};
  const float* c[2] = {gen_c0[0] ? gen_c0[0] : zero, gen_c0[1] ? gen_c0[1] : zero};
  if (stride != 1 || off != 0) {                     // the start state's rows i * stride + off, gathered once
    const float** init[4] = {&h[0], &h[1], &c[0], &c[1]};
    for (const float** p : init) {
      if (*p == zero) continue;
      float* t = arena.get<float>(N * H);
      repeat_rows(cx, t, *p + off * H, N, 1, H, stride * H);
      *p = t;
    }
  }
  if (draw_stride < 0) { draw_stride = stride; draw_off = off; }
  SampleCfg smp = {(uint32_t)seed, (uint32_t)(seed >> 32), 0, temperature, row_offset + draw_off, draw_stride, draw_rounds};
  // The step's decoder buffers alternate between two arena regions: step s reads the state step s-1 wrote into the other
  // one, so the new state feeds the next step without a copy.  Same allocations every step, so a region lands where it
  // did two steps earlier and the arena does not grow with L.
  Arena::Mark region[2] = {arena.mark(), {}};
  bool fused = false;
  for (int stp = 1; stp <= L; ++stp) {
    if (stp == 2) region[1] = arena.mark();
    arena.rewind(region[(stp - 1) & 1]);
    gen_decoder_step_lstm(N, tok, h, c);
    smp.step = (uint32_t)stp;
    bool took = false;
    if (tcmode() && !rows_route && (stp == 1 || fused)) {
      LaunchCtx::Scope sc(&cx, "vocab_sample", 2.0 * N * V * H, 4.0 * (N * (double)H + (double)V * H + 5.0 * N * nparts));
      took = vocab_sample_tc(cx, (int)N, V, H, gstep2.h, H, Wp(wo), H, Wp(wo + 1), smp, pm, ps, pk, pc, px);
      if (took) vocab_sample_finish(cx, pm, ps, pk, pc, px, nparts, N, stp, L, tok, ans, lp);
    }
    if (stp == 1) fused = took;
    VD_REQUIRE(took == fused, VD_E_STATE, "vocab_sample_tc changed its mind between steps");
    if (!fused) {
      // logits written once, read by the row's lse (two passes) and the draw (truncated: the lse and the row's staging in
      // shared memory, which the selection and the draw read)
      LaunchCtx::Scope sc(&cx, trunc ? "truncated_sample" : "sample_rows", 2.0 * N * V * H,
                          4.0 * (N * (double)H + (double)V * H + (trunc ? 4.0 : 2.0) * N * V));
      float* logits = arena.get<float>(N * V);
      linear_fwd(wo, gstep2.h, N, logits, 0);
      // the answer rules read each row's answer so far: positions 1 .. stp-1
      const AnswerRules ar = answer_rules(end_token > 0 ? end_token : V, stp, ans, L + 1);
      const AnswerRules* arp = rules.active ? &ar : nullptr;
      if (trunc) truncated_sample_rows(cx, logits, N, V, smp, tr, L, tok, ans, lp, arp);
      else logsoftmax_sample_rows(cx, logits, N, V, smp, L, tok, ans, lp, arp);
    }
    h[0] = gstep1.h; h[1] = gstep2.h;
    c[0] = gstep1.c; c[1] = gstep2.c;
  }
  return {ans, lp};
}

// Dialogs on the model's own answers (DESIGN §17): for r = 0 .. R-1, the encoder forward in eval mode on the batch with the
// engine-owned history (B, R, W), the search of round r's rows b*R + r only, its answers written into the outputs' rows
// b*R + r, and the history append of round r+1.  Everything is enqueued on the main stream; the batch's questions and
// image are staged once and the host waits only for the final copies.  `search(r)` enqueues round r's search and says where
// its answers are (DialogAnswers).
void Engine::gen_dialog(const vd_batch* b, int W, int max_ans_len, const std::function<DialogAnswers(int)>& search,
                        int32_t* hist_host) {
  // the decoder is the caller's to check: the gen searches, or the disc answer-pool retrieval
  VD_REQUIRE(cfg.useHist, VD_E_STATE, "dialogs on the model's own answers need a history encoder");
  VD_REQUIRE(b != nullptr && b->B > 0 && b->Tq > 0 && b->Th > 0, VD_E_SHAPE, "batch with B, Tq and Th > 0");
  VD_REQUIRE(W >= b->Th && max_ans_len >= 1, VD_E_BADARG, "hist_width >= the batch's Th, max_ans_len >= 1");
  VD_CUDA_CHECK(cudaSetDevice(cfg.gpuid));
  cx.stream = main_stream;
  const int saved_training = training;
  training = 0;
  try {
    stage_batch(b);
    wait_img();                                      // the rounds' batch aliases the staged image
    const int R = cfg.R, B = db.B;
    const int64_t N = db.N;
    int32_t* hist = (int32_t*)dialog_hist.ensure((size_t)N * W * sizeof(int32_t));
    hist_append(cx, hist, B, R, W, -1, db.hist, db.Th, nullptr, 0, nullptr, 0, 0, 0, false);   // round 0 <- the caption row
    vd_batch rb = {};
    rb.B = B; rb.Tq = db.Tq; rb.Th = W; rb.ques_fwd = db.ques; rb.hist = hist; rb.img_feat = db.img; rb.on_device = 1;
    rb.img_count = db.img_count;
    for (int r = 0; r < R; ++r) {
      encoder_forward(&rb);
      const DialogAnswers a = search(r);
      if (r + 1 < R)
        hist_append(cx, hist, B, R, W, r, rb.ques_fwd, rb.Tq, a.tokens, a.ld, a.len, a.max_tokens, a.end_token, max_ans_len,
                    cfg.fam_lf);             // the late-fusion encoders read concatenated history (opts.lua:59)
    }
    if (hist_host)
      VD_CUDA_CHECK(cudaMemcpyAsync(hist_host, hist, (size_t)N * W * sizeof(int32_t), cudaMemcpyDeviceToHost, cx.stream));
  } catch (...) { training = saved_training; throw; }
  training = saved_training;
}

// copies round r's n = B result rows (row pitch `bytes`) into rows b*R + r of an engine-owned (B*R, bytes) output
static void scatter_round(cudaStream_t s, void* dst, const void* src, size_t bytes, int R, int r, int64_t B) {
  VD_CUDA_CHECK(cudaMemcpy2DAsync((char*)dst + (size_t)r * bytes, (size_t)R * bytes, src, bytes, bytes, (size_t)B,
                                  cudaMemcpyDeviceToDevice, s));
}

void Engine::gen_dialog_beam_search(const vd_batch* b, int k, int G, float lam, int L, int start_token, int end_token, int W,
                                    int max_ans_len, int32_t* answer_host, int32_t* length_host, double* score_host,
                                    int32_t* hist_host, const NBestCfg& nc) {
  VD_REQUIRE(cfg.dec == DEC_GEN, VD_E_STATE, "gen_dialog_beam_search needs the gen decoder");
  check_beam_args(k, G, lam, L, nc);
  check_rules(L, end_token, true);
  VD_REQUIRE(answer_host && length_host && score_host, VD_E_BADARG, "null output pointer");
  VD_REQUIRE(b != nullptr && b->B > 0, VD_E_SHAPE, "batch B must be > 0");
  const int R = cfg.R;
  const int64_t Gn = (int64_t)G * nc.nbest;        // list entries per round
  const int64_t B = b->B, NG = B * R * Gn;
  int32_t* ans = (int32_t*)dialog_out[0].ensure((size_t)NG * L * sizeof(int32_t));
  int32_t* len = (int32_t*)dialog_out[1].ensure((size_t)NG * sizeof(int32_t));
  double* score = (double*)dialog_out[2].ensure((size_t)NG * sizeof(double));
  double* norm = nc.norm_host ? (double*)dialog_out[3].ensure((size_t)NG * sizeof(double)) : nullptr;
  VD_CUDA_CHECK(cudaSetDevice(cfg.gpuid));
  cx.stream = main_stream;
  const double* lp = length_penalty_table(nc.alpha, L);
  gen_dialog(b, W, max_ans_len, [&](int r) {
    const BeamResult res = beam_search_rows(B, R, r, k, G, lam, L, start_token, end_token, nc.nbest, lp);
    scatter_round(cx.stream, ans, res.gans, (size_t)Gn * L * sizeof(int32_t), R, r, B);
    scatter_round(cx.stream, len, res.glen, (size_t)Gn * sizeof(int32_t), R, r, B);
    scatter_round(cx.stream, score, res.gscore, (size_t)Gn * sizeof(double), R, r, B);
    if (norm) scatter_round(cx.stream, norm, res.gnorm, (size_t)Gn * sizeof(double), R, r, B);
    // the pick's tokens between <START> and the hypothesis' <END>
    return DialogAnswers{res.ans + 1, L, res.len, 0, end_token};
  }, hist_host);
  VD_CUDA_CHECK(cudaMemcpyAsync(answer_host, ans, (size_t)NG * L * sizeof(int32_t), cudaMemcpyDeviceToHost, cx.stream));
  VD_CUDA_CHECK(cudaMemcpyAsync(length_host, len, (size_t)NG * sizeof(int32_t), cudaMemcpyDeviceToHost, cx.stream));
  VD_CUDA_CHECK(cudaMemcpyAsync(score_host, score, (size_t)NG * sizeof(double), cudaMemcpyDeviceToHost, cx.stream));
  if (norm) VD_CUDA_CHECK(cudaMemcpyAsync(nc.norm_host, norm, (size_t)NG * sizeof(double), cudaMemcpyDeviceToHost, cx.stream));
  VD_CUDA_CHECK(cudaStreamSynchronize(cx.stream));
}

void Engine::gen_dialog_sample(const vd_batch* b, int L, int start_token, int end_token, float temperature, uint64_t seed,
                               int64_t row_offset, int W, int max_ans_len, int32_t* answer_host, float* logp_host,
                               int32_t* hist_host, const TruncCfg& tr) {
  VD_REQUIRE(cfg.dec == DEC_GEN, VD_E_STATE, "gen_dialog_sample needs the gen decoder");
  check_sample_args(L, start_token, temperature, row_offset, tr);
  VD_REQUIRE(end_token >= 1 && end_token <= cfg.V, VD_E_BADARG, "end_token in [1, V]");
  check_rules(L, end_token, false);
  VD_REQUIRE(answer_host, VD_E_BADARG, "null answer pointer");
  VD_REQUIRE(b != nullptr && b->B > 0, VD_E_SHAPE, "batch B must be > 0");
  const int R = cfg.R;
  const int64_t B = b->B, N = B * R;
  int32_t* ans = (int32_t*)dialog_out[0].ensure((size_t)N * (L + 1) * sizeof(int32_t));
  float* lp = (float*)dialog_out[3].ensure((size_t)N * L * sizeof(float));
  gen_dialog(b, W, max_ans_len, [&](int r) {
    const SampleResult res = sample_rows(B, R, r, L, start_token, temperature, seed, row_offset, -1, 0, nullptr, tr, end_token);
    scatter_round(cx.stream, ans, res.ans, (size_t)(L + 1) * sizeof(int32_t), R, r, B);
    scatter_round(cx.stream, lp, res.logp, (size_t)L * sizeof(float), R, r, B);
    // the samples before the first <END>
    return DialogAnswers{res.ans + 1, L + 1, nullptr, L, end_token};
  }, hist_host);
  VD_CUDA_CHECK(cudaMemcpyAsync(answer_host, ans, (size_t)N * (L + 1) * sizeof(int32_t), cudaMemcpyDeviceToHost, cx.stream));
  if (logp_host)
    VD_CUDA_CHECK(cudaMemcpyAsync(logp_host, lp, (size_t)N * L * sizeof(float), cudaMemcpyDeviceToHost, cx.stream));
  VD_CUDA_CHECK(cudaStreamSynchronize(cx.stream));
}

// ---- answer pool (DESIGN §18) ------------------------------------------------------------------------------------------
// Rows per option-LSTM run of the pool encoding.  Chunks are balanced (m split into equal parts of at most this many rows),
// so that at any m above 1 024 every chunk has at least 1 024 rows: the fp16 route of VD_MATH_F16 (lstm16_shape_ok) then runs
// for all of them, as it does for a batch's 100-option rows.
constexpr int64_t kPoolChunkRows = 16384;

void Engine::answer_pool_encode(const int32_t* tokens_host, int64_t m, int w) {
  VD_REQUIRE(cfg.dec == DEC_DISC, VD_E_STATE, "the answer pool is the disc decoder's (a gen engine has no option LSTM)");
  VD_REQUIRE(tokens_host && m >= 1 && m <= INT32_MAX && w >= 1, VD_E_BADARG, "answer pool: tokens, 1 <= m < 2^31, width >= 1");
  for (int64_t i = 0; i < m * w; ++i)
    VD_REQUIRE(tokens_host[i] >= 0 && tokens_host[i] <= cfg.V, VD_E_BADARG, "answer pool: a token outside [0, vocabSize]");
  VD_CUDA_CHECK(cudaSetDevice(cfg.gpuid));
  cx.stream = main_stream;
  join_options_backward();
  if (opt_fwd_pending) { VD_CUDA_CHECK(cudaStreamSynchronize(opt_stream)); opt_fwd_pending = false; }
  pool_valid = false;
  const int H = cfg.H, E = cfg.E;
  int32_t* tok = (int32_t*)pool_tok.ensure((size_t)m * w * sizeof(int32_t));
  float* emb = (float*)pool_emb.ensure((size_t)m * H * sizeof(float));
  VD_CUDA_CHECK(cudaMemcpyAsync(tok, tokens_host, (size_t)m * w * sizeof(int32_t), cudaMemcpyHostToDevice, cx.stream));
  refresh_shadows();
  const int64_t nchunks = (m + kPoolChunkRows - 1) / kPoolChunkRows, chunk = (m + nchunks - 1) / nchunks;
  const Arena::Mark mk = arena.mark();           // the last forward's activations stay as they are
  {
    LaunchCtx::Scope sc(&cx, "pool_encode", 2.0 * m * w * 4.0 * H * H, 4.0 * m * w + 4.0 * m * H);
    for (int64_t off = 0; off < m; off += chunk) {
      const int64_t n = std::min(chunk, m - off);
      int32_t* ids = arena.get<int32_t>(n * w);
      transpose_ids(cx, tok + off * w, ids, n, w);
      LstmRun r = make_run(w, n, E, H, seg("opt.lstm.weight"), nullptr, ids, nullptr);   // disc.lua:4-5: no maskzero
      lstm_forward(r, false);
      VD_CUDA_CHECK(cudaMemcpyAsync(emb + off * H, r.h_last(), (size_t)n * H * sizeof(float), cudaMemcpyDeviceToDevice, cx.stream));
      arena.rewind(mk);
    }
  }
  VD_CUDA_CHECK(cudaStreamSynchronize(cx.stream));
  pool_m = m; pool_w = w; pool_valid = true;
}

void Engine::pool_topk(const float* Q, int64_t ldq, int64_t rows, const float* E, int64_t m, int H, int k, float* topv,
                       int32_t* topi) {
  VD_REQUIRE(Q && E && topv && topi && rows >= 1 && m >= 1 && m <= INT32_MAX && H >= 1 && ldq >= H, VD_E_BADARG,
             "pool_topk: operands / shape");
  VD_REQUIRE(k >= 1 && k <= 32 && k <= m, VD_E_BADARG, "pool_topk: k in [1, min(32, m)]");
  const bool tc = tcmode() && pool_tc_ok(H, Q, ldq, E);
  PoolTcGeom g;
  const int slots = tc ? (g = pool_topk_tc_geom(cx, rows, m)).slots : pool_topk_simt_slots(cx, rows, m);
  const int64_t n = rows * slots * (int64_t)k;
  char* s = (char*)pool_scratch.ensure((size_t)n * 8);
  float* pv = (float*)s;
  int32_t* pi = (int32_t*)(s + n * 4);
  {
    LaunchCtx::Scope sc(&cx, tc ? "pool_topk" : "pool_topk_simt", 2.0 * rows * m * H,
                        4.0 * ((double)rows * H + (double)m * H) + 8.0 * n);
    if (tc) pool_topk_tc(cx, g, Q, ldq, rows, E, m, H, k, pv, pi);
    else pool_topk_simt(cx, slots, Q, ldq, rows, E, m, H, k, pv, pi);
  }
  LaunchCtx::Scope sc(&cx, "pool_topk_rows", 0.0, 8.0 * n + 8.0 * rows * k);
  pool_topk_merge(cx, pv, pi, rows, slots, k, tc ? g.num_n : 0, tc ? g.grid : 0, topv, topi);
}

void Engine::check_pool(int k) const {
  VD_REQUIRE(cfg.dec == DEC_DISC, VD_E_STATE, "answer-pool retrieval needs the disc decoder");
  VD_REQUIRE(pool_valid, VD_E_STATE, "no answer pool for the current weights and math mode: call vd_answer_pool_encode");
  VD_REQUIRE(k >= 1 && k <= 32 && k <= pool_m, VD_E_BADARG, "k in [1, min(32, pool rows)]");
}

// the batch as the encoder reads it: the retrieval never runs the batch's option LSTM (encoder_forward would start it)
static vd_batch encoder_only(const vd_batch* b) {
  vd_batch e = *b;
  e.To = 0; e.Ta = 0;
  e.options = e.answer_ind = e.answer_in = e.answer_out = e.option_in = e.option_out = nullptr;
  return e;
}

void Engine::answer_pool_retrieve(const vd_batch* b, int k, int32_t* index_host, float* score_host) {
  check_pool(k);
  VD_REQUIRE(b != nullptr && index_host && score_host, VD_E_BADARG, "null batch or output pointer");
  const vd_batch eb = encoder_only(b);
  const int saved_training = training;
  training = 0;
  try {
    encoder_forward(&eb);
    const int64_t N = db.N;
    float* tv = arena.get<float>(N * k);
    int32_t* ti = arena.get<int32_t>(N * k);
    pool_topk(encOut, cfg.H, N, (const float*)pool_emb.p, pool_m, cfg.H, k, tv, ti);
    VD_CUDA_CHECK(cudaMemcpyAsync(index_host, ti, (size_t)N * k * sizeof(int32_t), cudaMemcpyDeviceToHost, cx.stream));
    VD_CUDA_CHECK(cudaMemcpyAsync(score_host, tv, (size_t)N * k * sizeof(float), cudaMemcpyDeviceToHost, cx.stream));
    VD_CUDA_CHECK(cudaStreamSynchronize(cx.stream));
  } catch (...) { training = saved_training; throw; }
  training = saved_training;
}

// gen_dialog with the retrieval as the round's search: round r's rows of encOut (b*R + r, pitch R*H) against the pool, the
// top-1 pool row's tokens appended as the answer (its zero pads are not words; <END> = vocabSize ends it, as it ends a
// sampled answer)
void Engine::answer_pool_dialog(const vd_batch* b, int k, int W, int max_ans_len, int32_t* index_host, float* score_host,
                                int32_t* hist_host) {
  check_pool(k);
  VD_REQUIRE(index_host && score_host, VD_E_BADARG, "null output pointer");
  VD_REQUIRE(b != nullptr && b->B > 0, VD_E_SHAPE, "batch B must be > 0");
  const int R = cfg.R, H = cfg.H;
  const int64_t B = b->B, N = B * R;
  int32_t* idx = (int32_t*)dialog_out[0].ensure((size_t)N * k * sizeof(int32_t));
  int32_t* words = (int32_t*)dialog_out[1].ensure((size_t)B * pool_w * sizeof(int32_t));
  float* score = (float*)dialog_out[3].ensure((size_t)N * k * sizeof(float));
  const vd_batch eb = encoder_only(b);
  gen_dialog(&eb, W, max_ans_len, [&](int r) {
    float* tv = arena.get<float>(B * k);
    int32_t* ti = arena.get<int32_t>(B * k);
    pool_topk(encOut + (int64_t)r * H, (int64_t)R * H, B, (const float*)pool_emb.p, pool_m, H, k, tv, ti);
    scatter_round(cx.stream, idx, ti, (size_t)k * sizeof(int32_t), R, r, B);
    scatter_round(cx.stream, score, tv, (size_t)k * sizeof(float), R, r, B);
    gather_pool_rows(cx, (const int32_t*)pool_tok.p, pool_w, ti, k, B, words);
    return DialogAnswers{words, pool_w, nullptr, pool_w, cfg.V};
  }, hist_host);
  VD_CUDA_CHECK(cudaMemcpyAsync(index_host, idx, (size_t)N * k * sizeof(int32_t), cudaMemcpyDeviceToHost, cx.stream));
  VD_CUDA_CHECK(cudaMemcpyAsync(score_host, score, (size_t)N * k * sizeof(float), cudaMemcpyDeviceToHost, cx.stream));
  VD_CUDA_CHECK(cudaStreamSynchronize(cx.stream));
}

// ---- dialog sessions (DESIGN §19, §20) ----------------------------------------------------------------------------------
// A pool of C slots, each free (round -1) or one conversation at its own round.  Its state is allocated here, once, and
// indexed by slot; open changes nothing on the device.
void Engine::dialog_open(int C, int Tq, int W, int max_ans_len) {
  VD_REQUIRE(C >= 1 && Tq >= 1, VD_E_SHAPE, "a dialog pool with capacity and question width >= 1");
  // hist_append (as vd_gen_dialog_*'s loop calls it) needs a row to hold the caption row and a whole question row
  if (cfg.useHist) VD_REQUIRE(W >= Tq && max_ans_len >= 1, VD_E_BADARG, "hist_width >= the question width, max_ans_len >= 1");
  dses.open = dses.valid = false;
  dses.encOut = nullptr; dses.last_n = 0;
  VD_CUDA_CHECK(cudaSetDevice(cfg.gpuid));
  const int R = cfg.R, H = cfg.H;
  if (!cfg.useHist) W = 0;
  dses.img_cols = cfg.san ? (int64_t)cfg.P * H : cfg.img_in_q ? cfg.IE : cfg.useIm ? cfg.F : 0;
  if (cfg.useHist) {
    dses.hist.ensure((size_t)C * R * W * sizeof(int32_t));
    if (cfg.fam_mn || cfg.hre_att) dses.facts.ensure((size_t)C * R * H * sizeof(float));   // the attention's facts
    if (cfg.hre_att) dses.shc.ensure((size_t)C * R * sizeof(float));
    if (cfg.fam_hre)
      for (auto& g : dses.state) g.ensure((size_t)C * H * sizeof(float));
  }
  if (cfg.rnn_layers)
    for (auto& g : dses.rnn) g.ensure((size_t)C * H * sizeof(float));
  dses.ques.ensure((size_t)C * R * Tq * sizeof(int32_t));
  if (dses.img_cols) dses.img.ensure((size_t)C * dses.img_cols * sizeof(float));
  dses.enc.ensure((size_t)C * H * sizeof(float));
  dses.C = C; dses.Tq = Tq; dses.W = W; dses.max_ans_len = max_ans_len;
  dses.round.assign(C, -1);
  dses.draw_base.assign(C, 0);
  dses.count.assign(cfg.regions > 0 ? C : 0, cfg.P);
  dses.open = dses.valid = true;
}

// b's B dialogs (its image rows and round-0 history row; its questions, answers and options are not read) into the lowest
// free slots.  Their image products, which every round repeats, are computed here once, with the weights of this call.
void Engine::dialog_join(const vd_batch* b, const int64_t* draw_base, int32_t* slots_host) {
  VD_REQUIRE(dses.open, VD_E_STATE, "no dialog session: call vd_dialog_open");
  VD_REQUIRE(dses.valid, VD_E_STATE, "the weights or the math mode changed since the session was opened");
  VD_REQUIRE(b != nullptr && b->B > 0 && b->Tq > 0, VD_E_SHAPE, "join batch with B, Tq > 0");
  VD_REQUIRE(slots_host != nullptr, VD_E_BADARG, "null slot output");
  if (cfg.useHist) {
    VD_REQUIRE(b->hist && b->Th > 0, VD_E_SHAPE, "a history encoder's join needs the batch's round-0 history row");
    VD_REQUIRE(dses.W >= b->Th, VD_E_BADARG, "hist_width >= the batch's Th");
  }
  const int B = b->B;
  if (draw_base)
    for (int i = 0; i < B; ++i) VD_REQUIRE(draw_base[i] >= 0, VD_E_BADARG, "draw_base >= 0");
  std::vector<int32_t> slots;
  for (int s = 0; s < dses.C && (int)slots.size() < B; ++s)
    if (dses.round[s] < 0) slots.push_back(s);
  VD_REQUIRE((int)slots.size() == B, VD_E_STATE, "the pool has fewer free slots than dialogs to join");
  const vd_batch eb = encoder_only(b);
  dialog_join_images(&eb, slots.data());
  VD_CUDA_CHECK(cudaStreamSynchronize(cx.stream));
  const std::vector<int32_t> counts = batch_counts_host(b);
  for (int i = 0; i < B; ++i) {
    if (!counts.empty()) dses.count[slots[i]] = counts[i];
    dses.round[slots[i]] = 0;
    dses.draw_base[slots[i]] = draw_base ? draw_base[i] : 0;
    slots_host[i] = slots[i];
  }
}

std::vector<int32_t> Engine::batch_counts_host(const vd_batch* b) {
  std::vector<int32_t> c;
  if (cfg.regions <= 0) return c;
  c.assign(b->B, cfg.P);
  if (b->img_count && b->on_device) {
    VD_CUDA_CHECK(cudaStreamSynchronize(main_stream));   // a corpus batch's counts are gathered on the main stream
    VD_CUDA_CHECK(cudaMemcpy(c.data(), b->img_count, (size_t)b->B * sizeof(int32_t), cudaMemcpyDeviceToHost));
  }
  else if (b->img_count)
    std::copy_n(b->img_count, b->B, c.data());
  return c;
}

const int32_t* Engine::dialog_join_images(const vd_batch* b, const int32_t* slots) {
  const int B = b->B;
  quiesce();
  stage_batch(b);
  refresh_shadows();
  wait_img();
  int32_t* sd = arena.get<int32_t>(B);
  VD_CUDA_CHECK(cudaMemcpyAsync(sd, slots, (size_t)B * sizeof(int32_t), cudaMemcpyHostToDevice, cx.stream));
  if (cfg.useHist)                   // round 0 <- the caption row
    hist_append(cx, (int32_t*)dses.hist.p, B, cfg.R, dses.W, -1, db.hist, db.Th, nullptr, 0, nullptr, 0, 0, 0, false, sd);
  float* img = (float*)dses.img.p;
  if (cfg.san) {
    float* t = arena.get<float>((int64_t)B * dses.img_cols);
    san_image(db.img, B, t);
    scatter_rows(cx, img, t, sd, B, dses.img_cols);
  } else if (cfg.img_in_q) {         // eval mode: hrea's Dropout before img.embed is the identity
    float* e = arena.get<float>((int64_t)B * cfg.IE);
    linear_fwd(seg("img.embed.weight"), db.img, B, e, 0);
    scatter_rows(cx, img, e, sd, B, cfg.IE);
  } else if (cfg.useIm) {
    scatter_rows(cx, img, db.img, sd, B, cfg.F);
  }
  release_img();
  return sd;
}

// b's dialogs resumed in slots[i] at rounds[i] (DESIGN §21).  A conversation's cached state at round r depends only on its
// caption, image and rounds 0..r-1 (§17's causality), so it comes from one eval-mode pass over the P = sum r_i rows
// (slot s_i, round j < r_i).  The rows are packed time-major by round over the dialogs sorted by r descending: round j's
// rows are then a prefix block of the dialogs still going, so one dialog-LSTM step per round runs on a contiguous prefix
// and continues the previous step's rows.
void Engine::dialog_join_rounds(const vd_batch* b, const int32_t* rounds, const int32_t* answers, int Ta, const int64_t* draw_base,
                                const int32_t* slots) {
  VD_REQUIRE(dses.open, VD_E_STATE, "no dialog session: call vd_dialog_open");
  VD_REQUIRE(dses.valid, VD_E_STATE, "the weights or the math mode changed since the session was opened");
  VD_REQUIRE(b != nullptr && b->B > 0 && b->Tq > 0 && b->ques_fwd, VD_E_SHAPE, "resume batch with B, Tq > 0 and its questions");
  VD_REQUIRE(b->Tq <= dses.Tq, VD_E_SHAPE, "the batch's question width is above the session's");
  VD_REQUIRE(rounds != nullptr && slots != nullptr, VD_E_BADARG, "null rounds or slots");
  VD_REQUIRE(Ta >= 1, VD_E_BADARG, "answer width Ta >= 1");
  if (cfg.useHist) {
    VD_REQUIRE(b->hist && b->Th > 0, VD_E_SHAPE, "a history encoder's join needs the batch's round-0 history row");
    VD_REQUIRE(dses.W >= b->Th, VD_E_BADARG, "hist_width >= the batch's Th");
    VD_REQUIRE(answers != nullptr, VD_E_BADARG, "a history encoder's resume needs the answers");
  }
  const int B = b->B, R = cfg.R, H = cfg.H, Tq = b->Tq, Tw = dses.Tq, W = dses.W, V = cfg.V;
  std::vector<char> seen(dses.C, 0);
  for (int i = 0; i < B; ++i) {
    VD_REQUIRE(slots[i] >= 0 && slots[i] < dses.C, VD_E_BADARG, "a slot id outside [0, capacity)");
    VD_REQUIRE(!seen[slots[i]], VD_E_BADARG, "a slot named twice");
    seen[slots[i]] = 1;
    VD_REQUIRE(rounds[i] >= 0 && rounds[i] < R, VD_E_BADARG, "a round outside [0, maxQuesCount - 1]");
    if (draw_base) VD_REQUIRE(draw_base[i] >= 0, VD_E_BADARG, "draw_base >= 0");
  }
  std::vector<int32_t> ques((size_t)B * R * Tq);       // checked and packed on the host
  VD_CUDA_CHECK(cudaSetDevice(cfg.gpuid));
  if (b->on_device)
    VD_CUDA_CHECK(cudaMemcpy(ques.data(), b->ques_fwd, ques.size() * sizeof(int32_t), cudaMemcpyDeviceToHost));
  else
    std::copy_n(b->ques_fwd, ques.size(), ques.data());
  for (int i = 0; i < B; ++i)
    for (int j = 0; j < rounds[i]; ++j) {
      for (int t = 0; t < Tq; ++t) {
        const int32_t v = ques[((size_t)i * R + j) * Tq + t];
        VD_REQUIRE(v >= 0 && v <= V, VD_E_BADARG, "a question token outside [0, vocabSize]");
      }
      if (cfg.useHist)
        for (int t = 0; t < Ta; ++t) {
          const int32_t v = answers[((size_t)i * R + j) * Ta + t];
          VD_REQUIRE(v >= 0 && v <= V, VD_E_BADARG, "an answer token outside [0, vocabSize]");
        }
    }
  for (int i = 0; i < B; ++i) VD_REQUIRE(dses.round[slots[i]] < 0, VD_E_STATE, "an occupied slot");

  // sorted dialog i is batch row order[i]; round j has cnt[j] rows, from packed row row0[j] on
  std::vector<int> order(B);
  for (int i = 0; i < B; ++i) order[i] = i;
  std::stable_sort(order.begin(), order.end(), [&](int x, int y) { return rounds[x] > rounds[y]; });
  const int rmax = rounds[order[0]];
  std::vector<int32_t> cnt(R, 0), row0(R, 0);
  for (int i = 0; i < B; ++i)
    for (int j = 0; j < rounds[i]; ++j) ++cnt[j];
  for (int j = 1; j < R; ++j) row0[j] = row0[j - 1] + cnt[j - 1];
  const int64_t P = row0[R - 1] + cnt[R - 1];
  // upload: per packed row slot, round and question (right-aligned into the session's width); per sorted dialog slot and
  // round; row0; per sorted dialog its answers
  const int64_t o_round = P, o_q = 2 * P, o_sd = o_q + P * Tw, o_sr = o_sd + B, o_row0 = o_sr + B, o_ans = o_row0 + R;
  std::vector<int32_t> up((size_t)(o_ans + (cfg.useHist ? (int64_t)B * R * Ta : 0)), 0);
  for (int i = 0; i < B; ++i) {
    const int d = order[i];
    up[o_sd + i] = slots[d];
    up[o_sr + i] = rounds[d];
    for (int j = 0; j < rounds[d]; ++j) {
      const int64_t p = row0[j] + i;
      up[p] = slots[d];
      up[o_round + p] = j;
      std::copy_n(&ques[((size_t)d * R + j) * Tq], Tq, &up[o_q + p * Tw + Tw - Tq]);
    }
    if (cfg.useHist) std::copy_n(answers + (size_t)d * R * Ta, (size_t)R * Ta, &up[o_ans + (int64_t)i * R * Ta]);
  }
  std::copy(row0.begin(), row0.end(), &up[o_row0]);

  const int saved_training = training;
  training = 0;
  try {
    const vd_batch eb = encoder_only(b);
    dialog_join_images(&eb, slots);
    int32_t* u = arena.get<int32_t>((int64_t)up.size());
    VD_CUDA_CHECK(cudaMemcpyAsync(u, up.data(), up.size() * sizeof(int32_t), cudaMemcpyHostToDevice, cx.stream));
    const int32_t *slot_rows = u, *round_rows = u + o_round;
    if (cfg.useHist)                 // rows 1..r_i by §17's rule, before the gather reads them
      hist_prefill(cx, (int32_t*)dses.hist.p, B, R, W, u + o_sd, u + o_sr, u + o_row0, u + o_q, Tw, u + o_ans, Ta, V,
                   dses.max_ans_len, cfg.fam_lf);
    if (P > 0) {
      // hre / hrea's dialog LSTM reads q; mn caches facts only; late fusion re-reads the whole row at each ask
      const bool need_h = cfg.useHist && !cfg.fam_lf, need_q = cfg.fam_hre;
      DialogGather g;
      g.n = P; g.R = R; g.slot = slot_rows; g.round = round_rows;
      g.q = u + o_q; g.Tq = Tw; g.ques = (int32_t*)dses.ques.p; g.ids_q = ids_q = arena.get<int32_t>(P * Tw);
      ids_h = nullptr;
      if (need_h) { g.hist = (const int32_t*)dses.hist.p; g.W = W; g.ids_h = ids_h = arena.get<int32_t>(P * W); }
      float* img = nullptr;
      if (need_q && cfg.img_in_q) {
        g.img = (const float*)dses.img.p; g.img_cols = dses.img_cols; g.img_out = img = arena.get<float>(P * dses.img_cols);
      }
      {
        const double moved = 8.0 * P * (need_q && cfg.img_in_q ? dses.img_cols : 0) + 4.0 * P * (3 * Tw + (need_h ? W : 0));
        LaunchCtx::Scope sc(&cx, "dialog_gather", 0.0, moved);
        dialog_gather(cx, g);
      }
      if (need_h) {
        encoder_lstms(P, Tw, W, img, need_q);
        const float* h3 = hist2.h_last();
        float* facts = (float*)dses.facts.p;
        const int64_t fpitch = (int64_t)R * H;
        if (cfg.fam_mn) {
          dialog_cache_write(cx, facts, nullptr, h3, nullptr, P, R, H, 0, slot_rows, round_rows);
        } else {
          const float* q3 = ques2.h_last();
          float* j = arena.get<float>(P * 2 * H);
          if (cfg.hre_att) {         // every row's fact and score are cached before any attention reads them
            sq = arena.get<float>(P); sh = arena.get<float>(P);
            int sq_w = seg("att.q.weight"), sh_w = seg("att.h.weight");
            rowdot_fwd(cx, sq, q3, Wp(sq_w), Wp(sq_w + 1), P, H);
            rowdot_fwd(cx, sh, h3, Wp(sh_w), Wp(sh_w + 1), P, H);
            dialog_cache_write(cx, facts, (float*)dses.shc.p, h3, sh, P, R, H, 0, slot_rows, round_rows);
            hre_join_fwd(q3, facts, sq, (const float*)dses.shc.p, fpitch, (int)P, 0, 1, j, slot_rows, round_rows);
          } else {
            hre_join_fwd(q3, h3, nullptr, nullptr, fpitch, (int)P, 0, 1, j);
          }
          // round j's step continues the first cnt[j] rows of step j-1 (step 0 without state, as a full forward's first
          // step); each step's (h, c) go to its rows' slots, so a slot keeps the state of its last round r_i - 1
          float* out = arena.get<float>(P * H);
          const float *hp = nullptr, *cp = nullptr;
          for (int t = 0; t < rmax; ++t) {
            hre_dialog_fwd(j + (int64_t)row0[t] * 2 * H, cnt[t], 1, hp, cp, out + (int64_t)row0[t] * H);
            hp = dialog.h_last(); cp = dialog.c_last();
            dialog_cache_write(cx, nullptr, nullptr, nullptr, nullptr, cnt[t], R, H, 0, slot_rows + row0[t], nullptr,
                               (float*)dses.state[0].p, (float*)dses.state[1].p, hp, cp);
          }
        }
      }
    }
    VD_CUDA_CHECK(cudaStreamSynchronize(cx.stream));
  } catch (...) { training = saved_training; throw; }
  training = saved_training;
  const std::vector<int32_t> counts = batch_counts_host(b);
  for (int i = 0; i < B; ++i) {
    if (!counts.empty()) dses.count[slots[i]] = counts[i];
    dses.round[slots[i]] = rounds[i];
    dses.draw_base[slots[i]] = draw_base ? draw_base[i] : 0;
  }
}

void Engine::dialog_check_slots(const int32_t* slots, int64_t n) const {
  VD_REQUIRE(slots != nullptr && n >= 1, VD_E_BADARG, "at least one slot");
  std::vector<char> seen(dses.C, 0);
  for (int64_t i = 0; i < n; ++i) {
    VD_REQUIRE(slots[i] >= 0 && slots[i] < dses.C, VD_E_BADARG, "a slot id outside [0, capacity)");
    VD_REQUIRE(!seen[slots[i]], VD_E_BADARG, "a slot named twice");
    seen[slots[i]] = 1;
  }
  for (int64_t i = 0; i < n; ++i) VD_REQUIRE(dses.round[slots[i]] >= 0, VD_E_STATE, "a free slot");
}

// a freed slot's state is never read again; a later join overwrites what it reads
void Engine::dialog_leave(const int32_t* slots, int64_t n) {
  VD_REQUIRE(dses.open, VD_E_STATE, "no dialog session");
  dialog_check_slots(slots, n);
  for (int64_t i = 0; i < n; ++i) dses.round[slots[i]] = -1;
}

int Engine::dialog_lockstep_round() const {
  VD_REQUIRE(dses.open, VD_E_STATE, "no dialog session");
  const int r = dses.round[0];
  for (int s = 0; s < dses.C; ++s)
    VD_REQUIRE(dses.round[s] >= 0 && dses.round[s] == r, VD_E_STATE, "the session's slots are not all occupied at one round");
  return r;
}

std::vector<int32_t> Engine::dialog_all_slots() const {
  std::vector<int32_t> s(std::max(dses.C, 0));
  for (int i = 0; i < dses.C; ++i) s[i] = i;
  return s;
}

// the pool of b's B dialogs, all at round 0, sampling as vd_gen_dialog_sample's rows b*R + r
void Engine::dialog_begin(const vd_batch* b, int W, int max_ans_len) {
  VD_REQUIRE(b != nullptr && b->B > 0 && b->Tq > 0, VD_E_SHAPE, "session batch with B, Tq > 0");
  if (cfg.useHist) {
    VD_REQUIRE(b->hist && b->Th > 0, VD_E_SHAPE, "a history encoder's session needs the batch's round-0 history row");
    VD_REQUIRE(W >= b->Th && W >= b->Tq && max_ans_len >= 1, VD_E_BADARG,
               "hist_width >= the batch's Th and Tq, max_ans_len >= 1");
  }
  dialog_open(b->B, b->Tq, W, max_ans_len);
  std::vector<int64_t> base(b->B);
  for (int i = 0; i < b->B; ++i) base[i] = (int64_t)i * cfg.R;
  std::vector<int32_t> slots(b->B);
  try {
    dialog_join(b, base.data(), slots.data());
  } catch (...) { dses.open = dses.valid = false; throw; }
}

void Engine::dialog_end() { dses.open = dses.valid = false; dses.encOut = nullptr; dses.last_n = 0; }

void Engine::dialog_check_ask(const int32_t* slots, int64_t n, const int32_t* ques_host, int Tq) const {
  VD_REQUIRE(dses.open, VD_E_STATE, "no dialog session: call vd_dialog_open or vd_dialog_begin");
  VD_REQUIRE(dses.valid, VD_E_STATE, "the weights or the math mode changed since the session was opened");
  dialog_check_slots(slots, n);
  for (int64_t i = 0; i < n; ++i)
    VD_REQUIRE(dses.round[slots[i]] < cfg.R, VD_E_STATE, "a conversation that has had all maxQuesCount rounds");
  VD_REQUIRE(ques_host != nullptr, VD_E_BADARG, "null question rows");
  VD_REQUIRE(Tq >= 1 && Tq <= dses.Tq, VD_E_SHAPE, "question width in [1, the session's question width]");
  for (int64_t i = 0; i < n * Tq; ++i)
    VD_REQUIRE(ques_host[i] >= 0 && ques_host[i] <= cfg.V, VD_E_BADARG, "a question token outside [0, vocabSize]");
}

// The ask's rows in eval mode: row i is conversation slots[i] at its round r_i.  One upload of the rows, one gather launch
// (questions into the cache and time-major ids, history row r_i, the slot's image product and dialog-LSTM state), the
// question and history pairs over the n rows, then the family block with per-row attention over each slot's facts.  Leaves
// encOut = the (n, H) rows and ques1 / ques2 = this pass's runs, which forward_connect() reads; the last encoder_forward is
// no longer current.
Engine::AskRows Engine::dialog_encode(const int32_t* slots, int64_t n, const int32_t* ques_host, int Tq, int64_t row_offset) {
  quiesce();
  refresh_shadows();
  const int R = cfg.R, H = cfg.H, Tw = dses.Tq, W = dses.W;
  AskRows rows;
  rows.n = n;
  // slot, round, questions right-aligned into the session's width, then (region engines) the slot's region count
  const int64_t o_cnt = n * (2 + Tw);
  std::vector<int32_t> up((size_t)(o_cnt + (cfg.regions > 0 ? n : 0)), 0);
  std::vector<int64_t> draw(n);
  bool any_state = false;
  for (int64_t i = 0; i < n; ++i) {
    const int s = slots[i], r = dses.round[s];
    up[i] = s; up[n + i] = r;
    draw[i] = row_offset + dses.draw_base[s] + r;
    any_state |= r > 0;
    rows.any_next |= r + 1 < R;
    for (int t = 0; t < Tq; ++t) up[2 * n + i * Tw + Tw - Tq + t] = ques_host[i * Tq + t];
    if (cfg.regions > 0) up[o_cnt + i] = dses.count[s];
  }
  int64_t* draw_dev = arena.get<int64_t>(n);
  int32_t* up_dev = arena.get<int32_t>((int64_t)up.size());
  VD_CUDA_CHECK(cudaMemcpyAsync(draw_dev, draw.data(), draw.size() * sizeof(int64_t), cudaMemcpyHostToDevice, cx.stream));
  VD_CUDA_CHECK(cudaMemcpyAsync(up_dev, up.data(), up.size() * sizeof(int32_t), cudaMemcpyHostToDevice, cx.stream));
  rows.slot = up_dev; rows.round = up_dev + n; rows.draw = draw_dev;
  san_cnt = cfg.regions > 0 ? up_dev + o_cnt : nullptr;
  DialogGather g;
  g.n = n; g.R = R; g.slot = rows.slot; g.round = rows.round;
  g.q = up_dev + 2 * n; g.Tq = Tw; g.ques = (int32_t*)dses.ques.p; g.ids_q = ids_q = arena.get<int32_t>(n * Tw);
  ids_h = nullptr;
  if (cfg.useHist) { g.hist = (const int32_t*)dses.hist.p; g.W = W; g.ids_h = ids_h = arena.get<int32_t>(n * W); }
  float* img = nullptr;
  if (dses.img_cols) { g.img = (const float*)dses.img.p; g.img_cols = dses.img_cols; g.img_out = img = arena.get<float>(n * dses.img_cols); }
  if (cfg.fam_hre) {
    g.h = (const float*)dses.state[0].p; g.c = (const float*)dses.state[1].p; g.H = H;
    g.h_out = arena.get<float>(n * H); g.c_out = arena.get<float>(n * H);
  }
  {
    const double moved = 8.0 * n * (dses.img_cols + (cfg.fam_hre ? 2 * H : 0)) + 4.0 * n * (3 * Tw + W);
    LaunchCtx::Scope sc(&cx, "dialog_gather", 0.0, moved);
    dialog_gather(cx, g);
  }
  encoder_lstms(n, Tw, W, cfg.img_in_q ? img : nullptr);
  if (cfg.rnn_layers) {                  // the question LSTMs' last state, forward_connect's source, kept for vd_dialog_rnn_state
    const float* src[4] = {ques1.h_last(), ques1.c_last(), ques2.h_last(), ques2.c_last()};
    for (int i = 0; i < 4; ++i)
      VD_CUDA_CHECK(cudaMemcpyAsync(dses.rnn[i].p, src[i], (size_t)n * H * sizeof(float), cudaMemcpyDeviceToDevice, cx.stream));
  }
  const float* q3 = ques2.h_last();
  const float* h3 = cfg.useHist ? hist2.h_last() : nullptr;
  float* out = (float*)dses.enc.p;
  float* facts = (float*)dses.facts.p;
  const int64_t fpitch = (int64_t)R * H;
  if (cfg.fam_lf) {
    lf_block_fwd(q3, img, img, h3, (int)n, 1, out);
  } else if (cfg.fam_hre) {
    float* j = arena.get<float>(n * 2 * H);
    if (cfg.hre_att) {                   // the row's own fact and score are cached before its attention reads them
      sq = arena.get<float>(n); sh = arena.get<float>(n);
      int sq_w = seg("att.q.weight"), sh_w = seg("att.h.weight");
      rowdot_fwd(cx, sq, q3, Wp(sq_w), Wp(sq_w + 1), n, H);
      rowdot_fwd(cx, sh, h3, Wp(sh_w), Wp(sh_w + 1), n, H);
      dialog_cache_write(cx, facts, (float*)dses.shc.p, h3, sh, n, R, H, 0, rows.slot, rows.round);
      hre_join_fwd(q3, facts, sq, (const float*)dses.shc.p, fpitch, (int)n, 0, 1, j, rows.slot, rows.round);
    } else {                             // [q | h]: the row's own fact, no cache
      hre_join_fwd(q3, h3, nullptr, nullptr, fpitch, (int)n, 0, 1, j);
    }
    // A row at round 0 continues the zero state the gather wrote; when no row has state, the step runs without one, as the
    // full forward's first step does.  Either way the new state goes back to the rows' slots.
    hre_dialog_fwd(j, (int)n, 1, any_state ? g.h_out : nullptr, any_state ? g.c_out : nullptr, out);
    dialog_cache_write(cx, nullptr, nullptr, nullptr, nullptr, n, R, H, 0, rows.slot, nullptr, (float*)dses.state[0].p,
                       (float*)dses.state[1].p, dialog.h_last(), dialog.c_last());
  } else {
    dialog_cache_write(cx, facts, nullptr, h3, nullptr, n, R, H, 0, rows.slot, rows.round);
    mn_family_fwd(q3, img, img, facts, fpitch, (int)n, 0, 1, out, rows.slot, rows.round);
  }
  encOut = out;
  dses.encOut = out;
  dses.last_n = n;
  conn_dh_l1 = conn_dc_l1 = conn_dc_l2 = nullptr;
  have_fwd = true;                       // for forward_connect(); run_ask drops it again
  return rows;
}

void Engine::dialog_finish(const AskRows& rows, const DialogAnswers& a) {
  if (cfg.useHist && rows.any_next)      // rows at round R-1 write nothing
    hist_append(cx, (int32_t*)dses.hist.p, rows.n, cfg.R, dses.W, 0, (const int32_t*)dses.ques.p, dses.Tq, a.tokens, a.ld, a.len,
                a.max_tokens, a.end_token, dses.max_ans_len, cfg.fam_lf, rows.slot, rows.round);
}

// runs one ask: the encoder pass, `answer(rows)` (which enqueues the answerer and its copies to the host and says where the
// answers are), the history append, one synchronisation; eval mode throughout.  The rows' rounds advance only when all of
// it succeeded.
template <typename F>
static void run_ask(Engine* e, const int32_t* slots, int64_t n, const int32_t* ques_host, int Tq, int64_t row_offset, F&& answer) {
  const int saved_training = e->training;
  e->training = 0;
  try {
    const Engine::AskRows rows = e->dialog_encode(slots, n, ques_host, Tq, row_offset);
    const Engine::DialogAnswers a = answer(rows);
    e->dialog_finish(rows, a);
    VD_CUDA_CHECK(cudaStreamSynchronize(e->cx.stream));
  } catch (...) { e->training = saved_training; e->have_fwd = false; throw; }
  e->training = saved_training;
  e->have_fwd = false;
  for (int64_t i = 0; i < n; ++i) e->dses.round[slots[i]] += 1;
}

void Engine::dialog_ask_beam(const int32_t* slots, int64_t n, const int32_t* ques_host, int Tq, int k, int G, float lam, int L,
                             int start_token, int end_token, int32_t* answer_host, int32_t* length_host, double* score_host,
                             const NBestCfg& nc) {
  VD_REQUIRE(cfg.dec == DEC_GEN, VD_E_STATE, "a beam-search ask needs the gen decoder");
  check_beam_args(k, G, lam, L, nc);
  check_rules(L, end_token, true);
  VD_REQUIRE(start_token >= 1 && start_token <= cfg.V && end_token >= 1 && end_token <= cfg.V, VD_E_BADARG,
             "start_token and end_token in [1, vocabSize]");
  VD_REQUIRE(answer_host && length_host && score_host, VD_E_BADARG, "null output pointer");
  dialog_check_ask(slots, n, ques_host, Tq);
  run_ask(this, slots, n, ques_host, Tq, 0, [&](const AskRows&) {
    const BeamResult res = beam_search_rows(n, 1, 0, k, G, lam, L, start_token, end_token, nc.nbest,
                                            length_penalty_table(nc.alpha, L));
    const size_t nG = (size_t)n * G * nc.nbest;
    VD_CUDA_CHECK(cudaMemcpyAsync(answer_host, res.gans, nG * L * sizeof(int32_t), cudaMemcpyDeviceToHost, cx.stream));
    VD_CUDA_CHECK(cudaMemcpyAsync(length_host, res.glen, nG * sizeof(int32_t), cudaMemcpyDeviceToHost, cx.stream));
    VD_CUDA_CHECK(cudaMemcpyAsync(score_host, res.gscore, nG * sizeof(double), cudaMemcpyDeviceToHost, cx.stream));
    if (nc.norm_host)
      VD_CUDA_CHECK(cudaMemcpyAsync(nc.norm_host, res.gnorm, nG * sizeof(double), cudaMemcpyDeviceToHost, cx.stream));
    return DialogAnswers{res.ans + 1, L, res.len, 0, end_token};
  });
}

void Engine::dialog_ask_sample(const int32_t* slots, int64_t n, const int32_t* ques_host, int Tq, int L, int start_token,
                               int end_token, float temperature, uint64_t seed, int64_t row_offset, int32_t* answer_host,
                               float* logp_host, const TruncCfg& tr) {
  VD_REQUIRE(cfg.dec == DEC_GEN, VD_E_STATE, "a sampling ask needs the gen decoder");
  check_sample_args(L, start_token, temperature, row_offset, tr);
  VD_REQUIRE(end_token >= 1 && end_token <= cfg.V, VD_E_BADARG, "end_token in [1, V]");
  check_rules(L, end_token, false);
  VD_REQUIRE(answer_host, VD_E_BADARG, "null answer pointer");
  dialog_check_ask(slots, n, ques_host, Tq);
  run_ask(this, slots, n, ques_host, Tq, row_offset, [&](const AskRows& rows) {
    // row i draws as global round row_offset + draw_base[slot] + its round (vd_dialog_begin: vd_gen_dialog_sample's rows)
    const SampleResult res = sample_rows(n, 1, 0, L, start_token, temperature, seed, 0, -1, 0, rows.draw, tr, end_token);
    VD_CUDA_CHECK(cudaMemcpyAsync(answer_host, res.ans, (size_t)n * (L + 1) * sizeof(int32_t), cudaMemcpyDeviceToHost, cx.stream));
    if (logp_host)
      VD_CUDA_CHECK(cudaMemcpyAsync(logp_host, res.logp, (size_t)n * L * sizeof(float), cudaMemcpyDeviceToHost, cx.stream));
    return DialogAnswers{res.ans + 1, L + 1, nullptr, L, end_token};
  });
}

void Engine::dialog_ask_pool(const int32_t* slots, int64_t n, const int32_t* ques_host, int Tq, int k, int32_t* index_host,
                             float* score_host) {
  check_pool(k);
  VD_REQUIRE(index_host && score_host, VD_E_BADARG, "null output pointer");
  dialog_check_ask(slots, n, ques_host, Tq);
  run_ask(this, slots, n, ques_host, Tq, 0, [&](const AskRows&) {
    float* tv = arena.get<float>(n * k);
    int32_t* ti = arena.get<int32_t>(n * k);
    pool_topk(encOut, cfg.H, n, (const float*)pool_emb.p, pool_m, cfg.H, k, tv, ti);
    int32_t* words = arena.get<int32_t>(n * pool_w);
    gather_pool_rows(cx, (const int32_t*)pool_tok.p, pool_w, ti, k, n, words);
    VD_CUDA_CHECK(cudaMemcpyAsync(index_host, ti, (size_t)n * k * sizeof(int32_t), cudaMemcpyDeviceToHost, cx.stream));
    VD_CUDA_CHECK(cudaMemcpyAsync(score_host, tv, (size_t)n * k * sizeof(float), cudaMemcpyDeviceToHost, cx.stream));
    return DialogAnswers{words, pool_w, nullptr, pool_w, cfg.V};
  });
}

// model.lua:96-99 + optim_updates.lua:62-91
void Engine::clamp_adam_step(float lr) {
  VD_CUDA_CHECK(cudaSetDevice(cfg.gpuid));
  pool_valid = false;                 // the pool's encoding belongs to the weights before this step
  dses.valid = false;                 // so do a dialog session's cached facts and image products
  join_options_backward();
  float gscale = 1.f;
  if (world > 1) {
    allreduce_grads();
    // disc: loss is a mean over the local N rows -> average over ranks; gen: a sum -> plain sum (SURVEY §8e)
    if (cfg.dec == DEC_DISC) gscale = 1.f / (float)world;
  }
  adam_t += 1;
  const double b1 = 0.9, b2 = 0.999;
  double bc1 = 1.0 - pow(b1, (double)adam_t), bc2 = 1.0 - pow(b2, (double)adam_t);
  float step = (float)((double)lr * sqrt(bc2) / bc1);
  clamp_adam(cx, W, dW, m, v, nparams, step, (float)b1, (float)b2, 1e-8f, gscale);
}

}  // namespace vd
