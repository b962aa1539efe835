// HBM-resident dialog corpus + on-device batch assembly (include/visdial_b200.h, "dataloader" section).
//
// Replaces, for one split, the tensor preparation of dataloader:initialize and the per-batch indexing:
//   utils.rightAlign                       /root/reference/utils.lua:6-45
//   dataloader:prepareDataset              dataloader.lua:143-156
//   dataloader:processAnswers              :159-199
//   dataloader:processHistory              :202-278
//   dataloader:processOptions              :281-321
//   image L2 norm + NCHW->NHWC permute     :59-73
//   region features and their counts       DESIGN §26 (no reference counterpart)
//   getTrainBatch / getTestBatch           :324-375
//   getIndexData / getIndexOption          :378-478
// Everything here is int32/fp32 HBM-bound gather work: one thread per output element (or 16 B vector), fully
// coalesced writes, reads coalesced along the token axis.  The reference builds each prepared tensor with a
// sequential per-dialog loop; the kernels below evaluate the closed form of those loops per element (the "break"
// of rightAlign, utils.lua:20-22, becomes a prefix test on the lengths).
#include "engine.h"
#include <algorithm>
#include <memory>

namespace vd {

// ------------------------------------------------------------------------------------------------
// one-time preparation kernels
// ------------------------------------------------------------------------------------------------
// utils.rightAlign on a (n,R,M) volume.  A round is copied only while every earlier round of the same dialog has a
// non-zero length (the loop `break`s at the first empty round, utils.lua:20-22).
__global__ void k_right_align(const int32_t* __restrict__ src, const int32_t* __restrict__ len, int32_t* __restrict__ dst,
                              int64_t total, int R, int M) {
  int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= total) return;
  int64_t row = e / M; int m = (int)(e - row * M);
  int64_t i = row / R; int r = (int)(row - i * R);
  bool alive = true;
  for (int k = 0; k <= r; ++k) alive = alive && len[i * R + k] != 0;
  int L = len[row];
  int pos = m - (M - L);
  dst[e] = (alive && pos >= 0) ? src[row * M + pos] : 0;
}

// history lengths, dataloader.lua:229-271 (one thread per dialog: the recurrence is 10 steps long)
__global__ void k_hist_len(const int32_t* __restrict__ cap_len, const int32_t* __restrict__ ques_len,
                           const int32_t* __restrict__ ans_len, int32_t* __restrict__ hist_len, int n, int R, int Lqa,
                           int concat) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int lenH = min(cap_len[i], Lqa);                                   // :238
  hist_len[(int64_t)i * R] = lenH;
  for (int r = 1; r < R; ++r) {
    int lq = ques_len[(int64_t)i * R + r - 1], la = ans_len[(int64_t)i * R + r - 1];
    lenH = concat ? lenH + lq + la + 1 : lq + la;                    // :255 / :266
    hist_len[(int64_t)i * R + r] = lenH;
  }
}

// processHistory + rightAlign fused: element (i, r, m) of the right-aligned history, from the raw arrays.
__global__ void k_build_hist(const int32_t* __restrict__ cap, const int32_t* __restrict__ ques,
                             const int32_t* __restrict__ ans, const int32_t* __restrict__ ques_len,
                             const int32_t* __restrict__ hist_len, int32_t* __restrict__ dst, int64_t total, int R, int W,
                             int Lc, int Lq, int La, int concat, int end_tok) {
  int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= total) return;
  int64_t row = e / W; int m = (int)(e - row * W);
  int64_t i = row / R; int r = (int)(row - i * R);
  const int32_t* hl = hist_len + i * R;
  bool alive = true;
  for (int k = 0; k <= r; ++k) alive = alive && hl[k] != 0;
  int L = hl[r];
  int pos = m - (W - L);
  int32_t v = 0;
  if (alive && pos >= 0) {
    if (r == 0 || (concat && pos < hl[0])) {
      v = cap[i * Lc + pos];                                         // :236-237 (first lenH caption tokens)
    } else if (!concat) {                                            // :257-266: previous round's Q then A
      int64_t pr = i * R + r - 1;
      int lq = ques_len[pr];
      v = pos < lq ? ques[pr * Lq + pos] : ans[pr * La + pos - lq];
    } else {                                                         // :243-255: caption <END> Q1 A1 <END> Q2 A2 ...
      int k = 1;
      while (k < r && pos >= hl[k]) ++k;                             // segment k covers [hl[k-1], hl[k])
      int64_t pr = i * R + k - 1;
      int off = pos - hl[k - 1];
      int lq = ques_len[pr];
      v = off == 0 ? end_tok : (off - 1 < lq ? ques[pr * Lq + off - 1] : ans[pr * La + off - 1 - lq]);
    }
  }
  dst[e] = v;
}

// <START> a.. / a.. <END> wrapping of left-aligned rows (processAnswers :159-199, processOptions :281-321).
// end_when_empty: answers always get <END> at length+1 (:193); options only when length > 0 (:303-310).
__global__ void k_wrap_start_end(const int32_t* __restrict__ src, const int32_t* __restrict__ len,
                                 int32_t* __restrict__ in, int32_t* __restrict__ out, int64_t total, int La, int start_tok,
                                 int end_tok, int end_when_empty) {
  int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= total) return;
  int64_t row = e / (La + 1); int t = (int)(e - row * (La + 1));
  int L = len[row];
  in[e] = t == 0 ? start_tok : (t <= L ? src[row * La + t - 1] : 0);
  out[e] = t < L ? src[row * La + t] : ((t == L && (L > 0 || end_when_empty)) ? end_tok : 0);
}

// max_k (opt_len[opt[i,r,k]] + 1): the per-(dialog, round) bound getIndexOption('gen') trims to (:443-444)
__global__ void k_opt_maxlen(const int32_t* __restrict__ opt, const int32_t* __restrict__ opt_len,
                             int32_t* __restrict__ out, int64_t rows, int K) {
  int64_t row = (int64_t)blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
  if (row >= rows) return;
  int lane = threadIdx.x & 31, mx = 0;
  for (int k = lane; k < K; k += 32) mx = max(mx, opt_len[opt[row * K + k] - 1] + 1);
  for (int o = 16; o; o >>= 1) mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if (lane == 0) out[row] = mx;
}

// fc7: x / sqrt(sum x^2) per row, in place (dataloader.lua:64-68 on a 2-D tensor)
__global__ void k_img_norm_rows(float* __restrict__ x, int F) {
  float* row = x + (int64_t)blockIdx.x * F;
  __shared__ float red[32];
  float s = 0.f;
  for (int j = threadIdx.x; j < F; j += blockDim.x) s += row[j] * row[j];
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    s = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (threadIdx.x == 0) red[0] = sqrtf(s);
  }
  __syncthreads();
  const float nm = red[0];
  for (int j = threadIdx.x; j < F; j += blockDim.x) row[j] = row[j] / nm;
}

// pool5: per (image, position) channel norm of an (nimg, C, P) chunk (sum over dim 2 of the 4-D tensor, :65)
__global__ void k_img_norm_pos(const float* __restrict__ x, float* __restrict__ nm, int C, int P) {
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const float* base = x + (int64_t)blockIdx.y * C * P + p;
  float s = 0.f;
  for (int c = 0; c < C; ++c) { float v = base[(int64_t)c * P]; s += v * v; }
  nm[(int64_t)blockIdx.y * P + p] = sqrtf(s);
}

// (nimg, C, P) -> (nimg, P, C) through a 32x33 shared tile, optionally divided by nm[img, p] (:66-72)
__global__ void k_img_nchw_to_nhwc(const float* __restrict__ src, const float* __restrict__ nm, float* __restrict__ dst,
                                   int C, int P) {
  __shared__ float tile[32][33];
  const int64_t img = blockIdx.z;
  const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    int c = c0 + j, p = p0 + threadIdx.x;
    tile[j][threadIdx.x] = (c < C && p < P) ? src[(img * C + c) * P + p] : 0.f;
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    int p = p0 + j, c = c0 + threadIdx.x;
    if (p < P && c < C) {
      float v = tile[threadIdx.x][j];
      if (nm) v = v / nm[img * P + p];
      dst[(img * P + p) * C + c] = v;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// per-batch assembly kernels
// ------------------------------------------------------------------------------------------------
// One launch gathers every integer tensor of the batch.  Job j copies, for each dialog b of the batch and each of its
// `rows` rows, T tokens starting at column `off` of a width-W source row; the source row is ind[b]*rows + r, or (when
// rowidx is set) rowidx[ind[b]*rows + r] - 1 — the option-list indirection of getIndexOption (:452-459).
struct GatherJob {
  const int32_t* src; const int32_t* rowidx; int32_t* dst;
  int rows, W, T, off, vec;      // vec = 1: W, T, off are in units of int4 (16 B)
  int64_t total;                 // B * rows * T output units
};
struct GatherJobs { GatherJob j[8]; int n; };

__global__ void __launch_bounds__(256) k_gather_tokens(const GatherJobs jobs, const int32_t* __restrict__ ind) {
  const GatherJob& jb = jobs.j[blockIdx.y];
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < jb.total; e += stride) {
    int64_t orow = e / jb.T; int t = (int)(e - orow * jb.T);
    int64_t b = orow / jb.rows; int r = (int)(orow - b * jb.rows);
    int64_t srow = (int64_t)ind[b] * jb.rows + r;
    if (jb.rowidx) srow = (int64_t)jb.rowidx[srow] - 1;
    if (jb.vec) reinterpret_cast<int4*>(jb.dst)[e] = reinterpret_cast<const int4*>(jb.src)[srow * jb.W + jb.off + t];
    else jb.dst[e] = jb.src[srow * jb.W + jb.off + t];
  }
}

// region features: every row at or past its image's count of a (nimg, P, C4 float4) volume <- 0, once, so that the gathered
// batches hold exact zeros there
__global__ void k_zero_pad_regions(float4* __restrict__ x, const int32_t* __restrict__ cnt, int64_t total4, int P, int64_t C4) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total4) return;
  const int64_t row = i / C4;
  if ((int)(row % P) >= cnt[row / P]) x[i] = make_float4(0.f, 0.f, 0.f, 0.f);
}

// img_feat[b] = img_fv[img_pos[ind[b]]] (:394-398); 4 independent 16 B loads in flight per thread.  Region corpora with
// counts: img_count[b] = counts[img_pos[ind[b]]] as well
__global__ void __launch_bounds__(256) k_gather_img(const float4* __restrict__ src, const int32_t* __restrict__ img_pos,
                                                    const int32_t* __restrict__ ind, float4* __restrict__ dst,
                                                    int64_t elems4, const int32_t* __restrict__ counts,
                                                    int32_t* __restrict__ count_out) {
  const int64_t b = blockIdx.y;
  if (counts && blockIdx.x == 0 && threadIdx.x == 0) count_out[b] = counts[img_pos[ind[b]]];
  const float4* s = src + (int64_t)img_pos[ind[b]] * elems4;
  float4* d = dst + b * elems4;
  int64_t base = (int64_t)blockIdx.x * blockDim.x * 4 + threadIdx.x;
  float4 v[4];
#pragma unroll
  for (int u = 0; u < 4; ++u) { int64_t j = base + (int64_t)u * blockDim.x; if (j < elems4) v[u] = s[j]; }
#pragma unroll
  for (int u = 0; u < 4; ++u) { int64_t j = base + (int64_t)u * blockDim.x; if (j < elems4) d[j] = v[u]; }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
struct Corpus {
  Engine* eng = nullptr;
  int gpuid = 0;
  int n = 0, R = 0, Lq = 0, La = 0, Lc = 0, K = 0, m = 0, Wh = 0, nimg = 0;
  int useHist = 0, concat = 0, useIm = 0, maxHistoryLen = 0, start_tok = 0, end_tok = 0;
  int64_t img_elems = 0;
  int regions = 0;               // P of a region corpus (imgAtt 2), else 0
  int32_t* img_count = nullptr;  // (nimg) region counts, null = every region present
  bool has_ans_index = false;
  // raw (device)
  int32_t *ques = nullptr, *ques_len = nullptr, *ans = nullptr, *ans_len = nullptr, *cap = nullptr, *cap_len = nullptr,
          *opt = nullptr, *opt_list = nullptr, *opt_len = nullptr, *ans_index = nullptr, *img_pos = nullptr;
  // prepared (device)
  int32_t *ques_fwd = nullptr, *hist = nullptr, *hist_len = nullptr, *ans_in = nullptr, *ans_out = nullptr,
          *opt_in = nullptr, *opt_out = nullptr, *opt_maxlen = nullptr;
  float* img_fv = nullptr;
  // host metadata: the lengths getIndexData / getIndexOption take maxima over (:380-381,:388-389,:401-402,:443-444)
  std::vector<int32_t> h_ques_len, h_hist_len, h_ans_len1, h_opt_maxlen;
  std::vector<void*> owned;
  // two alternating output sets
  struct OutSet { GrowBuf ques, hist, ans_in, ans_out, ans_ind, options, opt_in, opt_out, img, ind, cnt; } out[2];
  int32_t* h_ind[2] = {nullptr, nullptr}; int h_ind_cap[2] = {0, 0};
  cudaEvent_t ind_free[2] = {nullptr, nullptr};
  int cur = 0;
  int64_t last_bytes = 0; int last_launches = 0;

  template <typename T> T* dalloc(int64_t elems) {
    void* p = nullptr;
    VD_CUDA_CHECK(cudaMalloc(&p, std::max<int64_t>(elems, 1) * sizeof(T)));
    owned.push_back(p);
    return (T*)p;
  }
  int32_t* upload(const int32_t* h, int64_t elems) {
    int32_t* d = dalloc<int32_t>(elems);
    VD_CUDA_CHECK(cudaMemcpy(d, h, elems * 4, cudaMemcpyHostToDevice));
    return d;
  }
  ~Corpus() {
    cudaSetDevice(gpuid);
    for (void* p : owned) cudaFree(p);
    for (int s = 0; s < 2; ++s) {
      OutSet& o = out[s];
      GrowBuf* bs[] = {&o.ques, &o.hist, &o.ans_in, &o.ans_out, &o.ans_ind, &o.options, &o.opt_in, &o.opt_out, &o.img, &o.ind,
                       &o.cnt};
      for (GrowBuf* b : bs) b->release();
      if (h_ind[s]) cudaFreeHost(h_ind[s]);
      if (ind_free[s]) cudaEventDestroy(ind_free[s]);
    }
  }
};

static void check_lengths(const int32_t* len, int64_t cnt, int lo, int hi, const char* what) {
  for (int64_t i = 0; i < cnt; ++i)
    if (len[i] < lo || len[i] > hi) {
      char buf[256];
      snprintf(buf, sizeof(buf), "%s[%lld] = %d outside [%d, %d]", what, (long long)i, len[i], lo, hi);
      throw CudaError(VD_E_SHAPE, buf);
    }
}

Corpus* corpus_create(Engine* eng, const vd_corpus_desc* d) {
  VD_REQUIRE(d != nullptr, VD_E_BADARG, "corpus descriptor is null");
  VD_REQUIRE(d->numThreads > 0 && d->numRounds > 0 && d->maxQuesLen > 0 && d->maxAnsLen > 0, VD_E_SHAPE, "corpus sizes");
  VD_REQUIRE(d->ques && d->ques_len && d->ans && d->ans_len, VD_E_BADARG, "ques / ans arrays missing");
  VD_REQUIRE(d->opt && d->opt_list && d->opt_len && d->numOptions > 0 && d->numOptList > 0, VD_E_BADARG, "option arrays missing");
  VD_REQUIRE(d->numRounds == eng->cfg.R, VD_E_SHAPE, "numRounds != params.maxQuesCount");
  VD_REQUIRE(d->numOptions == eng->cfg.K, VD_E_SHAPE, "opt:size(3) != params.numOptions");
  std::unique_ptr<Corpus> c(new Corpus());
  c->eng = eng;
  c->gpuid = eng->cfg.gpuid;
  c->n = d->numThreads; c->R = d->numRounds; c->Lq = d->maxQuesLen; c->La = d->maxAnsLen; c->Lc = d->maxCapLen;
  c->K = d->numOptions; c->m = d->numOptList; c->nimg = d->numImages;
  c->useHist = d->useHistory != 0; c->concat = d->concatHistory != 0; c->useIm = d->useIm != 0;
  c->start_tok = d->startToken; c->end_tok = d->endToken;
  const int n = c->n, R = c->R, Lq = c->Lq, La = c->La, K = c->K, m = c->m;
  const int64_t nr = (int64_t)n * R;
  cudaStream_t st = eng->main_stream;
  LaunchCtx& cx = eng->cx;
  auto grid1 = [](int64_t total) { return (unsigned)((total + 255) / 256); };

  // ---- validation the reference gets for free from Lua's bounds-checked indexing ----
  check_lengths(d->ques_len, nr, 0, Lq, "ques_length");
  check_lengths(d->ans_len, nr, 0, La, "ans_length");
  check_lengths(d->opt_len, m, 0, La, "opt_length");
  check_lengths(d->opt, nr * K, 1, m, "opt");
  if (d->ans_index) check_lengths(d->ans_index, nr, 0, K, "ans_index");

  // ---- raw arrays -> HBM ----
  c->ques = c->upload(d->ques, nr * Lq);
  c->ques_len = c->upload(d->ques_len, nr);
  c->ans = c->upload(d->ans, nr * La);
  c->ans_len = c->upload(d->ans_len, nr);
  c->opt = c->upload(d->opt, nr * K);
  c->opt_list = c->upload(d->opt_list, (int64_t)m * La);
  c->opt_len = c->upload(d->opt_len, m);
  if (d->ans_index) { c->ans_index = c->upload(d->ans_index, nr); c->has_ans_index = true; }
  c->h_ques_len.assign(d->ques_len, d->ques_len + nr);
  c->h_ans_len1.resize(nr);
  for (int64_t i = 0; i < nr; ++i) c->h_ans_len1[i] = d->ans_len[i] + 1;          // dataloader.lua:196

  // ---- prepareDataset on the device ----
  c->ques_fwd = c->dalloc<int32_t>(nr * Lq);                                       // :146-147
  k_right_align<<<grid1(nr * Lq), 256, 0, st>>>(c->ques, c->ques_len, c->ques_fwd, nr * Lq, R, Lq);
  check_launch(cx, "k_right_align");

  if (c->useHist) {                                                                // :150, :202-278
    VD_REQUIRE(d->cap && d->cap_len, VD_E_BADARG, "useHistory: cap / cap_length missing");
    VD_REQUIRE(c->Lc >= Lq + La, VD_E_SHAPE, "cap:size(2) < maxQuesLen + maxAnsLen (dataloader.lua:236 would raise)");
    check_lengths(d->cap_len, n, 0, c->Lc, "cap_length");
    c->cap = c->upload(d->cap, (int64_t)n * c->Lc);
    c->cap_len = c->upload(d->cap_len, n);
    c->maxHistoryLen = c->concat ? std::min(R * (Lq + La), 300) : d->maxHistoryLen; // :217 / :142
    c->Wh = c->concat ? c->maxHistoryLen : Lq + La;                                // :219 / :223
    VD_REQUIRE(c->maxHistoryLen > 0, VD_E_SHAPE, "maxHistoryLen must be > 0");
    c->hist_len = c->dalloc<int32_t>(nr);
    k_hist_len<<<grid1(n), 256, 0, st>>>(c->cap_len, c->ques_len, c->ans_len, c->hist_len, n, R, Lq + La, c->concat);
    check_launch(cx, "k_hist_len");
    c->h_hist_len.resize(nr);
    VD_CUDA_CHECK(cudaMemcpyAsync(c->h_hist_len.data(), c->hist_len, nr * 4, cudaMemcpyDeviceToHost, st));
    VD_CUDA_CHECK(cudaStreamSynchronize(st));
    check_lengths(c->h_hist_len.data(), nr, 0, c->Wh, "hist_len (history longer than the history tensor: dataloader.lua:246-253 would raise)");
    c->hist = c->dalloc<int32_t>(nr * c->Wh);
    k_build_hist<<<grid1(nr * c->Wh), 256, 0, st>>>(c->cap, c->ques, c->ans, c->ques_len, c->hist_len, c->hist,
                                                     nr * c->Wh, R, c->Wh, c->Lc, Lq, La, c->concat, c->end_tok);
    check_launch(cx, "k_build_hist");
  }

  c->opt_in = c->dalloc<int32_t>((int64_t)m * (La + 1));                           // :153, :281-321
  c->opt_out = c->dalloc<int32_t>((int64_t)m * (La + 1));
  k_wrap_start_end<<<grid1((int64_t)m * (La + 1)), 256, 0, st>>>(c->opt_list, c->opt_len, c->opt_in, c->opt_out,
                                                                  (int64_t)m * (La + 1), La, c->start_tok, c->end_tok, 0);
  check_launch(cx, "k_wrap_start_end");
  c->opt_maxlen = c->dalloc<int32_t>(nr);
  k_opt_maxlen<<<(unsigned)((nr + 7) / 8), 256, 0, st>>>(c->opt, c->opt_len, c->opt_maxlen, nr, K);
  check_launch(cx, "k_opt_maxlen");
  c->h_opt_maxlen.resize(nr);
  VD_CUDA_CHECK(cudaMemcpyAsync(c->h_opt_maxlen.data(), c->opt_maxlen, nr * 4, cudaMemcpyDeviceToHost, st));

  c->ans_in = c->dalloc<int32_t>(nr * (La + 1));                                   // :155, :159-199
  c->ans_out = c->dalloc<int32_t>(nr * (La + 1));
  k_wrap_start_end<<<grid1(nr * (La + 1)), 256, 0, st>>>(c->ans, c->ans_len, c->ans_in, c->ans_out, nr * (La + 1), La,
                                                          c->start_tok, c->end_tok, 1);
  check_launch(cx, "k_wrap_start_end");

  // ---- image features: (optional) L2 norm + NCHW -> NHWC, resident in HBM (:59-77) ----
  if (c->useIm) {
    VD_REQUIRE(d->images && d->img_pos && d->numImages > 0 && d->imgChannels > 0, VD_E_BADARG, "useIm: images / img_pos missing");
    check_lengths(d->img_pos, n, 0, d->numImages - 1, "img_pos");
    c->img_pos = c->upload(d->img_pos, n);
    VD_REQUIRE(d->imgAtt >= 0 && d->imgAtt <= 2, VD_E_BADARG, "imgAtt must be 0, 1 or 2");
    const bool region = d->imgAtt == 2;
    const int C = d->imgChannels, P = region ? d->imgSpatial : d->imgAtt ? d->imgSpatial * d->imgSpatial : 1;
    VD_REQUIRE(!d->imgAtt || d->imgSpatial > 0, VD_E_SHAPE, "imgSpatial");
    VD_REQUIRE(!region || !d->imgNorm, VD_E_BADARG, "region features are not L2-normalised (imgNorm = 0)");
    VD_REQUIRE(!region || C % 4 == 0, VD_E_SHAPE, "region feature channels must be a multiple of 4");
    VD_REQUIRE(!eng->cfg.useIm || region == (eng->cfg.regions > 0), VD_E_SHAPE,
               "region features need an engine with imgRegions = P, grid features one with imgRegions = 0");
    c->regions = region ? P : 0;
    c->img_elems = (int64_t)C * P;
    VD_REQUIRE(c->img_elems % 4 == 0, VD_E_SHAPE, "image feature row must be a multiple of 4 floats");
    const int64_t want = eng->cfg.att ? (int64_t)eng->cfg.P * eng->cfg.F : (int64_t)eng->cfg.F;
    VD_REQUIRE(!eng->cfg.useIm || c->img_elems == want, VD_E_SHAPE, "image feature size != params");
    c->img_fv = c->dalloc<float>((int64_t)c->nimg * c->img_elems);
    if (d->imgAtt != 1) {                       // fc7 rows, or region rows (N, P, C) as stored
      VD_CUDA_CHECK(cudaMemcpyAsync(c->img_fv, d->images, (size_t)c->nimg * c->img_elems * 4, cudaMemcpyHostToDevice, st));
      if (d->imgNorm) { k_img_norm_rows<<<c->nimg, 256, 0, st>>>(c->img_fv, C); check_launch(cx, "k_img_norm_rows"); }
    } else {
      // staged in chunks of <= 256 MB so a 33 GB feature file never needs a second full-size device buffer
      const int chunk = (int)std::max<int64_t>(1, std::min<int64_t>(c->nimg, (256ll << 20) / (c->img_elems * 4)));
      float* stage = nullptr; float* nm = nullptr;
      VD_CUDA_CHECK(cudaMalloc(&stage, (size_t)chunk * c->img_elems * 4));
      if (d->imgNorm) VD_CUDA_CHECK(cudaMalloc(&nm, (size_t)chunk * P * 4));
      for (int i0 = 0; i0 < c->nimg; i0 += chunk) {
        const int cnt = std::min(chunk, c->nimg - i0);
        VD_CUDA_CHECK(cudaMemcpyAsync(stage, d->images + (int64_t)i0 * c->img_elems, (size_t)cnt * c->img_elems * 4,
                                      cudaMemcpyHostToDevice, st));
        if (d->imgNorm) {
          k_img_norm_pos<<<dim3(cdiv(P, 128), cnt), 128, 0, st>>>(stage, nm, C, P);
          check_launch(cx, "k_img_norm_pos");
        }
        k_img_nchw_to_nhwc<<<dim3(cdiv(P, 32), cdiv(C, 32), cnt), dim3(32, 8), 0, st>>>(
            stage, d->imgNorm ? nm : nullptr, c->img_fv + (int64_t)i0 * c->img_elems, C, P);
        check_launch(cx, "k_img_nchw_to_nhwc");
      }
      VD_CUDA_CHECK(cudaStreamSynchronize(st));
      cudaFree(stage);
      if (nm) cudaFree(nm);
    }
  }
  VD_CUDA_CHECK(cudaStreamSynchronize(st));
  for (int s = 0; s < 2; ++s) VD_CUDA_CHECK(cudaEventCreateWithFlags(&c->ind_free[s], cudaEventDisableTiming));
  return c.release();
}

void corpus_destroy(Corpus* c) { delete c; }

void corpus_get_batch(Corpus* c, const int64_t* inds, int n, int decoder_gen, vd_batch* out) {
  VD_REQUIRE(inds != nullptr && out != nullptr, VD_E_BADARG, "inds / out is null");
  VD_REQUIRE(n > 0, VD_E_SHAPE, "batch must hold at least one dialog");
  VD_REQUIRE(decoder_gen >= 0 && decoder_gen <= 2, VD_E_BADARG, "decoder_gen must be 0, 1 or 2");
  Engine* eng = c->eng;
  VD_CUDA_CHECK(cudaSetDevice(c->gpuid));
  cudaStream_t st = eng->main_stream;
  LaunchCtx& cx = eng->cx;
  const int R = c->R, K = c->K, La = c->La, Lq = c->Lq;
  const int s = c->cur; c->cur ^= 1;
  Corpus::OutSet& o = c->out[s];

  // maxima over the batch: torch.max(batchQuesLen) etc. (dataloader.lua:380-381, 388-389, 401-402, 443-444)
  int Tq = 0, Th = 0, Ta = 0, To = 0;
  for (int b = 0; b < n; ++b) {
    VD_REQUIRE(inds[b] >= 0 && inds[b] < c->n, VD_E_SHAPE, "dialog index out of range");
    const int64_t base = inds[b] * R;
    for (int r = 0; r < R; ++r) {
      Tq = std::max(Tq, c->h_ques_len[base + r]);
      Ta = std::max(Ta, c->h_ans_len1[base + r]);
      if (c->useHist) Th = std::max(Th, c->h_hist_len[base + r]);
      if (decoder_gen == 2) To = std::max(To, c->h_opt_maxlen[base + r]);
    }
  }
  if (c->useHist) Th = std::min(Th, c->maxHistoryLen);                             // :389
  VD_REQUIRE(Tq > 0, VD_E_SHAPE, "every question of the batch is empty (the reference's {-0,-1} slice raises)");
  VD_REQUIRE(!c->useHist || Th > 0, VD_E_SHAPE, "every history of the batch is empty (the reference's {-0,-1} slice raises)");
  if (decoder_gen == 0) To = La;                                                   // raw opt_list rows, never trimmed (:452-459)

  // dialog indices -> device (the only per-batch PCIe traffic)
  if (c->h_ind_cap[s] < n) {
    if (c->h_ind[s]) { VD_CUDA_CHECK(cudaEventSynchronize(c->ind_free[s])); cudaFreeHost(c->h_ind[s]); c->h_ind[s] = nullptr; }
    VD_CUDA_CHECK(cudaMallocHost(&c->h_ind[s], (size_t)n * 4));
    c->h_ind_cap[s] = n;
  } else {
    VD_CUDA_CHECK(cudaEventSynchronize(c->ind_free[s]));                           // previous copy out of this slot is done
  }
  for (int b = 0; b < n; ++b) c->h_ind[s][b] = (int32_t)inds[b];
  int32_t* ind = (int32_t*)o.ind.ensure((size_t)n * 4);
  VD_CUDA_CHECK(cudaMemcpyAsync(ind, c->h_ind[s], (size_t)n * 4, cudaMemcpyHostToDevice, st));
  VD_CUDA_CHECK(cudaEventRecord(c->ind_free[s], st));

  GatherJobs jobs; jobs.n = 0;
  int64_t bytes = (int64_t)n * 4, max_total = 0;
  auto add = [&](const int32_t* src, const int32_t* rowidx, GrowBuf& buf, int rows, int W, int T, int off) -> int32_t* {
    GatherJob& j = jobs.j[jobs.n++];
    const int64_t elems = (int64_t)n * rows * T;
    int32_t* dst = (int32_t*)buf.ensure((size_t)elems * 4);
    j.src = src; j.rowidx = rowidx; j.dst = dst; j.rows = rows;
    j.vec = (W % 4 == 0 && T % 4 == 0 && off % 4 == 0) ? 1 : 0;
    j.W = j.vec ? W / 4 : W; j.T = j.vec ? T / 4 : T; j.off = j.vec ? off / 4 : off;
    j.total = (int64_t)n * rows * j.T;
    max_total = std::max(max_total, j.total);
    bytes += elems * 8 + (rowidx ? (int64_t)n * rows * 4 : 0);
    return dst;
  };
  memset(out, 0, sizeof(*out));
  out->B = n; out->Tq = Tq; out->Th = Th; out->To = To; out->Ta = Ta;
  out->ques_fwd = add(c->ques_fwd, nullptr, o.ques, R, Lq, Tq, Lq - Tq);             // :382-383 {-maxQuesLen,-1}
  if (c->useHist) out->hist = add(c->hist, nullptr, o.hist, R, c->Wh, Th, c->Wh - Th);  // :390-391
  out->answer_in = add(c->ans_in, nullptr, o.ans_in, R, La + 1, Ta, 0);              // :404-407 {1,maxAnsLen}
  out->answer_out = add(c->ans_out, nullptr, o.ans_out, R, La + 1, Ta, 0);
  if (c->has_ans_index) out->answer_ind = add(c->ans_index, nullptr, o.ans_ind, R, 1, 1, 0);   // :427-430
  if (decoder_gen == 0) {
    out->options = add(c->opt_list, c->opt, o.options, R * K, La, La, 0);            // :464-470
  } else if (decoder_gen == 2) {
    out->option_in = add(c->opt_in, c->opt, o.opt_in, R * K, La + 1, To, 0);         // :446-457
    out->option_out = add(c->opt_out, c->opt, o.opt_out, R * K, La + 1, To, 0);
  }
  int launches = 0;
  {
    const int gx = (int)std::min<int64_t>((max_total + 255) / 256, (int64_t)cx.sm_count * 8);
    LaunchCtx::Scope sc(&cx, "corpus_gather", 0, (double)bytes);
    k_gather_tokens<<<dim3(std::max(gx, 1), jobs.n), 256, 0, st>>>(jobs, ind);
    check_launch(cx, "k_gather_tokens");
    ++launches;
    if (c->useIm) {
      float* img = (float*)o.img.ensure((size_t)n * c->img_elems * 4);
      const int64_t e4 = c->img_elems / 4;
      int32_t* cnt = c->img_count ? (int32_t*)o.cnt.ensure((size_t)n * 4) : nullptr;
      k_gather_img<<<dim3(cdiv(e4, 1024), n), 256, 0, st>>>((const float4*)c->img_fv, c->img_pos, ind, (float4*)img, e4,
                                                              c->img_count, cnt);
      check_launch(cx, "k_gather_img");
      ++launches;
      out->img_feat = img;
      out->img_count = cnt;
      bytes += (int64_t)n * c->img_elems * 8 + (int64_t)n * 4 + (cnt ? (int64_t)n * 8 : 0);
    }
  }
  out->on_device = 1;
  c->last_bytes = bytes; c->last_launches = launches;
}

void corpus_read(Corpus* c, const char* name, void* host_dst, int64_t* elems) {
  VD_REQUIRE(name != nullptr && elems != nullptr, VD_E_BADARG, "name / elems is null");
  const int64_t nr = (int64_t)c->n * c->R;
  const void* p = nullptr; int64_t cnt = 0;
  const std::string k(name);
  if (k == "ques_fwd") { p = c->ques_fwd; cnt = nr * c->Lq; }
  else if (k == "hist") { p = c->hist; cnt = nr * c->Wh; }
  else if (k == "hist_len") { p = c->hist_len; cnt = nr; }
  else if (k == "ans_in") { p = c->ans_in; cnt = nr * (c->La + 1); }
  else if (k == "ans_out") { p = c->ans_out; cnt = nr * (c->La + 1); }
  else if (k == "opt_in") { p = c->opt_in; cnt = (int64_t)c->m * (c->La + 1); }
  else if (k == "opt_out") { p = c->opt_out; cnt = (int64_t)c->m * (c->La + 1); }
  else if (k == "img_fv") { p = c->img_fv; cnt = (int64_t)c->nimg * c->img_elems; }
  else if (k == "opt_list") { p = c->opt_list; cnt = (int64_t)c->m * c->La; }       // the split's answer pool (DESIGN §18)
  else VD_REQUIRE(false, VD_E_BADARG, "unknown prepared tensor name");
  VD_REQUIRE(p != nullptr, VD_E_STATE, "this corpus does not hold that tensor (useHistory / useIm off)");
  *elems = cnt;
  if (host_dst) {
    VD_CUDA_CHECK(cudaSetDevice(c->gpuid));
    VD_CUDA_CHECK(cudaStreamSynchronize(c->eng->main_stream));
    VD_CUDA_CHECK(cudaMemcpy(host_dst, p, (size_t)cnt * 4, cudaMemcpyDeviceToHost));
  }
}

void corpus_region_counts(Corpus* c, const int32_t* counts_host, int64_t numImages) {
  VD_REQUIRE(c->regions > 0 && c->img_fv, VD_E_STATE, "region counts need a corpus of region features (imgAtt = 2)");
  // the pad rows are zeroed in place: counts set once could not be raised later without the rows they zeroed
  VD_REQUIRE(c->img_count == nullptr, VD_E_STATE, "region counts are set once per corpus");
  VD_REQUIRE(counts_host != nullptr, VD_E_BADARG, "counts is null");
  VD_REQUIRE(numImages == c->nimg, VD_E_BADARG, "counts must hold one entry per image (numImages)");
  for (int64_t i = 0; i < numImages; ++i)
    if (counts_host[i] < 1 || counts_host[i] > c->regions) {
      char buf[160];
      snprintf(buf, sizeof(buf), "num_boxes[%lld] = %d outside [1, %d]", (long long)i, counts_host[i], c->regions);
      throw CudaError(VD_E_BADARG, buf);
    }
  VD_CUDA_CHECK(cudaSetDevice(c->gpuid));
  cudaStream_t st = c->eng->main_stream;
  c->img_count = c->dalloc<int32_t>(c->nimg);
  VD_CUDA_CHECK(cudaMemcpyAsync(c->img_count, counts_host, (size_t)c->nimg * 4, cudaMemcpyHostToDevice, st));
  const int64_t C4 = c->img_elems / c->regions / 4, total4 = (int64_t)c->nimg * c->img_elems / 4;
  k_zero_pad_regions<<<(unsigned)((total4 + 255) / 256), 256, 0, st>>>((float4*)c->img_fv, c->img_count, total4, c->regions, C4);
  check_launch(c->eng->cx, "k_zero_pad_regions");
  VD_CUDA_CHECK(cudaStreamSynchronize(st));
}

void corpus_batch_bytes(Corpus* c, int64_t* bytes, int32_t* launches) {
  if (bytes) *bytes = c->last_bytes;
  if (launches) *launches = c->last_launches;
}

}  // namespace vd
