// HBM-/latency-bound kernels of the hot path: everything that is not a dense contraction.
// Coalesced, float4-vectorised where the layout allows, warp-shuffle reductions.
#include "../../include/visdial_b200.h"
#include "kernels.cuh"

namespace vd {
namespace {

constexpr unsigned FULL = 0xffffffffu;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(FULL, v, o));
  return v;
}
// block-wide sum / max for blockDim.x <= 1024 (multiple of 32); `sh` has >= 33 floats
__device__ __forceinline__ float block_sum(float v, float* sh) {
  v = warp_sum(v);
  int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = blockDim.x >> 5;
  __syncthreads();
  if (l == 0) sh[w] = v;
  __syncthreads();
  if (w == 0) {
    float t = l < nw ? sh[l] : 0.f;
    t = warp_sum(t);
    if (l == 0) sh[32] = t;
  }
  __syncthreads();
  return sh[32];
}
__device__ __forceinline__ float block_max(float v, float* sh) {
  v = warp_max(v);
  int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = blockDim.x >> 5;
  __syncthreads();
  if (l == 0) sh[w] = v;
  __syncthreads();
  if (w == 0) {
    float t = l < nw ? sh[l] : -INFINITY;
    t = warp_max(t);
    if (l == 0) sh[32] = t;
  }
  __syncthreads();
  return sh[32];
}
__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

// ------------------------------------------------------------------------------------------------
__global__ void k_transpose_ids(const int32_t* __restrict__ src, int32_t* __restrict__ dst, int64_t rows, int T) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;      // index into dst (t, r)
  if (i >= rows * T) return;
  int64_t t = i / rows, r = i % rows;
  dst[i] = src[r * T + t];
}
// the same transpose over the K option rows of one selected round per dialog: dst row j = b*K + k reads source row
// (b*R + round[b])*K + k
__global__ void k_transpose_ids_rounds(const int32_t* __restrict__ src, const int32_t* __restrict__ round, int32_t* __restrict__ dst,
                                       int64_t rows, int T, int R, int K) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * T) return;
  int64_t t = i / rows, j = i % rows, b = j / K;
  dst[i] = src[(((b * R + round[b]) * K) + j % K) * T + t];
}
// dst[b,:] = src[b*R + round[b], :]  (gather = 1);  dst[b*R + round[b], :] = src[b,:] into a zeroed dst  (gather = 0)
__global__ void k_round_rows(const float* __restrict__ src, const int32_t* __restrict__ round, float* __restrict__ dst, int64_t B,
                             int R, int H, int gather) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * H) return;
  int64_t b = i / H, c = i % H, n = b * R + round[b];
  if (gather) dst[i] = src[n * H + c];
  else dst[n * H + c] = src[i];
}

__global__ void k_embed_rows(float* __restrict__ out, const float* __restrict__ emb, const int32_t* __restrict__ ids,
                             int64_t rows, int E4, DropCfg d, uint32_t site) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;      // float4 index
  if (i >= rows * E4) return;
  int64_t r = i / E4;
  int e4 = (int)(i % E4);
  int id = ids[r];
  float4 v = make_float4(0, 0, 0, 0);
  if (id != 0) v = reinterpret_cast<const float4*>(emb + (int64_t)id * E4 * 4)[e4];
  float f[4];
  drop_factor4(d, site, (uint64_t)i, f);      // element index = i*4 .. i*4+3  (E % 4 == 0)
  v.x *= f[0]; v.y *= f[1]; v.z *= f[2]; v.w *= f[3];
  reinterpret_cast<float4*>(out)[i] = v;
}

constexpr int SC_ROWS = 32, SC_THREADS = 128, SC_MAXACC = 8;   // E <= 1024
__global__ void __launch_bounds__(SC_THREADS) k_embed_scatter_add(float* __restrict__ demb, const float* __restrict__ dx,
                                                                 int64_t ldx, const int32_t* __restrict__ ids,
                                                                 int64_t rows, int E, DropCfg d, uint32_t site) {
  float pad_acc[SC_MAXACC];
#pragma unroll
  for (int a = 0; a < SC_MAXACC; ++a) pad_acc[a] = 0.f;
  int64_t r0 = (int64_t)blockIdx.x * SC_ROWS;
  for (int rr = 0; rr < SC_ROWS; ++rr) {
    int64_t r = r0 + rr;
    if (r >= rows) break;
    int id = ids[r];
#pragma unroll
    for (int a = 0; a < SC_MAXACC; ++a) {
      int e = threadIdx.x + a * SC_THREADS;
      if (e < E) {
        float v = dx[r * ldx + e] * drop_factor(d, site, (uint64_t)r * E + e);
        if (id == 0) pad_acc[a] += v;
        else atomicAdd(demb + (int64_t)id * E + e, v);
      }
    }
  }
#pragma unroll
  for (int a = 0; a < SC_MAXACC; ++a) {
    int e = threadIdx.x + a * SC_THREADS;
    if (e < E && pad_acc[a] != 0.f) atomicAdd(demb + e, pad_acc[a]);
  }
}

// ------------------------------------------------------------------------------------------------
__global__ void k_lstm_pw_fwd(float* __restrict__ gates, const float* __restrict__ bias, const float* __restrict__ c_prev,
                              const int32_t* __restrict__ mask_ids, float* __restrict__ c_out, float* __restrict__ h_out,
                              int64_t R, int H) {
  int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int H4 = H >> 2;
  if (idx >= R * H4) return;
  int64_t r = idx / H4;
  int j = (int)(idx % H4) * 4;
  float4* g4 = reinterpret_cast<float4*>(gates + r * 4 * H);
  float4 zero = make_float4(0, 0, 0, 0);
  if (mask_ids && mask_ids[r] == 0) {
    g4[(j) >> 2] = zero; g4[(H + j) >> 2] = zero; g4[(2 * H + j) >> 2] = zero; g4[(3 * H + j) >> 2] = zero;
    reinterpret_cast<float4*>(c_out + r * H)[j >> 2] = zero;
    reinterpret_cast<float4*>(h_out + r * H)[j >> 2] = zero;
    return;
  }
  float4 ai = g4[j >> 2], af = g4[(H + j) >> 2], ao = g4[(2 * H + j) >> 2], ag = g4[(3 * H + j) >> 2];
  float4 bi = reinterpret_cast<const float4*>(bias)[j >> 2], bf = reinterpret_cast<const float4*>(bias + H)[j >> 2],
         bo = reinterpret_cast<const float4*>(bias + 2 * H)[j >> 2], bg = reinterpret_cast<const float4*>(bias + 3 * H)[j >> 2];
  float4 cp = c_prev ? reinterpret_cast<const float4*>(c_prev + r * H)[j >> 2] : zero;
  float* pi = &ai.x; float* pf = &af.x; float* po = &ao.x; float* pg = &ag.x;
  const float* pbi = &bi.x; const float* pbf = &bf.x; const float* pbo = &bo.x; const float* pbg = &bg.x;
  const float* pc = &cp.x;
  float4 cn, hn;
  float* pcn = &cn.x; float* phn = &hn.x;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    float i = sigmoidf_(pi[q] + pbi[q]), f = sigmoidf_(pf[q] + pbf[q]), o = sigmoidf_(po[q] + pbo[q]);
    float g = tanhf(pg[q] + pbg[q]);
    float c = f * pc[q] + i * g;
    pi[q] = i; pf[q] = f; po[q] = o; pg[q] = g;
    pcn[q] = c; phn[q] = o * tanhf(c);
  }
  g4[j >> 2] = ai; g4[(H + j) >> 2] = af; g4[(2 * H + j) >> 2] = ao; g4[(3 * H + j) >> 2] = ag;
  reinterpret_cast<float4*>(c_out + r * H)[j >> 2] = cn;
  reinterpret_cast<float4*>(h_out + r * H)[j >> 2] = hn;
}

// SeqLSTM step with no recurrent term (t = 0 without h0): pre-activation = x-projection (+ bias), taken either from
// the gates buffer (in place) or gathered from the projection table.  One thread per (row, 4 hidden units).
__global__ void k_lstm_first_step(float* __restrict__ gates, const float* __restrict__ ptable, const int32_t* __restrict__ tok,
                                  const float* __restrict__ bias, const float* __restrict__ c_prev,
                                  const int32_t* __restrict__ mask_ids, float* __restrict__ c_out, float* __restrict__ h_out,
                                  int64_t R, int H) {
  int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int H4 = H >> 2;
  if (idx >= R * H4) return;
  const int64_t r = idx / H4;
  const int j = (int)(idx % H4) * 4;
  const float4 zero = make_float4(0, 0, 0, 0);
  const bool masked = mask_ids && mask_ids[r] == 0;
  const float* src = ptable ? ptable + (int64_t)tok[r] * 4 * H : gates + r * 4 * H;
  float4 a[4];
#pragma unroll
  for (int g = 0; g < 4; ++g) {
    a[g] = *reinterpret_cast<const float4*>(src + g * H + j);
    if (bias) { const float4 b = *reinterpret_cast<const float4*>(bias + g * H + j); a[g].x += b.x; a[g].y += b.y; a[g].z += b.z; a[g].w += b.w; }
  }
  const float4 cp = c_prev ? *reinterpret_cast<const float4*>(c_prev + r * H + j) : zero;
  float4 cn, hn;
  float* pa[4] = {&a[0].x, &a[1].x, &a[2].x, &a[3].x};
  const float* pc = &cp.x; float* pcn = &cn.x; float* phn = &hn.x;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    float gi = sigmoidf_(pa[0][q]), gf = sigmoidf_(pa[1][q]), go = sigmoidf_(pa[2][q]), gg = tanhf(pa[3][q]);
    float c = gf * pc[q] + gi * gg;
    float keep = masked ? 0.f : 1.f;
    pa[0][q] = gi * keep; pa[1][q] = gf * keep; pa[2][q] = go * keep; pa[3][q] = gg * keep;
    pcn[q] = c * keep; phn[q] = go * tanhf(c) * keep;
  }
  if (gates) {
#pragma unroll
    for (int g = 0; g < 4; ++g) *reinterpret_cast<float4*>(gates + r * 4 * H + g * H + j) = a[g];
  }
  *reinterpret_cast<float4*>(c_out + r * H + j) = cn;
  *reinterpret_cast<float4*>(h_out + r * H + j) = hn;
}

__global__ void k_lstm_pw_bwd(const float* __restrict__ gates, const float* __restrict__ c_prev, const float* __restrict__ c,
                              const float* __restrict__ dh_rec, const float* __restrict__ dh_ext,
                              const float* __restrict__ dc_ext, float* __restrict__ dc_carry,
                              const int32_t* __restrict__ mask_ids, float* __restrict__ da, int64_t R, int H) {
  int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= R * H) return;
  int64_t r = idx / H;
  int j = (int)(idx % H);
  const float* g = gates + r * 4 * H;
  float* d = da + r * 4 * H;
  if (mask_ids && mask_ids[r] == 0) {
    d[j] = 0.f; d[H + j] = 0.f; d[2 * H + j] = 0.f; d[3 * H + j] = 0.f;
    dc_carry[idx] = 0.f;
    return;
  }
  float gi = g[j], gf = g[H + j], go = g[2 * H + j], gg = g[3 * H + j];
  float cp = c_prev ? c_prev[idx] : 0.f;
  float dh = (dh_rec ? dh_rec[idx] : 0.f) + (dh_ext ? dh_ext[idx] : 0.f);
  float dc = dc_carry[idx] + (dc_ext ? dc_ext[idx] : 0.f);
  float tc = tanhf(c[idx]);
  dc += dh * go * (1.f - tc * tc);
  d[j] = dc * gg * gi * (1.f - gi);
  d[H + j] = dc * cp * gf * (1.f - gf);
  d[2 * H + j] = dh * tc * go * (1.f - go);
  d[3 * H + j] = dc * gi * (1.f - gg * gg);
  dc_carry[idx] = dc * gf;
}

// ---- beam search on the device (model.lua:510-570): the state shuffle
// next step's previous state of row r: parent >= 0 -> the state hypothesis `parent` PRODUCED in the last step; parent < 0 -> the
// state row (-1 - parent) was FED in the last step (a beam column that received no candidate keeps its old content, model.lua:560-569)
__global__ void k_beam_gather(float* __restrict__ dst, const float* __restrict__ out_prev, const float* __restrict__ in_prev,
                              const int32_t* __restrict__ parent, int64_t rows, int H) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * H) return;
  const int64_t r = i / H; const int c = (int)(i % H);
  const int p = parent[r];
  dst[i] = p >= 0 ? out_prev[(int64_t)p * H + c] : in_prev[(int64_t)(-1 - p) * H + c];
}

// row log-sum-exp from the per-slice (max, sum exp) partials of the fused vocabulary projection
__device__ __forceinline__ float parts_lse(const float* m, const float* s, int nparts) {
  float mx = -INFINITY;
  for (int i = 0; i < nparts; ++i) mx = fmaxf(mx, m[i]);
  float sum = 0.f;
  for (int i = 0; i < nparts; ++i) sum += s[i] * expf(m[i] - mx);
  return mx + logf(sum);
}

// row log-sum-exp from the partials, then the criterion / likelihood term
__global__ void k_vocab_lse_finish(const float* __restrict__ pm, const float* __restrict__ ps, int nparts,
                                   const float* __restrict__ tl, const int32_t* __restrict__ tgt, const int32_t* __restrict__ ids,
                                   float* __restrict__ lse, float* __restrict__ out, float sign, int accumulate, int64_t rows) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  const float l = parts_lse(pm + r * nparts, ps + r * nparts, nparts);
  if (lse) lse[r] = l;
  if (out) {
    const bool keep = ids[r] != 0 && tgt[r] > 0;
    const float v = keep ? sign * (tl[r] - l) : 0.f;
    out[r] = accumulate ? out[r] + v : v;
  }
}

// the sampling step's reduction over the slices of MODE_SAMPLE (thread per row): lse as k_vocab_lse_finish forms it, the
// winning slice by (key desc, class asc), then the token, the answer column and x_tok - lse
__global__ void k_vocab_sample_finish(const float* __restrict__ pm, const float* __restrict__ ps, const float* __restrict__ pk,
                                      const int32_t* __restrict__ pc, const float* __restrict__ px, int nparts, int64_t rows,
                                      int step, int L, int32_t* __restrict__ tokens, int32_t* __restrict__ answer,
                                      float* __restrict__ logp) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  const int64_t o = r * nparts;
  const float l = parts_lse(pm + o, ps + o, nparts);
  float bk = pk[o], bx = px[o];
  int bc = pc[o];
  for (int i = 1; i < nparts; ++i)
    if (sample_before(pk[o + i], pc[o + i], bk, bc)) { bk = pk[o + i]; bc = pc[o + i]; bx = px[o + i]; }
  tokens[r] = bc + 1;
  answer[r * (L + 1) + step] = bc + 1;
  if (logp) logp[r * L + step - 1] = bx - l;
}

// ------------------------------------------------------------------------------------------------
// out[c] += sum_r X[r, c] (bias gradients).  HBM-bound: a block covers 256 rows x 128 columns, a warp reads whole 512-byte row pieces
// (float4 per lane) of every 8th row with 4 loads in flight, the 8 warps are combined in shared memory, then one atomicAdd per column.
// SLOT (deterministic mode): the block's column sums go to its row of out (gridDim.y, cols) instead, for slot_reduce.
constexpr int CS_ROWS = 256;
template <bool SLOT>
__global__ void __launch_bounds__(256) k_colsum_add4(float* __restrict__ out, const float* __restrict__ X, int64_t rows, int cols, int64_t ldx) {
  __shared__ float4 red[8][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int c = (blockIdx.x * 32 + lane) * 4;
  const int64_t r0 = (int64_t)blockIdx.y * CS_ROWS, r1 = min(rows, r0 + CS_ROWS);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  if (c < cols) {
    const float* p = X + c;
    int64_t r = r0 + warp;
    for (; r + 24 < r1; r += 32) {
      const float4 a = *reinterpret_cast<const float4*>(p + r * ldx), b = *reinterpret_cast<const float4*>(p + (r + 8) * ldx);
      const float4 d = *reinterpret_cast<const float4*>(p + (r + 16) * ldx), e = *reinterpret_cast<const float4*>(p + (r + 24) * ldx);
      acc.x += (a.x + b.x) + (d.x + e.x); acc.y += (a.y + b.y) + (d.y + e.y);
      acc.z += (a.z + b.z) + (d.z + e.z); acc.w += (a.w + b.w) + (d.w + e.w);
    }
    for (; r < r1; r += 8) {
      const float4 a = *reinterpret_cast<const float4*>(p + r * ldx);
      acc.x += a.x; acc.y += a.y; acc.z += a.z; acc.w += a.w;
    }
  }
  red[warp][lane] = acc;
  __syncthreads();
  if (warp == 0 && c < cols) {
#pragma unroll
    for (int w = 1; w < 8; ++w) { const float4 o = red[w][lane]; acc.x += o.x; acc.y += o.y; acc.z += o.z; acc.w += o.w; }
    if constexpr (SLOT) {
      float* o = out + (int64_t)blockIdx.y * cols + c;
      o[0] = acc.x; o[1] = acc.y; o[2] = acc.z; o[3] = acc.w;
    } else {
      atomicAdd(out + c, acc.x); atomicAdd(out + c + 1, acc.y); atomicAdd(out + c + 2, acc.z); atomicAdd(out + c + 3, acc.w);
    }
  }
}
// any shape (odd column counts, unaligned leading dimension): one thread per column
template <bool SLOT>
__global__ void k_colsum_add(float* __restrict__ out, const float* __restrict__ X, int64_t rows, int cols, int64_t ldx) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= cols) return;
  int64_t r0 = (int64_t)blockIdx.y * CS_ROWS, r1 = min(rows, r0 + CS_ROWS);
  float acc = 0.f;
  for (int64_t r = r0; r < r1; ++r) acc += X[r * ldx + c];
  if constexpr (SLOT) out[(int64_t)blockIdx.y * cols + c] = acc;
  else atomicAdd(out + c, acc);
}

__global__ void k_dropout_apply(float* __restrict__ out, const float* __restrict__ in, int64_t n, DropCfg d, uint32_t site) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  out[i] = in[i] * drop_factor(d, site, (uint64_t)i);
}
__global__ void k_tanh_bwd(float* __restrict__ dpre, const float* __restrict__ dy, const float* __restrict__ y, int64_t n) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float yy = y[i];
  dpre[i] = dy[i] * (1.f - yy * yy);
}
__global__ void k_add_inplace(float* __restrict__ a, const float* __restrict__ b, int64_t n) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) a[i] += b[i];
}
__global__ void k_add_out(float* __restrict__ o, const float* __restrict__ a, const float* __restrict__ b, int64_t n) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) o[i] = a[i] + b[i];
}
__global__ void k_copy_cols(float* __restrict__ dst, int64_t ldd, const float* __restrict__ src, int64_t lds, int64_t rows, int cols) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * cols) return;
  int64_t r = i / cols; int c = (int)(i % cols);
  dst[r * ldd + c] = src[r * lds + c];
}
__global__ void k_repeat_rows(float* __restrict__ dst, const float* __restrict__ src, int64_t B, int R, int64_t cols,
                              int64_t lds) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * R * cols) return;
  int64_t n = i / cols, c = i % cols;
  dst[i] = src[(n / R) * lds + c];
}

// The history rule (DESIGN §17), the one place it lives on the device: row `prev` (W, right-aligned) -> the next row `out`
// from the question row q (src_w, right-aligned) and the answer tokens a, of which the first a_len[0] - 2 (a_len null:
// a_max) are read, cut at end_token, pads skipped, at most max_ans_len kept.  Every thread of the CTA calls it; a_s holds
// max_ans_len words.  The CTA synchronises once inside, before the writes; a caller that reads `out` next syncs again.
__device__ __forceinline__ void hist_next_row(const int32_t* __restrict__ prev, int32_t* __restrict__ out, int W,
                                              const int32_t* __restrict__ q, int src_w, const int32_t* __restrict__ a,
                                              const int32_t* __restrict__ a_len, int a_max, int end_token, int max_ans_len,
                                              int concat, int32_t* a_s, int* s_len) {
  if (threadIdx.x == 0) {
    int lp = 0, lq = 0, la = 0;                            // rows are pads then words: count the words from the right
    while (lp < W && prev[W - 1 - lp] != 0) ++lp;
    while (lq < src_w && q[src_w - 1 - lq] != 0) ++lq;
    if (lp > 0 && lq > 0) {
      const int n = a_len ? max(a_len[0] - 2, 0) : a_max;
      for (int i = 0; i < n && la < max_ans_len; ++i) {
        const int32_t t = a[i];
        if (t == end_token) break;
        if (t != 0) a_s[la++] = t;                          // a pad a stale beam column carried is not a word
      }
    }
    s_len[0] = lp; s_len[1] = lq; s_len[2] = la;
  }
  __syncthreads();
  const int lp = s_len[0], lq = s_len[1], la = s_len[2];
  const int keep = concat ? lp + 1 : 0;                    // row r ++ <END>
  const int total = lp == 0 ? 0 : keep + lq + la;
  for (int j = threadIdx.x; j < W; j += blockDim.x) {
    const int s = total - W + j;                           // position in the unbounded row; the rightmost W are kept
    int32_t t = 0;
    if (s >= 0) {
      if (s < keep) t = s < lp ? prev[W - lp + s] : end_token;
      else if (s < keep + lq) t = q[src_w - lq + (s - keep)];
      else t = a_s[s - keep - lq];
    }
    out[j] = t;
  }
}

// the dialog loop's history rows (hist_append in kernels.cuh), one CTA per dialog, or per asked row of a dialog pool
// (slot non-null: row b writes dialog slot[b], at round round[b] unless r < 0)
__global__ void k_hist_append(int32_t* __restrict__ hist, int R, int W, int r, const int32_t* __restrict__ src, int src_w,
                              const int32_t* __restrict__ ans, int64_t ans_ld, const int32_t* __restrict__ ans_len, int ans_max,
                              int end_token, int max_ans_len, int concat, const int32_t* __restrict__ slot,
                              const int32_t* __restrict__ round) {
  extern __shared__ int32_t a_s[];                        // the answer's kept words (max_ans_len)
  __shared__ int s_len[3];
  const int64_t b = blockIdx.x, d = slot ? slot[b] : b;
  int32_t* rows = hist + d * R * W;
  if (r >= 0 && round) {
    r = round[b];
    if (r >= R - 1) return;                                 // the conversation's last round: there is no row r + 1
  }
  if (r < 0) {
    const int32_t* s = src + b * R * src_w;
    for (int j = threadIdx.x; j < R * W; j += blockDim.x) {
      const int c = j - (W - src_w);
      rows[j] = (j < W && c >= 0) ? s[c] : 0;
    }
    return;
  }
  hist_next_row(rows + (int64_t)r * W, rows + (int64_t)(r + 1) * W, W, src + (d * R + r) * src_w, src_w, ans + b * ans_ld,
                ans_len ? ans_len + b : nullptr, ans_max, end_token, max_ans_len, concat, a_s, s_len);
}

// a resumed conversation's history rows 1..rounds[i] (hist_prefill in kernels.cuh): CTA i builds them in order, each from
// the one before, with the rule above
__global__ void k_hist_prefill(int32_t* __restrict__ hist, int R, int W, const int32_t* __restrict__ slot,
                               const int32_t* __restrict__ rounds, const int32_t* __restrict__ row0, const int32_t* __restrict__ q,
                               int src_w, const int32_t* __restrict__ ans, int Ta, int end_token, int max_ans_len, int concat) {
  extern __shared__ int32_t a_s[];
  __shared__ int s_len[3];
  const int64_t i = blockIdx.x;
  int32_t* rows = hist + (int64_t)slot[i] * R * W;
  const int r = rounds[i];
  for (int j = 0; j < r; ++j) {
    hist_next_row(rows + (int64_t)j * W, rows + (int64_t)(j + 1) * W, W, q + (row0[j] + i) * src_w, src_w,
                  ans + (i * R + j) * Ta, nullptr, Ta, end_token, max_ans_len, concat, a_s, s_len);
    __syncthreads();                                       // row j + 1 is the next row's `prev`; a_s and s_len are reused
  }
}
__global__ void k_sum_repeated_rows(float* __restrict__ dst, const float* __restrict__ src, int64_t B, int R, int64_t cols) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * cols) return;
  int64_t b = i / cols, c = i % cols;
  float acc = 0.f;
  for (int r = 0; r < R; ++r) acc += src[(b * R + r) * cols + c];
  dst[i] = acc;
}

// seg table: per segment {offset, rows, cols}; Wt[off + c*rows + r] = W[off + r*cols + c]
__global__ void k_transpose_segments(const float* __restrict__ W, float* __restrict__ Wt, const int64_t* __restrict__ tab) {
  __shared__ float tile[32][33];
  const int64_t off = tab[blockIdx.y * 3], rows = tab[blockIdx.y * 3 + 1], cols = tab[blockIdx.y * 3 + 2];
  const int64_t tiles_c = (cols + 31) / 32, tiles_r = (rows + 31) / 32;
  for (int64_t t = blockIdx.x; t < tiles_c * tiles_r; t += gridDim.x) {
    int64_t tr = t / tiles_c, tc = t % tiles_c;
    for (int y = threadIdx.y; y < 32; y += blockDim.y) {
      int64_t r = tr * 32 + y, c = tc * 32 + threadIdx.x;
      tile[y][threadIdx.x] = (r < rows && c < cols) ? W[off + r * cols + c] : 0.f;
    }
    __syncthreads();
    for (int y = threadIdx.y; y < 32; y += blockDim.y) {
      int64_t c = tc * 32 + y, r = tr * 32 + threadIdx.x;
      if (r < rows && c < cols) Wt[off + c * rows + r] = tile[threadIdx.x][y];
    }
    __syncthreads();
  }
}

// warp per row
__global__ void k_rowdot_fwd(float* __restrict__ out, const float* __restrict__ x, const float* __restrict__ w,
                             const float* __restrict__ b, int64_t rows, int H) {
  int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  int l = threadIdx.x & 31;
  if (r >= rows) return;
  float acc = 0.f;
  for (int c = l; c < H; c += 32) acc += x[r * H + c] * w[c];
  acc = warp_sum(acc);
  if (l == 0) out[r] = acc + b[0];
}
// block per 32-row chunk; threads over columns.  SLOT (deterministic mode): the block's dw / db sums go to its row of dw
// (gridDim.x, H) / its element of db (gridDim.x), for slot_reduce.
template <bool SLOT>
__global__ void k_rowdot_bwd(const float* __restrict__ ds, const float* __restrict__ x, const float* __restrict__ w,
                             float* __restrict__ dx, int accumulate_dx, float* __restrict__ dw, float* __restrict__ db,
                             int64_t rows, int H) {
  int64_t r0 = (int64_t)blockIdx.x * 32, r1 = min(rows, r0 + 32);
  for (int c = threadIdx.x; c < H; c += blockDim.x) {
    float wc = w[c], acc = 0.f;
    for (int64_t r = r0; r < r1; ++r) {
      float s = ds[r];
      acc += s * x[r * H + c];
      if (dx) { if (accumulate_dx) dx[r * H + c] += s * wc; else dx[r * H + c] = s * wc; }
    }
    if constexpr (SLOT) dw[(int64_t)blockIdx.x * H + c] = acc;
    else atomicAdd(dw + c, acc);
  }
  if (threadIdx.x == 0) {
    float acc = 0.f;
    for (int64_t r = r0; r < r1; ++r) acc += ds[r];
    if constexpr (SLOT) db[blockIdx.x] = acc;
    else atomicAdd(db, acc);
  }
}

// ------------------------------------------------------------------------------------------------
// history attention; one block per dialog, dynamic smem = (2 or 3)*R*H + R*R floats.  The forwards take a round range
// [r0, r1): the query / output rows are rounds r0..r1-1 of each dialog (B*(r1-r0) rows), the facts of dialog b are rows
// 0..r1-1 of h + b*hpitch, probs is (B, r1-r0, R).  The full forward passes [0, R) and hpitch = R*H; a dialog session
// passes [r, r+1) over its cached facts.  With slot / round non-null (a dialog pool's ask) block b is query row b alone, at
// round round[b] over the facts of dialog slot[b]: r0, r1 are ignored.  Each output element is reduced in the same order
// whatever the range.
__global__ void k_mn_att_fwd(const float* __restrict__ q, const float* __restrict__ h, float* __restrict__ probs,
                             float* __restrict__ hAtt, int R, int H, int r0, int r1, int64_t hpitch,
                             const int32_t* __restrict__ slot, const int32_t* __restrict__ round) {
  extern __shared__ float sm[];
  const int b = blockIdx.x, tid = threadIdx.x, nw = blockDim.x >> 5, w = tid >> 5, l = tid & 31;
  const int64_t d = slot ? slot[b] : b;
  if (slot) { r0 = round[b]; r1 = r0 + 1; }
  const int nr = r1 - r0;
  float* sq = sm; float* shh = sm + nr * H; float* S = shh + r1 * H;
  for (int i = tid; i < nr * H; i += blockDim.x) sq[i] = q[(int64_t)b * nr * H + i];
  for (int i = tid; i < r1 * H; i += blockDim.x) shh[i] = h[d * hpitch + i];
  __syncthreads();
  for (int p = w; p < nr * R; p += nw) {
    int i = r0 + p / R, j = p % R;
    float acc = 0.f;
    if (j <= i) {
      for (int c = l; c < H; c += 32) acc += sq[(i - r0) * H + c] * shh[j * H + c];
      acc = warp_sum(acc);
    }
    if (l == 0) S[p] = (j <= i) ? acc : -9999999.f;       // MaskSoftMax.lua:12
  }
  __syncthreads();
  if (tid < nr) {
    float mx = -INFINITY;
    for (int j = 0; j < R; ++j) mx = fmaxf(mx, S[tid * R + j]);
    float sum = 0.f;
    for (int j = 0; j < R; ++j) { float e = expf(S[tid * R + j] - mx); S[tid * R + j] = e; sum += e; }
    for (int j = 0; j < R; ++j) S[tid * R + j] /= sum;
  }
  __syncthreads();
  for (int i = tid; i < nr * R; i += blockDim.x) probs[(int64_t)b * nr * R + i] = S[i];
  for (int o = tid; o < nr * H; o += blockDim.x) {
    int i = o / H, c = o % H;
    float acc = 0.f;
    for (int j = 0; j <= i + r0; ++j) acc += S[i * R + j] * shh[j * H + c];
    hAtt[(int64_t)b * nr * H + o] = acc;
  }
}

__global__ void k_mn_att_bwd(const float* __restrict__ q, const float* __restrict__ h, const float* __restrict__ probs,
                             const float* __restrict__ dhAtt, float* __restrict__ dq, float* __restrict__ dh, int R, int H) {
  extern __shared__ float sm[];
  float* sq = sm; float* shh = sq + R * H; float* sd = shh + R * H; float* P = sd + R * H; float* dS = P + R * R;
  const int b = blockIdx.x, tid = threadIdx.x, nw = blockDim.x >> 5, w = tid >> 5, l = tid & 31;
  for (int i = tid; i < R * H; i += blockDim.x) {
    sq[i] = q[(int64_t)b * R * H + i]; shh[i] = h[(int64_t)b * R * H + i]; sd[i] = dhAtt[(int64_t)b * R * H + i];
  }
  for (int i = tid; i < R * R; i += blockDim.x) P[i] = probs[(int64_t)b * R * R + i];
  __syncthreads();
  for (int p = w; p < R * R; p += nw) {       // dP
    int i = p / R, j = p % R;
    float acc = 0.f;
    if (j <= i) {
      for (int c = l; c < H; c += 32) acc += sd[i * H + c] * shh[j * H + c];
      acc = warp_sum(acc);
    }
    if (l == 0) dS[p] = acc;
  }
  __syncthreads();
  if (tid < R) {
    float dot = 0.f;
    for (int j = 0; j < R; ++j) dot += P[tid * R + j] * dS[tid * R + j];
    for (int j = 0; j < R; ++j) dS[tid * R + j] = P[tid * R + j] * (dS[tid * R + j] - dot);
  }
  __syncthreads();
  for (int o = tid; o < R * H; o += blockDim.x) {
    int i = o / H, c = o % H;
    float aq = 0.f, ah = 0.f;
    for (int j = 0; j <= i; ++j) aq += dS[i * R + j] * shh[j * H + c];
    // dh[j=i here as row index] = sum_i' dS[i'][row] q[i'] + P[i'][row] dhAtt[i']
    for (int ii = i; ii < R; ++ii) ah += dS[ii * R + i] * sq[ii * H + c] + P[ii * R + i] * sd[ii * H + c];
    dq[(int64_t)b * R * H + o] = aq;
    dh[(int64_t)b * R * H + o] = ah;
  }
}

// rounds [r0, r1) as k_mn_att_fwd: sq (B*(r1-r0)), sh (B, R) with only columns j <= i read, Hs rows 0..r1-1 of
// Hs + b*hpitch.  The weighted sum runs over j <= i: a masked probability is exactly 0, so the terms j > i the sum skips
// add exact zeros (for finite facts) and the full forward keeps its bits.  slot / round as k_mn_att_fwd's (sh then
// (slots, R)).
__global__ void k_hrea_att_fwd(const float* __restrict__ sq, const float* __restrict__ sh, const float* __restrict__ Hs,
                               float* __restrict__ probs, float* __restrict__ att, int R, int H, int r0, int r1, int64_t hpitch,
                               const int32_t* __restrict__ slot, const int32_t* __restrict__ round) {
  extern __shared__ float sm[];
  const int b = blockIdx.x, tid = threadIdx.x;
  const int64_t d = slot ? slot[b] : b;
  if (slot) { r0 = round[b]; r1 = r0 + 1; }
  const int nr = r1 - r0;
  float* shh = sm; float* S = shh + r1 * H;
  for (int i = tid; i < r1 * H; i += blockDim.x) shh[i] = Hs[d * hpitch + i];
  if (tid < nr) {
    int i = r0 + tid;
    float row[32];
    float mx = -INFINITY;
    for (int j = 0; j < R; ++j) {
      float v = (j > i) ? 0.f : sq[b * nr + tid] + sh[d * R + j];  // MaskFuture.lua:17-19
      if (v == 0.f) v = -INFINITY;                                  // ReplaceZero.lua:13-18
      row[j] = v; mx = fmaxf(mx, v);
    }
    float sum = 0.f;
    for (int j = 0; j < R; ++j) { row[j] = expf(row[j] - mx); sum += row[j]; }
    for (int j = 0; j < R; ++j) S[tid * R + j] = row[j] / sum;
  }
  __syncthreads();
  for (int i = tid; i < nr * R; i += blockDim.x) probs[(int64_t)b * nr * R + i] = S[i];
  for (int o = tid; o < nr * H; o += blockDim.x) {
    int i = o / H, c = o % H;
    float acc = 0.f;
    for (int j = 0; j <= i + r0; ++j) acc += S[i * R + j] * shh[j * H + c];
    att[(int64_t)b * nr * H + o] = acc;
  }
}

// a dialog session's cache write (dialog_cache_write in kernels.cuh), one thread per element of every piece present:
// facts, then shc, then the dialog-LSTM state's h and c
__global__ void k_dialog_cache_write(float* __restrict__ facts, float* __restrict__ shc, const float* __restrict__ h3,
                                     const float* __restrict__ sh, int64_t B, int R, int H, int r, const int32_t* __restrict__ slot,
                                     const int32_t* __restrict__ round, float* __restrict__ st_h, float* __restrict__ st_c,
                                     const float* __restrict__ hn, const float* __restrict__ cn) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t nf = facts ? B * H : 0, ns = shc ? B : 0;
  if (i < nf) {
    const int64_t b = i / H, d = slot ? slot[b] : b, rr = round ? round[b] : r;
    facts[(d * R + rr) * H + i % H] = h3[i];
    return;
  }
  i -= nf;
  if (i < ns) {
    const int64_t d = slot ? slot[i] : i, rr = round ? round[i] : r;
    shc[d * R + rr] = sh[i];
    return;
  }
  i -= ns;
  if (st_h && i < 2 * B * H) {
    const bool is_c = i >= B * H;
    const int64_t e = is_c ? i - B * H : i, b = e / H, d = slot ? slot[b] : b;
    (is_c ? st_c : st_h)[d * H + e % H] = (is_c ? cn : hn)[e];
  }
}

// a dialog pool's ask gather (dialog_gather in kernels.cuh): blockIdx.y picks the piece, threads stride over its elements
__global__ void k_dialog_gather(DialogGather g) {
  const int64_t n = g.n, stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  switch (blockIdx.y) {
    case 0:                                                    // questions: the cache row, and time-major ids
      for (int64_t i = i0; i < n * g.Tq; i += stride) {
        const int64_t b = i / g.Tq, t = i % g.Tq;
        const int32_t v = g.q[i];
        g.ques[((int64_t)g.slot[b] * g.R + g.round[b]) * g.Tq + t] = v;
        g.ids_q[t * n + b] = v;
      }
      break;
    case 1:                                                    // history row round[b] of slot[b], time-major
      if (g.ids_h)
        for (int64_t i = i0; i < n * g.W; i += stride) {
          const int64_t b = i / g.W, t = i % g.W;
          g.ids_h[t * n + b] = g.hist[((int64_t)g.slot[b] * g.R + g.round[b]) * g.W + t];
        }
      break;
    case 2:                                                    // the slot's image product
      if (g.img_out)
        for (int64_t i = i0; i < n * g.img_cols; i += stride) {
          const int64_t b = i / g.img_cols;
          g.img_out[i] = g.img[(int64_t)g.slot[b] * g.img_cols + i % g.img_cols];
        }
      break;
    default:                                                   // the dialog-LSTM state; zeros for a conversation's round 0
      if (g.h_out)
        for (int64_t i = i0; i < n * g.H; i += stride) {
          const int64_t b = i / g.H, src = (int64_t)g.slot[b] * g.H + i % g.H;
          const bool first = g.round[b] == 0;
          g.h_out[i] = first ? 0.f : g.h[src];
          g.c_out[i] = first ? 0.f : g.c[src];
        }
      break;
  }
}

__global__ void k_scatter_rows(float* __restrict__ dst, const float* __restrict__ src, const int32_t* __restrict__ slot,
                               int64_t n, int64_t cols) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n * cols) dst[(int64_t)slot[i / cols] * cols + i % cols] = src[i];
}

__global__ void k_hrea_att_bwd(const float* __restrict__ Hs, const float* __restrict__ probs, const float* __restrict__ datt,
                               float* __restrict__ dsq, float* __restrict__ dsh, float* __restrict__ dHs, int R, int H) {
  extern __shared__ float sm[];
  float* shh = sm; float* sd = shh + R * H; float* P = sd + R * H; float* dS = P + R * R;
  const int b = blockIdx.x, tid = threadIdx.x, nw = blockDim.x >> 5, w = tid >> 5, l = tid & 31;
  for (int i = tid; i < R * H; i += blockDim.x) { shh[i] = Hs[(int64_t)b * R * H + i]; sd[i] = datt[(int64_t)b * R * H + i]; }
  for (int i = tid; i < R * R; i += blockDim.x) P[i] = probs[(int64_t)b * R * R + i];
  __syncthreads();
  for (int p = w; p < R * R; p += nw) {
    int i = p / R, j = p % R;
    float acc = 0.f;
    for (int c = l; c < H; c += 32) acc += sd[i * H + c] * shh[j * H + c];
    acc = warp_sum(acc);
    if (l == 0) dS[p] = acc;
  }
  __syncthreads();
  if (tid < R) {
    float dot = 0.f;
    for (int j = 0; j < R; ++j) dot += P[tid * R + j] * dS[tid * R + j];
    float rs = 0.f;
    for (int j = 0; j < R; ++j) { float v = P[tid * R + j] * (dS[tid * R + j] - dot); dS[tid * R + j] = v; rs += v; }
    dsq[b * R + tid] = rs;
  }
  __syncthreads();
  if (tid < R) {
    float cs = 0.f;
    for (int i = 0; i < R; ++i) cs += dS[i * R + tid];
    dsh[b * R + tid] = cs;
  }
  for (int o = tid; o < R * H; o += blockDim.x) {
    int j = o / H, c = o % H;
    float acc = 0.f;
    for (int i = 0; i < R; ++i) acc += P[i * R + j] * sd[i * H + c];
    dHs[(int64_t)b * R * H + o] = acc;
  }
}

__global__ void k_masktime_concat_fwd(float* __restrict__ out, const float* __restrict__ wemb, const float* __restrict__ img,
                                      const int32_t* __restrict__ ids, int64_t TN, int64_t N, int E, int I) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int W = E + I;
  if (i >= TN * W) return;
  int64_t row = i / W; int c = (int)(i % W);
  float v;
  if (c < E) v = wemb[row * E + c];
  else v = ids[row] != 0 ? img[(row % N) * I + (c - E)] : 0.f;     // MaskTime.lua:21-26
  out[i] = v;
}
__global__ void k_masktime_bwd(const float* __restrict__ dx, int64_t ldx, int off, const int32_t* __restrict__ ids,
                               float* __restrict__ dimg, int T, int64_t N, int I) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * I) return;
  int64_t n = i / I; int c = (int)(i % I);
  float acc = 0.f;
  for (int t = 0; t < T; ++t)
    if (ids[(int64_t)t * N + n] != 0) acc += dx[((int64_t)t * N + n) * ldx + off + c];   // MaskTime.lua:35-37
  dimg[i] = acc;
}

// ------------------------------------------------------------------------------------------------
// SAN
__global__ void k_san_expand_dropout(float* __restrict__ img_tr, const float* __restrict__ t, int64_t total4, int R,
                                     int64_t PH4, DropCfg d, uint32_t site) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;     // float4 index into (N,P,H)
  if (i >= total4) return;
  int64_t n = i / PH4, rem = i % PH4;
  float4 v = reinterpret_cast<const float4*>(t)[(n / R) * PH4 + rem];
  float f[4];
  drop_factor4(d, site, (uint64_t)i, f);
  v.x *= f[0]; v.y *= f[1]; v.z *= f[2]; v.w *= f[3];
  reinterpret_cast<float4*>(img_tr)[i] = v;
}

// tanh for the two score kernels (65 M evaluations per pass at the benched size): exp-based, absolute error ~1e-7
__device__ __forceinline__ float tanh_e(float x) {
  const float e = __expf(-2.f * fabsf(x));
  return copysignf(__fdividef(1.f - e, 1.f + e), x);
}
// Region features (DESIGN §26): with MASK, row n of the SAN kernels below attends over positions 0 .. cnt[n / R] - 1 only.
// Positions at or past the count are never loaded; their outputs (score, probability, ds, dic, dimg_tr, dt_pre) are written as
// zeros.  The count arguments come last so that the MASK = false instantiations keep the parameter offsets they had.

// warp per (n,p)
template <bool MASK>
__global__ void k_san_score_fwd(const float* __restrict__ ic, const float* __restrict__ qc, const float* __restrict__ w,
                                const float* __restrict__ b, float* __restrict__ s, int64_t NP, int P, int Cm, DropCfg d, uint32_t site,
                                const int32_t* __restrict__ cnt, int R) {
  int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  int l = threadIdx.x & 31;
  if (row >= NP) return;
  int64_t n = row / P;
  if (MASK && (int)(row - n * P) >= cnt[n / R]) {
    if (l == 0) s[row] = 0.f;
    return;
  }
  float acc = 0.f;
  for (int c4 = l; c4 < (Cm >> 2); c4 += 32) {
    float4 a = reinterpret_cast<const float4*>(ic + row * Cm)[c4];
    float4 q = reinterpret_cast<const float4*>(qc + n * Cm)[c4];
    float4 ww = reinterpret_cast<const float4*>(w)[c4];
    float f[4];
    drop_factor4(d, site, (uint64_t)(row * (Cm >> 2) + c4), f);
    acc += ww.x * f[0] * tanh_e(a.x + q.x) + ww.y * f[1] * tanh_e(a.y + q.y) + ww.z * f[2] * tanh_e(a.z + q.z) +
           ww.w * f[3] * tanh_e(a.w + q.w);
  }
  acc = warp_sum(acc);
  if (l == 0) s[row] = acc + b[0];
}

// The four kernels below stream (N, P, H) / (N, P, Cm) tensors (128 MB each at the benched size) once: they are HBM-bound, so every
// thread moves float4 pieces, keeps 4 independent loads in flight, and a dialog round's work is spread over several blocks.

// grid (N, 2 halves of H), block 256: softmax over the P scores (recomputed per half: P is 196), then u_out = p . img_tr + u_in for the
// half's columns — thread = float4 column piece x position group, groups combined in shared memory
template <bool MASK>
__global__ void __launch_bounds__(256) k_san_softmax_att_fwd(const float* __restrict__ s, float* __restrict__ p, const float* __restrict__ img_tr,
                                                             const float* __restrict__ u_in, float* __restrict__ u_out, int P, int H,
                                                             const int32_t* __restrict__ cnt, int R) {
  extern __shared__ float sm[];          // P floats + 33 + 256 float4
  float* sp = sm; float* red = sm + P;
  float4* part = reinterpret_cast<float4*>(sm + ((P + 33 + 3) & ~3));
  const int64_t n = blockIdx.x;
  const int c = MASK ? cnt[n / R] : P;   // positions attended
  float mx = -INFINITY;
  for (int i = threadIdx.x; i < c; i += blockDim.x) { float v = s[n * P + i]; sp[i] = v; mx = fmaxf(mx, v); }
  mx = block_max(mx, red);
  float sum = 0.f;
  for (int i = threadIdx.x; i < c; i += blockDim.x) { float e = expf(sp[i] - mx); sp[i] = e; sum += e; }
  sum = block_sum(sum, red);
  for (int i = threadIdx.x; i < c; i += blockDim.x) { float v = sp[i] / sum; sp[i] = v; if (blockIdx.y == 0) p[n * P + i] = v; }
  if (MASK && blockIdx.y == 0)
    for (int i = c + threadIdx.x; i < P; i += blockDim.x) p[n * P + i] = 0.f;
  __syncthreads();
  const int H4 = H >> 2, half = (H4 + 1) >> 1;
  const int c_lo = blockIdx.y * half, c_hi = min(H4, c_lo + half);
  const int tpc = min(half, (int)blockDim.x), npg = blockDim.x / tpc;
  const int tc = threadIdx.x % tpc, pg = threadIdx.x / tpc;
  const float4* base = reinterpret_cast<const float4*>(img_tr) + n * P * H4;
  for (int c0 = c_lo; c0 < c_hi; c0 += tpc) {
    const int c4 = c0 + tc;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (pg < npg && c4 < c_hi) {
      int i = pg;
      for (; i + 3 * npg < c; i += 4 * npg) {
        const float4 a = base[(int64_t)i * H4 + c4], b = base[(int64_t)(i + npg) * H4 + c4];
        const float4 g = base[(int64_t)(i + 2 * npg) * H4 + c4], e = base[(int64_t)(i + 3 * npg) * H4 + c4];
        const float w0 = sp[i], w1 = sp[i + npg], w2 = sp[i + 2 * npg], w3 = sp[i + 3 * npg];
        acc.x += w0 * a.x + w1 * b.x + w2 * g.x + w3 * e.x; acc.y += w0 * a.y + w1 * b.y + w2 * g.y + w3 * e.y;
        acc.z += w0 * a.z + w1 * b.z + w2 * g.z + w3 * e.z; acc.w += w0 * a.w + w1 * b.w + w2 * g.w + w3 * e.w;
      }
      for (; i < c; i += npg) {
        const float4 a = base[(int64_t)i * H4 + c4]; const float w0 = sp[i];
        acc.x += w0 * a.x; acc.y += w0 * a.y; acc.z += w0 * a.z; acc.w += w0 * a.w;
      }
    }
    part[threadIdx.x] = acc;
    __syncthreads();
    if (pg == 0 && c4 < c_hi) {
      for (int g = 1; g < npg; ++g) { const float4 o = part[g * tpc + tc]; acc.x += o.x; acc.y += o.y; acc.z += o.z; acc.w += o.w; }
      const float4 u = reinterpret_cast<const float4*>(u_in)[n * H4 + c4];
      reinterpret_cast<float4*>(u_out)[n * H4 + c4] = make_float4(acc.x + u.x, acc.y + u.y, acc.z + u.z, acc.w + u.w);
    }
    __syncthreads();
  }
}

// block per n (512 threads): dp = du . img_tr ; ds = p*(dp - sum p dp) ; dimg_tr = p * du
template <bool MASK>
__global__ void __launch_bounds__(512) k_san_att_bwd(const float* __restrict__ du, const float* __restrict__ p, const float* __restrict__ img_tr,
                                                     float* __restrict__ ds, float* __restrict__ dimg_tr, int P, int H,
                                                     const int32_t* __restrict__ cnt, int R) {
  extern __shared__ float sm[];          // H + P + P + 33
  float* sdu = sm; float* sp = sdu + H; float* sdp = sp + P; float* red = sdp + P;
  const int64_t n = blockIdx.x;
  const int tid = threadIdx.x, nw = blockDim.x >> 5, w = tid >> 5, l = tid & 31;
  const int H4 = H >> 2;
  const int cn = MASK ? cnt[n / R] : P;  // positions attended
  for (int c = tid; c < H; c += blockDim.x) sdu[c] = du[n * H + c];
  for (int i = tid; i < cn; i += blockDim.x) sp[i] = p[n * P + i];
  __syncthreads();
  const float4* sdu4 = reinterpret_cast<const float4*>(sdu);
  for (int i = w; i < cn; i += nw) {
    const float4* row = reinterpret_cast<const float4*>(img_tr) + (n * P + i) * H4;
    float acc = 0.f;
#pragma unroll 4
    for (int c = l; c < H4; c += 32) { const float4 a = row[c], b = sdu4[c]; acc += a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w; }
    acc = warp_sum(acc);
    if (l == 0) sdp[i] = acc;
  }
  __syncthreads();
  float part = 0.f;
  for (int i = tid; i < cn; i += blockDim.x) part += sp[i] * sdp[i];
  float dot = block_sum(part, red);
  for (int i = tid; i < cn; i += blockDim.x) ds[n * P + i] = sp[i] * (sdp[i] - dot);
  if (MASK)
    for (int i = cn + tid; i < P; i += blockDim.x) ds[n * P + i] = 0.f;
  float4* out = reinterpret_cast<float4*>(dimg_tr) + n * P * H4;
  for (int i = w; i < P; i += nw) {
    if (MASK && i >= cn) {
      for (int c = l; c < H4; c += 32) out[(int64_t)i * H4 + c] = make_float4(0.f, 0.f, 0.f, 0.f);
      continue;
    }
    const float pi = sp[i];
    for (int c = l; c < H4; c += 32) { const float4 b = sdu4[c]; out[(int64_t)i * H4 + c] = make_float4(pi * b.x, pi * b.y, pi * b.z, pi * b.w); }
  }
}

// grid (N, column slices), block 256: thread = float4 column piece x position group; a block walks ALL P positions of its columns, the
// position groups are combined in shared memory in a fixed order, so dqc — an intermediate gradient that flows on into the encoder — is
// written once and deterministically (only the leaf gradients dw, db use atomics).  Recomputes y = tanh(ic + qc) and the dropout factor.
// SLOT (deterministic mode): row n's dw / db sums go to row n of dw (N, Cm) / element n of db (N), for slot_reduce.
template <bool MASK, bool SLOT>
__global__ void __launch_bounds__(256) k_san_score_bwd(const float* __restrict__ ds, const float* __restrict__ ic, const float* __restrict__ qc,
                                                       const float* __restrict__ w, float* __restrict__ dic, float* __restrict__ dqc,
                                                       float* __restrict__ dw, float* __restrict__ db, int P, int Cm, DropCfg d, uint32_t site,
                                                       const int32_t* __restrict__ cnt, int R) {
  extern __shared__ float sm[];          // P floats (ds row), then 2 x 256 float4
  float4* part_q = reinterpret_cast<float4*>(sm + ((P + 3) & ~3));
  float4* part_w = part_q + 256;
  const int64_t n = blockIdx.x;
  const int cn = MASK ? cnt[n / R] : P;  // positions attended
  for (int i = threadIdx.x; i < cn; i += blockDim.x) sm[i] = ds[n * P + i];
  __syncthreads();
  const int C4 = Cm >> 2, per = (C4 + gridDim.y - 1) / gridDim.y;
  const int c_lo = blockIdx.y * per, c_hi = min(C4, c_lo + per);
  const int tpc = max(1, min(per, (int)blockDim.x)), npg = blockDim.x / tpc;
  const int tc = threadIdx.x % tpc, pg = threadIdx.x / tpc;
  const float4* ic4 = reinterpret_cast<const float4*>(ic);
  float4* dic4 = reinterpret_cast<float4*>(dic);
  for (int c0 = c_lo; c0 < c_hi; c0 += tpc) {
    const int c4 = c0 + tc;
    float4 aq = make_float4(0.f, 0.f, 0.f, 0.f), aw = aq;
    if (pg < npg && c4 < c_hi) {
      const float4 q = reinterpret_cast<const float4*>(qc)[n * C4 + c4], wc = reinterpret_cast<const float4*>(w)[c4];
#pragma unroll 4
      for (int i = pg; i < cn; i += npg) {
        const int64_t idx4 = (n * P + i) * C4 + c4;
        const float4 a = ic4[idx4];
        float f[4];
        drop_factor4(d, site, (uint64_t)idx4, f);
        const float g = sm[i];
        const float y0 = tanh_e(a.x + q.x), y1 = tanh_e(a.y + q.y), y2 = tanh_e(a.z + q.z), y3 = tanh_e(a.w + q.w);
        const float g0 = g * f[0], g1 = g * f[1], g2 = g * f[2], g3 = g * f[3];
        const float4 o = make_float4(g0 * wc.x * (1.f - y0 * y0), g1 * wc.y * (1.f - y1 * y1), g2 * wc.z * (1.f - y2 * y2), g3 * wc.w * (1.f - y3 * y3));
        dic4[idx4] = o;
        aq.x += o.x; aq.y += o.y; aq.z += o.z; aq.w += o.w;
        aw.x += g0 * y0; aw.y += g1 * y1; aw.z += g2 * y2; aw.w += g3 * y3;
      }
      if (MASK)
        for (int i = cn + pg; i < P; i += npg) dic4[(n * P + i) * C4 + c4] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    part_q[threadIdx.x] = aq; part_w[threadIdx.x] = aw;
    __syncthreads();
    if (pg == 0 && c4 < c_hi) {
      for (int g = 1; g < npg; ++g) {
        const float4 oq = part_q[g * tpc + tc], ow = part_w[g * tpc + tc];
        aq.x += oq.x; aq.y += oq.y; aq.z += oq.z; aq.w += oq.w;
        aw.x += ow.x; aw.y += ow.y; aw.z += ow.z; aw.w += ow.w;
      }
      reinterpret_cast<float4*>(dqc)[n * C4 + c4] = aq;
      if constexpr (SLOT) reinterpret_cast<float4*>(dw)[n * C4 + c4] = aw;
      else { atomicAdd(dw + 4 * c4, aw.x); atomicAdd(dw + 4 * c4 + 1, aw.y); atomicAdd(dw + 4 * c4 + 2, aw.z); atomicAdd(dw + 4 * c4 + 3, aw.w); }
    }
    __syncthreads();
  }
  // db: the scores of a row enter a softmax, so sum_i ds[n, i] is zero up to rounding — summed in a fixed order by one thread
  if (blockIdx.y == 0 && threadIdx.x == 0) {
    float acc = 0.f;
    for (int i = 0; i < cn; ++i) acc += sm[i];
    if constexpr (SLOT) db[n] = acc;
    else atomicAdd(db, acc);
  }
}

// thread = float4 of (B,P,H): sum over the R rounds that share the image (dropout factor recomputed), times tanh'.  With
// MASK, dialog b's positions at or past cnt[b] (H4 float4 per position) are written as zeros.
template <bool MASK>
__global__ void k_san_collapse_bwd(const float* __restrict__ dimg_tr, const float* __restrict__ t, float* __restrict__ dt_pre,
                                   int64_t total4, int R, int64_t PH4, DropCfg d, uint32_t site, const int32_t* __restrict__ cnt,
                                   int64_t H4) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;    // float4 index into (B,P,H)
  if (i >= total4) return;
  int64_t b = i / PH4, rem = i % PH4;
  if (MASK && rem / H4 >= cnt[b]) {
    reinterpret_cast<float4*>(dt_pre)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    return;
  }
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 5
  for (int r = 0; r < R; ++r) {
    const int64_t idx4 = (b * R + r) * PH4 + rem;
    const float4 v = reinterpret_cast<const float4*>(dimg_tr)[idx4];
    float f[4];
    drop_factor4(d, site, (uint64_t)idx4, f);
    acc.x += v.x * f[0]; acc.y += v.y * f[1]; acc.z += v.z * f[2]; acc.w += v.w * f[3];
  }
  const float4 tv = reinterpret_cast<const float4*>(t)[i];
  reinterpret_cast<float4*>(dt_pre)[i] = make_float4(acc.x * (1.f - tv.x * tv.x), acc.y * (1.f - tv.y * tv.y), acc.z * (1.f - tv.z * tv.z),
                                                     acc.w * (1.f - tv.w * tv.w));
}

// ------------------------------------------------------------------------------------------------
// warp per (n,k)
__global__ void k_disc_scores_fwd(const float* __restrict__ feat, const float* __restrict__ enc, float* __restrict__ scores,
                                  int64_t NK, int K, int H) {
  int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  int l = threadIdx.x & 31;
  if (row >= NK) return;
  const float4* f = reinterpret_cast<const float4*>(feat + row * H);
  const float4* e = reinterpret_cast<const float4*>(enc + (row / K) * H);
  float acc = 0.f;
  for (int c = l; c < (H >> 2); c += 32) {
    float4 a = f[c], b = e[c];
    acc += a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w;
  }
  acc = warp_sum(acc);
  if (l == 0) scores[row] = acc;
}
// block per n
__global__ void k_disc_scores_bwd(const float* __restrict__ dscores, const float* __restrict__ feat, const float* __restrict__ enc,
                                  float* __restrict__ dfeat, float* __restrict__ denc, int K, int H) {
  extern __shared__ float sm[];   // K floats
  const int64_t n = blockIdx.x;
  for (int k = threadIdx.x; k < K; k += blockDim.x) sm[k] = dscores[n * K + k];
  __syncthreads();
  for (int c = threadIdx.x; c < H; c += blockDim.x) {
    float e = enc[n * H + c], acc = 0.f;
    for (int k = 0; k < K; ++k) {
      int64_t idx = (n * K + k) * H + c;
      acc += sm[k] * feat[idx];
      dfeat[idx] = sm[k] * e;
    }
    denc[n * H + c] = acc;
  }
}

// block per row (blockDim >= 32)
__global__ void k_xent_fwd(const float* __restrict__ scores, const int32_t* __restrict__ gt, float* __restrict__ row_loss, int K) {
  __shared__ float red[33];
  const int64_t n = blockIdx.x;
  float mx = -INFINITY;
  for (int k = threadIdx.x; k < K; k += blockDim.x) mx = fmaxf(mx, scores[n * K + k]);
  mx = block_max(mx, red);
  float sum = 0.f;
  for (int k = threadIdx.x; k < K; k += blockDim.x) sum += expf(scores[n * K + k] - mx);
  sum = block_sum(sum, red);
  if (threadIdx.x == 0) row_loss[n] = -(scores[n * K + gt[n] - 1] - mx - logf(sum));
}
__global__ void k_xent_bwd(const float* __restrict__ scores, const int32_t* __restrict__ gt, float* __restrict__ dscores,
                           int K, float inv_n) {
  __shared__ float red[33];
  const int64_t n = blockIdx.x;
  float mx = -INFINITY;
  for (int k = threadIdx.x; k < K; k += blockDim.x) mx = fmaxf(mx, scores[n * K + k]);
  mx = block_max(mx, red);
  float sum = 0.f;
  for (int k = threadIdx.x; k < K; k += blockDim.x) sum += expf(scores[n * K + k] - mx);
  sum = block_sum(sum, red);
  int g = gt[n] - 1;
  for (int k = threadIdx.x; k < K; k += blockDim.x)
    dscores[n * K + k] = (expf(scores[n * K + k] - mx) / sum - (k == g ? 1.f : 0.f)) * inv_n;
}
// block per row, soft targets p = rel / sum(rel): row_loss = lse(s) - sum_k p_k s_k, dscores = (softmax(s) - p) * inv_n.
// Block reductions in a fixed order (no atomics): fp32 runs repeat bit for bit.
__global__ void k_soft_xent(const float* __restrict__ scores, const float* __restrict__ rel, float* __restrict__ row_loss,
                            float* __restrict__ dscores, int K, float inv_n) {
  __shared__ float red[33];
  const int64_t n = blockIdx.x;
  const float* s = scores + n * K;
  const float* r = rel + n * K;
  float mx = -INFINITY, rs = 0.f;
  for (int k = threadIdx.x; k < K; k += blockDim.x) { mx = fmaxf(mx, s[k]); rs += r[k]; }
  mx = block_max(mx, red);
  rs = block_sum(rs, red);
  float sum = 0.f, dot = 0.f;
  for (int k = threadIdx.x; k < K; k += blockDim.x) { sum += expf(s[k] - mx); dot += r[k] * s[k]; }
  sum = block_sum(sum, red);
  dot = block_sum(dot, red);
  const float inv_rs = 1.f / rs;
  if (threadIdx.x == 0) row_loss[n] = mx + logf(sum) - dot * inv_rs;
  for (int k = threadIdx.x; k < K; k += blockDim.x) dscores[n * K + k] = (expf(s[k] - mx) / sum - r[k] * inv_rs) * inv_n;
}
__global__ void k_reduce_sum(const float* __restrict__ x, float* __restrict__ out, int64_t n, float scale) {
  __shared__ float red[33];
  float acc = 0.f;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) acc += x[i];
  acc = block_sum(acc, red);
  if (threadIdx.x == 0) out[0] = acc * scale;
}

// block per row; thread k counts the options that beat option k
__global__ void k_rank_rows(const float* __restrict__ scores, const int32_t* __restrict__ gt, int32_t* __restrict__ ranks, int K) {
  extern __shared__ float sm[];
  const int64_t n = blockIdx.x;
  for (int k = threadIdx.x; k < K; k += blockDim.x) sm[k] = scores[n * K + k];
  __syncthreads();
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    float s = sm[k];
    int cnt = 0;
    for (int j = 0; j < K; ++j) { float t = sm[j]; cnt += (t > s) || (t == s && j < k); }
    if (gt) { if (k == gt[n] - 1) ranks[n] = cnt + 1; }
    else ranks[n * K + k] = cnt + 1;
  }
}

// log-sum-exp of one row, by the whole block.  k_logsoftmax_rows and k_logsoftmax_topk_rows both take their lse from here
// (same strided loops, same block reductions), so the log-probabilities x - lse they form are the same bits.
__device__ __forceinline__ float row_lse(const float* row, int V, float* red) {
  float mx = -INFINITY;
  for (int c = threadIdx.x; c < V; c += blockDim.x) mx = fmaxf(mx, row[c]);
  mx = block_max(mx, red);
  float sum = 0.f;
  for (int c = threadIdx.x; c < V; c += blockDim.x) sum += expf(row[c] - mx);
  sum = block_sum(sum, red);
  return mx + logf(sum);
}

// block per row
__global__ void k_logsoftmax_rows(float* __restrict__ x, const int32_t* __restrict__ mask_ids, int V) {
  __shared__ float red[33];
  const int64_t r = blockIdx.x;
  float* row = x + r * V;
  if (mask_ids && mask_ids[r] == 0) {
    for (int c = threadIdx.x; c < V; c += blockDim.x) row[c] = 0.f;
    return;
  }
  const float lse = row_lse(row, V, red);
  for (int c = threadIdx.x; c < V; c += blockDim.x) row[c] -= lse;
}

// ---- answer rules (common.cuh's AnswerRules, DESIGN §25) ------------------------------------------------------------
__device__ __forceinline__ bool is_barred(const uint32_t* bar, int c) { return (bar[c >> 5] >> (c & 31)) & 1u; }
__device__ __forceinline__ void set_barred(uint32_t* bar, int c) { atomicOr(&bar[c >> 5], 1u << (c & 31)); }

// Row r's barred set as a V-bit mask in shared memory (bit c: class c, token c + 1), built by the whole block: banned ids,
// <END> while stp <= min_words, the n-gram scan (start j = 1 .. stp-n per thread, n - 1 compares each), the fallback.
// Returns the number of allowed classes (>= 1) on every thread.  red: block_sum's 33 floats (exact: counts < 2^24).
__device__ __forceinline__ int build_barred(const AnswerRules& ar, int64_t r, int V, uint32_t* bar, float* red) {
  const int nw = (V + 31) >> 5, stp = ar.step, n = ar.no_repeat_ngram;
  for (int i = threadIdx.x; i < nw; i += blockDim.x) bar[i] = 0u;
  __syncthreads();
  for (int i = threadIdx.x; i < ar.n_banned; i += blockDim.x) set_barred(bar, ar.banned[i] - 1);
  if (threadIdx.x == 0 && stp <= ar.min_words) set_barred(bar, ar.end_token - 1);
  if (n > 0) {
    const int32_t* t = ar.hist + r * ar.ld;
    for (int j = 1 + (int)threadIdx.x; j <= stp - n; j += blockDim.x) {
      bool match = true;
      for (int i = 0; i < n - 1 && match; ++i) {
        const int32_t a = t[j + i];
        match = a != 0 && a == t[stp - n + 1 + i];
      }
      const int32_t w = t[j + n - 1];
      if (match && w != ar.end_token && (unsigned)(w - 1) < (unsigned)V) set_barred(bar, w - 1);
    }
  }
  __syncthreads();
  int cnt = 0;
  for (int i = threadIdx.x; i < nw; i += blockDim.x) cnt += __popc(bar[i]);
  const int allowed = V - (int)block_sum((float)cnt, red);
  if (allowed > 0) return allowed;
  if (threadIdx.x == 0) { const int c = ar.end_token - 1; bar[c >> 5] &= ~(1u << (c & 31)); }   // the fallback
  __syncthreads();
  return 1;
}

// (v, c) precedes (w, d) in torch.topk's order with the pinned tie rule: value descending, class ascending
__device__ __forceinline__ bool topk_before(float v, int c, float w, int d) { return v > w || (v == w && c < d); }

// The k best log-probabilities of every row and their classes, in torch.topk(sorted)'s order with the pinned tie rule
// (value descending, class ascending), without writing the (rows, V) log-probabilities: the logits are read three times
// whatever k is.  The lse comes from row_lse, so each x - lse is the value k_logsoftmax_rows would write, bit for bit.
// Each thread keeps the KMAX best (x - lse, class) pairs of its strided columns, sorted, in registers; the block then pops
// k winners from the thread heads.  A row whose mask id is 0 is all zeros in k_logsoftmax_rows (MaskZero): its top k is
// classes 0..k-1 with value 0.
// RULES: the answer rules' barred classes (ar, DESIGN §25) take no part; the list is the k best allowed classes, its entries
// past the allowed count (-inf, -1), and a pad row lists the first k allowed classes with value 0.
template <int KMAX, bool RULES>
__global__ void __launch_bounds__(256) k_logsoftmax_topk_rows(const float* __restrict__ x, const int32_t* __restrict__ mask_ids,
                                                              int V, int k, float* __restrict__ topv, int32_t* __restrict__ topi,
                                                              AnswerRules ar) {
  __shared__ float red[33];
  __shared__ float sv[8];
  __shared__ int si[8];
  __shared__ int win;
  __shared__ uint32_t bar[RULES ? RULES_MASK_WORDS : 1];
  const int64_t r = blockIdx.x;
  if (mask_ids && mask_ids[r] == 0) {
    if constexpr (RULES) {
      build_barred(ar, r, V, bar, red);
      if (threadIdx.x == 0) {
        int j = 0;
        for (int w = 0; w * 32 < V && j < k; ++w) {
          uint32_t f = ~bar[w] & (V - w * 32 >= 32 ? 0xffffffffu : (1u << (V - w * 32)) - 1u);   // allowed classes
          for (; f && j < k; f &= f - 1, ++j) { topv[r * k + j] = 0.f; topi[r * k + j] = w * 32 + __ffs(f) - 1; }
        }
        for (; j < k; ++j) { topv[r * k + j] = -INFINITY; topi[r * k + j] = -1; }
      }
    } else {
      for (int j = threadIdx.x; j < k; j += blockDim.x) { topv[r * k + j] = 0.f; topi[r * k + j] = j; }
    }
    return;
  }
  const float* row = x + r * V;
  const float lse = row_lse(row, V, red);
  if constexpr (RULES) build_barred(ar, r, V, bar, red);
  float lv[KMAX]; int lc[KMAX];
#pragma unroll
  for (int i = 0; i < KMAX; ++i) { lv[i] = -INFINITY; lc[i] = 0x7fffffff; }
  for (int c = threadIdx.x; c < V; c += blockDim.x) {
    if (RULES && is_barred(bar, c)) continue;
    float v = row[c] - lse;
    if (!topk_before(v, c, lv[KMAX - 1], lc[KMAX - 1])) continue;
    int ci = c;
#pragma unroll
    for (int i = 0; i < KMAX; ++i) {         // insertion: (v, ci) displaces every later entry by one
      if (topk_before(v, ci, lv[i], lc[i])) {
        const float tv = lv[i]; const int tc = lc[i];
        lv[i] = v; lc[i] = ci; v = tv; ci = tc;
      }
    }
  }
  for (int j = 0; j < k; ++j) {
    float bv = lv[0]; int bi = lc[0];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(FULL, bv, o);
      const int oi = __shfl_xor_sync(FULL, bi, o);
      if (topk_before(ov, oi, bv, bi)) { bv = ov; bi = oi; }
    }
    if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = bv; si[threadIdx.x >> 5] = bi; }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 1; w < (int)(blockDim.x >> 5); ++w)
        if (topk_before(sv[w], si[w], bv, bi)) { bv = sv[w]; bi = si[w]; }
      const bool none = RULES && bi == 0x7fffffff;           // fewer than k allowed classes
      topv[r * k + j] = none ? -INFINITY : bv; topi[r * k + j] = none ? -1 : bi;
      win = bi;
    }
    __syncthreads();
    if (lc[0] == win) {                        // the owner of the winning column pops its head
#pragma unroll
      for (int i = 0; i < KMAX - 1; ++i) { lv[i] = lv[i + 1]; lc[i] = lc[i + 1]; }
      lv[KMAX - 1] = -INFINITY; lc[KMAX - 1] = 0x7fffffff;
    }
    __syncthreads();
  }
}

// The Gumbel-max draw of common.cuh over row r's classes, by the whole block: y_of(j, y) gives class j's y = x_j / T and
// says whether j takes part.  Each thread takes Philox quadruples (4 consecutive element indices, one call) strided over
// the row, keeps its best (key, class), and the block reduces them with the same order.  The winning class is returned on
// thread 0.
template <typename Y>
__device__ __forceinline__ int row_gumbel_argmax(const SampleCfg& smp, int64_t r, int V, Y y_of, float* sk, int* sc) {
  const uint64_t base = (uint64_t)sample_round(smp, r) * (uint64_t)V;
  const uint64_t q0 = base >> 2, q1 = (base + V - 1) >> 2;
  float bk = -INFINITY;
  int bc = 0x7fffffff;
  for (uint64_t q = q0 + threadIdx.x; q <= q1; q += blockDim.x) {
    const int64_t j0 = (int64_t)(q * 4 - base);                 // class of word 0 (< 0 or >= V outside the row)
    float y[4];
    bool in[4];
    float ymax = -INFINITY;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int64_t j = j0 + e;
      in[e] = j >= 0 && j < V && y_of((int)j, y[e]);
      if (!in[e]) y[e] = -INFINITY;
      ymax = fmaxf(ymax, y[e]);
    }
    if (ymax + GUMBEL_MAX < bk) continue;                        // no key of the quadruple can reach the best one
    uint32_t o[4];
    sample_words(smp, q, o);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      if (!in[e]) continue;
      const int j = (int)(j0 + e);
      const float key = y[e] + gumbel_of_word(o[e]);
      if (sample_before(key, j, bk, bc)) { bk = key; bc = j; }
    }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    const float ok = __shfl_xor_sync(FULL, bk, off);
    const int oc = __shfl_xor_sync(FULL, bc, off);
    if (sample_before(ok, oc, bk, bc)) { bk = ok; bc = oc; }
  }
  if ((threadIdx.x & 31) == 0) { sk[threadIdx.x >> 5] = bk; sc[threadIdx.x >> 5] = bc; }
  __syncthreads();
  if (threadIdx.x == 0)
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w)
      if (sample_before(sk[w], sc[w], bk, bc)) { bk = sk[w]; bc = sc[w]; }
  return bc;
}

// The sampling step from materialised logits, one block per row.  The lse comes from row_lse, so x_tok - lse is the
// log-probability k_logsoftmax_rows would write.  RULES: the answer rules' barred classes (ar, DESIGN §25) take no part in
// the draw; the allowed classes' keys are unchanged.
template <bool RULES>
__global__ void __launch_bounds__(256) k_logsoftmax_sample_rows(const float* __restrict__ x, int V, SampleCfg smp, int L,
                                                                int32_t* __restrict__ tokens, int32_t* __restrict__ answer,
                                                                float* __restrict__ logp, AnswerRules ar) {
  __shared__ float red[33];
  __shared__ float sk[8];
  __shared__ int sc[8];
  __shared__ uint32_t bar[RULES ? RULES_MASK_WORDS : 1];
  const int64_t r = blockIdx.x;
  const float* row = x + r * V;
  const float lse = row_lse(row, V, red);
  if constexpr (RULES) build_barred(ar, r, V, bar, red);
  const int bc = row_gumbel_argmax(smp, r, V, [&](int j, float& y) {
    y = row[j] / smp.temperature;
    return !RULES || !is_barred(bar, j);
  }, sk, sc);
  if (threadIdx.x == 0) {
    tokens[r] = bc + 1;
    answer[r * (L + 1) + smp.step] = bc + 1;
    if (logp) logp[r * L + smp.step - 1] = row[bc] - lse;
  }
}

// ---- truncated sampling (common.cuh's rule, DESIGN §23) ------------------------------------------------------------
// Order-preserving 32-bit key of y: key(a) > key(b) <=> a > b, with -0 and +0 one key (they are equal y).
__device__ __forceinline__ uint32_t trunc_key(float y) {
  const uint32_t u = __float_as_uint(y == 0.f ? 0.f : y);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float trunc_y(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }
// integer mass q = rint(expf(y - m) 2^32) (2^32 at the maximum; the scaling by 2^32 is exact)
__device__ __forceinline__ unsigned long long trunc_mass(float y, float m) { return __float2ull_rn(expf(y - m) * 0x1p32f); }

struct TruncShared {
  unsigned long long hist[8][256];   // per-warp radix histograms: logits crowd into a few high digits
  unsigned long long scan[8];
  unsigned long long sel_excl;
  uint32_t sel_digit;
  int sel_class;
  float red[33];
  float sk[8];
  int sc[8];
};

// inclusive prefix sum over the 256 threads in thread order; sh holds >= 8 T
template <typename T>
__device__ __forceinline__ T block_incl_scan(T v, T* sh) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T n = __shfl_up_sync(FULL, v, o);
    if (lane >= o) v += n;
  }
  __syncthreads();
  if (lane == 31) sh[w] = v;
  __syncthreads();
  for (int i = 0; i < w; ++i) v += sh[i];
  return v;
}

// Radix select over the staged y, 8 bits per pass from the top: the key t with W(key > t) < need <= W(key >= t), W the sum
// of weight(j, key) (0: j takes no part), and above = W(key > t).  need must be in [1, W(all)].
struct TruncSel { uint32_t key; unsigned long long above; };
template <typename Wt>
__device__ __forceinline__ TruncSel trunc_radix_select(const float* ys, int V, unsigned long long need, Wt weight, TruncShared& s) {
  const int w = threadIdx.x >> 5;
  uint32_t prefix = 0;
  unsigned long long acc = 0;
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = threadIdx.x; i < 8 * 256; i += blockDim.x) (&s.hist[0][0])[i] = 0;
    __syncthreads();
    const uint32_t hmask = shift == 24 ? 0u : 0xffffffffu << (shift + 8);
    for (int j = threadIdx.x; j < V; j += blockDim.x) {
      const uint32_t k = trunc_key(ys[j]);
      if ((k & hmask) != prefix) continue;
      const unsigned long long wt = weight(j, k);
      if (wt) atomicAdd(&s.hist[w][(k >> shift) & 255u], wt);
    }
    __syncthreads();
    const uint32_t d = 255u - threadIdx.x;                       // thread t: digit 255 - t, so the scan runs key-descending
    unsigned long long tot = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) tot += s.hist[i][d];
    const unsigned long long incl = block_incl_scan(tot, s.scan), rem = need - acc;
    if (incl - tot < rem && rem <= incl) { s.sel_digit = d; s.sel_excl = incl - tot; }
    __syncthreads();
    prefix |= s.sel_digit << shift;
    acc += s.sel_excl;
  }
  return {prefix, acc};
}

// the class of the n-th (1-based) class of key t in class order among the classes in(j) admits: each thread counts a
// contiguous chunk, a block scan finds the chunk, its thread walks it
template <typename In>
__device__ __forceinline__ int trunc_nth_of_key(const float* ys, int V, uint32_t t, uint32_t n, TruncShared& s, In in) {
  const int per = (V + blockDim.x - 1) / blockDim.x, b = threadIdx.x * per, e = min(V, b + per);
  uint32_t c = 0;
  for (int j = b; j < e; ++j) c += trunc_key(ys[j]) == t && in(j);
  const uint32_t incl = block_incl_scan(c, reinterpret_cast<uint32_t*>(s.scan));
  if (incl - c < n && n <= incl) {
    uint32_t seen = incl - c;
    for (int j = b; j < e; ++j)
      if (trunc_key(ys[j]) == t && in(j) && ++seen == n) { s.sel_class = j; break; }
  }
  __syncthreads();
  return s.sel_class;
}

// The truncated sampling step from materialised logits, one 256-thread block per row (so row_lse reduces in
// k_logsoftmax_rows' order and logp is its bits).  y = x / T is staged in dynamic shared memory (4 V bytes).  The kept
// classes are a prefix of (y desc, class asc), held as its last element (tk, tc): key > tk, or key == tk and class <= tc.
// top-k and top-p each find their boundary key by radix select (counts, then integer masses over the top-k prefix) and
// the boundary class among that key's ties by a block scan in class order; the draw is row_gumbel_argmax over the prefix.
// RULES: the answer rules' barred classes (ar, DESIGN §25) are out of the row before truncation: they count in neither
// top-k nor the masses, m is the allowed classes' maximum, and the draw skips them.  Their bit mask follows ys in the stage.
template <bool RULES>
__global__ void __launch_bounds__(256) k_truncated_sample_rows(const float* __restrict__ x, int V, SampleCfg smp, TruncCfg tr,
                                                               int L, int32_t* __restrict__ tokens, int32_t* __restrict__ answer,
                                                               float* __restrict__ logp, AnswerRules ar) {
  extern __shared__ float ys[];
  __shared__ TruncShared s;
  const int64_t r = blockIdx.x;
  const float* row = x + r * V;
  uint32_t* bar = reinterpret_cast<uint32_t*>(ys + V);
  int nal = V;                                                   // allowed classes
  if constexpr (RULES) nal = build_barred(ar, r, V, bar, s.red);
  const auto in = [&](int j) { return !RULES || !is_barred(bar, j); };
  float m = -INFINITY;
  for (int j = threadIdx.x; j < V; j += blockDim.x) {
    const float y = row[j] / smp.temperature;
    ys[j] = y;
    if (in(j)) m = fmaxf(m, y);
  }
  m = block_max(m, s.red);                                       // its barriers also publish ys
  uint32_t tk = 0;                                               // key 0 is below every y: all classes kept
  int tc = 0x7fffffff;
  if (tr.top_k >= 1 && tr.top_k < nal) {
    const TruncSel k = trunc_radix_select(ys, V, (unsigned long long)tr.top_k,
                                          [&](int j, uint32_t) { return in(j) ? 1ull : 0ull; }, s);
    tk = k.key;
    tc = trunc_nth_of_key(ys, V, tk, (uint32_t)(tr.top_k - k.above), s, in);
  }
  if (tr.top_p < 1.f) {
    const uint32_t k0 = tk;
    const int c0 = tc;
    auto mass = [&](int j, uint32_t k) { return (in(j) && (k > k0 || (k == k0 && j <= c0))) ? trunc_mass(ys[j], m) : 0ull; };
    unsigned long long S = 0;
    for (int j = threadIdx.x; j < V; j += blockDim.x) S += mass(j, trunc_key(ys[j]));
    S = block_incl_scan(S, s.scan);
    if (threadIdx.x == blockDim.x - 1) s.sel_excl = S;
    __syncthreads();
    S = s.sel_excl;
    const unsigned long long tau = (unsigned long long)ceil((double)tr.top_p * (double)S);
    const TruncSel p = trunc_radix_select(ys, V, tau, mass, s);
    tk = p.key;
    const unsigned long long qt = trunc_mass(trunc_y(tk), m);    // every tie of tk has this mass (> 0: it was selected)
    // the ties it takes: the least n with above + n qt >= tau (a double quotient, corrected in integers)
    const unsigned long long rem = tau - p.above;
    unsigned long long n = (unsigned long long)((double)rem / (double)qt);
    while (n * qt < rem) ++n;
    while (n > 1 && (n - 1) * qt >= rem) --n;
    tc = trunc_nth_of_key(ys, V, tk, (uint32_t)n, s, in);
  }
  const int bc = row_gumbel_argmax(smp, r, V, [&](int j, float& y) {
    y = ys[j];
    const uint32_t k = trunc_key(y);
    return in(j) && (k > tk || (k == tk && j <= tc));
  }, s.sk, s.sc);
  const float lse = row_lse(row, V, s.red);                      // last: nothing long-lived across the selection
  if (threadIdx.x == 0) {
    tokens[r] = bc + 1;
    answer[r * (L + 1) + smp.step] = bc + 1;
    if (logp) logp[r * L + smp.step - 1] = row[bc] - lse;
  }
}

// The candidate merge of one beam-search step (model.lua:529-569 as model.py restates it), generalised to diverse beam
// search (DESIGN §22), one warp per round n.  Row n*k + c is hypothesis (column) c of round n.  The k columns form G
// groups of w = k / G; group g owns columns [g*w, (g+1)*w) and the groups are merged in order g = 0 .. G-1.
//  - Explored columns: all w of the group (only its first at step 1).  Explored column e of group g takes its w best
//    classes from its k top-k entries by (augmented desc, top-k position asc), augmented = (double)logp - lam * n_g(v),
//    n_g(v) = the columns of groups < g filled at this step with token v.  Group 0 has no penalties: its explored set is
//    the first w entries.  Candidate q = e*w + j is the j-th of them (G = 1: q = c*k + j, the reference's order).
//  - Candidates whose token is end_token enter group g's list of finished hypotheses (DESIGN §24) by their norm
//    x = s / lp[stp] (IEEE fp64 division; lp null: x = s), s = scores[c] + logp in fp64 unpenalised: the list keeps the n
//    best by (x desc, step asc, q asc).  Rounds take the step's finished candidates best first by (x desc, q asc), each
//    strictly after the last round's; a ballot over the list (lane i holds position i) gives a candidate's position, and the
//    rounds stop at the first that would land at position >= n.  A new entry's tokens go to a free slot or to the slot of
//    the evicted n-th entry, which is from an earlier step (so shorter, every token overwritten): no row moves, and only
//    the order array ord changes.  n = 1 with lp null is the reference's rule: the first maximum in (step, q) order.
//  - The others are ranked by (a desc, q asc), a = s - lam * n_g(v), and the first min(#, w) fill the group's columns
//    from the PRE-merge beams; a column stores the unpenalised s.  A column left unfilled keeps its beam and score, and
//    is fed next step the state it was fed this step (parent -1 - row) and its beam's next position (a pad, 0).
// Penalties only lower a score and group g's penalised tokens number at most g*w, so the w best classes of a row under
// the penalty lie inside its unpenalised top k: the decoder's top-k list holds every class DBS could pick.  The products
// lam * n are __dmul_rn so that no fused multiply-add changes a's rounding.  beams: (N, k, L) token histories; lists as
// BeamLists says.  At the last step (stp == L - 1) the lists are written in order to out_* (n > 1), and pick_* (N, L),
// (N), (N), or null, take the best of the G list heads by (x desc, group asc), groups without a finished hypothesis skipped
// (pick_len 0 when none).
// SKIP (the answer rules, DESIGN §25): a top-k entry of value -inf is no candidate; it finishes nothing and fills no column.
template <bool SKIP>
__global__ void __launch_bounds__(32) k_beam_merge(int stp, int k, int G, float lam, int L, int end_token, const BeamLists lst,
                                                   const float* __restrict__ topv, const int32_t* __restrict__ topi,
                                                   const double* __restrict__ sc_in, double* __restrict__ sc_out,
                                                   const int32_t* __restrict__ beams_in, int32_t* __restrict__ beams_out,
                                                   int32_t* __restrict__ tokens, int32_t* __restrict__ parent,
                                                   int32_t* __restrict__ pick_ans, int32_t* __restrict__ pick_len,
                                                   double* __restrict__ pick_score) {
  // per column: the filling candidate's source column, its token (0: unfilled) and its stored score
  __shared__ int win_c[32], win_t[32];
  __shared__ double win_s[32];
  // groups g > 0 (w <= 16): per explored entry its augmented value and penalty count; per candidate its top-k position
  // and penalty count
  __shared__ double e_aug[16 * 32];
  __shared__ unsigned char e_cnt[16 * 32], c_pos[16 * 16], c_cnt[16 * 16];
  __shared__ int s_ord[32];                                // the last step: a list's slot at each position
  const int n = blockIdx.x, lane = threadIdx.x;
  const int nb = lst.nbest;
  const double lpv = lst.lp ? lst.lp[stp] : 1.0;         // every candidate of this step has l = stp generated tokens
  const bool last = stp == L - 1;
  int best = -1, bslot = 0; double bnorm = 0.0;          // the pick so far (warp-uniform)
  const int w = k / G;
  const int ne = stp == 1 ? 1 : w;                       // explored columns per group
  const int ncand = ne * w;
  const double lamd = (double)lam;
  const float* tv = topv + (int64_t)n * k * k;          // rows n*k .. n*k+k-1, k entries each
  const int32_t* ti = topi + (int64_t)n * k * k;
  const double* sc = sc_in + (int64_t)n * k;
  const int32_t* bin = beams_in + (int64_t)n * k * L;
  for (int g = 0; g < G; ++g) {
    const int c0 = g * w;
    if (g > 0) {
      for (int i = lane; i < ne * k; i += 32) {
        const int t = ti[c0 * k + i] + 1;
        int cnt = 0;
        for (int c = 0; c < c0; ++c) cnt += win_t[c] == t;
        e_cnt[i] = (unsigned char)cnt;
        e_aug[i] = (double)tv[c0 * k + i] - __dmul_rn(lamd, (double)cnt);
      }
      __syncwarp();
      for (int i = lane; i < ne * k; i += 32) {
        const int e = i / k, p = i % k;
        const double a = e_aug[i];
        int rank = 0;
        for (int p2 = 0; p2 < k; ++p2) {
          const double a2 = e_aug[e * k + p2];
          rank += a2 > a || (a2 == a && p2 < p);
        }
        if (rank < w) { c_pos[e * w + rank] = (unsigned char)p; c_cnt[e * w + rank] = e_cnt[i]; }
      }
      __syncwarp();
    }
    // candidate q of group g: its top-k entry (column c0 + q / w), and its penalty count
    const auto entry = [&](int q) { return (c0 + q / w) * k + (g ? (int)c_pos[q] : q % w); };
    const auto count = [&](int q) { return g ? (int)c_cnt[q] : 0; };
    // finished hypotheses of this step into the group's list: lane i holds position i's slot and norm, m positions are
    // filled (slots fill in order, so slots 0 .. m-1 are the filled ones)
    const int64_t lb = ((int64_t)n * G + g) * nb;          // the group's first slot
    int m = __popc(__ballot_sync(FULL, lane < nb && lst.len[lb + lane] > 0));
    int pslot = 0; double pnorm = 0.0;
    if (lane < m) {
      pslot = lst.ord ? lst.ord[lb + lane] : lane;
      pnorm = lst.norm ? lst.norm[lb + pslot] : lst.score[lb + pslot];
    }
    __syncwarp();                                          // every lane has read the list before a round writes it
    double xn = INFINITY; int xq = -1;                     // the last round's candidate
    for (;;) {
      bool fnd = false; double fx = 0.0, fs = 0.0; int fq = 0x7fffffff;
      for (int q = lane; q < ncand; q += 32) {
        const int idx = entry(q);
        if (ti[idx] + 1 != end_token) continue;
        const double s = sc[idx / k] + (double)tv[idx];
        if (SKIP && s == -INFINITY) continue;                // scores are finite: only a -inf entry gives -inf
        const double x = __ddiv_rn(s, lpv);
        if (!(x < xn || (x == xn && q > xq))) continue;
        if (!fnd || x > fx) { fnd = true; fx = x; fs = s; fq = q; }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const bool of = __shfl_xor_sync(FULL, fnd, o);
        const double ox = __shfl_xor_sync(FULL, fx, o);
        const double os = __shfl_xor_sync(FULL, fs, o);
        const int oq = __shfl_xor_sync(FULL, fq, o);
        if (of && (!fnd || ox > fx || (ox == fx && oq < fq))) { fnd = true; fx = ox; fs = os; fq = oq; }
      }
      if (!fnd) break;                                     // warp-uniform
      // after every entry of an earlier step, or of an earlier round, whose norm is not below it
      const int pos = __popc(__ballot_sync(FULL, lane < m && pnorm >= fx));
      if (pos >= nb) break;
      const int slot = m < nb ? m : __shfl_sync(FULL, pslot, nb - 1);
      const int us = __shfl_up_sync(FULL, pslot, 1);
      const double un = __shfl_up_sync(FULL, pnorm, 1);
      if (lane > pos) { pslot = us; pnorm = un; }
      if (lane == pos) { pslot = slot; pnorm = fx; }
      m = min(m + 1, nb);
      const int c = c0 + fq / w;
      int32_t* dst = lst.ans + (lb + slot) * L;
      for (int p = lane; p < stp; p += 32) dst[p] = bin[(int64_t)c * L + p];
      if (lane == 0) {
        dst[stp] = end_token; lst.len[lb + slot] = stp + 1; lst.score[lb + slot] = fs;
        if (lst.norm) lst.norm[lb + slot] = fx;
      }
      if (pos == nb - 1) break;                            // the next candidate would land at position n
      xn = fx; xq = fq;
    }
    if (lst.ord && lane < m) lst.ord[lb + lane] = pslot;
    const double hn = __shfl_sync(FULL, pnorm, 0);
    const int hs = __shfl_sync(FULL, pslot, 0);
    if (m > 0 && (best < 0 || hn > bnorm)) { best = g; bnorm = hn; bslot = hs; }
    if (last && lst.out_ans) {                             // the list in order
      s_ord[lane] = pslot;
      __syncwarp();                                        // the order, and the slots' tokens other lanes wrote
      for (int i = lane; i < nb * L; i += 32) {
        const int ps = i / L, p = i % L;
        lst.out_ans[(lb + ps) * L + p] = ps < m ? lst.ans[(lb + s_ord[ps]) * L + p] : 0;
      }
      if (lane < nb) {
        lst.out_len[lb + lane] = lane < m ? lst.len[lb + pslot] : 0;
        lst.out_score[lb + lane] = lane < m ? lst.score[lb + pslot] : 0.0;
        lst.out_norm[lb + lane] = lane < m ? pnorm : 0.0;
      }
      __syncwarp();                                        // s_ord is the next group's
    }
    // the w best other candidates: round j takes the best one strictly after round j-1's winner
    int nfill = 0;
    double ps = INFINITY; int pq = -1;
    for (int j = 0; j < w; ++j) {
      bool ok = false; double bs = 0.0; int bq = 0x7fffffff;
      for (int q = lane; q < ncand; q += 32) {
        const int idx = entry(q);
        if (ti[idx] + 1 == end_token) continue;
        double s = sc[idx / k] + (double)tv[idx];
        if (SKIP && s == -INFINITY) continue;
        if (const int cnt = count(q)) s -= __dmul_rn(lamd, (double)cnt);
        if (!(s < ps || (s == ps && q > pq))) continue;
        if (!ok || s > bs) { ok = true; bs = s; bq = q; }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const bool of = __shfl_xor_sync(FULL, ok, o);
        const double os = __shfl_xor_sync(FULL, bs, o);
        const int oq = __shfl_xor_sync(FULL, bq, o);
        if (of && (!ok || os > bs || (os == bs && oq < bq))) { ok = true; bs = os; bq = oq; }
      }
      if (!ok) break;                                      // warp-uniform
      if (lane == 0) {
        const int idx = entry(bq);
        win_c[c0 + j] = idx / k; win_t[c0 + j] = ti[idx] + 1; win_s[c0 + j] = sc[idx / k] + (double)tv[idx];
      }
      nfill = j + 1; ps = bs; pq = bq;
    }
    for (int j = nfill + lane; j < w; j += 32) { win_c[c0 + j] = c0 + j; win_t[c0 + j] = 0; win_s[c0 + j] = sc[c0 + j]; }
    __syncwarp();                                          // the next group counts this one's tokens
  }
  const int row0 = n * k;
  for (int i = lane; i < k * (stp + 1); i += 32) {
    const int c = i / (stp + 1), p = i % (stp + 1);
    const int32_t t = p < stp ? bin[(int64_t)win_c[c] * L + p] : win_t[c];
    beams_out[((int64_t)row0 + c) * L + p] = t;
    if (p == stp) tokens[row0 + c] = t;
  }
  for (int c = lane; c < k; c += 32) {
    sc_out[row0 + c] = win_s[c];
    parent[row0 + c] = win_t[c] ? row0 + win_c[c] : -1 - (row0 + c);
  }
  if (pick_ans && last) {
    const int64_t src = ((int64_t)n * G + (best < 0 ? 0 : best)) * nb + bslot;
    for (int p = lane; p < L; p += 32) pick_ans[(int64_t)n * L + p] = best < 0 ? 0 : lst.ans[src * L + p];
    if (lane == 0) { pick_len[n] = best < 0 ? 0 : lst.len[src]; pick_score[n] = best < 0 ? 0.0 : lst.score[src]; }
  }
}

// start of a search: every hypothesis is <start> with score 0, no round has a finished hypothesis yet
__global__ void k_beam_init(int64_t rows, int L, int start_token, int32_t* __restrict__ beams, int32_t* __restrict__ tokens,
                            double* __restrict__ scores) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * L) return;
  const int64_t r = i / L; const int p = (int)(i % L);
  beams[i] = p == 0 ? start_token : 0;
  if (p == 0) { tokens[r] = start_token; scores[r] = 0.0; }
}
__global__ void k_nll_fwd(const float* __restrict__ logp, const int32_t* __restrict__ tgt, const int32_t* __restrict__ mask_ids,
                          float* __restrict__ row_loss, int64_t rows, int V) {
  int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  bool keep = mask_ids[r] != 0 && tgt[r] > 0;
  row_loss[r] = keep ? -logp[r * V + tgt[r] - 1] : 0.f;
}
__global__ void k_nll_bwd(const float* __restrict__ logp, const int32_t* __restrict__ tgt, const int32_t* __restrict__ mask_ids,
                          float* __restrict__ dlogits, int64_t total, int V) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  int64_t r = i / V; int c = (int)(i % V);
  bool keep = mask_ids[r] != 0 && tgt[r] > 0;
  dlogits[i] = keep ? expf(logp[i]) - (c == tgt[r] - 1 ? 1.f : 0.f) : 0.f;
}
// block per row of raw logits
__global__ void k_lhood_accumulate(const float* __restrict__ logits, const int32_t* __restrict__ tgt,
                                   const int32_t* __restrict__ mask_ids, float* __restrict__ lh, int V, float* __restrict__ lse) {
  __shared__ float red[33];
  const int64_t r = blockIdx.x;
  if (mask_ids[r] == 0 || tgt[r] <= 0) return;      // gen.lua:23-24 MaskZero rows are zero; utils.lua:92-97
  const float* row = logits + r * V;
  float mx = -INFINITY;
  for (int c = threadIdx.x; c < V; c += blockDim.x) mx = fmaxf(mx, row[c]);
  mx = block_max(mx, red);
  float sum = 0.f;
  for (int c = threadIdx.x; c < V; c += blockDim.x) sum += expf(row[c] - mx);
  sum = block_sum(sum, red);
  if (threadIdx.x == 0) {
    const float l = mx + logf(sum);
    lh[r] += row[tgt[r] - 1] - l;
    if (lse) lse[r] = l;
  }
}
__global__ void k_nll_bwd_scaled(const float* logits, const float* __restrict__ lse, const int32_t* __restrict__ tgt,
                                 const int32_t* __restrict__ mask_ids, const float* __restrict__ scale, float* dlogits,
                                 int64_t total, int V) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  int64_t r = i / V; int c = (int)(i % V);
  bool keep = mask_ids[r] != 0 && tgt[r] > 0;
  dlogits[i] = keep ? scale[r] * (expf(logits[i] - lse[r]) - (c == tgt[r] - 1 ? 1.f : 0.f)) : 0.f;
}
__global__ void k_scale_copy(float* __restrict__ dst, const float* __restrict__ src, int64_t n, float alpha) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = alpha * src[i];
}

__global__ void k_clamp_adam(float* __restrict__ W, float* __restrict__ dW, float* __restrict__ m, float* __restrict__ v,
                             int64_t n, float step, float b1, float b2, float omb1, float omb2, float eps, float gscale) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float g = dW[i] * gscale;
  g = fminf(fmaxf(g, -5.f), 5.f);                  // model.lua:96
  dW[i] = g;
  float mm = m[i] * b1 + omb1 * g;                 // optim_updates.lua:80
  float vv = v[i] * b2 + omb2 * g * g;             // :81
  m[i] = mm; v[i] = vv;
  float tmp = sqrtf(vv) + eps;                     // :82
  W[i] = W[i] - step * (mm / tmp);                 // :90
}
__global__ void k_fill(float* __restrict__ buf, int64_t n, float val) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) buf[i] = val;
}

// ---- rows grouped by token id (counting sort) + segmented row sum ---------------------------------------
// Half of the option tokens are the pad id 0 and a handful of words are very frequent, so one atomic per element
// serialises on a few addresses.  Pad ids are counted per block (one atomic per block); every other id is aggregated
// per warp with match.any (one atomic per distinct id per warp).
__global__ void __launch_bounds__(256) k_tok_hist(const int32_t* __restrict__ ids, int64_t n, int32_t* __restrict__ counts) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31;
  const int v = i < n ? ids[i] : -1;
  const int nz = __syncthreads_count(v == 0);
  if (threadIdx.x == 0 && nz) atomicAdd(counts, nz);
  const unsigned peers = __match_any_sync(0xffffffffu, v > 0 ? v : -1 - lane);
  if (v > 0 && lane == __ffs(peers) - 1) atomicAdd(counts + v, __popc(peers));
}
// single block: offsets[v] = exclusive prefix sum of counts[v]; cursor[v] = offsets[v]
__global__ void k_tok_scan(const int32_t* __restrict__ counts, int32_t* __restrict__ offsets, int32_t* __restrict__ cursor, int nv) {
  __shared__ int32_t part[1024];
  const int t = threadIdx.x, per = (nv + blockDim.x - 1) / blockDim.x;
  const int b = t * per, e = min(nv, b + per);
  int32_t s = 0;
  for (int i = b; i < e; ++i) s += counts[i];
  part[t] = s;
  __syncthreads();
  if (t == 0) { int32_t run = 0; for (int i = 0; i < (int)blockDim.x; ++i) { int32_t v = part[i]; part[i] = run; run += v; } }
  __syncthreads();
  int32_t run = part[t];
  for (int i = b; i < e; ++i) { offsets[i] = run; cursor[i] = run; run += counts[i]; }
}
__global__ void k_tok_fill(const int32_t* __restrict__ ids, int64_t n, int32_t* __restrict__ cursor, int32_t* __restrict__ perm,
                           int32_t* __restrict__ sorted_tok) {
  __shared__ int warp_z[8];
  __shared__ int block_base;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int v = i < n ? ids[i] : -1;
  // pad ids: rank inside the block from ballots, one cursor atomic per block
  const unsigned zb = __ballot_sync(0xffffffffu, v == 0);
  if (lane == 0) warp_z[warp] = __popc(zb);
  __syncthreads();
  if (threadIdx.x == 0) {
    int tot = 0;
    for (int w = 0; w < 8; ++w) { int c = warp_z[w]; warp_z[w] = tot; tot += c; }
    block_base = tot ? atomicAdd(cursor, tot) : 0;
  }
  __syncthreads();
  // other ids: one cursor atomic per distinct id per warp
  const unsigned peers = __match_any_sync(0xffffffffu, v > 0 ? v : -1 - lane);
  const int leader = __ffs(peers) - 1;
  int base = 0;
  if (v > 0 && lane == leader) base = atomicAdd(cursor + v, __popc(peers));
  base = __shfl_sync(0xffffffffu, base, leader);
  const unsigned lt = (1u << lane) - 1u;
  int pos = -1;
  if (v == 0) pos = block_base + warp_z[warp] + __popc(zb & lt);
  else if (v > 0) pos = base + __popc(peers & lt);
  if (pos >= 0) { perm[pos] = (int32_t)i; sorted_tok[pos] = v; }
}
// Each block owns SEG_ROWS consecutive positions of the token-sorted row list; it streams those rows (ncols floats
// each, coalesced) and flushes a running sum into out[token] whenever the token changes.  Balanced by construction.
constexpr int SEG_ROWS = 64;
__global__ void __launch_bounds__(256) k_segsum_rows(const float* __restrict__ X, int64_t ldx, const int32_t* __restrict__ perm,
                                                     const int32_t* __restrict__ sorted_tok, int64_t n, float* __restrict__ out,
                                                     int ncols) {
  const int64_t p0 = (int64_t)blockIdx.x * SEG_ROWS, p1 = min(n, p0 + SEG_ROWS);
  for (int c0 = threadIdx.x * 4; c0 < ncols; c0 += blockDim.x * 4) {
    float4 acc = make_float4(0, 0, 0, 0);
    int cur = sorted_tok[p0];
    for (int64_t p = p0; p < p1; ++p) {
      const int tok = sorted_tok[p];
      if (tok != cur) {
        float* o = out + (int64_t)cur * ncols + c0;
        asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(o), "f"(acc.x), "f"(acc.y), "f"(acc.z), "f"(acc.w) : "memory");
        acc = make_float4(0, 0, 0, 0);
        cur = tok;
      }
      const float4 v = __ldcs(reinterpret_cast<const float4*>(X + (int64_t)perm[p] * ldx + c0));
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    float* o = out + (int64_t)cur * ncols + c0;
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(o), "f"(acc.x), "f"(acc.y), "f"(acc.z), "f"(acc.w) : "memory");
  }
}

// ---- deterministic mode (DESIGN §27): reductions without float atomics ------------------------------------------------
// C[m, n] += ws[0][m][n] + ws[1][m][n] + ... + ws[S-1][m][n], summed in slot order (S slots of M x N, row pitch N)
__global__ void k_slot_reduce(float* __restrict__ C, int64_t ldc, const float* __restrict__ ws, int S, int64_t M, int N) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, MN = M * N;
  if (i >= MN) return;
  float acc = ws[i];
  for (int s = 1; s < S; ++s) acc += ws[(int64_t)s * MN + i];
  C[(i / N) * ldc + i % N] += acc;
}

// Stable counting sort of row ids by token: the rows are cut into blocks of TS_ROWS (from n alone), each walked in index order
// by one warp.  hist[b][v] = rows of block b with token v; after k_tsort_scan it is the rank of block b's first such row among
// the rows of token v, and total[v] their count.  Ranks inside a warp step come from match.any, so no cursor atomics: row i
// lands at base[v] + (rows of token v before row i).
constexpr int TS_ROWS = 2048;
__global__ void __launch_bounds__(32) k_tsort_hist(const int32_t* __restrict__ ids, int64_t n, int nv, int32_t* __restrict__ hist) {
  const int lane = threadIdx.x;
  int32_t* h = hist + (int64_t)blockIdx.x * nv;
  const int64_t r0 = (int64_t)blockIdx.x * TS_ROWS, r1 = min(n, r0 + TS_ROWS);
  for (int64_t i0 = r0; i0 < r1; i0 += 32) {
    const int64_t i = i0 + lane;
    const int v = i < r1 ? ids[i] : -1;
    const unsigned peers = __match_any_sync(0xffffffffu, v >= 0 ? v : -1 - lane);
    if (v >= 0 && lane == __ffs(peers) - 1) h[v] += __popc(peers);
    __syncwarp();
  }
}
__global__ void k_tsort_scan(int32_t* __restrict__ hist, int nblk, int nv, int32_t* __restrict__ total) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nv) return;
  int32_t run = 0;
  for (int b = 0; b < nblk; ++b) { const int32_t c = hist[(int64_t)b * nv + v]; hist[(int64_t)b * nv + v] = run; run += c; }
  total[v] = run;
}
__global__ void __launch_bounds__(32) k_tsort_fill(const int32_t* __restrict__ ids, int64_t n, int nv, int32_t* __restrict__ hist,
                                                   const int32_t* __restrict__ base, int32_t* __restrict__ perm,
                                                   int32_t* __restrict__ sorted_tok) {
  const int lane = threadIdx.x;
  int32_t* cur = hist + (int64_t)blockIdx.x * nv;
  const int64_t r0 = (int64_t)blockIdx.x * TS_ROWS, r1 = min(n, r0 + TS_ROWS);
  const unsigned lt = (1u << lane) - 1u;
  for (int64_t i0 = r0; i0 < r1; i0 += 32) {
    const int64_t i = i0 + lane;
    const int v = i < r1 ? ids[i] : -1;
    const unsigned peers = __match_any_sync(0xffffffffu, v >= 0 ? v : -1 - lane);
    const int leader = __ffs(peers) - 1;
    int c = 0;
    if (v >= 0 && lane == leader) c = cur[v];
    c = __shfl_sync(0xffffffffu, c, leader);
    if (v >= 0) {
      const int pos = base[v] + c + __popc(peers & lt);
      perm[pos] = (int32_t)i; sorted_tok[pos] = v;
      if (lane == leader) cur[v] = c + __popc(peers);
    }
    __syncwarp();
  }
}

// Segmented row sum without atomics: out[tok, :] += scale * sum of X[perm[p], :] over the positions p of each token, in p order.
// Pass 1: block b owns positions [b SD_ROWS, (b+1) SD_ROWS) (from n alone).  A token whose positions all lie in the block is
// added to out by the block; the part of a token that starts in an earlier block goes to head[b], that of a token that starts
// in the block and goes on into the next one to tail[b].  Pass 2 (k_segsum_det_join): the block where such a token starts
// adds tail[b] + head[b+1] + ... in block order.  T = float or __half (4 columns per thread); the dropout factor of element
// (row, c) is drop_factor(d, site, row ncols + c) (an embedding gradient; d.thresh = 0: none).
constexpr int SD_ROWS = 256;
__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ float4 ld4(const __half* p) {
  const uint2 u = *reinterpret_cast<const uint2*>(p);
  const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u.x)), b = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
  return make_float4(a.x, a.y, b.x, b.y);
}
__device__ __forceinline__ void add_scaled4(float* o, const float4& a, float s) {
  float4 v = *reinterpret_cast<float4*>(o);
  v.x += s * a.x; v.y += s * a.y; v.z += s * a.z; v.w += s * a.w;
  *reinterpret_cast<float4*>(o) = v;
}
__device__ __forceinline__ bool sd_cont_prev(const int32_t* tok, int64_t p0) { return p0 > 0 && tok[p0 - 1] == tok[p0]; }
__device__ __forceinline__ bool sd_cont_next(const int32_t* tok, int64_t p1, int64_t n) { return p1 < n && tok[p1] == tok[p1 - 1]; }
template <typename T>
__global__ void __launch_bounds__(256) k_segsum_det(const T* __restrict__ X, int64_t ldx, const int32_t* __restrict__ perm,
                                                    const int32_t* __restrict__ tok, int64_t n, float* __restrict__ out, int ncols,
                                                    const float* __restrict__ scale, DropCfg d, uint32_t site,
                                                    float* __restrict__ head, float* __restrict__ tail) {
  const int64_t p0 = (int64_t)blockIdx.x * SD_ROWS, p1 = min(n, p0 + SD_ROWS);
  const bool cprev = sd_cont_prev(tok, p0), cnext = sd_cont_next(tok, p1, n);
  const float sc = scale ? __ldg(scale) : 1.f;
  for (int c0 = threadIdx.x * 4; c0 < ncols; c0 += blockDim.x * 4) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    int cur = tok[p0];
    bool first = true;
    for (int64_t p = p0; p <= p1; ++p) {
      const int t = p < p1 ? tok[p] : -1;
      if (t != cur) {                      // the segment of `cur` ends at p (or the block ends)
        if (first && cprev) *reinterpret_cast<float4*>(head + (int64_t)blockIdx.x * ncols + c0) = acc;
        else if (p == p1 && cnext) *reinterpret_cast<float4*>(tail + (int64_t)blockIdx.x * ncols + c0) = acc;
        else add_scaled4(out + (int64_t)cur * ncols + c0, acc, sc);
        if (p == p1) break;
        acc = make_float4(0.f, 0.f, 0.f, 0.f);
        cur = t; first = false;
      }
      const int64_t row = perm[p];
      float4 v = ld4(X + row * ldx + c0);
      float f[4];
      drop_factor4(d, site, (uint64_t)(row * ncols + c0) >> 2, f);
      acc.x += v.x * f[0]; acc.y += v.y * f[1]; acc.z += v.z * f[2]; acc.w += v.w * f[3];
    }
  }
}
__global__ void __launch_bounds__(256) k_segsum_det_join(const int32_t* __restrict__ tok, int64_t n, float* __restrict__ out, int ncols,
                                                         const float* __restrict__ scale, const float* __restrict__ head,
                                                         const float* __restrict__ tail) {
  const int64_t nblk = (n + SD_ROWS - 1) / SD_ROWS, b = blockIdx.x;
  const int64_t p0 = b * SD_ROWS, p1 = min(n, p0 + SD_ROWS);
  // block b holds a tail when its last token goes on and did not come in from the block before as its only token
  if (!sd_cont_next(tok, p1, n) || (sd_cont_prev(tok, p0) && tok[p0] == tok[p1 - 1])) return;
  const int t = tok[p1 - 1];
  const float sc = scale ? __ldg(scale) : 1.f;
  for (int c0 = threadIdx.x * 4; c0 < ncols; c0 += blockDim.x * 4) {
    float4 acc = ld4(tail + b * ncols + c0);
    for (int64_t c = b + 1; c < nblk; ++c) {
      const float4 h = ld4(head + c * ncols + c0);
      acc.x += h.x; acc.y += h.y; acc.z += h.z; acc.w += h.w;
      const int64_t q0 = c * SD_ROWS, q1 = min(n, q0 + SD_ROWS);
      if (tok[q1 - 1] != t || !sd_cont_next(tok, q1, n)) break;   // the token ends in block c
    }
    add_scaled4(out + (int64_t)t * ncols + c0, acc, sc);
  }
}

inline int blocks_for(int64_t n, int threads) { return (int)((n + threads - 1) / threads); }
template <typename F>
void set_smem(F f, size_t bytes) {
  if (bytes > 48 * 1024) VD_CUDA_CHECK(cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
}
}  // namespace

#define L1D(kern, n, ...)                                                                  \
  do {                                                                                     \
    if ((n) > 0) {                                                                         \
      kern<<<blocks_for((n), 256), 256, 0, cx.stream>>>(__VA_ARGS__);                      \
      check_launch(cx, #kern);                                                             \
    }                                                                                      \
  } while (0)

template <typename T>
static void segsum_det(LaunchCtx& cx, const T* X, int64_t ldx, const int32_t* perm, const int32_t* sorted_tok, int64_t n, float* out,
                       int ncols, const float* scale, DropCfg d, uint32_t site) {
  if (n <= 0) return;
  const int nblk = cdiv(n, SD_ROWS);
  float* head = cx.scratch_get<float>((int64_t)nblk * ncols);
  float* tail = cx.scratch_get<float>((int64_t)nblk * ncols);
  k_segsum_det<T><<<nblk, 256, 0, cx.stream>>>(X, ldx, perm, sorted_tok, n, out, ncols, scale, d, site, head, tail);
  check_launch(cx, "k_segsum_det");
  k_segsum_det_join<<<nblk, 256, 0, cx.stream>>>(sorted_tok, n, out, ncols, scale, head, tail);
  check_launch(cx, "k_segsum_det_join");
}

void transpose_ids(LaunchCtx& cx, const int32_t* src, int32_t* dst, int64_t rows, int T) {
  L1D(k_transpose_ids, rows * T, src, dst, rows, T);
}
void transpose_ids_rounds(LaunchCtx& cx, const int32_t* src, const int32_t* round, int32_t* dst, int64_t B, int R, int K, int T) {
  L1D(k_transpose_ids_rounds, B * K * T, src, round, dst, B * K, T, R, K);
}
void gather_round_rows(LaunchCtx& cx, const float* src, const int32_t* round, float* dst, int64_t B, int R, int H) {
  L1D(k_round_rows, B * H, src, round, dst, B, R, H, 1);
}
void scatter_round_rows(LaunchCtx& cx, const float* src, const int32_t* round, float* dst, int64_t B, int R, int H) {
  VD_CUDA_CHECK(cudaMemsetAsync(dst, 0, (size_t)B * R * H * sizeof(float), cx.stream));
  L1D(k_round_rows, B * H, src, round, dst, B, R, H, 0);
}
void embed_rows(LaunchCtx& cx, float* out, const float* emb, const int32_t* ids, int64_t rows, int E, DropCfg d, uint32_t site) {
  VD_REQUIRE(E % 4 == 0, -1, "embedSize must be a multiple of 4");
  L1D(k_embed_rows, rows * (E / 4), out, emb, ids, rows, E / 4, d, site);
}
void embed_scatter_add(LaunchCtx& cx, float* demb, const float* dx, int64_t ldx, const int32_t* ids, int64_t rows, int E,
                       DropCfg d, uint32_t site, int nv) {
  VD_REQUIRE(E <= SC_THREADS * SC_MAXACC, -1, "embedSize too large for embed_scatter_add");
  if (rows <= 0) return;
  if (cx.deterministic) {
    VD_REQUIRE(nv > 0 && E % 4 == 0 && ldx % 4 == 0 && ((uintptr_t)dx & 15) == 0, -1, "embed_scatter_add: deterministic route shape");
    int32_t* s3 = cx.scratch_get<int32_t>(3 * (int64_t)nv);
    int32_t* perm = cx.scratch_get<int32_t>(rows);
    int32_t* stok = cx.scratch_get<int32_t>(rows);
    group_rows_by_token(cx, ids, rows, nv, s3, perm, stok);
    segsum_det(cx, dx, ldx, perm, stok, rows, demb, E, nullptr, d, site);
    return;
  }
  k_embed_scatter_add<<<blocks_for(rows, SC_ROWS), SC_THREADS, 0, cx.stream>>>(demb, dx, ldx, ids, rows, E, d, site);
  check_launch(cx, "embed_scatter_add");
}
void lstm_pointwise_fwd(LaunchCtx& cx, float* gates, const float* bias, const float* c_prev, const int32_t* mask_ids,
                        float* c_out, float* h_out, int64_t R, int H) {
  VD_REQUIRE(H % 4 == 0, -1, "rnnHiddenSize must be a multiple of 4");
  L1D(k_lstm_pw_fwd, R * (H / 4), gates, bias, c_prev, mask_ids, c_out, h_out, R, H);
}
void lstm_first_step_fwd(LaunchCtx& cx, float* gates, const float* ptable, const int32_t* tok, const float* bias,
                         const float* c_prev, const int32_t* mask_ids, float* c_out, float* h_out, int64_t R, int H) {
  VD_REQUIRE(H % 4 == 0 && (gates || ptable), -1, "lstm_first_step_fwd: bad arguments");
  L1D(k_lstm_first_step, R * (H / 4), gates, ptable, tok, bias, c_prev, mask_ids, c_out, h_out, R, H);
}
void lstm_pointwise_bwd(LaunchCtx& cx, const float* gates, const float* c_prev, const float* c, const float* dh_rec,
                        const float* dh_ext, const float* dc_ext, float* dc_carry, const int32_t* mask_ids, float* da,
                        int64_t R, int H) {
  L1D(k_lstm_pw_bwd, R * H, gates, c_prev, c, dh_rec, dh_ext, dc_ext, dc_carry, mask_ids, da, R, H);
}
void colsum_add(LaunchCtx& cx, float* out, const float* X, int64_t rows, int cols, int64_t ldx) {
  if (rows <= 0 || cols <= 0) return;
  dim3 grid(cdiv(cols, 128), cdiv(rows, CS_ROWS));
  const bool vec = cols % 4 == 0 && ldx % 4 == 0 && ((uintptr_t)X & 15) == 0;
  if (cx.deterministic) {
    float* ws = cx.scratch_get<float>((int64_t)grid.y * cols);
    if (vec) k_colsum_add4<true><<<grid, 256, 0, cx.stream>>>(ws, X, rows, cols, ldx);
    else k_colsum_add<true><<<grid, 128, 0, cx.stream>>>(ws, X, rows, cols, ldx);
    check_launch(cx, "colsum_add");
    slot_reduce(cx, out, cols, ws, (int)grid.y, 1, cols);
    return;
  }
  if (vec) k_colsum_add4<false><<<grid, 256, 0, cx.stream>>>(out, X, rows, cols, ldx);
  else k_colsum_add<false><<<grid, 128, 0, cx.stream>>>(out, X, rows, cols, ldx);
  check_launch(cx, "colsum_add");
}
void dropout_apply(LaunchCtx& cx, float* out, const float* in, int64_t n, DropCfg d, uint32_t site) {
  L1D(k_dropout_apply, n, out, in, n, d, site);
}
void tanh_bwd(LaunchCtx& cx, float* dpre, const float* dy, const float* y, int64_t n) { L1D(k_tanh_bwd, n, dpre, dy, y, n); }
void add_inplace(LaunchCtx& cx, float* a, const float* b, int64_t n) { L1D(k_add_inplace, n, a, b, n); }
void add_out(LaunchCtx& cx, float* out, const float* a, const float* b, int64_t n) { L1D(k_add_out, n, out, a, b, n); }
void copy_cols(LaunchCtx& cx, float* dst, int64_t ldd, const float* src, int64_t lds, int64_t rows, int cols) {
  L1D(k_copy_cols, rows * cols, dst, ldd, src, lds, rows, cols);
}
void repeat_rows(LaunchCtx& cx, float* dst, const float* src, int64_t B, int R, int64_t cols, int64_t lds) {
  L1D(k_repeat_rows, B * R * cols, dst, src, B, R, cols, lds < 0 ? cols : lds);
}
void hist_append(LaunchCtx& cx, int32_t* hist, int64_t B, int R, int W, int r, const int32_t* src, int src_w, const int32_t* ans,
                 int64_t ans_ld, const int32_t* ans_len, int ans_max, int end_token, int max_ans_len, bool concat,
                 const int32_t* slot, const int32_t* round) {
  VD_REQUIRE(W >= src_w && src_w > 0 && r < R - 1 && (r < 0 || max_ans_len >= 1), VD_E_BADARG, "hist_append: widths / round");
  VD_REQUIRE(round == nullptr || slot != nullptr, VD_E_BADARG, "hist_append: per-row rounds need per-row slots");
  if (B <= 0) return;
  const int cap = r < 0 ? 0 : (int)std::min<int64_t>(max_ans_len, ans_ld);   // an answer row holds at most ans_ld words
  k_hist_append<<<(unsigned)B, 128, (size_t)cap * sizeof(int32_t), cx.stream>>>(hist, R, W, r, src, src_w, ans, ans_ld, ans_len,
                                                                               ans_max, end_token, cap, concat ? 1 : 0, slot, round);
  check_launch(cx, "k_hist_append");
}
void hist_prefill(LaunchCtx& cx, int32_t* hist, int64_t n, int R, int W, const int32_t* slot, const int32_t* rounds,
                  const int32_t* row0, const int32_t* q, int src_w, const int32_t* ans, int Ta, int end_token, int max_ans_len,
                  bool concat) {
  VD_REQUIRE(W >= src_w && src_w > 0 && Ta >= 1 && max_ans_len >= 1, VD_E_BADARG, "hist_prefill: widths");
  if (n <= 0) return;
  const int cap = std::min(max_ans_len, Ta);
  k_hist_prefill<<<(unsigned)n, 128, (size_t)cap * sizeof(int32_t), cx.stream>>>(hist, R, W, slot, rounds, row0, q, src_w, ans, Ta,
                                                                              end_token, cap, concat ? 1 : 0);
  check_launch(cx, "k_hist_prefill");
}
void sum_repeated_rows(LaunchCtx& cx, float* dst, const float* src, int64_t B, int R, int64_t cols) {
  L1D(k_sum_repeated_rows, B * cols, dst, src, B, R, cols);
}
void transpose_segments(LaunchCtx& cx, const float* W, float* Wt, const int64_t* seg_table_dev, int nseg, int64_t max_elems) {
  if (nseg <= 0) return;
  int gx = (int)std::min<int64_t>((max_elems + 1023) / 1024, 4096);
  dim3 grid(gx, nseg), block(32, 8);
  k_transpose_segments<<<grid, block, 0, cx.stream>>>(W, Wt, seg_table_dev);
  check_launch(cx, "transpose_segments");
}
void rowdot_fwd(LaunchCtx& cx, float* out, const float* x, const float* w, const float* b, int64_t rows, int H) {
  L1D(k_rowdot_fwd, rows * 32, out, x, w, b, rows, H);
}
void rowdot_bwd(LaunchCtx& cx, const float* ds, const float* x, const float* w, float* dx, int accumulate_dx, float* dw,
                float* db, int64_t rows, int H) {
  if (rows <= 0) return;
  const int nb = blocks_for(rows, 32);
  if (cx.deterministic) {
    float* ws = cx.scratch_get<float>((int64_t)nb * (H + 1));
    k_rowdot_bwd<true><<<nb, 256, 0, cx.stream>>>(ds, x, w, dx, accumulate_dx, ws, ws + (int64_t)nb * H, rows, H);
    check_launch(cx, "rowdot_bwd");
    slot_reduce(cx, dw, H, ws, nb, 1, H);
    slot_reduce(cx, db, 1, ws + (int64_t)nb * H, nb, 1, 1);
    return;
  }
  k_rowdot_bwd<false><<<nb, 256, 0, cx.stream>>>(ds, x, w, dx, accumulate_dx, dw, db, rows, H);
  check_launch(cx, "rowdot_bwd");
}

void mn_attention_fwd(LaunchCtx& cx, const float* q, const float* h, float* probs, float* hAtt, int B, int R, int H) {
  mn_attention_rows_fwd(cx, q, h, (int64_t)R * H, probs, hAtt, B, R, H, 0, R);
}
void mn_attention_rows_fwd(LaunchCtx& cx, const float* q, const float* h, int64_t hpitch, float* probs, float* hAtt, int B,
                           int R, int H, int r0, int r1, const int32_t* slot, const int32_t* round) {
  VD_REQUIRE((slot == nullptr) == (round == nullptr), VD_E_BADARG, "mn_attention: per-row slots and rounds go together");
  if (slot) { r0 = 0; r1 = R; }                   // one row per block; shared memory for the deepest round
  VD_REQUIRE(0 <= r0 && r0 < r1 && r1 <= R && hpitch >= (int64_t)r1 * H, VD_E_BADARG, "mn_attention: round range / fact pitch");
  const int nr = slot ? 1 : r1 - r0;
  size_t smem = (size_t)(nr * H + r1 * H + nr * R) * sizeof(float);
  set_smem(k_mn_att_fwd, smem);
  k_mn_att_fwd<<<B, 256, smem, cx.stream>>>(q, h, probs, hAtt, R, H, r0, r1, hpitch, slot, round);
  check_launch(cx, "mn_attention_fwd");
}
void mn_attention_bwd(LaunchCtx& cx, const float* q, const float* h, const float* probs, const float* dhAtt, float* dq,
                      float* dh, int B, int R, int H) {
  size_t smem = (size_t)(3 * R * H + 2 * R * R) * sizeof(float);
  set_smem(k_mn_att_bwd, smem);
  k_mn_att_bwd<<<B, 256, smem, cx.stream>>>(q, h, probs, dhAtt, dq, dh, R, H);
  check_launch(cx, "mn_attention_bwd");
}
void hrea_attention_fwd(LaunchCtx& cx, const float* sq, const float* sh, const float* Hs, float* probs, float* att, int B,
                        int R, int H) {
  hrea_attention_rows_fwd(cx, sq, sh, Hs, (int64_t)R * H, probs, att, B, R, H, 0, R);
}
void hrea_attention_rows_fwd(LaunchCtx& cx, const float* sq, const float* sh, const float* Hs, int64_t hpitch, float* probs,
                             float* att, int B, int R, int H, int r0, int r1, const int32_t* slot, const int32_t* round) {
  VD_REQUIRE(R <= 32, -2, "maxQuesCount must be <= 32");
  VD_REQUIRE((slot == nullptr) == (round == nullptr), VD_E_BADARG, "hrea_attention: per-row slots and rounds go together");
  if (slot) { r0 = 0; r1 = R; }
  VD_REQUIRE(0 <= r0 && r0 < r1 && r1 <= R && hpitch >= (int64_t)r1 * H, VD_E_BADARG, "hrea_attention: round range / fact pitch");
  const int nr = slot ? 1 : r1 - r0;
  size_t smem = (size_t)(r1 * H + nr * R) * sizeof(float);
  set_smem(k_hrea_att_fwd, smem);
  k_hrea_att_fwd<<<B, 256, smem, cx.stream>>>(sq, sh, Hs, probs, att, R, H, r0, r1, hpitch, slot, round);
  check_launch(cx, "hrea_attention_fwd");
}
void dialog_cache_write(LaunchCtx& cx, float* facts, float* shc, const float* h3, const float* sh, int64_t B, int R, int H, int r,
                        const int32_t* slot, const int32_t* round, float* st_h, float* st_c, const float* hn, const float* cn) {
  VD_REQUIRE(0 <= r && r < R && (shc == nullptr) == (sh == nullptr) && (facts == nullptr) == (h3 == nullptr) &&
             (st_h == nullptr) == (hn == nullptr) && (st_c == nullptr) == (cn == nullptr) && (st_h == nullptr) == (st_c == nullptr),
             VD_E_BADARG, "dialog_cache_write: round / (destination, source) pairs");
  VD_REQUIRE((round == nullptr || slot != nullptr) && (slot == nullptr || round != nullptr || (!facts && !shc)), VD_E_BADARG,
             "dialog_cache_write: per-row rounds need per-row slots, and the facts need per-row rounds");
  L1D(k_dialog_cache_write, (facts ? B * H : 0) + (shc ? B : 0) + (st_h ? 2 * B * H : 0), facts, shc, h3, sh, B, R, H, r, slot, round,
      st_h, st_c, hn, cn);
}
void dialog_gather(LaunchCtx& cx, const DialogGather& g) {
  if (g.n <= 0) return;
  const int64_t most = std::max({g.n * g.Tq, g.n * g.W, g.n * g.img_cols, g.n * (int64_t)g.H});
  const unsigned gx = (unsigned)std::min<int64_t>(blocks_for(most, 256), 2048);
  k_dialog_gather<<<dim3(gx, 4), 256, 0, cx.stream>>>(g);
  check_launch(cx, "dialog_gather");
}
void scatter_rows(LaunchCtx& cx, float* dst, const float* src, const int32_t* slot, int64_t n, int64_t cols) {
  L1D(k_scatter_rows, n * cols, dst, src, slot, n, cols);
}
void hrea_attention_bwd(LaunchCtx& cx, const float* sq, const float* sh, const float* Hs, const float* probs,
                        const float* datt, float* dsq, float* dsh, float* dHs, int B, int R, int H) {
  (void)sq; (void)sh;
  size_t smem = (size_t)(2 * R * H + 2 * R * R) * sizeof(float);
  set_smem(k_hrea_att_bwd, smem);
  k_hrea_att_bwd<<<B, 256, smem, cx.stream>>>(Hs, probs, datt, dsq, dsh, dHs, R, H);
  check_launch(cx, "hrea_attention_bwd");
}
void masktime_concat_fwd(LaunchCtx& cx, float* out, const float* wemb, const float* img, const int32_t* ids_tm, int T,
                         int64_t N, int E, int I) {
  L1D(k_masktime_concat_fwd, (int64_t)T * N * (E + I), out, wemb, img, ids_tm, (int64_t)T * N, N, E, I);
}
void masktime_bwd(LaunchCtx& cx, const float* dx, int64_t ldx, int off, const int32_t* ids_tm, float* dimg, int T, int64_t N,
                  int I) {
  L1D(k_masktime_bwd, N * I, dx, ldx, off, ids_tm, dimg, T, N, I);
}

void san_expand_dropout(LaunchCtx& cx, float* img_tr, const float* t, int B, int R, int P, int H, DropCfg d, uint32_t site) {
  VD_REQUIRE(H % 4 == 0, -1, "H % 4");
  int64_t PH4 = (int64_t)P * H / 4, total4 = (int64_t)B * R * PH4;
  L1D(k_san_expand_dropout, total4, img_tr, t, total4, R, PH4, d, site);
}
void san_score_fwd(LaunchCtx& cx, const float* img_common, const float* ques_common, const float* w, const float* b, float* s,
                   int64_t N, int P, int Cm, DropCfg d, uint32_t site, const int32_t* cnt, int R) {
  VD_REQUIRE(Cm % 4 == 0, -1, "commonEmbeddingSize % 4");
  if (N * P <= 0) return;
  auto k = cnt ? k_san_score_fwd<true> : k_san_score_fwd<false>;
  k<<<blocks_for(N * P * 32, 256), 256, 0, cx.stream>>>(img_common, ques_common, w, b, s, N * P, P, Cm, d, site, cnt, R);
  check_launch(cx, "k_san_score_fwd");
}
void san_softmax_att_fwd(LaunchCtx& cx, const float* s, float* p, const float* img_tr, const float* u_in, float* u_out,
                         int64_t N, int P, int H, const int32_t* cnt, int R) {
  if (N <= 0) return;
  VD_REQUIRE(H % 4 == 0, -1, "H % 4");
  size_t smem = (size_t)(((P + 33 + 3) & ~3) + 256 * 4) * sizeof(float);
  auto k = cnt ? k_san_softmax_att_fwd<true> : k_san_softmax_att_fwd<false>;
  k<<<dim3((unsigned)N, 2), 256, smem, cx.stream>>>(s, p, img_tr, u_in, u_out, P, H, cnt, R);
  check_launch(cx, "san_softmax_att_fwd");
}
void san_att_bwd(LaunchCtx& cx, const float* du, const float* p, const float* img_tr, float* ds, float* dimg_tr, int64_t N,
                 int P, int H, const int32_t* cnt, int R) {
  if (N <= 0) return;
  VD_REQUIRE(H % 4 == 0, -1, "H % 4");
  size_t smem = (size_t)(H + 2 * P + 33) * sizeof(float);
  auto k = cnt ? k_san_att_bwd<true> : k_san_att_bwd<false>;
  k<<<(int)N, 512, smem, cx.stream>>>(du, p, img_tr, ds, dimg_tr, P, H, cnt, R);
  check_launch(cx, "san_att_bwd");
}
void san_score_bwd(LaunchCtx& cx, const float* ds, const float* img_common, const float* ques_common, const float* w,
                   float* d_img_common, float* d_ques_common, float* dw, float* db, int64_t N, int P, int Cm, DropCfg d,
                   uint32_t site, const int32_t* cnt, int R) {
  if (N <= 0) return;
  VD_REQUIRE(Cm % 4 == 0, -1, "commonEmbeddingSize % 4");
  const int CS = Cm >= 512 ? 4 : 1;                      // column slices per dialog round
  const size_t smem = (size_t)(((P + 3) & ~3) + 2 * 256 * 4) * sizeof(float);
  if (cx.deterministic) {
    float* ws = cx.scratch_get<float>(N * (Cm + 1));
    auto k = cnt ? k_san_score_bwd<true, true> : k_san_score_bwd<false, true>;
    k<<<dim3((unsigned)N, CS), 256, smem, cx.stream>>>(ds, img_common, ques_common, w, d_img_common, d_ques_common, ws, ws + N * Cm, P,
                                                        Cm, d, site, cnt, R);
    check_launch(cx, "san_score_bwd");
    slot_reduce(cx, dw, Cm, ws, (int)N, 1, Cm);
    slot_reduce(cx, db, 1, ws + N * Cm, (int)N, 1, 1);
    return;
  }
  auto k = cnt ? k_san_score_bwd<true, false> : k_san_score_bwd<false, false>;
  k<<<dim3((unsigned)N, CS), 256, smem, cx.stream>>>(ds, img_common, ques_common, w, d_img_common, d_ques_common, dw, db, P, Cm, d,
                                                      site, cnt, R);
  check_launch(cx, "san_score_bwd");
}
void san_collapse_bwd(LaunchCtx& cx, const float* dimg_tr, const float* t, float* dt_pre, int B, int R, int P, int H,
                      DropCfg d, uint32_t site, const int32_t* cnt) {
  VD_REQUIRE(H % 4 == 0, -1, "H % 4");
  int64_t PH4 = (int64_t)P * H / 4, total4 = (int64_t)B * PH4;
  if (total4 <= 0) return;
  auto k = cnt ? k_san_collapse_bwd<true> : k_san_collapse_bwd<false>;
  k<<<blocks_for(total4, 256), 256, 0, cx.stream>>>(dimg_tr, t, dt_pre, total4, R, PH4, d, site, cnt, (int64_t)H / 4);
  check_launch(cx, "k_san_collapse_bwd");
}

void disc_scores_fwd(LaunchCtx& cx, const float* feat, const float* encOut, float* scores, int64_t N, int K, int H) {
  VD_REQUIRE(H % 4 == 0, -1, "H % 4");
  L1D(k_disc_scores_fwd, N * K * 32, feat, encOut, scores, N * K, K, H);
}
void disc_scores_bwd(LaunchCtx& cx, const float* dscores, const float* feat, const float* encOut, float* dfeat, float* dencOut,
                     int64_t N, int K, int H) {
  if (N <= 0) return;
  k_disc_scores_bwd<<<(int)N, 256, K * sizeof(float), cx.stream>>>(dscores, feat, encOut, dfeat, dencOut, K, H);
  check_launch(cx, "disc_scores_bwd");
}
void xent_fwd(LaunchCtx& cx, const float* scores, const int32_t* gt, float* row_loss, int64_t N, int K) {
  if (N <= 0) return;
  k_xent_fwd<<<(int)N, 128, 0, cx.stream>>>(scores, gt, row_loss, K);
  check_launch(cx, "xent_fwd");
}
void xent_bwd(LaunchCtx& cx, const float* scores, const int32_t* gt, float* dscores, int64_t N, int K) {
  if (N <= 0) return;
  k_xent_bwd<<<(int)N, 128, 0, cx.stream>>>(scores, gt, dscores, K, 1.f / (float)N);
  check_launch(cx, "xent_bwd");
}
void soft_xent(LaunchCtx& cx, const float* scores, const float* rel, float* row_loss, float* dscores, int64_t N, int K) {
  if (N <= 0) return;
  k_soft_xent<<<(int)N, 128, 0, cx.stream>>>(scores, rel, row_loss, dscores, K, 1.f / (float)N);
  check_launch(cx, "soft_xent");
}
void reduce_sum(LaunchCtx& cx, const float* x, float* out, int64_t n, float scale) {
  k_reduce_sum<<<1, 1024, 0, cx.stream>>>(x, out, n, scale);
  check_launch(cx, "reduce_sum");
}
void rank_rows(LaunchCtx& cx, const float* scores, const int32_t* gt, int32_t* ranks, int64_t N, int K) {
  if (N <= 0) return;
  k_rank_rows<<<(int)N, 128, K * sizeof(float), cx.stream>>>(scores, gt, ranks, K);
  check_launch(cx, "rank_rows");
}
void logsoftmax_rows(LaunchCtx& cx, float* logits, const int32_t* mask_ids, int64_t rows, int V) {
  if (rows <= 0) return;
  k_logsoftmax_rows<<<(int)rows, 256, 0, cx.stream>>>(logits, mask_ids, V);
  check_launch(cx, "logsoftmax_rows");
}
void nll_fwd(LaunchCtx& cx, const float* logp, const int32_t* tgt, const int32_t* mask_ids, float* row_loss, int64_t rows, int V) {
  L1D(k_nll_fwd, rows, logp, tgt, mask_ids, row_loss, rows, V);
}
void nll_bwd(LaunchCtx& cx, const float* logp, const int32_t* tgt, const int32_t* mask_ids, float* dlogits, int64_t rows, int V) {
  L1D(k_nll_bwd, rows * V, logp, tgt, mask_ids, dlogits, rows * V, V);
}
void lhood_accumulate(LaunchCtx& cx, const float* logits, const int32_t* tgt, const int32_t* mask_ids, float* lh, int64_t rows,
                      int V, float* lse) {
  if (rows <= 0) return;
  k_lhood_accumulate<<<(int)rows, 256, 0, cx.stream>>>(logits, tgt, mask_ids, lh, V, lse);
  check_launch(cx, "lhood_accumulate");
}
void nll_bwd_scaled(LaunchCtx& cx, const float* logits, const float* lse, const int32_t* tgt, const int32_t* mask_ids,
                    const float* scale, float* dlogits, int64_t rows, int V) {
  L1D(k_nll_bwd_scaled, rows * V, logits, lse, tgt, mask_ids, scale, dlogits, rows * V, V);
}
void scale_copy(LaunchCtx& cx, float* dst, const float* src, int64_t n, float alpha) { L1D(k_scale_copy, n, dst, src, n, alpha); }
void vocab_lse_finish(LaunchCtx& cx, const float* part_max, const float* part_sum, int nparts, const float* tgt_logit,
                      const int32_t* tgt, const int32_t* row_ids, float* lse, float* out, float sign, int accumulate, int64_t rows) {
  L1D(k_vocab_lse_finish, rows, part_max, part_sum, nparts, tgt_logit, tgt, row_ids, lse, out, sign, accumulate, rows);
}
void vocab_sample_finish(LaunchCtx& cx, const float* part_max, const float* part_sum, const float* part_key, const int32_t* part_cls,
                         const float* part_x, int nparts, int64_t rows, int step, int L, int32_t* tokens, int32_t* answer, float* logp) {
  L1D(k_vocab_sample_finish, rows, part_max, part_sum, part_key, part_cls, part_x, nparts, rows, step, L, tokens, answer, logp);
}
static void check_rules(const AnswerRules* ar, int V) {
  if (!ar) return;
  VD_REQUIRE(V >= 1 && V <= TRUNC_MAX_V, VD_E_BADARG, "answer rules need V in [1, 49152] (the row's bit mask)");
  VD_REQUIRE(ar->min_words >= 0 && ar->no_repeat_ngram >= 0 && ar->n_banned >= 0 && ar->n_banned <= 1024 &&
             (ar->banned || ar->n_banned == 0) && ar->end_token >= 1 && ar->end_token <= V && ar->step >= 1 &&
             (ar->hist || ar->no_repeat_ngram == 0) && ar->ld > 0,
             VD_E_BADARG, "answer rules: counts, banned ids, end_token, step or history");
}
void logsoftmax_sample_rows(LaunchCtx& cx, const float* logits, int64_t rows, int V, const SampleCfg& smp, int L, int32_t* tokens,
                            int32_t* answer, float* logp, const AnswerRules* ar) {
  check_rules(ar, V);
  if (rows <= 0) return;
  if (ar) k_logsoftmax_sample_rows<true><<<(unsigned)rows, 256, 0, cx.stream>>>(logits, V, smp, L, tokens, answer, logp, *ar);
  else k_logsoftmax_sample_rows<false><<<(unsigned)rows, 256, 0, cx.stream>>>(logits, V, smp, L, tokens, answer, logp, {});
  check_launch(cx, "k_logsoftmax_sample_rows");
}
void truncated_sample_rows(LaunchCtx& cx, const float* logits, int64_t rows, int V, const SampleCfg& smp, const TruncCfg& tr,
                           int L, int32_t* tokens, int32_t* answer, float* logp, const AnswerRules* ar) {
  VD_REQUIRE(V >= 1 && V <= TRUNC_MAX_V, VD_E_BADARG, "truncated_sample_rows: V must be in [1, 49152] (the staged row)");
  VD_REQUIRE(tr.top_k >= 0 && std::isfinite(tr.top_p) && tr.top_p > 0.f && tr.top_p <= 1.f, VD_E_BADARG,
             "truncated_sample_rows: top_k >= 0, top_p in (0, 1]");
  check_rules(ar, V);
  if (rows <= 0) return;
  // the dynamic stage beside the static histograms passes the 48 KB default from V = 8 121 on: always opted in.  With the
  // rules the row's barred bits follow it (6 KB at V = 49 152: 198 KB beside 16.3 KB static, within a CTA's 227 KB)
  const size_t smem = (size_t)V * sizeof(float) + (ar ? (size_t)((V + 31) / 32) * sizeof(uint32_t) : 0);
  if (ar) {
    VD_CUDA_CHECK(cudaFuncSetAttribute(k_truncated_sample_rows<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_truncated_sample_rows<true><<<(unsigned)rows, 256, smem, cx.stream>>>(logits, V, smp, tr, L, tokens, answer, logp, *ar);
  } else {
    VD_CUDA_CHECK(cudaFuncSetAttribute(k_truncated_sample_rows<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_truncated_sample_rows<false><<<(unsigned)rows, 256, smem, cx.stream>>>(logits, V, smp, tr, L, tokens, answer, logp, {});
  }
  check_launch(cx, "k_truncated_sample_rows");
}
void beam_gather(LaunchCtx& cx, float* dst, const float* out_prev, const float* in_prev, const int32_t* parent, int64_t rows, int H) {
  L1D(k_beam_gather, rows * H, dst, out_prev, in_prev, parent, rows, H);
}
template <bool RULES>
static void launch_topk_rows(LaunchCtx& cx, const float* logits, const int32_t* mask_ids, int64_t rows, int V, int k, float* topv,
                             int32_t* topi, const AnswerRules& ar) {
  const unsigned g = (unsigned)rows;
  if (k <= 4) k_logsoftmax_topk_rows<4, RULES><<<g, 256, 0, cx.stream>>>(logits, mask_ids, V, k, topv, topi, ar);
  else if (k <= 8) k_logsoftmax_topk_rows<8, RULES><<<g, 256, 0, cx.stream>>>(logits, mask_ids, V, k, topv, topi, ar);
  else if (k <= 16) k_logsoftmax_topk_rows<16, RULES><<<g, 256, 0, cx.stream>>>(logits, mask_ids, V, k, topv, topi, ar);
  else k_logsoftmax_topk_rows<32, RULES><<<g, 256, 0, cx.stream>>>(logits, mask_ids, V, k, topv, topi, ar);
}
void logsoftmax_topk_rows(LaunchCtx& cx, const float* logits, const int32_t* mask_ids, int64_t rows, int V, int k, float* topv,
                          int32_t* topi, const AnswerRules* ar) {
  VD_REQUIRE(k >= 1 && k <= 32 && k <= V, VD_E_BADARG, "logsoftmax_topk_rows: k");
  check_rules(ar, V);
  if (rows == 0) return;
  if (ar) launch_topk_rows<true>(cx, logits, mask_ids, rows, V, k, topv, topi, *ar);
  else launch_topk_rows<false>(cx, logits, mask_ids, rows, V, k, topv, topi, {});
  check_launch(cx, "k_logsoftmax_topk_rows");
}
void beam_init(LaunchCtx& cx, int64_t rows, int L, int start_token, int32_t* beams, int32_t* tokens, double* scores) {
  L1D(k_beam_init, rows * L, rows, L, start_token, beams, tokens, scores);
}
void beam_merge(LaunchCtx& cx, int64_t N, int stp, int k, int G, float lam, int L, int end_token, const float* topv,
                const int32_t* topi, const double* scores_in, double* scores_out, const int32_t* beams_in, int32_t* beams_out,
                int32_t* tokens, int32_t* parent, const BeamLists& lists, int32_t* pick_ans, int32_t* pick_len,
                double* pick_score, bool skip_empty) {
  VD_REQUIRE(k >= 1 && k <= 32 && stp >= 1 && stp < L, VD_E_BADARG, "beam_merge: k / step");
  VD_REQUIRE(G >= 1 && k % G == 0 && std::isfinite(lam) && lam >= 0.f, VD_E_BADARG, "beam_merge: groups / diversity");
  VD_REQUIRE(!pick_ans == !pick_len && !pick_ans == !pick_score, VD_E_BADARG, "beam_merge: all pick outputs or none");
  const BeamLists& b = lists;
  VD_REQUIRE(b.nbest >= 1 && b.nbest <= 32 && b.ans && b.len && b.score && (b.norm || !b.lp), VD_E_BADARG,
             "beam_merge: n in [1, 32], the list slots, and norms with a length-penalty table");
  const bool many = b.nbest > 1;
  VD_REQUIRE(!b.ord == !many && !b.out_ans == !many && !b.out_len == !many && !b.out_score == !many && !b.out_norm == !many &&
             (!many || b.norm), VD_E_BADARG, "beam_merge: n > 1 takes norms, the order and every ordered output");
  if (N == 0) return;
  if (skip_empty)
    k_beam_merge<true><<<(unsigned)N, 32, 0, cx.stream>>>(stp, k, G, lam, L, end_token, b, topv, topi, scores_in, scores_out,
                                                          beams_in, beams_out, tokens, parent, pick_ans, pick_len, pick_score);
  else
    k_beam_merge<false><<<(unsigned)N, 32, 0, cx.stream>>>(stp, k, G, lam, L, end_token, b, topv, topi, scores_in, scores_out,
                                                           beams_in, beams_out, tokens, parent, pick_ans, pick_len, pick_score);
  check_launch(cx, "k_beam_merge");
}
void clamp_adam(LaunchCtx& cx, float* W, float* dW, float* m, float* v, int64_t n, float step, float beta1, float beta2,
                float eps, float grad_scale) {
  float omb1 = (float)(1.0 - (double)beta1), omb2 = (float)(1.0 - (double)beta2);
  L1D(k_clamp_adam, n, W, dW, m, v, n, step, beta1, beta2, omb1, omb2, eps, grad_scale);
}
void group_rows_by_token(LaunchCtx& cx, const int32_t* ids, int64_t n, int nv, int32_t* scratch3nv, int32_t* perm,
                         int32_t* sorted_tok) {
  if (n <= 0) return;
  int32_t *counts = scratch3nv, *offsets = scratch3nv + nv, *cursor = scratch3nv + 2 * (int64_t)nv;
  if (cx.deterministic) {                  // stable: the rows of a token in index order
    const int nblk = cdiv(n, TS_ROWS);
    int32_t* hist = cx.scratch_get<int32_t>((int64_t)nblk * nv);
    VD_CUDA_CHECK(cudaMemsetAsync(hist, 0, (size_t)nblk * nv * sizeof(int32_t), cx.stream));
    k_tsort_hist<<<nblk, 32, 0, cx.stream>>>(ids, n, nv, hist);
    check_launch(cx, "k_tsort_hist");
    k_tsort_scan<<<cdiv(nv, 256), 256, 0, cx.stream>>>(hist, nblk, nv, counts);
    check_launch(cx, "k_tsort_scan");
    k_tok_scan<<<1, 1024, 0, cx.stream>>>(counts, offsets, cursor, nv);
    check_launch(cx, "k_tok_scan");
    k_tsort_fill<<<nblk, 32, 0, cx.stream>>>(ids, n, nv, hist, offsets, perm, sorted_tok);
    check_launch(cx, "k_tsort_fill");
    return;
  }
  VD_CUDA_CHECK(cudaMemsetAsync(counts, 0, (size_t)nv * sizeof(int32_t), cx.stream));
  L1D(k_tok_hist, n, ids, n, counts);
  k_tok_scan<<<1, 1024, 0, cx.stream>>>(counts, offsets, cursor, nv);
  check_launch(cx, "k_tok_scan");
  L1D(k_tok_fill, n, ids, n, cursor, perm, sorted_tok);
}
void segsum_rows(LaunchCtx& cx, const float* X, int64_t ldx, const int32_t* perm, const int32_t* sorted_tok, int64_t n,
                 float* out, int ncols) {
  if (n <= 0) return;
  VD_REQUIRE(ncols % 4 == 0 && ldx % 4 == 0, -1, "segsum_rows: ncols, ldx must be multiples of 4");
  if (cx.deterministic) { segsum_det(cx, X, ldx, perm, sorted_tok, n, out, ncols, nullptr, DropCfg{}, 0); return; }
  k_segsum_rows<<<blocks_for(n, SEG_ROWS), 256, 0, cx.stream>>>(X, ldx, perm, sorted_tok, n, out, ncols);
  check_launch(cx, "k_segsum_rows");
}
void segsum_rows16_det(LaunchCtx& cx, const __half* X, int64_t ldx, const int32_t* perm, const int32_t* sorted_tok, int64_t n,
                       float* out, int ncols, const float* inv_scale) {
  segsum_det(cx, X, ldx, perm, sorted_tok, n, out, ncols, inv_scale, DropCfg{}, 0);
}
void slot_reduce(LaunchCtx& cx, float* C, int64_t ldc, const float* ws, int S, int64_t M, int N) {
  L1D(k_slot_reduce, M * N, C, ldc, ws, S, M, N);
}
void fill_l2_flush(LaunchCtx& cx, float* buf, int64_t n) {
  k_fill<<<cx.sm_count * 8, 256, 0, cx.stream>>>(buf, n, 0.f);
  check_launch(cx, "fill_l2_flush");
}

}  // namespace vd
