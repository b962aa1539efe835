// Answer-pool retrieval (DESIGN §18): the k best pool rows of every query row by (score desc, pool index asc), score =
// query . pool embedding (disc.lua:22-29's dot product against every answer of opt_list_<split>), without the (rows, m)
// score matrix in HBM.  Two routes write the same partial lists — per (row, slot) the slot's k best, best first, empty
// entries as (-inf, -1) — and one merge reduces them:
//   tensor cores : k_tc_gemm MODE_TOPK (gemm_tc.cu), one slot per (CTA, column half)
//   CUDA cores   : k_pool_topk_simt below, fp32 scores over 256-column chunks, one slot per chunk column of the grid
// Both keep their scratch independent of m: the slots are bounded by the grid.
#include "../../include/visdial_b200.h"
#include "kernels.cuh"

namespace vd {

namespace {

constexpr unsigned FULL = 0xffffffffu;

constexpr int PS_ROWS = 16;      // query rows per CTA of the CUDA-core route
constexpr int PS_COLS = 256;     // pool rows per chunk (one per thread)
constexpr int POOL_TC_BM = 128;  // the tensor-core route's row block (tc::BM)
constexpr int POOL_TC_NH = 2;    // its slots per CTA (column halves of a tile)

// (v, c) precedes (w, d): score descending, pool index ascending
__device__ __forceinline__ bool pool_before(float v, int c, float w, int d) { return v > w || (v == w && c < d); }

// One CTA: PS_ROWS query rows against the chunks blockIdx.x, blockIdx.x + gridDim.x, ... of 256 pool rows.  Each thread
// scores one pool row against the CTA's query rows in fp32 (one fma chain over H); then warp w merges the chunk into the
// running lists of rows 2w, 2w + 1 (candidates in ascending pool index, so an equal score never displaces an entry).
__global__ void __launch_bounds__(256) k_pool_topk_simt(const float* __restrict__ Q, int64_t ldq, int64_t rows,
                                                        const float* __restrict__ E, int64_t m, int H, int k,
                                                        float* __restrict__ part_v, int32_t* __restrict__ part_i, int slots) {
  extern __shared__ float ps_sm[];
  float* qs = ps_sm;                                   // (PS_ROWS, H)
  float* sc = qs + PS_ROWS * H;                        // (PS_ROWS, PS_COLS)
  float* lv = sc + PS_ROWS * PS_COLS;                  // (PS_ROWS, k)
  int32_t* li = reinterpret_cast<int32_t*>(lv + PS_ROWS * k);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t r0 = (int64_t)blockIdx.y * PS_ROWS;
  for (int i = tid; i < PS_ROWS * H; i += blockDim.x) {
    const int64_t r = r0 + i / H;
    qs[i] = r < rows ? Q[r * ldq + i % H] : 0.f;
  }
  for (int i = tid; i < PS_ROWS * k; i += blockDim.x) { lv[i] = -INFINITY; li[i] = -1; }
  __syncthreads();
  for (int64_t chunk = blockIdx.x; chunk * PS_COLS < m; chunk += gridDim.x) {
    const int64_t j = chunk * PS_COLS + tid;
    float acc[PS_ROWS];
#pragma unroll
    for (int r = 0; r < PS_ROWS; ++r) acc[r] = 0.f;
    if (j < m) {
      const float* e = E + j * H;
#pragma unroll 4
      for (int c = 0; c < H; ++c) {
        const float ev = __ldg(e + c);
#pragma unroll
        for (int r = 0; r < PS_ROWS; ++r) acc[r] = fmaf(qs[r * H + c], ev, acc[r]);
      }
    }
#pragma unroll
    for (int r = 0; r < PS_ROWS; ++r) sc[r * PS_COLS + tid] = acc[r];
    __syncthreads();
    for (int rr = 2 * warp; rr < 2 * warp + 2; ++rr) {
      if (r0 + rr >= rows) break;                      // warp-uniform
      float* rv = lv + rr * k;
      int32_t* ri = li + rr * k;
      float thr = rv[k - 1];
      for (int g = 0; g < PS_COLS / 32; ++g) {
        const int64_t jj = chunk * PS_COLS + g * 32 + lane;
        const float x = sc[rr * PS_COLS + g * 32 + lane];
        unsigned msk = __ballot_sync(FULL, jj < m && x > thr);
        while (msk) {
          const int src = __ffs(msk) - 1;
          msk &= msk - 1;
          const float cv = __shfl_sync(FULL, x, src);
          if (!(cv > thr)) continue;                   // thr rose since the ballot (warp-uniform)
          if (lane == 0) {
            int pos = k - 1;
            while (pos > 0 && cv > rv[pos - 1]) { rv[pos] = rv[pos - 1]; ri[pos] = ri[pos - 1]; --pos; }
            rv[pos] = cv; ri[pos] = (int32_t)(chunk * PS_COLS + g * 32 + src);
          }
          __syncwarp();
          thr = rv[k - 1];
        }
      }
    }
    __syncthreads();
  }
  for (int i = tid; i < PS_ROWS * k; i += blockDim.x) {
    const int64_t r = r0 + i / k;
    if (r >= rows) continue;
    const int64_t o = (r * slots + blockIdx.x) * k + i % k;
    part_v[o] = lv[i]; part_i[o] = li[i];
  }
}

// One CTA per row: the k best of the row's partial lists, in k_logsoftmax_topk_rows' way — each thread keeps the KMAX best
// entries of its strided slots in registers (a slot's list is sorted, so its first entry that does not beat the thread's
// KMAX-th ends it), then the CTA pops k winners from the thread heads.  tc_grid > 0: the tensor-core route's slots, of which
// only those whose CTA walked the row's row block were written.
template <int KMAX>
__global__ void __launch_bounds__(128) k_pool_topk_merge(const float* __restrict__ part_v, const int32_t* __restrict__ part_i,
                                                         int slots, int k, int tc_num_n, int tc_grid, float* __restrict__ topv,
                                                         int32_t* __restrict__ topi) {
  __shared__ float sv[4];
  __shared__ int si[4];
  __shared__ int win;
  const int64_t r = blockIdx.x;
  float lv[KMAX]; int lc[KMAX];
#pragma unroll
  for (int i = 0; i < KMAX; ++i) { lv[i] = -INFINITY; lc[i] = 0x7fffffff; }
  const int64_t lo = (r / POOL_TC_BM) * (int64_t)tc_num_n, hi = lo + tc_num_n;
  for (int s = threadIdx.x; s < slots; s += blockDim.x) {
    if (tc_grid > 0) {                                 // first tile of CTA s / NH at or after lo; the CTA walked the block iff < hi
      const int64_t c = s / POOL_TC_NH;
      const int64_t first = c >= lo ? c : c + (lo - c + tc_grid - 1) / tc_grid * tc_grid;
      if (first >= hi) continue;
    }
    const int64_t base = (r * slots + s) * k;
    for (int e = 0; e < k; ++e) {
      float v = part_v[base + e];
      int ci = part_i[base + e];
      if (ci < 0 || !pool_before(v, ci, lv[KMAX - 1], lc[KMAX - 1])) break;
#pragma unroll
      for (int i = 0; i < KMAX; ++i) {
        if (pool_before(v, ci, lv[i], lc[i])) {
          const float tv = lv[i]; const int tc = lc[i];
          lv[i] = v; lc[i] = ci; v = tv; ci = tc;
        }
      }
    }
  }
  for (int j = 0; j < k; ++j) {
    float bv = lv[0]; int bi = lc[0];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(FULL, bv, o);
      const int oi = __shfl_xor_sync(FULL, bi, o);
      if (pool_before(ov, oi, bv, bi)) { bv = ov; bi = oi; }
    }
    if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = bv; si[threadIdx.x >> 5] = bi; }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 1; w < (int)(blockDim.x >> 5); ++w)
        if (pool_before(sv[w], si[w], bv, bi)) { bv = sv[w]; bi = si[w]; }
      topv[r * k + j] = bv; topi[r * k + j] = bi;
      win = bi;
    }
    __syncthreads();
    if (lc[0] == win) {                                // pool indices are unique: only the owner pops
#pragma unroll
      for (int i = 0; i < KMAX - 1; ++i) { lv[i] = lv[i + 1]; lc[i] = lc[i + 1]; }
      lv[KMAX - 1] = -INFINITY; lc[KMAX - 1] = 0x7fffffff;
    }
    __syncthreads();
  }
}

__global__ void k_gather_pool_rows(const int32_t* __restrict__ pool_tok, int w, const int32_t* __restrict__ idx, int64_t idx_ld,
                                   int64_t n, int32_t* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * w) return;
  const int64_t b = i / w;
  out[i] = pool_tok[(int64_t)idx[b * idx_ld] * w + i % w];
}

size_t simt_smem(int H, int k) { return (size_t)(PS_ROWS * H + PS_ROWS * PS_COLS + 2 * PS_ROWS * k) * sizeof(float); }

}  // namespace

int pool_topk_simt_slots(const LaunchCtx& cx, int64_t rows, int64_t m) {
  const int64_t row_blocks = (rows + PS_ROWS - 1) / PS_ROWS;
  const int64_t want = std::max<int64_t>(1, 2LL * cx.sm_count / row_blocks);
  return (int)std::min<int64_t>((m + PS_COLS - 1) / PS_COLS, want);
}

void pool_topk_simt(LaunchCtx& cx, int slots, const float* Q, int64_t ldq, int64_t rows, const float* E, int64_t m, int H, int k,
                    float* part_v, int32_t* part_i) {
  VD_REQUIRE(rows >= 1 && m >= 1 && H >= 1 && k >= 1 && k <= 32 && slots >= 1, VD_E_BADARG, "pool_topk_simt: shape");
  const size_t smem = simt_smem(H, k);
  VD_REQUIRE(smem <= 227 * 1024, VD_E_BADARG, "pool_topk_simt: H too large for the query tile");
  static bool attr_set = false;
  if (!attr_set) {
    VD_CUDA_CHECK(cudaFuncSetAttribute(k_pool_topk_simt, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    attr_set = true;
  }
  dim3 grid((unsigned)slots, (unsigned)((rows + PS_ROWS - 1) / PS_ROWS));
  k_pool_topk_simt<<<grid, 256, smem, cx.stream>>>(Q, ldq, rows, E, m, H, k, part_v, part_i, slots);
  check_launch(cx, "k_pool_topk_simt");
}

void pool_topk_merge(LaunchCtx& cx, const float* part_v, const int32_t* part_i, int64_t rows, int slots, int k, int tc_num_n,
                     int tc_grid, float* topv, int32_t* topi) {
  VD_REQUIRE(k >= 1 && k <= 32 && slots >= 1, VD_E_BADARG, "pool_topk_merge: k / slots");
  if (rows <= 0) return;
  const unsigned g = (unsigned)rows;
  if (k <= 4) k_pool_topk_merge<4><<<g, 128, 0, cx.stream>>>(part_v, part_i, slots, k, tc_num_n, tc_grid, topv, topi);
  else if (k <= 8) k_pool_topk_merge<8><<<g, 128, 0, cx.stream>>>(part_v, part_i, slots, k, tc_num_n, tc_grid, topv, topi);
  else if (k <= 16) k_pool_topk_merge<16><<<g, 128, 0, cx.stream>>>(part_v, part_i, slots, k, tc_num_n, tc_grid, topv, topi);
  else k_pool_topk_merge<32><<<g, 128, 0, cx.stream>>>(part_v, part_i, slots, k, tc_num_n, tc_grid, topv, topi);
  check_launch(cx, "k_pool_topk_merge");
}

void gather_pool_rows(LaunchCtx& cx, const int32_t* pool_tok, int w, const int32_t* idx, int64_t idx_ld, int64_t n, int32_t* out) {
  if (n <= 0) return;
  const int64_t total = n * w;
  k_gather_pool_rows<<<cdiv(total, 256), 256, 0, cx.stream>>>(pool_tok, w, idx, idx_ld, n, out);
  check_launch(cx, "k_gather_pool_rows");
}

}  // namespace vd
