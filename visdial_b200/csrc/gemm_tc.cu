// Dense contractions on the Hopper tensor cores: wgmma kind tf32 (fp32 operands in shared memory, TF32 multiply,
// fp32 accumulate in registers), operands staged by TMA (128B-swizzled tiles) through an mbarrier ring, one
// persistent CTA per SM, warp-specialised: warpgroup 0 = TMA producer (one thread), warpgroups 1-2 = consumers, each
// contracting a 64-row half of the 128-row tile; the accumulators then go through shared memory so that the fused
// pointwise epilogue runs "thread = row" (consumer warp w: rows 32 (w % 4) .., column half w / 4).
//
//   MODE_GENERIC : C = act(beta*C + bias + A B^T)                          (nn.Linear and friends)
//   MODE_LSTM_FWD: gates = A_h Wh^T (+ x-projection) -> SeqLSTM pointwise   (one launch per time step)
//   MODE_LSTM_BWD: dh = da_{t+1} Wh -> SeqLSTM backward pointwise -> da_t   (one launch per time step)
//   k_tc_atb     : C += A^T B with both operands MN-major                   (weight gradients, split-K)
#include <cuda.h>
#include <mutex>
#include "kernels.cuh"
#include "tc_ptx.cuh"

namespace vd {
namespace tc {

constexpr int BM = 128;          // rows per tile (two 64-row wgmma slabs)
constexpr int BK = 32;           // fp32 elements per k-block = one 128-byte swizzle row
constexpr int MMA_K = 8;         // tf32: 32 bytes per instruction
constexpr int EPI_WARPS = 8;     // the consumer warps: 2 per 32-row quarter, each takes half of the tile's columns
constexpr int GEMM_THREADS = 128 + 32 * EPI_WARPS;

enum { MODE_GENERIC = 0, MODE_LSTM_FWD = 1, MODE_LSTM_BWD = 2, MODE_LSE = 3, MODE_DLOGIT = 4, MODE_SAMPLE = 5 };
// MODE_LSE    : vocabulary projection whose (rows, V) logits never leave the chip: per row and column slice only the running
//               max, the sum of exponentials and the target's logit are written (gen.lua:23-24 + the criterion of model.lua:33-36
//               / utils.computeLhood, utils.lua:86-102)
// MODE_DLOGIT : the same contraction recomputed in the backward pass with the epilogue  C = keep * (exp(x - lse[row]) - onehot)
// MODE_SAMPLE : MODE_LSE's statistics plus the slice's best Gumbel key x / T + g (common.cuh), its class and its logit
//               (the sampling step of model.lua:584-593 without the logits in HBM)

struct Params {
  int M, N, K;                    // GEMM sizes (N = output columns; LSTM_FWD: N = 4H, LSTM_BWD: N = H)
  int H;
  // generic
  float* C; int64_t ldc; float beta; const float* bias; int act;
  // lstm fwd
  float* gates;                   // (R,4H): in = x-projection pre-activations (if has_xproj), out = activated gates
  int has_xproj;
  const float* ptable; const int32_t* tok;   // optional gathered x-projection: ptable[tok[r], 4H]
  const float* c_prev; float* c_out; float* h_out; const int32_t* mask_ids;
  // lstm bwd
  const float* gsave; const float* c_cur; const float* dh_ext; float* dc_carry; float* da;
  // fused vocabulary softmax (MODE_LSE / MODE_DLOGIT): 1-based target class per row (0 = none), maskzero ids per row
  const int32_t* tgt; const int32_t* row_ids; const float* lse;
  float* part_max; float* part_sum; float* tgt_logit; int nparts;      // (M, nparts) partials, nparts = column tiles * slices
  // MODE_SAMPLE: (M, nparts) best key, its class and its logit
  float* part_key; int32_t* part_cls; float* part_x; SampleCfg smp;
};

__device__ __forceinline__ void ld8(const float* p, float* d) {
  const float4 x0 = __ldg(reinterpret_cast<const float4*>(p)), x1 = __ldg(reinterpret_cast<const float4*>(p) + 1);
  d[0] = x0.x; d[1] = x0.y; d[2] = x0.z; d[3] = x0.w; d[4] = x1.x; d[5] = x1.y; d[6] = x1.z; d[7] = x1.w;
}
__device__ __forceinline__ void add8(const float* p, float* d) {
  const float4 x0 = __ldg(reinterpret_cast<const float4*>(p)), x1 = __ldg(reinterpret_cast<const float4*>(p) + 1);
  d[0] += x0.x; d[1] += x0.y; d[2] += x0.z; d[3] += x0.w; d[4] += x1.x; d[5] += x1.y; d[6] += x1.z; d[7] += x1.w;
}
__device__ __forceinline__ void st8(float* p, const float* v) {
  reinterpret_cast<float4*>(p)[0] = make_float4(v[0], v[1], v[2], v[3]);
  reinterpret_cast<float4*>(p)[1] = make_float4(v[4], v[5], v[6], v[7]);
}
// streaming store: saved activations are not read again before the backward pass — keep them out of L2's way
__device__ __forceinline__ void st8_cs(float* p, const float* v) {
  __stcs(reinterpret_cast<float4*>(p), make_float4(v[0], v[1], v[2], v[3]));
  __stcs(reinterpret_cast<float4*>(p) + 1, make_float4(v[4], v[5], v[6], v[7]));
}

// Epilogue staging of the generic / d-logit modes: per consumer warp one array of [32 rows][16 floats].  The 16-byte
// chunks of a row are XOR-swizzled by (row>>1)&3 so that both access patterns are bank-conflict free: "thread = row" and
// "4 lanes = one row's 64 bytes" (coalesced 64-byte runs on the global side).  C leaves by TMA tensor stores.
constexpr int STG_ARR_BYTES = 32 * 16 * 4;
template <int MODE> struct StageCfg {
  static constexpr bool ON = MODE == MODE_GENERIC || MODE == MODE_DLOGIT;
  static constexpr int ARR = ON ? 1 : 0;
  static constexpr int BYTES = EPI_WARPS * ARR * STG_ARR_BYTES;
};
template <int BN, int STG_BYTES = 0> struct SmemLayout {
  static constexpr int A_BYTES = BM * BK * 4;        // 16 KB
  static constexpr int B_BYTES = BN * BK * 4;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int ACC_BYTES = BN * ACC_LD * 4;  // the accumulator tile on its way to the epilogue
  static constexpr int WANT = (B_BYTES == 16384) ? 6 : (B_BYTES == 8192) ? 8 : 10;   // small tiles are latency-bound: deeper
  static constexpr int FIT = (232448 - 1024 - 256 - STG_BYTES - ACC_BYTES) / STAGE_BYTES;
  static constexpr int STAGES = WANT < FIT ? WANT : FIT;
  static constexpr int TOTAL = STAGES * STAGE_BYTES + STG_BYTES + ACC_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
};

__device__ __forceinline__ float4* stg_at(float* stg, int arr, int row, int q) {
  return reinterpret_cast<float4*>(stg + (arr * 32 + row) * 16 + ((q ^ ((row >> 1) & 3)) << 2));
}
// global -> staging: `mine` = this lane's row base (16 floats) or nullptr (zeros); coalesced 4 lanes per row, cp.async;
// the caller ends the group with stg_load_wait().
__device__ __forceinline__ void stg_load(float* stg, int arr, const float* mine, int lane) {
#pragma unroll
  for (int ps = 0; ps < 4; ++ps) {
    const int row = ps * 8 + (lane >> 2), q = lane & 3;
    const float* src = shfl_ptr(mine, row);
    float4* dst = stg_at(stg, arr, row, q);
    if (src) asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst)), "l"(src + q * 4) : "memory");
    else *dst = make_float4(0.f, 0.f, 0.f, 0.f);
  }
}
struct EpiMaps { CUtensorMap g4; };      // C as 64B-swizzled boxes of 32 rows x 16 floats
__device__ __forceinline__ void stg_load_wait() {
  asm volatile("cp.async.wait_all;" ::: "memory");
  __syncwarp();
}
__device__ __forceinline__ void stg_get8(float* stg, int arr, int row, int sub, float* d) {
  const float4 a = *stg_at(stg, arr, row, sub * 2), b = *stg_at(stg, arr, row, sub * 2 + 1);
  d[0] = a.x; d[1] = a.y; d[2] = a.z; d[3] = a.w; d[4] = b.x; d[5] = b.y; d[6] = b.z; d[7] = b.w;
}
__device__ __forceinline__ void stg_put8(float* stg, int arr, int row, int sub, const float* v) {
  *stg_at(stg, arr, row, sub * 2) = make_float4(v[0], v[1], v[2], v[3]);
  *stg_at(stg, arr, row, sub * 2 + 1) = make_float4(v[4], v[5], v[6], v[7]);
}

template <int BN> __device__ __forceinline__ void wgmma_tf32(float (&d)[BN / 2], uint64_t a, uint64_t b, uint32_t acc) {
  if constexpr (BN == 128) wgmma_tf32_n128(d, a, b, acc);
  else if constexpr (BN == 64) wgmma_tf32_n64(d, a, b, acc);
  else { static_assert(BN == 32, "tile width"); wgmma_tf32_n32(d, a, b, acc); }
}

// ------------------------------------------------------------------------------------------------
template <int BN, int MODE>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
k_tc_gemm(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
          const __grid_constant__ EpiMaps em, const Params p) {
  using SC = StageCfg<MODE>;
  using L = SmemLayout<BN, SC::BYTES>;
  constexpr int NH = EPI_WARPS / 4;                  // consumer warps per 32-row quarter = column slices per tile
  constexpr int STAGES = L::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  float* stg_all = (float*)(smem + STAGES * L::STAGE_BYTES);
  float* acc = (float*)(smem + STAGES * L::STAGE_BYTES + SC::BYTES);
  uint64_t* full = (uint64_t*)(smem + STAGES * L::STAGE_BYTES + SC::BYTES + L::ACC_BYTES);
  uint64_t* empty = full + STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_m = (p.M + BM - 1) / BM;
  const int num_n = (p.N + BN - 1) / BN;
  const int num_tiles = num_m * num_n;
  const int num_kb = (p.K + BK - 1) / BK;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < 4) {
    if (threadIdx.x == 0) {
      // ===== TMA producer =====
      int s = 0; uint32_t ph = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m0 = (tile / num_n) * BM;
        const int nt = tile % num_n;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty[s], ph ^ 1);
          uint8_t* sa = smem + s * L::STAGE_BYTES;
          uint8_t* sb = sa + L::A_BYTES;
          mbar_expect_tx(&full[s], L::STAGE_BYTES);
          tma_load_2d(sa, &tmA, &full[s], kb * BK, m0);
          if (MODE == MODE_LSTM_FWD) {
            // interleave the 4 gate blocks of this hidden-unit slice: tile columns = [i | f | o | g]
            constexpr int HB = BN / 4;
#pragma unroll
            for (int g = 0; g < 4; ++g) tma_load_2d(sb + g * HB * BK * 4, &tmB, &full[s], kb * BK, g * p.H + nt * HB);
          } else {
            tma_load_2d(sb, &tmB, &full[s], kb * BK, nt * BN);
          }
          if (++s == STAGES) { s = 0; ph ^= 1; }
        }
      }
    }
  } else {
    // ===== consumers: warpgroup wg contracts rows [64 wg, 64 wg + 64) of the tile, then all 8 warps run the epilogue =====
    const int cw = warp - 4, wg = cw >> 2;
    const int q = cw & 3;
    const int half = cw >> 2;
    const float* arow = acc + q * 32 + lane;
    int s = 0; uint32_t ph = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int m0 = (tile / num_n) * BM;
      const int nt = tile % num_n;
      float d[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) d[i] = 0.f;
      int prev = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full[s], ph);
        const uint32_t sa = smem_u32(smem + s * L::STAGE_BYTES);
        const uint64_t adesc = make_desc(sa + wg * 64 * 128, 16, 1024), bdesc = make_desc(sa + L::A_BYTES, 16, 1024);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / MMA_K; ++k)
          wgmma_tf32<BN>(d, adesc + (uint64_t)(k * MMA_K * 4 >> 4), bdesc + (uint64_t)(k * MMA_K * 4 >> 4), (kb | k) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();                              // the previous k-block's MMAs are done with their stage
        if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty[prev]);
        prev = s;
        if (++s == STAGES) { s = 0; ph ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_hold(d);
      if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty[prev]);
      bar_named(1, 32 * EPI_WARPS);                    // the previous tile's epilogue is done with the accumulator tile
      acc_store(acc, d, wg * 64);
      bar_named(1, 32 * EPI_WARPS);
      const int64_t row = (int64_t)m0 + q * 32 + lane;
      const bool row_ok = row < p.M;

      if (MODE == MODE_LSE || MODE == MODE_SAMPLE) {
        // online softmax statistics of this warp's column slice of the tile: nothing but (max, sum exp, target logit) leaves
        const int n0 = nt * BN;
        const int tcol = (MODE == MODE_LSE && row_ok) ? p.tgt[row] - 1 : -1;
        float mrun = -INFINITY, srun = 0.f, tl = 0.f;
        bool has = false;
        // MODE_SAMPLE: the slice's best (key, class, logit); columns ascend, so a strictly greater key keeps ties on the
        // lower class.  N % 4 == 0 and 8-column groups: element (row, n0 + c) starts a Philox quadruple.
        float bkey = -INFINITY, bx = 0.f;
        int bcls = 0x7fffffff;
        const uint64_t ebase = MODE == MODE_SAMPLE ? (uint64_t)(p.smp.row_offset + row * p.smp.row_stride) * (uint64_t)p.N : 0;
#pragma unroll 1
        for (int c = half * (BN / NH); c < (half + 1) * (BN / NH); c += 8) {
          if (n0 + c >= p.N) break;                 // warp-uniform
          float v[8];
          acc_ld8(arow, c, v);
          float mx = -INFINITY;
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int n = n0 + c + j;
            const bool ok = n < p.N;
            const float x = ok ? v[j] + (p.bias ? __ldg(p.bias + n) : 0.f) : -INFINITY;
            v[j] = x;
            if (ok && n == tcol) { tl = x; has = true; }
            mx = fmaxf(mx, x);
          }
          const float mnew = fmaxf(mrun, mx);
          float add = 0.f;
#pragma unroll
          for (int j = 0; j < 8; ++j) add += __expf(v[j] - mnew);      // exp(-inf) = 0 for the clipped columns
          srun = srun * __expf(mrun - mnew) + add;
          mrun = mnew;
          if (MODE == MODE_SAMPLE && row_ok) {
#pragma unroll
            for (int h4 = 0; h4 < 2; ++h4) {
              const int nb = n0 + c + 4 * h4;
              if (nb >= p.N) break;
              float y[4];
              float ymax = -INFINITY;
#pragma unroll
              for (int j = 0; j < 4; ++j) { y[j] = v[4 * h4 + j] / p.smp.temperature; ymax = fmaxf(ymax, y[j]); }
              if (ymax + GUMBEL_MAX < bkey) continue;          // no key of the quadruple can reach the best one
              uint32_t o[4];
              sample_words(p.smp, (ebase + (uint64_t)nb) >> 2, o);
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                const float key = y[j] + gumbel_of_word(o[j]);
                if (key > bkey) { bkey = key; bcls = nb + j; bx = v[4 * h4 + j]; }
              }
            }
          }
        }
        if (row_ok) {
          const int64_t pi = row * p.nparts + nt * NH + half;
          p.part_max[pi] = mrun; p.part_sum[pi] = srun;
          if (MODE == MODE_SAMPLE) { p.part_key[pi] = bkey; p.part_cls[pi] = bcls; p.part_x[pi] = bx; }
          else if (has) p.tgt_logit[row] = tl;
        }
      } else if (MODE == MODE_GENERIC || MODE == MODE_DLOGIT) {
        // 16 output columns at a time through the warp's staging array; C leaves (and, for beta != 0, enters)
        // as 64-byte-swizzled boxes: TMA tensor store / cp.async load.  Rows >= M and columns >= N are clipped.
        const int n0 = nt * BN;
        float* stg = stg_all + cw * (SC::ARR * 32 * 16);
#pragma unroll 1
        for (int c = half * (BN / NH); c < (half + 1) * (BN / NH); c += 16) {
          if (n0 + c >= p.N) break;                 // warp-uniform
          if (lane == 0) bulk_wait_read0();
          __syncwarp();
          if (p.beta != 0.f) {
            const bool full16 = n0 + c + 16 <= p.N;
            stg_load(stg, 0, (row_ok && full16) ? p.C + row * p.ldc + n0 + c : nullptr, lane);
            stg_load_wait();
            if (!full16 && row_ok) {               // ragged last group: element-wise
#pragma unroll
              for (int sub = 0; sub < 2; ++sub) {
                float t[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) { const int n = n0 + c + sub * 8 + j; t[j] = n < p.N ? p.C[row * p.ldc + n] : 0.f; }
                stg_put8(stg, 0, lane, sub, t);
              }
            }
          }
#pragma unroll
          for (int sub = 0; sub < 2; ++sub) {
            float v[8], old[8];
            acc_ld8(arow, c + sub * 8, v);
              if (p.beta != 0.f) stg_get8(stg, 0, lane, sub, old);
            if (MODE == MODE_DLOGIT) {
              // d loss / d logit of the sum criterion: softmax - onehot on kept rows (input token != pad, target != pad)
              const int tg = row_ok ? p.tgt[row] : 0;
              const bool keepr = row_ok && tg > 0 && p.row_ids[row] != 0;
              const float l = keepr ? p.lse[row] : 0.f;
#pragma unroll
              for (int j = 0; j < 8; ++j) {
                const int n = n0 + c + sub * 8 + j;
                const float x = v[j] + ((p.bias && n < p.N) ? __ldg(p.bias + n) : 0.f);
                v[j] = keepr ? __expf(x - l) - (n == tg - 1 ? 1.f : 0.f) : 0.f;
              }
            } else {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const int n = n0 + c + sub * 8 + j;
              float x = v[j];
              if (p.bias && n < p.N) x += __ldg(p.bias + n);
              if (p.beta != 0.f) x += p.beta * old[j];
              v[j] = p.act == 1 ? ftanh(x) : x;
            }
            }
            stg_put8(stg, 0, lane, sub, v);
          }
          fence_proxy_async_smem();
          __syncwarp();
          if (lane == 0) { tma_store_2d(&em.g4, stg, n0 + c, m0 + q * 32); bulk_commit(); }
          __syncwarp();
        }
      } else if (MODE == MODE_LSTM_FWD) {
        constexpr int HB = BN / 4;                  // hidden units per tile
        const int H = p.H, j0 = nt * HB;
        const bool masked = row_ok && p.mask_ids && p.mask_ids[row] == 0;
        const float* prow = (row_ok && p.ptable) ? p.ptable + (int64_t)p.tok[row] * 4 * H : nullptr;
        float* grow = p.gates ? p.gates + row * 4 * H : nullptr;
#pragma unroll 1
        for (int c = half * (HB / NH); c < (half + 1) * (HB / NH); c += 8) {
          const int j = j0 + c;
          float a[4][8], x[4][8], cp[8];
          // issue the global loads first so that they overlap the accumulator read
          if (row_ok && !masked) {
#pragma unroll
            for (int g = 0; g < 4; ++g) {
              if (p.bias) ld8(p.bias + g * H + j, x[g]);
              else {
#pragma unroll
                for (int e = 0; e < 8; ++e) x[g][e] = 0.f;
              }
              if (p.has_xproj) add8(grow + g * H + j, x[g]);
              if (prow) add8(prow + g * H + j, x[g]);
            }
            if (p.c_prev) ld8(p.c_prev + row * H + j, cp);
            else {
#pragma unroll
              for (int e = 0; e < 8; ++e) cp[e] = 0.f;
            }
          }
#pragma unroll
          for (int g = 0; g < 4; ++g) acc_ld8(arow, g * HB + c, a[g]);
          if (row_ok) {
            float cn[8], hn[8];
            if (masked) {
#pragma unroll
              for (int e = 0; e < 8; ++e) { a[0][e] = a[1][e] = a[2][e] = a[3][e] = 0.f; cn[e] = 0.f; hn[e] = 0.f; }
            } else {
#pragma unroll
              for (int e = 0; e < 8; ++e) {
                const float zi = (p.K ? a[0][e] : 0.f) + x[0][e], zf = (p.K ? a[1][e] : 0.f) + x[1][e];
                const float zo = (p.K ? a[2][e] : 0.f) + x[2][e], zg = (p.K ? a[3][e] : 0.f) + x[3][e];
                const float gi = fsigmoid(zi), gf = fsigmoid(zf), go = fsigmoid(zo), gg = ftanh(zg);
                const float c_ = gf * cp[e] + gi * gg;
                a[0][e] = gi; a[1][e] = gf; a[2][e] = go; a[3][e] = gg;
                cn[e] = c_; hn[e] = go * ftanh(c_);
              }
            }
            if (grow) {
#pragma unroll
              for (int g = 0; g < 4; ++g) st8_cs(grow + g * H + j, a[g]);
            }
            st8(p.c_out + row * H + j, cn);
            st8(p.h_out + row * H + j, hn);
          }
          __syncwarp();
        }
      } else {   // MODE_LSTM_BWD: accumulator = dh_rec for hidden units [nt*BN, nt*BN + BN)
        const int H = p.H, j0 = nt * BN;
        const bool masked = row_ok && p.mask_ids && p.mask_ids[row] == 0;
#pragma unroll 1
        for (int c = half * (BN / NH); c < (half + 1) * (BN / NH); c += 8) {
          const int j = j0 + c;
          float dh[8], g[4][8], cp[8], cc[8], dc[8], ex[8];
          if (row_ok && !masked) {
#pragma unroll
            for (int gg = 0; gg < 4; ++gg) ld8(p.gsave + row * 4 * H + gg * H + j, g[gg]);
            if (p.c_prev) ld8(p.c_prev + row * H + j, cp);
            else {
#pragma unroll
              for (int e = 0; e < 8; ++e) cp[e] = 0.f;
            }
            ld8(p.c_cur + row * H + j, cc);
            ld8(p.dc_carry + row * H + j, dc);
            if (p.dh_ext) ld8(p.dh_ext + row * H + j, ex);
            else {
#pragma unroll
              for (int e = 0; e < 8; ++e) ex[e] = 0.f;
            }
          }
          acc_ld8(arow, c, dh);
          if (row_ok) {
            float out[4][8], dcn[8];
            if (masked) {
#pragma unroll
              for (int e = 0; e < 8; ++e) { out[0][e] = out[1][e] = out[2][e] = out[3][e] = 0.f; dcn[e] = 0.f; }
            } else {
#pragma unroll
              for (int e = 0; e < 8; ++e) {
                const float dhe = (p.K ? dh[e] : 0.f) + ex[e];
                const float gi = g[0][e], gf = g[1][e], go = g[2][e], gg_ = g[3][e];
                const float tcv = ftanh(cc[e]);
                const float d = dc[e] + dhe * go * (1.f - tcv * tcv);
                out[0][e] = d * gg_ * gi * (1.f - gi);
                out[1][e] = d * cp[e] * gf * (1.f - gf);
                out[2][e] = dhe * tcv * go * (1.f - go);
                out[3][e] = d * gi * (1.f - gg_ * gg_);
                dcn[e] = d * gf;
              }
            }
#pragma unroll
            for (int gg = 0; gg < 4; ++gg) st8(p.da + row * 4 * H + gg * H + j, out[gg]);
            st8(p.dc_carry + row * H + j, dcn);
          }
          __syncwarp();
        }
      }
    }
    if (SC::ON && lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");   // all TMA stores performed
  }
}

// ------------------------------------------------------------------------------------------------
// Weight gradients: C[M,N] += sum_k A[k,m] B[k,n].  Both operands are "MN-major" (the contraction index k is the row
// index of the activations in HBM), and wgmma takes tf32 operands K-major only: the two consumer warpgroups load each
// k-block (32 rows of A and B) from global memory and transpose it into the K-major 128B-swizzled layout while storing
// it (double-buffered: the next k-block's loads fly while the current one's MMAs run).  One (tile, K-split) per CTA; the
// fp32 partial sums are reduced into C with red.global.add.
constexpr int ATB_KB = 32;       // k-rows per k-block (4 MMAs)
constexpr int ATB_BN = 128;
constexpr int ATB_THREADS = 256;
constexpr int ATB_OP_BYTES = 128 * ATB_KB * 4;            // one operand tile: 128 rows of 128 B
constexpr int ATB_SMEM = 2 * 2 * ATB_OP_BYTES + 1024;
struct AtbParams { int M, N; int64_t K, k_per_split; const float* A; int64_t lda; const float* B; int64_t ldb; float* C; int64_t ldc; };

// thread's share of a k-block of one operand: 32 k-rows x 128 columns = 1024 chunks of (4 consecutive k, one column), 4 per
// thread; a warp reads 32 consecutive columns of a k-row per load (coalesced), zero outside the operand
__device__ __forceinline__ void atb_load(float4 (&r)[4], const float* X, int64_t ldx, int ncols, int c0, int64_t k0, int64_t kend) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int idx = (int)threadIdx.x + ATB_THREADS * i;
    const int c = c0 + (idx & 127);
    const int64_t k = k0 + (idx >> 7) * 4;
    float v[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) v[e] = (c < ncols && k + e < kend) ? __ldg(X + (k + e) * ldx + c) : 0.f;
    r[i] = make_float4(v[0], v[1], v[2], v[3]);
  }
}
// chunk (k/4, col) of the K-major tile: row `col` of 128 bytes, 16-byte chunk k/4 swizzled with col % 8 — one vector store;
// the 8 lanes of a store phase hold 8 consecutive columns, i.e. 8 different chunks: no bank conflict
__device__ __forceinline__ void atb_store(uint8_t* tile, const float4 (&r)[4]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int idx = (int)threadIdx.x + ATB_THREADS * i;
    const int col = idx & 127, kq = idx >> 7;
    *reinterpret_cast<float4*>(tile + col * 128 + ((kq ^ (col & 7)) << 4)) = r[i];
  }
}

__global__ void __launch_bounds__(ATB_THREADS, 1)
k_tc_atb(const AtbParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  const int wg = threadIdx.x >> 7;
  const int num_n = (p.N + ATB_BN - 1) / ATB_BN;
  const int m0 = (blockIdx.x / num_n) * BM, n0 = (blockIdx.x % num_n) * ATB_BN;
  const int64_t kbeg = (int64_t)blockIdx.y * p.k_per_split;
  const int64_t kend = min(p.K, kbeg + p.k_per_split);
  const int num_kb = (int)((kend - kbeg + ATB_KB - 1) / ATB_KB);
  if (num_kb <= 0) return;

  float d[ATB_BN / 2];
#pragma unroll
  for (int i = 0; i < ATB_BN / 2; ++i) d[i] = 0.f;
  float4 ra[4], rb[4];
  atb_load(ra, p.A, p.lda, p.M, m0, kbeg, kend);
  atb_load(rb, p.B, p.ldb, p.N, n0, kbeg, kend);
  atb_store(smem, ra);
  atb_store(smem + ATB_OP_BYTES, rb);
  fence_proxy_async_smem();
  __syncthreads();
  for (int kb = 0; kb < num_kb; ++kb) {
    uint8_t* cur = smem + (kb & 1) * 2 * ATB_OP_BYTES;
    const uint32_t sa = smem_u32(cur);
    const uint64_t adesc = make_desc(sa + wg * 64 * 128, 16, 1024), bdesc = make_desc(sa + ATB_OP_BYTES, 16, 1024);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < ATB_KB / MMA_K; ++k)
      wgmma_tf32_n128(d, adesc + (uint64_t)(k * MMA_K * 4 >> 4), bdesc + (uint64_t)(k * MMA_K * 4 >> 4), (kb | k) ? 1u : 0u);
    wgmma_commit();
    if (kb + 1 < num_kb) {
      const int64_t k0 = kbeg + (int64_t)(kb + 1) * ATB_KB;
      atb_load(ra, p.A, p.lda, p.M, m0, k0, kend);
      atb_load(rb, p.B, p.ldb, p.N, n0, k0, kend);
      uint8_t* nxt = smem + ((kb + 1) & 1) * 2 * ATB_OP_BYTES;   // its last readers (k-block kb - 1) have completed
      atb_store(nxt, ra);
      atb_store(nxt + ATB_OP_BYTES, rb);
      fence_proxy_async_smem();
    }
    wgmma_wait<0>();
    wgmma_hold(d);
    __syncthreads();
  }
  // fragment -> red.add into C
  const int lane = threadIdx.x & 31, w = (threadIdx.x >> 5) & 3;
  const int r0 = m0 + wg * 64 + 16 * w + (lane >> 2), c0 = n0 + 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < ATB_BN / 8; ++j) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = r0 + 8 * h, n = c0 + 8 * j;
      if (m < p.M) {
        float* crow = p.C + (int64_t)m * p.ldc + n;
        if (n < p.N) atomicAdd(crow, d[4 * j + 2 * h]);
        if (n + 1 < p.N) atomicAdd(crow + 1, d[4 * j + 2 * h + 1]);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ host
PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = (PFN_encodeTiled)p;
  });
  VD_REQUIRE(fn != nullptr, -3, "cuTensorMapEncodeTiled not available from the driver");
  return fn;
}

// 2-D fp32 tensor map: `rows` x `cols` (cols contiguous), row pitch ld floats, box = box_rows x box_cols floats
static CUtensorMap make_tmap(const float* base, int64_t rows, int64_t cols, int64_t ld, int box_rows, int box_cols = BK,
                             CUtensorMapSwizzle swz = CU_TENSOR_MAP_SWIZZLE_128B) {
  CUtensorMap tm;
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 4};
  cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = get_encode()(&tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)base, dims, strides, box, estr,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char buf[256];
    snprintf(buf, sizeof(buf), "cuTensorMapEncodeTiled failed (%d): base %p rows %lld cols %lld ld %lld box %dx%d", (int)r, (void*)base,
             (long long)rows, (long long)cols, (long long)ld, box_rows, box_cols);
    throw CudaError(-3, buf);
  }
  return tm;
}

static bool tma_ok(const float* p, int64_t ld) { return ((uintptr_t)p % 16 == 0) && (ld % 4 == 0); }

template <int BN, int MODE>
static void launch(LaunchCtx& cx, const CUtensorMap& tA, const CUtensorMap& tB, const Params& p, int num_tiles,
                   const EpiMaps* epi = nullptr) {
  using L = SmemLayout<BN, StageCfg<MODE>::BYTES>;
  static EpiMaps none = {};
  const EpiMaps& em = epi ? *epi : none;
  static bool attr_set = false;
  if (!attr_set) {
    VD_CUDA_CHECK(cudaFuncSetAttribute(k_tc_gemm<BN, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL));
    attr_set = true;
  }
  // Persistent grid, balanced waves: with pmax CTAs available the tiles need ceil(tiles/pmax) rounds; the smallest grid
  // that still finishes in that many rounds is used, so no CTA idles through a ragged last round and the SMs not needed
  // stay free for concurrent streams.
  const int pmax = cx.sms();
  int grid = num_tiles;
  if (num_tiles > pmax) { const int rounds = cdiv(num_tiles, pmax); grid = cdiv(num_tiles, rounds); }
  k_tc_gemm<BN, MODE><<<grid, GEMM_THREADS, L::TOTAL, cx.stream>>>(tA, tB, em, p);
  check_launch(cx, "k_tc_gemm");
}

}  // namespace tc

// ---- public entry points ------------------------------------------------------------------------
bool gemm_tn_tc(LaunchCtx& cx, int M, int N, int K, const float* A, int64_t lda, const int32_t* a_gather, const float* B,
                int64_t ldb, float* C, int64_t ldc, float beta, const float* bias, int act) {
  using namespace tc;
  if (a_gather) return false;                               // gathered rows go through the projection table instead
  if (M < 64 || N < 16 || K < 32) return false;             // tiny contractions stay on CUDA cores
  // N % 4: the TMA store of C clips the box at N only in whole 16-byte chunks — with N % 4 != 0 it writes zeros into
  // the (up to 3) columns of each row past N, which belong to the caller when ldc > N
  if (N % 4 != 0) return false;
  if (!tma_ok(A, lda) || !tma_ok(B, ldb) || !tma_ok(C, ldc)) return false;
  Params p = {};
  p.M = M; p.N = N; p.K = K; p.C = C; p.ldc = ldc; p.beta = beta; p.bias = bias; p.act = act;
  EpiMaps em = {};
  em.g4 = make_tmap(C, M, N, ldc, 32, 16, CU_TENSOR_MAP_SWIZZLE_64B);      // C leaves through TMA tensor stores
  CUtensorMap tA = make_tmap(A, M, K, lda, BM);
  if (N > 64) {
    CUtensorMap tB = make_tmap(B, N, K, ldb, 128);
    launch<128, MODE_GENERIC>(cx, tA, tB, p, cdiv(M, BM) * cdiv(N, 128), &em);
  } else {
    CUtensorMap tB = make_tmap(B, N, K, ldb, 64);
    launch<64, MODE_GENERIC>(cx, tA, tB, p, cdiv(M, BM) * cdiv(N, 64), &em);
  }
  return true;
}

bool gemm_atb_tc(LaunchCtx& cx, int M, int N, int64_t K, const float* A, int64_t lda, const int32_t* a_gather, const float* B,
                 int64_t ldb, float* C, int64_t ldc) {
  using namespace tc;
  if (a_gather) return false;
  if (M < 32 || N < 32 || K < 64) return false;
  if (!tma_ok(A, lda) || !tma_ok(B, ldb)) return false;
  const int tiles = cdiv(M, BM) * cdiv(N, ATB_BN);
  // whole waves: the largest split count with tiles * splits <= 2 * #SM
  // (under an SM budget — the option stream sharing the GPU with the encoder's chains — a single wave of budget CTAs, so
  // that the reserved SMs really stay free: a second wave would be placed on them)
  const int64_t cta_cap = cx.sm_budget > 0 ? cx.sm_budget : 2LL * cx.sm_count;
  int64_t splits = std::max<int64_t>(1, std::min<int64_t>(cta_cap / tiles, K / (ATB_KB * 4)));
  int64_t kps = ((K + splits - 1) / splits + ATB_KB - 1) / ATB_KB * ATB_KB;
  splits = (K + kps - 1) / kps;
  AtbParams p = {M, N, K, kps, A, lda, B, ldb, C, ldc};
  static bool attr_set = false;
  if (!attr_set) {
    VD_CUDA_CHECK(cudaFuncSetAttribute(k_tc_atb, cudaFuncAttributeMaxDynamicSharedMemorySize, ATB_SMEM));
    attr_set = true;
  }
  dim3 grid(tiles, (unsigned)splits);
  k_tc_atb<<<grid, ATB_THREADS, ATB_SMEM, cx.stream>>>(p);
  check_launch(cx, "k_tc_atb");
  return true;
}

// Vocabulary projection with the softmax statistics fused into the epilogue (no (rows, V) tensor in HBM):
//   part_max / part_sum (M, nparts): per column slice running max and sum of exp(x - max);  tgt_logit[m] = x[m, tgt[m]-1]
int vocab_lse_nparts(int N) { return cdiv(N, 128) * (tc::EPI_WARPS / 4); }
// The shapes both halves of the fused vocabulary softmax take.  The backward writes its (M, N) d-logits with row pitch N
// through TMA, so N must be a multiple of 4; the forward refuses that shape too, because once it has taken a shape the
// logits are never materialised and the backward has no other route.
bool vocab_tc_ok(int M, int N, int K, const float* A, int64_t lda, const float* B, int64_t ldb) {
  return M >= 64 && N >= 256 && N % 4 == 0 && K >= 32 && tc::tma_ok(A, lda) && tc::tma_ok(B, ldb);
}
bool vocab_lse_tc(LaunchCtx& cx, int M, int N, int K, const float* A, int64_t lda, const float* B, int64_t ldb, const float* bias,
                  const int32_t* tgt, float* part_max, float* part_sum, float* tgt_logit) {
  using namespace tc;
  if (!vocab_tc_ok(M, N, K, A, lda, B, ldb)) return false;
  Params p = {};
  p.M = M; p.N = N; p.K = K; p.bias = bias; p.tgt = tgt; p.part_max = part_max; p.part_sum = part_sum; p.tgt_logit = tgt_logit;
  p.nparts = vocab_lse_nparts(N);
  CUtensorMap tA = make_tmap(A, M, K, lda, BM), tB = make_tmap(B, N, K, ldb, 128);
  launch<128, MODE_LSE>(cx, tA, tB, p, cdiv(M, BM) * cdiv(N, 128));
  return true;
}
// Vocabulary projection with the sampling step fused into the epilogue: vocab_lse_tc's part_max / part_sum plus, per column
// slice, the best Gumbel key, its class and its logit (M, nparts each).  vocab_sample_finish reduces them.
bool vocab_sample_tc(LaunchCtx& cx, int M, int N, int K, const float* A, int64_t lda, const float* B, int64_t ldb, const float* bias,
                     const SampleCfg& smp, float* part_max, float* part_sum, float* part_key, int32_t* part_cls, float* part_x) {
  using namespace tc;
  if (!vocab_tc_ok(M, N, K, A, lda, B, ldb)) return false;
  Params p = {};
  p.M = M; p.N = N; p.K = K; p.bias = bias; p.part_max = part_max; p.part_sum = part_sum;
  p.part_key = part_key; p.part_cls = part_cls; p.part_x = part_x; p.smp = smp;
  p.nparts = vocab_lse_nparts(N);
  CUtensorMap tA = make_tmap(A, M, K, lda, BM), tB = make_tmap(B, N, K, ldb, 128);
  launch<128, MODE_SAMPLE>(cx, tA, tB, p, cdiv(M, BM) * cdiv(N, 128));
  return true;
}
// C[m,n] = keep[m] * (exp(A B^T + bias - lse[m]) - [n == tgt[m]-1])   (backward of log-softmax + ClassNLL, recomputed)
bool vocab_dlogits_tc(LaunchCtx& cx, int M, int N, int K, const float* A, int64_t lda, const float* B, int64_t ldb, const float* bias,
                      const int32_t* tgt, const int32_t* row_ids, const float* lse, float* C, int64_t ldc) {
  using namespace tc;
  if (!vocab_tc_ok(M, N, K, A, lda, B, ldb) || !tma_ok(C, ldc)) return false;
  Params p = {};
  p.M = M; p.N = N; p.K = K; p.C = C; p.ldc = ldc; p.bias = bias; p.tgt = tgt; p.row_ids = row_ids; p.lse = lse;
  EpiMaps em = {};
  em.g4 = make_tmap(C, M, N, ldc, 32, 16, CU_TENSOR_MAP_SWIZZLE_64B);
  CUtensorMap tA = make_tmap(A, M, K, lda, BM), tB = make_tmap(B, N, K, ldb, 128);
  launch<128, MODE_DLOGIT>(cx, tA, tB, p, cdiv(M, BM) * cdiv(N, 128), &em);
  return true;
}

// The weights the fused forward step takes; the engine routes a SeqLSTM to lstm_step_fwd_tc only if this holds.
bool lstm_step_fwd_tc_ok(int H, const float* WtS_h, int64_t ldw) { return H % 64 == 0 && tc::tma_ok(WtS_h, ldw); }

// One SeqLSTM forward step on the tensor cores: gates = h_prev Wh^T (+ xproj | + ptable[tok]) + bias, then the
// pointwise half, fused.  WtS_h = transposed shadow weight offset to the h columns: [4H, ld] with K = H.
// *tile (optional) receives the tile width that ran.
bool lstm_step_fwd_tc(LaunchCtx& cx, int64_t R, int H, const float* h_prev, const float* WtS_h, int64_t ldw, const float* bias,
                      float* gates, int has_xproj, const float* ptable, const int32_t* tok, const float* c_prev, float* c_out,
                      float* h_out, const int32_t* mask_ids, int* tile) {
  using namespace tc;
  if (!lstm_step_fwd_tc_ok(H, WtS_h, ldw) || R < 1) return false;
  if (h_prev && !tma_ok(h_prev, H)) return false;
  Params p = {};
  p.M = (int)R; p.N = 4 * H; p.K = h_prev ? H : 0; p.H = H;      // K == 0: no recurrent term (t = 0 without h0)
  if (!h_prev) h_prev = WtS_h;                                      // any valid address for the (unused) tensor map
  p.bias = bias; p.gates = gates; p.has_xproj = has_xproj; p.ptable = ptable; p.tok = tok;
  p.c_prev = c_prev; p.c_out = c_out; p.h_out = h_out; p.mask_ids = mask_ids;
  CUtensorMap tA = make_tmap(h_prev, p.K ? R : 128, H, H, BM);
  if (cdiv(R, BM) * (H / 32) >= cx.sm_count) {   // 32 hidden units (x 4 gates = 128 columns) per tile
    CUtensorMap tB = make_tmap(WtS_h, 4 * (int64_t)H, H, ldw, 32);
    launch<128, MODE_LSTM_FWD>(cx, tA, tB, p, cdiv(R, BM) * (H / 32));
    if (tile) *tile = 128;
  } else {                                   // few rows (encoder LSTMs): 16 hidden units per tile, 2x the CTAs
    CUtensorMap tB = make_tmap(WtS_h, 4 * (int64_t)H, H, ldw, 16);
    launch<64, MODE_LSTM_FWD>(cx, tA, tB, p, cdiv(R, BM) * (H / 16));
    if (tile) *tile = 64;
  }
  return true;
}

// The weights the fused backward step takes; the engine routes a SeqLSTM's BPTT to lstm_step_bwd_tc only if this holds.
bool lstm_step_bwd_tc_ok(int H, const float* Wh) { return H % 128 == 0 && tc::tma_ok(Wh, 4 * H); }

// One SeqLSTM backward step: dh_rec = da_next Wh (Wh rows = reference layout rows D.., [H, 4H]) fused with the
// backward pointwise half producing da_t and the cell-gradient carry.  *tile (optional) receives the tile width that ran.
bool lstm_step_bwd_tc(LaunchCtx& cx, int64_t R, int H, const float* da_next, const float* Wh, const float* gsave,
                      const float* c_prev, const float* c_cur, const float* dh_ext, float* dc_carry, const int32_t* mask_ids,
                      float* da, int* tile) {
  using namespace tc;
  if (!lstm_step_bwd_tc_ok(H, Wh) || R < 1) return false;
  if (da_next && !tma_ok(da_next, 4 * H)) return false;
  Params p = {};
  p.M = (int)R; p.N = H; p.K = da_next ? 4 * H : 0; p.H = H;       // K == 0: last time step, no recurrent gradient
  if (!da_next) da_next = Wh;
  p.gsave = gsave; p.c_prev = c_prev; p.c_cur = c_cur; p.dh_ext = dh_ext;
  p.dc_carry = dc_carry; p.mask_ids = mask_ids; p.da = da;
  CUtensorMap tA = make_tmap(da_next, p.K ? R : 128, 4 * (int64_t)H, 4 * (int64_t)H, BM);
  if (cdiv(R, BM) * (H / 128) >= cx.sm_count) {
    CUtensorMap tB = make_tmap(Wh, H, 4 * (int64_t)H, 4 * (int64_t)H, 128);
    launch<128, MODE_LSTM_BWD>(cx, tA, tB, p, cdiv(R, BM) * (H / 128));
    if (tile) *tile = 128;
  } else {                                   // few rows: 32 hidden units per tile
    CUtensorMap tB = make_tmap(Wh, H, 4 * (int64_t)H, 4 * (int64_t)H, 32);
    launch<32, MODE_LSTM_BWD>(cx, tA, tB, p, cdiv(R, BM) * (H / 32));
    if (tile) *tile = 32;
  }
  return true;
}

}  // namespace vd
