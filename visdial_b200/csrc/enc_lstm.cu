// Persistent two-layer SeqLSTM for the FEW-ROW encoder LSTMs (question / history: R = B*10 = 320 rows, T = 20 / 40 steps,
// encoders/mn-att-ques-im-hist.lua:27-45, hrea-ques-im-hist.lua:36,76, lf-*.lua): ONE launch runs both stacked layers over
// all T time steps, forward (k_enc_pair_fwd) or BPTT (k_enc_pair_bwd), instead of 3 launches per time step.
//
// Why: the per-step kernels are latency-bound — 3 launches per time step for < 1 % of the FLOPs, each re-streaming the 4 MB
// recurrent weight through L2.  Here the weight is STATIONARY: every CTA keeps a 128 KB fp16 slice of it (32 hidden units)
// in shared memory for the whole sequence, and per step only a (128-row x K) fp16 panel moves (TMA, 5-stage ring).  Three
// CTA roles per 128-row block, H/32 CTAs each, so that NO role contracts more than one panel per step:
//
//   forward   L1  cell of layer 1:   gates = xproj1[t] (batched GEMM, up front) + h1_{t-1} Wh1^T      -> h1_t      K = H
//             X2  input half of 2:   gates2[t] <- h1_t Wx2^T + b2   (off the recurrent critical path)              K = H
//             L2  cell of layer 2:   gates = gates2[t] (from X2)    + h2_{t-1} Wh2^T                  -> h2_t      K = H
//   BPTT      T   cell of layer 2:   dh2_t = da2_{t+1} Wh2 [+ dL/dh2 at the last step]                -> da2_t     K = 4H
//             X   input half:        da1[t][:, 0:H] <- da2_t Wx2    (partial of dh1_t, parked in the output rows)  K = 4H
//             B   cell of layer 1:   dh1_t = partial + da1_{t+1} Wh1 [+ dL/dh1 at the last step]      -> da1_t     K = 4H
//   (BPTT as listed = k_enc_pair_bwd<false>, the split by hidden unit.  When H % 128 == 0 the BPTT splits BY GATE instead,
//   k_enc_pair_bwd<true>: CTA (gate, 128-unit slice) contracts K = H against N = 128 and the four gate CTAs of a slice sum their
//   partials in a zeroed fp32 dh[t] with red.add before each runs the pointwise of 32 units — see the comment at the kernel.)
//
// f16 wgmma, two consumer warpgroups of 64 rows each, N = 4 gates x 32 (forward) / 32 or 128 (BPTT), fp32 accumulators in
// registers that leave through a 32-column shared-memory chunk; the pointwise half runs in the same warps (two threads per row,
// 16 hidden units each) with the cell state / its gradient held in REGISTERS across the sequence.  Time steps are chained
// through global-memory flags: a CTA publishes "step t of my slice is stored" (barrier + release atomic), the TMA producer (and,
// for the parked partials, the epilogue threads) of a consumer CTA spin on the count of the row block (ld.acquire) — no cluster
// / grid barrier.  A stuck wait traps.  All CTAs must be co-resident (3 H/32 x row-block groups <= SM count, one CTA per SM):
// enc_pair_shape_ok.
//
// Numerics: fp16 operands (h, da, weights) with fp32 accumulation = the VD_MATH_F16 class (10-bit mantissa like TF32); cell
// state, gate pre-activations, saved activations and all gradients fp32.  The BPTT runs in a power-of-two scaled space (s from
// the largest dL/dh_T, dL/dc_T input, enc_pair_backward): the encoder gradients are small enough (~1e-6 for da at B = 32) that
// fp16 da would otherwise be subnormal, with a few significant bits or none.
#include <cuda.h>
#include <cuda_fp16.h>
#include "../../include/visdial_b200.h"
#include "kernels.cuh"
#include "tc_ptx.cuh"

namespace vd {
namespace tc {

constexpr int EP_THREADS = 288;          // warps 0-7 = two consumer warpgroups (64 rows each), warp 8 = TMA producer
constexpr int EP_STAGES = 5;
constexpr int EP_STAGE_BYTES = 128 * 64 * 2;      // 128 rows x 64 halves
constexpr int EP_W_BYTES_MAX = 131072;            // weight slice: fwd 128 x H, BPTT 32 x 4H halves = 256*H bytes (H <= 512)
constexpr int EP_ACC_BYTES = 32 * ACC_LD * 4;     // one 32-column chunk of the accumulator on its way to the epilogue
constexpr int EP_SMEM = EP_W_BYTES_MAX + EP_STAGES * EP_STAGE_BYTES + EP_ACC_BYTES + 1024 + 256;
constexpr int EP_HS = 32;                         // hidden units per CTA slice
static_assert(EP_SMEM <= 227 * 1024, "persistent encoder LSTM: shared memory budget");

__device__ __forceinline__ uint32_t ep_pack2(float a, float b) {
  uint32_t r;
  asm("{\n .reg .f16 lo, hi;\n cvt.rn.satfinite.f16.f32 lo, %1;\n cvt.rn.satfinite.f16.f32 hi, %2;\n mov.b32 %0, {lo, hi};\n}"
      : "=r"(r) : "f"(a), "f"(b));
  return r;
}
// spin until *flag >= want (published with fence + atomicAdd by the producers of that step); traps instead of hanging
__device__ __forceinline__ void wait_flag_generic(const int* flag, int want) {
  uint32_t spins = 0;
  for (;;) {
    int v;
    asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(flag) : "memory");
    if (v >= want) break;
    if (++spins > 64) __nanosleep(40);
    if (spins > (1u << 27)) __trap();
  }
}
__device__ __forceinline__ void wait_flag(const int* flag, int want) {
  wait_flag_generic(flag, want);
  asm volatile("fence.proxy.async;" ::: "memory");       // the TMA (async proxy) reads what generic-proxy stores published
}
// two threads per row, 16 hidden units each: every access of a thread is a whole 64-byte half line of its row (four 16-byte
// accesses of the same thread, which the LSU merges far better than pieces of different lines)
constexpr int EP_HW = 16;                         // hidden units per epilogue thread
__device__ __forceinline__ void ld16g(const float* p, float* d) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float4 v = *reinterpret_cast<const float4*>(p + 4 * i);
    d[4 * i] = v.x; d[4 * i + 1] = v.y; d[4 * i + 2] = v.z; d[4 * i + 3] = v.w;
  }
}
__device__ __forceinline__ void st16g(float* p, const float* v) {
#pragma unroll
  for (int i = 0; i < 4; ++i) reinterpret_cast<float4*>(p)[i] = make_float4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
}
__device__ __forceinline__ void st16gs(float* p, const float* v, float s) {     // v * s
#pragma unroll
  for (int i = 0; i < 4; ++i)
    reinterpret_cast<float4*>(p)[i] = make_float4(v[4 * i] * s, v[4 * i + 1] * s, v[4 * i + 2] * s, v[4 * i + 3] * s);
}
__device__ __forceinline__ void st16h(__half* p, const float* v) {            // 16 halves = 32 bytes
#pragma unroll
  for (int i = 0; i < 2; ++i)
    reinterpret_cast<uint4*>(p)[i] = make_uint4(ep_pack2(v[8 * i], v[8 * i + 1]), ep_pack2(v[8 * i + 2], v[8 * i + 3]),
                                                ep_pack2(v[8 * i + 4], v[8 * i + 5]), ep_pack2(v[8 * i + 6], v[8 * i + 7]));
}
__device__ __forceinline__ void zero16(float* d) {
#pragma unroll
  for (int e = 0; e < EP_HW; ++e) d[e] = 0.f;
}

enum { EP_CELL1 = 0, EP_PROJ = 1, EP_CELL2 = 2 };      // forward: L1, X2, L2;  BPTT: T (layer 2), X, B (layer 1) — see the header

struct EncFwdParams {
  int T, R, H, RB;                 // RB = number of 128-row blocks
  int nS, groups;                  // slices per role (H/32); CTA groups of 3 nS (each owns row blocks g, g+groups, ...)
  float* gates1; float* c1; float* h1; __half* h1_16;      // gates1: in = x-projection (+bias), out = activated gates
  float* gates2; float* c2; float* h2; __half* h2_16;      // gates2: parked x-half (+bias) per step, then activated gates
  const float* bias2;
  const int32_t* mask;             // (T,R) token ids for maskzero, or null
  int* flags;                      // [3][RB][T]: completed slices of (role, row block, step)
};

// carve-up shared by both kernels
struct EpSmem {
  uint8_t* wsm; uint8_t* stages; float* acc; uint64_t* full; uint64_t* empty; uint64_t* wbar;
  __device__ explicit EpSmem(uint8_t* raw) {
    uint8_t* smem = (uint8_t*)(((uintptr_t)raw + 1023) & ~(uintptr_t)1023);
    wsm = smem;                                               // resident weight slice: k-block tiles of [N rows][128 B]
    stages = smem + EP_W_BYTES_MAX;
    acc = (float*)(stages + EP_STAGES * EP_STAGE_BYTES);
    full = (uint64_t*)(stages + EP_STAGES * EP_STAGE_BYTES + EP_ACC_BYTES);
    empty = full + EP_STAGES;
    wbar = empty + EP_STAGES;
  }
  __device__ void init_barriers() {
    for (int s = 0; s < EP_STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 2); }
    mbar_init(wbar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
};

// k-block order of a CTA: rotated by `koff`, so that the CTAs streaming the same panel at the same moment (the H/32 slices of a role, and
// the projection role beside the cell that shares its panel) ask L2 for different lines instead of queueing on the same ones
__device__ __forceinline__ int ep_koff(int role, int slice, int nS, int KB) {
  const int stride = KB >= 2 * nS ? KB / (2 * nS) : 1;
  return ((2 * slice + (role == EP_PROJ ? 1 : 0)) * stride) % KB;
}
template <int N> __device__ __forceinline__ void ep_wgmma(float (&d)[N / 2], uint64_t a, uint64_t b, uint32_t acc) {
  if constexpr (N == 128) wgmma_f16_n128(d, a, b, acc);
  else { static_assert(N == 32, "accumulator width"); wgmma_f16_n32(d, a, b, acc); }
}
// contraction of one step by a consumer warpgroup: KB k-blocks of the streamed panel (its 64 rows) against the resident slice
template <int N>
__device__ __forceinline__ void ep_mma_step(const EpSmem& sm, float (&d)[N / 2], int wg, int KB, int koff, int& s, uint32_t& ph) {
  int prev = -1;
  for (int kb = 0; kb < KB; ++kb) {
    mbar_wait(&sm.full[s], ph);
    int kr = kb + koff; if (kr >= KB) kr -= KB;
    const uint32_t sa = smem_u32(sm.stages + s * EP_STAGE_BYTES) + wg * 64 * 128;
    const uint32_t sb = smem_u32(sm.wsm + kr * N * 128);
    const uint64_t adesc = make_desc(sa, 16, 1024), bdesc = make_desc(sb, 16, 1024);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) ep_wgmma<N>(d, adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2), (kb | k) ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<1>();
    if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&sm.empty[prev]);
    prev = s;
    if (++s == EP_STAGES) { s = 0; ph ^= 1; }
  }
  wgmma_wait<0>();
  wgmma_hold(d);
  if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&sm.empty[prev]);
}
// accumulator columns [32 C, 32 C + 32) of this warpgroup's 64 rows -> the shared chunk (rows 64 wg ..); the warps of the warpgroup
// then read their half row from it.  C is a compile-time constant at every call.
template <int NR>
__device__ __forceinline__ void ep_chunk(float* acc, const float (&d)[NR], int wg, int C) {
  bar_named(2 + wg, 128);                          // the previous chunk has been read
  const int lane = threadIdx.x & 31, w = (threadIdx.x >> 5) & 3;
  const int r = wg * 64 + 16 * w + (lane >> 2), c = 2 * (lane & 3);
#pragma unroll
  for (int jj = 0; jj < 4; ++jj) {
    const int j = 4 * C + jj;
    float* p = acc + (c + 8 * jj) * ACC_LD + r;
    p[0] = d[4 * j]; p[ACC_LD] = d[4 * j + 1]; p[8] = d[4 * j + 2]; p[ACC_LD + 8] = d[4 * j + 3];
  }
  bar_named(2 + wg, 128);
}
__device__ __forceinline__ void ep_ld16(const float* arow, float* v) {
#pragma unroll
  for (int e = 0; e < EP_HW; ++e) v[e] = arow[e * ACC_LD];
}

// publish step t of this slice: barrier of the consumer warps, then ONE gpu-scope release (cumulative over what the barrier made
// visible to the signalling thread) that counts the slice in — the grid-sync idiom of cooperative groups
__device__ __forceinline__ void ep_publish(int* flag) {
  bar_named(1, 256);
  if (threadIdx.x == 0) asm volatile("red.release.gpu.global.add.s32 [%0], 1;" ::"l"(flag) : "memory");
}

__global__ void __launch_bounds__(EP_THREADS, 1)
k_enc_pair_fwd(const __grid_constant__ CUtensorMap tmH1, const __grid_constant__ CUtensorMap tmH2,
               const __grid_constant__ CUtensorMap tmW1, const __grid_constant__ CUtensorMap tmW2, const EncFwdParams p) {
  extern __shared__ uint8_t smem_raw[];
  EpSmem sm(smem_raw);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int H = p.H, T = p.T;
  const int per_group = 3 * p.nS;
  const int group = blockIdx.x / per_group, idx = blockIdx.x % per_group;
  const int role = idx / p.nS, slice = idx % p.nS;
  constexpr int HS = EP_HS, N = 4 * EP_HS;          // accumulator columns [i | f | o | g]
  const int KB = H / 64;                           // k-blocks of the streamed panel = of the resident slice
  const int koff = ep_koff(role, slice, p.nS, KB);
  int* flagL1 = p.flags;
  int* flagX = p.flags + (size_t)p.RB * T;
  int* flagL2 = p.flags + 2 * (size_t)p.RB * T;

  if (threadIdx.x == 0) sm.init_barriers();
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      // ---- weights, once: tile kb = 4 gate boxes of HS rows x 64 halves.  W1 = Wh1 [4H, H]; W2 = [Wx2 | Wh2] [4H, 2H]
      const CUtensorMap* tw = role == EP_CELL1 ? &tmW1 : &tmW2;
      const int kofs = role == EP_CELL2 ? H : 0;
      mbar_expect_tx(sm.wbar, (uint32_t)(KB * N * 128));
      for (int kb = 0; kb < KB; ++kb)
        for (int g = 0; g < 4; ++g) tma_load_2d(sm.wsm + kb * N * 128 + g * HS * 128, tw, sm.wbar, kofs + kb * 64, g * H + slice * HS);
      // ---- per step: the state panel of this row block
      int s = 0; uint32_t ph = 0;
      for (int rb = group; rb < p.RB; rb += p.groups) {
        for (int t = 0; t < T; ++t) {
          const CUtensorMap* tm; int ts;
          if (role == EP_PROJ) { wait_flag(flagL1 + (size_t)rb * T + t, p.nS); tm = &tmH1; ts = t; }
          else {
            if (t == 0) continue;
            wait_flag((role == EP_CELL1 ? flagL1 : flagL2) + (size_t)rb * T + (t - 1), p.nS);
            tm = role == EP_CELL1 ? &tmH1 : &tmH2; ts = t - 1;
          }
          for (int kb = 0; kb < KB; ++kb) {
            int kr = kb + koff; if (kr >= KB) kr -= KB;
            mbar_wait(&sm.empty[s], ph ^ 1);
            mbar_expect_tx(&sm.full[s], EP_STAGE_BYTES);
            tma_load_2d(sm.stages + s * EP_STAGE_BYTES, tm, &sm.full[s], kr * 64, ts * p.R + rb * 128);
            if (++s == EP_STAGES) { s = 0; ph ^= 1; }
          }
        }
      }
    }
  } else if (warp < 8) {
    // ---- consumers: warpgroup wg contracts rows [64 wg, 64 wg + 64) of the block; its first two warps run the epilogue, thread = row
    const int wg = warp >> 2;
    const int hh = (warp >> 1) & 1;                          // which 16 of the slice's 32 hidden units
    const int rloc = wg * 64 + (warp & 1) * 32 + lane;
    const float* arow = sm.acc + hh * EP_HW * ACC_LD + rloc;
    const int u0 = slice * HS + hh * EP_HW;
    mbar_wait(sm.wbar, 0);
    int s = 0; uint32_t ph = 0;
    if (role == EP_PROJ) {
      // gates2[t] <- h1_t Wx2^T + b2 for the 4 x 32 gate columns of this slice (the layer-2 cell of the same slice adds its recurrent half)
      for (int rb = group; rb < p.RB; rb += p.groups) {
        const int64_t row = (int64_t)rb * 128 + rloc;
        const bool row_ok = row < p.R;
        for (int t = 0; t < T; ++t) {
          const int64_t tr = (int64_t)t * p.R + row;
          float d[N / 2];
          ep_mma_step<N>(sm, d, wg, KB, koff, s, ph);
#pragma unroll
          for (int g = 0; g < 4; ++g) {                        // one gate = one 128-byte line of the row per pass
            ep_chunk(sm.acc, d, wg, g);
            if (row_ok) {
              float a[EP_HW], bb[EP_HW];
              ep_ld16(arow, a);
              ld16g(p.bias2 + g * H + u0, bb);
#pragma unroll
              for (int e = 0; e < EP_HW; ++e) a[e] += bb[e];
              st16g(p.gates2 + tr * 4 * H + g * H + u0, a);
            }
          }
          ep_publish(flagX + (size_t)rb * T + t);
        }
      }
    } else {
      // LSTM cell, state c in registers across the sequence.  One gate at a time over all 32 units of the slice (order i, g, f, o), so
      // that every global access of a thread is a whole 128-byte line; the activated gates overwrite the x rows in place
      const bool l1 = role == EP_CELL1;
      float* gates = l1 ? p.gates1 : p.gates2;
      float* cst = l1 ? p.c1 : p.c2;
      float* hst = l1 ? p.h1 : p.h2;
      __half* h16 = l1 ? p.h1_16 : p.h2_16;
      int* flag = l1 ? flagL1 : flagL2;
      for (int rb = group; rb < p.RB; rb += p.groups) {
        const int64_t row = (int64_t)rb * 128 + rloc;
        const bool row_ok = row < p.R;
        float c[EP_HW];
        zero16(c);
        for (int t = 0; t < T; ++t) {
          const bool has_acc = t > 0;
          const int64_t tr = (int64_t)t * p.R + row;
          const float keep = (row_ok && p.mask && p.mask[tr] == 0) ? 0.f : 1.f;
          // additive term of the pre-activation: the x-half (+ bias) rows — layer 1: batched GEMM before the kernel; layer 2: parked in
          // gates2[t] by the projection CTAs of this step (acquire their count first)
          if (!l1 && row_ok) wait_flag_generic(flagX + (size_t)rb * T + t, p.nS);
          float* xrow = gates + tr * 4 * H + u0;
          if (l1 && row_ok && t + 1 < T) {                     // next step's x-projection rows: pull them into L2 now
#pragma unroll
            for (int g = 0; g < 4; ++g) asm volatile("prefetch.global.L2 [%0];" ::"l"(xrow + (int64_t)p.R * 4 * H + g * H) : "memory");
          }
          float d[N / 2];
          if (has_acc) ep_mma_step<N>(sm, d, wg, KB, koff, s, ph);
          float x[EP_HW], a[EP_HW], ig[EP_HW];
          // ---- i
          if (has_acc) ep_chunk(sm.acc, d, wg, 0);
          if (row_ok) {
            if (has_acc) ep_ld16(arow, a); else zero16(a);
            ld16g(xrow + 0 * H, x);
#pragma unroll
            for (int e = 0; e < EP_HW; ++e) { a[e] = fsigmoid(a[e] + x[e]) * keep; ig[e] = a[e]; }
            st16g(xrow + 0 * H, a);
          }
          // ---- g
          if (has_acc) ep_chunk(sm.acc, d, wg, 3);
          if (row_ok) {
            if (has_acc) ep_ld16(arow, a); else zero16(a);
            ld16g(xrow + 3 * H, x);
#pragma unroll
            for (int e = 0; e < EP_HW; ++e) { a[e] = ftanh(a[e] + x[e]) * keep; ig[e] *= a[e]; }
            st16g(xrow + 3 * H, a);
          }
          // ---- f  (maskzero: keep = 0 resets the state of an all-zero input row)
          if (has_acc) ep_chunk(sm.acc, d, wg, 1);
          if (row_ok) {
            if (has_acc) ep_ld16(arow, a); else zero16(a);
            ld16g(xrow + 1 * H, x);
#pragma unroll
            for (int e = 0; e < EP_HW; ++e) { a[e] = fsigmoid(a[e] + x[e]) * keep; c[e] = (a[e] * c[e] + ig[e]) * keep; }
            st16g(xrow + 1 * H, a);
          }
          // ---- o, h
          if (has_acc) ep_chunk(sm.acc, d, wg, 2);
          if (row_ok) {
            if (has_acc) ep_ld16(arow, a); else zero16(a);
            ld16g(xrow + 2 * H, x);
#pragma unroll
            for (int e = 0; e < EP_HW; ++e) { a[e] = fsigmoid(a[e] + x[e]) * keep; ig[e] = a[e] * ftanh(c[e]) * keep; }     // ig <- h_t
            st16g(xrow + 2 * H, a);
            st16h(h16 + tr * H + u0, ig);                      // what the next step's TMA reads
          }
          ep_publish(flag + (size_t)rb * T + t);
          // after the flag: saved state for the backward pass
          if (row_ok) { st16g(cst + tr * H + u0, c); st16g(hst + tr * H + u0, ig); }
        }
      }
    }
  }
}


// ------------------------------------------------------------------------------------------------
// BPTT of the pair, same structure mirrored in time (roles T / X / B of the header).  The SeqLSTM backward pointwise reads the saved
// gates, c_{t-1}, c_t, carries dc in registers and writes da_t as fp32 (what the weight / input gradients after the kernel read) and
// fp16 (the A operand of the steps that follow).  Layer 2 runs ahead; the X CTAs turn each da2_t into the layer-1 partial right behind it.
// Everything inside runs scaled by s = scale2[0]: dh_last / dc_last are multiplied by s when loaded, so dh, dc, the partials and the
// fp16 da are s times the true values; only the fp32 da is stored times 1/s (exact: s is a power of two).
struct EncBwdParams {
  int T, R, H, RB;
  int nS, groups;
  const float* gates1; const float* c1; float* da1; __half* da1_16;
  const float* gates2; const float* c2; float* da2; __half* da2_16;
  const float* dh_last1; const float* dc_last1; const float* dh_last2; const float* dc_last2;   // (R,H) each or null
  const int32_t* mask;
  int* flags;                      // [3][RB][T] step flags, then (gate split) [2][RB][T][H/128] partial-sum counts
  float* dh2; float* dh1;          // gate split: (T*R, H) fp32 each, zeroed — the partial products of a step are summed here with red.add
  const float* scale2;             // device {s, 1/s}
};

// GS = gate split (H % 128 == 0): a CTA contracts ONE gate's quarter of the da panel (K = H) against a 128-unit slice of the weight
// (same 128 KB): N = 128 per instruction instead of N = 32 and a quarter of the panel bytes.  The four gate CTAs of a unit slice add
// their partials into dh (red.add), count themselves in, and each then runs the pointwise for 32 of the slice's 128 units once the
// count is complete.
template <bool GS>
__global__ void __launch_bounds__(EP_THREADS, 1)
k_enc_pair_bwd(const __grid_constant__ CUtensorMap tmA1, const __grid_constant__ CUtensorMap tmA2,
               const __grid_constant__ CUtensorMap tmW1, const __grid_constant__ CUtensorMap tmW2, const EncBwdParams p) {
  extern __shared__ uint8_t smem_raw[];
  EpSmem sm(smem_raw);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int H = p.H, T = p.T;
  const int per_group = 3 * p.nS;
  const int group = blockIdx.x / per_group, idx = blockIdx.x % per_group;
  const int role = idx / p.nS, slice = idx % p.nS;         // EP_CELL1 = T (layer 2), EP_PROJ = X, EP_CELL2 = B (layer 1)
  constexpr int HS = EP_HS;                                // hidden units this CTA runs the pointwise for
  constexpr int N = GS ? 128 : EP_HS;                      // accumulator columns
  const int nU = H / 128;                                  // GS: unit slices of 128; slice = gate * nU + unit slice
  const int gq = GS ? slice / nU : 0, us = GS ? slice % nU : 0;
  const int j0 = GS ? us * 128 + gq * HS : slice * HS;     // first hidden unit of the pointwise
  const int KB = (GS ? H : 4 * H) / 64;                    // k-blocks of the streamed panel (piece) = of the resident slice
  const int koff = ep_koff(role, slice, p.nS, KB);
  int* flagT = p.flags;
  int* flagX = p.flags + (size_t)p.RB * T;
  int* flagB = p.flags + 2 * (size_t)p.RB * T;
  int* cntT = p.flags + 3 * (size_t)p.RB * T;              // GS: [RB][T][nU] partials summed into dh2 / dh1
  int* cntB = cntT + (size_t)p.RB * T * nU;

  if (threadIdx.x == 0) sm.init_barriers();
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      // W2 = Wh2 as [H, 4H]; W1 = [Wx2 | Wh1] as [H, 8H]
      const CUtensorMap* tw = role == EP_CELL1 ? &tmW2 : &tmW1;
      const int kofs = role == EP_CELL2 ? 4 * H : 0;
      mbar_expect_tx(sm.wbar, (uint32_t)(KB * N * 128));
      for (int kb = 0; kb < KB; ++kb)
        tma_load_2d(sm.wsm + kb * N * 128, tw, sm.wbar, kofs + (GS ? gq * H : 0) + kb * 64, GS ? us * 128 : slice * HS);
      int s = 0; uint32_t ph = 0;
      for (int rb = group; rb < p.RB; rb += p.groups) {
        for (int t = T - 1; t >= 0; --t) {
          const CUtensorMap* tm; int ts;
          if (role == EP_PROJ) { wait_flag(flagT + (size_t)rb * T + t, p.nS); tm = &tmA2; ts = t; }
          else {
            if (t == T - 1) continue;
            wait_flag((role == EP_CELL1 ? flagT : flagB) + (size_t)rb * T + (t + 1), p.nS);
            tm = role == EP_CELL1 ? &tmA2 : &tmA1; ts = t + 1;
          }
          for (int kb = 0; kb < KB; ++kb) {
            int kr = kb + koff; if (kr >= KB) kr -= KB;
            mbar_wait(&sm.empty[s], ph ^ 1);
            mbar_expect_tx(&sm.full[s], EP_STAGE_BYTES);
            tma_load_2d(sm.stages + s * EP_STAGE_BYTES, tm, &sm.full[s], (GS ? gq * H : 0) + kr * 64, ts * p.R + rb * 128);
            if (++s == EP_STAGES) { s = 0; ph ^= 1; }
          }
        }
      }
    }
  } else if (warp < 8) {
    const int wg = warp >> 2;
    const int hh = (warp >> 1) & 1;                          // which 16 of the slice's 32 hidden units
    const int rloc = wg * 64 + (warp & 1) * 32 + lane;
    const float* arow = sm.acc + hh * EP_HW * ACC_LD + rloc;
    const int u0 = j0 + hh * EP_HW;
    mbar_wait(sm.wbar, 0);
    int s = 0; uint32_t ph = 0;
    // GS: add this CTA's (128 rows x 128 units) partial product into dh[t] and count it in for the unit slice
    auto add_partial = [&](const float (&d)[N / 2], float* dhbuf, int* cnt, int rb, int t, int64_t tr, bool row_ok) {
#pragma unroll
      for (int sb = 0; sb < N / 32; ++sb) {
        ep_chunk(sm.acc, d, wg, sb);
        if (row_ok) {
          float a[EP_HW];
          ep_ld16(arow, a);
          float* dst = dhbuf + tr * H + us * 128 + sb * 32 + hh * EP_HW;
#pragma unroll
          for (int e = 0; e < EP_HW; e += 4) red_add_v4(dst + e, a[e], a[e + 1], a[e + 2], a[e + 3]);
        }
      }
      bar_named(1, 256);
      if (threadIdx.x == 0) asm volatile("red.release.gpu.global.add.s32 [%0], 1;" ::"l"(cnt + ((size_t)rb * T + t) * nU + us) : "memory");
    };
    if (role == EP_PROJ) {
      // GS: partial of dh1_t = da2_t Wx2 (this gate's quarter, this unit slice), summed into dh1[t];  otherwise the partial of
      // dh1_t = da2_t Wx2, parked in the first H columns of da1[t] (the B cell of the same slice reads it, then overwrites)
      for (int rb = group; rb < p.RB; rb += p.groups) {
        const int64_t row = (int64_t)rb * 128 + rloc;
        const bool row_ok = row < p.R;
        for (int t = T - 1; t >= 0; --t) {
          const int64_t tr = (int64_t)t * p.R + row;
          float d[N / 2];
          ep_mma_step<N>(sm, d, wg, KB, koff, s, ph);
          if constexpr (GS) {
            add_partial(d, p.dh1, cntB, rb, t, tr, row_ok);
          } else {
            ep_chunk(sm.acc, d, wg, 0);
            if (row_ok) { float a[EP_HW]; ep_ld16(arow, a); st16g(p.da1 + tr * 4 * H + u0, a); }
            ep_publish(flagX + (size_t)rb * T + t);
          }
        }
      }
    } else {
      // SeqLSTM backward pointwise, dc in registers across the sequence; whole 128-byte lines per thread and access (three passes: o, then
      // i and g, then f), da_t stored as fp16 (the operand of the steps that follow) and fp32 (read after the kernel)
      const bool top = role == EP_CELL1;
      const float* gates = top ? p.gates2 : p.gates1;
      const float* cst = top ? p.c2 : p.c1;
      float* da = top ? p.da2 : p.da1;
      __half* da16 = top ? p.da2_16 : p.da1_16;
      const float* dh_last = top ? p.dh_last2 : p.dh_last1;
      const float* dc_last = top ? p.dc_last2 : p.dc_last1;
      int* flag = top ? flagT : flagB;
      float* dhbuf = top ? p.dh2 : p.dh1;
      int* cnt = top ? cntT : cntB;
      const float sc = p.scale2[0], isc = p.scale2[1];
      for (int rb = group; rb < p.RB; rb += p.groups) {
        const int64_t row = (int64_t)rb * 128 + rloc;
        const bool row_ok = row < p.R;
        float dc[EP_HW];
        zero16(dc);
        for (int t = T - 1; t >= 0; --t) {
          const bool has_acc = t < T - 1;
          const int64_t tr = (int64_t)t * p.R + row;
          const float keep = (row_ok && p.mask && p.mask[tr] == 0) ? 0.f : 1.f;
          const float* grow = gates + tr * 4 * H + u0;
          float* darow = da + tr * 4 * H + u0;
          __half* da16row = da16 + tr * 4 * H + u0;
          float va[EP_HW], vb[EP_HW], dh[EP_HW];
          float d[N / 2];
          if (has_acc) ep_mma_step<N>(sm, d, wg, KB, koff, s, ph);
          if constexpr (GS) {
            // my partial into dh[t]; then the complete sum of my 32 units once every contributor of the unit slice has counted in:
            // layer 2: its 4 gate CTAs; layer 1: 4 projection CTAs (every step) + its own 4 gate CTAs (all steps but the last)
            if (has_acc) add_partial(d, dhbuf, cnt, rb, t, tr, row_ok);
            const int want = top ? 4 : (has_acc ? 8 : 4);
            if (!row_ok || (top && !has_acc)) zero16(dh);
            else {
              wait_flag_generic(cnt + ((size_t)rb * T + t) * nU + us, want);
              ld16g(dhbuf + tr * H + u0, dh);
            }
          } else {
            if (has_acc) ep_chunk(sm.acc, d, wg, 0);
            if (has_acc && row_ok) ep_ld16(arow, dh); else zero16(dh);
            if (!top && row_ok) {                              // the parked partial of this step
              wait_flag_generic(flagX + (size_t)rb * T + t, p.nS);
              ld16g(darow, va);
#pragma unroll
              for (int e = 0; e < EP_HW; ++e) dh[e] += va[e];
            }
          }
          if (row_ok) {
            if (t == T - 1) {
              if (dh_last) { ld16g(dh_last + row * H + u0, va);
#pragma unroll
                for (int e = 0; e < EP_HW; ++e) dh[e] += va[e] * sc; }
              if (dc_last) { ld16g(dc_last + row * H + u0, dc);
#pragma unroll
                for (int e = 0; e < EP_HW; ++e) dc[e] *= sc; }
            }
            // ---- o:  da_o = dh tanh(c) o (1-o);  d = dc + dh o (1 - tanh(c)^2)
            ld16g(grow + 2 * H, va); ld16g(cst + tr * H + u0, vb);
#pragma unroll
            for (int e = 0; e < EP_HW; ++e) {
              const float tcv = ftanh(vb[e]), go = va[e], dhe = dh[e] * keep;
              dc[e] = (dc[e] + dhe * go * (1.f - tcv * tcv)) * keep;           // dc <- d
              dh[e] = dhe * tcv * go * (1.f - go);
            }
            st16h(da16row + 2 * H, dh); st16gs(darow + 2 * H, dh, isc);
            // ---- i, g:  da_i = d g i (1-i);  da_g = d i (1-g^2)
            ld16g(grow, va); ld16g(grow + 3 * H, vb);
#pragma unroll
            for (int e = 0; e < EP_HW; ++e) dh[e] = dc[e] * vb[e] * va[e] * (1.f - va[e]);
            st16h(da16row, dh); st16gs(darow, dh, isc);
#pragma unroll
            for (int e = 0; e < EP_HW; ++e) dh[e] = dc[e] * va[e] * (1.f - vb[e] * vb[e]);
            st16h(da16row + 3 * H, dh); st16gs(darow + 3 * H, dh, isc);
            // ---- f:  da_f = d c_{t-1} f (1-f);  dc_{t-1} = d f
            ld16g(grow + 1 * H, va);
            if (t > 0) ld16g(cst + (tr - p.R) * H + u0, vb); else zero16(vb);
#pragma unroll
            for (int e = 0; e < EP_HW; ++e) { dh[e] = dc[e] * vb[e] * va[e] * (1.f - va[e]); dc[e] *= va[e]; }
            st16h(da16row + 1 * H, dh); st16gs(darow + 1 * H, dh, isc);
          }
          ep_publish(flag + (size_t)rb * T + t);
        }
      }
    }
  }
}

// scale2 = {s, 1/s}: the power of two s that brings the largest |x| over the non-null inputs (n4 float4 each) to [2^5, 2^6); s = 1
// when that is 0 or infinite, NaN elements do not take part (fmaxf).  One CTA: the inputs are (R, H), a few hundred KB each, and one
// launch costs less on the BPTT's critical path than a grid-wide reduction and a second launch.
__global__ void __launch_bounds__(1024) k_ep_pick_scale(const float* x0, const float* x1, const float* x2, const float* x3, int64_t n4,
                                                        float* __restrict__ scale2) {
  __shared__ float red[32];
  const float* xs[4] = {x0, x1, x2, x3};
  float m = 0.f;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    if (!xs[k]) continue;
    const float4* x = reinterpret_cast<const float4*>(xs[k]);
    for (int64_t i = threadIdx.x; i < n4; i += blockDim.x) {
      const float4 v = __ldg(x + i);
      m = fmaxf(m, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x < 32) {
    m = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (threadIdx.x == 0) {
      float sc = 1.f;
      if (m > 0.f && isfinite(m)) {
        int e; frexpf(m, &e);                        // m = f * 2^e, f in [0.5, 1)
        sc = ldexpf(1.f, max(-60, min(60, 6 - e)));
      }
      scale2[0] = sc; scale2[1] = 1.f / sc;
    }
  }
}

// ------------------------------------------------------------------------------------------------ host
static CUtensorMap ep_tmap_h(const __half* base, int64_t rows, int64_t cols, int64_t ld, int box_rows) {
  CUtensorMap tm;
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {64u, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = get_encode()(&tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (void*)base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char buf[256];
    snprintf(buf, sizeof(buf), "cuTensorMapEncodeTiled (enc_lstm) failed (%d): rows %lld cols %lld ld %lld box %d", (int)r, (long long)rows,
             (long long)cols, (long long)ld, box_rows);
    throw CudaError(-3, buf);
  }
  return tm;
}

}  // namespace tc

bool enc_pair_shape_ok(int64_t R, int H, int sm_count) {
  return H % 64 == 0 && H <= 512 && R >= 64 && 3 * (H / 32) <= sm_count;
}

// flags: int32 [3 * RB * T] (zeroed here).  gates1 holds the layer-1 x-projection (+ bias) on entry.
void enc_pair_forward(LaunchCtx& cx, int T, int64_t R, int H, const __half* W1h16, const __half* W2cat16, const float* bias2,
                      const int32_t* mask, float* gates1, float* c1, float* h1, __half* h1_16, float* gates2, float* c2, float* h2,
                      __half* h2_16, int* flags) {
  using namespace tc;
  VD_REQUIRE(enc_pair_shape_ok(R, H, cx.sm_count), VD_E_STATE, "enc_pair_forward: shape");
  EncFwdParams p = {};
  p.T = T; p.R = (int)R; p.H = H; p.RB = cdiv(R, 128);
  p.nS = H / 32;
  p.groups = std::max(1, std::min(p.RB, cx.sm_count / (3 * p.nS)));
  p.gates1 = gates1; p.c1 = c1; p.h1 = h1; p.h1_16 = h1_16;
  p.gates2 = gates2; p.c2 = c2; p.h2 = h2; p.h2_16 = h2_16;
  p.bias2 = bias2; p.mask = mask; p.flags = flags;
  VD_CUDA_CHECK(cudaMemsetAsync(flags, 0, (size_t)3 * p.RB * T * sizeof(int), cx.stream));
  const int64_t TR = (int64_t)T * R;
  CUtensorMap tH1 = ep_tmap_h(h1_16, TR, H, H, 128), tH2 = ep_tmap_h(h2_16, TR, H, H, 128);
  CUtensorMap tW1 = ep_tmap_h(W1h16, 4 * (int64_t)H, H, H, EP_HS), tW2 = ep_tmap_h(W2cat16, 4 * (int64_t)H, 2 * (int64_t)H, 2 * (int64_t)H, EP_HS);
  static bool attr_set = false;
  if (!attr_set) {
    VD_CUDA_CHECK(cudaFuncSetAttribute(k_enc_pair_fwd, cudaFuncAttributeMaxDynamicSharedMemorySize, EP_SMEM));
    attr_set = true;
  }
  k_enc_pair_fwd<<<p.groups * 3 * p.nS, EP_THREADS, EP_SMEM, cx.stream>>>(tH1, tH2, tW1, tW2, p);
  check_launch(cx, "k_enc_pair_fwd");
}


// gates*/c* = the activations the forward saved; da*/da*_16 out (all T steps); flags int32 [enc_pair_bwd_flag_ints()].
// dh1 / dh2: (T*R, H) fp32 scratch each for the gate-split variant (H % 128 == 0), or null -> unit-split variant.
// scale: float[2] out, {s, 1/s}: da*_16 = fp16(s da*), so the fp16 weight gradients take 1/s as their inv_scale.
// s brings the largest |dh_last*|, |dc_last*| to [2^5, 2^6): 10 binades of head-room below the fp16 maximum, because dc sums the
// dh of up to T steps and da_f = d c_{t-1} f (1-f) grows with |c|, which can reach T; the fp16 normal range still reaches
// 20 binades below the largest input, where the option LSTM's 2^10 target would leave only 6 binades of head-room.
int64_t enc_pair_bwd_flag_ints(int T, int64_t R, int H) { return (int64_t)cdiv(R, 128) * T * (3 + 2 * std::max(1, H / 128)); }
bool enc_pair_gate_split(int H) { return H % 128 == 0; }
void enc_pair_backward(LaunchCtx& cx, int T, int64_t R, int H, const __half* B1cat16, const __half* Whb2_16, const int32_t* mask,
                       const float* gates1, const float* c1, const float* gates2, const float* c2, const float* dh_last1,
                       const float* dc_last1, const float* dh_last2, const float* dc_last2, float* da1, __half* da1_16, float* da2,
                       __half* da2_16, int* flags, float* dh1, float* dh2, float* scale) {
  using namespace tc;
  VD_REQUIRE(enc_pair_shape_ok(R, H, cx.sm_count), VD_E_STATE, "enc_pair_backward: shape");
  const bool gs = dh1 && dh2 && enc_pair_gate_split(H);
  EncBwdParams p = {};
  p.T = T; p.R = (int)R; p.H = H; p.RB = cdiv(R, 128);
  p.nS = H / 32;
  p.groups = std::max(1, std::min(p.RB, cx.sm_count / (3 * p.nS)));
  p.gates1 = gates1; p.c1 = c1; p.da1 = da1; p.da1_16 = da1_16;
  p.gates2 = gates2; p.c2 = c2; p.da2 = da2; p.da2_16 = da2_16;
  p.dh_last1 = dh_last1; p.dc_last1 = dc_last1; p.dh_last2 = dh_last2; p.dc_last2 = dc_last2;
  p.mask = mask; p.flags = flags; p.dh1 = dh1; p.dh2 = dh2; p.scale2 = scale;
  k_ep_pick_scale<<<1, 1024, 0, cx.stream>>>(dh_last1, dc_last1, dh_last2, dc_last2, R * H / 4, scale);
  check_launch(cx, "k_ep_pick_scale");
  VD_CUDA_CHECK(cudaMemsetAsync(flags, 0, (size_t)enc_pair_bwd_flag_ints(T, R, H) * sizeof(int), cx.stream));
  const int64_t TR = (int64_t)T * R;
  const int64_t G = 4 * (int64_t)H;
  if (gs) {
    VD_CUDA_CHECK(cudaMemsetAsync(dh1, 0, (size_t)TR * H * sizeof(float), cx.stream));
    VD_CUDA_CHECK(cudaMemsetAsync(dh2, 0, (size_t)TR * H * sizeof(float), cx.stream));
  }
  CUtensorMap tA1 = ep_tmap_h(da1_16, TR, G, G, 128), tA2 = ep_tmap_h(da2_16, TR, G, G, 128);
  const int wbox = gs ? 128 : EP_HS;
  CUtensorMap tW1 = ep_tmap_h(B1cat16, H, 2 * G, 2 * G, wbox), tW2 = ep_tmap_h(Whb2_16, H, G, G, wbox);
  static bool attr_set = false;
  if (!attr_set) {
    VD_CUDA_CHECK(cudaFuncSetAttribute(k_enc_pair_bwd<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, EP_SMEM));
    VD_CUDA_CHECK(cudaFuncSetAttribute(k_enc_pair_bwd<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, EP_SMEM));
    attr_set = true;
  }
  if (gs) k_enc_pair_bwd<true><<<p.groups * 3 * p.nS, EP_THREADS, EP_SMEM, cx.stream>>>(tA1, tA2, tW1, tW2, p);
  else k_enc_pair_bwd<false><<<p.groups * 3 * p.nS, EP_THREADS, EP_SMEM, cx.stream>>>(tA1, tA2, tW1, tW2, p);
  check_launch(cx, "k_enc_pair_bwd");
}

}  // namespace vd
