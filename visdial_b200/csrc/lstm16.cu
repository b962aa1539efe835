// SeqLSTM over MANY rows (the disc decoder's option LSTM, decoders/disc.lua:4-20: R = N*100 = 32 000 rows at B = 32)
// with 16-bit operands and 16-bit saved state: VD_MATH_F16.
//
// Why: the TF32 step kernels are bound by BYTES, not by the tensor pipe — the L2->SM operand stream of fp32 tiles and the
// HBM traffic of the fp32 saved activations (at B = 32: 0.5 GB forward, 1.05 GB backward per step).  A TF32 operand keeps 10 mantissa bits of the fp32
// word it reads; an fp16 word carries the same 10 bits in half the bytes (the exponent range is what is given up: h and
// the weights live well inside it, the gradients are scaled by a power of two chosen from max|dL/dh_T| so that they do
// too — exact, undone in the weight-gradient epilogue).  So: h_t, the x-projection table, the activated gates and da_t
// are stored as fp16, the contractions run as f16 wgmma (2x the TF32 rate) with fp32 accumulation,
// and c_t, dc, every accumulator, the weight gradients and the final h_T that meets the encoder stay fp32.
//
//   k_lstm16<0>    : gates = h_{t-1} Wh^T (wgmma, 128x128 tiles) + P16[token] + bias -> pointwise -> fp16 gates,
//                    fp32 c_t, fp16 h_t (+ fp32 h_T on the last step).  Each CTA keeps one 128-row column slice of Wh
//                    resident in shared memory (128 KB at H = 512) and streams only h_{t-1}; its two consumer warpgroups
//                    contract their 64-row halves and take turns, so that one's main loop runs under the other's
//                    epilogue; one 5-stage ring carries both halves' h_{t-1} rows in the order of the turns.
//   k_lstm16_bptt  : BPTT steps t_hi .. 0 in one launch: dh = da_{t+1} Wh (wgmma) -> backward pointwise -> fp16 da_t.  One
//                    cluster of H / 128 CTAs per 128-row block (CTA u: hidden units 128u .. 128u + 127), a cluster barrier
//                    between the steps (da_t of the whole block, written by the cluster, is the next step's A operand, read
//                    back from L2); the fp32 dc carry stays on chip for all steps (half in registers, half in shared
//                    memory).  A 4-stage ring of 32 KB (A and B) stages shared by both consumer warpgroups; 8 KB of
//                    staging per consumer warp; 32 KB of carry: 224 KB of shared memory, 168 registers, no spills.
//                    Launched in waves of as many clusters as fit in the SM budget (lstm16_bptt_plan); a one-step launch
//                    is the step test hook.  Per row and step it moves 12 KB of HBM at H = 512 (gates in, da out, c_{t-1}
//                    and c_t in) where one launch per step moved 20 KB (also da_{t+1} in and the carry in and out).
//   Both run their pointwise epilogue on the accumulator registers (no shared-memory accumulator tile); the epilogue inputs
//   are fetched by cp.async before the tile's contraction (the backward: those of its first 32 hidden units, during the
//   cluster barrier before the step).
//   k_atb16        : dWh += inv_scale * h^T da  (both operands MN-major fp16, 128 x 256 tiles, stream-K, red.global.add)
//   k_lstm16_first / k_lstm16_bwd_last / k_segsum16 / k_cvt16 / k_amax / k_pick_scale : streaming helpers
#include <cuda.h>
#include <cuda_fp16.h>
#include <map>
#include <mutex>
#include "../../include/visdial_b200.h"
#include "kernels.cuh"
#include "tc_ptx.cuh"

namespace vd {
namespace tc {

constexpr int BM16 = 128;        // rows per tile (two 64-row wgmma slabs)
constexpr int BK16 = 64;         // halves per k-block = one 128-byte swizzle row
constexpr int UK16 = 16;         // f16 wgmma: 32 bytes per instruction
constexpr int BN16 = 128;        // accumulator columns per tile: forward 32 hidden units x 4 gates, backward 128 hidden units
constexpr int EW16 = 8;          // consumer warps = epilogue warps: 16 rows of a tile each
constexpr int STAGE16 = 32768;   // 16 KB of A (128 rows) + 16 KB of B (128 rows)

// Activations of the fp16 option LSTM: ONE special-function op each (tanh.approx.f32, relative error 2^-11 — the rounding class of the fp16
// the gates and h are stored in right after; sigmoid(x) = 0.5 tanh(x/2) + 0.5) instead of the two of ex2 + rcp: the pointwise half of the
// forward step is issue / MUFU-bound.  Against the ex2 + rcp forms (abs error ~1e-7), measured at the benched size
// (tests/test_c4_b32_gpu.py, DESIGN.md 7): rank agreement with the fp64 oracle 0.9781 vs 0.9777, top-1 0.99375 both, R@k deltas 0 both.
__device__ __forceinline__ float tanh16(float x) { float y; asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float sig16(float x) { return fmaf(0.5f, tanh16(0.5f * x), 0.5f); }

// ---- fp16 <-> fp32 packing (round to nearest even, saturating: a scaled gradient that outgrows the range clamps to
// +-65504 instead of becoming inf)
__device__ __forceinline__ uint32_t pack2(float a, float b) {
  uint32_t r;
  asm("{\n .reg .f16 lo, hi;\n cvt.rn.satfinite.f16.f32 lo, %1;\n cvt.rn.satfinite.f16.f32 hi, %2;\n mov.b32 %0, {lo, hi};\n}"
      : "=r"(r) : "f"(a), "f"(b));
  return r;
}
__device__ __forceinline__ uint4 pack8(const float* v) {
  return make_uint4(pack2(v[0], v[1]), pack2(v[2], v[3]), pack2(v[4], v[5]), pack2(v[6], v[7]));
}
__device__ __forceinline__ void unpack8(const uint4 u, float* v) {
  const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) { const float2 f = __half22float2(h[i]); v[2 * i] = f.x; v[2 * i + 1] = f.y; }
}

// ---- epilogue staging tiles (one set per consumer warp: the warp's 16 rows x 32 hidden units).  Laid out exactly like the
// TMA box that leaves them, so stores are single bulk-tensor instructions:
//   T16: [16 rows][32 halves] = 64-byte rows, 16-byte chunk c of row r at  r*64 + ((c ^ ((r>>1)&3)) << 4)    (SWIZZLE_64B)
//   T32: [16 rows][32 floats] = 128-byte rows, 16-byte chunk c of row r at r*128 + ((c ^ (r&7)) << 4)        (SWIZZLE_128B)
// A thread reads and writes them at its accumulator fragment's positions (rows l/4 and l/4 + 8, units 2(l%4) + 8jj, +1):
// a warp's half2 / float2 accesses are bank-conflict free.  The inputs land here by cp.async, 16-byte chunks per lane.
constexpr int T16_BYTES = 1024, T32_BYTES = 2048;
__device__ __forceinline__ uint8_t* t16_at(uint8_t* base, int row, int unit) {   // the half2 at (row, unit), unit even
  return base + row * 64 + (((unit >> 3) ^ ((row >> 1) & 3)) << 4) + (unit & 7) * 2;
}
__device__ __forceinline__ uint8_t* t32_at(uint8_t* base, int row, int unit) {   // the float2 at (row, unit), unit even
  return base + row * 128 + (((unit >> 2) ^ (row & 7)) << 4) + (unit & 3) * 4;
}
__device__ __forceinline__ const void* shfl_vptr(const void* p, int src_lane) {
  unsigned long long v = (unsigned long long)p;
  unsigned lo = __shfl_sync(0xffffffffu, (unsigned)v, src_lane), hi = __shfl_sync(0xffffffffu, (unsigned)(v >> 32), src_lane);
  return (const void*)(((unsigned long long)hi << 32) | lo);
}
__device__ __forceinline__ void cp16(void* dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
// global -> T16 tile: `mine` = the row base (32 halves) of row (lane & 15), or nullptr (zeros); 4 lanes per row, 2 passes
__device__ __forceinline__ void t16_load(uint8_t* base, const void* mine, int lane) {
#pragma unroll
  for (int ps = 0; ps < 2; ++ps) {
    const int row = ps * 8 + (lane >> 2), c = lane & 3;
    const uint8_t* src = (const uint8_t*)shfl_vptr(mine, row);
    uint8_t* dst = base + row * 64 + ((c ^ ((row >> 1) & 3)) << 4);
    if (src) cp16(dst, src + c * 16); else *reinterpret_cast<uint4*>(dst) = make_uint4(0, 0, 0, 0);
  }
}
// global -> T32 tile: 8 lanes per row, 4 passes
__device__ __forceinline__ void t32_load(uint8_t* base, const void* mine, int lane) {
#pragma unroll
  for (int ps = 0; ps < 4; ++ps) {
    const int row = ps * 4 + (lane >> 3), c = lane & 7;
    const uint8_t* src = (const uint8_t*)shfl_vptr(mine, row);
    uint8_t* dst = base + row * 128 + ((c ^ (row & 7)) << 4);
    if (src) cp16(dst, src + c * 16); else *reinterpret_cast<float4*>(dst) = make_float4(0.f, 0.f, 0.f, 0.f);
  }
}
__device__ __forceinline__ void cp_wait_all() {
  asm volatile("cp.async.wait_all;" ::: "memory");
  __syncwarp();
}
__device__ __forceinline__ float2 ld_h2(uint8_t* p) { return __half22float2(*reinterpret_cast<const __half2*>(p)); }
__device__ __forceinline__ void st_h2(uint8_t* p, float a, float b) { *reinterpret_cast<uint32_t*>(p) = pack2(a, b); }

struct Lstm16Params {
  int R, H;
  // forward
  const __half* ptable; const int32_t* tok;   // x-projection table (V+1, 4H) WITHOUT bias, token id per row
  const float* bias;                           // (4H) fp32, added in the epilogue
  const float* c_prev;                         // (R,H) fp32 or null (zeros)
  const int32_t* mask_ids;                     // maskzero ids or null
  float* h32_out;                              // optional fp32 copy of h (the step whose h meets fp32 consumers)
  int save_gates;
};
struct Lstm16Maps { CUtensorMap g16, c, h16; };   // [R,4H] fp16 gates / da ; [R,H] fp32 c / dc ; [R,H] fp16 h: 16 x 32 boxes

// ------------------------------------------------------------------------------------------------
// MODE 0 = forward step (the only specialisation); warpgroup 0 = TMA producers, warpgroups 1-2 = consumers (64 rows each).
// Each consumer warp runs the pointwise epilogue of its 16 rows straight from its accumulator registers, 32 hidden units at a
// time, with the inputs staged by cp.async in the T16 / T32 tiles above.
template <int MODE> struct Cfg16;

// Forward: each CTA owns one column slice (32 hidden units x 4 gates = 128 rows of Wh, all H of K) for the whole launch and
// keeps it resident in shared memory; only h_{t-1} streams.  The two consumer warpgroups each contract their own 64-row half of
// a 128-row block against the whole slice and take turns (named-barrier token): one warpgroup's main loop runs while the other
// runs its epilogue.  The turns fix the order in which the halves are consumed, so one ring of 64-row stages carries both,
// in that order, and keeps four stages in flight across the hand-over from one warpgroup to the other.
template <>
struct Cfg16<0> {
  static constexpr int THREADS = 128 + 32 * EW16;
  static constexpr int KB_MAX = 512 / BK16;                       // k-blocks of the slice at the largest H (lstm16_shape_ok)
  static constexpr int SLICE_KB = 4 * 32 * BK16 * 2;              // one k-block of the slice: 4 gate boxes of 32 rows = 16 KB
  static constexpr int RES_BYTES = KB_MAX * SLICE_KB;             // 128 KB
  static constexpr int A_STAGE = 64 * BK16 * 2;                   // 64 rows of h_{t-1} x one k-block = 8 KB
  static constexpr int A_STAGES = 5;                              // as many as fit beside the slice and the staging
  // per-warp staging {4 gate tiles T16, h tile T16, c tile T32} = 7 KB: the inputs, x-projection rows and c_prev, land in the
  // gate and c tiles; the outputs overwrite them in place
  static constexpr int STG_PER_WARP = 5 * T16_BYTES + T32_BYTES;
  static constexpr int STG_BYTES = EW16 * STG_PER_WARP;           // 56 KB
  static constexpr int BAR_BYTES = 8 * (KB_MAX + 2 * A_STAGES);
  static constexpr int TOTAL = RES_BYTES + A_STAGES * A_STAGE + STG_BYTES + BAR_BYTES + 1024;   // + alignment slack
  static_assert(TOTAL <= 232448, "k_lstm16<0>: shared memory");
};

// The forward step is the k_lstm16<0> specialisation below; the BPTT runs k_lstm16_bptt.
template <int MODE>
__global__ void k_lstm16(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                         const __grid_constant__ Lstm16Maps em, const Lstm16Params p);

// Forward step.  CTA b owns the column slice nt = b % num_n and walks the 128-row blocks b / num_n, + P, + 2P, ... (P =
// gridDim.x / num_n CTAs per slice).  Thread 0 loads the slice once (one barrier per k-block, so the first contraction starts
// on the first 16 KB) and then streams h_{t-1} through the ring.  Warpgroup w contracts rows 64w .. 64w + 63 of each block
// with the m64n128k16 instructions, operands and k order of a 128 x 128 tile: the accumulators are bit for bit those of a
// kernel that streams both operands.  The turn is a token on two named barriers of the 256 consumer
// threads: warpgroup 1 runs its main loop, arrives on barrier 2 (warpgroup 2's main loop may start) and runs its epilogue;
// warpgroup 2 arrives on barrier 1 after its main loop, except after its last block, so that every barrier phase that is
// arrived on is also waited on.  Without the token the two start together and stay in lockstep.
template <>
__global__ void __launch_bounds__(Cfg16<0>::THREADS, 1)
k_lstm16<0>(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
            const __grid_constant__ Lstm16Maps em, const Lstm16Params p) {
  using C = Cfg16<0>;
  constexpr int AS = C::A_STAGES;
  constexpr int TOKEN_WG1 = 1, TOKEN_WG2 = 2;                 // named barriers (0 is __syncthreads')
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint8_t* slice = smem;                                      // [k-block][gate i f o g][32 rows][64 halves], 128B swizzle
  uint8_t* ring = slice + C::RES_BYTES;                       // [stage][64 rows][64 halves], 128B swizzle
  uint8_t* stg_all = ring + AS * C::A_STAGE;
  uint64_t* wfull = (uint64_t*)(stg_all + C::STG_BYTES);      // [k-block]: that k-block of the slice has landed
  uint64_t* full = wfull + C::KB_MAX;                         // [stage]
  uint64_t* empty = full + AS;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int H = p.H;
  const int num_m = (p.R + BM16 - 1) / BM16;
  const int num_n = H / 32;
  const int num_kb = H / BK16;
  const int nt = blockIdx.x % num_n, per = gridDim.x / num_n;   // this CTA's slice; CTAs per slice
  const int mb0 = blockIdx.x / num_n;                           // this CTA's first row block (none if >= num_m)

  if (threadIdx.x == 0) {
    for (int kb = 0; kb < num_kb; ++kb) mbar_init(&wfull[kb], 1);
    for (int s = 0; s < AS; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 1); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < 4) {
    if (threadIdx.x == 0 && mb0 < num_m) {
      // ===== TMA producer: the slice once, then per row block warpgroup 1's 64 rows of A, k-block by k-block, then
      // warpgroup 2's: the order of the turns
      for (int kb = 0; kb < num_kb; ++kb) {
        uint8_t* sb = slice + kb * C::SLICE_KB;
        mbar_expect_tx(&wfull[kb], C::SLICE_KB);
        // slice rows = [i | f | o | g] of 32 hidden units
#pragma unroll
        for (int g = 0; g < 4; ++g) tma_load_2d(sb + g * 4096, &tmB, &wfull[kb], kb * BK16, g * H + nt * 32);
      }
      int s = 0; uint32_t ph = 0;
      for (int mb = mb0; mb < num_m; mb += per) {
        for (int w = 0; w < 2; ++w) {
          for (int kb = 0; kb < num_kb; ++kb) {
            mbar_wait(&empty[s], ph ^ 1);
            mbar_expect_tx(&full[s], C::A_STAGE);
            tma_load_2d(ring + s * C::A_STAGE, &tmA, &full[s], kb * BK16, mb * BM16 + w * 64);
            if (++s == AS) { s = 0; ph ^= 1; }
          }
        }
      }
    }
  } else {
    const int cw = warp - 4, wg = cw >> 2;
    uint8_t* stg = stg_all + cw * C::STG_PER_WARP;
    // fragment rows of this thread within the warp's 16, and the unit pair within a group of 8 columns
    const int fr = lane >> 2, fu = 2 * (lane & 3);
    // main loop of one row block: this warpgroup's 64 rows x 128 columns against the resident slice.  Its k-blocks take
    // ring positions (2 j + wg) num_kb .. + num_kb - 1 in its j-th turn; (s, ph) = the ring position of the next one.
    int s = 0; uint32_t ph = 0;
    auto skip = [&](int n) {                                   // the other warpgroup's turn
      for (s += n; s >= AS; s -= AS) ph ^= 1;
    };
    skip(wg * num_kb);
    auto contract = [&](float (&d)[BN16 / 2], bool first) {
#pragma unroll
      for (int i = 0; i < BN16 / 2; ++i) d[i] = 0.f;
      int prev = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        if (first) mbar_wait(&wfull[kb], 0);
        mbar_wait(&full[s], ph);
        const uint64_t adesc = make_desc(smem_u32(ring + s * C::A_STAGE), 16, 1024),
                       bdesc = make_desc(smem_u32(slice + kb * C::SLICE_KB), 16, 1024);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK16 / UK16; ++k)
          wgmma_f16_n128(d, adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2), (kb | k) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty[prev]);
        prev = s;
        if (++s == AS) { s = 0; ph ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_hold(d);
      if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty[prev]);
      skip(num_kb);
    };
    // Tile columns [i | f | o | g] x 32 hidden units, so the thread holding column 8jj + fu of gate i holds the same unit of
    // f, o and g in fragments jj + 4, jj + 8, jj + 12: the pointwise step runs where the accumulators are.
    uint8_t* sG = stg; uint8_t* sH = stg + 4 * T16_BYTES; uint8_t* sC = sH + T16_BYTES;
    for (int mb = mb0; mb < num_m; mb += per) {
      // first hidden unit of the slice.  Opaque to the compiler, so that the bias and output addresses derived from it are
      // formed in the epilogue instead of being hoisted out of the loop, where they would spill
      int j0 = nt * 32;
      asm volatile("" : "+r"(j0));
      const int r0 = mb * BM16 + wg * 64 + (cw & 3) * 16;      // first of the warp's 16 rows
      const int64_t row = (int64_t)r0 + (lane & 15);           // lanes l and l + 16 both describe row l % 16
      const bool row_ok = row < p.R;
      const float keep = (row_ok && p.mask_ids && p.mask_ids[row] == 0) ? 0.f : 1.f;
      // A pad token's x-projection is exactly zero (LookupTableMaskZero: embedding row 0 is zero, and the table carries no
      // bias), so finished sequences skip the gather: at late time steps most of the 100 x 20-token options have ended, and
      // every row would otherwise read the same 4 KB of L2
      const int32_t tk = row_ok ? __ldg(p.tok + row) : 0;
      const __half* prow = tk != 0 ? p.ptable + (int64_t)tk * 4 * H + j0 : nullptr;
      const float* cprow = (row_ok && p.c_prev) ? p.c_prev + row * H + j0 : nullptr;
      if (lane == 0) bulk_wait_read0();                        // the previous block's TMA stores have read the staging tiles
      __syncwarp();
#pragma unroll
      for (int g = 0; g < 4; ++g) t16_load(sG + g * T16_BYTES, prow ? prow + g * H : nullptr, lane);
      t32_load(sC, cprow, lane);
      const bool first = mb == mb0;
      if (wg == 0) {
        if (!first) bar_named(TOKEN_WG1, 256);                 // warpgroup 2's main loop is done
      } else {
        bar_named(TOKEN_WG2, 256);                             // warpgroup 1's main loop is done
      }
      float d[BN16 / 2];
      contract(d, first);                                      // the loads fly while the MMAs of this block run
      if (wg == 0) bar_arrive_named(TOKEN_WG2, 256);
      else if (mb + per < num_m) bar_arrive_named(TOKEN_WG1, 256);
      cp_wait_all();
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int r = fr + 8 * hh;
        const float kp = __shfl_sync(0xffffffffu, keep, r);
        const int64_t grow = (int64_t)r0 + r;
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
          const int u = 8 * jj + fu;
          float a[4][2], cp[2], hn[2];
#pragma unroll
          for (int g = 0; g < 4; ++g) {
            const float2 x = ld_h2(t16_at(sG + g * T16_BYTES, r, u));
            const float2 b = __ldg(reinterpret_cast<const float2*>(p.bias + g * H + j0 + u));
            a[g][0] = d[4 * (jj + 4 * g) + 2 * hh] + (x.x + b.x);
            a[g][1] = d[4 * (jj + 4 * g) + 2 * hh + 1] + (x.y + b.y);
          }
          const float2 c2 = *reinterpret_cast<const float2*>(t32_at(sC, r, u));
          cp[0] = c2.x; cp[1] = c2.y;
#pragma unroll
          for (int e2 = 0; e2 < 2; ++e2) {
            const float gi = sig16(a[0][e2]), gf = sig16(a[1][e2]), go = sig16(a[2][e2]), gg = tanh16(a[3][e2]);
            const float c_ = (gf * cp[e2] + gi * gg) * kp;
            a[0][e2] = gi * kp; a[1][e2] = gf * kp; a[2][e2] = go * kp; a[3][e2] = gg * kp;
            cp[e2] = c_; hn[e2] = go * tanh16(c_) * kp;
          }
#pragma unroll
          for (int g = 0; g < 4; ++g) st_h2(t16_at(sG + g * T16_BYTES, r, u), a[g][0], a[g][1]);
          *reinterpret_cast<float2*>(t32_at(sC, r, u)) = make_float2(cp[0], cp[1]);
          st_h2(t16_at(sH, r, u), hn[0], hn[1]);
          if (p.h32_out && grow < p.R)                    // last step only: the fp32 h that meets the encoder output
            *reinterpret_cast<float2*>(p.h32_out + grow * H + j0 + u) = make_float2(hn[0], hn[1]);
        }
      }
      fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) {
        if (p.save_gates) {
#pragma unroll
          for (int g = 0; g < 4; ++g) tma_store_2d(&em.g16, sG + g * T16_BYTES, g * H + j0, r0);
        }
        tma_store_2d(&em.c, sC, j0, r0);
        tma_store_2d(&em.h16, sH, j0, r0);
        bulk_commit();
      }
      __syncwarp();
    }
    if (lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");   // all TMA stores performed
  }
}

// ------------------------------------------------------------------------------------------------
// Backward (BPTT): one cluster of H / 128 CTAs per 128-row block runs the block's whole time loop, t = t_hi .. 0, in one
// launch.  CTA u of the cluster owns hidden units 128u .. 128u + 127 of the block (its tile: dh = da_{t+1} Whb[units]^T over
// all 4H of k), so the cluster's CTAs together write all 4H columns of the block's da_t, which is what every one of them reads
// as its A operand at step t - 1: a cluster barrier between the steps is the only coupling (option rows are independent
// sequences), clusters never wait on each other.  The fp32 cell-gradient carry dc stays on chip for the whole loop, in the
// accumulator-fragment layout (64 floats per consumer thread: 32 in registers beside the 64 accumulators, 32 in shared
// memory): it is read once before the first step and written once after the last.
//
// Visibility of da_t to the next step's TMA loads (async proxy -> global -> async proxy, across the CTAs of the cluster):
//   1. every consumer warp waits until its bulk stores of da_t are complete (cp.async.bulk.wait_group 0 — not .read, which
//      only says that the staging tiles may be reused);
//   2. fence.proxy.async.global orders them against the generic-proxy release that follows;
//   3. barrier.cluster.arrive.release by every thread, barrier.cluster.wait.acquire by every thread;
//   4. only then does the producer thread, after one more fence.proxy.async.global, issue the TMA loads of da_t.
// The producer may run ahead of its consumers into the next step's loads only as far as this barrier.
struct Bptt16 {
  static constexpr int THREADS = 128 + 32 * EW16;
  // per-warp staging: {4 gate tiles T16 (the inputs, overwritten by da), c_{t-1}, c_t T32} = 8 KB
  static constexpr int STG_PER_WARP = 4 * T16_BYTES + 2 * T32_BYTES;
  static constexpr int STG_BYTES = EW16 * STG_PER_WARP;                       // 64 KB
  static constexpr int DCS_BYTES = 256 * (BN16 / 4) * 4;                    // half of the dc carry: 32 KB
  static constexpr int STAGES = (232448 - 1024 - 256 - STG_BYTES - DCS_BYTES) / STAGE16;   // 4
  static constexpr int TOTAL = STAGES * STAGE16 + STG_BYTES + DCS_BYTES + 1024 + 256;    // + alignment slack + barriers
  static_assert(STAGES >= 4 && TOTAL <= 232448, "k_lstm16_bptt: shared memory");
  // the producer warpgroup hands registers to the consumers (128 x 40 + 256 x 232 <= 64 K): without it the consumers spill
  static constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;
};
struct Bptt16Params {
  int R, H;
  int mb0;                                 // row block of cluster 0; cluster c runs block mb0 + c
  int t_hi;                                // steps t_hi, t_hi - 1, ..., 0
  const __half* gates; int64_t g_step;     // saved fp16 gates of step t at gates + t g_step, (R, 4H)
  const float* c; int64_t c_step;          // c_t at c + t c_step, (R, H); c_{t-1} likewise, and c0 (null: zeros) for t = 0
  const float* c0;
  const int32_t* mask; int64_t m_step;     // maskzero ids of step t at mask + t m_step, or null
  float* dc_carry;                         // (R, H) fp32: the carry into step t_hi in, the carry out of step 0 out
};

__device__ __forceinline__ void cluster_arrive_release() { asm volatile("barrier.cluster.arrive.release;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait_acquire() { asm volatile("barrier.cluster.wait.acquire;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }

// tmA: da_{t+1} of step t as slice z = t of an (R, 4H) x z tensor, 128 x 64 boxes; tmB: Whb (H, 4H), 128 x 64 boxes;
// tmD: da_t as slice z = t, 16 x 32 boxes (SWIZZLE_64B, the T16 staging tiles)
__global__ void __launch_bounds__(Bptt16::THREADS, 1)
k_lstm16_bptt(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
              const __grid_constant__ CUtensorMap tmD, const Bptt16Params p) {
  using C = Bptt16;
  constexpr int STAGES = C::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint8_t* stg_all = smem + STAGES * STAGE16;
  uint64_t* full = (uint64_t*)(stg_all + C::STG_BYTES + C::DCS_BYTES);
  uint64_t* empty = full + STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int H = p.H;
  const int num_n = H / BN16;                                  // = the cluster size (a 1-D grid of 1-D clusters)
  const int nt = blockIdx.x % num_n;
  const int m0 = (p.mb0 + blockIdx.x / num_n) * BM16;
  const int num_kb = 4 * H / BK16;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(C::PRODUCER_REGS));
    // ===== TMA producer: 128 rows of A, 128 rows of B per k-block.  Every thread of the warpgroup takes part in the
    // cluster barrier between the steps; thread 0 issues the loads.
    int s = 0; uint32_t ph = 0;
    for (int t = p.t_hi; t >= 0; --t) {
      if (t < p.t_hi) { cluster_arrive_release(); cluster_wait_acquire(); }   // da_t of step t + 1 is in global memory
      if (threadIdx.x == 0) {
        if (t < p.t_hi) fence_proxy_async_global();
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty[s], ph ^ 1);
          uint8_t* sa = smem + s * STAGE16;
          uint8_t* sb = sa + 16384;
          mbar_expect_tx(&full[s], STAGE16);
          tma_load_3d(sa, &tmA, &full[s], kb * BK16, m0, t);
          tma_load_2d(sb, &tmB, &full[s], kb * BK16, nt * BN16);
          if (++s == STAGES) { s = 0; ph ^= 1; }
        }
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(C::CONSUMER_REGS));
    const int cw = warp - 4, wg = cw >> 2;
    uint8_t* stg = stg_all + cw * C::STG_PER_WARP;
    // fragment rows of this thread within the warp's 16, and the unit pair within a group of 8 columns
    const int fr = lane >> 2, fu = 2 * (lane & 3);
    int s = 0; uint32_t ph = 0;
    // main loop of one step: this warpgroup's 64 rows x 128 columns, accumulated in registers
    auto contract = [&](float (&d)[BN16 / 2]) {
#pragma unroll
      for (int i = 0; i < BN16 / 2; ++i) d[i] = 0.f;
      int prev = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full[s], ph);
        const uint32_t sa = smem_u32(smem + s * STAGE16);
        const uint64_t adesc = make_desc(sa + wg * 64 * 128, 16, 1024), bdesc = make_desc(sa + 16384, 16, 1024);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK16 / UK16; ++k)
          wgmma_f16_n128(d, adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2), (kb | k) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty[prev]);
        prev = s;
        if (++s == STAGES) { s = 0; ph ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_hold(d);
      if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty[prev]);
    };
    // 128 hidden units per tile = 4 groups of 32; fragment columns are hidden units, so the thread reads the gates / c of
    // exactly the units its accumulators (and its dc carry) hold
    uint8_t* sG = stg; uint8_t* sCP = stg + 4 * T16_BYTES; uint8_t* sCC = sCP + T32_BYTES;
    const int r0 = m0 + wg * 64 + (cw & 3) * 16;               // first of the warp's 16 rows
    const int64_t row = (int64_t)r0 + (lane & 15);             // lanes l and l + 16 both describe row l % 16
    const bool row_ok = row < p.R;
    const int j0 = nt * BN16;
    // the dc carry in d's layout: element i = 4 jb + 2 hh + e is dc of row r0 + fr + 8 hh, unit j0 + 8 jb + fu + e.  The
    // first two groups' (i < 32) live in registers, the last two's in shared memory, [i - 32][consumer thread] (a warp's
    // accesses are 32 consecutive words): all 64 beside the 64 accumulators do not fit in the 168 registers of a thread.
    float dcr[BN16 / 4];
    float* dcs = reinterpret_cast<float*>(stg_all + C::STG_BYTES) + (threadIdx.x - 128);
    auto dc_at = [&](int i) -> float& { return i < BN16 / 4 ? dcr[i] : dcs[(i - BN16 / 4) * 256]; };
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int64_t rr = (int64_t)r0 + fr + 8 * hh;
#pragma unroll
      for (int jb = 0; jb < BN16 / 8; ++jb) {
        const float2 v = rr < p.R ? *reinterpret_cast<const float2*>(p.dc_carry + rr * H + j0 + 8 * jb + fu) : make_float2(0.f, 0.f);
        dc_at(4 * jb + 2 * hh) = v.x; dc_at(4 * jb + 2 * hh + 1) = v.y;
      }
    }
    // inputs of step t, hidden units j .. j + 31 -> staging.  The row is made opaque to the compiler, so that the addresses
    // derived from it are formed here instead of being hoisted out of the step loop, where they would spill
    auto fetch = [&](int t, int j) {
      int64_t row = (int64_t)r0 + (lane & 15);
      asm volatile("" : "+l"(row));
      const __half* grow = row_ok ? p.gates + t * p.g_step + row * 4 * H : nullptr;
      const float* cpbase = t > 0 ? p.c + (t - 1) * p.c_step : p.c0;
      const float* cprow = (row_ok && cpbase) ? cpbase + row * H : nullptr;
      const float* ccrow = row_ok ? p.c + t * p.c_step + row * H : nullptr;
      if (lane == 0) bulk_wait_read0();
      __syncwarp();
#pragma unroll
      for (int g = 0; g < 4; ++g) t16_load(sG + g * T16_BYTES, grow ? grow + g * H + j : nullptr, lane);
      t32_load(sCP, cprow ? cprow + j : nullptr, lane);
      t32_load(sCC, ccrow ? ccrow + j : nullptr, lane);
    };
    fetch(p.t_hi, j0);
    for (int t = p.t_hi; t >= 0; --t) {
      const float keep = (row_ok && p.mask && p.mask[t * p.m_step + row] == 0) ? 0.f : 1.f;
      float d[BN16 / 2];
      contract(d);
#pragma unroll
      for (int grp = 0; grp < BN16 / 32; ++grp) {
        const int j = j0 + grp * 32;
        if (grp > 0) fetch(t, j);
        cp_wait_all();
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int r = fr + 8 * hh;
          const float keep_r = __shfl_sync(0xffffffffu, keep, r);
#pragma unroll
          for (int jj = 0; jj < 4; ++jj) {
            const int u = 8 * jj + fu;
            float g[4][2], cp[2], cc[2], out[4][2];
#pragma unroll
            for (int gg = 0; gg < 4; ++gg) {
              const float2 x = ld_h2(t16_at(sG + gg * T16_BYTES, r, u));
              g[gg][0] = x.x; g[gg][1] = x.y;
            }
            const float2 cp2 = *reinterpret_cast<const float2*>(t32_at(sCP, r, u));
            const float2 cc2 = *reinterpret_cast<const float2*>(t32_at(sCC, r, u));
            cp[0] = cp2.x; cp[1] = cp2.y; cc[0] = cc2.x; cc[1] = cc2.y;
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int i = 4 * (4 * grp + jj) + 2 * hh + e;
              const float dh = d[i];
              const float gi = g[0][e], gf = g[1][e], go = g[2][e], gg_ = g[3][e];
              const float tcv = tanh16(cc[e]);
              const float dd = (dc_at(i) + dh * go * (1.f - tcv * tcv)) * keep_r;
              const float dhe = dh * keep_r;
              out[0][e] = dd * gg_ * gi * (1.f - gi);
              out[1][e] = dd * cp[e] * gf * (1.f - gf);
              out[2][e] = dhe * tcv * go * (1.f - go);
              out[3][e] = dd * gi * (1.f - gg_ * gg_);
              dc_at(i) = dd * gf;
            }
#pragma unroll
            for (int gg = 0; gg < 4; ++gg) st_h2(t16_at(sG + gg * T16_BYTES, r, u), out[gg][0], out[gg][1]);
          }
        }
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) {
#pragma unroll
          for (int gg = 0; gg < 4; ++gg) tma_store_3d(&tmD, sG + gg * T16_BYTES, gg * H + j, r0, t);
          bulk_commit();
        }
        __syncwarp();
      }
      if (t > 0) {
        if (lane == 0) {
          asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");   // this warp's da_t is in global memory
          fence_proxy_async_global();
        }
        __syncwarp();
        cluster_arrive_release();
        fetch(t - 1, j0);                                      // the next step's first inputs fly across the barrier
        cluster_wait_acquire();                                // (pairs the arrive; nothing here reads da_t)
      }
    }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int64_t rr = (int64_t)r0 + fr + 8 * hh;
      if (rr < p.R) {
#pragma unroll
        for (int jb = 0; jb < BN16 / 8; ++jb)
          *reinterpret_cast<float2*>(p.dc_carry + rr * H + j0 + 8 * jb + fu) = make_float2(dc_at(4 * jb + 2 * hh), dc_at(4 * jb + 2 * hh + 1));
      }
    }
    if (lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");   // all TMA stores performed
  }
}

// ------------------------------------------------------------------------------------------------
// Weight gradient of the recurrent block:  C[m,n] += inv_scale * sum_k A[k,m] B[k,n],  A = h (K rows x H) fp16,
// B = da (K rows x 4H) fp16 — both MN-major (the contraction index is the row index in HBM).  A TMA box of 64 columns
// x KB rows lands as KB rows of 128 bytes = the canonical MN-major SWIZZLE_128B layout (8 k-rows per 1024-byte atom:
// SBO = 1024; 64-column groups LBO bytes apart), which the f16 wgmma reads transposed; one K = 16 instruction consumes
// two atoms.  Warpgroup 0 = TMA producer, warpgroups 1-2 = consumers (64 rows of the 128 x 256 tile each, m64n256k16).
//
// Stream-K: every tile's k-blocks are cut into chunks of `chunk` k-blocks (the last one of a tile shorter), numbered
// k-range-major — chunk c = (k-range c / tiles, tile c % tiles) — so that the CTAs running at one time work on the same rows
// of A and B for different tiles, and those rows come from HBM once and are reused from L2 (tile-major order would read
// the operands once per tile).  The producer claims chunks from a device counter and tags the chunk's first stage with its
// number; the consumers add each finished partial tile into C with red.global.add (C is accumulated with atomics anyway,
// so no fix-up pass).  A CTA that starts late, behind kernels of other streams, claims fewer chunks.  The last CTA to
// finish resets the counter, so one zeroed counter per stream serves every launch on it.
// SLOT (deterministic mode): the chunk plan follows from the shape alone, and a chunk's partial tile is stored into the slot of
// its k-range (ws: k-ranges x M x N) instead; slot_reduce then adds the slots to C in k-range order, so the sum does not depend
// on which CTA claimed which chunk.
constexpr int A16_KB = 64;                 // k-rows per stage (4 MMAs)
constexpr int A16_BM = 128, A16_BN = 256;
constexpr int A16_THREADS = 384;
constexpr int A16_A_BYTES = (A16_BM / 64) * A16_KB * 128;  // 2 boxes of 64 columns
constexpr int A16_B_BYTES = (A16_BN / 64) * A16_KB * 128;  // 4 boxes
constexpr int A16_STAGE = A16_A_BYTES + A16_B_BYTES;       // 48 KB
constexpr int A16_STAGES = 4;
constexpr int A16_TOTAL = A16_STAGES * A16_STAGE + 1024 + 256;
constexpr int A16_CHUNKS_PER_CTA = 24;     // chunk length: ~24 claims per CTA (tail imbalance < 1/24), at least
constexpr int A16_MIN_CHUNK = 32;          // 32 k-blocks (the partial-tile reduction stays a few % of the chunk)
struct Atb16Params {
  int M, N, tiles_n, tiles, kbt;           // kbt = k-blocks per tile
  int chunk, num_chunks;                   // k-blocks per chunk, chunks (tiles x k-ranges)
  float* C; int64_t ldc; const float* inv_scale;
  int* counter;                            // [0] next chunk, [1] CTAs done; both zero between launches
  float* ws;                               // SLOT: the k-range slots
};
constexpr int A16_DET_RANGES = 16;         // SLOT: k-ranges (partial tiles per tile) at most

template <bool VEC4, bool SLOT>   // VEC4: C 16-byte aligned with ldc % 4 == 0: the partial tiles go out as red.global.add.v4
__global__ void __launch_bounds__(A16_THREADS, 1)
k_atb16(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const Atb16Params p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint64_t* full = (uint64_t*)(smem + A16_STAGES * A16_STAGE);
  uint64_t* empty = full + A16_STAGES;
  int* tag = (int*)(empty + A16_STAGES);                     // chunk of a chunk's first stage, -1 = no more work
  const int warp = threadIdx.x >> 5;

  if (threadIdx.x == 0) {
    for (int s = 0; s < A16_STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < 4) {
    if (threadIdx.x == 0) {
      int s = 0; uint32_t ph = 0;
      for (;;) {
        const int c = atomicAdd(p.counter, 1);
        if (c >= p.num_chunks) break;
        const int tile = c % p.tiles, kb0 = (c / p.tiles) * p.chunk, kb1 = min(p.kbt, kb0 + p.chunk);
        const int m0 = (tile / p.tiles_n) * A16_BM, n0 = (tile % p.tiles_n) * A16_BN;
        for (int kb = kb0; kb < kb1; ++kb) {
          const int krow = kb * A16_KB;
          mbar_wait(&empty[s], ph ^ 1);
          uint8_t* sa = smem + s * A16_STAGE;
          uint8_t* sb = sa + A16_A_BYTES;
          if (kb == kb0) tag[s] = c;
          mbar_expect_tx(&full[s], A16_STAGE);       // out-of-range rows / columns land as zeros and still count
#pragma unroll
          for (int b = 0; b < A16_BM / 64; ++b) tma_load_2d(sa + b * A16_KB * 128, &tmA, &full[s], m0 + b * 64, krow);
#pragma unroll
          for (int b = 0; b < A16_BN / 64; ++b) tma_load_2d(sb + b * A16_KB * 128, &tmB, &full[s], n0 + b * 64, krow);
          if (++s == A16_STAGES) { s = 0; ph ^= 1; }
        }
      }
      mbar_wait(&empty[s], ph ^ 1);
      tag[s] = -1;
      mbar_arrive(&full[s]);
      // every CTA has made its last claim once all have counted themselves here: the last one resets the counter
      __threadfence();
      if (atomicAdd(p.counter + 1, 1) == (int)gridDim.x - 1) {
        atomicExch(p.counter, 0);
        atomicExch(p.counter + 1, 0);
      }
    }
  } else {
    const int wg = (warp - 4) >> 2, lane = threadIdx.x & 31, w = warp & 3;
    const float sc = p.inv_scale ? __ldg(p.inv_scale) : 1.f;
    float d[A16_BN / 2];
    int s = 0; uint32_t ph = 0;
    for (;;) {
      mbar_wait(&full[s], ph);
      const int c = tag[s];
      if (c < 0) break;
      const int tile = c % p.tiles, kb0 = (c / p.tiles) * p.chunk;
      const int nseg = min(p.kbt - kb0, p.chunk);        // k-blocks of this partial tile
      int prev = -1;
      for (int i = 0; i < nseg; ++i) {
        if (i > 0) mbar_wait(&full[s], ph);
        const uint32_t sa = smem_u32(smem + s * A16_STAGE);
        const uint32_t sb = sa + A16_A_BYTES;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < A16_KB / UK16; ++k)
          wgmma_f16_n256_mn(d, make_desc(sa + wg * A16_KB * 128 + k * 2048, A16_KB * 128, 1024),
                            make_desc(sb + k * 2048, A16_KB * 128, 1024), (i | k) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty[prev]);
        prev = s;
        if (++s == A16_STAGES) { s = 0; ph ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_hold(d);
      if ((threadIdx.x & 127) == 0) mbar_arrive(&empty[prev]);
      const int m = (tile / p.tiles_n) * A16_BM + wg * 64 + 16 * w + (lane >> 2);
      const int n0 = (tile % p.tiles_n) * A16_BN + 2 * (lane & 3);
      if constexpr (VEC4) {
        // lane pairs (q, q^1) swap half their fragment: the even lane adds 4 consecutive columns of row m, the odd one of row m + 8
        const bool odd = lane & 1;
        const int row = odd ? m + 8 : m;
#pragma unroll
        for (int j = 0; j < A16_BN / 8; ++j) {
          const float s0 = odd ? d[4 * j] : d[4 * j + 2], s1 = odd ? d[4 * j + 1] : d[4 * j + 3];
          const float k0 = odd ? d[4 * j + 2] : d[4 * j], k1 = odd ? d[4 * j + 3] : d[4 * j + 1];
          const float r0 = __shfl_xor_sync(0xffffffffu, s0, 1), r1 = __shfl_xor_sync(0xffffffffu, s1, 1);
          const int col = n0 + 8 * j - (odd ? 2 : 0);
          const float4 v = odd ? make_float4(r0 * sc, r1 * sc, k0 * sc, k1 * sc) : make_float4(k0 * sc, k1 * sc, r0 * sc, r1 * sc);
          if (row < p.M && col < p.N) {                // M, N multiples of 64: a 4-column group is all in or all out
            if constexpr (SLOT)
              *reinterpret_cast<float4*>(p.ws + ((int64_t)(c / p.tiles) * p.M + row) * p.N + col) = v;
            else red_add_v4(p.C + (int64_t)row * p.ldc + col, v.x, v.y, v.z, v.w);
          }
        }
      } else {
#pragma unroll
        for (int j = 0; j < A16_BN / 8; ++j) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = m + 8 * h, col = n0 + 8 * j;
            const float v0 = d[4 * j + 2 * h] * sc, v1 = d[4 * j + 2 * h + 1] * sc;
            if (row < p.M && col < p.N) {
              float* dst = p.C + (int64_t)row * p.ldc + col;
              atomicAdd(dst, v0);
              atomicAdd(dst + 1, v1);
            }
          }
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ streaming helpers
// t = 0 without initial state: pre-activation = P16[tok] + bias.  One thread per (row, 8 hidden units).
__global__ void __launch_bounds__(256)
k_lstm16_first(const __half* __restrict__ ptable, const int32_t* __restrict__ tok, const float* __restrict__ bias,
               const float* __restrict__ c_prev, const int32_t* __restrict__ mask_ids, __half* __restrict__ gates,
               float* __restrict__ c_out, __half* __restrict__ h16, float* __restrict__ h32, int64_t R, int H) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int H8 = H >> 3;
  if (idx >= R * H8) return;
  const int64_t r = idx / H8;
  const int j = (int)(idx % H8) * 8;
  const float keep = (mask_ids && mask_ids[r] == 0) ? 0.f : 1.f;
  const int32_t tk = tok[r];
  const __half* src = ptable + (int64_t)tk * 4 * H;
  float a[4][8], cp[8], cn[8], hn[8];
#pragma unroll
  for (int g = 0; g < 4; ++g) {
    unpack8(tk != 0 ? __ldg(reinterpret_cast<const uint4*>(src + g * H + j)) : make_uint4(0, 0, 0, 0), a[g]);   // pad: exactly zero
    const float4 b0 = __ldg(reinterpret_cast<const float4*>(bias + g * H + j)), b1 = __ldg(reinterpret_cast<const float4*>(bias + g * H + j) + 1);
    a[g][0] += b0.x; a[g][1] += b0.y; a[g][2] += b0.z; a[g][3] += b0.w; a[g][4] += b1.x; a[g][5] += b1.y; a[g][6] += b1.z; a[g][7] += b1.w;
  }
  if (c_prev) {
    const float4 c0 = *reinterpret_cast<const float4*>(c_prev + r * H + j), c1 = *(reinterpret_cast<const float4*>(c_prev + r * H + j) + 1);
    cp[0] = c0.x; cp[1] = c0.y; cp[2] = c0.z; cp[3] = c0.w; cp[4] = c1.x; cp[5] = c1.y; cp[6] = c1.z; cp[7] = c1.w;
  } else {
#pragma unroll
    for (int e = 0; e < 8; ++e) cp[e] = 0.f;
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const float gi = fsigmoid(a[0][e]), gf = fsigmoid(a[1][e]), go = fsigmoid(a[2][e]), gg = ftanh(a[3][e]);
    const float c_ = gf * cp[e] + gi * gg;
    a[0][e] = gi * keep; a[1][e] = gf * keep; a[2][e] = go * keep; a[3][e] = gg * keep;
    cn[e] = c_ * keep; hn[e] = go * ftanh(c_) * keep;
  }
  if (gates) {
#pragma unroll
    for (int g = 0; g < 4; ++g) __stcs(reinterpret_cast<uint4*>(gates + r * 4 * H + g * H + j), pack8(a[g]));
  }
  float4* co = reinterpret_cast<float4*>(c_out + r * H + j);
  co[0] = make_float4(cn[0], cn[1], cn[2], cn[3]); co[1] = make_float4(cn[4], cn[5], cn[6], cn[7]);
  *reinterpret_cast<uint4*>(h16 + r * H + j) = pack8(hn);
  if (h32) {
    float4* ho = reinterpret_cast<float4*>(h32 + r * H + j);
    ho[0] = make_float4(hn[0], hn[1], hn[2], hn[3]); ho[1] = make_float4(hn[4], hn[5], hn[6], hn[7]);
  }
}

// t = T-1 of the BPTT: no recurrent gradient yet; dh = scale * dh_last (the power-of-two gradient scale enters here)
__global__ void __launch_bounds__(256)
k_lstm16_bwd_last(const __half* __restrict__ gates, const float* __restrict__ c_prev, const float* __restrict__ c_cur,
                  const float* __restrict__ dh_last, const float* __restrict__ scale, const int32_t* __restrict__ mask_ids,
                  float* __restrict__ dc_carry, __half* __restrict__ da, int64_t R, int H) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int H8 = H >> 3;
  if (idx >= R * H8) return;
  const int64_t r = idx / H8;
  const int j = (int)(idx % H8) * 8;
  const float keep = (mask_ids && mask_ids[r] == 0) ? 0.f : 1.f;
  const float s = __ldg(scale);
  float g[4][8], cp[8], cc[8], dh[8], out[4][8], dcn[8];
#pragma unroll
  for (int gg = 0; gg < 4; ++gg) unpack8(__ldcs(reinterpret_cast<const uint4*>(gates + r * 4 * H + gg * H + j)), g[gg]);
  auto ld8f = [](const float* p, float* d) {
    const float4 x0 = *reinterpret_cast<const float4*>(p), x1 = *(reinterpret_cast<const float4*>(p) + 1);
    d[0] = x0.x; d[1] = x0.y; d[2] = x0.z; d[3] = x0.w; d[4] = x1.x; d[5] = x1.y; d[6] = x1.z; d[7] = x1.w;
  };
  if (c_prev) ld8f(c_prev + r * H + j, cp);
  else {
#pragma unroll
    for (int e = 0; e < 8; ++e) cp[e] = 0.f;
  }
  ld8f(c_cur + r * H + j, cc);
  ld8f(dh_last + r * H + j, dh);
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const float gi = g[0][e], gf = g[1][e], go = g[2][e], gg_ = g[3][e];
    const float dhe = dh[e] * s * keep;
    const float tcv = tanh16(cc[e]);
    const float d = dhe * go * (1.f - tcv * tcv);
    out[0][e] = d * gg_ * gi * (1.f - gi);
    out[1][e] = d * cp[e] * gf * (1.f - gf);
    out[2][e] = dhe * tcv * go * (1.f - go);
    out[3][e] = d * gi * (1.f - gg_ * gg_);
    dcn[e] = d * gf;
  }
#pragma unroll
  for (int gg = 0; gg < 4; ++gg) *reinterpret_cast<uint4*>(da + r * 4 * H + gg * H + j) = pack8(out[gg]);
  float4* o = reinterpret_cast<float4*>(dc_carry + r * H + j);
  o[0] = make_float4(dcn[0], dcn[1], dcn[2], dcn[3]); o[1] = make_float4(dcn[4], dcn[5], dcn[6], dcn[7]);
}

// 2-D fp32 -> fp16 (weights, projection table)
__global__ void k_cvt16(__half* __restrict__ dst, int64_t ldd, const float* __restrict__ src, int64_t lds, int64_t rows, int cols) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int c4 = cols >> 2;
  if (idx >= rows * c4) return;
  const int64_t r = idx / c4;
  const int c = (int)(idx % c4) * 4;
  const float4 v = *reinterpret_cast<const float4*>(src + r * lds + c);
  *reinterpret_cast<uint2*>(dst + r * ldd + c) = make_uint2(pack2(v.x, v.y), pack2(v.z, v.w));
}

// max |x| -> bits[0] (atomicMax on the IEEE bit pattern of a non-negative float)
__global__ void __launch_bounds__(256) k_amax(const float* __restrict__ x, int64_t n4, uint32_t* __restrict__ bits) {
  float m = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(x) + i);
    m = fmaxf(m, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(bits, __float_as_uint(m));
}
// scale = the power of two that brings max|dh| to [2^9, 2^10): 6 binades of head-room below the fp16 maximum for the
// growth of da through the recurrence, 24 binades (normal + subnormal) below for the small gradients
__global__ void k_pick_scale(const uint32_t* __restrict__ bits, float* __restrict__ out2) {
  const float amax = __uint_as_float(bits[0]);
  float s = 1.f;
  if (amax > 0.f && isfinite(amax)) {
    int e; frexpf(amax, &e);                         // amax = f * 2^e, f in [0.5, 1)
    int k = 10 - e;
    k = max(-60, min(60, k));
    s = ldexpf(1.f, k);
  }
  out2[0] = s; out2[1] = 1.f / s;
}

// segmented row sum over fp16 rows (see k_segsum_rows in pointwise.cu): out[tok,:] += inv_scale * sum of X[perm[p],:]
constexpr int SEG16_ROWS = 64;
__global__ void __launch_bounds__(256)
k_segsum16(const __half* __restrict__ X, int64_t ldx, const int32_t* __restrict__ perm, const int32_t* __restrict__ sorted_tok,
           int64_t n, float* __restrict__ out, int ncols, const float* __restrict__ inv_scale) {
  const int64_t p0 = (int64_t)blockIdx.x * SEG16_ROWS, p1 = min(n, p0 + SEG16_ROWS);
  const float sc = inv_scale ? __ldg(inv_scale) : 1.f;
  for (int c0 = threadIdx.x * 8; c0 < ncols; c0 += blockDim.x * 8) {
    float acc[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] = 0.f;
    int cur = sorted_tok[p0];
    auto flush = [&](int tok) {
      float* o = out + (int64_t)tok * ncols + c0;
      red_add_v4(o, acc[0] * sc, acc[1] * sc, acc[2] * sc, acc[3] * sc);
      red_add_v4(o + 4, acc[4] * sc, acc[5] * sc, acc[6] * sc, acc[7] * sc);
    };
    for (int64_t p = p0; p < p1; ++p) {
      const int tok = sorted_tok[p];
      if (tok != cur) {
        flush(cur);
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] = 0.f;
        cur = tok;
      }
      float v[8];
      unpack8(__ldcs(reinterpret_cast<const uint4*>(X + (int64_t)perm[p] * ldx + c0)), v);
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[e] += v[e];
    }
    flush(cur);
  }
}

// ------------------------------------------------------------------------------------------------ host
static CUtensorMap make_tmap16(const void* base, CUtensorMapDataType dt, int esize, int64_t rows, int64_t cols, int64_t ld,
                               int box_rows, int box_cols, CUtensorMapSwizzle swz) {
  CUtensorMap tm;
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * esize};
  cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = get_encode()(&tm, dt, 2, (void*)base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
                            CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char buf[256];
    snprintf(buf, sizeof(buf), "cuTensorMapEncodeTiled (lstm16) failed (%d): base %p rows %lld cols %lld ld %lld box %dx%d", (int)r, base,
             (long long)rows, (long long)cols, (long long)ld, box_rows, box_cols);
    throw CudaError(-3, buf);
  }
  return tm;
}
static CUtensorMap tmap_h(const __half* base, int64_t rows, int64_t cols, int64_t ld, int box_rows, int box_cols,
                          CUtensorMapSwizzle swz) {
  return make_tmap16(base, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, rows, cols, ld, box_rows, box_cols, swz);
}
static CUtensorMap tmap_f(const float* base, int64_t rows, int64_t cols, int64_t ld, int box_rows, int box_cols,
                          CUtensorMapSwizzle swz) {
  return make_tmap16(base, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, rows, cols, ld, box_rows, box_cols, swz);
}

// persistent, balanced waves (see gemm_tc.cu::launch): the fewest workers, at most pmax, that take cdiv(n, pmax) items each
static int balanced_workers(int n, int pmax) { return n <= pmax ? n : cdiv(n, cdiv(n, pmax)); }

template <int MODE>
static void launch16(LaunchCtx& cx, const CUtensorMap& tA, const CUtensorMap& tB, const Lstm16Maps& em, const Lstm16Params& p,
                     int grid) {
  using C = Cfg16<MODE>;
  static bool attr_set = false;
  if (!attr_set) {
    VD_CUDA_CHECK(cudaFuncSetAttribute(k_lstm16<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::TOTAL));
    attr_set = true;
  }
  k_lstm16<MODE><<<grid, C::THREADS, C::TOTAL, cx.stream>>>(tA, tB, em, p);
  check_launch(cx, "k_lstm16");
}

}  // namespace tc

// H = 256 or 512: the BPTT's clusters are H / 128 = 2 or 4 CTAs
bool lstm16_shape_ok(int64_t R, int H) { return (H == 256 || H == 512) && R >= 1024; }

void lstm16_step_fwd(LaunchCtx& cx, int64_t R, int H, const __half* h_prev16, const __half* Wh16, const __half* ptable16,
                     const int32_t* tok, const float* bias, const float* c_prev, const int32_t* mask_ids, __half* gates16,
                     float* c_out, __half* h16_out, float* h32_out) {
  using namespace tc;
  VD_REQUIRE(lstm16_shape_ok(R, H), VD_E_STATE, "lstm16_step_fwd: shape");
  Lstm16Params p = {};
  p.R = (int)R; p.H = H; p.ptable = ptable16; p.tok = tok; p.bias = bias; p.c_prev = c_prev; p.mask_ids = mask_ids;
  p.h32_out = h32_out; p.save_gates = gates16 != nullptr;
  CUtensorMap tA = tmap_h(h_prev16, R, H, H, 64, BK16, CU_TENSOR_MAP_SWIZZLE_128B);       // one warpgroup's 64 rows
  CUtensorMap tB = tmap_h(Wh16, 4 * (int64_t)H, H, H, 32, BK16, CU_TENSOR_MAP_SWIZZLE_128B);
  Lstm16Maps em;
  em.g16 = gates16 ? tmap_h(gates16, R, 4 * (int64_t)H, 4 * (int64_t)H, 16, 32, CU_TENSOR_MAP_SWIZZLE_64B)
                   : tmap_h(h16_out, R, H, H, 16, 32, CU_TENSOR_MAP_SWIZZLE_64B);
  em.c = tmap_f(c_out, R, H, H, 16, 32, CU_TENSOR_MAP_SWIZZLE_128B);
  em.h16 = tmap_h(h16_out, R, H, H, 16, 32, CU_TENSOR_MAP_SWIZZLE_64B);
  // each of the H / 32 column slices gets the same number of CTAs, which split its 128-row blocks evenly
  const int slices = H / 32;
  launch16<0>(cx, tA, tB, em, p, slices * balanced_workers(cdiv(R, BM16), std::max(1, cx.sms() / slices)));
}

Bptt16Plan lstm16_bptt_plan(LaunchCtx& cx, int64_t R, int H) {
  using namespace tc;
  VD_REQUIRE(lstm16_shape_ok(R, H), VD_E_STATE, "lstm16_bptt_plan: shape");
  const int csize = H / BN16;
  // clusters of k_lstm16_bptt the device can hold at once, per cluster size (the kernel's shared memory gives one CTA per SM)
  static std::mutex mu;
  static std::map<std::pair<int, int>, int> fit;
  int dev = 0;
  VD_CUDA_CHECK(cudaGetDevice(&dev));
  int maxc = 0;
  {
    std::lock_guard<std::mutex> lock(mu);
    int& f = fit[{dev, csize}];
    if (f == 0) {
      VD_CUDA_CHECK(cudaFuncSetAttribute(k_lstm16_bptt, cudaFuncAttributeMaxDynamicSharedMemorySize, Bptt16::TOTAL));
      cudaLaunchConfig_t cfg = {};
      cudaLaunchAttribute attr[1];
      attr[0].id = cudaLaunchAttributeClusterDimension;
      attr[0].val.clusterDim.x = csize; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
      cfg.gridDim = dim3(csize * std::max(1, cx.sm_count / csize)); cfg.blockDim = dim3(Bptt16::THREADS); cfg.dynamicSmemBytes = Bptt16::TOTAL;
      cfg.attrs = attr; cfg.numAttrs = 1;
      VD_CUDA_CHECK(cudaOccupancyMaxActiveClusters(&f, k_lstm16_bptt, &cfg));
      VD_REQUIRE(f >= 1, VD_E_STATE, "k_lstm16_bptt: no cluster fits on the device");
    }
    maxc = f;
  }
  // as many clusters as fit and as the SM budget allows, balanced over the waves
  const int num_m = cdiv(R, BM16);
  Bptt16Plan pl;
  pl.csize = csize;
  pl.clusters = balanced_workers(num_m, std::max(1, std::min(maxc, cx.sms() / csize)));
  pl.waves = cdiv(num_m, pl.clusters);
  return pl;
}

// steps t_hi .. 0 of every row block, a wave of clusters per launch.  The tensors of step t: da_{t+1} = slice t of da_in
// (z slices of (R, 4H)), da_t -> slice t of da_out, gates / c / mask at base + t step.
static void lstm16_bptt_run(LaunchCtx& cx, int64_t R, int H, int t_hi, const __half* da_in, __half* da_out, const __half* Whb16,
                            const __half* gates16, int64_t g_step, const float* c, int64_t c_step, const float* c0,
                            const int32_t* mask, int64_t m_step, float* dc_carry) {
  using namespace tc;
  const Bptt16Plan pl = lstm16_bptt_plan(cx, R, H);
  const int64_t G = 4 * (int64_t)H;
  auto map3 = [&](const __half* base, int box_rows, int box_cols, CUtensorMapSwizzle swz) {
    CUtensorMap tm;
    cuuint64_t dims[3] = {(cuuint64_t)G, (cuuint64_t)R, (cuuint64_t)(t_hi + 1)};
    cuuint64_t strides[2] = {(cuuint64_t)G * 2, (cuuint64_t)(R * G * 2)};
    cuuint32_t box[3] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = get_encode()(&tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, (void*)base, dims, strides, box, estr,
                              CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) throw CudaError(-3, "cuTensorMapEncodeTiled (lstm16 bptt) failed (" + std::to_string((int)r) + ")");
    return tm;
  };
  const CUtensorMap tA = map3(da_in, BM16, BK16, CU_TENSOR_MAP_SWIZZLE_128B);
  const CUtensorMap tB = tmap_h(Whb16, H, G, G, 128, BK16, CU_TENSOR_MAP_SWIZZLE_128B);
  const CUtensorMap tD = map3(da_out, 16, 32, CU_TENSOR_MAP_SWIZZLE_64B);
  Bptt16Params p = {};
  p.R = (int)R; p.H = H; p.t_hi = t_hi;
  p.gates = gates16; p.g_step = g_step; p.c = c; p.c_step = c_step; p.c0 = c0; p.mask = mask; p.m_step = m_step;
  p.dc_carry = dc_carry;
  const int num_m = cdiv(R, BM16);
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = pl.csize; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  for (int mb0 = 0; mb0 < num_m; mb0 += pl.clusters) {
    p.mb0 = mb0;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(pl.csize * std::min(pl.clusters, num_m - mb0)); cfg.blockDim = dim3(Bptt16::THREADS);
    cfg.dynamicSmemBytes = Bptt16::TOTAL; cfg.stream = cx.stream; cfg.attrs = attr; cfg.numAttrs = 1;
    VD_CUDA_CHECK(cudaLaunchKernelEx(&cfg, k_lstm16_bptt, tA, tB, tD, p));
    check_launch(cx, "k_lstm16_bptt");
  }
}

void lstm16_step_bwd(LaunchCtx& cx, int64_t R, int H, const __half* da_next16, const __half* Whb16, const __half* gates16,
                     const float* c_prev, const float* c_cur, float* dc_carry, const int32_t* mask_ids, __half* da16) {
  VD_REQUIRE(lstm16_shape_ok(R, H), VD_E_STATE, "lstm16_step_bwd: shape");
  lstm16_bptt_run(cx, R, H, 0, da_next16, da16, Whb16, gates16, 0, c_cur, 0, c_prev, mask_ids, 0, dc_carry);
}

void lstm16_bptt(LaunchCtx& cx, int64_t R, int H, int T, __half* da16, const __half* Whb16, const __half* gates16, const float* c,
                 const float* c0, const int32_t* mask, float* dc_carry) {
  VD_REQUIRE(lstm16_shape_ok(R, H) && T >= 2, VD_E_STATE, "lstm16_bptt: shape");
  const int64_t RG = R * 4 * H;
  lstm16_bptt_run(cx, R, H, T - 2, da16 + RG, da16, Whb16, gates16, RG, c, R * H, c0, mask, R, dc_carry);
}

void lstm16_first_step(LaunchCtx& cx, int64_t R, int H, const __half* ptable16, const int32_t* tok, const float* bias,
                       const float* c_prev, const int32_t* mask_ids, __half* gates16, float* c_out, __half* h16_out, float* h32_out) {
  const int64_t n = R * (H / 8);
  tc::k_lstm16_first<<<(unsigned)((n + 255) / 256), 256, 0, cx.stream>>>(ptable16, tok, bias, c_prev, mask_ids, gates16, c_out,
                                                                          h16_out, h32_out, R, H);
  check_launch(cx, "k_lstm16_first");
}

void lstm16_bwd_last(LaunchCtx& cx, int64_t R, int H, const __half* gates16, const float* c_prev, const float* c_cur,
                     const float* dh_last, const float* scale, const int32_t* mask_ids, float* dc_carry, __half* da16) {
  const int64_t n = R * (H / 8);
  tc::k_lstm16_bwd_last<<<(unsigned)((n + 255) / 256), 256, 0, cx.stream>>>(gates16, c_prev, c_cur, dh_last, scale, mask_ids,
                                                                             dc_carry, da16, R, H);
  check_launch(cx, "k_lstm16_bwd_last");
}

void cvt_f32_to_f16(LaunchCtx& cx, __half* dst, int64_t ldd, const float* src, int64_t lds, int64_t rows, int cols) {
  VD_REQUIRE(cols % 4 == 0 && lds % 4 == 0 && ldd % 4 == 0, VD_E_STATE, "cvt_f32_to_f16: alignment");
  const int64_t n = rows * (cols / 4);
  if (n == 0) return;
  tc::k_cvt16<<<(unsigned)((n + 255) / 256), 256, 0, cx.stream>>>(dst, ldd, src, lds, rows, cols);
  check_launch(cx, "k_cvt16");
}

// scale2[0] = power-of-two scale for max|x| -> [2^9, 2^10), scale2[1] = its inverse; bits = 1 scratch word
void pick_grad_scale(LaunchCtx& cx, const float* x, int64_t n, uint32_t* bits, float* scale2) {
  VD_REQUIRE(n % 4 == 0, VD_E_STATE, "pick_grad_scale: n % 4");
  VD_CUDA_CHECK(cudaMemsetAsync(bits, 0, sizeof(uint32_t), cx.stream));
  const int blocks = (int)std::min<int64_t>((n / 4 + 255) / 256, 4 * cx.sm_count);
  tc::k_amax<<<blocks, 256, 0, cx.stream>>>(x, n / 4, bits);
  check_launch(cx, "k_amax");
  tc::k_pick_scale<<<1, 1, 0, cx.stream>>>(bits, scale2);
  check_launch(cx, "k_pick_scale");
}

void segsum_rows16(LaunchCtx& cx, const __half* X, int64_t ldx, const int32_t* perm, const int32_t* sorted_tok, int64_t n,
                   float* out, int ncols, const float* inv_scale) {
  VD_REQUIRE(ncols % 8 == 0 && ldx % 8 == 0, VD_E_STATE, "segsum_rows16: alignment");
  if (n == 0) return;
  if (cx.deterministic) { segsum_rows16_det(cx, X, ldx, perm, sorted_tok, n, out, ncols, inv_scale); return; }
  tc::k_segsum16<<<(unsigned)((n + tc::SEG16_ROWS - 1) / tc::SEG16_ROWS), 256, 0, cx.stream>>>(X, ldx, perm, sorted_tok, n, out, ncols,
                                                                                               inv_scale);
  check_launch(cx, "k_segsum16");
}

// one zeroed claim / done counter pair per (device, stream): launches on one stream are ordered, and each leaves it zeroed
static int* atb16_counter(cudaStream_t stream) {
  static std::mutex mu;
  static std::map<std::pair<int, cudaStream_t>, int*> counters;
  int dev = 0;
  VD_CUDA_CHECK(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lock(mu);
  int*& c = counters[{dev, stream}];
  if (!c) {
    VD_CUDA_CHECK(cudaMalloc((void**)&c, 2 * sizeof(int)));
    VD_CUDA_CHECK(cudaMemsetAsync(c, 0, 2 * sizeof(int), stream));
  }
  return c;
}

// C[M,N] += inv_scale * A^T B, A (K x M) and B (K x N) fp16 row-major; stream-K over at most cx.sms() CTAs
void gemm_atb16(LaunchCtx& cx, int M, int N, int64_t K, const __half* A, int64_t lda, const __half* B, int64_t ldb, float* C,
                int64_t ldc, const float* inv_scale) {
  using namespace tc;
  VD_REQUIRE(M % 64 == 0 && N % 64 == 0 && K >= A16_KB && lda % 8 == 0 && ldb % 8 == 0, VD_E_STATE, "gemm_atb16: shape");
  Atb16Params p = {};
  p.M = M; p.N = N; p.tiles_n = cdiv(N, A16_BN); p.tiles = cdiv(M, A16_BM) * p.tiles_n;
  VD_REQUIRE((K + A16_KB - 1) / A16_KB <= INT32_MAX, VD_E_STATE, "gemm_atb16: K");
  p.kbt = (int)((K + A16_KB - 1) / A16_KB);
  const int64_t sms = cx.sms(), total = (int64_t)p.tiles * p.kbt;
  if (cx.deterministic) {
    const int ranges = std::max(1, std::min(A16_DET_RANGES, cdiv(p.kbt, A16_MIN_CHUNK)));
    p.chunk = cdiv(p.kbt, ranges);
    p.ws = cx.scratch_get<float>((int64_t)cdiv(p.kbt, p.chunk) * M * N);
  } else {
    p.chunk = (int)std::min<int64_t>(p.kbt, std::max<int64_t>(A16_MIN_CHUNK, cdiv(total, sms * A16_CHUNKS_PER_CTA)));
  }
  p.num_chunks = p.tiles * cdiv(p.kbt, p.chunk);
  p.C = C; p.ldc = ldc; p.inv_scale = inv_scale;
  p.counter = atb16_counter(cx.stream);
  CUtensorMap tA = tmap_h(A, K, M, lda, A16_KB, 64, CU_TENSOR_MAP_SWIZZLE_128B),
              tB = tmap_h(B, K, N, ldb, A16_KB, 64, CU_TENSOR_MAP_SWIZZLE_128B);
  static bool attr_set = false;
  if (!attr_set) {
    VD_CUDA_CHECK(cudaFuncSetAttribute(k_atb16<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, A16_TOTAL));
    VD_CUDA_CHECK(cudaFuncSetAttribute(k_atb16<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, A16_TOTAL));
    VD_CUDA_CHECK(cudaFuncSetAttribute(k_atb16<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, A16_TOTAL));
    attr_set = true;
  }
  const unsigned grid = (unsigned)std::min<int64_t>(sms, p.num_chunks);
  if (cx.deterministic) {
    k_atb16<true, true><<<grid, A16_THREADS, A16_TOTAL, cx.stream>>>(tA, tB, p);
    check_launch(cx, "k_atb16");
    slot_reduce(cx, C, ldc, p.ws, cdiv(p.kbt, p.chunk), M, N);
    return;
  }
  if (ldc % 4 == 0 && ((uintptr_t)C & 15) == 0) k_atb16<true, false><<<grid, A16_THREADS, A16_TOTAL, cx.stream>>>(tA, tB, p);
  else k_atb16<false, false><<<grid, A16_THREADS, A16_TOTAL, cx.stream>>>(tA, tB, p);
  check_launch(cx, "k_atb16");
}

}  // namespace vd
