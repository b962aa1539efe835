// fp32 CUDA-core GEMMs: the VD_MATH_FP32 verification path, and the fallback for contraction
// shapes the wgmma kernels do not take (tiny M / N).  Same contract as the tensor-core kernels
// in gemm_tc.cu.
//
//   gemm_tn : C[m,n] = act(beta*C[m,n] + bias[n] + sum_k A[row(m),k] * B[n,k])
//             A (M x K) row-major with optional row gather, B (N x K) row-major ("K-major" both).
//   gemm_atb: C[m,n] += sum_k A[row(k),m] * B[k,n]      (weight gradients; split-K + atomics)
#include "kernels.cuh"

namespace vd {

namespace {
constexpr int BM = 128, BN = 128, BK = 16, TM = 8, TN = 8, NT = 256;

__device__ __forceinline__ float act_apply(float v, int act) { return act == 1 ? tanhf(v) : v; }

__global__ void __launch_bounds__(NT) k_gemm_tn(int M, int N, int K, const float* __restrict__ A, int64_t lda,
                                                const int32_t* __restrict__ a_gather,
                                                const float* __restrict__ B, int64_t ldb,
                                                float* __restrict__ C, int64_t ldc, float beta,
                                                const float* __restrict__ bias, int act, int vec) {
  __shared__ float As[BK][BM + 4];
  __shared__ float Bs[BK][BN + 4];
  const int tid = threadIdx.x;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const int lrow = tid >> 2, lk = (tid & 3) * 4;      // 64 rows x 4 float4 per pass, 2 passes
  const float* arow[2];
  const float* brow[2];
#pragma unroll
  for (int p = 0; p < 2; ++p) {
    int m = m0 + lrow + p * 64;
    if (m < M) {
      int64_t r = a_gather ? (int64_t)a_gather[m] : (int64_t)m;
      arow[p] = A + r * lda;
    } else arow[p] = nullptr;
    int n = n0 + lrow + p * 64;
    brow[p] = n < N ? B + (int64_t)n * ldb : nullptr;
  }
  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;
  const int ty = tid >> 4, tx = tid & 15;
  for (int k0 = 0; k0 < K; k0 += BK) {
#pragma unroll
    for (int p = 0; p < 2; ++p) {
      float4 va = make_float4(0, 0, 0, 0), vb = make_float4(0, 0, 0, 0);
      int k = k0 + lk;
      if (vec) {
        if (arow[p] && k < K) va = *reinterpret_cast<const float4*>(arow[p] + k);
        if (brow[p] && k < K) vb = *reinterpret_cast<const float4*>(brow[p] + k);
      } else {
        if (arow[p]) { const float* q = arow[p] + k; if (k < K) va.x = q[0]; if (k + 1 < K) va.y = q[1]; if (k + 2 < K) va.z = q[2]; if (k + 3 < K) va.w = q[3]; }
        if (brow[p]) { const float* q = brow[p] + k; if (k < K) vb.x = q[0]; if (k + 1 < K) vb.y = q[1]; if (k + 2 < K) vb.z = q[2]; if (k + 3 < K) vb.w = q[3]; }
      }
      int r = lrow + p * 64;
      As[lk + 0][r] = va.x; As[lk + 1][r] = va.y; As[lk + 2][r] = va.z; As[lk + 3][r] = va.w;
      Bs[lk + 0][r] = vb.x; Bs[lk + 1][r] = vb.y; Bs[lk + 2][r] = vb.z; Bs[lk + 3][r] = vb.w;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float a[TM], b[TN];
      *reinterpret_cast<float4*>(a) = *reinterpret_cast<const float4*>(&As[k][ty * TM]);
      *reinterpret_cast<float4*>(a + 4) = *reinterpret_cast<const float4*>(&As[k][ty * TM + 4]);
      *reinterpret_cast<float4*>(b) = *reinterpret_cast<const float4*>(&Bs[k][tx * TN]);
      *reinterpret_cast<float4*>(b + 4) = *reinterpret_cast<const float4*>(&Bs[k][tx * TN + 4]);
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    int m = m0 + ty * TM + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      int n = n0 + tx * TN + j;
      if (n >= N) continue;
      float v = acc[i][j];
      if (bias) v += bias[n];
      float* c = C + (int64_t)m * ldc + n;
      if (beta != 0.f) v += beta * (*c);
      *c = act_apply(v, act);
    }
  }
}

// C[m,n] += sum_k A[row(k), m] * B[k, n];  grid.z splits K.
__global__ void __launch_bounds__(NT) k_gemm_atb(int M, int N, int64_t K, int64_t k_per_split,
                                                 const float* __restrict__ A, int64_t lda,
                                                 const int32_t* __restrict__ a_gather,
                                                 const float* __restrict__ B, int64_t ldb,
                                                 float* __restrict__ C, int64_t ldc, int vec) {
  __shared__ float As[BK][BM + 4];
  __shared__ float Bs[BK][BN + 4];
  const int tid = threadIdx.x;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int64_t kbeg = (int64_t)blockIdx.z * k_per_split;
  const int64_t kend = min(K, kbeg + k_per_split);
  const int lk = tid >> 5, lc = (tid & 31) * 4;       // 8 k-rows x 32 float4 per pass, 2 passes
  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;
  const int ty = tid >> 4, tx = tid & 15;
  for (int64_t k0 = kbeg; k0 < kend; k0 += BK) {
#pragma unroll
    for (int p = 0; p < 2; ++p) {
      int64_t k = k0 + lk + p * 8;
      float4 va = make_float4(0, 0, 0, 0), vb = make_float4(0, 0, 0, 0);
      if (k < kend) {
        int64_t r = a_gather ? (int64_t)a_gather[k] : k;
        int m = m0 + lc, n = n0 + lc;
        if (vec) {
          if (m < M) va = *reinterpret_cast<const float4*>(A + r * lda + m);
          if (n < N) vb = *reinterpret_cast<const float4*>(B + k * ldb + n);
        } else {
          const float* ap = A + r * lda + m; const float* bp = B + k * ldb + n;
          if (m + 0 < M) va.x = ap[0]; if (m + 1 < M) va.y = ap[1]; if (m + 2 < M) va.z = ap[2]; if (m + 3 < M) va.w = ap[3];
          if (n + 0 < N) vb.x = bp[0]; if (n + 1 < N) vb.y = bp[1]; if (n + 2 < N) vb.z = bp[2]; if (n + 3 < N) vb.w = bp[3];
        }
      }
      *reinterpret_cast<float4*>(&As[lk + p * 8][lc]) = va;
      *reinterpret_cast<float4*>(&Bs[lk + p * 8][lc]) = vb;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float a[TM], b[TN];
      *reinterpret_cast<float4*>(a) = *reinterpret_cast<const float4*>(&As[k][ty * TM]);
      *reinterpret_cast<float4*>(a + 4) = *reinterpret_cast<const float4*>(&As[k][ty * TM + 4]);
      *reinterpret_cast<float4*>(b) = *reinterpret_cast<const float4*>(&Bs[k][tx * TN]);
      *reinterpret_cast<float4*>(b + 4) = *reinterpret_cast<const float4*>(&Bs[k][tx * TN + 4]);
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    int m = m0 + ty * TM + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      int n = n0 + tx * TN + j;
      if (n >= N) continue;
      atomicAdd(C + (int64_t)m * ldc + n, acc[i][j]);
    }
  }
}
}  // namespace

void gemm_tn_simt(LaunchCtx& cx, int M, int N, int K, const float* A, int64_t lda, const int32_t* a_gather,
                  const float* B, int64_t ldb, float* C, int64_t ldc, float beta, const float* bias, int act) {
  if (M <= 0 || N <= 0) return;
  int vec = (K % 4 == 0 && lda % 4 == 0 && ldb % 4 == 0 && ((uintptr_t)A % 16 == 0) && ((uintptr_t)B % 16 == 0)) ? 1 : 0;
  dim3 grid(cdiv(M, BM), cdiv(N, BN));
  k_gemm_tn<<<grid, NT, 0, cx.stream>>>(M, N, K, A, lda, a_gather, B, ldb, C, ldc, beta, bias, act, vec);
  check_launch(cx, "gemm_tn_simt");
}

void gemm_atb_simt(LaunchCtx& cx, int M, int N, int64_t K, const float* A, int64_t lda, const int32_t* a_gather,
                   const float* B, int64_t ldb, float* C, int64_t ldc) {
  if (M <= 0 || N <= 0 || K <= 0) return;
  int vec = (M % 4 == 0 && N % 4 == 0 && lda % 4 == 0 && ldb % 4 == 0 &&
             ((uintptr_t)A % 16 == 0) && ((uintptr_t)B % 16 == 0)) ? 1 : 0;
  int tiles = cdiv(N, BN) * cdiv(M, BM);
  int splits = (int)std::max<int64_t>(1, std::min<int64_t>((4LL * cx.sm_count + tiles - 1) / tiles, (K + 511) / 512));
  int64_t kps = ((K + splits - 1) / splits + BK - 1) / BK * BK;
  splits = (int)((K + kps - 1) / kps);
  dim3 grid(cdiv(N, BN), cdiv(M, BM), splits);
  k_gemm_atb<<<grid, NT, 0, cx.stream>>>(M, N, K, kps, A, lda, a_gather, B, ldb, C, ldc, vec);
  check_launch(cx, "gemm_atb_simt");
}

}  // namespace vd
