"""The engine's dense contractions (Engine::gemm_tn / gemm_atb) on paper: which kernel takes a call, how the weight-gradient
kernels split K, the per-element error bound of a result, and a numpy emulation of each kernel's arithmetic.

    gemm_tn : C[m, n] = act(beta C[m, n] + bias[n] + sum_k A[row(m), k] B[n, k])      k_tc_gemm (MODE_GENERIC) | k_gemm_tn
    gemm_atb: C[m, n] += sum_k A[row(k), m] B[k, n]                                      k_tc_atb | k_gemm_atb

Bound (U = 2^-24, first order).  The result of a chain of n fp32 additions is within n U sum|terms| of the exact sum.  The
epilogue adds bias, then beta C (one product and one sum), hence

    pre = (n + 3) U (sum_k |a_k b_k| + |bias| + |beta C0|)                 n = K (gemm_tn), kps + splits (gemm_atb)

On the tensor cores the operands are TF32 (10 explicit mantissa bits, the low 13 of fp32 dropped): products of TF32-exact
operands are exact in fp32, so `pre` holds as it stands; fp32 operands add 2^-9 sum_k |a_k b_k| (each factor off by < 2^-10).
The CUDA-core kernels use one fmaf per k.  With act = 1 the bound goes through tanh' = 1 - tanh^2 and picks up the tanh's own
error: 2 ulp of tanhf on the CUDA cores (4 U relative), and 3e-7 absolute plus 4 U relative for the tensor-core epilogue's
exp-based ftanh."""
import numpy as np

U = 2.0 ** -24
TF32_PROD = 2.0 ** -9        # relative error of a product of two fp32 operands truncated (or rounded) to TF32
FTANH_ABS = 3e-7             # ftanh (tc_ptx.cuh): __expf near 1 - e, as TANH_E_ABS of test_kernels_gpu.py
TANH_REL = 4 * U             # 2 ulp of tanhf / __fdividef

TC_BK = 32                   # k_tc_gemm / k_tc_atb k-block
SIMT_BK = 16                 # k_gemm_tn / k_gemm_atb k-block
ATB_BM, ATB_BN = 128, 128    # both weight-gradient kernels' output tiles

# A value that TF32 cannot hold under any rounding (1 + 2^-11 is a tie between 1 and 1 + 2^-10): a row and a column of
# it make one output element whose TF32 error, about 2^-10 of its value, exceeds the fp32-only bound while K < 2^14.
WITNESS = np.float32(1 + 2.0 ** -11)


def tf32(x):
    """fp32 -> TF32 by truncation (the low 13 mantissa bits cleared), as numpy float32"""
    x = np.ascontiguousarray(x, np.float32)
    return (x.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def bf16(x):
    x = np.ascontiguousarray(x, np.float32)
    return (x.view(np.uint32) & np.uint32(0xFFFF0000)).view(np.float32)


# ---------------------------------------------------------------------------------------------- routes
def tn_takes_tc(tcmode, M, N, K, gather, aligned_a, aligned_b, aligned_c):
    """gemm_tn_tc's acceptance predicate (gemm_tc.cu), behind Engine::gemm_tn's tcmode()"""
    return bool(tcmode and not gather and M >= 64 and N >= 16 and K >= 32 and N % 4 == 0 and aligned_a and aligned_b
                and aligned_c)


def atb_takes_tc(tcmode, M, N, K, gather, aligned_a, aligned_b):
    """gemm_atb_tc's acceptance predicate"""
    return bool(tcmode and not gather and M >= 32 and N >= 32 and K >= 64 and aligned_a and aligned_b)


def aligned(off, ld):
    """a float operand at element offset `off` of a 256-byte aligned allocation, row pitch ld: 16-byte rows"""
    return off % 4 == 0 and ld % 4 == 0


def _cdiv(a, b):
    return -(-a // b)


def atb_tc_splits(M, N, K, sms, budget=0):
    """(splits, k per split) of gemm_atb_tc: whole waves of at most 2 #SM CTAs, or one wave of `budget` CTAs"""
    tiles = _cdiv(M, ATB_BM) * _cdiv(N, ATB_BN)
    cap = budget if budget > 0 else 2 * sms
    splits = max(1, min(cap // tiles, K // (TC_BK * 4)))
    kps = _cdiv(_cdiv(K, splits), TC_BK) * TC_BK
    return _cdiv(K, kps), kps


def atb_simt_splits(M, N, K, sms):
    """(splits, k per split) of gemm_atb_simt: about 4 #SM CTAs, at least 512 k-rows each"""
    tiles = _cdiv(N, ATB_BN) * _cdiv(M, ATB_BM)
    splits = max(1, min(_cdiv(4 * sms, tiles), _cdiv(K, 512)))
    kps = _cdiv(_cdiv(K, splits), SIMT_BK) * SIMT_BK
    return _cdiv(K, kps), kps


# ---------------------------------------------------------------------------------------------- bound
def chain(op, K, tc, M=0, N=0, sms=132, budget=0):
    """the addition chain n of the bound: K for gemm_tn, the longest split plus the split count for gemm_atb"""
    if op == "tn":
        return K
    splits, kps = atb_tc_splits(M, N, K, sms, budget) if tc else atb_simt_splits(M, N, K, sms)
    return min(kps, K) + splits


def bound(n, sabs, extra, tc, tf32_exact, act=0, ref=None):
    """per-element bound.  sabs = sum_k |a_k b_k|, extra = |bias| + |beta C0| (gemm_atb: |C0|), ref = the fp64 result
    (after the activation); all broadcast, numpy arrays or torch tensors"""
    pre = (n + 3) * U * (sabs + extra)
    if tc and not tf32_exact:
        pre = pre + TF32_PROD * sabs
    if not act:
        return pre
    t = abs(ref)
    return (1 - t * t) * pre + TANH_REL * t + (FTANH_ABS if tc else 0.0)


# ---------------------------------------------------------------------------------------------- emulation
def _acc(prods, kb, bf16_blocks=False, drop_last_partial=False):
    """fp32 sequential accumulation of the products (K, ...) in k-blocks of kb"""
    K = prods.shape[0]
    acc = np.zeros(prods.shape[1:], np.float32)
    for k0 in range(0, K, kb):
        blk = prods[k0:k0 + kb]
        if drop_last_partial and k0 + kb > K:
            break
        acc = np.cumsum(np.concatenate([acc[None], blk]), axis=0, dtype=np.float32)[-1]
        if bf16_blocks:
            acc = bf16(acc)
    return acc


def emulate_tn(A, B, C0=None, beta=0.0, bias=None, act=0, tc=True, mutant=None):
    """gemm_tn on fp32 numpy: A (M, K), B (N, K) -> C (M, N)"""
    f = np.float32
    if tc or mutant == "tf32_on_fp32_route":
        A, B = tf32(A), tf32(B)
    prods = (A.T[:, :, None] * B.T[:, None, :]).astype(f)           # (K, M, N), exact for TF32 operands
    acc = _acc(prods, TC_BK if tc else SIMT_BK, mutant == "bf16_blocks", mutant == "drop_last_kblock")
    x = acc
    if bias is not None:
        x = (x + (tf32(bias) if mutant == "bias_tf32" else bias.astype(f))[None, :]).astype(f)
    if beta != 0:
        bc = (f(beta) * C0).astype(f)
        x = (x + (tf32(bc) if mutant == "betac_tf32" else bc)).astype(f)
    if act:
        x = np.tanh(x.astype(np.float64)).astype(f)
    return x


def emulate_atb(A, B, C0, tc=True, sms=132, budget=0, mutant=None, MN=None):
    """gemm_atb on fp32 numpy: A (K, M), B (K, N), C0 (M, N) -> C0 + A^T B, split-K partials added to C in split order.
    MN: the call's (M, N) when A and B hold only some of its columns (the split count follows the call's shape)"""
    f = np.float32
    K = A.shape[0]
    M, N = MN or (A.shape[1], B.shape[1])
    if tc or mutant == "tf32_on_fp32_route":
        A, B = tf32(A), tf32(B)
    splits, kps = atb_tc_splits(M, N, K, sms, budget) if tc else atb_simt_splits(M, N, K, sms)
    C = C0.astype(f).copy()
    for s in range(splits):
        if mutant == "split_lost" and s == splits - 1:
            continue
        a, b = A[s * kps:(s + 1) * kps], B[s * kps:(s + 1) * kps]
        prods = (a[:, :, None] * b[:, None, :]).astype(f)
        part = _acc(prods, TC_BK if tc else SIMT_BK, mutant == "bf16_blocks", mutant == "drop_last_kblock")
        C = (C + part).astype(f)
        if mutant == "split_twice" and s == 0:
            C = (C + part).astype(f)
    return C
