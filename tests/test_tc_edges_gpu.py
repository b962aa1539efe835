"""Tensor-core kernels at ragged, strided and odd shapes, against fp64 numpy.

GEMM primitives (vd_gemm_tn / vd_gemm_atb / vd_gemm_atb16): shapes on both sides of every routing predicate and tile
edge, strided and offset operands, NaN guard bands around C (padding columns and rows past M must come back untouched,
and with beta = 0 the NaN inside C must never be read).  The route is asserted, not only the result: a Python mirror of
the acceptance predicate says "tensor cores" or "CUDA cores", and the error class must agree.  The natural error scale of
an output element is s = sqrt(sum_k (a_k b_k)^2) (times tanh' after act = 1); TF32 operands (10-bit mantissa) leave a
normalised rms error rms(err) / rms(s) of about 3e-4, an fp32 contraction about 1e-7, so 1e-5 separates the classes.  The
bounds of test_tensorcore_gpu.py hold on top: rms <= 1.5e-3 sqrt(K), max <= 8e-3 sqrt(K) for unit-variance operands.

SeqLSTM step hooks (vd_lstm_step_fwd / _bwd): per element against the numpy step of tests/helpers.py, which
test_oracle_units.py pins to the oracle.  Inputs are O(1) (x-projection and bias ~ N(0, 0.5^2), h in (-1, 1), weights
~ N(0, 1/H)), so a pre-activation carries a TF32 error of about 1e-3 sqrt(H) * |w| |h| ~ 5e-4 and every output an error
below 1e-3 rms, 8e-3 max (1.5e-5 / 1e-4 on CUDA cores).  Swapping two gate blocks, dropping the bias or reading the
wrong c_prev row changes outputs by O(0.1).

Whole graphs at odd sizes (embedSize 36, vocabSize 301, H = 192) in TF32 and F16 against the oracle and the engine's
own FP32 mode, with the kernel classes that ran read from the launch profile."""
import ctypes as C

import numpy as np
import pytest
import torch

from helpers import (Buf, _image, _view, lstm_step_bwd_ref, lstm_step_fwd_ref, seg_slices, small_params, torch_batch,
                     torch_params)
from oracle import philox
from oracle import visdial_oracle as O
from visdial_b200 import VD_MATH_F16, VD_MATH_FP32, VD_MATH_TF32, Batch, Engine, init_parameters
from visdial_b200._lib import check
from visdial_b200.synthetic import make_batch

pytestmark = pytest.mark.gpu


def _aligned(off, ld):
    return off % 4 == 0 and ld % 4 == 0        # cudaMalloc bases are 256-byte aligned: 16 bytes <=> off % 4 == 0


def _r4(x):
    return (x + 3) // 4 * 4


@pytest.fixture(scope="module")
def eng():
    e = Engine(small_params("lf-ques", "disc"))
    e.set_math_mode(VD_MATH_TF32)
    yield e
    e.close()


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _check_class(err, scale, K, tc, what):
    rms = float(np.sqrt(np.mean(err ** 2)))
    norm = rms / max(float(np.sqrt(np.mean(scale ** 2))), 1e-30)
    assert rms <= 1.5e-3 * np.sqrt(K) and float(np.abs(err).max()) <= 8e-3 * np.sqrt(K), (what, rms, float(np.abs(err).max()))
    if tc:
        assert norm > 1e-5, ("expected the TF32 tensor-core route", what, norm)
        assert norm < 3e-3, (what, norm)
    else:
        assert norm < 1e-5, ("expected the fp32 CUDA-core route", what, norm)


# ---------------------------------------------------------------------------------------------- C = act(beta C + bias + A B^T)
def _run_tn(eng, M, N, K, beta=0.0, bias=False, act=0, offA=0, lda=None, offB=0, ldb=None, offC=0, ldc=None, seed=0):
    lda = lda or _r4(K)
    ldb = ldb or _r4(K)
    ldc = ldc or _r4(N) + 4
    rng = np.random.default_rng(seed + 1000 * M + 10 * N + K)
    sa = 1.0 / np.sqrt(K) if act else 1.0             # keep tanh off its saturated flanks
    A = (rng.standard_normal((M, K)) * sa).astype(np.float32)
    B = rng.standard_normal((N, K)).astype(np.float32)
    C0 = rng.standard_normal((M, N)).astype(np.float32)
    bv = rng.standard_normal(N).astype(np.float32) if bias else None
    imgC = _image(C0 if beta != 0 else np.full((M, N), np.nan, np.float32), offC, ldc, rows_extra=3)
    bufs = [Buf(eng, _image(A, offA, lda)), Buf(eng, _image(B, offB, ldb)), Buf(eng, imgC)]
    if bias:
        bufs.append(Buf(eng, bv))
    dA, dB, dC = bufs[:3]
    check(eng.lib.vd_gemm_tn(eng.h, M, N, K, dA.ptr(offA), lda, dB.ptr(offB), ldb, dC.ptr(offC), ldc, beta,
                             bufs[3].ptr() if bias else None, act))
    out = dC.get()
    for b in bufs:
        b.free()
    A64, B64 = A.astype(np.float64), B.astype(np.float64)
    pre = A64 @ B64.T + (bv[None, :] if bias else 0) + (beta * C0.astype(np.float64) if beta != 0 else 0)
    ref = np.tanh(pre) if act else pre
    scale = np.sqrt((A64 ** 2) @ (B64 ** 2).T)
    if act:
        scale = scale * (1 - ref ** 2)
    got = _view(out, offC, M, N, ldc)
    assert np.isfinite(got).all(), "C produced non-finite values (NaN read from the guard band or, with beta = 0, from C)"
    guard = out.copy()
    _view(guard, offC, M, N, ldc)[:] = np.nan
    assert np.isnan(guard).all(), "vd_gemm_tn wrote outside C[0:M, 0:N]"
    tc = M >= 64 and N >= 16 and N % 4 == 0 and K >= 32 and _aligned(offA, lda) and _aligned(offB, ldb) and _aligned(offC, ldc)
    return got - ref, scale, tc


TN_M = [63, 64, 65, 127, 128, 129, 257]
TN_N = [15, 16, 17, 20, 33, 36, 64, 65, 68, 127, 128, 129, 132]     # N % 4 != 0 stays on CUDA cores (see gemm_tn_tc)
TN_K = [31, 32, 33, 36, 63, 300]


@pytest.mark.parametrize("M", TN_M)
def test_gemm_tn_tile_edges(eng, M):
    """every N of the sweep for this M (both BN = 64 and BN = 128 tiles, ragged last tiles), K cycling through the
    k-block edges; the epilogue cycles through beta in {0, 1, 0.5}, bias on / off and act = tanh"""
    for j, N in enumerate(TN_N):
        i = TN_M.index(M) * len(TN_N) + j
        K = TN_K[i % len(TN_K)]
        beta, bias, act = (0.0, 1.0, 0.5)[i % 3], (i // 3) % 2 == 1, int(i % 5 == 0)
        err, scale, tc = _run_tn(eng, M, N, K, beta=beta, bias=bias, act=act, seed=i)
        _check_class(err, scale, K, tc, (M, N, K, beta, bias, act))


@pytest.mark.parametrize("N", [17, 20, 68, 132])
def test_gemm_tn_k_edges(eng, N):
    for K in TN_K:
        err, scale, tc = _run_tn(eng, 129, N, K, beta=0.5, bias=True, seed=K)
        _check_class(err, scale, K, tc, (129, N, K))


# (offA, lda+, offB, ldb+, offC, ldc+): pitches are round_up(K or N, 4) + the extra
TN_STRIDES = [(4, 8, 4, 4, 4, 12), (0, 4, 0, 8, 0, 4), (1, 0, 0, 0, 0, 0), (0, 0, 5, 4, 0, 0), (0, 0, 0, 0, 1, 4),
              (0, 1, 0, 0, 0, 0), (0, 0, 0, 3, 0, 0), (0, 0, 0, 0, 0, 1)]


@pytest.mark.parametrize("M,N,K", [(129, 68, 33), (64, 20, 63), (257, 132, 300), (65, 17, 32)])
@pytest.mark.parametrize("strides", TN_STRIDES)
def test_gemm_tn_strided_views(eng, M, N, K, strides):
    """offset / strided operands: 16-byte aligned ones stay on the tensor cores, misaligned ones (offset 1 float or
    ld % 4 != 0) go to the CUDA cores; either way C's padding columns and the rows past M stay untouched"""
    oA, eA, oB, eB, oC, eC = strides
    err, scale, tc = _run_tn(eng, M, N, K, beta=1.0, bias=True, offA=oA, lda=_r4(K) + eA, offB=oB, ldb=_r4(K) + eB,
                             offC=oC, ldc=_r4(N) + eC, seed=sum(strides))
    _check_class(err, scale, K, tc, (M, N, K, strides))


def test_gemm_tn_fp32_mode_never_takes_the_tensor_cores(eng):
    eng.set_math_mode(VD_MATH_FP32)
    try:
        for M, N, K in ((128, 128, 64), (257, 65, 300)):
            err, scale, _ = _run_tn(eng, M, N, K, beta=1.0, bias=True)
            _check_class(err, scale, K, False, (M, N, K))
    finally:
        eng.set_math_mode(VD_MATH_TF32)


# ---------------------------------------------------------------------------------------------- C += A^T B  (weight gradients)
def _run_atb(eng, M, N, K, offA=0, lda=None, offB=0, ldb=None, offC=0, ldc=None, seed=0):
    lda = lda or _r4(M)
    ldb = ldb or _r4(N)
    ldc = ldc or _r4(N) + 4
    rng = np.random.default_rng(seed + 7 * M + 3 * N + K)
    A = rng.standard_normal((K, M)).astype(np.float32)
    B = rng.standard_normal((K, N)).astype(np.float32)
    C0 = rng.standard_normal((M, N)).astype(np.float32)
    dA, dB, dC = Buf(eng, _image(A, offA, lda)), Buf(eng, _image(B, offB, ldb)), Buf(eng, _image(C0, offC, ldc, rows_extra=3))
    check(eng.lib.vd_gemm_atb(eng.h, M, N, K, dA.ptr(offA), lda, dB.ptr(offB), ldb, dC.ptr(offC), ldc))
    out = dC.get()
    for b in (dA, dB, dC):
        b.free()
    A64, B64 = A.astype(np.float64), B.astype(np.float64)
    ref = C0 + A64.T @ B64
    got = _view(out, offC, M, N, ldc)
    assert np.isfinite(got).all()
    guard = out.copy()
    _view(guard, offC, M, N, ldc)[:] = np.nan
    assert np.isnan(guard).all(), "vd_gemm_atb wrote outside C[0:M, 0:N]"
    tc = M >= 32 and N >= 32 and K >= 64 and _aligned(offA, lda) and _aligned(offB, ldb)
    return got - ref, np.sqrt((A64 ** 2).T @ (B64 ** 2)), tc


ATB_MN = [31, 32, 33, 127, 128, 129]
ATB_K = [63, 64, 65, 255, 256, 257, 1000]


@pytest.mark.parametrize("M", ATB_MN)
def test_gemm_atb_tile_and_split_edges(eng, M):
    """M, N around the 32 threshold and the 128-wide tile, K around the 64 threshold, the 32-row k-block and the
    K / 128 split-K steps (one 128 x 128 tile: the split count is K // 128 up to two waves)"""
    for j, N in enumerate(ATB_MN):
        K = ATB_K[(ATB_MN.index(M) * len(ATB_MN) + j) % len(ATB_K)]
        err, scale, tc = _run_atb(eng, M, N, K)
        _check_class(err, scale, K, tc, (M, N, K))
    for K in ATB_K:
        err, scale, tc = _run_atb(eng, M, 129, K, seed=1)
        _check_class(err, scale, K, tc, (M, 129, K))


@pytest.mark.parametrize("strides", [(4, 4, 4, 8, 1, 3), (1, 0, 0, 0, 0, 0), (0, 0, 0, 1, 0, 0), (0, 2, 0, 0, 4, 8)])
@pytest.mark.parametrize("M,N,K", [(129, 65, 257), (33, 128, 64)])
def test_gemm_atb_strided_views(eng, M, N, K, strides):
    """the tensor-core weight gradient needs aligned A and B only: C may sit anywhere (it is reduced with atomics)"""
    oA, eA, oB, eB, oC, eC = strides
    err, scale, tc = _run_atb(eng, M, N, K, offA=oA, lda=_r4(M) + eA, offB=oB, ldb=_r4(N) + eB, offC=oC, ldc=_r4(N) + eC)
    _check_class(err, scale, K, tc, (M, N, K, strides))


@pytest.mark.parametrize("M,N,K,offA,offB,offC,ldc_extra", [(64, 64, 64, 0, 0, 0, 4), (64, 128, 65, 4, 8, 1, 3),
                                                          (192, 64, 333, 0, 4, 0, 12), (128, 192, 127, 8, 0, 5, 1)])
def test_gemm_atb16_edges(eng, M, N, K, offA, offB, offC, ldc_extra):
    """VD_MATH_F16 weight gradient at the shapes its VD_REQUIRE takes (M, N multiples of 64, K >= 64), ragged K, offset
    fp32 sources with padded pitches, C anywhere with a guard band: exact products of the fp16-rounded operands, so only
    the fp32 accumulation order separates it from fp64"""
    rng = np.random.default_rng(M + N + K)
    lda, ldb, ldc = M + 4, N + 8, N + ldc_extra
    A = rng.standard_normal((K, M)).astype(np.float16).astype(np.float32)
    B = rng.standard_normal((K, N)).astype(np.float16).astype(np.float32)
    C0 = rng.standard_normal((M, N)).astype(np.float32)
    dA, dB, dC = Buf(eng, _image(A, offA, lda, fill=0)), Buf(eng, _image(B, offB, ldb, fill=0)), Buf(eng, _image(C0, offC, ldc, 2))
    check(eng.lib.vd_gemm_atb16(eng.h, M, N, K, dA.ptr(offA), lda, dB.ptr(offB), ldb, dC.ptr(offC), ldc, 0.5))
    out = dC.get()
    for b in (dA, dB, dC):
        b.free()
    ref = C0 + 0.5 * (A.astype(np.float64).T @ B.astype(np.float64))
    got = _view(out, offC, M, N, ldc)
    assert float(np.abs(got - ref).max()) < 2e-6 * K * 0.5 + 1e-5
    guard = out.copy()
    _view(guard, offC, M, N, ldc)[:] = np.nan
    assert np.isnan(guard).all(), "vd_gemm_atb16 wrote outside C[0:M, 0:N]"


# ---------------------------------------------------------------------------------------------- SeqLSTM step hooks
def _fwd_tile(R, H, sms):
    return 128 if -(-R // 128) * (H // 32) >= sms else 64


def _bwd_tile(R, H, sms):
    return 128 if -(-R // 128) * (H // 128) >= sms else 32


def _rows_for(H, per_block, sms, big):
    """R with the given tile choice: the smallest row-block count that fills the SMs (big) or one below it (not big),
    with a partial last block; 1 if not even one full wave is reachable below"""
    need = -(-sms // per_block)                          # row blocks that make the wide tile win
    return 128 * (need - 1) + 77 if big else max(1, 128 * (need - 2) + 77)


def _mask_rows(R, rng):
    m = rng.random(R) < 0.1
    for r in (0, 127, 128, R - 1):                       # first / last row of a tile, first row of the next, the last row
        if r < R:
            m[r] = True
    return m


def _lstm_fwd_case(eng, R, H, sms, gather, with_c, with_h, masked, seed):
    rng = np.random.default_rng(seed)
    G = 4 * H
    Wh = (rng.standard_normal((H, G)) / np.sqrt(H)).astype(np.float32)       # (H, 4H): the h rows of the weight
    WhT = np.ascontiguousarray(Wh.T)                                         # (4H, H) as the transposed shadow holds it
    ldw = H + 4 * (seed % 2)                                                 # padded pitch, like [4H, D+H] with the h columns
    bias = (rng.standard_normal(G) * 0.5).astype(np.float32)
    h_prev = np.tanh(rng.standard_normal((R, H))).astype(np.float32) if with_h else None
    c_prev = rng.standard_normal((R, H)).astype(np.float32) if with_c else None
    mask = _mask_rows(R, rng) if masked else np.zeros(R, bool)
    ids = np.where(mask, 0, 1).astype(np.int32)
    bufs = {"WhT": Buf(eng, _image(WhT, 0, ldw, fill=0)), "bias": Buf(eng, bias), "c": Buf(eng, np.zeros(R * H, np.float32)),
            "h": Buf(eng, np.zeros(R * H, np.float32)), "ids": Buf(eng, ids)}
    if gather:
        V1 = 37
        table = (rng.standard_normal((V1, G)) * 0.5).astype(np.float32)
        tok = rng.integers(0, V1, R).astype(np.int32)
        xz = table[tok]
        bufs["pt"], bufs["tok"] = Buf(eng, table), Buf(eng, tok)
        bufs["g"] = Buf(eng, np.full(R * G, np.nan, np.float32))
    else:
        xz = (rng.standard_normal((R, G)) * 0.5).astype(np.float32)
        bufs["g"] = Buf(eng, xz)
    if with_h:
        bufs["hp"] = Buf(eng, h_prev)
    if with_c:
        bufs["cp"] = Buf(eng, c_prev)
    path = C.c_int32(-1)
    b = lambda k: bufs[k].ptr() if k in bufs else None
    check(eng.lib.vd_lstm_step_fwd(eng.h, R, H, b("hp"), b("WhT"), ldw, b("bias"), b("g"), int(not gather), b("pt"),
                                   37 if gather else 0, b("tok"), b("cp"), b("c"), b("h"), b("ids") if masked else None,
                                   C.byref(path)))
    got = {k: bufs[k].get().reshape(R, -1) for k in ("g", "c", "h")}
    for v in bufs.values():
        v.free()
    ref = lstm_step_fwd_ref(xz.astype(np.float64) + bias, h_prev, Wh, c_prev, mask)
    return got, ref, path.value


@pytest.mark.parametrize("H", [64, 128, 192, 512])
def test_lstm_step_fwd_vs_fp64(eng, sms, H):
    """both tile widths where H allows (the wide one needs cdiv(R,128) * H/32 >= #SM rows), R in {1, 127, 128, 129, a
    partial last block}, table gather and dense x-projection, with and without c_prev, masked rows on tile edges, and the
    first step without h_prev (the streaming kernel the engine uses there)"""
    Rs = [1, 127, 128, 129, _rows_for(H, H // 32, sms, big=False)]
    if H == 512:
        Rs.append(_rows_for(H, H // 32, sms, big=True))
    seen = set()
    for n, R in enumerate(Rs):
        for gather in (True, False):
            with_c = (n + gather) % 2 == 0
            got, ref, path = _lstm_fwd_case(eng, R, H, sms, gather, with_c, True, True, seed=H + 10 * n + gather)
            assert path == _fwd_tile(R, H, sms), (R, H, path)
            seen.add(path)
            for name, g, r in (("gates", got["g"], ref[0]), ("c", got["c"], ref[1]), ("h", got["h"], ref[2])):
                e = np.abs(g - r)
                assert float(e.max()) < 8e-3 and float(np.sqrt(np.mean(e ** 2))) < 1e-3, (name, R, H, gather, float(e.max()))
    assert seen == ({64, 128} if H == 512 else {64})
    # first step without h_prev: no recurrent term, the pointwise kernel
    got, ref, path = _lstm_fwd_case(eng, 129, H, sms, True, False, False, True, seed=H)
    assert path == 0
    for g, r in zip((got["g"], got["c"], got["h"]), ref):
        assert float(np.abs(g - r).max()) < 1e-5


def test_lstm_step_fwd_cuda_core_route(eng):
    """FP32 mode: recurrent GEMM + pointwise kernel (the engine's CUDA-core route), fp32-class error"""
    eng.set_math_mode(VD_MATH_FP32)
    try:
        got, ref, path = _lstm_fwd_case(eng, 129, 64, 132, False, True, True, True, seed=5)
    finally:
        eng.set_math_mode(VD_MATH_TF32)
    assert path == 0
    for g, r in zip((got["g"], got["c"], got["h"]), ref):
        assert float(np.abs(g - r).max()) < 1e-4


def _lstm_bwd_case(eng, R, H, with_next, with_ext, with_c, masked, seed):
    rng = np.random.default_rng(seed)
    G = 4 * H
    Wh = (rng.standard_normal((H, G)) / np.sqrt(G)).astype(np.float32)
    z = rng.standard_normal((R, G))
    gates = np.concatenate([1 / (1 + np.exp(-z[:, :3 * H])), np.tanh(z[:, 3 * H:])], 1).astype(np.float32)
    c_prev = rng.standard_normal((R, H)).astype(np.float32) if with_c else None
    c_cur = rng.standard_normal((R, H)).astype(np.float32)
    da_next = (rng.standard_normal((R, G)) * 0.5).astype(np.float32) if with_next else None
    dh_ext = (rng.standard_normal((R, H)) * 0.5).astype(np.float32) if with_ext else None
    dc = (rng.standard_normal((R, H)) * 0.5).astype(np.float32)
    mask = _mask_rows(R, rng) if masked else np.zeros(R, bool)
    ids = np.where(mask, 0, 1).astype(np.int32)
    bufs = {"Wh": Buf(eng, Wh), "g": Buf(eng, gates), "cc": Buf(eng, c_cur), "dc": Buf(eng, dc), "ids": Buf(eng, ids),
            "da": Buf(eng, np.full(R * G, np.nan, np.float32))}
    for k, v in (("cp", c_prev), ("dn", da_next), ("ex", dh_ext)):
        if v is not None:
            bufs[k] = Buf(eng, v)
    b = lambda k: bufs[k].ptr() if k in bufs else None
    path = C.c_int32(-1)
    check(eng.lib.vd_lstm_step_bwd(eng.h, R, H, b("dn"), b("Wh"), b("g"), b("cp"), b("cc"), b("ex"), b("dc"),
                                   b("ids") if masked else None, b("da"), C.byref(path)))
    got_da, got_dc = bufs["da"].get().reshape(R, G), bufs["dc"].get().reshape(R, H)
    for v in bufs.values():
        v.free()
    dh = np.zeros((R, H))
    if with_next:
        dh += da_next.astype(np.float64) @ Wh.astype(np.float64).T
    if with_ext:
        dh += dh_ext
    ref_da, ref_dc = lstm_step_bwd_ref(gates, c_prev, c_cur, dh, dc, mask)
    return (got_da, got_dc), (ref_da, ref_dc), path.value


@pytest.mark.parametrize("H", [64, 128, 192, 512])
def test_lstm_step_bwd_vs_fp64(eng, sms, H):
    """both backward tile widths (BN 128 needs cdiv(R,128) * H/128 >= #SM), R in {1, 127, 128, 129, partial blocks},
    with and without dh_ext and c_prev, masked rows on tile edges; H % 128 != 0 and the last step (no da_next) take the
    CUDA cores, as in the engine"""
    Rs = [1, 127, 128, 129, 1000]
    if H == 512:
        Rs += [_rows_for(H, H // 128, sms, big=False), _rows_for(H, H // 128, sms, big=True)]
    seen = set()
    for n, R in enumerate(Rs):
        with_ext, with_c = n % 2 == 0, n % 3 != 1
        got, ref, path = _lstm_bwd_case(eng, R, H, True, with_ext, with_c, True, seed=H + n)
        want = _bwd_tile(R, H, sms) if H % 128 == 0 else 0
        assert path == want, (R, H, path)
        seen.add(path)
        for name, g, r in (("da", got[0], ref[0]), ("dc", got[1], ref[1])):
            e = np.abs(g - r)
            assert float(e.max()) < 8e-3 and float(np.sqrt(np.mean(e ** 2))) < 1e-3, (name, R, H, float(e.max()))
    assert seen == ({32, 128} if H == 512 else {32} if H % 128 == 0 else {0})
    got, ref, path = _lstm_bwd_case(eng, 129, H, False, True, True, True, seed=H)
    assert path == 0
    for g, r in zip(got, ref):
        assert float(np.abs(g - r).max()) < 1e-5


def test_lstm_step_hooks_refuse_routes_the_engine_never_takes(eng):
    rng = np.random.default_rng(0)
    H, R = 256, 1024
    path = C.c_int32(-1)
    bufs = [Buf(eng, np.zeros(n, np.float32)) for n in (4 * H * H, 4 * H, R * 4 * H, R * H, R * H, 37 * 4 * H)]
    tok = Buf(eng, rng.integers(0, 37, R).astype(np.int32))
    WhT, bias, g, c, h, pt = (x.ptr() for x in bufs)
    try:
        eng.set_math_mode(VD_MATH_F16)      # this shape is the fp16 option LSTM's (lstm16.cu), which has no hook
        assert eng.lib.vd_lstm_step_fwd(eng.h, R, H, h, WhT, H, bias, g, 0, pt, 37, tok.ptr(), None, c, h, None, C.byref(path)) != 0
        eng.set_math_mode(VD_MATH_FP32)     # the CUDA-core route gathers in its x-projection GEMM, never from a table
        assert eng.lib.vd_lstm_step_fwd(eng.h, R, H, h, WhT, H, bias, g, 0, pt, 37, tok.ptr(), None, c, h, None, C.byref(path)) != 0
    finally:
        eng.set_math_mode(VD_MATH_TF32)
        for x in bufs + [tok]:
            x.free()


# ---------------------------------------------------------------------------------------------- odd sizes, whole graphs
def _rel(a, b):
    a = np.asarray(a, np.float64).ravel()
    b = np.asarray(b, np.float64).ravel()
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def _train_and_eval(p, flat, nb, mode, profile=False):
    eng = Engine(p)
    eng.set_math_mode(mode)
    eng.set_parameters(flat)
    eng.set_training(1)
    eng.set_dropout_seed(11, 3)
    eng.zero_grad()
    if profile:
        eng.profile(True)
    loss = eng.forward_backward(Batch(nb))
    g = eng.get_gradients()
    stats = {}
    if profile:
        for name in ("enc_pair_fwd", "enc_pair_bwd", "vocab_lse", "vocab_dlogits", "lstm_step_first", "lstm_step_small",
                     "lstm_step_bwd_last", "lstm_step_bwd_small"):
            stats[name] = eng.kernel_stats(name)["launches"]
        eng.profile(False)
    eng.set_training(0)
    b = Batch(nb)
    eng.encoder_forward(b)
    out = eng.decoder_forward(b)
    dec = out.numpy() if out is not None else None
    eng.close()
    return loss, g, dec, stats


ODD = {
    # embedSize 36: x-projections with a ragged last k-block, [4H, D+H] weights with D % 32 != 0
    "e36_h64": dict(enc="hre-ques-hist", dec="gen", kw=dict(embedSize=36, rnnHiddenSize=64, vocabSize=200), B=7),
    "e36_h128": dict(enc="lf-ques-im-hist", dec="disc", kw=dict(embedSize=36, rnnHiddenSize=128, vocabSize=200, numOptions=10), B=7),
    # vocabSize 301: d-logits rows of 301 floats (not 16-byte aligned) behind a fused forward that used to take the shape
    "v301": dict(enc="lf-ques", dec="gen", kw=dict(embedSize=64, rnnHiddenSize=128, vocabSize=301), B=13),
    # H = 192: tensor-core forward steps with CUDA-core BPTT (TF32), unit-split persistent encoder BPTT (F16)
    "h192": dict(enc="hre-ques-hist", dec="disc", kw=dict(embedSize=64, rnnHiddenSize=192, vocabSize=200, numOptions=10), B=7),
}


@pytest.mark.parametrize("mode", [VD_MATH_TF32, VD_MATH_F16])
@pytest.mark.parametrize("cfg", sorted(ODD))
def test_odd_size_graph_matches_oracle_and_fp32(cfg, mode):
    c = ODD[cfg]
    p = small_params(c["enc"], c["dec"], **c["kw"])
    flat = init_parameters(p, seed=3)
    nb = make_batch(p, c["B"], seed=7, max_ques_len=9, max_ans_len=6, max_cap_len=12, max_hist_len=14, max_hist_concat=40,
                    empty_round_every=4)
    loss, g, dec, st = _train_and_eval(p, flat, nb, mode, profile=True)
    loss32, g32, dec32, _ = _train_and_eval(p, flat, nb, VD_MATH_FP32)
    P, tb = torch_params(p, flat), torch_batch(nb)
    psite = {O.SITE_FUSION: p["dropout"]}
    ref = O.forward_backward(O.Ctx(train=True, mask_fn=philox.make_mask_fn(11, 3, psite), structure="batched"), p, P, tb)
    assert abs(loss - ref["loss"]) < 5e-3 * max(1.0, abs(ref["loss"])), (loss, ref["loss"])
    assert abs(loss - loss32) < 5e-3 * max(1.0, abs(loss32)), (loss, loss32)
    for name, s in seg_slices(p).items():
        r = ref["grads"][name].numpy().ravel()
        if np.abs(r).max() < 1e-7:
            continue
        assert _rel(g[s], r) < 3e-2, (name, _rel(g[s], r))
        assert _rel(g[s], g32[s]) < 3e-2, (name, _rel(g[s], g32[s]))
    if dec is not None:
        assert float(np.abs(dec - dec32).max()) < 5e-3 * max(1.0, float(np.abs(dec32).max()))
    # the intended kernel classes ran
    if cfg == "v301":
        assert st["vocab_dlogits"] == 0     # V % 4 != 0: materialised logits ("vocab_lse" counts the refused attempt too)
    if cfg == "h192" and mode == VD_MATH_F16:
        assert st["enc_pair_fwd"] > 0 and st["enc_pair_bwd"] > 0    # H % 128 != 0: the unit-split k_enc_pair_bwd<false>
    if cfg == "h192" and mode == VD_MATH_TF32:
        assert st["lstm_step_first"] > 0                             # tensor-core forward steps ...
        assert st["lstm_step_bwd_last"] == 0 and st["lstm_step_bwd_small"] > 0   # ... CUDA-core BPTT
    if cfg.startswith("e36") and mode == VD_MATH_TF32:
        assert st["lstm_step_first"] > 0                             # D % 32 != 0 still on the fused tensor-core steps
        assert (st["lstm_step_bwd_last"] > 0) == (p["rnnHiddenSize"] % 128 == 0)


def test_gen_vocab_fused_route_at_aligned_odd_vocab():
    """vocabSize 300 + 4 = 304 (a multiple of 4 but not of 16 or 128): the fused forward and the fused d-logits both run,
    with a ragged last column tile, and agree with the oracle"""
    p = small_params("lf-ques", "gen", embedSize=64, rnnHiddenSize=128, vocabSize=304)
    flat = init_parameters(p, seed=3)
    nb = make_batch(p, 13, seed=7, max_ques_len=9, max_ans_len=6, empty_round_every=4)
    loss, g, _, st = _train_and_eval(p, flat, nb, VD_MATH_TF32, profile=True)
    assert st["vocab_lse"] > 0 and st["vocab_dlogits"] > 0
    ref = O.forward_backward(O.Ctx(train=True, mask_fn=philox.make_mask_fn(11, 3), structure="batched"), p,
                             torch_params(p, flat), torch_batch(nb))
    assert abs(loss - ref["loss"]) < 5e-3 * abs(ref["loss"])
    for name, s in seg_slices(p).items():
        r = ref["grads"][name].numpy().ravel()
        if np.abs(r).max() >= 1e-7:
            assert _rel(g[s], r) < 3e-2, name

