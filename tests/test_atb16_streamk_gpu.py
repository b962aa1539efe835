"""The stream-K fp16 weight gradient (lstm16.cu::k_atb16, C += inv_scale * A^T B, A (K x M), B (K x N) fp16) against an
fp64 product of the same fp16 operands: the option LSTM's shape, grids from one CTA to every SM, back-to-back launches
(the claim counter must come back to zero after each), launches on two streams at once, tile widths N % 256 != 0, K off
and below the chunk size, and C anywhere inside a NaN guard band (only C[0:M, 0:N] may be written)."""
import ctypes as C

import pytest
import torch

from helpers import run, small_params
from visdial_b200 import Engine

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    e = Engine(small_params("lf-ques", "disc"))
    yield e
    e.close()


def _ptr(t, off=0):
    return C.c_void_p(t.data_ptr() + t.element_size() * off)


def _atb16(eng, M, N, K, inv=1.0, ctas=0, launches=1, streams=1, off=(0, 0), ldc_extra=0, seed=0):
    """runs `launches` launches onto one C with a NaN guard band; returns (C, fp64 reference, the fp32 error bound)"""
    g = torch.Generator(device="cuda").manual_seed(seed * 7919 + M + N + K)
    A = torch.randn(K, M, device="cuda", generator=g).half()
    B = torch.randn(K, N, device="cuda", generator=g).half()
    ldc = N + ldc_extra
    r0, c0 = off
    rows = M + r0 + 1
    Cbuf = torch.full((rows * ldc + c0 + 64,), float("nan"), device="cuda", dtype=torch.float32)
    view = Cbuf[r0 * ldc + c0:].as_strided((M, N), (ldc, 1))
    C0 = torch.randn(M, N, device="cuda", generator=g)
    view.copy_(C0)
    sc = torch.tensor([inv], device="cuda", dtype=torch.float32)
    ref = torch.zeros(M, N, device="cuda", dtype=torch.float64)
    for k in range(0, K, 65536):
        ref += A[k:k + 65536].double().T @ B[k:k + 65536].double()
    ref = C0.double() + launches * inv * ref
    torch.cuda.synchronize()
    run(eng, "gemm_atb16", [_ptr(A), _ptr(B), _ptr(Cbuf, r0 * ldc + c0), _ptr(sc)],
        [M, N, K, M, N, ldc, ctas, launches, streams])
    torch.cuda.synchronize()
    got = view.double().clone()
    guard = Cbuf.clone()
    guard[r0 * ldc + c0:].as_strided((M, N), (ldc, 1)).fill_(float("nan"))
    assert torch.isnan(guard).all(), "k_atb16 wrote outside C[0:M, 0:N]"
    bound = launches * (2e-6 * K * inv) + 1e-5 * launches
    return got, ref, bound


def _check(got, ref, bound, what):
    err = float((got - ref).abs().max())
    assert torch.isfinite(got).all() and err < bound, (what, err, bound)


def test_option_lstm_shape(eng):
    """dWh of the benched option LSTM: H = 512, 4H = 2048, K = 19 steps x 32 000 rows, gradient scale 2^-7"""
    got, ref, bound = _atb16(eng, 512, 2048, 19 * 32000, inv=2.0 ** -7, off=(1, 4), ldc_extra=8)
    _check(got, ref, bound, "option shape")


@pytest.mark.parametrize("ctas", [1, 2, 5, 31, 64, 0])
def test_grid_sizes(eng, ctas):
    """the same chunks whatever the number of CTAs claiming them (0 = every SM)"""
    got, ref, bound = _atb16(eng, 256, 512, 20011, inv=0.5, ctas=ctas)
    _check(got, ref, bound, ctas)


@pytest.mark.parametrize("M,N,K", [(128, 320, 5000), (192, 384, 64 * 33 + 5), (64, 448, 1000), (256, 2048, 100), (128, 256, 64),
                                   (512, 2048, 64 * 32 * 3 + 1)])
def test_ragged_shapes(eng, M, N, K):
    """N % 256 in {64, 128, 192}, M % 128 == 64, K off the chunk size and below one chunk (32 k-blocks)"""
    got, ref, bound = _atb16(eng, M, N, K, inv=0.25)
    _check(got, ref, bound, (M, N, K))


@pytest.mark.parametrize("off,ldc_extra", [((1, 1), 3), ((0, 2), 0), ((2, 4), 4)])
def test_unaligned_c(eng, off, ldc_extra):
    """C at an offset and pitch that are not 16-byte multiples takes the scalar-atomic epilogue, the last case the v4 one"""
    got, ref, bound = _atb16(eng, 128, 320, 3000, inv=1.0, off=off, ldc_extra=ldc_extra)
    _check(got, ref, bound, (off, ldc_extra))


def test_back_to_back_launches(eng):
    """200 launches on one stream: each starts from a counter the previous one reset"""
    got, ref, bound = _atb16(eng, 128, 256, 4096 + 17, inv=1.0 / 64, launches=200)
    _check(got, ref, bound, "200 launches")


@pytest.mark.parametrize("ctas", [0, 40])
def test_two_streams(eng, ctas):
    """launches alternating between two streams, running at the same time onto one C: one counter per stream"""
    got, ref, bound = _atb16(eng, 256, 1024, 30000, inv=0.125, ctas=ctas, launches=24, streams=2)
    _check(got, ref, bound, "two streams")
