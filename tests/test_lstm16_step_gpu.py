"""The fp16 option-LSTM step kernels (lstm16.cu, VD_MATH_F16) through their test hooks vd_lstm16_step_fwd / _bwd, per
element against the numpy step of tests/helpers.py on the same fp16-rounded inputs.

The contraction has exact fp16 products and fp32 accumulation, so what separates the kernels from fp64 is tanh.approx
(relative error 2^-11) and the fp16 rounding of the stored gates, h and da (2^-11 relative): a few 1e-3 of (1 + |ref|).
Swapping two gate blocks, dropping the c_prev term or reading another row's inputs changes outputs by O(0.1).

Shapes: H = 256 and 512; R = 1 024, a ragged R (R % 128 != 0) and one large enough that the persistent CTAs take unequal
numbers of tiles; c_prev absent and present, gates saved or not, the fp32 copy of h, pad tokens and masked rows."""
import ctypes as C

import numpy as np
import pytest

from helpers import lstm_step_bwd_ref, lstm_step_fwd_ref, small_params
from visdial_b200 import Engine
from visdial_b200._lib import check

pytestmark = pytest.mark.gpu

TOL = 4e-3
V1 = 41                                    # rows of the x-projection table; row 0 = the pad token's, all zero


@pytest.fixture(scope="module")
def eng():
    e = Engine(small_params("lf-ques", "disc"))
    yield e
    e.close()


class Dev:
    """Device copies of host arrays; get(name) reads one back with its original dtype and shape."""

    def __init__(self, eng, **arrays):
        self.eng, self.img, self.p = eng, {}, {}
        for k, a in arrays.items():
            if a is None:
                continue
            a = np.ascontiguousarray(a)
            p = C.c_void_p()
            check(eng.lib.vd_device_alloc(eng.h, C.byref(p), a.nbytes))
            check(eng.lib.vd_memcpy_h2d(eng.h, p, a.ctypes.data, a.nbytes))
            self.img[k], self.p[k] = a, p

    def __call__(self, k):
        return self.p.get(k)

    def get(self, k):
        out = np.empty_like(self.img[k])
        check(self.eng.lib.vd_memcpy_d2h(self.eng.h, out.ctypes.data, self.p[k], out.nbytes))
        return out

    def free(self):
        for p in self.p.values():
            check(self.eng.lib.vd_device_free(self.eng.h, p))


def _f16(x):
    return np.asarray(x, np.float32).astype(np.float16)


def _mask_rows(R, rng):
    m = rng.random(R) < 0.1
    m[[0, 127, 128, R - 1]] = True                 # tile edges and the last row
    return m


def _close(name, got, ref):
    err = np.abs(np.asarray(got, np.float64) - ref) / (1.0 + np.abs(ref))
    assert np.isfinite(got).all(), name
    assert float(err.max()) < TOL and float(np.sqrt(np.mean(err ** 2))) < TOL / 4, (name, float(err.max()))


CASES = [  # (H, R, with_c, save_gates, h32)
    (256, 1024, True, True, False),
    (256, 1101, False, True, True),
    (512, 1024, False, False, True),
    (512, 1101, True, True, False),
    (512, 8910, True, True, True),                  # 1 120 forward / 280 backward tiles: CTAs take unequal tile counts
]


@pytest.mark.parametrize("H,R,with_c,save_gates,h32", CASES)
def test_lstm16_step_fwd(eng, H, R, with_c, save_gates, h32):
    rng = np.random.default_rng(H + R)
    G = 4 * H
    Wh = _f16(rng.standard_normal((G, H)) / np.sqrt(H))                        # (4H, H): gates = h Wh^T
    table = _f16(rng.standard_normal((V1, G)) * 0.5)
    table[0] = 0
    tok = rng.integers(0, V1, R).astype(np.int32)
    tok[rng.random(R) < 0.3] = 0                                               # ended sequences: pad tokens
    bias = (rng.standard_normal(G) * 0.5).astype(np.float32)
    h_prev = _f16(np.tanh(rng.standard_normal((R, H))))
    c_prev = rng.standard_normal((R, H)).astype(np.float32) if with_c else None
    mask = _mask_rows(R, rng)
    ids = np.where(mask, 0, 1).astype(np.int32)
    nan16 = np.full((R, G), np.nan, np.float16)
    d = Dev(eng, h=h_prev, W=Wh, pt=table, tok=tok, bias=bias, cp=c_prev, ids=ids, g=nan16,
            c=np.full((R, H), np.nan, np.float32), h16=nan16[:, :H], h32=np.full((R, H), np.nan, np.float32) if h32 else None)
    try:
        check(eng.lib.vd_lstm16_step_fwd(eng.h, R, H, d("h"), d("W"), d("pt"), d("tok"), d("bias"), d("cp"), d("ids"),
                                         d("g") if save_gates else None, d("c"), d("h16"), d("h32")))
        got = {k: d.get(k) for k in ("g", "c", "h16") + (("h32",) if h32 else ())}
    finally:
        d.free()
    z_x = table.astype(np.float64)[tok] + bias
    ref_g, ref_c, ref_h = lstm_step_fwd_ref(z_x, h_prev, Wh.astype(np.float64).T, c_prev, mask)
    if save_gates:
        _close("gates", got["g"], ref_g)
    else:
        assert np.isnan(got["g"].astype(np.float32)).all(), "gates written although not asked for"
    _close("c", got["c"], ref_c)
    _close("h16", got["h16"], ref_h)
    if h32:
        _close("h32", got["h32"], ref_h)
        assert np.array_equal(got["h32"].astype(np.float16), got["h16"]), "h16 is not the rounded fp32 h"


@pytest.mark.parametrize("H,R,with_c", [(H, R, c) for H, R, c, _, _ in CASES])
def test_lstm16_step_bwd(eng, H, R, with_c):
    rng = np.random.default_rng(7 * H + R)
    G = 4 * H
    Whb = _f16(rng.standard_normal((H, G)) / np.sqrt(G))                       # (H, 4H): dh = da Whb^T
    z = rng.standard_normal((R, G))
    gates = _f16(np.concatenate([1 / (1 + np.exp(-z[:, :3 * H])), np.tanh(z[:, 3 * H:])], 1))
    c_prev = rng.standard_normal((R, H)).astype(np.float32) if with_c else None
    c_cur = rng.standard_normal((R, H)).astype(np.float32)
    da_next = _f16(rng.standard_normal((R, G)) * 0.5)
    dc = (rng.standard_normal((R, H)) * 0.5).astype(np.float32)
    mask = _mask_rows(R, rng)
    ids = np.where(mask, 0, 1).astype(np.int32)
    d = Dev(eng, dn=da_next, W=Whb, g=gates, cp=c_prev, cc=c_cur, dc=dc, ids=ids, da=np.full((R, G), np.nan, np.float16))
    try:
        check(eng.lib.vd_lstm16_step_bwd(eng.h, R, H, d("dn"), d("W"), d("g"), d("cp"), d("cc"), d("dc"), d("ids"), d("da")))
        got_da, got_dc = d.get("da"), d.get("dc")
    finally:
        d.free()
    dh = da_next.astype(np.float64) @ Whb.astype(np.float64).T
    ref_da, ref_dc = lstm_step_bwd_ref(gates, c_prev, c_cur, dh, dc, mask)
    _close("da", got_da, ref_da)
    _close("dc", got_dc, ref_dc)


def test_lstm16_hooks_refuse_other_shapes(eng):
    """the hooks take what lstm16_shape_ok takes and nothing else"""
    R = 1024
    d = Dev(eng, a=np.zeros(R * 4 * 512, np.float16), f=np.zeros(R * 512, np.float32), tok=np.zeros(R, np.int32))
    try:
        for h, r in ((192, 1024), (256, 1023), (768, 2048)):
            assert eng.lib.vd_lstm16_step_fwd(eng.h, r, h, d("a"), d("a"), d("a"), d("tok"), d("f"), None, None, None,
                                              d("f"), d("a"), None) != 0
            assert eng.lib.vd_lstm16_step_bwd(eng.h, r, h, d("a"), d("a"), d("a"), None, d("f"), d("f"), None, d("a")) != 0
    finally:
        d.free()
