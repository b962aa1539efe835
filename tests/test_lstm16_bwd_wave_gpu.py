"""The fp16 option-LSTM BPTT (lstm16.cu, k_lstm16_bptt) over T - 1 steps in one call, through vd_test_kernel's lstm16_bptt:
a cluster of H / 128 CTAs per 128-row block runs steps T - 2 .. 0 with the cell-gradient carry on chip, in waves of as many
clusters as the device and the SM budget hold.  Per case:

* every da_t (t = T - 2 .. 0) and the final carry are bitwise equal to T - 1 chained one-step launches through
  vd_lstm16_step_bwd, which tests/test_lstm16_bwd_step_gpu.py pins to the outputs of the step kernel it replaced.  A row
  block run twice, or not at all, would leave a different carry;
* the guard rows past the last slice of da and past R of the carry are untouched, and every input (the slice of da the
  run starts from included) is bitwise unchanged;
* the launch plan: clusters of H / 128 CTAs, waves x row blocks per wave covers the row blocks, and no wave is empty; the
  case's wave shape (one wave with fewer row blocks than fit, or several with an unequal last one) is the one intended.

The inputs of step t are rows 7t .. 7t + R - 1 of one seeded table per tensor, so that the benched shape (R = 32 000,
H = 512, T = 20) does not need T tables of random numbers."""
import ctypes as C

import numpy as np
import pytest
import torch

from helpers import call, small_params
from lstm16_bwd_cases import GUARD, NAN16, SCALES, case_seed
from visdial_b200 import Engine
from visdial_b200._lib import check

pytestmark = pytest.mark.gpu

RESERVE = 16           # the SMs the overlapped option BPTT leaves to the encoder (Engine::opt_reserve_sms)
SHIFT = 7              # step t reads rows SHIFT t .. SHIFT t + R - 1 of each table

# (name, H, R, T, SM budget: "all" or "reserve", mask ids, initial cell state, expected waves: "one" or "several")
CASES = [
    ("c4", 512, 32000, 20, "all", True, False, "several"),             # the benched shape: 250 row blocks
    ("c4_reserve", 512, 32000, 20, "reserve", True, False, "several"),  # the overlapped step's budget
    ("c4_h256", 256, 32000, 6, "all", True, True, "several"),           # clusters of 2
    ("rag37", 512, 1024 + 3 * 128 + 37, 5, "all", True, True, "one"),   # ragged last block, fewer blocks than fit
    ("rag100_h256", 256, 1024 + 5 * 128 + 100, 4, "reserve", True, False, "one"),
    ("r1024", 512, 1024, 3, "all", True, True, "one"),
    ("no_mask", 256, 2000, 2, "all", False, False, "one"),              # one step, every row kept
]


def _alloc(eng, nbytes):
    p = C.c_void_p()
    check(eng.lib.vd_device_alloc(eng.h, C.byref(p), nbytes))
    return p


def _at(p, off):
    return C.c_void_p(p.value + off)


def _put(eng, p, a, off=0):
    a = np.ascontiguousarray(a)
    check(eng.lib.vd_memcpy_h2d(eng.h, _at(p, off), a.ctypes.data, a.nbytes))


def _get(eng, p, shape, dtype, off=0):
    out = np.empty(shape, dtype)
    check(eng.lib.vd_memcpy_d2h(eng.h, out.ctypes.data, _at(p, off), out.nbytes))
    return out


def make_tables(H, R, T, masked, with_c0, seed):
    rng = np.random.default_rng(seed)
    G, n = 4 * H, R + SHIFT * T
    s_dn, s_dc = SCALES["engine"]
    z = rng.standard_normal((n, G), np.float32) * np.float32(1.5)
    gates = np.concatenate([1 / (1 + np.exp(-z[:, :3 * H])), np.tanh(z[:, 3 * H:])], 1).astype(np.float16)
    return dict(
        Whb=(rng.standard_normal((H, G), np.float32) / np.float32(np.sqrt(G))).astype(np.float16),
        gates=gates,
        c=rng.standard_normal((n, H), np.float32) * np.float32(1.5),
        c0=rng.standard_normal((R, H), np.float32) * np.float32(1.5) if with_c0 else None,
        da_last=(rng.standard_normal((R, G), np.float32) * np.float32(s_dn)).astype(np.float16),
        dc=rng.standard_normal((R, H), np.float32) * np.float32(s_dc),
        ids=np.where(rng.random((T, R)) < 0.1, 0, 1).astype(np.int32) if masked else None)


@pytest.fixture(scope="module")
def eng():
    e = Engine(small_params("lf-ques", "disc"))
    yield e
    e.close()


@pytest.mark.parametrize("name,H,R,T,budget,masked,with_c0,waves", CASES, ids=[c[0] for c in CASES])
def test_lstm16_bptt_waves(eng, name, H, R, T, budget, masked, with_c0, waves):
    G = 4 * H
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    sm_budget = 0 if budget == "all" else sms - RESERVE
    tb = make_tables(H, R, T, masked, with_c0, case_seed(name))
    SG, SC = R * G * 2, R * H * 4                                   # bytes of one slice of da / gates, of c
    nan_da = np.full((R, G), NAN16, np.uint16)
    ptr = {}
    try:
        for k, nb in (("Whb", H * G * 2), ("gates", T * SG), ("c", T * SC), ("dc_new", (R + GUARD) * H * 4),
                      ("dc_ref", (R + GUARD) * H * 4), ("da_new", T * SG + GUARD * G * 2), ("da_ref", T * SG + GUARD * G * 2),
                      ("plan", 3 * 8)):
            ptr[k] = _alloc(eng, nb)
        if with_c0:
            ptr["c0"] = _alloc(eng, SC)
            _put(eng, ptr["c0"], tb["c0"])
        if masked:
            ptr["ids"] = _alloc(eng, T * R * 4)
            _put(eng, ptr["ids"], tb["ids"])
        _put(eng, ptr["Whb"], tb["Whb"])
        for t in range(T):
            _put(eng, ptr["gates"], tb["gates"][SHIFT * t:SHIFT * t + R], t * SG)
            _put(eng, ptr["c"], tb["c"][SHIFT * t:SHIFT * t + R], t * SC)
        dc_img = np.concatenate([tb["dc"], np.full((GUARD, H), np.nan, np.float32)])
        for run in ("new", "ref"):
            for t in range(T - 1):
                _put(eng, ptr["da_" + run], nan_da, t * SG)
            _put(eng, ptr["da_" + run], tb["da_last"], (T - 1) * SG)
            _put(eng, ptr["da_" + run], np.full((GUARD, G), NAN16, np.uint16), T * SG)
            _put(eng, ptr["dc_" + run], dc_img)

        # the T - 1 steps in one call, in waves
        rc = call(eng, "lstm16_bptt", [ptr["da_new"], ptr["Whb"], ptr["gates"], ptr["c"], ptr.get("c0"), ptr.get("ids"),
                                       ptr["dc_new"], ptr["plan"]], [R, H, T, sm_budget])
        check(rc)
        # the same steps as chained one-step launches
        for t in range(T - 2, -1, -1):
            c_prev = _at(ptr["c"], (t - 1) * SC) if t > 0 else ptr.get("c0")
            ids = _at(ptr["ids"], t * R * 4) if masked else None
            check(eng.lib.vd_lstm16_step_bwd(eng.h, R, H, _at(ptr["da_ref"], (t + 1) * SG), ptr["Whb"],
                                             _at(ptr["gates"], t * SG), c_prev, _at(ptr["c"], t * SC), ptr["dc_ref"], ids,
                                             _at(ptr["da_ref"], t * SG)))

        csize, per_wave, nwaves = (int(v) for v in _get(eng, ptr["plan"], (3,), np.int64))
        blocks = -(-R // 128)
        print("WAVES %-12s H %d R %5d T %2d budget %3d SMs: %d row blocks, %d launches of %d clusters of %d CTAs, the last "
              "of %d" % (name, H, R, T, sm_budget or sms, blocks, nwaves, per_wave, csize, blocks - (nwaves - 1) * per_wave))
        assert csize == H // 128 and per_wave * csize <= (sm_budget or sms)
        assert (nwaves - 1) * per_wave < blocks <= nwaves * per_wave, (name, "the waves do not cover the row blocks once")
        if waves == "one":
            assert nwaves == 1 and per_wave == blocks, name
        else:
            assert nwaves > 1 and blocks % per_wave != 0, (name, "the case should end in an unequal wave")

        for t in range(T - 1):
            a = _get(eng, ptr["da_new"], (R, G), np.uint16, t * SG)
            b = _get(eng, ptr["da_ref"], (R, G), np.uint16, t * SG)
            assert (a != NAN16).all(), (name, t, "da_t not written everywhere")
            assert np.array_equal(a, b), (name, t, "da_t differs from the chained one-step launches")
        dc_new = _get(eng, ptr["dc_new"], (R + GUARD, H), np.float32)
        dc_ref = _get(eng, ptr["dc_ref"], (R + GUARD, H), np.float32)
        assert dc_new[:R].tobytes() == dc_ref[:R].tobytes(), (name, "the final carry differs from the chained launches")
        assert dc_new[R:].tobytes() == dc_img[R:].tobytes(), (name, "carry rows past R written")
        if masked:
            assert (dc_new[:R][tb["ids"][0] == 0] == 0).all(), (name, "masked rows of the carry must be exact zeros")

        # guard rows, and every input unchanged
        assert (_get(eng, ptr["da_new"], (GUARD, G), np.uint16, T * SG) == NAN16).all(), (name, "rows past da written")
        assert _get(eng, ptr["da_new"], (R, G), np.float16, (T - 1) * SG).tobytes() == tb["da_last"].tobytes(), name
        assert _get(eng, ptr["Whb"], (H, G), np.float16).tobytes() == tb["Whb"].tobytes(), name
        for t in range(T):
            assert _get(eng, ptr["gates"], (R, G), np.float16, t * SG).tobytes() == \
                tb["gates"][SHIFT * t:SHIFT * t + R].tobytes(), (name, t, "gates written")
            assert _get(eng, ptr["c"], (R, H), np.float32, t * SC).tobytes() == \
                tb["c"][SHIFT * t:SHIFT * t + R].tobytes(), (name, t, "c written")
        if with_c0:
            assert _get(eng, ptr["c0"], (R, H), np.float32).tobytes() == tb["c0"].tobytes(), name
        if masked:
            assert np.array_equal(_get(eng, ptr["ids"], (T, R), np.int32), tb["ids"]), name
    finally:
        for p in ptr.values():
            check(eng.lib.vd_device_free(eng.h, p))


def test_lstm16_bptt_refuses_one_step(eng):
    """T = 1 has no recurrent step: the call is refused before anything runs"""
    p = _alloc(eng, 8)
    try:
        assert call(eng, "lstm16_bptt", [p, p, p, p, None, None, p, None], [1024, 512, 1, 0]) != 0
    finally:
        check(eng.lib.vd_device_free(eng.h, p))
