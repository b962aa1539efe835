"""Seeded inputs for the fp16 option-LSTM forward step (lstm16.cu, k_lstm16<0>) and one run of it through the test hook
vd_lstm16_step_fwd, shared by tests/test_lstm16_fwd_resident_gpu.py and the script that writes its bit-exact fixture
(tests/golden/make_lstm16_fwd_golden.py).

Every output buffer has GUARD rows past R, filled with a NaN pattern: the kernel must leave them alone."""
import ctypes as C
import hashlib

import numpy as np

from visdial_b200._lib import check

V1 = 41                 # rows of the x-projection table; row 0 = the pad token's, all zero
GUARD = 64              # rows past R in every output buffer
NAN16 = np.uint16(0x7E01)

# (name, H, R, with_c, save_gates, h32)
CASES = [
    ("c4_h512", 512, 32000, True, True, True),        # the benched shape: 250 row blocks over 16 slices x 8 CTAs
    ("h256", 256, 4000, True, True, True),            # 8 slices, 32 row blocks (the last one ragged)
    ("r1024_h512", 512, 1024, False, True, False),    # 8 row blocks: one per CTA of a slice
    ("r1024_h256", 256, 1024, True, False, True),
    ("half_empty", 512, 1024 + 3 * 128 + 37, True, True, True),     # R % 128 = 37: the last block's second half is empty
    ("half_ragged", 256, 1024 + 5 * 128 + 100, False, True, True),  # R % 128 = 100: the second half is ragged
    ("one_row", 512, 1024 + 128 + 1, True, True, False),            # R % 128 = 1
    ("last_half_full", 256, 1024 + 64, True, True, True),           # R % 128 = 64: the second half is exactly empty
]


def _f16(x):
    return np.asarray(x, np.float32).astype(np.float16)


def make_inputs(H, R, with_c, seed):
    rng = np.random.default_rng(seed)
    G = 4 * H
    Wh = _f16(rng.standard_normal((G, H)) / np.sqrt(H))                        # (4H, H): gates = h Wh^T
    table = _f16(rng.standard_normal((V1, G)) * 0.5)
    table[0] = 0
    tok = rng.integers(0, V1, R).astype(np.int32)
    tok[rng.random(R) < 0.3] = 0                                               # ended sequences: pad tokens
    bias = (rng.standard_normal(G) * 0.5).astype(np.float32)
    h_prev = _f16(np.tanh(rng.standard_normal((R, H))))
    c_prev = rng.standard_normal((R, H)).astype(np.float32) if with_c else None
    mask = rng.random(R) < 0.1
    mask[[0, 63, 64, 127, 128, R - 1]] = True                                  # half-block and block edges, the last row
    ids = np.where(mask, 0, 1).astype(np.int32)
    return dict(Wh=Wh, table=table, tok=tok, bias=bias, h_prev=h_prev, c_prev=c_prev, mask=mask, ids=ids)


def _alloc(eng, a):
    a = np.ascontiguousarray(a)
    p = C.c_void_p()
    check(eng.lib.vd_device_alloc(eng.h, C.byref(p), a.nbytes))
    check(eng.lib.vd_memcpy_h2d(eng.h, p, a.ctypes.data, a.nbytes))
    return p


def run_fwd(eng, H, R, inp, save_gates, h32, launches=1):
    """Runs the step `launches` times into the same output buffers; returns a list (one entry per launch) of dicts of the
    full output buffers, guard rows included: g (R + GUARD, 4H) fp16, c (R + GUARD, H) fp32, h16 fp16, h32 fp32."""
    G = 4 * H
    outs0 = {"g": np.full((R + GUARD, G), NAN16, np.uint16).view(np.float16) if save_gates else None,
             "c": np.full((R + GUARD, H), np.nan, np.float32),
             "h16": np.full((R + GUARD, H), NAN16, np.uint16).view(np.float16),
             "h32": np.full((R + GUARD, H), np.nan, np.float32) if h32 else None}
    ins = {"h": inp["h_prev"], "W": inp["Wh"], "pt": inp["table"], "tok": inp["tok"], "bias": inp["bias"],
           "cp": inp["c_prev"], "ids": inp["ids"]}
    ptr = {k: _alloc(eng, a) for k, a in ins.items() if a is not None}
    optr = {k: _alloc(eng, a) for k, a in outs0.items() if a is not None}
    res = []
    try:
        for _ in range(launches):
            check(eng.lib.vd_lstm16_step_fwd(eng.h, R, H, ptr["h"], ptr["W"], ptr["pt"], ptr["tok"], ptr["bias"], ptr.get("cp"),
                                             ptr["ids"], optr.get("g"), optr["c"], optr["h16"], optr.get("h32")))
            got = {}
            for k, p in optr.items():
                out = np.empty_like(outs0[k])
                check(eng.lib.vd_memcpy_d2h(eng.h, out.ctypes.data, p, out.nbytes))
                got[k] = out
            res.append(got)
    finally:
        for p in list(ptr.values()) + list(optr.values()):
            check(eng.lib.vd_device_free(eng.h, p))
    return res


def digest(a, R):
    """sha-256 of the first R rows' bytes"""
    return hashlib.sha256(np.ascontiguousarray(a[:R]).tobytes()).hexdigest()


def case_seed(name):
    return int.from_bytes(hashlib.sha256(name.encode()).digest()[:4], "little")
