"""Seeded inputs for the fp16 option-LSTM backward step (lstm16.cu, k_lstm16<1>), one run of it through the test hook
vd_lstm16_step_bwd, and the per-element check of its outputs against fp64.  Shared by tests/test_lstm16_bwd_step_gpu.py, the
CPU test that the check rejects subtly wrong kernels (tests/test_lstm16_bwd_bound.py) and the script that writes the bit-exact
fixture (tests/golden/make_lstm16_bwd_golden.py).

The step, per row r and hidden unit u, with [i f o g] = the saved fp16 gates of step t and keep = 0 on masked rows:
  dh  = sum_k da_{t+1}[r, k] Whb[u, k]                      (f16 wgmma, fp32 accumulation, K = 4H)
  tc  = tanh.approx(c_t);  dd = (dc + dh o (1 - tc^2)) keep
  da  = fp16 of [dd g i(1-i), dd c_{t-1} f(1-f), dh keep tc o(1-o), dd i(1-g^2)]   (round to nearest, saturating)
  dc <- dd f                                                (fp32, in place)

Every buffer, inputs included, has GUARD rows past R (past H for Whb) filled with a NaN pattern (a sentinel for the int32
mask ids): the kernel must read none of them into a result and write none of them."""
import ctypes as C
from collections import Counter

import numpy as np

from helpers import lstm_step_bwd_ref
from lstm16_fwd_cases import GUARD, NAN16, case_seed, digest  # noqa: F401  (re-exported for the tests and the fixture script)
from seq_lstm_ref import U, bptt_bound
from visdial_b200._lib import check

BM, BN = 128, 128            # rows and hidden units of one k_lstm16<1> tile
IGUARD = -123456789          # guard rows of the int32 mask ids
MASKED = (0, 15, 16, 63, 64, 127, 128)   # warp, warpgroup and tile edges; R - 1 too

# da_{t+1} and the incoming cell-gradient carry are N(0, 1) times these.  "engine" is the engine's gradient scale: the BPTT
# runs on gradients scaled so that max|dh_T| is in [2^9, 2^10) (k_pick_scale).  "subnormal" puts da in fp16's subnormal
# range (below 2^-14); "saturate" makes dd g i(1-i) and dd i(1-g^2) pass 65 504, so that the saturating store must clamp.
SCALES = {"unit": (1.0, 1.0), "engine": (2.0 ** 8, 2.0 ** 8), "subnormal": (2.0 ** -16, 2.0 ** -16),
          "saturate": (2.0 ** 8, 2.0 ** 20)}

# (name, H, R, kind); kind = the scale regime, or an engine-scale case without c_prev or without mask ids.  The tile
# figures assume 132 SMs; tile_plan computes them from the device's SM count.
CASES = [
    ("c4_h512", 512, 32000, "engine"),              # the benched shape: 1 000 tiles, 8 per CTA; CTAs reuse their staging
                                                    # tiles across tiles (bulk_wait_read0 / cp.async hand-over)
    ("c4_h256", 256, 32000, "engine"),              # 500 tiles, 4 per CTA
    ("unequal", 512, 8910, "engine"),               # 280 tiles on 94 CTAs: 92 take 3, 2 take 2
    ("r1024_h512", 512, 1024, "engine"),            # 32 tiles, fewer than SMs: one per CTA
    ("r1024_h256", 256, 1024, "engine"),            # 16 tiles
    # R % 128 = r: the last row block holds r rows (warps own 16 rows, warpgroups 64)
    ("rag1", 512, 1024 + 1 * 128 + 1, "engine"),    # one row: warp 0 holds 1 row, the second warpgroup is empty
    ("rag16", 256, 1024 + 2 * 128 + 16, "engine"),  # warp 0 full, warps 1-7 empty
    ("rag37", 512, 1024 + 3 * 128 + 37, "engine"),  # warp 2 cut at 5 rows, the second warpgroup empty
    ("rag64", 256, 1024 + 4 * 128 + 64, "engine"),  # the first warpgroup full, the second exactly empty
    ("rag100", 512, 1024 + 5 * 128 + 100, "engine"),  # the second warpgroup ragged: warp 6 holds 4 rows, warp 7 none
    ("rag127", 256, 1024 + 6 * 128 + 127, "engine"),  # warp 7 holds 15 rows
    ("no_c_prev", 256, 2000, "no_c_prev"),          # c_prev null: the forget-gate gradient reads zeros
    ("no_mask", 512, 1500, "no_mask"),              # mask_ids null: every row kept
    ("subnormal", 256, 1536, "subnormal"),          # da_{t+1} and dc ~ 2^-16: da lands among fp16 subnormals
    ("saturate", 512, 1280, "saturate"),            # dc ~ 2^20: da past 65 504 must come back as +-65504, not inf
]

FP16_MAX = 65504.0
SAT = 65520.0                # fp16 rounds to nearest up to here; past it only the saturating store keeps a value finite
TANH = 2.0 ** -10            # tanh.approx.f32: relative error 2^-11 of a value at most 1, doubled as in bptt_bound's callers
STORE = 2.0 ** -11           # fp16 round to nearest: half an ulp, relative
STORE_ABS = 2.0 ** -25       # half of fp16's smallest subnormal
CONTRACTION = 1.0            # factor on the (4H + 2) U S contraction term: 1 = fp32 accumulation rounded to nearest


def _f16(x):
    return np.asarray(x, np.float32).astype(np.float16)


def make_inputs(H, R, kind, seed):
    """the hook's inputs as host arrays (no guard rows): da_next (R, 4H) and Whb (H, 4H) fp16, gates (R, 4H) fp16, c_prev (or
    None), c_cur and dc (R, H) fp32, mask (R,) bool (or None) and its ids"""
    rng = np.random.default_rng(seed)
    G = 4 * H
    s_dn, s_dc = SCALES.get(kind, SCALES["engine"])
    Whb = _f16(rng.standard_normal((H, G)) / np.sqrt(G))                        # (H, 4H): dh = da_next Whb^T
    z = rng.standard_normal((R, G)) * 1.5
    gates = _f16(np.concatenate([1 / (1 + np.exp(-z[:, :3 * H])), np.tanh(z[:, 3 * H:])], 1))
    c_prev = None if kind == "no_c_prev" else (rng.standard_normal((R, H)) * 1.5).astype(np.float32)
    c_cur = (rng.standard_normal((R, H)) * 1.5).astype(np.float32)
    da_next = _f16(rng.standard_normal((R, G)) * s_dn)
    dc = (rng.standard_normal((R, H)) * s_dc).astype(np.float32)
    mask = None
    if kind != "no_mask":
        mask = rng.random(R) < 0.1
        mask[[r for r in MASKED if r < R] + [R - 1]] = True
    ids = None if mask is None else np.where(mask, 0, 1).astype(np.int32)
    return dict(da_next=da_next, Whb=Whb, gates=gates, c_prev=c_prev, c_cur=c_cur, dc=dc, mask=mask, ids=ids)


def guarded(a):
    """a with GUARD more rows of the guard pattern"""
    a = np.ascontiguousarray(a)
    fill = {np.dtype(np.float16): NAN16, np.dtype(np.float32): np.float32(np.nan), np.dtype(np.int32): IGUARD}[a.dtype]
    out = np.empty((a.shape[0] + GUARD,) + a.shape[1:], a.dtype)
    if a.dtype == np.float16:
        out.view(np.uint16)[a.shape[0]:] = fill
    else:
        out[a.shape[0]:] = fill
    out[:a.shape[0]] = a
    return out


def _alloc(eng, nbytes):
    p = C.c_void_p()
    check(eng.lib.vd_device_alloc(eng.h, C.byref(p), nbytes))
    return p


def _put(eng, p, a):
    check(eng.lib.vd_memcpy_h2d(eng.h, p, a.ctypes.data, a.nbytes))


def _get(eng, p, like):
    out = np.empty_like(like)
    check(eng.lib.vd_memcpy_d2h(eng.h, out.ctypes.data, p, out.nbytes))
    return out


def run_bwd(eng, H, R, inp, launches=1):
    """Runs the step `launches` times.  Before each launch da16 is filled with NaN again and dc_carry, which the step reads
    and overwrites in place, is uploaded again, so every launch starts from the same state.  Returns (outs, ins): outs has one
    dict per launch of the full output buffers, guard rows included: da (R + GUARD, 4H) fp16, dc (R + GUARD, H) fp32; ins
    maps each input to (the image uploaded, the image read back after the last launch)."""
    G = 4 * H
    init = {"da": guarded(np.full((R, G), NAN16, np.uint16).view(np.float16)), "dc": guarded(inp["dc"])}
    imgs = {k: guarded(inp[k]) for k in ("da_next", "Whb", "gates", "c_prev", "c_cur", "ids") if inp[k] is not None}
    ptr = {k: _alloc(eng, a.nbytes) for k, a in list(imgs.items()) + list(init.items())}
    outs = []
    try:
        for k, a in imgs.items():
            _put(eng, ptr[k], a)
        for _ in range(launches):
            for k, a in init.items():
                _put(eng, ptr[k], a)
            check(eng.lib.vd_lstm16_step_bwd(eng.h, R, H, ptr["da_next"], ptr["Whb"], ptr["gates"], ptr.get("c_prev"),
                                             ptr["c_cur"], ptr["dc"], ptr.get("ids"), ptr["da"]))
            outs.append({k: _get(eng, ptr[k], a) for k, a in init.items()})
        ins = {k: (a, _get(eng, ptr[k], a)) for k, a in imgs.items()}
    finally:
        for p in ptr.values():
            check(eng.lib.vd_device_free(eng.h, p))
    return outs, ins


def tile_plan(H, R, sms):
    """the tiles of k_lstm16<1> and how its persistent grid splits them (lstm16.cu: balanced_workers over the SMs; CTA b takes
    tiles b, b + grid, ...): (tiles, grid, {tiles per CTA: CTAs})"""
    tiles = -(-R // BM) * (H // BN)
    grid = tiles if tiles <= sms else -(-tiles // -(-tiles // sms))
    return tiles, grid, dict(Counter(len(range(b, tiles, grid)) for b in range(grid)))


def reference(inp, r0, r1):
    """fp64 da and dc of rows r0 .. r1 - 1 and their per-element bounds.

    dh = da_next Whb^T and S = |da_next| |Whb|^T; the operands are exact fp16 and the accumulation fp32, so |dh error| <=
    (4H + 2) U S.  The pointwise part is bptt_bound's model at T = 1 (tanh.approx within TANH, 3 U of the fp32 carry terms,
    U of the product dd f); the gate gradients add 4 U of their fp32 products, and the fp16 store half an ulp of the stored
    value: STORE |da| relative (with STORE of the fp32 error itself) and STORE_ABS among the subnormals."""
    G = inp["Whb"].shape[1]
    dn, W = inp["da_next"][r0:r1].astype(np.float64), inp["Whb"].astype(np.float64)
    dh, S = dn @ W.T, np.abs(dn) @ np.abs(W).T
    e_dh = CONTRACTION * (G + 2) * U * S
    g, cc, dc = (inp[k][r0:r1].astype(np.float64) for k in ("gates", "c_cur", "dc"))
    cp = None if inp["c_prev"] is None else inp["c_prev"][r0:r1].astype(np.float64)
    m = None if inp["mask"] is None else inp["mask"][r0:r1]
    da, dcn = lstm_step_bwd_ref(g, cp, cc, dh, dc, m)
    eda, edc = bptt_bound(g[None], cc[None], cp, None if m is None else m[None], dh[None], e_dh[None], dc, TANH)
    eda = (eda[0] + 4 * U * np.abs(da)) * (1 + STORE) + STORE * np.abs(da) + STORE_ABS
    return da, dcn, eda, edc


def check_step(inp, da16, dc, block=4096):
    """The per-element check of one step's outputs, rows 0 .. R-1, against reference(), in blocks of `block` rows (one fp64
    (R, 4H) array is 524 MB at R = 32 000, H = 512).  Returns
      da, dc: the worst |out - ref| / bound, with da's reference clipped to +-65504 as the saturating store clips; inf for a
              non-finite output, or for an element whose reference is past SAT by more than its bound (a store rounding to
              nearest would give inf) that is not exactly 65 504 with the reference's sign;
      clamped: the number of such elements;
      subnormals: the number of da elements that are nonzero fp16 subnormals;
      flushed: the number of da elements that are zero where |ref| > 1.5 2^-24 (they round to at least 2^-24)."""
    R = inp["dc"].shape[0]
    res = {"da": 0.0, "dc": 0.0, "clamped": 0, "subnormals": 0, "flushed": 0}
    for r0 in range(0, R, block):
        r1 = min(R, r0 + block)
        ref_da, ref_dc, eda, edc = reference(inp, r0, r1)
        got_da, got_dc = da16[r0:r1].astype(np.float64), dc[r0:r1].astype(np.float64)
        sat = np.abs(ref_da) > SAT + eda
        res["clamped"] += int(sat.sum())
        a = np.abs(got_da)
        res["subnormals"] += int(((a > 0) & (a < 2.0 ** -14)).sum())
        res["flushed"] += int(((got_da == 0) & (np.abs(ref_da) > 1.5 * 2.0 ** -24)).sum())
        if not (np.isfinite(got_da).all() and (got_da[sat] == np.sign(ref_da[sat]) * FP16_MAX).all()):
            res["da"] = np.inf
        else:
            # the saturating store is clip(round(x)); clipping shrinks distances, so |out - clip(ref)| <= |round(x) - ref|
            res["da"] = max(res["da"], float(np.max(np.abs(got_da - np.clip(ref_da, -FP16_MAX, FP16_MAX)) / eda)))
        if not np.isfinite(got_dc).all():
            res["dc"] = np.inf
        else:
            res["dc"] = max(res["dc"], float(np.max(np.abs(got_dc - ref_dc) / np.maximum(edc, 1e-300))))
    return res
