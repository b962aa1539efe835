"""The per-element check of the fp16 option-LSTM backward step (tests/lstm16_bwd_cases.py: check_step, used by
test_lstm16_bwd_step_gpu.py) has teeth, without a GPU.

A numpy emulation of the step on the hook's inputs, as the kernel computes it: dh an fp32 matmul of the fp16 operands; the
pointwise part in fp32, in the kernel's order of operations, with tanh perturbed by up to 2^-11 relative (tanh.approx); the
stores of da rounded to nearest fp16, saturating.  The faithful emulation must pass the check in every regime: unit-scale
gradients, the engine's scale (2^8), fp16's subnormal range (2^-16) and the saturating one (dc ~ 2^20).  Each mutant, a
plausible kernel bug, must fail it in every regime where it changes the result.  All but do_from_dd stay within a third of
the older 4e-3 (1 + |ref|) tolerance of test_lstm16_step_gpu.py at unit scale."""
import numpy as np
import pytest

from lstm16_bwd_cases import case_seed, check_step, make_inputs

H, R = 256, 640
F16_MIN_NORMAL = 2.0 ** -14
REGIMES = ("unit", "engine", "subnormal", "saturate")

# mutant: the regimes where it changes the result (all but the saturating one, whose clamped outputs hide the store's rounding)
MUTANTS = {
    "carry_store16": ("unit", "engine", "subnormal"),   # the cell-gradient carry written as fp16
    "carry_read16": ("unit", "engine", "subnormal"),    # the incoming carry read as fp16
    "dd16": ("unit", "engine", "subnormal"),            # dd rounded to fp16
    "ftz": ("subnormal",),                              # fp16 subnormals of da flushed to zero
    "rtz": ("unit", "engine", "subnormal"),             # da stored rounding toward zero
    "do_from_dd": ("unit", "engine", "subnormal"),      # the output-gate gradient from dd instead of dh
    "no_satfinite": ("saturate",),                      # a store that overflows to inf instead of clamping to 65 504
}


def _f16_round(x, mutant):
    """fp32 -> fp16 -> fp32 as the kernel's cvt.rn.satfinite stores it, or as a mutant would"""
    if mutant == "no_satfinite":
        with np.errstate(over="ignore"):
            return x.astype(np.float16).astype(np.float32)
    y = np.clip(x, -65504, 65504).astype(np.float16)
    if mutant == "rtz":
        y = np.where(np.abs(y.astype(np.float32)) > np.abs(x), np.nextafter(y, np.float16(0)), y)
    if mutant == "ftz":
        y = np.where(np.abs(y) < F16_MIN_NORMAL, np.float16(0), y)
    return y.astype(np.float32)


def emulate(inp, mutant=None, seed=0):
    """da (R, 4H) fp16 and the new carry (R, H) fp32 of one backward step"""
    f32 = np.float32
    rng = np.random.default_rng(seed)
    dh = inp["da_next"].astype(f32) @ inp["Whb"].astype(f32).T
    g = inp["gates"].astype(f32)
    gi, gf, go, gg = np.split(g, 4, axis=1)
    cp = np.zeros_like(gi) if inp["c_prev"] is None else inp["c_prev"]
    dc = inp["dc"]
    if mutant == "carry_read16":
        dc = dc.astype(np.float16).astype(f32)
    cc = inp["c_cur"].astype(np.float64)
    tcv = (np.tanh(cc) * (1 + rng.uniform(-2.0 ** -11, 2.0 ** -11, cc.shape))).astype(f32)
    keep = np.ones((dh.shape[0], 1), f32) if inp["mask"] is None else np.where(inp["mask"], 0, 1).astype(f32)[:, None]
    one = f32(1)
    dd = (dc + dh * go * (one - tcv * tcv)) * keep
    if mutant == "dd16":
        dd = dd.astype(np.float16).astype(f32)
    dhe = (dd if mutant == "do_from_dd" else dh) * keep
    out = [dd * gg * gi * (one - gi), dd * cp * gf * (one - gf), dhe * tcv * go * (one - go), dd * gi * (one - gg * gg)]
    dcn = dd * gf
    if mutant == "carry_store16":
        dcn = dcn.astype(np.float16).astype(f32)
    with np.errstate(over="ignore"):
        da = _f16_round(np.concatenate(out, 1), mutant).astype(np.float16)
    return da, dcn


def _inputs(regime):
    return make_inputs(H, R, regime, case_seed("bound-" + regime))


@pytest.mark.parametrize("regime", REGIMES)
def test_faithful_emulation_passes(regime):
    inp = _inputs(regime)
    da, dcn = emulate(inp, seed=1)
    res = check_step(inp, da, dcn, block=256)
    print("RATIO emulation %-10s da %.3g dc %.3g" % (regime, res["da"], res["dc"]))
    assert res["da"] <= 1 and res["dc"] <= 1, (regime, res)
    assert res["clamped"] > 0 if regime == "saturate" else res["clamped"] == 0, (regime, res)
    if regime == "subnormal":
        assert res["subnormals"] > 0 and res["flushed"] == 0, res


@pytest.mark.parametrize("mutant,regime", [(m, r) for m, rs in MUTANTS.items() for r in rs])
def test_mutant_fails(mutant, regime):
    inp = _inputs(regime)
    da, dcn = emulate(inp, mutant, seed=1)
    res = check_step(inp, da, dcn, block=256)
    print("RATIO %-14s %-10s da %.3g dc %.3g" % (mutant, regime, res["da"], res["dc"]))
    assert max(res["da"], res["dc"]) > 1, (mutant, regime, res)
