"""The fp16 option-LSTM backward step (lstm16.cu, k_lstm16<1>) through its test hook vd_lstm16_step_bwd, per case of
tests/lstm16_bwd_cases.py:

* da and the cell-gradient carry, element by element, against fp64 within lstm16_bwd_cases.reference's bound: the fp32
  accumulation of exact fp16 products ((4H + 2) U S), bptt_bound's pointwise model (tanh.approx, fp32 products) and half an
  ulp of the fp16 store of da.  The worst err / bound of each is printed (pytest -s);
* masked rows of da and of the carry are exact zeros; the guard rows past R of both are bitwise untouched; every input,
  guard rows included, is bitwise unchanged; a second launch from the same carry gives the same bits;
* the sha-256 of rows 0 .. R-1 of da and of the carry equals tests/golden/lstm16_bwd_step.json: every output element comes
  from one tile, through the same m64n128k16 instructions in the same k order and the same fp32 epilogue expressions, so
  its bits do not depend on the tile schedule;
* saturate: no da is inf, and those whose reference is past 65 520 by more than their bound are exactly +-65504;
  subnormal: da holds nonzero fp16 subnormals, and none whose reference rounds to at least 2^-24 comes back as zero.

The cases' tile distribution over the device's SMs is printed too.  On an H100 the contraction stays within the
round-to-nearest term (lstm16_bwd_cases.CONTRACTION = 1)."""
import json
import os

import numpy as np
import pytest
import torch

from helpers import small_params
from lstm16_bwd_cases import CASES, GUARD, NAN16, case_seed, check_step, digest, make_inputs, run_bwd, tile_plan
from visdial_b200 import Engine

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lstm16_bwd_step.json")


@pytest.fixture(scope="module")
def eng():
    e = Engine(small_params("lf-ques", "disc"))
    yield e
    e.close()


@pytest.fixture(scope="module")
def golden():
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.mark.parametrize("name,H,R,kind", CASES, ids=[c[0] for c in CASES])
def test_lstm16_bwd_step(eng, golden, name, H, R, kind):
    tiles, grid, per = tile_plan(H, R, torch.cuda.get_device_properties(0).multi_processor_count)
    print("TILES %-10s H %d R %5d: %4d tiles on %3d CTAs, %s" % (name, H, R, tiles, grid,
          ", ".join("%d take %d" % (n, k) for k, n in sorted(per.items(), reverse=True))))
    inp = make_inputs(H, R, kind, case_seed(name))
    (first, second), ins = run_bwd(eng, H, R, inp, launches=2)

    for k, (sent, back) in ins.items():
        assert sent.tobytes() == back.tobytes(), (name, k, "an input was written")
    for k, a in first.items():
        assert a.tobytes() == second[k].tobytes(), (name, k, "two launches differ")
    guard_da = first["da"][R:].view(np.uint16)
    assert guard_da.shape[0] == GUARD and (guard_da == NAN16).all(), (name, "da rows past R written")
    assert np.isnan(first["dc"][R:]).all() and \
        (first["dc"][R:].view(np.uint32) == np.float32(np.nan).view(np.uint32)).all(), (name, "dc rows past R written")

    da, dc = first["da"][:R], first["dc"][:R]
    if inp["mask"] is not None:
        assert (da[inp["mask"]] == 0).all() and (dc[inp["mask"]] == 0).all(), (name, "masked rows must be exact zeros")

    res = check_step(inp, da, dc)
    print("RATIO %-10s da %.3g dc %.3g  (clamped %d, subnormal %d)" % (name, res["da"], res["dc"], res["clamped"],
                                                                       res["subnormals"]))
    assert res["da"] <= 1 and res["dc"] <= 1, (name, res)
    if kind == "saturate":
        assert not np.isinf(da).any() and res["clamped"] > 0, (name, res)
    else:
        assert res["clamped"] == 0, (name, res)
    if kind == "subnormal":
        assert res["subnormals"] > 0 and res["flushed"] == 0, (name, res)

    assert {"da": digest(da, R), "dc": digest(dc, R)} == golden[name], (name, "not bitwise equal to the pinned outputs")
