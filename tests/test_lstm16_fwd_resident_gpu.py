"""The fp16 option-LSTM forward step (lstm16.cu, k_lstm16<0>: a CTA-resident Wh column slice, two row-half pipelines that
take turns) through its test hook vd_lstm16_step_fwd.

Per case of tests/lstm16_fwd_cases.py: every output against the numpy step of tests/helpers.py at the tolerance of
test_lstm16_step_gpu.py; gates, c, h and the fp32 h bit for bit against tests/golden/lstm16_fwd_step.json, written by the
kernel this one replaced, which streamed both operands (same m64n128k16 instructions, operands and k order, so the same
bits); the guard rows past R untouched; and a second launch into the same buffers bitwise equal to the first.

Shapes: the benched one (R = 32 000, H = 512), H = 256, R = 1 024 (one row block per CTA of a slice), and R % 128 in
{1, 37, 64, 100}: the last block's second 64-row half empty, exactly empty or ragged."""
import json
import os

import numpy as np
import pytest

from helpers import lstm_step_fwd_ref, small_params
from lstm16_fwd_cases import CASES, GUARD, case_seed, digest, make_inputs, run_fwd
from visdial_b200 import Engine

pytestmark = pytest.mark.gpu

TOL = 4e-3
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lstm16_fwd_step.json")


@pytest.fixture(scope="module")
def eng():
    e = Engine(small_params("lf-ques", "disc"))
    yield e
    e.close()


@pytest.fixture(scope="module")
def golden():
    with open(GOLDEN) as f:
        return json.load(f)


def _close(name, got, ref):
    err = np.abs(np.asarray(got, np.float64) - ref) / (1.0 + np.abs(ref))
    assert np.isfinite(got).all(), name
    assert float(err.max()) < TOL and float(np.sqrt(np.mean(err ** 2))) < TOL / 4, (name, float(err.max()))


@pytest.mark.parametrize("name,H,R,with_c,save_gates,h32", CASES, ids=[c[0] for c in CASES])
def test_lstm16_fwd_resident(eng, golden, name, H, R, with_c, save_gates, h32):
    inp = make_inputs(H, R, with_c, case_seed(name))
    first, second = run_fwd(eng, H, R, inp, save_gates, h32, launches=2)
    assert set(first) == set(golden[name]), (name, sorted(first), sorted(golden[name]))

    for k, a in first.items():
        assert a.tobytes() == second[k].tobytes(), (name, k, "two launches differ")
        guard = a[R:].view(np.uint16 if a.dtype == np.float16 else np.uint32)
        assert guard.shape[0] == GUARD and (guard == guard.ravel()[0]).all() and np.isnan(a[R:]).all(), \
            (name, k, "rows past R written")

    z_x = inp["table"].astype(np.float64)[inp["tok"]] + inp["bias"]
    ref_g, ref_c, ref_h = lstm_step_fwd_ref(z_x, inp["h_prev"], inp["Wh"].astype(np.float64).T, inp["c_prev"], inp["mask"])
    if save_gates:
        _close("gates", first["g"][:R], ref_g)
    _close("c", first["c"][:R], ref_c)
    _close("h16", first["h16"][:R], ref_h)
    if h32:
        _close("h32", first["h32"][:R], ref_h)
        assert np.array_equal(first["h32"][:R].astype(np.float16), first["h16"][:R]), "h16 is not the rounded fp32 h"

    for k, a in first.items():
        assert digest(a, R) == golden[name][k], (name, k, "not bitwise equal to the shared-ring kernel's output")
