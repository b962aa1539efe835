"""Bit-exact fixture of the fp16 option-LSTM backward step (lstm16.cu, k_lstm16<1>): for every case of
tests/lstm16_bwd_cases.py, the sha-256 of the da (fp16) and the cell-gradient carry (fp32) the step writes for rows 0 .. R-1
on the case's seeded inputs.  tests/test_lstm16_bwd_step_gpu.py checks the kernel against it.

What the pin covers: the contraction dh = da_{t+1} Whb^T as m64n128k16 f16 wgmma instructions with fp32 accumulation, 16 k at a
time in increasing k order, and the epilogue's fp32 expressions in their order of operations (dd = (dc + dh o (1 - tc tc))
keep, the four gate gradients left to right, dd f), tanh.approx and the round-to-nearest saturating fp16 store.  Each output
element comes from one tile, so the tile schedule, the ring and the staging do not enter: a rewrite of those must reproduce
these bits.  A rewrite that changes the instructions, the k order or an epilogue expression must regenerate this fixture and
justify the change in its own commit.

Written on an H100 by the backward kernel whose consumer warpgroups share one 4-stage ring and both run their epilogue after
the tile's contraction; re-run (needs a GPU and a built library):  python tests/golden/make_lstm16_bwd_golden.py [out.json]"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
sys.path.insert(0, os.path.join(HERE, ".."))

from helpers import small_params  # noqa: E402
from lstm16_bwd_cases import CASES, case_seed, digest, make_inputs, run_bwd  # noqa: E402
from visdial_b200 import Engine  # noqa: E402

OUT = os.path.join(HERE, "lstm16_bwd_step.json")


def main():
    eng = Engine(small_params("lf-ques", "disc"))
    fixture = {}
    try:
        for name, H, R, kind in CASES:
            inp = make_inputs(H, R, kind, case_seed(name))
            got = run_bwd(eng, H, R, inp)[0][0]
            fixture[name] = {k: digest(a, R) for k, a in sorted(got.items())}
            print(name, fixture[name], flush=True)
    finally:
        eng.close()
    with open(sys.argv[1] if len(sys.argv) > 1 else OUT, "w") as f:
        json.dump(fixture, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
