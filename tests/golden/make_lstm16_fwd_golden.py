"""Bit-exact fixture of the fp16 option-LSTM forward step (lstm16.cu, k_lstm16<0>): for every case of
tests/lstm16_fwd_cases.py, the sha-256 of the gates, c, h and fp32 h the step writes for rows 0 .. R-1 on the case's seeded
inputs.  tests/test_lstm16_fwd_resident_gpu.py checks the kernel against it, so a rewrite of the kernel that keeps the same
MMAs on the same operands in the same k order must reproduce these bits.

Written on an H100 by the forward kernel that streamed both operands (one 128 x 128 tile per CTA and round);
re-run (needs a GPU and a built library):  python tests/golden/make_lstm16_fwd_golden.py"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
sys.path.insert(0, os.path.join(HERE, ".."))

from helpers import small_params  # noqa: E402
from lstm16_fwd_cases import CASES, case_seed, digest, make_inputs, run_fwd  # noqa: E402
from visdial_b200 import Engine  # noqa: E402

OUT = os.path.join(HERE, "lstm16_fwd_step.json")


def main():
    eng = Engine(small_params("lf-ques", "disc"))
    fixture = {}
    try:
        for name, H, R, with_c, save_gates, h32 in CASES:
            inp = make_inputs(H, R, with_c, case_seed(name))
            got = run_fwd(eng, H, R, inp, save_gates, h32)[0]
            fixture[name] = {k: digest(a, R) for k, a in sorted(got.items())}
            print(name, fixture[name], flush=True)
    finally:
        eng.close()
    with open(sys.argv[1] if len(sys.argv) > 1 else OUT, "w") as f:
        json.dump(fixture, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
