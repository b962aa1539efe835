"""What deterministic training costs (vd_set_deterministic, DESIGN §27): the training step (zero_grad, forward_backward,
clamp_adam_step) of bench.py's configs C1-C4 in VD_MATH_F16, TF32 and FP32, default routes against deterministic ones on
one engine and one device-resident batch.  Both are warmed up, then timed with device events (vd_timer_start / _stop) over
--steps steps each, alternating the two in --rounds rounds so that both see the same machine.  C5 is C4's graph in an
evaluation step, which has no gradient reductions.  Prints one JSON line per (config, mode) with the card's name and power
limit, read in the same run.
usage: python tools/bench_deterministic.py [--configs C1,C2,C3,C4] [--modes f16,tf32,fp32] [--steps 10] [--warmup 3] [--rounds 3]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import CONFIGS, config_params  # noqa: E402
from visdial_b200 import VD_MATH_F16, VD_MATH_FP32, VD_MATH_TF32, Batch, Engine, init_parameters  # noqa: E402
from visdial_b200.synthetic import make_batch  # noqa: E402

MODES = {"f16": VD_MATH_F16, "tf32": VD_MATH_TF32, "fp32": VD_MATH_FP32}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    except FileNotFoundError:
        q = None
    if q is None or q.returncode != 0:
        raise SystemExit("nvidia-smi failed: this benchmark needs the GPU")
    name, power = [s.strip() for s in q.stdout.splitlines()[0].split(",")]
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="C1,C2,C3,C4")
    ap.add_argument("--modes", default="f16,tf32,fp32")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    name, power = card()
    for cfg in args.configs.split(","):
        c = CONFIGS[cfg]
        p = config_params(cfg)
        nb = make_batch(p, c["batch"], seed=3)
        for mode in args.modes.split(","):
            eng = Engine(p)
            eng.set_math_mode(MODES[mode])
            eng.set_parameters(init_parameters(p, seed=1))
            eng.set_training(1)
            b = Batch(nb).to_device(eng)

            def step():
                eng.zero_grad()
                eng.forward_backward(b)
                eng.clamp_adam_step(1e-3)

            def timed(det, n):
                eng.set_deterministic(det)
                eng.synchronize()
                eng.timer_start()
                for _ in range(n):
                    step()
                return eng.timer_stop() / n

            for det in (False, True):
                timed(det, args.warmup)
            ms = {False: [], True: []}
            for _ in range(args.rounds):
                for det in (False, True):
                    ms[det].append(timed(det, args.steps))
            eng.close()
            d, t = float(np.median(ms[False])), float(np.median(ms[True]))
            print(json.dumps({"config": cfg, "math": mode, "batch": c["batch"], "default_ms": [round(x, 3) for x in ms[False]],
                              "deterministic_ms": [round(x, 3) for x in ms[True]], "ratio_median": round(t / d, 3),
                              "card": name, "power_limit": power}), flush=True)


if __name__ == "__main__":
    main()
