"""The dense fine-tuning step (vd_forward_backward_dense) against the standard training step (vd_forward_backward) on the
same batches: C4's graph (`mn-att-ques-im-hist + disc`, pool5 14x14x512, 10 rounds, 100 options x 20 tokens, V = 10000),
B = 32 dialogs, VD_MATH_F16, device-resident batches.  Both steps are warmed up at their shapes, then timed with device
events (vd_timer_start / vd_timer_stop) over --steps steps each, alternating the two in --rounds rounds so that both see
the same machine.  Also reports the option-LSTM step class's rows of work per step (profiling counts, a separate pass).
Prints one JSON line with the card's name and power limit, read in the same run.
usage: python tools/bench_dense.py [--batch 32] [--steps 20] [--warmup 5] [--rounds 3]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from visdial_b200 import VD_MATH_F16, Batch, Engine, init_parameters  # noqa: E402
from visdial_b200.engine import DEFAULT_PARAMS, derive_flags  # noqa: E402
from visdial_b200.synthetic import make_batch  # noqa: E402


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
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    name, power = card()
    p = derive_flags(dict(DEFAULT_PARAMS, encoder="mn-att-ques-im-hist", decoder="disc", vocabSize=10000, imgFeatureSize=512))
    B, K, R = args.batch, p["numOptions"], p["maxQuesCount"]
    eng = Engine(p)
    eng.set_math_mode(VD_MATH_F16)
    eng.set_parameters(init_parameters(p, seed=3))
    eng.set_training(1)
    rng = np.random.default_rng(5)
    batches = []
    for i in range(2):
        b = Batch(make_batch(p, B, seed=1234 + i)).to_device(eng)
        rel = rng.choice([0.0, 0.0, 0.0, 0.5, 1.0], size=(B, K)).astype(np.float32)
        rel[:, 0] = 1.0
        batches.append((b, rng.integers(0, R, size=B).astype(np.int32), rel))
    steps = {"standard": lambda x: eng.forward_backward(x[0]), "dense": lambda x: eng.forward_backward_dense(*x)}

    def run(kind, n, it0):
        for i in range(n):
            eng.zero_grad()
            eng.set_dropout_seed(1234, it0 + i)
            steps[kind](batches[i % 2])

    for kind in steps:
        run(kind, args.warmup, 0)
    ms = {k: [] for k in steps}
    for r in range(args.rounds):
        for kind in steps:
            eng.synchronize()
            eng.timer_start()
            run(kind, args.steps, 1000 * (r + 1))
            eng.synchronize()
            ms[kind].append(eng.timer_stop() / args.steps)
    rows = {}
    eng.profile(True)
    for kind in steps:
        eng.profile_reset()
        run(kind, 1, 0)
        eng.synchronize()
        st = eng.kernel_stats("lstm_step")
        To = batches[0][0].c.To
        rows[kind] = st["flops"] / ((To - 1) * 2.0 * 4 * p["rnnHiddenSize"] ** 2)
    eng.close()
    out = {"card": name, "power_limit": power, "workload": "C4 mn-att-ques-im-hist+disc, B=%d, VD_MATH_F16" % B,
           "ms_per_step": {k: round(float(np.median(v)), 3) for k, v in ms.items()},
           "ms_per_step_rounds": {k: [round(x, 3) for x in v] for k, v in ms.items()},
           "speedup": round(float(np.median(ms["standard"]) / np.median(ms["dense"])), 2),
           "option_lstm_rows_per_step": rows}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
