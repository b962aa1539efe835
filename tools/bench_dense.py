"""The dense fine-tuning step against the standard training step on the same batches, device-resident, B = 32 dialogs.
Both steps are warmed up at their shapes, then timed with device events (vd_timer_start / vd_timer_stop) over --steps
steps each, alternating the two in --rounds rounds so that both see the same machine.  Prints one JSON line with the
card's name and power limit, read in the same run.

--decoder disc (default): vd_forward_backward_dense against vd_forward_backward on C4's graph (`mn-att-ques-im-hist +
  disc`, pool5 14x14x512, 10 rounds, 100 options x 20 tokens, V = 10000) in VD_MATH_F16.  Also reports the option-LSTM
  step class's rows of work per step (profiling counts, a separate pass).
--decoder gen: vd_forward_backward_dense_gen against the standard gen step on `mn-att-ques-im-hist + gen` (V = 10000,
  option_in / option_out batches) in VD_MATH_F16 and VD_MATH_TF32.  Also reports, from a profiled pass, the time of the
  fused vocabulary classes (vocab_lse, vocab_dlogits) and the four vocabulary passes' algorithmic FLOPs per step.
usage: python tools/bench_dense.py [--decoder disc|gen] [--batch 32] [--steps 20] [--warmup 5] [--rounds 3]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from visdial_b200 import VD_MATH_F16, VD_MATH_TF32, Batch, Engine, init_parameters  # noqa: E402
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


def timed(eng, steps, batches, args):
    """Warm-up, then --rounds rounds of --steps steps of each kind, alternating: ms per step of each kind per round."""
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
    return ms, run


def main_gen(args, name, power):
    p = derive_flags(dict(DEFAULT_PARAMS, encoder="mn-att-ques-im-hist", decoder="gen", vocabSize=10000, imgFeatureSize=512))
    B, K, R, H, V = args.batch, p["numOptions"], p["maxQuesCount"], p["rnnHiddenSize"], p["vocabSize"]
    out = {"card": name, "power_limit": power, "workload": "mn-att-ques-im-hist+gen, V=%d, B=%d" % (V, B), "modes": {}}
    for mode, mname in ((VD_MATH_F16, "f16"), (VD_MATH_TF32, "tf32")):
        eng = Engine(p)
        eng.set_math_mode(mode)
        eng.set_parameters(init_parameters(p, seed=3))
        eng.set_training(1)
        rng = np.random.default_rng(5)
        batches = []
        for i in range(2):
            b = Batch(make_batch(p, B, seed=1234 + i, gen_eval=True)).to_device(eng)
            rel = rng.choice([0.0, 0.0, 0.0, 0.5, 1.0], size=(B, K)).astype(np.float32)
            rel[:, 0] = 1.0
            batches.append((b, rng.integers(0, R, size=B).astype(np.int32), rel))
        To = batches[0][0].c.To
        steps = {"standard": lambda x: eng.forward_backward(x[0]), "dense": lambda x: eng.forward_backward_dense_gen(*x)}
        ms, run = timed(eng, steps, batches, args)
        eng.profile(True)
        eng.profile_reset()
        run("dense", 1, 0)
        eng.synchronize()
        vocab = {k: round(eng.kernel_stats(k)["ms"], 3) for k in ("vocab_lse", "vocab_dlogits")}
        eng.profile(False)
        eng.close()
        out["modes"][mname] = {
            "ms_per_step": {k: round(float(np.median(v)), 3) for k, v in ms.items()},
            "ms_per_step_rounds": {k: [round(x, 3) for x in v] for k, v in ms.items()},
            "dense_over_standard": round(float(np.median(ms["dense"]) / np.median(ms["standard"])), 2),
            "dense_vocab_ms_profiled": vocab, "To": To}
    # forward statistics, d-logit recompute, dec.out's dW and dh: four (To*B*K, V, H) contractions
    out["dense_vocab_tflop_per_step"] = round(4 * 2.0 * To * B * K * V * H / 1e12, 3)
    print(json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--decoder", choices=("disc", "gen"), default="disc")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    name, power = card()
    if args.decoder == "gen":
        return main_gen(args, name, power)
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
