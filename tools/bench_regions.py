"""Region features (DESIGN §26) against the grid: ms per training step of `mn-att-ques-im-hist + disc` at B = 32 in
VD_MATH_F16 and VD_MATH_TF32 for three inputs, alternated round by round so that all three see the same machine:
  grid      the 14 x 14 pool5 grid, P = 196, C = 512 (no counts: the unmasked kernels)
  fixed36   36 region rows, C = 2048, no counts (the unmasked kernels at P = 36)
  adaptive  100 region rows, C = 2048, counts uniform in [10, 100] (the masked kernels)
  adaptive-unmasked  the same rows without counts (the unmasked kernels at P = 100: what skipping pad rows saves)
then one beam-search generate call (encoder forward + vd_gen_beam_search, beam 5) of `mn-att-ques-im-hist + gen` on D = 32
dialogs for each input.  Device-resident batches, device-event timing (vd_timer_start / vd_timer_stop).  Prints one JSON
line with the card's name and power limit, read in the same run.
usage: python tools/bench_regions.py [--steps 20] [--warmup 5] [--rounds 3]"""
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

INPUTS = {"grid": dict(imgFeatureSize=512, imgSpatialSize=14),
          "fixed36": dict(imgFeatureSize=2048, imgRegions=36),
          "adaptive": dict(imgFeatureSize=2048, imgRegions=100),
          "adaptive-unmasked": dict(imgFeatureSize=2048, imgRegions=100)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    if q.returncode != 0:
        raise SystemExit("nvidia-smi failed: this benchmark needs the GPU")
    return [s.strip() for s in q.stdout.splitlines()[0].split(",")]


def params(kind, dec):
    p = derive_flags(dict(DEFAULT_PARAMS, encoder="mn-att-ques-im-hist", decoder=dec, vocabSize=10000, batchSize=32,
                          **INPUTS[kind]))
    return p


def batch(p, kind, B, seed):
    nb = make_batch(p, B, seed=seed, gen_eval=False)
    if kind == "adaptive":
        nb["img_count"] = np.random.default_rng(seed).integers(10, 101, size=B).astype(np.int32)
    else:
        nb.pop("img_count", None)
    return nb


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    name, power = card()
    out = {"card": name, "power_limit": power, "B": 32, "train_ms": {}, "generate_ms": {}}
    for mode, mname in ((VD_MATH_F16, "f16"), (VD_MATH_TF32, "tf32")):
        engs = {}
        for kind in INPUTS:
            p = params(kind, "disc")
            e = Engine(p)
            e.set_math_mode(mode)
            e.set_parameters(init_parameters(p, seed=1))
            e.set_training(1)
            engs[kind] = (e, Batch(batch(p, kind, 32, 3)).to_device(e))
            for _ in range(a.warmup):
                e.zero_grad()
                e.forward_backward(engs[kind][1])
            e.synchronize()
        times = {k: [] for k in INPUTS}
        for _ in range(a.rounds):
            for kind, (e, b) in engs.items():
                e.timer_start()
                for _ in range(a.steps):
                    e.forward_backward(b)
                times[kind].append(e.timer_stop() / a.steps)
        out["train_ms"][mname] = {k: {"median": float(np.median(v)), "rounds": [round(x, 3) for x in v]} for k, v in times.items()}
        for e, _ in engs.values():
            e.close()
    for kind in INPUTS:
        p = params(kind, "gen")
        e = Engine(p)
        e.set_math_mode(VD_MATH_TF32)
        e.set_parameters(init_parameters(p, seed=2))
        e.set_training(0)
        b = Batch(batch(p, kind, 32, 4)).to_device(e)
        ms = []
        for i in range(1 + a.rounds):
            e.timer_start()
            e.encoder_forward(b)
            e.gen_beam_search(5, 20, p["vocabSize"] - 1, p["vocabSize"])
            t = e.timer_stop()
            if i:
                ms.append(t)
        out["generate_ms"][kind] = {"median": float(np.median(ms)), "rounds": [round(x, 3) for x in ms]}
        e.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
