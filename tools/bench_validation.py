"""Cost of validating while training (DESIGN §28): one `-valIter` pass over a val split next to one training epoch.

For C4 (mn-att-ques-im-hist + disc, pool5 14x14x512) and C3 (hrea-ques-im-hist + gen, fc7), V = 10000, 32 dialogs per
step, in F16 and TF32: a device dataloader over synthetic train and val splits of `--dialogs` dialogs each, one timed
training epoch (ceil(dialogs / 32) Model.trainIteration calls, ended by a device synchronise) and one timed validation
pass (Validator.rank_lists + the ground-truth ranks: every round's 100-option rank list, batches of 32).  The per-dialog
rates are also scaled to VisDial v0.9's split sizes (82 783 train, 40 504 val dialogs); those two columns are
extrapolations.  The card's name and power limit are printed in the same run.

    python tools/bench_validation.py [--dialogs 1024] [--repeats 2]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from helpers import full_params  # noqa: E402
from visdial_b200 import VD_MATH_F16, VD_MATH_TF32, Model  # noqa: E402
from visdial_b200.dataloader import Dataloader  # noqa: E402
from visdial_b200.synthetic import make_corpus  # noqa: E402
from visdial_b200.validation import Validator, gt_ranks  # noqa: E402

B, V = 32, 10000
CONFIGS = [("C4", "mn-att-ques-im-hist", "disc"), ("C3", "hrea-ques-im-hist", "gen")]
V09_TRAIN, V09_VAL = 82783, 40504


def run(enc, dec, math, n, repeats):
    p = full_params(enc, dec, vocabSize=V, batchSize=B)
    data = {s: make_corpus(p, num_threads=n, num_opt_list=8000, seed=5 + i) for i, s in enumerate(("train", "val"))}
    m = Model(p, seed=1234)
    m.engine.set_math_mode({"f16": VD_MATH_F16, "tf32": VD_MATH_TF32}[math])
    dl = Dataloader(m.engine, seed=1234).initialize(p, ["train", "val"], data)
    val = Validator(m, dl, {"savePath": ""}, 0, 1, lambda *a: None)
    answer = dl.corpus["val"].raw["ans_index"]
    steps = -(-n // B)
    for _ in range(5):
        m.trainIteration(dl)
    gt_ranks(val.rank_lists(), answer)                       # warm: the eval shapes' workspace
    epoch_s, pass_s = [], []
    for _ in range(repeats):
        m.engine.synchronize()
        t = time.perf_counter()
        for _ in range(steps):
            m.trainIteration(dl)
        m.engine.synchronize()
        epoch_s.append(time.perf_counter() - t)
        t = time.perf_counter()
        gt_ranks(val.rank_lists(), answer)                   # vd_retrieve ends each batch with a stream synchronise
        m.engine.synchronize()
        pass_s.append(time.perf_counter() - t)
    dl.close()
    m.engine.close()
    e, v = float(np.median(epoch_s)), float(np.median(pass_s))
    return {"epoch_s": round(e, 3), "val_pass_s": round(v, 3), "val_over_epoch": round(v / e, 3),
            "train_ms_per_dialog": round(1e3 * e / (steps * B), 4), "val_ms_per_dialog": round(1e3 * v / n, 4),
            "v09_epoch_s_extrapolated": round(e / (steps * B) * V09_TRAIN, 1),
            "v09_val_pass_s_extrapolated": round(v / n * V09_VAL, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dialogs", type=int, default=1024, help="dialogs of each synthetic split")
    ap.add_argument("--repeats", type=int, default=2)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    print(json.dumps({"gpu": card[0] if card else None, "dialogs_per_split": a.dialogs, "batch": B, "V": V}), flush=True)
    for name, enc, dec in CONFIGS:
        for math in ("f16", "tf32"):
            out = {"config": "%s %s + %s" % (name, enc, dec), "math": math}
            out.update(run(enc, dec, math, a.dialogs, a.repeats))
            print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
