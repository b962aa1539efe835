"""Cost of keeping the image features in pinned host memory (DESIGN §29) against keeping them on the device.

C4 (mn-att-ques-im-hist + disc, F16, V = 10 000, B = 32) over synthetic train and val splits of `--dialogs` dialogs, once
with pool5 grid features (196 x 512) and once with 100 detector regions of 2048 channels and per-image counts.  One model;
two dataloaders over the same arrays, one device-resident and one host-placed (its device budget set to 0 bytes), used
in alternation, `--rounds` times:
  - step:  `--steps` Model.trainIteration calls (each prefetching the next batch's rows), ended by a device synchronise;
  - val:   one validation pass over val (Validator.rank_lists, batches of 32, each prefetching the next);
  - batch: engine-stream events around one vd_corpus_get_batch of 32 random dialogs with nothing prefetched, so the
           engine stream waits for the copy engines' host-to-device copies (device placement: the gather kernels).
Medians per placement.  The card's name and power limit are printed in the same run.

    python tools/bench_host_images.py [--dialogs 1024] [--steps 20] [--rounds 3]"""
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
from visdial_b200 import VD_MATH_F16, Model  # noqa: E402
from visdial_b200 import dataloader as DL  # noqa: E402
from visdial_b200.synthetic import make_corpus  # noqa: E402
from visdial_b200.validation import Validator  # noqa: E402

B, V = 32, 10000
FEATURES = {"pool5": dict(imgFeatureSize=512), "regions100": dict(imgFeatureSize=2048, imgRegions=100)}


def _dataloader(m, p, data, host):
    real = DL.device_memory
    if host:
        DL.device_memory = lambda gpuid: 0
    try:
        dl = DL.Dataloader(m.engine, seed=1234).initialize(p, ["train", "val"], data)
    finally:
        DL.device_memory = real
    assert all(c.images_on_host == host for c in dl.corpus.values())
    return dl


def run(features, n, steps, rounds):
    p = full_params("mn-att-ques-im-hist", "disc", vocabSize=V, batchSize=B, **FEATURES[features])
    data = {s: make_corpus(p, num_threads=n, num_opt_list=8000, seed=5 + i) for i, s in enumerate(("train", "val"))}
    m = Model(p, seed=1234)
    m.engine.set_math_mode(VD_MATH_F16)
    dls = {"device": _dataloader(m, p, data, False), "host": _dataloader(m, p, data, True)}
    vals = {k: Validator(m, dl, {"savePath": ""}, 0, 1, lambda *a: None) for k, dl in dls.items()}
    rng = np.random.default_rng(0)
    for k, dl in dls.items():                                 # warm both: every shape the timed window uses
        for _ in range(3):
            m.trainIteration(dl)
        vals[k].rank_lists()
    res = {k: {"step_ms": [], "val_s": [], "batch_ms": []} for k in dls}
    for _ in range(rounds):
        for k, dl in dls.items():
            m.engine.synchronize()
            t = time.perf_counter()
            for _ in range(steps):
                m.trainIteration(dl)
            m.engine.synchronize()
            res[k]["step_ms"].append(1e3 * (time.perf_counter() - t) / steps)
            t = time.perf_counter()
            vals[k].rank_lists()
            m.engine.synchronize()
            res[k]["val_s"].append(time.perf_counter() - t)
            c = dl.corpus["train"]
            ms = []
            for _ in range(10):
                inds = rng.integers(0, n, size=B)
                m.engine.synchronize()
                m.engine.timer_start()
                c.get_batch(inds, 0)
                ms.append(m.engine.timer_stop())
            res[k]["batch_ms"].append(float(np.median(ms)))
    for dl in dls.values():
        dl.close()
    m.engine.close()
    row_bytes = int(np.prod(data["train"]["images"].shape[1:])) * 4
    out = {"features": features, "image_MB_per_batch": round(B * row_bytes / 1e6, 2)}
    for k in dls:
        out[k] = {name: round(float(np.median(v)), 4) for name, v in res[k].items()}
        out[k]["step_ms_all"] = [round(x, 3) for x in res[k]["step_ms"]]
    out["host_over_device_step"] = round(out["host"]["step_ms"] / out["device"]["step_ms"], 4)
    out["host_over_device_val"] = round(out["host"]["val_s"] / out["device"]["val_s"], 4)
    out["copy_GB_per_s"] = round(B * row_bytes / (out["host"]["batch_ms"] * 1e-3) / 1e9, 2)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dialogs", type=int, default=1024, help="dialogs (and images) of each synthetic split")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    print(json.dumps({"gpu": card[0] if card else None, "dialogs_per_split": a.dialogs, "batch": B, "V": V,
                      "math": "f16"}), flush=True)
    for features in FEATURES:
        print(json.dumps(run(features, a.dialogs, a.steps, a.rounds)), flush=True)


if __name__ == "__main__":
    main()
