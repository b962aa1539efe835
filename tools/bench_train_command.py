"""QA-rounds/s of `python -m visdial_b200.train` against the same Model.trainIteration loop in-process, on C4-shaped synthetic
files (mn-att-ques-im-hist+disc, pool5 14x14x512, V = 10000, 32 dialogs per step).

The command's rate is taken from two runs that differ only in -numEpochs: the difference of their wall times covers the
extra iterations alone, so start-up, file reading, the corpus upload and the final checkpoint cancel out.  The in-process
rate times `--steps` trainIteration calls on a Dataloader over the same files, ended by a device synchronise.  Both arms
alternate `--repeats` times; the card's name and power limit are printed with the numbers.

    python tools/bench_train_command.py [--math f16] [--dialogs 512] [--steps 400] [--repeats 2]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from visdial_b200 import VD_MATH_F16, VD_MATH_FP32, VD_MATH_TF32, Model, h5lite  # noqa: E402
from visdial_b200.dataloader import Dataloader  # noqa: E402
from visdial_b200.engine import DEFAULT_PARAMS, derive_flags  # noqa: E402
from visdial_b200.synthetic import make_corpus  # noqa: E402

ENC, DEC, V, F, B = "mn-att-ques-im-hist", "disc", 10000, 512, 32


def write_files(d, n):
    p = derive_flags(dict(DEFAULT_PARAMS, encoder=ENC, decoder=DEC, vocabSize=V, imgFeatureSize=F))
    raw = make_corpus(p, num_threads=n, num_opt_list=8000, seed=99)
    h5lite.write(os.path.join(d, "data_img.h5"), {"images_train": raw.pop("images")})
    h5lite.write(os.path.join(d, "visdial_data.h5"), {k + "_train": np.asarray(v, np.uint32) for k, v in raw.items()})
    with open(os.path.join(d, "visdial_params.json"), "w") as f:
        json.dump({"word2ind": {"w%d" % i: i for i in range(1, V - 1)}}, f)
    files = {k: os.path.join(d, v) for k, v in (("inputJson", "visdial_params.json"), ("inputQues", "visdial_data.h5"),
                                                 ("inputImg", "data_img.h5"))}
    return p, files


def command_seconds(files, epochs, math, d):
    args = [sys.executable, "-m", "visdial_b200.train", "-encoder", ENC, "-decoder", DEC, "-imgFeatureSize", str(F),
            "-batchSize", str(B), "-numEpochs", str(epochs), "-saveIter", "0", "-math", math,
            "-savePath", os.path.join(d, "ck%d" % epochs)] + [x for k, v in files.items() for x in ("-" + k, v)]
    t = time.perf_counter()
    subprocess.run(args, cwd=ROOT, check=True, stdout=subprocess.DEVNULL)
    return time.perf_counter() - t


def inprocess_seconds(p, files, steps, math):
    m = Model(dict(p, batchSize=B), seed=1234)
    m.engine.set_math_mode({"f16": VD_MATH_F16, "tf32": VD_MATH_TF32, "fp32": VD_MATH_FP32}[math])
    dl = Dataloader(m.engine, seed=1234).initialize_from_files(dict(p, **files), ["train"])
    for _ in range(10):
        m.trainIteration(dl)
    m.engine.synchronize()
    t = time.perf_counter()
    for _ in range(steps):
        m.trainIteration(dl)
    m.engine.synchronize()
    sec = time.perf_counter() - t
    dl.close()
    m.engine.close()
    return sec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--math", default="f16", choices=["f16", "tf32", "fp32"])
    ap.add_argument("--dialogs", type=int, default=512, help="train split size (an epoch is dialogs / 32 iterations)")
    ap.add_argument("--steps", type=int, default=400, help="extra iterations of the long command run, and timed in-process steps")
    ap.add_argument("--repeats", type=int, default=2)
    a = ap.parse_args()
    per_epoch = -(-a.dialogs // B)
    short, long_ = 2, 2 + -(-a.steps // per_epoch)
    extra = (long_ - short) * per_epoch
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    with tempfile.TemporaryDirectory() as d:
        p, files = write_files(d, a.dialogs)
        cmd, inproc = [], []
        for _ in range(a.repeats):
            inproc.append(a.steps * B * 10 / inprocess_seconds(p, files, a.steps, a.math))
            dt = command_seconds(files, long_, a.math, d) - command_seconds(files, short, a.math, d)
            cmd.append(extra * B * 10 / dt)
    print(json.dumps({"workload": "train %s+%s, pool5 14x14x%d, V=%d, %d dialogs per step, math %s" % (ENC, DEC, F, V, B, a.math),
                      "unit": "QA-rounds/s", "train_command": [round(x, 1) for x in cmd],
                      "trainIteration_in_process": [round(x, 1) for x in inproc],
                      "command_extra_iterations": extra, "in_process_steps": a.steps, "gpu": card[0] if card else None}))


if __name__ == "__main__":
    main()
