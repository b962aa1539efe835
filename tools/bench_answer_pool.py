"""Answer-pool retrieval (DESIGN §18) on the benched graph C4 (`mn-att-ques-im-hist + disc`, V = 10 000, H = 512) against
a synthetic pool of m = 100 000 answers of width 20 (the real opt_list_val size is not known here).  Per math mode
(F16, TF32, FP32), all in one run:
  encode           vd_answer_pool_encode over the whole pool (device events around the call)
  retrieve/<d>     vd_answer_pool_retrieve, top-1, d dialogs per call: host wall time per dialog, launch overhead included
                   (every call ends in a device synchronisation), the encoder forward included
  encoder/<d>      the same call's encoder forward alone (vd_encoder_forward on the batch without its options, then a
                   synchronisation), per dialog
  topk/<d>         the scoring kernel alone (the pool_topk / pool_topk_simt class of vd_kernel_stats, device events): ms per
                   call, achieved TFLOP/s from 2 * rows * m * H, and its share of the 495 TFLOP/s TF32 data-sheet rate
Every path is warmed up at its shape first, then timed over whole calls for at least --window seconds.  Prints one JSON
line per (mode, path) and the card's name and power limit, read in the same run.
usage: python tools/bench_answer_pool.py [--modes f16,tf32,fp32] [--dpc 1,8,32,128] [--m 100000] [--window 1.0] [--out F]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from visdial_b200 import VD_MATH_F16, VD_MATH_FP32, VD_MATH_TF32, init_parameters  # noqa: E402
from visdial_b200.engine import DEFAULT_PARAMS, Batch, Engine, derive_flags  # noqa: E402
from visdial_b200.synthetic import make_batch  # noqa: E402

MODES = {"f16": VD_MATH_F16, "tf32": VD_MATH_TF32, "fp32": VD_MATH_FP32}
TF32_PEAK = 495e12          # H100 SXM data sheet, dense TF32
WIDTH = 20


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    except FileNotFoundError:
        q = None
    if q is None or q.returncode != 0:
        raise SystemExit("nvidia-smi failed: this benchmark needs the GPU")
    name, power = [s.strip() for s in q.stdout.splitlines()[0].split(",")]
    return name, power


def timed(fn, window):
    fn()                                                        # warm-up at this shape
    n, t0 = 0, time.perf_counter()
    while True:
        fn()
        n += 1
        dt = time.perf_counter() - t0
        if dt >= window:
            return dt / n, n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--modes", default="f16,tf32,fp32")
    ap.add_argument("--dpc", default="1,8,32,128")
    ap.add_argument("--m", type=int, default=100000)
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power = card()
    p = dict(DEFAULT_PARAMS)
    p.update(encoder="mn-att-ques-im-hist", decoder="disc", vocabSize=10000, imgFeatureSize=512)
    p = derive_flags(p)
    H = p["rnnHiddenSize"]
    rng = np.random.default_rng(0)
    lens = rng.integers(1, WIDTH + 1, a.m)
    pool = np.zeros((a.m, WIDTH), np.int32)
    for j in range(a.m):
        pool[j, :lens[j]] = rng.integers(1, p["vocabSize"] + 1, lens[j])
    eng = Engine(p)
    eng.set_parameters(init_parameters(p, seed=1))
    eng.set_training(0)
    batches, enc_only = {}, {}
    for d in map(int, a.dpc.split(",")):
        nb = make_batch(p, d, seed=d)
        batches[d] = Batch(nb).to_device(eng)
        # the encoder as the retrieval runs it: a batch with options would also start the N * 100-row option LSTM
        enc_only[d] = Batch({k: v for k, v in nb.items() if k != "options"}).to_device(eng)
    lines = []

    def emit(rec):
        rec.update(card=name, power_limit=power, m=a.m, width=WIDTH, H=H, V=p["vocabSize"])
        print(json.dumps(rec), flush=True)
        lines.append(rec)

    for mname in a.modes.split(","):
        eng.set_math_mode(MODES[mname])
        eng.answer_pool_encode(pool)                            # warm-up
        ms = []
        for _ in range(2):
            eng.timer_start()
            eng.answer_pool_encode(pool)
            ms.append(eng.timer_stop())
        emit({"mode": mname, "path": "encode", "ms": float(np.mean(ms))})
        for d, b in batches.items():
            t, n = timed(lambda: eng.answer_pool_retrieve(b, 1), a.window)
            emit({"mode": mname, "path": "retrieve/%d" % d, "ms_per_dialog": 1e3 * t / d, "calls": n})
            t, n = timed(lambda: (eng.encoder_forward(enc_only[d]), eng.synchronize()), a.window)
            emit({"mode": mname, "path": "encoder/%d" % d, "ms_per_dialog": 1e3 * t / d, "calls": n})
            eng.profile(True)
            eng.profile_reset()
            cls = "pool_topk_simt" if mname == "fp32" else "pool_topk"
            calls = 0
            t0 = time.perf_counter()
            while time.perf_counter() - t0 < a.window:
                eng.answer_pool_retrieve(b, 1)
                calls += 1
            st = eng.kernel_stats(cls)
            eng.profile(False)
            kms = st["ms"] / st["launches"]
            tflops = st["flops"] / (st["ms"] * 1e-3) / 1e12
            emit({"mode": mname, "path": "topk/%d" % d, "class": cls, "ms": kms, "tflops": tflops,
                  "tf32_peak_share": tflops * 1e12 / TF32_PEAK, "launches": st["launches"]})
    eng.close()
    if a.out:
        with open(a.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
