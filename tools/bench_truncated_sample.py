"""Truncated sampling's cost (DESIGN §23): ms per call of vd_gen_sample (untruncated: the fused projection route where the
math mode and shape take it) and of vd_gen_truncated_sample at top-k 50, top-p 0.9 and both, on D dialogs' rounds (N =
10 D rows) of one encoder forward, at the default sizes with V = 10 000 and beam length 20, in the F16 and FP32 math
modes, for hrea-ques-im-hist and mn-att-ques-im-hist with the gen decoder.  The paths are warmed up at their shape and then
timed alternately, round after round, over whole calls (each follows an untimed encoder forward and ends in a device
synchronisation) until every path's timed calls add up to --window seconds.  The device time of the draw's class
(vd_kernel_stats truncated_sample for the truncated calls, vocab_sample + sample_rows for the untruncated one: CUDA
events around each step's projection and draw) comes from a separate profiled call.  Prints one JSON line per (encoder, mode, D,
path) with the card's name and power limit, read in the same run.
usage: python tools/bench_truncated_sample.py [--encoders E1,E2] [--modes f16,fp32] [--dialogs 1,8,32,128] [--window 1.0]
       [--out F]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from visdial_b200 import VD_MATH_F16, VD_MATH_FP32, init_parameters  # noqa: E402
from visdial_b200.engine import DEFAULT_PARAMS, Batch, Engine, derive_flags  # noqa: E402
from visdial_b200.synthetic import make_batch  # noqa: E402

LEN, V, T, SEED = 20, 10000, 1.0, 1234
PATHS = [("untruncated", 0, 1.0), ("k=50", 50, 1.0), ("p=0.9", 0, 0.9), ("k=50,p=0.9", 50, 0.9)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    if q.returncode != 0:
        raise SystemExit("nvidia-smi failed: this benchmark needs the GPU")
    return [s.strip() for s in q.stdout.splitlines()[0].split(",")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--encoders", default="hrea-ques-im-hist,mn-att-ques-im-hist")
    ap.add_argument("--modes", default="f16,fp32")
    ap.add_argument("--dialogs", default="1,8,32,128")
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power = card()
    out = open(a.out, "w") if a.out else None

    def emit(rec):
        line = json.dumps(dict(rec, card=name, power_limit=power))
        print(line, flush=True)
        if out:
            out.write(line + "\n")

    for enc in a.encoders.split(","):
        p = dict(DEFAULT_PARAMS, encoder=enc, decoder="gen", vocabSize=V)
        derive_flags(p)
        flat = init_parameters(p, seed=1)
        for mode in a.modes.split(","):
            eng = Engine(p)
            eng.set_math_mode({"f16": VD_MATH_F16, "fp32": VD_MATH_FP32}[mode])
            eng.set_training(0)
            eng.set_parameters(flat)
            for D in [int(x) for x in a.dialogs.split(",")]:
                batch = Batch(make_batch(p, D, seed=7)).to_device(eng)

                def forward():
                    eng.encoder_forward(batch)
                    eng.synchronize()

                def call(k, pp):
                    if k == 0 and pp == 1.0:
                        return eng.gen_sample(LEN, V - 1, T, SEED, 0)
                    return eng.gen_truncated_sample(LEN, V - 1, T, SEED, 0, k, pp)
                for _, k, pp in PATHS:                    # warm-up of every shape
                    forward()
                    call(k, pp)
                total, n = {x[0]: 0.0 for x in PATHS}, {x[0]: 0 for x in PATHS}
                while min(n.values()) < 2 or min(total.values()) < a.window:
                    for path, k, pp in PATHS:
                        forward()
                        t0 = time.perf_counter()
                        call(k, pp)
                        total[path] += time.perf_counter() - t0
                        n[path] += 1
                for path, k, pp in PATHS:
                    forward()
                    eng.profile(True)
                    eng.profile_reset()
                    call(k, pp)
                    # the untruncated call brackets its steps as vocab_sample (the fused route's attempt) and sample_rows
                    classes = ["truncated_sample"] if k or pp < 1.0 else ["vocab_sample", "sample_rows"]
                    st = [eng.kernel_stats(c) for c in classes]
                    eng.profile(False)
                    emit({"encoder": enc, "mode": mode, "dialogs": D, "rows": 10 * D, "path": path,
                          "ms_per_call": round(1e3 * total[path] / n[path], 3), "calls": n[path], "class": "+".join(classes),
                          "class_ms": round(sum(x["ms"] for x in st), 3), "class_launches": sum(x["launches"] for x in st)})
            eng.close()
    if out:
        out.close()


if __name__ == "__main__":
    main()
