"""Diverse beam search's cost (DESIGN §22): ms per call of vd_gen_diverse_beam_search at beam_size k = 10 in G groups, and
of vd_gen_beam_search at k = 10 and at k = w = 10 / G, on D dialogs' rounds (N = 10 D searches) of one encoder forward,
hrea-ques-im-hist + gen at the default sizes, V = 10 000, beam length 20, in the F16 and FP32 math modes.  The merge's
share is the merge's time (vd_kernel_stats class beam_merge, CUDA events around each launch) over the call's wall time
in a separate profiled call.  Every path is warmed up at its shape, then timed over whole calls (each ends in a device
synchronisation, and follows an untimed encoder forward) until the timed calls add up to --window seconds.  Prints one JSON line per (mode, D, path) and the card's name and power limit,
read in the same run.
usage: python tools/bench_diverse_beam.py [--modes f16,fp32] [--dialogs 1,32,128] [--groups 2,5] [--window 1.0] [--out F]"""
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

K, LEN, V, ENC = 10, 20, 10000, "hrea-ques-im-hist"


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    if q.returncode != 0:
        raise SystemExit("nvidia-smi failed: this benchmark needs the GPU")
    return [s.strip() for s in q.stdout.splitlines()[0].split(",")]


def timed(forward, call, seconds):
    """ms per search call, after one warm-up call of the same shape.  Each call follows an encoder forward, outside the
    timed region, as in generateAnswers: a search's buffers live in the activation arena until the next forward."""
    forward()
    call()
    n, total = 0, 0.0
    while n < 2 or total < seconds:
        forward()
        t0 = time.perf_counter()
        call()
        total += time.perf_counter() - t0
        n += 1
    return 1e3 * total / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--modes", default="f16,fp32")
    ap.add_argument("--dialogs", default="1,32,128")
    ap.add_argument("--groups", default="2,5")
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

    p = dict(DEFAULT_PARAMS, encoder=ENC, decoder="gen", vocabSize=V)
    derive_flags(p)
    flat = init_parameters(p, seed=1)
    start, end = V - 1, V
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
            paths = [("beam/k=%d" % K, K, 1)]
            for G in [int(x) for x in a.groups.split(",")]:
                paths += [("diverse/k=%d,G=%d" % (K, G), K, G), ("beam/k=%d" % (K // G), K // G, 1)]
            seen = set()
            for path, k, G in paths:
                if path in seen:
                    continue
                seen.add(path)
                if G > 1:
                    call = lambda: eng.gen_diverse_beam_search(k, G, 0.5, LEN, start, end)  # noqa: E731
                else:
                    call = lambda: eng.gen_beam_search(k, LEN, start, end)  # noqa: E731
                ms = timed(forward, call, a.window)
                forward()
                eng.profile(True)
                eng.profile_reset()
                t0 = time.perf_counter()
                call()
                wall = 1e3 * (time.perf_counter() - t0)
                merge = eng.kernel_stats("beam_merge")
                eng.profile(False)
                emit({"mode": mode, "dialogs": D, "searches": 10 * D, "path": path, "ms_per_call": round(ms, 3),
                      "merge_ms": round(merge["ms"], 3), "merge_launches": merge["launches"],
                      "merge_share": round(merge["ms"] / wall, 4)})
        eng.close()
    if out:
        out.close()


if __name__ == "__main__":
    main()
