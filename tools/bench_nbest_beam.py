"""n-best lists' cost (DESIGN §24): ms per call of vd_gen_nbest_beam_search at beam_size k = 10 with (nbest, length
penalty) in (1, 0.7), (5, 0.7) and (32, 0.7), against vd_gen_beam_search at k = 10, on D dialogs' rounds (N = 10 D
searches) of one encoder forward, hrea-ques-im-hist and mn-att-ques-im-hist + gen at the default sizes, V = 10 000, beam
length 20, in the F16 and FP32 math modes.  The paths are alternated: each repetition times every path once, over whole
calls (each ends in a device synchronisation and follows an untimed encoder forward) until the timed calls add up to
--window seconds, and a path's figure is the median over the repetitions, with the spread (max - min).  The merge's
device time per call (vd_kernel_stats class beam_merge, CUDA events around each launch) is read in a separate profiled
call.  Prints one JSON line per (encoder, mode, D, path) and the card's name and power limit, read in the same run.
usage: python tools/bench_nbest_beam.py [--encoders a,b] [--modes f16,fp32] [--dialogs 1,32,128] [--reps 5] [--window 0.5]
       [--out F]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from visdial_b200 import VD_MATH_F16, VD_MATH_FP32, init_parameters  # noqa: E402
from visdial_b200.engine import DEFAULT_PARAMS, Batch, Engine, derive_flags  # noqa: E402
from visdial_b200.synthetic import make_batch  # noqa: E402

K, LEN, V = 10, 20, 10000
LISTS = [(1, 0.7), (5, 0.7), (32, 0.7)]


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
    ap.add_argument("--encoders", default="hrea-ques-im-hist,mn-att-ques-im-hist")
    ap.add_argument("--modes", default="f16,fp32")
    ap.add_argument("--dialogs", default="1,32,128")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--window", type=float, default=0.5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power = card()
    out = open(a.out, "w") if a.out else None

    def emit(rec):
        line = json.dumps(dict(rec, card=name, power_limit=power))
        print(line, flush=True)
        if out:
            out.write(line + "\n")

    start, end = V - 1, V
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
                paths = [("beam/k=%d" % K, lambda: eng.gen_beam_search(K, LEN, start, end))]
                for nb, alpha in LISTS:
                    paths.append(("nbest/k=%d,n=%d,alpha=%g" % (K, nb, alpha),
                                  lambda nb=nb, alpha=alpha: eng.gen_nbest_beam_search(K, 1, 0.0, alpha, nb, LEN, start, end)))
                times = {path: [] for path, _ in paths}
                for _ in range(a.reps):
                    for path, call in paths:
                        times[path].append(timed(forward, call, a.window))
                for path, call in paths:
                    forward()
                    eng.profile(True)
                    eng.profile_reset()
                    call()
                    merge = eng.kernel_stats("beam_merge")
                    eng.profile(False)
                    t = times[path]
                    emit({"encoder": enc, "mode": mode, "dialogs": D, "searches": 10 * D, "path": path,
                          "ms_per_call": round(statistics.median(t), 3), "spread_ms": round(max(t) - min(t), 3),
                          "merge_ms": round(merge["ms"], 3), "merge_launches": merge["launches"]})
            eng.close()
    if out:
        out.close()


if __name__ == "__main__":
    main()
