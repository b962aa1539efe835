"""The answer rules' cost (DESIGN §25): ms per call with the rules off and with minWords 2, noRepeatNgram 2 and <UNK>
(a word id of the vocabulary standing in for it) banned, on five paths: beam search at k = 10, diverse beam search
(k = 10, G = 2), n-best lists (k = 10, n = 5, alpha = 0.7), untruncated sampling and top-p 0.9 sampling, on D dialogs'
rounds (N = 10 D rows) of one encoder forward, hrea-ques-im-hist + gen at the default sizes, V = 10 000, length 20, in the
F16 and FP32 math modes.  Rules off and on are alternated: each repetition times every (path, rules) pair once over whole
calls (each ends in a device synchronisation and follows an untimed encoder forward) until the timed calls add up to
--window seconds; a figure is the median over the repetitions, with the spread.  The step classes' device time per call
(vd_kernel_stats: beam_merge for the searches; vocab_sample + sample_rows or truncated_sample for sampling) is read in a
separate profiled call.  Prints one JSON line per (mode, D, path, rules) and the card's name and power limit, read in
the same run.
usage: python tools/bench_answer_rules.py [--encoders a] [--modes f16,fp32] [--dialogs 1,32,128] [--reps 5] [--window 0.5]
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
UNK = 1                      # the synthetic vocabulary has no words: any id stands for <UNK>
RULES = dict(min_words=2, no_repeat_ngram=2, banned=[UNK])
CLASSES = {"beam": ["beam_merge"], "sample": ["vocab_sample", "sample_rows", "truncated_sample"]}


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
    ap.add_argument("--encoders", default="hrea-ques-im-hist")
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
                paths = [("beam/k=%d" % K, "beam", lambda: eng.gen_beam_search(K, LEN, start, end)),
                         ("diverse/k=%d,G=2" % K, "beam", lambda: eng.gen_diverse_beam_search(K, 2, 0.5, LEN, start, end)),
                         ("nbest/k=%d,n=5,alpha=0.7" % K, "beam",
                          lambda: eng.gen_nbest_beam_search(K, 1, 0.0, 0.7, 5, LEN, start, end)),
                         ("sample", "sample", lambda: eng.gen_sample(LEN, start, 1.0, 1234, 0)),
                         ("sample/topP=0.9", "sample", lambda: eng.gen_truncated_sample(LEN, start, 1.0, 1234, 0, 0, 0.9))]

                def ruled(call, on):
                    def f():
                        if on:
                            eng.set_answer_rules(**RULES)
                        try:
                            call()
                        finally:
                            if on:
                                eng.set_answer_rules()
                    return f
                runs = [(path, cls, on, ruled(call, on)) for path, cls, call in paths for on in (False, True)]
                times = {(path, on): [] for path, _, on, _ in runs}
                for _ in range(a.reps):
                    for path, _, on, call in runs:
                        times[path, on].append(timed(forward, call, a.window))
                for path, cls, on, call in runs:
                    forward()
                    eng.profile(True)
                    eng.profile_reset()
                    call()
                    st = [eng.kernel_stats(c) for c in CLASSES[cls]]
                    eng.profile(False)
                    t = times[path, on]
                    emit({"encoder": enc, "mode": mode, "dialogs": D, "rows": 10 * D, "path": path, "rules": on,
                          "ms_per_call": round(statistics.median(t), 3), "spread_ms": round(max(t) - min(t), 3),
                          "class_ms": round(sum(x["ms"] for x in st), 3), "class_launches": sum(x["launches"] for x in st)})
            eng.close()
    if out:
        out.close()


if __name__ == "__main__":
    main()
