"""Resuming conversations in a dialog pool (DESIGN §21), in one run, with the card's name and power limit read in the same
run.  For n conversations resumed at round r (n = 1, 8, 32, 128; r = 1, 5, 9), alternated, medians over --reps:
  join_rounds  ms of one vd_dialog_join_rounds of the n conversations at round r (their rounds 0..r-1 in one encoder pass);
  ask          ms of one beam ask of n conversations at round 0 (a join, then the timed ask);
  replay       ms of what join_rounds replaces: a join at round 0 and r beam asks.  The asks also decode and append
               their own answers, so this is an upper bound on replaying given answers.
Gen decoder, beam 5 x 20, V = 10 000, default sizes (H = 512, E = 300).  Host clock around calls that end in a device
synchronisation; every shape is warmed up first.  One JSON line per (encoder, mode, n, r).
usage: python tools/bench_dialog_resume.py [--encoders a,b] [--modes f16,fp32] [--dialogs 1,8,32,128] [--rounds 1,5,9]
                                           [--reps 3] [--out FILE]"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_generate import card  # noqa: E402
from visdial_b200 import VD_MATH_F16, VD_MATH_FP32, init_parameters  # noqa: E402
from visdial_b200.engine import DEFAULT_PARAMS, Batch, Engine, derive_flags, split_parameters  # noqa: E402
from visdial_b200.synthetic import make_batch  # noqa: E402

BEAM, LEN, V, MAX_ANS, CAP = 5, 20, 10000, 19, 128


def _rows(nb, ds):
    return {k: np.ascontiguousarray(v[ds]) for k, v in nb.items() if k in ("ques_fwd", "hist", "img_feat")}


def _timed(fn):
    t0 = time.perf_counter()
    fn()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--encoders", default="hrea-ques-im-hist,mn-att-ques-im-hist,lf-ques-im-hist")
    ap.add_argument("--modes", default="f16,fp32")
    ap.add_argument("--dialogs", default="1,8,32,128")
    ap.add_argument("--rounds", default="1,5,9")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power = card()
    rows = []
    for enc in a.encoders.split(","):
        p = dict(DEFAULT_PARAMS)
        p.update(encoder=enc, decoder="gen", vocabSize=V, imgFeatureSize=512 if "att" in enc else 4096, batchSize=1)
        p = derive_flags(p)
        eng = Engine(p)
        flat = init_parameters(p, seed=3)
        split_parameters(p, flat)["dec.out.bias"][V - 1] += 4.0           # answers of realistic length, not all 20 words
        eng.set_parameters(flat)
        eng.set_training(0)
        nb = make_batch(p, CAP, seed=7)
        R, Tq = nb["ques_fwd"].shape[1:]
        W = max(300 if p["concatHistory"] else Tq + MAX_ANS, nb["hist"].shape[2])
        for mode in a.modes.split(","):
            eng.set_math_mode({"f16": VD_MATH_F16, "fp32": VD_MATH_FP32}[mode])
            for n in [int(x) for x in a.dialogs.split(",")]:
                ds = list(range(n))
                batch = Batch(_rows(nb, ds))
                answers = np.ascontiguousarray(nb["answer_out"][ds])     # the dialogs' own answers, <END>-terminated

                def ask(r):
                    eng.dialog_ask_beam_slots(ds, nb["ques_fwd"][:n, r], BEAM, LEN, V - 1, V)

                def one_ask():
                    eng.dialog_open(n, Tq, W, MAX_ANS)
                    eng.dialog_join(batch)
                    return _timed(lambda: ask(0))

                for r in [int(x) for x in a.rounds.split(",")]:
                    def resume():
                        eng.dialog_open(n, Tq, W, MAX_ANS)
                        return _timed(lambda: eng.dialog_join_rounds(batch, np.full(n, r, np.int32), answers, ds))

                    def replay():
                        eng.dialog_open(n, Tq, W, MAX_ANS)
                        return _timed(lambda: (eng.dialog_join(batch), [ask(t) for t in range(r)]))

                    resume(); one_ask(); replay()                 # warm-up of every shape
                    t = {"join_rounds": [], "ask": [], "replay": []}
                    for _ in range(a.reps):
                        t["join_rounds"].append(resume())
                        t["ask"].append(one_ask())
                        t["replay"].append(replay())
                    ms = {k: 1e3 * float(np.median(v)) for k, v in t.items()}
                    row = {"bench": "dialog_resume", "encoder": enc, "mode": mode, "n": n, "r": r, "reps": a.reps,
                           "join_rounds_ms": round(ms["join_rounds"], 3), "ask_ms": round(ms["ask"], 3),
                           "replay_ms": round(ms["replay"], 3),
                           "replay_over_join_rounds": round(ms["replay"] / ms["join_rounds"], 2),
                           "gpu": name, "power_limit": power}
                    print(json.dumps(row), flush=True)
                    rows.append(row)
        eng.close()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
