"""Dialog sessions (DESIGN §19) against vd_gen_dialog_beam_search (§17) on the same batches, in one run, alternated.
  session  ms per ask at each round r = 0..9: vd_dialog_ask_beam on d dialogs, round r only over the cached state (host
           clock around the call, which ends in a device synchronisation)
  dialog   vd_gen_dialog_beam_search's call on the same d dialogs and questions, divided by the 10 rounds: its per-round
           share, which encodes all d*10 rounds at every round
Gen decoder, beam 5 x 20, V = 10 000, the default sizes (H = 512, E = 300); encoders hrea-ques-im-hist, mn-att-ques-im-hist
and lf-ques-im-hist; F16 and FP32; d = 1, 8, 32, 128 dialogs per session.  Every shape is warmed up with one whole session
and one call first; then --reps alternations of {one session of 10 asks, one call}.  Reports the median over the reps and
the card's name and power limit, read in the same run; one JSON line per (encoder, mode, d).
usage: python tools/bench_dialog_session.py [--encoders a,b] [--modes f16,fp32] [--dialogs 1,8,32,128] [--reps 5]
                                            [--out FILE]"""
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

BEAM, LEN, V, MAX_ANS = 5, 20, 10000, 19


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--encoders", default="hrea-ques-im-hist,mn-att-ques-im-hist,lf-ques-im-hist")
    ap.add_argument("--modes", default="f16,fp32")
    ap.add_argument("--dialogs", default="1,8,32,128")
    ap.add_argument("--reps", type=int, default=5)
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
        for mode in a.modes.split(","):
            eng.set_math_mode({"f16": VD_MATH_F16, "fp32": VD_MATH_FP32}[mode])
            for d in [int(x) for x in a.dialogs.split(",")]:
                nb = {k: v for k, v in make_batch(p, d, seed=7).items() if k in ("ques_fwd", "hist", "img_feat")}
                R, Tq = nb["ques_fwd"].shape[1:]
                W = 300 if p["concatHistory"] else Tq + MAX_ANS
                W = max(W, nb["hist"].shape[2])
                batch = Batch(nb)

                def session():
                    eng.dialog_begin(batch, W, MAX_ANS)
                    t = []
                    for r in range(R):
                        t0 = time.perf_counter()
                        eng.dialog_ask_beam(nb["ques_fwd"][:, r], BEAM, LEN, V - 1, V)
                        t.append(time.perf_counter() - t0)
                    return t

                def dialog():
                    t0 = time.perf_counter()
                    got = eng.gen_dialog_beam_search(batch, BEAM, LEN, V - 1, V, W, MAX_ANS)
                    return time.perf_counter() - t0, got

                session(); dialog()                                      # warm-up of every shape
                asks, calls = [], []
                for _ in range(a.reps):
                    asks.append(session())
                    t, want = dialog()
                    calls.append(t)
                same = bool(np.array_equal(eng.dialog_history(W), want[3]))   # same history rows as the call
                row = {"encoder": enc, "mode": mode, "dialogs": d, "reps": a.reps,
                       "session_ms_per_ask": [round(1e3 * float(np.median([x[r] for x in asks])), 3) for r in range(R)],
                       "dialog_ms_per_round": round(1e3 * float(np.median(calls)) / R, 3),
                       "same_history_as_dialog_call": same, "gpu": name, "power_limit": power}
                print(json.dumps(row), flush=True)
                rows.append(row)
        eng.close()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
