"""Dialog pools (DESIGN §20), in one run, with the card's name and power limit read in the same run.
  (a) mixed    ms per ask of n conversations at n different rounds (slot i at round i % 5 when timing starts), against
      lockstep ms per ask of n conversations all at one round (a vd_dialog_begin session), alternated, n = 1, 8, 32, 128.
      gather_ms is the ask gather's device time per ask at n, from a separate profiled pass (CUDA events).
  (b) traffic  a seeded mix: --conversations conversations of 10 questions join at a steady rate (--join-rate per ask)
      into a pool of capacity 128; every ask answers each live conversation's next question.  Reports answers per
      second and asks per conversation (device calls between its join and its last answer), against serving the
      conversations one session at a time (one engine, one begin of one dialog each), timed on the first
      --serial conversations.
Gen decoder, beam 5 x 20, V = 10 000, default sizes (H = 512, E = 300).  Host clock around calls that end in a device
synchronisation; every shape is warmed up first; medians over --reps.  One JSON line per (encoder, mode, ...).
usage: python tools/bench_dialog_pool.py [--encoders a,b] [--modes f16,fp32] [--dialogs 1,8,32,128] [--reps 3]
                                         [--conversations 512] [--serial 32] [--out FILE]"""
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

BEAM, LEN, V, MAX_ANS, CAP, SPREAD, TIMED = 5, 20, 10000, 19, 128, 5, 5


def _rows(nb, ds):
    return {k: np.ascontiguousarray(v[ds]) for k, v in nb.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--encoders", default="hrea-ques-im-hist,mn-att-ques-im-hist,lf-ques-im-hist")
    ap.add_argument("--modes", default="f16,fp32")
    ap.add_argument("--dialogs", default="1,8,32,128")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--conversations", type=int, default=512)
    ap.add_argument("--join-rate", type=int, default=16)
    ap.add_argument("--serial", type=int, default=32)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power = card()
    rows = []

    def emit(row):
        row.update(gpu=name, power_limit=power)
        print(json.dumps(row), flush=True)
        rows.append(row)

    for enc in a.encoders.split(","):
        p = dict(DEFAULT_PARAMS)
        p.update(encoder=enc, decoder="gen", vocabSize=V, imgFeatureSize=512 if "att" in enc else 4096, batchSize=1)
        p = derive_flags(p)
        eng = Engine(p)
        flat = init_parameters(p, seed=3)
        split_parameters(p, flat)["dec.out.bias"][V - 1] += 4.0           # answers of realistic length, not all 20 words
        eng.set_parameters(flat)
        eng.set_training(0)
        nb = {k: v for k, v in make_batch(p, CAP, seed=7).items() if k in ("ques_fwd", "hist", "img_feat")}
        R, Tq = nb["ques_fwd"].shape[1:]
        W = max(300 if p["concatHistory"] else Tq + MAX_ANS, nb["hist"].shape[2])

        def ask(slots):
            rounds = eng.dialog_slots()
            q = np.stack([nb["ques_fwd"][s % CAP, rounds[s]] for s in slots])
            eng.dialog_ask_beam_slots(slots, q, BEAM, LEN, V - 1, V)

        for mode in a.modes.split(","):
            eng.set_math_mode({"f16": VD_MATH_F16, "fp32": VD_MATH_FP32}[mode])
            # ---- (a) mixed-round against lockstep asks of the same n
            for n in [int(x) for x in a.dialogs.split(",")]:
                batch = Batch(_rows(nb, list(range(n))))
                all_slots = list(range(n))

                def lockstep():
                    eng.dialog_begin(batch, W, MAX_ANS)
                    t = []
                    for r in range(TIMED):
                        t0 = time.perf_counter()
                        eng.dialog_ask_beam(nb["ques_fwd"][:n, r], BEAM, LEN, V - 1, V)
                        t.append(time.perf_counter() - t0)
                    return float(np.median(t))

                def mixed():
                    eng.dialog_open(n, Tq, W, MAX_ANS)
                    eng.dialog_join(batch)
                    for k in range(1, SPREAD):                       # slot i to round i % SPREAD
                        behind = [i for i in all_slots if i % SPREAD >= k]
                        if behind:
                            ask(behind)
                    t = []
                    for _ in range(TIMED):
                        t0 = time.perf_counter()
                        ask(all_slots)
                        t.append(time.perf_counter() - t0)
                    return float(np.median(t))

                lockstep(); mixed()                                  # warm-up of every shape
                ls, mx = [], []
                for _ in range(a.reps):
                    ls.append(lockstep())
                    mx.append(mixed())
                eng.profile(True)                                    # the gather's device time, in a pass of its own
                eng.dialog_open(n, Tq, W, MAX_ANS)
                eng.dialog_join(batch)
                eng.profile_reset()
                for _ in range(TIMED):
                    ask(all_slots)
                g = eng.kernel_stats("dialog_gather")
                eng.profile(False)
                emit({"bench": "mixed_vs_lockstep", "encoder": enc, "mode": mode, "n": n, "reps": a.reps,
                      "lockstep_ms_per_ask": round(1e3 * float(np.median(ls)), 3),
                      "mixed_ms_per_ask": round(1e3 * float(np.median(mx)), 3),
                      "gather_ms_per_ask": round(g["ms"] / TIMED, 4),
                      "gather_mb_per_ask": round(g["bytes"] / TIMED / 1e6, 2)})
            # ---- (b) the traffic mix against one session at a time
            rng = np.random.default_rng(13)
            order = rng.integers(0, CAP, a.conversations)            # each conversation: a dialog of the batch
            eng.dialog_open(CAP, Tq, W, MAX_ANS)
            live, joined, answers, asks, span = {}, 0, 0, 0, []
            t0 = time.perf_counter()
            while joined < a.conversations or live:
                k = min(a.join_rate, a.conversations - joined, CAP - len(live))
                if k > 0:
                    ds = order[joined:joined + k].tolist()
                    for s, d in zip(eng.dialog_join(Batch(_rows(nb, ds))).tolist(), ds):
                        live[s] = (d, asks)
                    joined += k
                slots = sorted(live)
                rounds = eng.dialog_slots()
                q = np.stack([nb["ques_fwd"][live[s][0], rounds[s]] for s in slots])
                eng.dialog_ask_beam_slots(slots, q, BEAM, LEN, V - 1, V)
                asks += 1
                answers += len(slots)
                done = [s for s in slots if rounds[s] + 1 == R]
                for s in done:
                    span.append(asks - live.pop(s)[1])
                if done:
                    eng.dialog_leave(done)
            pooled = time.perf_counter() - t0
            t0 = time.perf_counter()
            for d in order[:a.serial].tolist():
                eng.dialog_begin(Batch(_rows(nb, [d])), W, MAX_ANS)
                for r in range(R):
                    eng.dialog_ask_beam(nb["ques_fwd"][[d], r], BEAM, LEN, V - 1, V)
            serial = time.perf_counter() - t0
            emit({"bench": "traffic", "encoder": enc, "mode": mode, "conversations": a.conversations, "capacity": CAP,
                  "join_rate": a.join_rate, "asks": asks, "pool_answers_per_s": round(answers / pooled, 1),
                  "asks_per_conversation": round(float(np.mean(span)), 2),
                  "one_at_a_time_answers_per_s": round(a.serial * R / serial, 1), "one_at_a_time_measured_on": a.serial})
        eng.close()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
