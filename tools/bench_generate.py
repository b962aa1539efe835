"""Model:generateAnswers (model.lua:432-613) wall time per dialog: beam search (beamSize 5, beamLen 20) or sampling (beamLen
20, sampleWords = 1) over the 10 rounds of each dialog, V = 10 000, for `hrea-ques-im-hist + gen` (C3's graph) and
`mn-att-ques-im-hist + gen`, in the F16 and FP32 math modes.  Paths, all in one run:
  device/<d>   beam search, the default: vd_gen_beam_search, d dialogs per encoder forward and call (params.dialogsPerCall)
  host_search  the tests' host reference search (tests/host_decode.py::host_beam_search), per dialog: the state and
               log-probabilities through the host at every vd_gen_decoder_step, the top-k and the candidate merge on the host
  sample/<d>   sampling: vd_gen_sample, d dialogs per encoder forward and call
  host_sample  sampling as the engine ran it before it moved to the device: per dialog and step, the state up, one
               vd_gen_decoder_step, the log-probabilities and state down, one numpy categorical draw per round (host_sample)
Dialogs on the model's own answers (history "generated", DESIGN §17; kinds dialog-beam, dialog-sample; history encoders):
  dialog/<d>         vd_gen_dialog_beam_search, d dialogs per call
  host_dialog/<d>    the loop a user would otherwise write: per round, the history rebuilt on the host, the batch uploaded,
                     the encoder forward and vd_gen_beam_search over all the batch's rounds, one round kept (10 calls)
  enc/<d>            the device loop's 10 encoder forwards alone (same batch and history width), for the encoder's share
  dsample/<d>        vd_gen_dialog_sample, d dialogs per call
  host_dsample/<d>   the host loop with vd_gen_sample
Every path is warmed up at its shape first, then timed over whole calls until the window lasts at least --window seconds
(host clock; every call ends in a device synchronisation).  Prints one JSON line per (encoder, mode, path) and the card's name
and power limit, read in the same run.
usage: python tools/bench_generate.py [--encoders a,b] [--modes f16,fp32] [--dpc 1,8,32,128]
                                      [--kinds beam,sample,dialog-beam,dialog-sample]
                                      [--window 1.0] [--out FILE]"""
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
from visdial_b200 import VD_MATH_F16, VD_MATH_FP32, Model  # noqa: E402
from visdial_b200.dataloader import Dataloader  # noqa: E402
from visdial_b200.engine import DEFAULT_PARAMS, derive_flags  # noqa: E402
from visdial_b200.synthetic import make_corpus  # noqa: E402
from host_decode import HostStep, host_beam_search, start_state  # noqa: E402
from dialog_history import beam_words, next_row, right_aligned, row_words, sample_words  # noqa: E402
from visdial_b200.engine import Batch  # noqa: E402

BEAM, LEN, V = 5, 20, 10000


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    except FileNotFoundError:
        q = None
    if q is None or q.returncode != 0:
        raise SystemExit("nvidia-smi failed: this benchmark needs the GPU")
    name, power = [s.strip() for s in q.stdout.splitlines()[0].split(",")]
    return name, power


def host_sample(eng, encOut, L, start, T, rng):
    """the sampling branch of Model.generateAnswers before it moved to the device (one dialog: all its rounds per step)"""
    h, c = start_state(eng, encOut)                                             # forwardConnect, gen.lua:30-42
    tok = np.full(encOut.shape[0], start, dtype=np.int64)
    seq = [tok.copy()]
    with HostStep(eng, encOut.shape[0]) as step:
        for _ in range(L):
            decOut, h, c = step(tok, h, c)                                      # :586-588 (+ decoderConnect)
            p = np.exp(decOut.astype(np.float64) / T)                           # :590
            p /= p.sum(1, keepdims=True)
            tok = np.array([rng.choice(p.shape[1], p=p[i]) + 1 for i in range(len(tok))], dtype=np.int64)
            seq.append(tok.copy())
    return np.stack(seq, 1)


def hist_width(dl):
    """the history width generateAnswers passes for generated history"""
    return dl.maxHistoryLen if dl.concatHistory else min(dl.maxQuesLen + dl.maxAnsLen, dl.maxHistoryLen)


def host_dialog(m, dl, d, start, end, sample):
    """d dialogs on their own answers with one engine call per round: the history rebuilt and uploaded every round"""
    m.wrapper.evaluate()
    nb = dl.getIndexData(np.arange(d), m.params, "val").numpy()
    B, R = nb["ques_fwd"].shape[:2]
    W, mal = hist_width(dl), dl.maxAnsLen
    hist = np.zeros((B, R, W), np.int32)
    for b in range(B):
        hist[b, 0] = right_aligned(row_words(nb["hist"][b, 0]), W)
    for r in range(R):
        m.engine.encoder_forward(Batch(dict(nb, hist=hist)))
        if sample:
            ans, _ = m.engine.gen_sample(LEN, start, 1.0, 1234, 0)
            words = [sample_words(ans[b * R + r], end) for b in range(B)]
        else:
            ans, length, _ = m.engine.gen_beam_search(BEAM, LEN, start, end)
            words = [beam_words(ans[b * R + r], length[b * R + r]) for b in range(B)]
        if r + 1 < R:
            for b in range(B):
                hist[b, r + 1] = next_row(hist[b, r], row_words(nb["ques_fwd"][b, r]), words[b], dl.concatHistory, end, W, mal)
    m.wrapper.training()


def encoders_only(m, dl, d):
    """the device loop's R encoder forwards on d dialogs at the loop's history width"""
    m.wrapper.evaluate()
    nb = dl.getIndexData(np.arange(d), m.params, "val").numpy()
    B, R = nb["ques_fwd"].shape[:2]
    W = hist_width(dl)
    hist = np.zeros((B, R, W), np.int32)
    hist[:, :, W - nb["hist"].shape[2]:] = nb["hist"]
    b = Batch(dict(nb, hist=hist)).to_device(m.engine)
    for _ in range(R):
        m.engine.encoder_forward(b)
    m.engine.synchronize()
    m.wrapper.training()


def window(call, dialogs_per_call, seconds):
    """ms per dialog over whole calls, after one warm-up call of the same shape"""
    call()
    n, t0 = 0, time.perf_counter()
    while True:
        call()
        n += dialogs_per_call
        dt = time.perf_counter() - t0
        if dt >= seconds:
            return dt / n * 1e3, n, dt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--encoders", default="hrea-ques-im-hist,mn-att-ques-im-hist")
    ap.add_argument("--modes", default="f16,fp32")
    ap.add_argument("--dpc", default="1,8,32,128")
    ap.add_argument("--kinds", default="beam,sample")
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dpcs = [int(x) for x in a.dpc.split(",")]
    kinds = a.kinds.split(",")
    name, power = card()
    rows = []
    for enc in a.encoders.split(","):
        p = dict(DEFAULT_PARAMS)
        p.update(encoder=enc, decoder="gen", vocabSize=V, imgFeatureSize=512 if "att" in enc else 4096, batchSize=1)
        p = derive_flags(p)
        raw = make_corpus(p, max(dpcs), 2000, seed=5, ques_len_cap=8 if p["concatHistory"] else None,
                          ans_len_cap=8 if p["concatHistory"] else None)
        m = Model(p, seed=3)
        dl = Dataloader(m.engine).initialize(dict(p, maxHistoryLen=60), ["val"], {"val": raw})
        start, end = dl.word2ind["<START>"], dl.word2ind["<END>"]
        for mode in a.modes.split(","):
            m.engine.set_math_mode({"f16": VD_MATH_F16, "fp32": VD_MATH_FP32}[mode])
            beam = {"beamSize": BEAM, "beamLen": LEN}

            def host_search():
                m.wrapper.evaluate()
                b = dl.getIndexData(np.array([0]), m.params, "val")
                encOut = m.forwardBackward(b, True, True).numpy()
                host_beam_search(m.engine, encOut, BEAM, LEN, start, end)
                m.wrapper.training()

            samp = {"sampleWords": 1, "beamLen": LEN, "temperature": 1.0}
            rng = np.random.default_rng(1234)

            def host_samp():
                m.wrapper.evaluate()
                b = dl.getIndexData(np.array([0]), m.params, "val")
                encOut = m.forwardBackward(b, True, True).numpy()
                host_sample(m.engine, encOut, LEN, start, 1.0, rng)
                m.wrapper.training()

            paths = []
            if "beam" in kinds:
                paths += [("device/%d" % d, d, lambda d=d: m.generateAnswers(dl, "val", dict(beam, maxThreads=d, dialogsPerCall=d),
                                                                             strict=False)) for d in dpcs]
                paths += [("host_search", 1, host_search)]
            if "sample" in kinds:
                paths += [("sample/%d" % d, d, lambda d=d: m.generateAnswers(dl, "val", dict(samp, maxThreads=d, dialogsPerCall=d)))
                          for d in dpcs]
                paths += [("host_sample", 1, host_samp)]
            dialog = {"history": "generated", "beamSize": BEAM, "beamLen": LEN}
            if "dialog-beam" in kinds:
                paths += [("dialog/%d" % d, d, lambda d=d: m.generateAnswers(dl, "val", dict(dialog, maxThreads=d, dialogsPerCall=d),
                                                                             strict=False)) for d in dpcs]
                paths += [("host_dialog/%d" % d, d, lambda d=d: host_dialog(m, dl, d, start, end, False)) for d in dpcs]
                paths += [("enc/%d" % d, d, lambda d=d: encoders_only(m, dl, d)) for d in dpcs]
            if "dialog-sample" in kinds:
                paths += [("dsample/%d" % d, d, lambda d=d: m.generateAnswers(dl, "val", dict(dialog, sampleWords=1,
                                                                                              maxThreads=d, dialogsPerCall=d)))
                          for d in dpcs]
                paths += [("host_dsample/%d" % d, d, lambda d=d: host_dialog(m, dl, d, start, end, True)) for d in dpcs]
            for path, d, call in paths:
                ms, n, dt = window(call, d, a.window)
                r = {"encoder": enc, "mode": mode, "path": path, "ms_per_dialog": round(ms, 3), "dialogs_timed": n,
                     "window_s": round(dt, 2), "beamSize": BEAM, "beamLen": LEN, "vocabSize": V, "gpu": name, "power_limit": power}
                print(json.dumps(r), flush=True)
                rows.append(r)
        dl.close(); m.engine.close()
    print("\n%s, power limit %s: ms per dialog (beam %d x %d / sampling x %d, V = %d)" % (name, power, BEAM, LEN, LEN, V))
    order = ["device", "host_search", "sample", "host_sample", "dialog", "host_dialog", "enc", "dsample", "host_dsample"]
    paths = sorted({r["path"] for r in rows}, key=lambda s: (order.index(s.split("/")[0]), int(s.split("/")[1]) if "/" in s else 0))
    print("| encoder | mode | " + " | ".join(paths) + " |")
    print("|---|---|" + "---|" * len(paths))
    for enc in a.encoders.split(","):
        for mode in a.modes.split(","):
            got = {r["path"]: r["ms_per_dialog"] for r in rows if r["encoder"] == enc and r["mode"] == mode}
            print("| %s | %s | " % (enc, mode) + " | ".join("%.2f" % got[p] for p in paths) + " |")
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
