"""Synthetic VisDial-shaped batches that reproduce the OUTPUT CONTRACT of the reference dataloader
(/root/reference/dataloader.lua:143-478, SURVEY.md Appendix A and §8d): right-aligned questions and
history, left-aligned START/END-wrapped answers, raw left-aligned options, 1-based ids with 0 = pad.
There is no VisDial data (and no h5py) in this environment; `data` is always "synthetic"."""
from __future__ import annotations

from typing import Dict

import numpy as np


def _right_align(rows, width):
    out = np.zeros((len(rows), width), dtype=np.int32)
    for i, r in enumerate(rows):
        r = r[-width:] if len(r) > width else r
        if len(r):
            out[i, width - len(r):] = r
    return out


def make_batch(params: dict, B: int, seed: int = 1234, max_ques_len: int = 20, max_ans_len: int = 19,
               max_cap_len: int = 40, max_hist_len: int = 40, max_hist_concat: int = 300,
               gen_eval: bool = False, empty_round_every: int = 16) -> Dict[str, np.ndarray]:
    """dataloader:getTrainBatch / getTestBatch analogue.  Keys as in the reference batch table."""
    rng = np.random.default_rng(seed)
    V = int(params["vocabSize"])
    R = int(params.get("maxQuesCount", 10))
    K = int(params.get("numOptions", 100))
    enc = params["encoder"]
    START, END = V - 1, V                                    # dataloader.lua:17-22
    tok = lambda n: rng.integers(1, V - 1, size=n, dtype=np.int32)   # U{1..V-2}

    ques, ans, cap = [], [], []
    for b in range(B):
        cap.append(tok(max_cap_len if b == 0 else int(rng.integers(1, max_cap_len + 1))))
        for r in range(R):
            ql = int(rng.integers(1, max_ques_len + 1))
            al = int(rng.integers(1, max_ans_len + 1))
            if b == 0 and r == 0:                            # one max-length sequence -> deterministic trim
                ql, al = max_ques_len, max_ans_len
            if empty_round_every and b % empty_round_every == empty_round_every - 1 and r == R - 1:
                ql, al = 0, 0                                # a fully padded round (v1.0 test has < 10 rounds)
            ques.append(tok(ql))
            ans.append(tok(al))
    Tq = max(1, max(len(q) for q in ques))
    out = {"ques_fwd": _right_align(ques, Tq).reshape(B, R, Tq)}          # dataloader.lua:146-147,380-384

    if "hist" in enc:
        rows = []
        concat = "lf" in enc                                               # opts.lua:59
        for b in range(B):
            run = list(cap[b])
            for r in range(R):
                if r == 0:
                    h = list(cap[b])
                else:
                    qa = list(ques[b * R + r - 1]) + list(ans[b * R + r - 1])
                    if concat:                                             # dataloader.lua:217-255
                        run = run + [END] + qa
                        h = run
                    else:                                                  # :234-267
                        h = qa
                rows.append(np.asarray(h, dtype=np.int32))
        width = max_hist_concat if concat else max_hist_len
        Th = max(1, min(width, max(len(h) for h in rows)))
        out["hist"] = _right_align(rows, Th).reshape(B, R, Th)

    if "im" in enc:
        if int(params.get("imgRegions", 0)) > 0:                           # region rows with adaptive counts (DESIGN §26)
            out["img_feat"], out["img_count"] = region_features(rng, B, int(params["imgRegions"]),
                                                                int(params["imgFeatureSize"]), adaptive=True)
        elif "att" in enc:                                                 # pool5 NHWC, un-normalised (opts.lua:66)
            S, Cc = int(params["imgSpatialSize"]), int(params["imgFeatureSize"])
            out["img_feat"] = np.maximum(rng.standard_normal((B, S, S, Cc), dtype=np.float32), 0)
        else:                                                              # fc7, L2-normalised (dataloader.lua:64-68)
            F = int(params["imgFeatureSize"])
            f = np.maximum(rng.standard_normal((B, F), dtype=np.float32), 0)
            out["img_feat"] = (f / np.linalg.norm(f, axis=1, keepdims=True)).astype(np.float32)

    N = B * R
    Ta = max(len(a) for a in ans) + 1                                       # dataloader.lua:401-407
    a_in = np.zeros((N, Ta), dtype=np.int32)
    a_out = np.zeros((N, Ta), dtype=np.int32)
    for i, a in enumerate(ans):
        a_in[i, 0] = START
        a_in[i, 1:1 + len(a)] = a
        a_out[i, :len(a)] = a
        a_out[i, len(a)] = END
    out["answer_in"] = a_in.reshape(B, R, Ta)
    out["answer_out"] = a_out.reshape(B, R, Ta)

    gt = rng.integers(1, K + 1, size=N).astype(np.int32)                    # 1-based (prepro.py:166-170)
    out["answer_ind"] = gt
    To = 20                                                                 # never trimmed (dataloader.lua:463-470)
    lens = rng.integers(1, max_ans_len + 1, size=(N, K))
    opts = rng.integers(1, V - 1, size=(N, K, To), dtype=np.int32)
    opts *= (np.arange(To)[None, None, :] < lens[:, :, None])
    for n in range(N):                                                      # the ground-truth option is the answer
        if len(ans[n]) > 0:
            opts[n, gt[n] - 1, :] = 0
            opts[n, gt[n] - 1, :len(ans[n])] = ans[n]
    out["options"] = opts

    if gen_eval:                                                            # dataloader.lua:281-321,437-462
        olen = (opts != 0).sum(-1)
        To2 = int(olen.max()) + 1
        oi = np.zeros((N, K, To2), dtype=np.int32)
        oo = np.zeros((N, K, To2), dtype=np.int32)
        oi[:, :, 0] = START
        oi[:, :, 1:] = opts[:, :, :To2 - 1]
        oo[:, :, :To2 - 1] = opts[:, :, :To2 - 1]
        np.put_along_axis(oo, olen[:, :, None], END, axis=2)
        out["option_in"] = oi.reshape(B, R, K, To2)
        out["option_out"] = oo.reshape(B, R, K, To2)
        del out["options"]          # the dataloader emits either raw options (disc) or option_in/out (gen eval)
    return out


class SyntheticDataloader:
    """Minimal dataloader with the reference's method names (dataloader.lua:324-375)."""

    def __init__(self, params: dict, num_threads: int = 256, seed: int = 1234):
        self.params = params
        self.numThreads = {"train": num_threads, "val": num_threads}
        self.seed = seed
        self.iter = 0

    def getTrainBatch(self, params: dict, B: int = None):
        self.iter += 1
        return make_batch(params, B or int(params.get("batchSize", 40)), seed=self.seed + self.iter)

    def getTestBatch(self, start_id: int, params: dict, dtype: str = "val"):
        B = int(params.get("batchSize", 40))
        return make_batch(params, B, seed=self.seed + 100003 + start_id,
                          gen_eval=params.get("decoder") == "gen")


def region_features(rng, n: int, P: int, C: int, adaptive: bool = True, lo: int = 1):
    """Detector region features as a v1.0 features file holds them: (n, P, C) float32 rows, and with `adaptive` the
    per-image counts (n,) int32 in [lo, P] (the first image has P regions and, for n >= 2, the second has lo), else None
    (a fixed P boxes per image).  Rows at or past an image's count hold nonzero junk, as a file's padding may."""
    feats = (np.maximum(rng.standard_normal((n, P, C), dtype=np.float32), 0) + 0.01).astype(np.float32)
    if not adaptive:
        return feats, None
    counts = rng.integers(lo, P + 1, size=n).astype(np.int32)
    counts[0] = P
    if n >= 2:
        counts[1] = lo
    pad = np.arange(P)[None, :] >= counts[:, None]
    feats[pad] = rng.uniform(-3.0, 3.0, size=(int(pad.sum()), C)).astype(np.float32)
    return feats, counts


def write_region_features(path: str, splits: Dict[str, tuple]):
    """An image features h5 of region features: {split: (images (n, P, C), counts (n,) or None)} as images_<split> and,
    when counts are given, num_boxes_<split>."""
    from . import h5lite
    data = {}
    for split, (feats, counts) in splits.items():
        data["images_" + split] = np.ascontiguousarray(feats, dtype=np.float32)
        if counts is not None:
            data["num_boxes_" + split] = np.ascontiguousarray(counts, dtype=np.int32)
    h5lite.write(path, data)


def make_corpus(params: dict, num_threads: int = 64, num_opt_list: int = 512, seed: int = 4321, max_ques_len: int = 20,
                max_ans_len: int = 20, max_cap_len: int = 40, ques_len_cap: int = None, ans_len_cap: int = None,
                edge_cases: bool = True, num_images: int = None, region_adaptive: bool = True) -> Dict[str, np.ndarray]:
    """One split of visdial_data.h5 + data_img.h5 in the layout data/prepro.py:105-183 writes (dataset names without
    the `_<split>` suffix): left-aligned zero-padded token matrices with separate length arrays, 1-based option rows
    into `opt_list`, 1-based `ans_index`, 0-based `img_pos`.  `edge_cases` plants what the reference's loops treat
    specially: an empty question / empty answer round in the middle of a dialog (utils.lua:20-22 `break`), an empty
    caption, an empty option, and one dialog with every sequence at full length.  With params' imgRegions = P > 0 the
    images are region features (numImages, P, imgFeatureSize) with `num_boxes` (region_features; region_adaptive)."""
    rng = np.random.default_rng(seed)
    V = int(params["vocabSize"])
    R = int(params.get("maxQuesCount", 10))
    K = int(params.get("numOptions", 100))
    enc = params["encoder"]
    n, m = int(num_threads), int(num_opt_list)
    qcap = int(ques_len_cap or max_ques_len)
    acap = int(ans_len_cap or max_ans_len)
    tok = lambda shape: rng.integers(1, V - 1, size=shape, dtype=np.int32)
    mask = lambda lens, width: (np.arange(width)[None, :] < np.asarray(lens).reshape(-1, 1)).astype(np.int32)

    ques_len = rng.integers(1, qcap + 1, size=(n, R)).astype(np.int32)
    ans_len = rng.integers(1, acap + 1, size=(n, R)).astype(np.int32)
    cap_len = rng.integers(1, max_cap_len + 1, size=n).astype(np.int32)
    opt_len = rng.integers(1, acap + 1, size=m).astype(np.int32)
    if edge_cases and n >= 8:
        ques_len[0, :], ans_len[0, :], cap_len[0] = qcap, acap, max_cap_len      # everything at full length
        ques_len[1, 4] = 0                                                       # empty question mid-dialog
        ans_len[2, 3] = 0                                                        # empty answer
        ques_len[3, 2], ans_len[3, 2] = 0, 0                                     # empty Q and A -> empty history round
        cap_len[4] = 0                                                           # empty caption
        ques_len[5, R - 1], ans_len[5, R - 1] = 0, 0                             # v1.0-test style short dialog
        opt_len[1] = 0                                                           # empty option
    out = {
        "ques": tok((n, R, max_ques_len)) * mask(ques_len, max_ques_len).reshape(n, R, max_ques_len),
        "ques_length": ques_len,
        "ans": tok((n, R, max_ans_len)) * mask(ans_len, max_ans_len).reshape(n, R, max_ans_len),
        "ans_length": ans_len,
        "cap": tok((n, max_cap_len)) * mask(cap_len, max_cap_len),
        "cap_length": cap_len,
        "opt_list": tok((m, max_ans_len)) * mask(opt_len, max_ans_len),
        "opt_length": opt_len,
        "opt": rng.integers(1, m + 1, size=(n, R, K)).astype(np.int32),           # prepro.py:151-160 (1-based)
        "ans_index": rng.integers(1, K + 1, size=(n, R)).astype(np.int32),        # prepro.py:166-170
        "num_rounds": np.full(n, R, dtype=np.int32),
    }
    if edge_cases and n >= 8:
        out["opt"][0, 0, 0] = 2                                                   # the empty option is referenced
        out["num_rounds"][5] = R - 1
    if "im" in enc:
        nimg = int(num_images or n)
        out["img_pos"] = rng.permutation(nimg)[:n].astype(np.int32) if nimg >= n else \
            rng.integers(0, nimg, size=n).astype(np.int32)
        if int(params.get("imgRegions", 0)) > 0:                                  # region rows N x P x C (DESIGN §26)
            out["images"], nb = region_features(rng, nimg, int(params["imgRegions"]), int(params["imgFeatureSize"]),
                                                adaptive=region_adaptive)
            if nb is not None:
                out["num_boxes"] = nb
        elif "att" in enc:                                                        # pool5 as stored: N x C x S x S
            S, Cc = int(params["imgSpatialSize"]), int(params["imgFeatureSize"])
            out["images"] = np.maximum(rng.standard_normal((nimg, Cc, S, S), dtype=np.float32), 0) + 0.01
        else:
            out["images"] = np.maximum(rng.standard_normal((nimg, int(params["imgFeatureSize"])), dtype=np.float32), 0) + 0.01
    return out
