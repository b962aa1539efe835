"""Device-resident corpus + on-device batch assembly (visdial_b200/csrc/corpus.cu through the C ABI) against
oracle/dataloader_oracle.py — bit-exact for every integer tensor, 1e-6 relative for the normalised image features.
Reference: /root/reference/dataloader.lua:143-478, utils.lua:6-45."""
import numpy as np
import pytest

from oracle import dataloader_oracle as D
from helpers import small_params
from host_decode import host_beam_search
from visdial_b200._lib import VdError
from visdial_b200.dataloader import Dataloader
from visdial_b200.engine import Batch, Engine
from visdial_b200.model import Model
from visdial_b200.synthetic import make_corpus

pytestmark = pytest.mark.gpu

CONFIGS = [("lf-ques", "gen"), ("lf-ques-im-hist", "disc"), ("hrea-ques-im-hist", "gen"), ("mn-att-ques-im-hist", "disc"),
           ("lf-ques-im-hist", "gen"), ("mn-att-ques-im-hist", "gen"), ("lf-ques-im", "disc"), ("hre-ques-hist", "gen"),
           ("mn-ques-im-hist", "disc"), ("lf-att-ques-im-hist", "disc")]


def _opt(params, img_norm):
    enc = params["encoder"]
    return dict(params, useHistory="hist" in enc, concatHistory="lf" in enc, useIm="im" in enc,
                maxHistoryLen=60, imgNorm=int(img_norm))


def _setup(enc, dec, n=40, m=300, img_norm=True, seed=11, **kw):
    params = small_params(enc, dec)
    concat = "lf" in enc and "hist" in enc
    raw = make_corpus(params, n, m, seed=seed, ques_len_cap=14 if concat else None, ans_len_cap=13 if concat else None, **kw)
    opt = _opt(params, img_norm)
    V = params["vocabSize"]
    orc = D.DataloaderOracle(raw, use_history=opt["useHistory"], concat_history=opt["concatHistory"], use_im=opt["useIm"],
                             start=V - 1, end=V, img_norm=img_norm, att="att" in enc)
    eng = Engine(params)
    dl = Dataloader(eng, seed=5).initialize(opt, ["train", "val"], {"train": raw, "val": raw})
    return params, raw, orc, eng, dl


def _same_batch(dev, ref, keys_float=("img_feat",)):
    got = dev.numpy()
    want_keys = {k for k in ref if k != "num_rounds"}
    assert set(got) == want_keys, (sorted(got), sorted(want_keys))
    for k in want_keys:
        if k in keys_float:
            np.testing.assert_allclose(got[k], ref[k], rtol=1e-6, atol=1e-7, err_msg=k)
        else:
            assert got[k].shape == ref[k].shape, (k, got[k].shape, ref[k].shape)
            assert np.array_equal(got[k], ref[k]), k


@pytest.mark.parametrize("enc,dec", CONFIGS)
def test_prepared_tensors_match_oracle(enc, dec):
    params, raw, orc, eng, dl = _setup(enc, dec)
    c = dl.corpus["train"]
    n, R = raw["ques"].shape[:2]
    assert np.array_equal(c.read("ques_fwd").reshape(orc.ques_fwd.shape), orc.ques_fwd)
    assert np.array_equal(c.read("ans_in").reshape(orc.ans_in.shape), orc.ans_in)
    assert np.array_equal(c.read("ans_out").reshape(orc.ans_out.shape), orc.ans_out)
    assert np.array_equal(c.read("opt_in").reshape(orc.opt_in.shape), orc.opt_in)
    assert np.array_equal(c.read("opt_out").reshape(orc.opt_out.shape), orc.opt_out)
    if "hist" in enc:
        assert np.array_equal(c.read("hist_len").reshape(n, R), orc.hist_len)
        assert np.array_equal(c.read("hist").reshape(orc.hist.shape), orc.hist)
        assert dl.maxHistoryLen == orc.maxHistoryLen
    if "im" in enc:
        np.testing.assert_allclose(c.read("img_fv").reshape(orc.img_fv.shape), orc.img_fv, rtol=1e-6, atol=1e-7)
    dl.close(); eng.close()


@pytest.mark.parametrize("enc,dec", CONFIGS)
def test_batches_match_oracle(enc, dec):
    params, raw, orc, eng, dl = _setup(enc, dec)
    n = raw["ques"].shape[0]
    rng = np.random.default_rng(0)
    cases = [np.arange(0, 8), np.array([6, 6, 7, 39, 6]), rng.integers(0, n, size=32), np.array([9])]
    for inds in cases:
        for mode, kw in ((0 if dec == "disc" else 1, dict(test_batch=False)), (0 if dec == "disc" else 2, dict(test_batch=True))):
            dev = dl.corpus["train"].get_batch(inds, mode)
            _same_batch(dev, orc.get_batch(inds, dec, **kw))
            assert dev.num_answer_tokens == int((orc.get_batch(inds, dec, **kw)["answer_out"] > 0).sum())
    # getTestBatch walks the split in order and the last batch is ragged (dataloader.lua:347-357)
    p = dict(params, batchSize=16)
    start, seen = 0, 0
    while start < n:
        dev, nxt = dl.getTestBatch(start, p, "val")
        ref = orc.get_batch(np.arange(start, nxt), dec, test_batch=True)
        _same_batch(dev, ref)
        assert np.array_equal(dev["num_rounds"], ref["num_rounds"])
        seen += dev.c.B; start = nxt
    assert seen == n
    by, launches = dl.corpus["val"].batch_bytes()
    assert launches == (2 if "im" in enc else 1) and by > 0
    dl.close(); eng.close()


def test_unnormalised_fc7_and_shared_images():
    # imgNorm = 0 and several dialogs pointing at the same image row (img_pos is an arbitrary map, dataloader.lua:395-397)
    params, raw, orc, eng, dl = _setup("lf-ques-im-hist", "disc", img_norm=False, num_images=7)
    inds = np.arange(0, 20)
    _same_batch(dl.corpus["train"].get_batch(inds, 0), orc.get_batch(inds, "disc", test_batch=False), keys_float=())
    dl.close(); eng.close()


def test_two_batches_stay_valid():
    # the corpus alternates two output sets: batch k is still intact after batch k+1 has been assembled
    params, raw, orc, eng, dl = _setup("mn-att-ques-im-hist", "disc")
    a = dl.corpus["train"].get_batch(np.arange(0, 8), 0)
    b = dl.corpus["train"].get_batch(np.arange(20, 30), 0)
    _same_batch(a, orc.get_batch(np.arange(0, 8), "disc", test_batch=False))
    _same_batch(b, orc.get_batch(np.arange(20, 30), "disc", test_batch=False))
    dl.close(); eng.close()


def test_errors_are_reported_not_swallowed():
    params = small_params("lf-ques-im-hist", "disc")
    raw = make_corpus(params, 16, 50, seed=2)              # full-length rounds: concat history exceeds 300 tokens
    eng = Engine(params)
    with pytest.raises(VdError):                           # dataloader.lua:246-253 would raise an index error
        Dataloader(eng).initialize(_opt(params, True), ["train"], {"train": raw})
    raw = make_corpus(params, 16, 50, seed=2, ques_len_cap=14, ans_len_cap=13)
    bad = dict(raw); bad["opt"] = raw["opt"].copy(); bad["opt"][3, 2, 1] = 51
    with pytest.raises(VdError):
        Dataloader(eng).initialize(_opt(params, True), ["train"], {"train": bad})
    dl = Dataloader(eng).initialize(_opt(params, True), ["train"], {"train": raw})
    with pytest.raises(VdError):
        dl.corpus["train"].get_batch(np.array([16]), 0)
    with pytest.raises(VdError):
        dl.corpus["train"].get_batch(np.array([], dtype=np.int64), 0)
    dl.close(); eng.close()


@pytest.mark.parametrize("enc,dec", [("mn-att-ques-im-hist", "disc"), ("hrea-ques-im-hist", "gen")])
def test_training_from_device_batches_equals_host_batches(enc, dec):
    """Model:trainIteration fed by the device dataloader == the same step fed by the oracle's host batch."""
    params, raw, orc, eng, dl = _setup(enc, dec)
    eng.close()
    inds = np.array([0, 5, 9, 13, 21, 21, 30, 38])

    class Fixed:
        def __init__(self, fn): self.fn = fn
        def getTrainBatch(self, p, B=None): return self.fn()

    losses = []
    for source in ("device", "host"):
        model = Model(dict(params, batchSize=len(inds)), seed=7)
        model.engine.set_math_mode(1)
        if source == "device":
            d2 = Dataloader(model.engine).initialize(_opt(params, True), ["train"], {"train": raw})
            feed = Fixed(lambda: d2.corpus["train"].get_batch(inds, 0 if dec == "disc" else 1))
        else:
            ref = orc.get_batch(inds, dec, test_batch=False)
            feed = Fixed(lambda: Batch({k: v for k, v in ref.items()}))
        losses.append([model.trainIteration(feed) for _ in range(3)])
        w = model.engine.get_parameters()
        losses[-1].append(w)
        model.engine.close()
    # the inputs differ only by the last-ulp of the normalised image features; Adam turns that into O(lr) noise on
    # parameters whose gradient is ~0, so the parameters are compared in aggregate and the losses tightly
    for a, b in zip(losses[0][:3], losses[1][:3]):
        assert abs(a - b) <= 1e-5 * max(1.0, abs(b))
    d = np.abs(losses[0][3] - losses[1][3])
    assert d.max() <= 7e-3 and (d > 1e-5).mean() < 1e-3


# ---- committed fixtures: the device path against tests/golden/dataloader/*.npz, no oracle in the loop ------------
import glob
import os

GOLD = sorted(glob.glob(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dataloader", "*.npz")))
GOLD_INDS = np.array([0, 1, 3, 4, 5, 5, 11])


@pytest.mark.parametrize("path", GOLD, ids=[os.path.basename(g)[:-4] for g in GOLD])
def test_device_dataloader_reproduces_golden(path):
    enc, dec = os.path.basename(path)[:-4].split("__")
    z = np.load(path)
    params = small_params(enc, dec)
    raw = {k[4:]: z[k] for k in z.files if k.startswith("raw_")}
    eng = Engine(params)
    dl = Dataloader(eng).initialize(_opt(params, True), ["train"], {"train": raw})
    c = dl.corpus["train"]
    for k in z.files:
        if not k.startswith("prep_"):
            continue
        got = c.read(k[5:]).reshape(z[k].shape)
        if z[k].dtype.kind == "f":
            np.testing.assert_allclose(got, z[k], rtol=1e-6, atol=1e-7, err_msg=k)
        else:
            assert np.array_equal(got, z[k]), k
    for tag, mode in (("train", 0 if dec == "disc" else 1), ("test", 0 if dec == "disc" else 2)):
        ref = {k[len(tag) + 1:]: z[k] for k in z.files if k.startswith(tag + "_") and k != tag + "_num_rounds"}
        _same_batch(c.get_batch(GOLD_INDS, mode), ref)
    dl.close(); eng.close()


@pytest.mark.parametrize("enc,dec", [("mn-att-ques-im-hist", "disc"), ("lf-ques-im-hist", "gen")])
def test_model_retrieve_over_the_device_dataloader(enc, dec):
    """Model:retrieve (model.lua:142-189) walking a split through getTestBatch: ranks from device-assembled batches ==
    ranks from the oracle's host batches, exactly (forward-only path, no atomics)."""
    params, raw, orc, eng, dl = _setup(enc, dec, n=20)
    eng.close()
    p = dict(params, batchSize=8)
    model = Model(p, seed=4)
    model.engine.set_math_mode(1)
    d2 = Dataloader(model.engine).initialize(_opt(params, True), ["val"], {"val": raw})
    got = model.retrieve(d2, "val")

    class HostLoader:
        numThreads = {"val": 20}
        def getTestBatch(self, start, pp, dtype):
            nxt = min(20, start + pp["batchSize"])
            return orc.get_batch(np.arange(start, nxt), dec, test_batch=True), nxt
    want = model.retrieve(HostLoader(), "val")
    assert got.shape == (20, 10) and np.array_equal(got, want)
    d2.close(); model.engine.close()


@pytest.mark.parametrize("enc", ["lf-ques", "hrea-ques-im-hist", "mn-att-ques-im-hist", "lf-ques-im-hist", "lf-ques-im", "hre-ques-im-hist",
                                 "mn-ques-hist", "lf-att-ques-im-hist"])
def test_generate_answers_matches_oracle(enc):
    """Model:generateAnswers (model.lua:432-613) — beam search and sampling on batches the device dataloader assembles —
    against the host reference search (tests/host_decode.py) on the same encoder forward, and against
    oracle.generate_answers on the same dialog (fp32 math mode)."""
    import torch
    from helpers import torch_batch, torch_params
    from oracle import visdial_oracle as O
    from visdial_b200 import init_parameters
    params = small_params(enc, "gen", vocabSize=9)
    concat = "lf" in enc and "hist" in enc
    raw = make_corpus(params, 12, 40, seed=77, max_ques_len=8, max_ans_len=6, max_cap_len=14,
                      ques_len_cap=5 if concat else None, ans_len_cap=4 if concat else None)
    V = params["vocabSize"]
    orc = D.DataloaderOracle(raw, use_history="hist" in enc, concat_history=concat, use_im="im" in enc, start=V - 1, end=V,
                             img_norm=True, att="att" in enc)
    model = Model(dict(params, batchSize=1), seed=3)
    model.engine.set_math_mode(1)
    flat = init_parameters(params, seed=3)
    model.engine.set_parameters(flat)
    dl = Dataloader(model.engine).initialize(_opt(params, True), ["val"], {"val": raw})
    P = torch_params(params, flat)
    for conv in (0, 3, 7):
        got = model.generateAnswers(dl, "val", {"beamSize": 3, "beamLen": 6, "maxThreads": conv + 1}, strict=False)[conv]["dialog"]
        # the device search walks exactly the hypotheses of the host reference (state, log-probabilities, top-k and merge
        # through the host) on the same dialog's encoder forward
        model.wrapper.evaluate()
        encOut = model.forwardBackward(dl.getIndexData(np.array([conv]), model.params, "val"), True, True).numpy()
        model.wrapper.training()
        answer, length, score = host_beam_search(model.engine, encOut, 3, 6, dl.word2ind["<START>"], dl.word2ind["<END>"])
        assert [None if g is None else (g["answer"], g["length"], g["score"]) for g in got] == \
               [None if n == 0 else (a.tolist(), int(n), float(s)) for a, n, s in zip(answer, length, score)]
        tb = torch_batch(orc.get_index_data(np.array([conv])))
        with torch.no_grad():
            want = O.generate_answers(O.Ctx(), params, P, tb, V - 1, V, beam_size=3, beam_len=6, strict=False)
        assert len(got) == len(want) == 10
        for g, w in zip(got, want):
            assert (g is None) == (w is None)
            if g is not None:
                assert g["length"] == w["length"] and abs(g["score"] - w["score"]) < 1e-4
                # a winner that passed through a stale beam column (pad token inside, model.lua:559) took a top-k over
                # an all-zero row: which of the tied tokens it picked is implementation-defined (torch.topk vs argsort)
                if 0 not in w["answer"][1:w["length"]].tolist():
                    assert g["answer"] == w["answer"].tolist()
    samp = model.generateAnswers(dl, "val", {"sampleWords": 1, "temperature": 0.8, "beamLen": 5, "maxThreads": 2, "seed": 4})
    assert len(samp) == 2 and all(len(d["dialog"]) == 10 for d in samp)
    assert all(len(r["answer"]) == 6 and r["answer"][0] == V - 1 and all(1 <= t <= V for t in r["answer"])
               for d in samp for r in d["dialog"])
    dl.close(); model.engine.close()


def test_initialize_from_files(tmp_path):
    """dataloader:initialize's file half (dataloader.lua:13-129): visdial_params.json + visdial_data.h5 + data_img.h5
    named as prepro.py / prepro_img_*.lua name them -> the same batches as the in-memory path."""
    import json
    from visdial_b200 import h5lite
    params, raw, orc, eng, dl = _setup("mn-att-ques-im-hist", "disc", n=16)
    dl.close()
    V = params["vocabSize"]
    h5lite.write(str(tmp_path / "visdial_data.h5"),
                 {k + "_val": np.asarray(v, np.uint32) for k, v in raw.items() if k != "images"})       # prepro.py:267-277
    h5lite.write(str(tmp_path / "data_img.h5"), {"images_val": raw["images"]})
    json.dump({"word2ind": {"w%d" % i: i for i in range(1, V - 1)}, "ind2word": {}, "unique_img_val": []},
              open(str(tmp_path / "visdial_params.json"), "w"))
    opt = dict(_opt(params, True), inputJson=str(tmp_path / "visdial_params.json"),
               inputQues=str(tmp_path / "visdial_data.h5"), inputImg=str(tmp_path / "data_img.h5"))
    d2 = Dataloader(eng).initialize_from_files(opt, ["val"])
    assert d2.vocabSize == V and d2.word2ind["<START>"] == V - 1 and d2.word2ind["<END>"] == V and d2.word2ind["w3"] == 3
    inds = np.array([1, 4, 4, 15])
    _same_batch(d2.corpus["val"].get_batch(inds, 0), orc.get_batch(inds, "disc", test_batch=True))
    d2.close(); eng.close()
