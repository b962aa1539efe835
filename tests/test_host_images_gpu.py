"""Image features in pinned host memory (DESIGN §29) on the device: with host placement forced by a budget of 0 bytes, every
batch, training step, command checkpoint and command output is bit for bit what the device-resident corpus gives for the
same synthetic data."""
import json
import os

import numpy as np
import pytest

import test_cli_gpu as T
from helpers import small_params
from test_regions_gpu import region_params
from visdial_b200 import VD_MATH_F16, VD_MATH_TF32
from visdial_b200 import dataloader as DL
from visdial_b200.dataloader import Dataloader
from visdial_b200.engine import Engine
from visdial_b200.model import Model
from visdial_b200.synthetic import make_corpus

pytestmark = pytest.mark.gpu

N = 40
# (name, encoder, imgNorm, regions P or 0, counts)
LAYOUTS = [("fc7", "hrea-ques-im-hist", 1, 0, False), ("pool5-norm0", "mn-att-ques-im-hist", 0, 0, False),
           ("pool5-norm1", "mn-att-ques-im-hist", 1, 0, False), ("regions36", "lf-att-ques-im-hist", 0, 36, False),
           ("regions100", "mn-att-ques-im-hist", 0, 100, True)]


def _host_budget(monkeypatch):
    """A device of 0 bytes: every split's features go to pinned host memory."""
    monkeypatch.setattr(DL, "device_memory", lambda gpuid: 0)


def _params(enc, dec, P):
    return region_params(enc, dec, P) if P else small_params(enc, dec)


def _raw(p, P, counts, seed=11):
    concat = "lf" in p["encoder"]
    raw = make_corpus(p, N, 300, seed=seed, num_images=N - 9, ques_len_cap=14 if concat else None,
                      ans_len_cap=13 if concat else None, region_adaptive=counts)
    if P and not counts:
        raw.pop("num_boxes", None)
    return raw


def _opt(p, img_norm, B=8):
    enc = p["encoder"]
    return dict(p, useHistory="hist" in enc, concatHistory="lf" in enc, useIm=True, maxHistoryLen=60, imgNorm=img_norm,
                batchSize=B)


def _pair(monkeypatch, p, opt, raw, seed=5):
    """(device-resident dataloader, host-placed dataloader) over the same splits, on one engine each."""
    dev_eng, host_eng = Engine(p), Engine(p)
    dev = Dataloader(dev_eng, seed=seed).initialize(opt, ["train", "val"], {"train": raw, "val": raw})
    with monkeypatch.context() as m:
        _host_budget(m)
        host = Dataloader(host_eng, seed=seed).initialize(opt, ["train", "val"], {"train": raw, "val": raw})
    return dev, host


def _close(*dls):
    for dl in dls:
        dl.close()
        dl.eng.close()


def _bits(batch):
    out = {}
    for k, v in batch.numpy().items():
        out[k] = v.view(np.uint32) if v.dtype == np.float32 else v
    return out


def _same(a, b, what):
    ga, gb = _bits(a), _bits(b)
    assert sorted(ga) == sorted(gb), what
    for k in ga:
        assert ga[k].shape == gb[k].shape and np.array_equal(ga[k], gb[k]), (what, k)


@pytest.mark.parametrize("name,enc,img_norm,P,counts", LAYOUTS)
def test_batches_are_bit_identical(monkeypatch, name, enc, img_norm, P, counts):
    dec = "disc" if name != "fc7" else "gen"
    p = _params(enc, dec, P)
    raw = _raw(p, P, counts)
    dev, host = _pair(monkeypatch, p, _opt(p, img_norm), raw)
    for dtype in ("train", "val"):
        on_host, by = host.corpus[dtype].images_on_host, host.corpus[dtype].image_bytes
        assert on_host and by == raw["images"].nbytes
        assert not dev.corpus[dtype].images_on_host and dev.corpus[dtype].image_bytes == by
        assert np.array_equal(dev.corpus[dtype].read("img_fv").view(np.uint32), host.corpus[dtype].read("img_fv").view(np.uint32))
    rng = np.random.default_rng(0)
    # repeated indices, dialogs that share an image row (num_images < N), runs of consecutive rows, a single dialog
    cases = [np.arange(0, 8), np.array([6, 6, 7, 39, 6]), rng.integers(0, N, size=32), np.array([9]), np.arange(31, 40)]
    for inds in cases:
        for mode in (0, 1, 2):
            _same(dev.corpus["train"].get_batch(inds, mode), host.corpus["train"].get_batch(inds, mode), (name, inds, mode))
    # the prefetching paths: training draws, and a validation walk with a ragged last batch (40 = 5 x 7 + 5)
    prm = dict(p, batchSize=7)
    for _ in range(4):
        _same(dev.getTrainBatch(prm), host.getTrainBatch(prm), (name, "train"))
    start = 0
    while start < N:
        (bd, nd), (bh, nh) = dev.getTestBatch(start, prm, "val"), host.getTestBatch(start, prm, "val")
        assert nd == nh
        _same(bd, bh, (name, "val", start))
        start = nd
    if counts:
        b = host.corpus["train"].get_batch(np.arange(N), 0)
        assert np.array_equal(b["img_count"], raw["num_boxes"][raw["img_pos"]])
    _close(dev, host)


def test_lifetime_and_prefetch_misses(monkeypatch):
    p = _params("mn-att-ques-im-hist", "disc", 0)
    raw = _raw(p, 0, False)
    dev, host = _pair(monkeypatch, p, _opt(p, 1), raw)
    prm = dict(p, batchSize=6)
    first = host.getTrainBatch(prm)
    kept = _bits(first)
    host.getTrainBatch(prm)                       # prefetches the third batch's rows while `first` is still valid
    host.eng.synchronize()
    got = _bits(first)
    assert all(np.array_equal(kept[k], got[k]) for k in kept)
    # a prefetch followed by a get-batch of other indices: that batch's own rows, and the prefetch is dropped
    c, cd = host.corpus["val"], dev.corpus["val"]
    c.prefetch(np.arange(0, 6))
    _same(cd.get_batch(np.arange(10, 16), 0), c.get_batch(np.arange(10, 16), 0), "miss")
    _same(cd.get_batch(np.arange(0, 6), 0), c.get_batch(np.arange(0, 6), 0), "after the miss")
    c.prefetch(np.array([3, 3, 1]))
    _same(cd.get_batch(np.array([3, 3]), 0), c.get_batch(np.array([3, 3]), 0), "shorter")
    _close(dev, host)


def test_no_budget_keeps_features_on_the_device():
    p = _params("mn-att-ques-im-hist", "disc", 0)
    raw = _raw(p, 0, False)
    eng = Engine(p)
    dl = Dataloader(eng).initialize(_opt(p, 1), ["train"], {"train": raw})
    assert not dl.corpus["train"].images_on_host and dl.corpus["train"].image_bytes == raw["images"].nbytes
    _close(dl)


@pytest.mark.parametrize("dec", ["disc", "gen"])
@pytest.mark.parametrize("mode", [VD_MATH_F16, VD_MATH_TF32])
def test_deterministic_steps_are_bit_identical(monkeypatch, dec, mode):
    p = _params("mn-att-ques-im-hist", dec, 0)
    raw = _raw(p, 0, False)
    opt = _opt(p, 0, B=6)
    weights = []
    for place in ("device", "host"):
        m = Model(dict(p, batchSize=6), seed=3)
        m.engine.set_math_mode(mode)
        m.engine.set_deterministic(True)
        with monkeypatch.context() as mp:
            if place == "host":
                _host_budget(mp)
            dl = Dataloader(m.engine, seed=9).initialize(opt, ["train"], {"train": raw})
        assert dl.corpus["train"].images_on_host == (place == "host")
        for _ in range(3):
            m.trainIteration(dl)
        weights.append(m.engine.get_parameters().tobytes())
        dl.close()
        m.engine.close()
    assert weights[0] == weights[1]


# ---- the commands, in process, with the budget substituted ---------------------------------------------------------------
def _train_dense(path, n):
    rng = np.random.default_rng(5)
    entries = [{"image_id": j, "round_id": int(rng.integers(1, 10)),
                "gt_relevance": rng.choice([0.0, 0.5, 1.0], size=100).tolist()} for j in range(n)]
    with open(str(path), "w") as f:
        json.dump(entries, f)
    return str(path)


def _read(path):
    with open(str(path), "rb") as f:
        return f.read()


def _in_process(monkeypatch, capsys, host, fn, opt, out, keep):
    """fn(opt) with the host budget substituted when `host`; then `out` (the run's output path, the same for both
    placements, since checkpoints record it) is moved to `keep`.  Returns what the run printed."""
    capsys.readouterr()
    with monkeypatch.context() as m:
        if host:
            _host_budget(m)
        fn(opt)
    os.rename(str(out), str(keep))
    return capsys.readouterr().out


def test_commands_write_the_same_files(monkeypatch, capsys, tmp_path):
    from visdial_b200 import cli, evaluate, finetune, generate, train
    flags = {}
    for enc, dec in (("mn-att-ques-im-hist", "disc"), ("hrea-ques-im-hist", "gen")):
        (tmp_path / enc).mkdir()
        flags[enc], _ = T.write_files(str(tmp_path / enc), enc, dec)
        sizes = T._size_flags(T._params(enc, dec))
        save = tmp_path / "run"
        for place in ("device", "host"):
            opt = cli.train_opts([str(a) for a in sizes + flags[enc] + [
                "-batchSize", 4, "-numEpochs", 2, "-saveIter", 1, "-valIter", 1, "-math", "f16", "-deterministic", 1,
                "-savePath", save]])
            _in_process(monkeypatch, capsys, place == "host", train.main, opt, save, tmp_path / (enc + place))
        dev, host = tmp_path / (enc + "device"), tmp_path / (enc + "host")
        names = sorted(os.listdir(str(dev)))
        assert names == sorted(os.listdir(str(host))) and "model_best.t7" in names
        for f in names:
            if f.endswith(".t7"):
                assert _read(dev / f) == _read(host / f), (enc, f)
        logs = [json.load(open(str(s / "val_log.json"))) for s in (dev, host)]
        for log in logs:                     # the wall time of each pass is the one entry that is not a result
            for e in log:
                e.pop("seconds")
        assert logs[0] == logs[1]

    # finetune and evaluate the disc checkpoint, generate with the gen one
    enc = "mn-att-ques-im-hist"
    dense = _train_dense(tmp_path / "dense.json", T.SPLITS["train"])
    ck = tmp_path / (enc + "device") / "model_epoch_1.t7"
    gen_ck = tmp_path / "hrea-ques-im-histdevice" / "model_final.t7"
    out = {}
    for place in ("device", "host"):
        host = place == "host"
        save, ranks, res = tmp_path / "run", tmp_path / "ranks.json", tmp_path / "results"
        opt = finetune.finetune_opts([str(a) for a in flags[enc] + [
            "-loadPath", ck, "-denseAnnotations", dense, "-batchSize", 4, "-numEpochs", 1, "-saveIter", 1, "-math", "tf32",
            "-deterministic", 1, "-savePath", save]])
        _in_process(monkeypatch, capsys, host, finetune.main, opt, save, tmp_path / ("finetune-" + place))
        opt = cli.parse(cli.EVALUATE_OPTIONS, [str(a) for a in flags[enc] + [
            "-loadPath", ck, "-useGt", "-saveRanks", "-saveRankPath", ranks, "-batchSize", 4, "-math", "fp32"]])
        printed = _in_process(monkeypatch, capsys, host, evaluate.main, opt, ranks, tmp_path / ("ranks-%s.json" % place))
        opt = cli.parse(cli.GENERATE_COMMAND_OPTIONS, [str(a) for a in flags["hrea-ques-im-hist"] + [
            "-loadPath", gen_ck, "-resultPath", res, "-maxThreads", 5, "-math", "fp32"]])
        _in_process(monkeypatch, capsys, host, generate.main, opt, res, tmp_path / ("results-" + place))
        out[place] = [_read(tmp_path / ("finetune-" + place) / f) for f in ("model_epoch_1.t7", "model_final.t7")] + [
            _read(tmp_path / ("ranks-%s.json" % place)), _read(tmp_path / ("results-" + place) / "results.json"), printed]
    assert "r@1" in out["device"][-1]
    assert out["device"] == out["host"]
