"""`python -m visdial_b200.train | evaluate | generate` as subprocesses on small visdial_params.json / visdial_data.h5 /
data_img.h5 files, against the same work done in-process through Model (fp32 math, the rank-exact mode)."""
import json
import math
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from helpers import small_params
from visdial_b200.synthetic import make_corpus

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
V = 40
SPLITS = {"train": 60, "val": 13, "test": 9}
CASES = [("mn-att-ques-im-hist", "disc"), ("hrea-ques-im-hist", "gen"), ("lf-ques", "gen")]   # pool5, fc7, no image file
LOG = re.compile(r"^\[[^\]]+\]\[Epoch:\d+\.\d\d\]\[Iter:\d+\]\[Loss:-?\d+\.\d{5}\]\[lr:\d+\.\d{6}\]$")


def _params(enc, dec):
    return small_params(enc, dec, vocabSize=V, numOptions=100)


def _size_flags(p):
    return ["-encoder", p["encoder"], "-decoder", p["decoder"]] + [
        x for k in ("embedSize", "rnnHiddenSize", "imgFeatureSize", "imgSpatialSize", "imgEmbedSize", "commonEmbeddingSize")
        for x in ("-" + k, str(p[k]))]


def write_files(d, enc, dec):
    """visdial_params.json / visdial_data.h5 / data_img.h5 with every split, in prepro.py's layout, under directory `d`.
    Returns (the -input* flags, the dataloader's file options)."""
    from visdial_b200 import h5lite
    p = _params(enc, dec)
    concat = "lf" in enc and "hist" in enc
    ques, imgs, info = {}, {}, {"word2ind": {"w%d" % i: i for i in range(1, V - 1)}}
    for i, (split, n) in enumerate(SPLITS.items()):
        raw = make_corpus(p, n, 40, seed=11 + i, max_ques_len=8, max_ans_len=6, max_cap_len=14,
                          ques_len_cap=5 if concat else None, ans_len_cap=4 if concat else None)
        if "images" in raw:
            imgs["images_" + split] = raw.pop("images")
        ques.update({k + "_" + split: np.asarray(v, np.uint32) for k, v in raw.items()})
        info["unique_img_" + split] = ["COCO_%s2014_%012d.jpg" % (split, 1000 * i + j) for j in range(n)]
    h5lite.write(os.path.join(d, "visdial_data.h5"), ques)
    with open(os.path.join(d, "visdial_params.json"), "w") as f:
        json.dump(info, f)
    fo = {"inputJson": os.path.join(d, "visdial_params.json"), "inputQues": os.path.join(d, "visdial_data.h5")}
    if imgs:
        h5lite.write(os.path.join(d, "data_img.h5"), imgs)
        fo["inputImg"] = os.path.join(d, "data_img.h5")
    return [x for k, v in fo.items() for x in ("-" + k, v)], fo


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    """{(enc, dec): (dir, the -input* flags, the dataloader's file options)}."""
    out = {}
    for enc, dec in CASES:
        d = tmp_path_factory.mktemp(enc)
        out[(enc, dec)] = (d,) + write_files(str(d), enc, dec)
    return out


def _run(mod, *args, ok=True):
    r = subprocess.run([sys.executable, "-m", "visdial_b200." + mod] + [str(a) for a in args], cwd=ROOT,
                       capture_output=True, text=True, timeout=1200)
    if ok:
        assert r.returncode == 0, (r.stdout[-3000:], r.stderr[-3000:])
    return r


def _model(p, fo, split, ck=None, init_seed=1234, data_seed=1234, rank=0, world=1):
    """Model + device dataloader in fp32 math, by default with the commands' seeds (visdial_b200.cli.SEED)."""
    from visdial_b200 import VD_MATH_FP32, Model
    from visdial_b200.checkpoint import restore
    from visdial_b200.dataloader import Dataloader
    from visdial_b200.engine import derive_flags
    m = Model(p, seed=init_seed)
    m.engine.set_math_mode(VD_MATH_FP32)
    if ck is not None:
        restore(m, ck)
    dl = Dataloader(m.engine, seed=data_seed, rank=rank, world=world).initialize_from_files(derive_flags(dict(p, **fo)), [split])
    return m, dl


def train_inproc(p, fo, iters, ck=None, **seeds):
    """The train command's loop in-process: (weights, learning rate) after `iters` Model.trainIteration calls."""
    m, dl = _model(p, fo, "train", ck, **seeds)
    for _ in range(iters):
        m.trainIteration(dl)
    w, lr = m.engine.get_parameters(), m.optims["learningRate"]
    dl.close(); m.engine.close()
    return w, lr


def weight_distance(a, b):
    """How far two weight vectors are apart: the largest difference, and the share of weights that differ by more than
    1e-5 (tools/measure_train_spread.py measures both between repeated runs and under a wrong seed, rate or length)."""
    d = np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64))
    return {"max": float(d.max()), "frac_1e-5": float((d > 1e-5).mean())}


# fp32 training sums some gradients with atomics, so repeated runs of one loop are not always bit-identical, and Adam carries
# a last-bit difference into the weights.  tools/measure_train_spread.py, on an H100 80GB HBM3 (400 W), 10 in-process runs
# of each case below (45 pairs): mn-att-ques-im-hist+disc never bit-identical, hrea-ques-im-hist+gen in 21 of 45 pairs,
# lf-ques+gen in all 45 (though it has differed in the last bits in other runs).  The share of weights that differ by more
# than 1e-5 was at most 0.045 % between repeated runs, and at least 93.8 % under any of: another data, initialisation or
# dropout seed, learningRate x1.01, no rate decay, one iteration fewer.  The largest difference does not separate the two
# (up to 1.3e-3 between repeated runs, 6.7e-4 for the 1 % rate change), so it only gets a loose bound.
MAX_SHARE_OFF, MAX_DIFF = 1e-2, 1e-2


def _same_as_inproc(got, ref, what):
    """The command's weights against an in-process run of the same loop, to the tolerance measured above."""
    dist = weight_distance(got, ref)
    print("%s: %s" % (what, "bit-identical" if dist["max"] == 0.0 else "%.3g %% of the weights differ by more than 1e-5, "
                      "by at most %.3g" % (100 * dist["frac_1e-5"], dist["max"])))
    assert dist["frac_1e-5"] <= MAX_SHARE_OFF and dist["max"] <= MAX_DIFF, (what, dist)


def _decayed(lr, iters, rate=0.9997592083):
    for _ in range(iters):                                                   # model.lua:102-105, the same float steps
        lr *= rate
    return lr


@pytest.mark.parametrize("enc,dec", CASES)
def test_train_writes_the_reference_checkpoints(files, tmp_path, enc, dec):
    from visdial_b200.checkpoint import load_checkpoint
    d, flags, fo = files[(enc, dec)]
    p = dict(_params(enc, dec), batchSize=1)
    save = tmp_path / "run"
    r = _run("train", *_size_flags(p), *flags, "-batchSize", 1, "-numEpochs", 2, "-saveIter", 1, "-math", "fp32",
             "-savePath", save)
    per_epoch = math.ceil(SPLITS["train"] / 1)
    assert "\n%d iter per epoch." % per_epoch in r.stdout
    logs = [ln for ln in r.stdout.splitlines() if ln.startswith("[")]
    assert len(logs) == 2 * per_epoch // 100 and all(LOG.match(ln) for ln in logs), logs
    assert "[Iter:100]" in logs[0]
    assert sorted(os.listdir(save)) == ["model_epoch_1.t7", "model_epoch_2.t7", "model_final.t7"]
    ck1 = load_checkpoint(str(save / "model_epoch_1.t7"))
    assert ck1["optims"]["learningRate"] == _decayed(1e-3, per_epoch)
    assert ck1["modelParams"]["numIterPerEpoch"] == per_epoch and ck1["modelParams"]["numTrainThreads"] == SPLITS["train"]
    fin = load_checkpoint(str(save / "model_final.t7"))
    assert "optims" not in fin and fin["modelW"].dtype == np.float32
    w, lr = train_inproc(p, fo, 2 * per_epoch)
    assert load_checkpoint(str(save / "model_epoch_2.t7"))["optims"]["learningRate"] == lr
    _same_as_inproc(fin["modelW"], w, "train %s+%s" % (enc, dec))

    if enc != "lf-ques":
        return
    # -loadPath: the file's weights and learning rate, fresh Adam moments, the file's numEpochs / saveIter
    again = tmp_path / "resumed"
    _run("train", *flags, "-loadPath", save / "model_epoch_1.t7", "-batchSize", 1, "-math", "fp32", "-savePath", again)
    got = load_checkpoint(str(again / "model_epoch_1.t7"))
    w, lr = train_inproc(p, fo, per_epoch, ck=ck1)
    assert got["optims"]["learningRate"] == lr == _decayed(ck1["optims"]["learningRate"], per_epoch)
    _same_as_inproc(got["modelW"], w, "train -loadPath")


@pytest.fixture(scope="module")
def checkpoints(files, tmp_path_factory):
    """A model_final.t7 per case (initial weights; the generative ones with a raised <END> bias so that beams finish)."""
    from visdial_b200 import Model, init_parameters
    from visdial_b200.engine import layout
    out = {}
    for enc, dec in CASES:
        p = _params(enc, dec)
        m = Model(p, seed=1234)
        w = init_parameters(p, seed=5)
        if dec == "gen":
            seg = [s for s in layout(p)[0] if s.name == "dec.out.bias"][0]
            w[seg.offset + V - 1] += 2.0                                      # class V-1 = token V = <END>
        m.engine.set_parameters(w)
        path = str(tmp_path_factory.mktemp("ck") / "model.t7")
        m.save(path, final=True)
        m.engine.close()
        out[(enc, dec)] = path
    return out


def _metrics(stdout):
    return {k: float(v) for k, v in re.findall(r"^\t(r@1|r@5|r@10|medianR|meanR|meanRR): (\S+)$", stdout, re.M)}


@pytest.mark.parametrize("enc,dec", CASES)
def test_evaluate(files, checkpoints, tmp_path, enc, dec):
    from visdial_b200.checkpoint import load_checkpoint
    from visdial_b200.utils import processRanks
    d, flags, fo = files[(enc, dec)]
    ckp = checkpoints[(enc, dec)]
    ck = load_checkpoint(ckp)
    gt = tmp_path / "gt.json"
    r = _run("evaluate", *flags, "-loadPath", ckp, "-useGt", "-saveRanks", "-saveRankPath", gt, "-math", "fp32")
    m, dl = _model(dict(ck["modelParams"], batchSize=30, useGt=True), fo, "val", ck)
    want = m.retrieve(dl, "val", as_table=True)
    ranks = m.retrieve(dl, "val")
    full = m.predict(dl, "val")
    dl.close(); m.engine.close()
    assert json.load(open(gt)) == want
    assert _metrics(r.stdout) == {k: float("%f" % v) for k, v in processRanks(ranks, verbose=False).items()}
    assert "No. questions: %d" % ranks.size in r.stdout

    allr = tmp_path / "all.json"
    _run("evaluate", *flags, "-loadPath", ckp, "-saveRanks", "-saveRankPath", allr, "-math", "fp32")
    got = json.load(open(allr))
    assert got == full and len(got[0]["ranks"]) == 100 and got[0]["image_id"] == 1000

    test = tmp_path / "test.json"
    r = _run("evaluate", *flags, "-loadPath", ckp, "-split", "test", "-useGt", "-saveRanks", "-saveRankPath", test,
             "-math", "fp32")
    assert "Warning: No ground truth avaiilable in test split, changing useGt to false." in r.stdout
    m, dl = _model(dict(ck["modelParams"], batchSize=30, useGt=False), fo, "test", ck)
    want = m.predict(dl, "test")
    nr = dl.corpus["test"].num_rounds
    dl.close(); m.engine.close()
    got = json.load(open(test))
    assert got == want and [e["round_id"] for e in got] == [int(n) for n in nr]


def _texts(answers, ind2word):
    from visdial_b200.utils import idToWords
    return [{"image_id": a["image_id"], "dialog": [{"question": idToWords(x["question"], ind2word),
                                                     "answer": idToWords(x["answer"], ind2word)} for x in a["dialog"]]}
            for a in answers]


@pytest.mark.parametrize("sample", [0, 1], ids=["beam", "sample"])
@pytest.mark.parametrize("enc,dec", [c for c in CASES if c[1] == "gen"])
def test_generate(files, checkpoints, tmp_path, enc, dec, sample):
    from visdial_b200.checkpoint import load_checkpoint
    d, flags, fo = files[(enc, dec)]
    ckp = checkpoints[(enc, dec)]
    _run("generate", *flags, "-loadPath", ckp, "-resultPath", tmp_path / "vis", "-maxThreads", 6, "-sampleWords", sample,
         "-temperature", 0.7, "-math", "fp32")
    res = json.load(open(str(tmp_path / "vis" / "results.json")))
    for k in ("encoder", "decoder", "beamSize", "beamLen", "sampleWords", "temperature"):      # vis/static/main.js
        assert k in res["opts"], k
    assert (res["opts"]["encoder"], res["opts"]["sampleWords"], res["opts"]["beamLen"]) == (enc, sample, 20)
    ck = load_checkpoint(ckp)
    m, dl = _model(ck["modelParams"], fo, "val", ck)
    answers = m.generateAnswers(dl, "val", {"maxThreads": 6, "sampleWords": sample, "temperature": 0.7, "beamSize": 5,
                                            "beamLen": 20})
    want = _texts(answers, dl.ind2word)
    dl.close(); m.engine.close()
    assert res["data"] == want
    assert len(want) == 6 and want[0]["image_id"] == 1000 and all(len(a["dialog"]) == 10 for a in want)
    assert all(x["answer"].startswith(" <START>") for a in want for x in a["dialog"])


def test_generate_stops_without_a_file_when_no_beam_finishes(files, tmp_path):
    """model.lua:575: a round where no beam reaches <END> within beamLen ends the run; no results.json is written."""
    from visdial_b200 import Model, init_parameters
    from visdial_b200.engine import layout
    enc, dec = "lf-ques", "gen"
    d, flags, fo = files[(enc, dec)]
    p = _params(enc, dec)
    m = Model(p, seed=1234)
    w = init_parameters(p, seed=5)
    seg = [s for s in layout(p)[0] if s.name == "dec.out.bias"][0]
    w[seg.offset + V - 1] -= 1e4                                              # <END> is never among the top beams
    m.engine.set_parameters(w)
    ckp = str(tmp_path / "never_ends.t7")
    m.save(ckp, final=True)
    m.engine.close()
    r = _run("generate", *flags, "-loadPath", ckp, "-resultPath", tmp_path / "vis", "-maxThreads", 2, "-math", "fp32", ok=False)
    assert r.returncode != 0 and "no beam reached <END>" in r.stderr
    assert not (tmp_path / "vis" / "results.json").exists()


# ---- two GPUs -----------------------------------------------------------------------------------------------------------
def _two_gpus():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")


def test_two_gpus_evaluate_and_generate_write_the_one_gpu_files(files, checkpoints, tmp_path):
    _two_gpus()
    for enc, dec in [("mn-att-ques-im-hist", "disc"), ("hrea-ques-im-hist", "gen")]:
        d, flags, fo = files[(enc, dec)]
        ckp = checkpoints[(enc, dec)]
        for extra in ([], ["-useGt"]):
            outs = []
            for n in (1, 2):
                path = tmp_path / ("%s%s_%d.json" % (enc, "".join(extra), n))
                _run("evaluate", *flags, "-loadPath", ckp, *extra, "-saveRanks", "-saveRankPath", path, "-math", "fp32",
                     "-gpus", n)
                outs.append(path.read_bytes())
            assert outs[0] == outs[1], (enc, extra)
    d, flags, fo = files[("hrea-ques-im-hist", "gen")]
    ckp = checkpoints[("hrea-ques-im-hist", "gen")]
    for sample in (0, 1):
        outs = []
        for n in (1, 2):
            res = tmp_path / ("gen%d_%d" % (sample, n))
            _run("generate", *flags, "-loadPath", ckp, "-resultPath", res, "-maxThreads", 5, "-sampleWords", sample,
                 "-math", "fp32", "-gpus", n)
            outs.append((res / "results.json").read_bytes())
        assert outs[0] == outs[1], sample
        assert len(json.loads(outs[0])["data"]) == 5


def test_two_gpus_train(files, tmp_path):
    _two_gpus()
    from visdial_b200.checkpoint import load_checkpoint
    p = _params("mn-att-ques-im-hist", "disc")
    d, flags, fo = files[("mn-att-ques-im-hist", "disc")]
    save = tmp_path / "run"
    r = _run("train", *_size_flags(p), *flags, "-batchSize", 1, "-numEpochs", 2, "-saveIter", 1, "-math", "fp32",
             "-savePath", save, "-gpus", 2)
    per_epoch = math.ceil(SPLITS["train"] / 2)
    assert "\n%d iter per epoch." % per_epoch in r.stdout and r.stdout.count("iter per epoch") == 1
    assert "weights identical on 2 ranks" in r.stdout
    assert sorted(os.listdir(save)) == ["model_epoch_1.t7", "model_epoch_2.t7", "model_final.t7"]
    ck1 = load_checkpoint(str(save / "model_epoch_1.t7"))
    assert ck1["optims"]["learningRate"] == _decayed(1e-3, per_epoch)


# ---- per-rank work of evaluate / generate, and the split's num_rounds -------------------------------------------------
def test_dataloader_keeps_num_rounds_for_predict_and_retrieve():
    """dataloader.lua:110 keeps `<split>_num_rounds`; model.lua:175-243 walks rounds 1..num_rounds of each dialog (every
    one on val, the last one on test).  make_corpus gives dialog 5 nine rounds."""
    from visdial_b200 import VD_MATH_FP32, Model
    from visdial_b200.dataloader import Dataloader
    p = _params("lf-ques", "disc")
    raw = make_corpus(p, 8, 40, seed=3, max_ques_len=8, max_ans_len=6, max_cap_len=14)
    m = Model(dict(p, batchSize=4), seed=3)
    m.engine.set_math_mode(VD_MATH_FP32)
    dl = Dataloader(m.engine).initialize(dict(p, maxHistoryLen=60), ["val", "test"], {"val": raw, "test": raw})
    assert np.array_equal(dl.val_num_rounds, raw["num_rounds"]) and raw["num_rounds"][5] == 9
    for table in (m.retrieve(dl, "val", as_table=True), m.predict(dl, "val")):
        rounds = [e["round_id"] for e in table if e["image_id"] == 5]
        assert rounds == list(range(1, 10)) and len(table) == 8 * 10 - 1
    test = m.predict(dl, "test")
    assert [e["round_id"] for e in test] == [10] * 5 + [9] + [10] * 2
    dl.close(); m.engine.close()


@pytest.mark.parametrize("world", [2, 3])
def test_rank_shares_concatenate_to_the_one_gpu_result(files, checkpoints, world):
    """What each rank of `evaluate -gpus N` / `generate -gpus N` computes, run here rank after rank on one GPU: the
    rank-ordered concatenation is the 1-GPU result (fp32), and a rank with an empty share contributes nothing."""
    from visdial_b200 import evaluate, generate
    from visdial_b200.checkpoint import load_checkpoint
    for (enc, dec), use_gt in ((("mn-att-ques-im-hist", "disc"), True), (("hrea-ques-im-hist", "gen"), False)):
        d, flags, fo = files[(enc, dec)]
        ck = load_checkpoint(checkpoints[(enc, dec)])
        mp = dict(ck["modelParams"], batchSize=30, useGt=use_gt)
        shares = []
        for rank, n in [(0, 1)] + [(r, world) for r in range(world)] + [(world + 12, world + 13)]:    # 13 val dialogs
            m, dl = _model(mp, fo, "val", ck, rank=rank, world=n)
            shares.append(evaluate.rank_share(m, dl, "val", use_gt))
            dl.close(); m.engine.close()
        one, parts, empty = shares[0], shares[1:-1], shares[-1]
        assert [e for _, t in parts for e in t] == one[1] and empty[1] == []
        if use_gt:
            assert np.array_equal(np.concatenate([r for r, _ in parts]), one[0]) and empty[0].shape == (0, 10)
    d, flags, fo = files[("hrea-ques-im-hist", "gen")]
    ck = load_checkpoint(checkpoints[("hrea-ques-im-hist", "gen")])
    for sample in (0, 1):
        opt = {"beamSize": 5, "beamLen": 20, "temperature": 0.7, "dialogsPerCall": 1, "sampleWords": sample,
               "maxThreads": world + 2}
        shares = []
        for rank, n in [(0, 1)] + [(r, world) for r in range(world)] + [(world + 2, world + 3)]:
            m, dl = _model(ck["modelParams"], fo, "val", ck, rank=rank, world=n)
            shares.append(generate.rank_share(m, dl, opt))
            dl.close(); m.engine.close()
        assert len(shares[0]) == world + 2
        assert [e for s in shares[1:-1] for e in s] == shares[0] and shares[-1] == []
