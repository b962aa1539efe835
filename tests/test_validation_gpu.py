"""Validation while training (DESIGN §28) on the device: `train -valIter` logs what `evaluate -useGt` and `ndcg` compute
for the same checkpoints, keeps the best one, stops early with -valPatience, and leaves training exactly as it was."""
import hashlib
import json
import os
import re
import shutil

import numpy as np
import pytest

import test_cli_gpu as T
from test_dense_gpu import data  # noqa: F401  (fixture: lf-ques disc files with train and val dense annotations)
from test_regions_gpu import _write as write_region_files

pytestmark = pytest.mark.gpu

B = 4
METRICS = ("r@1", "r@5", "r@10", "medianR", "meanR", "meanRR")


def _grid_files(d, enc, dec):
    flags, _ = T.write_files(str(d), enc, dec)
    return flags, T._size_flags(T._params(enc, dec))


def _val_dense(path, n, first_image=1000, seed=3):
    rng = np.random.default_rng(seed)
    entries = [{"image_id": first_image + j, "round_id": int(rng.integers(1, 10)),
                "gt_relevance": rng.choice([0.0, 0.0, 0.5, 1.0], size=100).tolist()} for j in range(n)]
    for e in entries:
        e["gt_relevance"][0] = 1.0
    with open(str(path), "w") as f:
        json.dump(entries, f)
    return str(path)


def _printed(value):
    return float("%f" % value)


def _check_against_evaluate(save, flags, log, dense_file=None, tmp=None):
    """Every logged epoch against evaluate -useGt (and evaluate -saveRanks + ndcg) of that epoch's checkpoint."""
    from visdial_b200 import dense
    for e in log:
        ck = save / ("model_epoch_%d.t7" % e["epoch"])
        r = T._run("evaluate", *flags, "-loadPath", ck, "-useGt", "-batchSize", B, "-math", "fp32")
        assert {k: _printed(e[k]) for k in METRICS} == T._metrics(r.stdout), (e, r.stdout[-800:])
        if dense_file is None:
            continue
        ranks = tmp / ("ranks%d.json" % e["epoch"])
        T._run("evaluate", *flags, "-loadPath", ck, "-saveRanks", "-saveRankPath", ranks, "-batchSize", B, "-math", "fp32")
        r = T._run("ndcg", "-ranks", ranks, "-denseAnnotations", dense_file)
        assert "NDCG: %f" % e["ndcg"] in r.stdout, (e, r.stdout)
        assert e["ndcg"] == dense.score_ranks(json.load(open(str(ranks))), dense.read(dense_file, 100))


def _best(log, metric):
    best = None
    for e in log:
        if best is None or e[metric] > best[metric]:
            best = e
    return best["epoch"]


CASES = [("mn-att-ques-im-hist", "disc", "grid"), ("hrea-ques-im-hist", "gen", "fc7"),
         ("lf-att-ques-im-hist", "gen", "region")]


@pytest.mark.parametrize("enc,dec,features", CASES)
def test_logged_metrics_are_evaluates(tmp_path, enc, dec, features):
    d = tmp_path / "data"
    d.mkdir()
    if features == "region":
        flags, sizes = write_region_files(str(d), enc, dec, 10)
        n_train, n_val = 40, 9
    else:
        flags, sizes = _grid_files(d, enc, dec)
        n_train, n_val = T.SPLITS["train"], T.SPLITS["val"]
    dense_file = _val_dense(tmp_path / "val_dense.json", n_val) if features == "grid" else None
    save = tmp_path / "run"
    extra = ["-valDenseAnnotations", dense_file] if dense_file else []
    r = T._run("train", *sizes, *flags, "-batchSize", B, "-numEpochs", 2, "-saveIter", 1, "-valIter", 1, *extra,
               "-math", "fp32", "-savePath", save)
    per_epoch = -(-n_train // B)
    log = json.load(open(str(save / "val_log.json")))
    assert [(e["epoch"], e["iter"]) for e in log] == [(1, per_epoch), (2, 2 * per_epoch)]
    assert all(list(e) == ["epoch", "iter", *METRICS] + (["ndcg"] if dense_file else []) + ["seconds"] for e in log)
    val_lines = [ln for ln in r.stdout.splitlines() if "][Val] " in ln]
    assert len(val_lines) == 2 and all(("NDCG" in ln) == bool(dense_file) for ln in val_lines), r.stdout[-2000:]
    _check_against_evaluate(save, flags, log, dense_file, tmp_path)
    best = _best(log, "ndcg" if dense_file else "meanRR")
    assert "Best validation: epoch %d " % best in r.stdout
    assert (save / "model_best.t7").read_bytes() == (save / ("model_epoch_%d.t7" % best)).read_bytes()
    assert sorted(os.listdir(save)) == ["model_best.t7", "model_epoch_1.t7", "model_epoch_2.t7", "model_final.t7",
                                        "val_log.json"]


def _checkpoints(save):
    return {f: (save / f).read_bytes() for f in sorted(os.listdir(save)) if f.startswith("model_epoch") or f == "model_final.t7"}


@pytest.mark.parametrize("math", ["f16", "tf32"])
@pytest.mark.parametrize("enc,dec", [("hre-ques-im-hist", "disc"), ("hrea-ques-im-hist", "gen")])
def test_validation_leaves_training_alone(tmp_path, enc, dec, math):
    """-deterministic 1: every checkpoint of a run that validates each epoch is the same file as without validation."""
    d = tmp_path / "data"
    d.mkdir()
    flags, sizes = _grid_files(d, enc, dec)
    got = []
    save = tmp_path / "run"                       # one path for both runs: modelParams records savePath
    for extra in ([], ["-valIter", 1]):
        T._run("train", *sizes, *flags, "-batchSize", B, "-numEpochs", 2, "-saveIter", 1, "-math", math,
               "-deterministic", 1, *extra, "-savePath", save)
        got.append(_checkpoints(save))
        shutil.rmtree(str(save))
    assert sorted(got[0]) == ["model_epoch_1.t7", "model_epoch_2.t7", "model_final.t7"]
    assert [f for f in got[0] if got[0][f] != got[1][f]] == []


def _digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def _state(model, dl):
    m, v, t = model.engine.optim_state()
    return {"rng": json.dumps(dl.rng.bit_generator.state, default=int), "iteration": model.iteration,
            "lr": model.optims["learningRate"], "runningLoss": model.runningLoss, "t": t, "m": _digest(m), "v": _digest(v),
            "W": _digest(model.engine.get_parameters())}


@pytest.mark.parametrize("math", ["f16", "tf32"])
@pytest.mark.parametrize("enc,dec", [("mn-att-ques-im-hist", "disc"), ("hrea-ques-im-hist", "gen")])
def test_a_pass_reads_the_training_state_only(tmp_path, enc, dec, math):
    """In process, deterministic: the train RNG, iteration, learning rate, running loss, Adam's m, v and t and W are
    unchanged by a pass, and the steps after it (dropout on, the fp16 mirrors and gradient scale, the option overlap and the
    train batch ring as the pass left them) give the bits of a twin that never validated."""
    from visdial_b200 import cli
    from visdial_b200.engine import derive_flags
    from visdial_b200.validation import Validator
    flags, fo = T.write_files(str(tmp_path), enc, dec)
    mp = dict(T._params(enc, dec), batchSize=B)
    opt = derive_flags(dict(mp, **fo, math=math, deterministic=1, gpuid=0, savePath=str(tmp_path / "run")))
    os.makedirs(opt["savePath"])
    runs = []
    for validating in (False, True):
        model, dl = cli.build(dict(mp), opt, 0, 1, ["train", "val"] if validating else ["train"])
        losses = [model.trainIteration(dl) for _ in range(3)]
        if validating:
            before = _state(model, dl)
            Validator(model, dl, opt, 0, 1, lambda *a: None)(3, 1)
            assert _state(model, dl) == before
        losses += [model.trainIteration(dl) for _ in range(3)]
        runs.append((losses, _state(model, dl)))
        dl.close()
        model.engine.close()
    assert runs[0] == runs[1]
    assert json.load(open(os.path.join(opt["savePath"], "val_log.json")))[0]["iter"] == 3


def test_patience_stops_the_run(tmp_path):
    """Learning rate 0: the second validation ties the first, so -valPatience 1 stops there with epoch 1 the best."""
    from visdial_b200.checkpoint import load_checkpoint
    d = tmp_path / "data"
    d.mkdir()
    flags, sizes = _grid_files(d, "mn-att-ques-im-hist", "disc")
    save = tmp_path / "run"
    r = T._run("train", *sizes, *flags, "-batchSize", B, "-numEpochs", 6, "-saveIter", 1, "-valIter", 1, "-valPatience", 1,
               "-learningRate", 0, "-math", "fp32", "-savePath", save)
    log = json.load(open(str(save / "val_log.json")))
    assert [e["epoch"] for e in log] == [1, 2] and all(log[1][k] == log[0][k] for k in METRICS)
    assert "Stopping early: MRR has not improved for 1 validations" in r.stdout
    assert "Best validation: epoch 1 " in r.stdout
    assert sorted(os.listdir(save)) == ["model_best.t7", "model_epoch_1.t7", "model_epoch_2.t7", "model_final.t7",
                                        "val_log.json"]
    fin = load_checkpoint(str(save / "model_final.t7"))
    assert "optims" not in fin
    assert np.array_equal(fin["modelW"], load_checkpoint(str(save / "model_epoch_2.t7"))["modelW"])


def test_finetune_validates_on_ndcg(data, tmp_path):  # noqa: F811
    from visdial_b200 import dense
    _, flags, ann, ck = data
    save = tmp_path / "run"
    r = T._run("finetune", *flags, "-loadPath", ck, "-denseAnnotations", ann["train"], "-valIter", 1,
               "-valDenseAnnotations", ann["val"], "-numEpochs", 2, "-saveIter", 1, "-batchSize", B, "-math", "fp32",
               "-savePath", save)
    log = json.load(open(str(save / "val_log.json")))
    assert [e["epoch"] for e in log] == [1, 2] and all("ndcg" in e for e in log)
    assert len(re.findall(r"\]\[Val\] .* NDCG \d\.\d{5}$", r.stdout, re.M)) == 2, r.stdout[-2000:]
    best = _best(log, "ndcg")
    assert (save / "model_best.t7").read_bytes() == (save / ("model_epoch_%d.t7" % best)).read_bytes()
    ranks = tmp_path / "ranks.json"
    T._run("evaluate", *flags, "-loadPath", save / "model_epoch_1.t7", "-saveRanks", "-saveRankPath", ranks,
           "-batchSize", B, "-math", "fp32")
    assert log[0]["ndcg"] == dense.score_ranks(json.load(open(str(ranks))), dense.read(ann["val"], 100))


# ---- two GPUs -----------------------------------------------------------------------------------------------------------
def test_two_gpus(tmp_path):
    T._two_gpus()
    d = tmp_path / "data"
    d.mkdir()
    flags, sizes = _grid_files(d, "mn-att-ques-im-hist", "disc")
    dense_file = _val_dense(tmp_path / "val_dense.json", T.SPLITS["val"])
    save = tmp_path / "run"
    T._run("train", *sizes, *flags, "-batchSize", B, "-numEpochs", 2, "-saveIter", 1, "-valIter", 1,
           "-valDenseAnnotations", dense_file, "-math", "fp32", "-gpus", 2, "-savePath", save)
    log = json.load(open(str(save / "val_log.json")))
    assert [e["epoch"] for e in log] == [1, 2]
    _check_against_evaluate(save, flags, log, dense_file, tmp_path)
    # an early stop reaches both ranks: the run ends (within _run's timeout) with its final checkpoint
    stop = tmp_path / "stop"
    r = T._run("train", *sizes, *flags, "-batchSize", B, "-numEpochs", 8, "-saveIter", 1, "-valIter", 1, "-valPatience", 1,
               "-learningRate", 0, "-math", "fp32", "-gpus", 2, "-savePath", stop)
    assert "Stopping early" in r.stdout and "weights identical on 2 ranks" in r.stdout
    assert [e["epoch"] for e in json.load(open(str(stop / "val_log.json")))] == [1, 2]
    assert (stop / "model_final.t7").exists() and not (stop / "model_epoch_3.t7").exists()
    shutil.rmtree(str(stop))
