"""Validation while training (DESIGN §28), the host half: the -valIter / -valDenseAnnotations / -valPatience options and
their refusals, the best-so-far and patience bookkeeping, and the metric step against utils.processRanks and
dense.score_ranks."""
import json
import time

import numpy as np
import pytest

from test_cli_gpu import SPLITS, write_files
from visdial_b200 import cli, dense, h5lite
from visdial_b200.engine import derive_flags
from visdial_b200.finetune import finetune_opts
from visdial_b200.finetune_gen import finetune_gen_opts
from visdial_b200.synthetic import make_corpus
from visdial_b200.utils import processRanks
from visdial_b200.validation import Selection, annotated_rows, gt_ranks, metrics

NOW = time.struct_time((2026, 3, 4, 5, 6, 7, 0, 0, 0))
VAL_OPTS = ("valIter", "valDenseAnnotations", "valPatience")


def _today(options):
    """What train_opts returned before the validation options existed, restated from the tables."""
    opt = {n: d for n, d, _ in options + cli.RUN_OPTIONS}
    del opt["deterministic"]
    opt["savePath"] = "checkpoints/model-3-4-2026-5:6:7-lf-ques-hist-gen/"
    return derive_flags(opt)


@pytest.mark.parametrize("parse,options", [
    (lambda a: cli.train_opts(a, now=NOW), cli.TRAIN_OPTIONS),
    (lambda a: cli.train_opts(a, now=NOW, options=cli.FINETUNE_OPTIONS, prog="finetune"), cli.FINETUNE_OPTIONS),
])
def test_defaults_leave_the_options_as_they_were(parse, options):
    assert parse([]) == _today(options)
    assert parse(["-valIter", "0", "-valPatience", "0", "-valDenseAnnotations", ""]) == _today(options)


def test_the_commands_parse_the_options(monkeypatch):
    monkeypatch.setattr(time, "localtime", lambda: NOW)
    for f in (finetune_opts, finetune_gen_opts):
        assert not set(VAL_OPTS) & set(f([]))
        assert f([]) == _today(cli.FINETUNE_OPTIONS)


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    """lf-ques gen files with train / val / test splits, a val dense annotation file, and a question file without val."""
    d = tmp_path_factory.mktemp("val")
    flags, fo = write_files(str(d), "lf-ques", "gen")
    rng = np.random.default_rng(2)
    ann = [{"image_id": 1000 + j, "round_id": int(rng.integers(1, 10)), "gt_relevance": rng.random(100).tolist()}
           for j in range(SPLITS["val"])]
    path = str(d / "val_dense.json")
    with open(path, "w") as f:
        json.dump(ann, f)
    raw = make_corpus(derive_flags(dict(cli.model_params(_today(cli.TRAIN_OPTIONS)), encoder="lf-ques", vocabSize=40,
                                        numOptions=100, maxQuesCount=10)), 5, 40, seed=1, max_ques_len=8, max_ans_len=6,
                      max_cap_len=14)
    raw.pop("images", None)
    h5lite.write(str(d / "train_only.h5"), {k + "_train": np.asarray(v, np.uint32) for k, v in raw.items()})
    return d, flags, ann, path


def _refused(capsys, argv, what):
    with pytest.raises(SystemExit) as e:
        cli.train_opts(argv, now=NOW)
    assert e.value.code == 2
    err = capsys.readouterr().err
    assert what in err, err


def test_validation_options_pass_on_good_files(files):
    d, flags, ann, path = files
    opt = cli.train_opts(flags + ["-valIter", "2", "-valPatience", "3", "-valDenseAnnotations", path], now=NOW)
    assert (opt["valIter"], opt["valPatience"], opt["valDenseAnnotations"]) == (2, 3, path)
    mp = cli.model_params(opt)
    assert not set(VAL_OPTS) & set(mp)
    assert mp == cli.model_params(cli.train_opts(flags, now=NOW))


def test_refusals(files, capsys, tmp_path):
    d, flags, ann, path = files
    _refused(capsys, flags + ["-valIter", "-1"], "-valIter and -valPatience must be >= 0")
    _refused(capsys, flags + ["-valIter", "1", "-valPatience", "-2"], "-valIter and -valPatience must be >= 0")
    _refused(capsys, flags + ["-valPatience", "2"], "-valPatience needs -valIter")
    _refused(capsys, flags + ["-valDenseAnnotations", path], "-valDenseAnnotations needs -valIter")
    # a file dense.read refuses against the val split: an image of another split, a short relevance list, a bad round
    for n, bad in enumerate(({"image_id": 5, "round_id": 1}, {"gt_relevance": [1.0] * 99}, {"round_id": 11})):
        f = tmp_path / ("bad%d.json" % n)
        f.write_text(json.dumps([dict(ann[0], **bad)] + ann[1:]))
        _refused(capsys, flags + ["-valIter", "1", "-valDenseAnnotations", str(f)], "-valDenseAnnotations: ")
    f = tmp_path / "zeros.json"
    f.write_text(json.dumps([dict(a, gt_relevance=[0.0] * 100) for a in ann]))
    _refused(capsys, flags + ["-valIter", "1", "-valDenseAnnotations", str(f)], "no usable annotated round")
    # a data file without a val split
    q = flags.index("-inputQues")
    no_val = flags[:q + 1] + [str(d / "train_only.h5")] + flags[q + 2:]
    _refused(capsys, no_val + ["-valIter", "1"], "has no val split")
    cli.train_opts(no_val, now=NOW)                   # fine without -valIter: the val split is never read


def test_model_params_never_carry_the_validation_options():
    opt = dict(_today(cli.TRAIN_OPTIONS), valIter=1, valPatience=2, valDenseAnnotations="x.json", gpus=2, math="f16")
    assert not set(VAL_OPTS + ("gpus", "math")) & set(cli.model_params(opt))


# ---- the best-so-far and the patience ------------------------------------------------------------------------------------
def _drive(values, patience):
    """(the validation after which the run stops or None, best epoch, the improvements) for one value per epoch."""
    s = Selection(patience)
    improved = []
    for epoch, v in enumerate(values, 1):
        improved.append(s.record(epoch, v))
        if s.stop:
            return epoch, s.best_epoch, improved
    return None, s.best_epoch, improved


def test_ties_are_not_improvements():
    assert _drive([0.5, 0.5, 0.5], 0) == (None, 1, [True, False, False])
    assert _drive([0.5, 0.6, 0.6, 0.7], 0) == (None, 4, [True, True, False, True])


@pytest.mark.parametrize("patience", [1, 2, 3])
def test_stop_after_exactly_patience_non_improvements(patience):
    flat = [0.4] * 10
    assert _drive(flat, patience)[:2] == (1 + patience, 1)
    # an improvement resets the count: best at epoch 3, then patience non-improvements (one a tie)
    seq = [0.1, 0.3, 0.5] + [0.5, 0.2, 0.4, 0.1][:patience] + [0.9]
    assert _drive(seq, patience)[:2] == (3 + patience, 3)
    assert _drive([0.1 * i for i in range(10)], patience)[:2] == (None, 10)


def test_no_patience_never_stops():
    assert _drive([1.0] + [0.0] * 20, 0)[:2] == (None, 1)


# ---- the metric step -----------------------------------------------------------------------------------------------------
def _rank_lists(rng, D, R, K):
    return np.argsort(rng.random((D, R, K)), axis=2).argsort(axis=2).astype(np.int32) + 1


def test_metrics_equal_process_ranks_and_score_ranks(tmp_path):
    rng = np.random.default_rng(7)
    D, R, K = 23, 10, 100
    full = _rank_lists(rng, D, R, K)
    answer = rng.integers(1, K + 1, size=(D, R)).astype(np.int32)
    want_gt = np.array([[full[i, j, answer[i, j] - 1] for j in range(R)] for i in range(D)])
    gt = gt_ranks(full, answer)
    assert np.array_equal(gt, want_gt)

    unique_img = ["COCO_val2014_%012d.jpg" % (500 + i) for i in range(D)]
    entries = [{"image_id": 500 + int(i), "round_id": int(rng.integers(1, R + 1)),
                "gt_relevance": rng.choice([0.0, 0.0, 0.5, 1.0], size=K).tolist()} for i in rng.permutation(D)[:17]]
    entries[3]["gt_relevance"] = [0.0] * K                                     # skipped by dense.read
    f = tmp_path / "val_dense.json"
    f.write_text(json.dumps(entries))
    ann = dense.read(str(f), K, unique_img=unique_img)
    table = [{"image_id": 500 + i, "round_id": j + 1, "ranks": full[i, j].tolist()} for i in range(D) for j in range(R)]

    pos, rows = annotated_rows(full, 0, ann)
    got = metrics(gt, rows, ann.relevance)
    assert {k: v for k, v in got.items() if k != "ndcg"} == processRanks(want_gt, verbose=False)
    assert got["ndcg"] == dense.score_ranks(table, ann)
    assert list(pos) == list(range(len(ann)))
    assert metrics(gt) == processRanks(want_gt, verbose=False)

    # the shares of several ranks, gathered in rank order and put back in annotation order, give the same numbers
    from visdial_b200.dist import shard_range
    for world in (2, 3, 5):
        shares = [shard_range(D, r, world) for r in range(world)]
        parts = [annotated_rows(full[lo:hi], lo, ann) for lo, hi in shares]
        p = np.concatenate([a for a, _ in parts])
        rows = np.concatenate([b for _, b in parts])[np.argsort(p, kind="stable")]
        g = np.concatenate([gt_ranks(full[lo:hi], answer[lo:hi]) for lo, hi in shares])
        assert metrics(g, rows, ann.relevance) == got
