"""The history rule of dialogs generated on their own answers (tests/dialog_history.py, DESIGN §17) against the reference
dataloader's history (oracle/dataloader_oracle.py::process_history + getIndexData's rightmost cut): fed the ground-truth
answers, the round-by-round rule rebuilds the dataset's rows.  And the generate command's -history option."""
import os
import subprocess
import sys

import numpy as np
import pytest

from dialog_history import beam_words, dialog_history, next_row, sample_words
from helpers import small_params
from oracle import dataloader_oracle as D
from visdial_b200 import cli
from visdial_b200.synthetic import make_corpus

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
V, R, LQ, LA = 40, 10, 6, 5
END = V


def _corpus(concat, seed=5, ans_cut=None):
    p = small_params("lf-ques-hist" if concat else "hre-ques-hist", "gen", vocabSize=V)
    raw = make_corpus(p, 12, 40, seed=seed, max_ques_len=LQ, max_ans_len=LA, max_cap_len=14,   # concat: rows fit the width
                      ques_len_cap=4 if concat else None, ans_len_cap=4 if concat else None)
    if ans_cut is not None:                                   # the dataset the rule should see when answers are cut
        raw = dict(raw, ans=raw["ans"].copy(), ans_length=np.minimum(raw["ans_length"], ans_cut))
        raw["ans"][:, :, ans_cut:] = 0
    return raw, D.DataloaderOracle(raw, use_history=True, concat_history=concat, use_im=False, start=V - 1, end=END)


def _rule(raw, orc, d, concat, W, max_ans_len):
    answers = [raw["ans"][d, r, :raw["ans_length"][d, r]].tolist() for r in range(R)]
    return dialog_history(orc.hist[d, 0], orc.ques_fwd[d], answers, concat, END, W, max_ans_len)


def _trimmed(rows, W):
    """the dataset's right-aligned rows at width W: the rightmost W columns (dataloader.lua:387-392), or pads in front"""
    if W <= rows.shape[-1]:
        return rows[..., rows.shape[-1] - W:]
    return np.concatenate([np.zeros(rows.shape[:-1] + (W - rows.shape[-1],), rows.dtype), rows], -1)


# make_corpus' dialog 1 has an empty question with a non-empty answer, where the rule writes no answer.  Dialogs 1 and 3 have
# an empty question before their last round: rightAlign's break (utils.lua:20-22) empties their later question rows in
# ques_fwd, the questions the loop reads, while processHistory writes the raw questions; per-round history rows are empty
# from there on either way, concatenated ones are not.
def _same(concat):
    return [d for d in range(12) if d not in ((1, 3) if concat else (1,))]


@pytest.mark.parametrize("concat,W", [(False, LQ + LA), (False, 8), (False, 14), (True, R * (LQ + LA)), (True, 150)],
                         ids=["per_round", "per_round_narrow", "per_round_wide", "concat", "concat_wide"])
def test_ground_truth_answers_rebuild_the_dataset_history(concat, W):
    raw, orc = _corpus(concat)
    assert orc.hist.shape[-1] == (R * (LQ + LA) if concat else LQ + LA)
    for d in _same(concat):
        assert np.array_equal(_rule(raw, orc, d, concat, W, LA), _trimmed(orc.hist[d], W)), d
    # the edge cases are there: an empty caption (every row empty), an empty round, an empty last round
    assert not orc.hist[4].any() and (orc.hist_len[3] == 0).any() != concat


def test_concat_history_that_overflows_its_width_keeps_the_rightmost_words():
    raw, orc = _corpus(True)
    W = 20
    assert (orc.hist_len > W).any()
    for d in _same(True):
        assert np.array_equal(_rule(raw, orc, d, True, W, LA), _trimmed(orc.hist[d], W)), d


@pytest.mark.parametrize("concat", [False, True], ids=["per_round", "concat"])
def test_answers_longer_than_max_ans_len_are_cut_to_their_first_words(concat):
    raw, _ = _corpus(concat)
    cut, ocut = _corpus(concat, ans_cut=3)
    assert (raw["ans_length"] > 3).any()
    W = R * (LQ + LA) if concat else LQ + LA
    for d in _same(concat):
        assert np.array_equal(_rule(raw, ocut, d, concat, W, 3), _trimmed(ocut.hist[d], W)), d


@pytest.mark.parametrize("concat", [False, True], ids=["per_round", "concat"])
def test_a_question_of_pads_writes_no_answer(concat):
    raw, orc = _corpus(concat)
    W = orc.hist.shape[-1]
    got = _rule(raw, orc, 1, concat, W, LA)
    assert raw["ques_length"][1, 4] == 0 and raw["ans_length"][1, 4] > 0 and not orc.ques_fwd[1, 5:].any()
    assert np.array_equal(got[:5], orc.hist[1, :5])
    if concat:                                                # row 4 ++ <END>: the question and answer add nothing
        assert np.array_equal(got[5], next_row(got[4], [], [7, 8], True, END, W, LA))
        assert got[5][-1] == END and np.count_nonzero(got[5]) == np.count_nonzero(got[4]) + 1
    else:                                                     # an empty row, and rightAlign's break empties the rest
        assert not got[5:].any() and orc.hist[1, 5].any()


def test_answer_words():
    assert beam_words([39, 5, 0, 7, 40, 0], 5) == [5, 7]     # a pad a stale beam column carried is not a word
    assert beam_words([39, 40, 0], 2) == [] and beam_words([39, 5, 6], 0) == []
    assert sample_words([39, 5, 6, 40, 7], 40) == [5, 6] and sample_words([39, 5, 6], 40) == [5, 6]


def test_history_option():
    assert cli.parse(cli.GENERATE_COMMAND_OPTIONS, [])["history"] == "gt"
    opt = cli.parse(cli.GENERATE_COMMAND_OPTIONS, ["-history", "generated", "-sampleWords", "1", "-dialogsPerCall", "4",
                                                   "-gpus", "2"])
    assert (opt["history"], opt["sampleWords"], opt["dialogsPerCall"], opt["gpus"]) == ("generated", 1, 4, 2)
    with pytest.raises(SystemExit):
        cli.parse(cli.GENERATE_COMMAND_OPTIONS, ["-history", "model"])
    with pytest.raises(SystemExit):                           # the other commands do not take it
        cli.parse(cli.EVALUATE_OPTIONS, ["-history", "gt"])


def test_generate_refuses_an_unknown_history_before_any_gpu_work(tmp_path):
    r = subprocess.run([sys.executable, "-m", "visdial_b200.generate", "-history", "own", "-loadPath", str(tmp_path / "none.t7"),
                        "-resultPath", str(tmp_path / "vis")], cwd=ROOT, capture_output=True, text=True, timeout=120,
                       env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
    assert r.returncode == 2 and "-history is one of gt|generated" in r.stderr, r.stderr
    assert not (tmp_path / "vis").exists()
