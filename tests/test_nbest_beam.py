"""The beam search's n-best lists on the host (tests/host_nbest.py, DESIGN §24): with n = 1 and no length penalty the list
is host_diverse.merge_step's best finished hypothesis and the pick its pick; equal norms keep (step, q) order; the lp table
is math.pow's; without a penalty a list holds the top n raw scores of every <END> candidate; with one a longer
hypothesis can outrank a shorter one of higher raw score.  And the commands' -lengthPenalty / -nBest options."""
import math

import numpy as np
import pytest

from host_diverse import merge_step, pick_answers
from host_nbest import empty_lists, end_candidates, list_step, lp_table, nbest_merge_step, pick_lists
from visdial_b200 import cli


def _tables(rng, N, k, V, end, pad=0.15, end_boost=1.2):
    """top-k tables as the decoder's are (value desc, class asc) on a coarse grid (ties), <END> likely, pad rows"""
    x = np.round(rng.normal(0.0, 1.0, (N * k, V)), 1).astype(np.float32)
    x[:, end - 1] += end_boost
    logp = (x - np.log(np.exp(x.astype(np.float64)).sum(1, keepdims=True))).astype(np.float32)
    logp[rng.random(N * k) < pad] = 0.0
    top = np.argsort(-logp, axis=1, kind="stable")[:, :k]
    return np.take_along_axis(logp, top, 1), top.astype(np.int32)


def _run(rng, N, k, G, lam, alpha, nb, L, V, **kw):
    """every merge of a search on random tables, the twin with lists beside merge_step; yields per step both results"""
    lp = lp_table(alpha, L) if alpha else None
    beams = np.zeros((N, k, L), np.int32)
    beams[:, :, 0] = V - 1
    scores = np.zeros((N, k))
    lists = empty_lists(N, G, nb, L)
    ref = (np.zeros((N, G, L), np.int32), np.zeros((N, G), np.int32), np.zeros((N, G)))
    for stp in range(1, L):
        topv, topi = _tables(rng, N, k, V, V, **kw)
        got = nbest_merge_step(stp, k, G, lam, lp, L, V, topv, topi, scores, beams, *lists)
        want = merge_step(stp, k, G, lam, L, V, topv, topi, scores, beams, *ref)
        yield stp, got, want, (topv, topi, scores, beams)
        scores, beams, lists, ref = got[0], got[1], got[4:], want[4:]


@pytest.mark.parametrize("k,G", [(6, 1), (6, 2), (6, 3), (8, 2), (5, 5)])
def test_one_entry_no_penalty_is_merge_step(k, G):
    rng = np.random.default_rng(10 * k + G)
    N, L, V = 5, 8, 12
    for lam in (0.0, 0.5):
        for stp, got, want, _ in _run(rng, N, k, G, lam, 0.0, 1, L, V):
            for a, b in zip(got[:4], want[:4]):
                assert np.array_equal(a, b), stp
            ans, length, score, norm = got[4:]
            assert np.array_equal(ans[:, :, 0], want[4]) and np.array_equal(length[:, :, 0], want[5])
            assert np.array_equal(score[:, :, 0], want[6]) and np.array_equal(norm, score)
            pa, pl, ps, _ = pick_lists(ans, length, score, norm)
            for x, y in zip((pa, pl, ps), pick_answers(*want[4:])):
                assert np.array_equal(x, y), stp


def test_one_entry_hand_made_ties_and_pad_rows():
    """<END> at two steps with equal scores: the first stays; equal <END> candidates within a step: the lower q; a pad
    row (all zero) whose <END> entry ties the others"""
    k, G, L, V = 3, 1, 5, 6
    end = V
    topi = np.array([[end - 1, 0, 1], [0, end - 1, 1], [0, 1, end - 1]], np.int32)
    topv = np.array([[-1.0, -1.0, -2.0], [-0.5, -1.0, -3.0], [0.0, 0.0, 0.0]], np.float32)
    scores = np.array([[-1.0, -1.0, -2.0]])
    beams = np.zeros((1, k, L), np.int32)
    beams[0, :, 0] = end - 1
    beams[0, :, 1] = [2, 3, 4]
    lists = empty_lists(1, G, 1, L)
    got = nbest_merge_step(2, k, G, 0.0, None, L, end, topv, topi, scores, beams, *lists)
    want = merge_step(2, k, G, 0.0, L, end, topv, topi, scores, beams, np.zeros((1, 1, L), np.int32),
                      np.zeros((1, 1), np.int32), np.zeros((1, 1)))
    assert got[5][0, 0, 0] == want[5][0, 0] == 3 and got[6][0, 0, 0] == want[6][0, 0] == -2.0
    assert np.array_equal(got[4][0, 0, 0], want[4][0, 0]) and got[4][0, 0, 0, 1] == 2      # column 0's, q = 0
    # a later step's equal score does not replace it
    later = nbest_merge_step(3, k, G, 0.0, None, L, end, topv, topi, scores, got[1], *got[4:])
    assert later[5][0, 0, 0] == 3 and later[6][0, 0, 0] == -2.0


def test_equal_norms_keep_step_then_q_order():
    N, G, nb, L, end = 1, 1, 4, 6, 9
    beams = np.arange(1, 1 + 2 * L, dtype=np.int32).reshape(1, 2, L)
    lists = empty_lists(N, G, nb, L)
    lists = list_step(2, L, end, None, beams, [[[(3, 1, -2.0), (1, 0, -2.0)]]], *lists)
    lists = list_step(3, L, end, None, beams, [[[(0, 0, -2.0), (2, 1, -1.0)]]], *lists)
    ans, length, score, norm = lists
    assert list(score[0, 0]) == [-1.0, -2.0, -2.0, -2.0]
    assert list(length[0, 0]) == [4, 3, 3, 4]
    assert ans[0, 0, 1, 1] == beams[0, 0, 1] and ans[0, 0, 2, 1] == beams[0, 1, 1]       # step 2: q 1 (column 0), q 3
    assert ans[0, 0, 0, 3] == end and ans[0, 0, 0, 4] == 0


def test_lp_table_is_math_pow():
    for alpha in (0.0, 0.6, 0.7, 1.0, 2.0, 1e-3):
        t = lp_table(alpha, 20)
        a = float(np.float32(alpha))
        assert all(t[l] == math.pow((5.0 + l) / 6.0, a) for l in range(20))
    assert (lp_table(0.0, 20) == 1.0).all()
    assert lp_table(1.0, 2)[1] == 1.0                    # lp(1) = 1 at every alpha


@pytest.mark.parametrize("k,G,nb", [(6, 1, 5), (6, 2, 3), (8, 2, 32), (4, 4, 2)])
def test_no_penalty_lists_hold_the_top_raw_scores_of_every_end_candidate(k, G, nb):
    rng = np.random.default_rng(7 * k + nb)
    N, L, V = 4, 7, 10
    seen = [[[] for _ in range(G)] for _ in range(N)]
    for stp, got, _, (topv, topi, scores, beams) in _run(rng, N, k, G, 0.5, 0.0, nb, L, V):
        for n, per in enumerate(end_candidates(stp, k, G, 0.5, V, topv, topi, scores, got[2])):
            for g, cs in enumerate(per):
                seen[n][g] += [s for _, _, s in cs]
        _, length, score, norm = got[4:]
        assert np.array_equal(norm, score)
        for n in range(N):
            for g in range(G):
                top = sorted(seen[n][g], reverse=True)[:nb]
                m = int((length[n, g] > 0).sum())
                assert list(score[n, g, :m]) == top and (length[n, g, m:] == 0).all(), (stp, n, g)
    if nb < 32:
        assert any(len(x) > nb for s in seen for x in s)  # some lists were full and evicted


def test_length_penalty_lets_a_longer_answer_outrank_a_shorter_one():
    L, end, nb = 8, 9, 2
    beams = np.zeros((1, 1, L), np.int32)
    beams[0, 0, :6] = [8, 1, 2, 3, 4, 5]
    cands = {2: [[[(0, 0, -3.0)]]], 6: [[[(0, 0, -3.3)]]]}
    for alpha, want in ((0.0, [3, 7]), (1.0, [7, 3])):
        lp = lp_table(alpha, L) if alpha else None
        lists = empty_lists(1, 1, nb, L)
        for stp in (2, 6):
            lists = list_step(stp, L, end, lp, beams, cands[stp], *lists)
        ans, length, score, norm = lists
        assert list(length[0, 0]) == want, alpha
        if alpha:
            assert norm[0, 0, 0] == -3.3 / lp[6] and norm[0, 0, 1] == -3.0 / lp[2]
            assert score[0, 0, 0] == -3.3                  # the score stays the summed log-probability
    pa, pl, ps, pg = pick_lists(ans, length, score, norm)
    assert pl[0] == 7 and ps[0] == -3.3 and pg[0] == 0


def test_pick_is_the_best_head_by_norm_lower_group_on_ties():
    L = 4
    ans = np.zeros((1, 3, 2, L), np.int32)
    length = np.array([[[3, 2], [0, 0], [3, 0]]], np.int32)
    score = np.array([[[-1.0, -2.0], [0.0, 0.0], [-0.5, 0.0]]])
    norm = np.array([[[-0.5, -2.0], [0.0, 0.0], [-0.5, 0.0]]])
    ans[0, 0, 0, 1], ans[0, 2, 0, 1] = 5, 6
    pa, pl, ps, pg = pick_lists(ans, length, score, norm)
    assert pg[0] == 0 and pa[0, 1] == 5 and ps[0] == -1.0          # the empty group 1 (norm 0) is skipped
    pa, pl, ps, pg = pick_lists(ans, np.zeros_like(length), score, norm)
    assert pg[0] == -1 and pl[0] == 0 and ps[0] == 0.0


@pytest.mark.parametrize("table", [cli.GENERATE_COMMAND_OPTIONS, cli.CHAT_OPTIONS], ids=["generate", "chat"])
def test_options_parse_and_refuse(table):
    opt = cli.parse(table, ["-lengthPenalty", "0.7", "-nBest", "5"])
    assert opt["lengthPenalty"] == 0.7 and opt["nBest"] == 5
    d = cli.parse(table, ["-nBest", "1", "-lengthPenalty", "0"])
    assert "lengthPenalty" not in d and "nBest" not in d                    # options that change nothing are dropped
    for bad in (["-lengthPenalty", "-0.1"], ["-lengthPenalty", "nan"], ["-lengthPenalty", "inf"], ["-nBest", "0"],
                ["-nBest", "33"], ["-nBest", "-1"]):
        with pytest.raises(SystemExit) as e:
            cli.parse(table, bad)
        assert e.value.code == 2, bad
    assert cli.parse(table, ["-nBest", "32"])["nBest"] == 32
    assert not {"lengthPenalty", "nBest"} & {o[0] for o in cli.GENERATE_OPTIONS}   # generate.lua's table stays its own
    assert not {"lengthPenalty", "nBest"} & {o[0] for o in cli.DIVERSE_OPTIONS}


def test_written_opts_record_the_options_only_when_they_differ_from_the_defaults():
    table = cli.GENERATE_COMMAND_OPTIONS
    base = cli.written_opts(cli.parse(table, []))
    for argv in (["-nBest", "1"], ["-lengthPenalty", "0"], ["-nBest", "1", "-lengthPenalty", "0.0"]):
        w = cli.written_opts(cli.parse(table, argv))
        assert w == base and list(w) == list(base), argv
        assert "nBest" not in w and "lengthPenalty" not in w
    w = cli.written_opts(cli.parse(table, ["-nBest", "5"]))
    assert w["nBest"] == 5 and w["lengthPenalty"] == 0.0
    w = cli.written_opts(cli.parse(table, ["-lengthPenalty", "0.7"]))
    assert w["lengthPenalty"] == 0.7 and w["nBest"] == 1
    c = cli.written_opts(cli.parse(cli.CHAT_OPTIONS, []))
    assert "nBest" not in c and "lengthPenalty" not in c
