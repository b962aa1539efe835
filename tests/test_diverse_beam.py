"""Diverse beam search's merge rule on the host (tests/host_diverse.py, DESIGN §22): with one group it is the reference's
merge; selecting a group's candidates from the decoder's top-k list equals selecting them from the whole sorted row; with
no penalty every group is a search of width k / G; with a large one the groups start with distinct words.  And the
commands' -beamGroups / -diversity options."""
import numpy as np
import pytest

from host_diverse import diverse_search, merge_step, pick_index
from visdial_b200 import cli


def _ref_merge(stp, k, L, end, topv, topi, scores, beams, ans, ans_len, ans_score):
    """model.lua:529-569 as host_decode.host_beam_search restates it, on beams (N, k, L)"""
    N = scores.shape[0]
    scores_o, beams_o = scores.copy(), beams.copy()
    ans, ans_len, ans_score = ans.copy(), ans_len.copy(), ans_score.copy()
    tokens, parent = np.zeros(N * k, np.int32), np.zeros(N * k, np.int32)
    for it in range(N):
        cands, finish = [], []
        for wordId in range(1 if stp == 1 else k):
            r = it * k + wordId
            for p in range(k):
                tok = int(topi[r, p]) + 1
                sc = float(scores[it, wordId]) + float(topv[r, p])
                if tok == end:
                    finish.append((sc, wordId))
                else:
                    cands.append((sc, wordId, tok))
        finish.sort(key=lambda t: -t[0])
        if finish and (ans_len[it, 0] == 0 or finish[0][0] > ans_score[it, 0]):
            ans[it, 0, :stp] = beams[it, finish[0][1], :stp]
            ans[it, 0, stp] = end
            ans_len[it, 0], ans_score[it, 0] = stp + 1, finish[0][0]
        cands.sort(key=lambda t: -t[0])
        for c in range(k):
            r = it * k + c
            if c < len(cands):
                sc, wordId, tok = cands[c]
                beams_o[it, c, :stp] = beams[it, wordId, :stp]
                beams_o[it, c, stp] = tok
                scores_o[it, c] = sc
                tokens[r], parent[r] = tok, it * k + wordId
            else:
                beams_o[it, c, stp] = 0
                tokens[r], parent[r] = 0, -1 - r
    return scores_o, beams_o, tokens, parent, ans, ans_len, ans_score


def _topk(logp, k):
    top = np.argsort(-logp, axis=1, kind="stable")[:, :k]
    return np.take_along_axis(logp, top, 1), top.astype(np.int32)


def _state(rng, N, k, G, L, stp, V):
    """a mid-search state: beams with stp filled positions, scores with ties, some groups already finished"""
    beams = np.zeros((N, k, L), np.int32)
    beams[:, :, 0] = V - 1
    beams[:, :, 1:stp] = rng.integers(1, V - 1, (N, k, stp - 1))
    scores = np.round(rng.normal(-2.0, 1.0, (N, k)), 1)
    ans, ans_len, ans_score = np.zeros((N, G, L), np.int32), np.zeros((N, G), np.int32), np.zeros((N, G))
    done = rng.random((N, G)) < 0.3
    ans_len[done], ans_score[done] = 2, -3.0
    return scores, beams, ans, ans_len, ans_score


def _logp(rng, rows, V, end, pad_rows=0):
    """log-probability rows with ties (values on a coarse grid), a likely <END>, and all-zero (pad) rows"""
    x = np.round(rng.normal(0.0, 1.0, (rows, V)), 1).astype(np.float32)
    x[:, end - 1] += 1.0
    logp = (x - np.log(np.exp(x).sum(1, keepdims=True))).astype(np.float32)
    logp[:pad_rows] = 0.0
    return logp


@pytest.mark.parametrize("stp", [1, 2, 5])
@pytest.mark.parametrize("k", [1, 3, 8])
def test_one_group_is_the_reference_merge(stp, k):
    rng = np.random.default_rng(100 * stp + k)
    N, L, V = 4, 7, 12
    for _ in range(5):
        topv, topi = _topk(_logp(rng, N * k, V, V, pad_rows=k), k)
        state = _state(rng, N, k, 1, L, stp, V)
        got = merge_step(stp, k, 1, 0.7, L, V, topv, topi, *state)
        want = _ref_merge(stp, k, L, V, topv, topi, *state)
        for g, w, name in zip(got, want, ("scores", "beams", "tokens", "parent", "ans", "ans_len", "ans_score")):
            assert np.array_equal(g, w), name


def test_one_group_hand_made_ties():
    """equal scores across columns, <END> tied with a word, and a pad row: ties go to the lower candidate index"""
    k, L, end = 2, 4, 5
    topv = np.array([[-1.0, -1.0], [-0.5, -1.5], [0.0, 0.0], [-1.0, -2.0]], np.float32)
    topi = np.array([[4, 0], [1, 2], [0, 1], [2, 4]], np.int32)            # classes: token = class + 1, <END> = 5
    scores = np.array([[-1.0, -1.5], [0.0, 0.0]])
    beams = np.zeros((2, k, L), np.int32)
    beams[:, :, 0] = 4
    beams[:, 0, 1], beams[:, 1, 1] = 2, 3
    ans, ans_len, ans_score = np.zeros((2, 1, L), np.int32), np.zeros((2, 1), np.int32), np.zeros((2, 1))
    got = merge_step(2, k, 1, 0.0, L, end, topv, topi, scores, beams, ans, ans_len, ans_score)
    want = _ref_merge(2, k, L, end, topv, topi, scores, beams, ans, ans_len, ans_score)
    for g, w in zip(got, want):
        assert np.array_equal(g, w)
    assert got[5][0, 0] == 3 and got[6][0, 0] == -2.0                       # round 0 finished from column 0
    assert got[2][:2].tolist() == [1, 2]                                     # -2.0 (column 0, class 0) before -2.0 (column 1)


def test_top_k_list_holds_every_class_the_groups_pick():
    """Group g's w best classes under the penalty, chosen from the whole sorted row, are the ones chosen from its
    unpenalised top k (k = G w): at most g w tokens carry a penalty, and a penalty only lowers a score."""
    rng = np.random.default_rng(3)
    for _ in range(400):
        V = int(rng.integers(8, 40))
        G = int(rng.integers(1, 5))
        w = int(rng.integers(1, max(2, min(8, V // G) + 1)))
        k = G * w
        if k > V:
            continue
        g = int(rng.integers(0, G))
        lam = float(np.float32(rng.choice([0.0, 0.1, 0.5, 3.0, 1e6])))
        row = np.round(rng.normal(0, 1, V), 1).astype(np.float32)
        order = np.argsort(-row, kind="stable")
        pen = rng.choice(V, size=int(rng.integers(0, g * w + 1)), replace=True)     # the tokens earlier groups filled
        cnt = np.bincount(pen, minlength=V)

        def best(classes):
            aug = [(float(row[c]) - lam * int(cnt[c]), i, int(c)) for i, c in enumerate(classes)]
            return [c for _, _, c in sorted(aug, key=lambda t: (-t[0], t[1]))[:w]]
        assert best(order) == best(order[:k])


def _toy_step(V, H, seed=0):
    """a decoder step on the host, row by row (no row's result depends on another's): embedding + state -> tanh ->
    log-softmax, <END> (class V-1) favoured"""
    rng = np.random.default_rng(seed)
    emb = rng.normal(0, 1, (V + 1, H)).astype(np.float32)
    wout = rng.normal(0, 1.5, (H, V)).astype(np.float32)

    def step(tokens, h, c):
        hn = [np.tanh(emb[tokens] + 0.5 * h[0]).astype(np.float32), h[1]]
        logits = np.stack([r @ wout for r in hn[0]]).astype(np.float32)
        logits[:, V - 1] += 2.0                                              # <END>: hypotheses finish at varied steps
        lse = np.log(np.exp(logits.astype(np.float64)).sum(1, keepdims=True))
        logp = (logits - lse).astype(np.float32)
        logp[tokens == 0] = 0.0                                              # MaskZero: a pad row is all zeros
        return logp, hn, [c[0], c[1]]
    return step


def _search(N, k, G, lam, L=8, V=11, H=6, seed=0):
    rng = np.random.default_rng(seed + 1)
    h0 = np.repeat(rng.normal(0, 1, (N, H)).astype(np.float32), k, 0)
    h, c = [h0, np.zeros_like(h0)], [np.zeros_like(h0), np.zeros_like(h0)]
    stats = {"stale": 0, "pad_rows": 0, "end_steps": set()}
    out = diverse_search(_toy_step(V, H, seed), h, c, N, k, G, lam, L, V - 1, V, stats)
    return out, stats


@pytest.mark.parametrize("G,w", [(2, 2), (3, 1), (2, 3)])
def test_no_penalty_makes_every_group_a_search_of_width_w(G, w):
    (ans, ln, sc), _ = _search(5, G * w, G, 0.0)
    (a1, l1, s1), _ = _search(5, w, 1, 0.0)
    for g in range(G):
        assert np.array_equal(ans[:, g], a1[:, 0]) and np.array_equal(ln[:, g], l1[:, 0]) and np.array_equal(sc[:, g], s1[:, 0])
    assert (ln > 0).any()


def test_large_penalty_gives_distinct_first_words():
    rng = np.random.default_rng(9)
    N, G, w, V, L = 6, 4, 2, 20, 5
    k = G * w
    topv, topi = _topk(_logp(rng, N * k, V, V), k)
    state = _state(rng, N, k, G, L, 1, V)
    _, beams, tokens, parent, *_ = merge_step(1, k, G, 1e4, L, V, topv, topi, *state)
    for n in range(N):
        first = [int(t) for t in tokens[n * k:(n + 1) * k] if t != 0]
        assert len(first) == len(set(first)) and len(first) >= k - G          # at most one <END> per group finishes
    (ans, ln, _), stats = _search(6, 6, 3, 1e4, L=9)
    for n in range(6):
        # a column left without a candidate at step 1 carries on from a pad: that is no word
        words = [int(ans[n, g, 1]) for g in range(3) if ln[n, g] > 2 and ans[n, g, 1] != 0]
        assert len(words) == len(set(words))
    (a0, _, _), _ = _search(6, 6, 3, 0.0, L=9)
    assert not np.array_equal(a0, ans)
    assert stats["pad_rows"] > 0 and stats["stale"] > 0 and len(stats["end_steps"]) > 1, stats


def test_pick_is_the_best_group_lower_group_on_ties():
    assert pick_index([0, 3, 4], [0.0, -1.0, -1.0]) == 1
    assert pick_index([0, 0], [0.0, 0.0]) == -1
    assert pick_index([2, 3], [-2.0, -1.0]) == 1
    from visdial_b200.model import pick_group, ranked_groups
    assert pick_group(np.array([0, 3, 4]), np.array([0.0, -1.0, -1.0])) == 1
    e = {"groups": [None, {"score": -1.0, "g": 1}, {"score": -0.5, "g": 2}, {"score": -1.0, "g": 3}]}
    assert [x["g"] for x in ranked_groups(e)] == [2, 1, 3]


@pytest.mark.parametrize("table", ["GENERATE_COMMAND_OPTIONS", "CHAT_OPTIONS"])
def test_options(table):
    options = getattr(cli, table)
    opt = cli.parse(options, [])
    assert opt["beamGroups"] == 1 and opt["diversity"] == 0.5
    opt = cli.parse(options, ["-beamGroups", "5", "-beamSize", "10", "-diversity", "2"])
    assert (opt["beamGroups"], opt["beamSize"], opt["diversity"]) == (5, 10, 2.0)
    for bad in (["-beamGroups", "0"], ["-beamGroups", "3"], ["-beamGroups", "2", "-beamSize", "5"], ["-diversity", "-1"],
                ["-diversity", "nan"], ["-diversity", "inf"]):
        with pytest.raises(SystemExit) as e:
            cli.parse(options, bad)
        assert e.value.code == 2, bad
    assert "beamGroups" not in dict((n, d) for n, d, _ in cli.GENERATE_OPTIONS)      # generate.lua's table stays its own


def test_written_opts_leave_plain_beam_search_files_unchanged():
    opt = cli.parse(cli.GENERATE_COMMAND_OPTIONS, [])
    assert "beamGroups" not in cli.written_opts(opt) and "diversity" not in cli.written_opts(opt)
    assert list(cli.written_opts(opt)) == [k for k in opt if k not in ("beamGroups", "diversity")]
    opt = cli.parse(cli.GENERATE_COMMAND_OPTIONS, ["-beamGroups", "5", "-beamSize", "10"])
    assert cli.written_opts(opt)["beamGroups"] == 5 and cli.written_opts(opt)["diversity"] == 0.5
