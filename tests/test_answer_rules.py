"""The answer rules (DESIGN §25) on the host: the barred set on hand-made histories, the twin searches with the rules off and
on, constrained sampling's coupling and distribution, the command options and the Python parameters."""
import numpy as np
import pytest

import answer_rules_twin as art
import sampling_twin
from host_diverse import merge_step
from host_nbest import empty_lists, nbest_merge_step, nbest_search
from visdial_b200 import cli
from visdial_b200.model import answer_rules

END = 9


def _bar(t, stp, V=END, **kw):
    return set(np.flatnonzero(art.barred(np.asarray(t), stp, V, END, art.Rules(**kw))) + 1)


# ---- the barred set ------------------------------------------------------------------------------------------------
def test_ngram_blocking_by_hand():
    t = [8, 1, 2, 3, 1, 2, 0, 0]                   # <START> = 8, then 1 2 3 1 2
    assert _bar(t, 6, no_repeat_ngram=1) == {1, 2, 3}
    assert _bar(t, 6, no_repeat_ngram=2) == {3}     # "2 3" was seen after 2
    assert _bar(t, 6, no_repeat_ngram=3) == {3}     # "1 2 3" was seen after "1 2"
    assert _bar(t, 5, no_repeat_ngram=2) == {2}     # after "... 1": "1 2"
    assert _bar(t, 3, no_repeat_ngram=3) == set()   # too short for a 3-gram
    assert _bar([8, 8, 5, 8, 0], 4, no_repeat_ngram=2) == {5}       # a word equal to <START> counts; position 0 does not
    assert _bar([8, 5, 0, 0], 2, no_repeat_ngram=2) == set()        # <START> (position 0) is in no n-gram


def test_windows_with_a_pad_match_nothing():
    assert _bar([8, 1, 0, 1, 0], 4, no_repeat_ngram=2) == set()     # "1 0" is no bigram
    assert _bar([8, 1, 2, 0, 1, 2], 5, no_repeat_ngram=2) == {2}
    assert _bar([8, 1, 2, 0, 1, 2], 4, no_repeat_ngram=2) == set()  # the suffix is the pad


def test_end_is_never_barred_by_ngrams_and_barred_exactly_while_short():
    assert _bar([8, 4, END, 4, 0], 4, no_repeat_ngram=2) == set()
    assert _bar([8, END, END, 0], 3, no_repeat_ngram=1) == set()
    for stp in range(1, 7):
        assert (END in _bar([8] * 7, stp, min_words=3)) == (stp <= 3)


def test_banned_and_the_fallback():
    assert _bar([8, 0], 1, banned=[2, 5]) == {2, 5}
    # every class barred: <END> comes back
    assert _bar([8, 1, 2, 3, 4, 5, 6, 7, 8], 9, V=END, min_words=20, no_repeat_ngram=1) == set(range(1, 9))
    assert _bar([8, 0], 1, banned=list(range(1, 9)), min_words=3) == set(range(1, 9))


# ---- twin searches -------------------------------------------------------------------------------------------------
def _table_step(V, seed, end_early=False):
    """a row-wise decoder step from a fixed random logit table indexed by (step, fed token): no state"""
    rng = np.random.default_rng(seed)
    tab = rng.normal(0, 1.5, (40, V + 1, V)).astype(np.float32)
    if end_early:
        tab[:, :, END - 1] += 6.0                   # <END> dominates from the first step
    cnt = [0]

    def step(tokens, h, c):
        s = cnt[0]
        cnt[0] += 1
        x = tab[s, np.asarray(tokens)]
        logp = (x - np.log(np.exp(x.astype(np.float64)).sum(1, keepdims=True))).astype(np.float32)
        logp[np.asarray(tokens) == 0] = 0.0        # MaskZero pad rows
        return logp, h, c
    return step


def _search(step, N, k, G, nb, alpha, L, rules):
    z = [np.zeros((N * k, 2), np.float32)] * 2
    if rules is None:
        return nbest_search(step, z, z, N, k, G, 0.5, alpha, nb, L, 8, END)
    return art.rules_search(step, z, z, N, k, G, 0.5, alpha, nb, L, 8, END, rules)


@pytest.mark.parametrize("k,G,nb,alpha", [(4, 1, 1, 0.0), (6, 2, 1, 0.0), (6, 3, 3, 0.7)])
def test_rules_off_equal_the_existing_twins(k, G, nb, alpha):
    for seed in range(3):
        want = _search(_table_step(END, seed), 3, k, G, nb, alpha, 10, None)
        got = _search(_table_step(END, seed), 3, k, G, nb, alpha, 10, art.Rules())
        for g, w in zip(got, want):
            assert np.array_equal(g, w)


def test_unfill_keeps_plain_merges_and_empties_columns():
    rng = np.random.default_rng(0)
    N, k, L, stp = 2, 4, 6, 3
    beams = rng.integers(1, 8, (N, k, L)).astype(np.int32)
    scores = rng.normal(size=(N, k))
    topv = np.sort(rng.normal(size=(N * k, k)).astype(np.float32), 1)[:, ::-1].copy()
    topi = np.tile(np.arange(k, dtype=np.int32), (N * k, 1))
    lists = empty_lists(N, 1, 1, L)
    plain = nbest_merge_step(stp, k, 1, 0.0, None, L, END, topv, topi, scores, beams, *lists)
    ruled = art.rules_merge_step(stp, k, 1, 0.0, None, L, END, topv, topi, scores, beams, *lists)
    for a, b in zip(plain, ruled):
        assert np.array_equal(a, b)
    topv[:, 1:], topi[:, 1:] = -np.inf, -1          # one allowed class per row: explored rows give k candidates at stp > 1
    out = art.rules_merge_step(1, k, 1, 0.0, None, L, END, topv, topi, scores, beams, *lists)
    assert (out[3].reshape(N, k)[:, 1:] < 0).all() and (out[2].reshape(N, k)[:, 1:] == 0).all()
    assert np.isfinite(out[0]).all()
    ref = merge_step(1, k, 1, 0.0, L, END, topv, topi, scores, beams, *empty_lists(N, 1, 1, L)[:3])
    assert np.array_equal(ref[1][:, 0], out[1][:, 0])


@pytest.mark.parametrize("k,G,nb", [(4, 1, 1), (6, 2, 1), (6, 1, 5)])
def test_rules_on_every_finished_answer_obeys(k, G, nb):
    V, L = 30, 14
    rules = art.Rules(min_words=3, no_repeat_ngram=2, banned=[4, 7])
    seen = 0
    for seed in range(4):
        rng = np.random.default_rng(seed)
        tab = rng.normal(0, 1.5, (L, V + 1, V)).astype(np.float32)
        tab[:, :, 2] += 3.0                         # a favourite word: repeats are tempting
        cnt = [0]

        def step(tokens, h, c):
            x = tab[cnt[0], np.asarray(tokens)]
            cnt[0] += 1
            logp = (x - np.log(np.exp(x.astype(np.float64)).sum(1, keepdims=True))).astype(np.float32)
            logp[np.asarray(tokens) == 0] = 0.0
            return logp, h, c
        z = [np.zeros((3 * k, 2), np.float32)] * 2
        ans, length, _, _ = art.rules_search(step, z, z, 3, k, G, 0.5, 0.0, nb, L, V - 1, V, rules)
        for a, n in zip(ans.reshape(-1, L), length.ravel()):
            if n > 0:
                assert a[n - 1] == V and art.obeys(a[1:n - 1], rules)
                seen += 1
    assert seen > 0


def test_min_words_changes_the_pick_on_a_table_that_finishes_early():
    plain = _search(_table_step(END, 1, end_early=True), 2, 4, 1, 1, 0.0, 10, None)
    ruled = _search(_table_step(END, 1, end_early=True), 2, 4, 1, 1, 0.0, 10, art.Rules(min_words=3))
    assert (plain[1][:, 0, 0] == 2).all()           # <START> <END>: the empty answer wins unconstrained
    assert (ruled[1][:, 0, 0] >= 5).all()


# ---- constrained sampling ------------------------------------------------------------------------------------------
def _rows(R, V, seed):
    return np.random.default_rng(seed).normal(0, 2, (R, V)).astype(np.float32)


@pytest.mark.parametrize("top_k,top_p", [(0, 1.0), (5, 1.0), (0, 0.9), (8, 0.8)])
def test_constrained_draw_is_coupled_to_the_free_draw(top_k, top_p):
    V = 37
    x = _rows(400, V, 3)
    rng = np.random.default_rng(4)
    bar = rng.random((400, V)) < 0.3
    bar[:, V - 1] = False
    # the free (untruncated, unconstrained) draw: a constrained draw takes its token whenever the rules and the
    # truncation of the allowed classes keep it, as the keys of the allowed classes are the free draw's
    free, _ = sampling_twin.draw(x, 1.3, 11, 2, 0)
    allowed = ~bar[np.arange(400), free - 1]
    if top_k == 0 and top_p == 1.0:
        got, _ = art.sample_draw(x, bar, 1.3, 11, 2, 0)
    else:
        got = art.truncated_draw(x, bar, 1.3, 11, 2, top_k, top_p)[0]
        allowed &= np.array([art.probabilities(x[r], bar[r], 1.3, top_k, top_p)[free[r] - 1] > 0 for r in range(400)])
    assert allowed.sum() > 100
    assert np.array_equal(got[allowed], free[allowed])
    assert not bar[np.arange(400), got - 1].any()


@pytest.mark.parametrize("top_k,top_p", [(0, 1.0), (4, 1.0), (0, 0.8)])
def test_chi_square_of_constrained_draws(top_k, top_p):
    from scipy.stats import chisquare
    V, n = 12, 10000
    x = np.tile(_rows(1, V, 5), (n, 1))
    bar = np.zeros((n, V), bool)
    bar[:, [1, 4, 7]] = True
    p = art.probabilities(x[0], bar[0], 1.0, top_k, top_p)
    if top_k == 0 and top_p == 1.0:
        tok, _ = art.sample_draw(x, bar, 1.0, 21, 3, 0)
    else:
        tok = art.truncated_draw(x, bar, 1.0, 21, 3, top_k, top_p)[0]
    obs = np.bincount(tok - 1, minlength=V)
    keep = p > 0
    assert obs[~keep].sum() == 0
    assert chisquare(obs[keep], p[keep] * n).pvalue > 1e-3


# ---- options and parameters ----------------------------------------------------------------------------------------
def test_options_refusals_and_written_opts():
    table = cli.GENERATE_COMMAND_OPTIONS
    o = cli.parse(table, [])
    assert "minWords" not in o and "bannedWords" not in o and "noRepeatNgram" not in o
    o = cli.parse(table, ["-minWords", "0", "-noRepeatNgram", "0", "-bannedWords", ""])
    assert "minWords" not in o
    o = cli.parse(table, ["-minWords", "2", "-bannedWords", "UNK, yes"])
    assert cli.answer_rule_params(o) == {"minWords": 2, "noRepeatNgram": 0, "bannedWords": ["UNK", "yes"]}
    w = cli.written_opts(o)
    assert w["minWords"] == 2 and w["bannedWords"] == "UNK, yes"
    assert "minWords" not in cli.written_opts(cli.parse(table, []))
    for bad in (["-minWords", "-1"], ["-noRepeatNgram", "-2"]):
        with pytest.raises(SystemExit):
            cli.parse(table, bad)
    assert "minWords" in dict((n, d) for n, d, _ in cli.CHAT_OPTIONS)
    assert not any(n == "minWords" for n, _, _ in cli.GENERATE_OPTIONS)


def test_python_parameters_map_words_and_refuse_unknown_ones():
    w2i = {"yes": 1, "UNK": 2, "<START>": 3, "<END>": 4}
    assert answer_rules({}, w2i) is None
    assert answer_rules({"minWords": 0, "noRepeatNgram": 0, "bannedWords": []}, w2i) is None
    assert answer_rules({"noRepeatNgram": 2, "bannedWords": ["UNK"]}, w2i) == (0, 2, [2])
    with pytest.raises(ValueError):
        answer_rules({"bannedWords": ["nope"]}, w2i)


def test_ctypes_struct_mirrors_the_header():
    from test_abi import _struct_fields
    from visdial_b200 import _lib
    assert [f[0] for f in _lib.vd_answer_rules._fields_] == _struct_fields("vd_answer_rules")
    assert "vd_set_answer_rules" in _lib.SIGNATURES
