"""The truncated-sampling rule's numpy twin (tests/truncation_twin.py, DESIGN §23) checked on its own, and the generate /
chat options that select it."""
import numpy as np
import pytest
from scipy import stats

import sampling_twin
import truncation_twin as tt
from visdial_b200 import cli
from visdial_b200.model import truncates

SEED = (5 << 32) | 11


def _rows(n, V, spread=2.0, seed=0):
    return (np.random.default_rng(seed).normal(size=(n, V)) * spread).astype(np.float32)


def test_no_truncation_is_the_untruncated_draw():
    x = _rows(64, 37)
    for T in (0.5, 1.0, 2.0):
        want, _ = sampling_twin.draw(x.astype(np.float64), T, SEED, 3, 17)
        for k, p in ((0, 1.0), (37, 1.0), (100, 1.0)):
            got, _, _, small, large = tt.draw(x, T, SEED, 3, k, p, row_offset=17)
            np.testing.assert_array_equal(got, want)
            assert small.all() and large.all()


@pytest.mark.parametrize("k,p", [(1, 1.0), (5, 1.0), (0, 0.5), (0, 0.9), (5, 0.9), (20, 0.3)])
def test_coupling_with_the_untruncated_draw(k, p):
    """a truncated draw equals the untruncated one whenever the untruncated winner is kept, and is always kept itself"""
    x = _rows(400, 50, seed=1)
    free, _ = sampling_twin.draw(x.astype(np.float64), 0.8, SEED, 2, 0)
    got, either, _, small, large = tt.draw(x, 0.8, SEED, 2, k, p)
    rows = np.arange(x.shape[0])
    assert large[rows, got - 1].all()
    inside = small[rows, free - 1]
    np.testing.assert_array_equal(got[inside], free[inside])
    assert inside.any() and (~inside).any()
    assert all(got[r] in either[r] for r in rows)


def _chisquare(counts, p):
    e = p * counts.sum()
    keep = e > 0
    assert counts[~keep].sum() == 0                      # nothing drawn outside the kept set
    counts, e = counts[keep], e[keep]
    small = e < 5
    if small.any():
        counts = np.append(counts[~small], counts[small].sum())
        e = np.append(e[~small], e[small].sum())
    if counts.shape[0] == 1:
        return 1.0
    return stats.chisquare(counts, e)[1]


@pytest.mark.parametrize("T", [0.7, 1.3])
@pytest.mark.parametrize("k,p", [(1, 1.0), (5, 1.0), (50, 1.0), (0, 0.5), (0, 0.9), (50, 0.9), (5, 0.5)])
def test_draws_follow_the_renormalised_truncated_softmax(k, p, T):
    """>= 10 000 draws from one row (every row of the call a fresh Philox round) against softmax(x / T) restricted to the
    kept classes and renormalised"""
    V, n = 64, 10000
    x = _rows(1, V, spread=1.0, seed=2)[0]
    got, _, _, _, _ = tt.draw(np.repeat(x[None], n, 0), T, 1234, 1, k, p)
    counts = np.bincount(got - 1, minlength=V).astype(np.float64)
    assert _chisquare(counts, tt.probabilities(x, T, k, p)) > 1e-4


def test_k1_and_a_tiny_p_give_the_argmax():
    x = _rows(200, 30, seed=3)
    want = np.argmax(x, 1) + 1
    for k, p in ((1, 1.0), (0, 1e-6), (1, 1e-6), (7, 1e-30)):
        got, _, _, _, _ = tt.draw(x, 1.1, SEED, 5, k, p)
        np.testing.assert_array_equal(got, want)


def test_ties_at_both_boundaries_keep_the_lower_classes():
    x = np.array([1, 3, 3, 3, 2], np.float32)
    o, n, _, _ = tt.kept(x, 1.0, 2, 1.0)
    assert sorted(o[:n]) == [1, 2]
    o, n, _, _ = tt.kept(np.zeros(4, np.float32), 1.0, 0, 0.5)      # four equal masses: tau = 2 of them
    assert sorted(o[:n]) == [0, 1]
    o, n, _, _ = tt.kept(np.array([0, 5, 5, 5, 5, 1], np.float32), 1.0, 3, 0.5)   # top-k cuts a tie, top-p within it
    assert list(o[:n]) == [1, 2]
    o, n, _, _ = tt.kept(np.array([0.0, -0.0, 0.0], np.float32), 1.0, 2, 1.0)    # -0 and +0 are equal y
    assert list(o[:n]) == [0, 1]


def test_boundary_ambiguity_is_reported():
    # masses 1, 1, 1, 1: P = 0.5 reaches tau exactly at two classes; a 2^-20 perturbation moves it
    _, n, n_lo, n_hi = tt.kept(np.zeros(4, np.float32), 1.0, 0, 0.5)
    assert n == 2 and (n_lo, n_hi) == (2, 3)
    _, n, n_lo, n_hi = tt.kept(np.array([2, 0, 0], np.float32), 1.0, 0, 0.6)
    assert n == n_lo == n_hi == 1


def test_truncates():
    assert not truncates(0, 1.0, 10) and not truncates(10, 1.0, 10) and not truncates(11, 1.0, 10)
    assert truncates(1, 1.0, 10) and truncates(9, 1.0, 10) and truncates(0, 0.99, 10)


# ---- options ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("table", [cli.GENERATE_COMMAND_OPTIONS, cli.CHAT_OPTIONS], ids=["generate", "chat"])
def test_options_parse_and_refuse(table):
    opt = cli.parse(table, ["-sampleWords", "1", "-topK", "50", "-topP", "0.9"])
    assert opt["topK"] == 50 and opt["topP"] == 0.9
    for bad in (["-topK", "-1"], ["-topP", "0"], ["-topP", "1.5"], ["-topP", "-0.1"], ["-topP", "nan"]):
        with pytest.raises(SystemExit) as e:
            cli.parse(table, ["-sampleWords", "1"] + bad)
        assert e.value.code == 2, bad
    assert not {"topK", "topP"} & {o[0] for o in cli.GENERATE_OPTIONS}        # generate.lua's table stays its own


def test_written_opts_record_truncation_only_when_it_truncates_a_sampling_run():
    table = cli.GENERATE_COMMAND_OPTIONS
    for argv in ([], ["-sampleWords", "1"], ["-topK", "50"], ["-topP", "0.9"], ["-sampleWords", "1", "-topK", "0"],
                 ["-sampleWords", "1", "-topP", "1"]):
        opt = cli.parse(table, argv)
        w = cli.written_opts(opt)
        assert "topK" not in w and "topP" not in w, argv
        pairs = list(zip(argv[::2], argv[1::2]))
        base = cli.parse(table, [a for n, v in pairs if n not in ("-topK", "-topP") for a in (n, v)])
        assert list(w) == list(cli.written_opts(base)), argv
    w = cli.written_opts(cli.parse(table, ["-sampleWords", "1", "-topP", "0.9"]))
    assert w["topK"] == 0 and w["topP"] == 0.9
    w = cli.written_opts(cli.parse(table, ["-sampleWords", "1", "-topK", "5"]))
    assert w["topK"] == 5 and w["topP"] == 1.0
