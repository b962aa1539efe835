"""The sampling rule of generateAnswers (Gumbel-max over x / T with counter-based Philox draws, common.cuh) as its numpy twin
states it: the transform, the counter layout, independence from how the rounds are split into calls, the distribution it
draws from, and the low-temperature limit."""
import math

import numpy as np
import pytest
import torch
from scipy import stats

from helpers import small_batch, small_params, torch_batch, torch_params
from oracle.philox import philox4x32_10
from sampling_twin import SITE_SAMPLE, draw, generate_answers_sample, gumbel_keys, gumbel_of_words, sample_words
from visdial_b200 import engine as E


def test_gumbel_transform_known_answers():
    w = np.array([0, 0xFF, 0x100, 0x7FFFFFFF, 0x80000000, 0xFFFFFFFF], np.uint32)
    want = [-math.log(25 * math.log(2)),                                    # u = 2^-25 (the low 8 bits are dropped)
            -math.log(25 * math.log(2)),
            -math.log(24 * math.log(2) - math.log(1.5)),                    # u = 1.5 2^-24
            -math.log(-math.log(0.5 - 2 ** -25)),                           # the two sides of u = 1/2
            -math.log(-math.log(0.5 + 2 ** -25)),
            -math.log(-math.log1p(-2 ** -25))]                              # u = 1 - 2^-25: the largest g, 17.33
    np.testing.assert_allclose(gumbel_of_words(w), want, rtol=1e-12)
    assert gumbel_of_words(np.array([0xFFFFFFFF], np.uint32))[0] < 17.5    # GUMBEL_MAX of common.cuh bounds every g


def test_counter_layout():
    """element idx = (row_offset + r) V + j takes word idx % 4 of counter (idx // 4, 0, SITE_SAMPLE, step), key = seed"""
    seed, step, V = (7 << 32) | 1234, 3, 9
    w = sample_words(seed, step, 5, 3, V)
    for r in range(3):
        for j in range(V):
            idx = (5 + r) * V + j
            o = philox4x32_10(idx // 4, 0, SITE_SAMPLE, step, seed & 0xFFFFFFFF, seed >> 32)
            assert int(w[r, j]) == int(o[idx % 4])
    assert not np.array_equal(sample_words(seed, step + 1, 5, 3, V), w)
    assert not np.array_equal(sample_words(seed + 1, step, 5, 3, V), w)


def test_row_offset_selects_the_same_draws():
    rng = np.random.default_rng(0)
    x = rng.normal(size=(12, 37))
    full, _ = draw(x, 0.8, 99, 2, row_offset=0)
    for r0 in (1, 4, 7):
        part, _ = draw(x[r0:], 0.8, 99, 2, row_offset=r0)
        assert np.array_equal(part, full[r0:])
    np.testing.assert_array_equal(gumbel_keys(x[3:5], 0.8, 99, 2, 3), gumbel_keys(x, 0.8, 99, 2, 0)[3:5])


@pytest.mark.parametrize("T", [0.5, 1.0, 2.0])
def test_frequencies_match_the_tempered_softmax(T):
    """chi-square of 40 000 draws (one row of logits, every row index and step a fresh draw) against softmax(x / T)"""
    x = np.array([1.2, -0.3, 0.0, 2.1, -1.7, 0.4, 0.9])
    rows, steps = 8000, 5
    X = np.repeat(x[None], rows, 0)
    counts = np.zeros(len(x))
    for t in range(1, steps + 1):
        tok, _ = draw(X, T, 1234, t)
        counts += np.bincount(tok - 1, minlength=len(x))
    p = np.exp(x / T - np.max(x / T))
    p /= p.sum()
    chi2, pval = stats.chisquare(counts, p * rows * steps)
    assert pval > 1e-4, (chi2, pval, counts)


def test_low_temperature_gives_the_argmax():
    rng = np.random.default_rng(1)
    x = rng.normal(size=(500, 50)) * 2
    srt = np.sort(x, 1)
    keep = srt[:, -1] - srt[:, -2] >= 0.1
    assert keep.sum() > 300
    tok, _ = draw(x[keep], 1e-3, 5, 1)
    assert np.array_equal(tok - 1, np.argmax(x[keep], 1))


def test_oracle_sampler_feeds_its_own_tokens_and_respects_row_offset():
    """the model-level twin: deterministic per seed; its log-probabilities are the step decoder's at its own tokens; a
    shifted row_offset changes the draws"""
    p = small_params("hrea-ques-im-hist", "gen", vocabSize=9)
    P = torch_params(p, E.init_parameters(p, seed=3))
    b = torch_batch(small_batch(p, B=1, seed=5))
    V = p["vocabSize"]
    a, lp, gap = generate_answers_sample(p, P, b, V - 1, 6, 0.7, 11)
    a2, lp2, _ = generate_answers_sample(p, P, b, V - 1, 6, 0.7, 11)
    assert a.shape == (10, 7) and (a[:, 0] == V - 1).all() and ((a >= 1) & (a <= V)).all()
    assert np.array_equal(a, a2) and np.array_equal(lp, lp2)
    assert (lp <= 0).all() and (gap >= 0).all()
    # replay with the oracle's step decoder: the recorded log-probabilities are those of the fed-back tokens
    from oracle import visdial_oracle as O
    with torch.no_grad():
        encOut, state = O.ENCODERS[p["encoder"]](O.Ctx(train=False), p, P, O.prepare_inputs(p, b))
        H0, C0 = O.gen_forward_connect(state, encOut)
        H = [h if h is not None else encOut.new_zeros(encOut.shape) for h in H0]
        C = [c if c is not None else encOut.new_zeros(encOut.shape) for c in C0]
        for t in range(6):
            logp, H, C = O.decoder_gen_step(p, P, torch.from_numpy(a[:, t]), H, C)
            np.testing.assert_allclose(logp.double().numpy()[np.arange(10), a[:, t + 1] - 1], lp[:, t], rtol=0, atol=1e-12)
    a3, _, _ = generate_answers_sample(p, P, b, V - 1, 6, 0.7, 11, row_offset=10)
    assert not np.array_equal(a, a3)
