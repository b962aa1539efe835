"""TEST INFRASTRUCTURE ONLY.  numpy twin of the answer rules (visdial_b200/csrc/common.cuh's AnswerRules, DESIGN §25): the
barred set of a row at a step, the constrained top-k list the beam search merges, the merge's treatment of (-inf, -1)
entries, whole constrained searches driven by a decoder step (host_decode.HostStep) through host_nbest's merge, and the
constrained draws of sampling_twin / truncation_twin.  The existing twins are used as they are: a rule only removes classes
from a choice, so it is applied to their inputs (the top-k list, the Gumbel keys, the logits) and their outputs."""
import numpy as np

import sampling_twin
import truncation_twin
from host_decode import HostStep, start_state
from host_nbest import empty_lists, lp_table, nbest_merge_step


class Rules:
    """min_words m, no_repeat_ngram n (0 = off), banned token ids (1-based)"""

    def __init__(self, min_words=0, no_repeat_ngram=0, banned=()):
        self.min_words, self.no_repeat_ngram, self.banned = int(min_words), int(no_repeat_ngram), [int(b) for b in banned]

    @property
    def active(self):
        return self.min_words > 0 or self.no_repeat_ngram > 0 or bool(self.banned)


def barred(t, stp, V, end, rules):
    """bool (V,) of the classes (token - 1) barred at step stp for a row whose tokens are t (t[0] = <START>, t[1 .. stp-1]
    the answer so far; 0 = a pad)"""
    b = np.zeros(V, bool)
    for x in rules.banned:
        b[x - 1] = True
    if stp <= rules.min_words:
        b[end - 1] = True
    n = rules.no_repeat_ngram
    if n > 0:
        suffix = [int(x) for x in t[stp - n + 1:stp]]
        for j in range(1, stp - n + 1):
            win = [int(x) for x in t[j:j + n - 1]]
            w = int(t[j + n - 1])
            if 0 not in win and 0 not in suffix and win == suffix and w != 0 and w != end:
                b[w - 1] = True
    if b.all():
        b[end - 1] = False                                  # the fallback
    return b


def barred_rows(hist, stp, V, end, rules):
    """(rows, V) barred sets of every row of hist (rows, >= stp)"""
    return np.stack([barred(h, stp, V, end, rules) for h in hist])


def topk(logp, bar, k):
    """the k best allowed classes of every row by (value desc, class asc): (topv float32, topi int32), entries past a row's
    allowed count (-inf, -1).  A pad row's logp is all zeros, so it lists its first k allowed classes with value 0."""
    rows, V = logp.shape
    topv = np.full((rows, k), -np.inf, np.float32)
    topi = np.full((rows, k), -1, np.int32)
    for r in range(rows):
        cls = np.flatnonzero(~bar[r])
        o = cls[np.lexsort((cls, -logp[r, cls]))][:k]
        topv[r, :len(o)], topi[r, :len(o)] = logp[r, o], o
    return topv, topi


def unfill_empty(stp, scores, beams, out):
    """k_beam_merge's SKIP rule on a merge's outputs (scores_o, beams_o, tokens, parent, ...): host_diverse's merge ranks a
    (-inf, -1) entry after every real candidate, so it can only fill the columns no real candidate filled; such a column is
    restored to the unfilled form (its beam and score kept, a pad at stp, parent -1 - row)."""
    scores_o, beams_o, tokens, parent = [a.copy() for a in out[:4]]
    N, k = scores.shape
    for n in range(N):
        for c in range(k):
            if scores_o[n, c] == -np.inf:
                r = n * k + c
                scores_o[n, c] = scores[n, c]
                beams_o[n, c, :stp] = beams[n, c, :stp]
                beams_o[n, c, stp] = 0
                tokens[r], parent[r] = 0, -1 - r
    return (scores_o, beams_o, tokens, parent) + tuple(out[4:])


def rules_merge_step(stp, k, G, lam, lp, L, end, topv, topi, scores, beams, ans, length, score, norm):
    """host_nbest.nbest_merge_step with -inf entries taken as no candidate"""
    out = nbest_merge_step(stp, k, G, lam, lp, L, end, topv, topi, scores, beams, ans, length, score, norm)
    return unfill_empty(stp, scores, beams, out)


def rules_search(step, h, c, N, k, G, lam, alpha, nb, L, start, end, rules, check=None):
    """host_nbest.nbest_search under the rules: (answer (N, G, nb, L), length, score, norm).  `check(stp, beams, bar)`, if
    given, sees every step's pre-merge beams (N, k, L) and barred sets."""
    lp = lp_table(alpha, L) if alpha != 0 else None
    beams = np.zeros((N, k, L), np.int32)
    beams[:, :, 0] = start
    scores = np.zeros((N, k), np.float64)
    lists = empty_lists(N, G, nb, L)
    tokens = np.full(N * k, start, np.int32)
    for stp in range(1, L):
        logp, out_h, out_c = step(tokens, h, c)
        bar = barred_rows(beams.reshape(N * k, L), stp, logp.shape[1], end, rules)
        if check is not None:
            check(stp, beams, bar)
        topv, top = topk(logp, bar, k)
        scores, beams, tokens, parent, *lists = rules_merge_step(stp, k, G, lam, lp, L, end, topv, top, scores, beams,
                                                                 *lists)
        keep = parent < 0
        src = np.where(keep, 0, parent)
        h = [np.where(keep[:, None], a, o[src]) for a, o in zip(h, out_h)]
        c = [np.where(keep[:, None], a, o[src]) for a, o in zip(c, out_c)]
    return tuple(lists)


def host_rules_beam_search(eng, encOut, k, G, lam, alpha, nb, L, start, end, rules):
    """vd_gen_nbest_beam_search's search under the engine's rules on the host, stepped through vd_gen_decoder_step"""
    N = encOut.shape[0]
    h, c = start_state(eng, encOut, k)
    with HostStep(eng, N * k) as step:
        return rules_search(step, h, c, N, k, G, lam, alpha, nb, L, start, end, rules)


def sample_draw(x, bar, temperature, seed, step, row_offset=0, rounds=None):
    """sampling_twin.draw over the allowed classes: (1-based tokens, gap between the two best allowed keys)"""
    x = np.asarray(x, np.float32)
    if rounds is None:
        k = sampling_twin.gumbel_keys(x, temperature, seed, step, row_offset)
    else:
        k = np.concatenate([sampling_twin.gumbel_keys(x[i:i + 1], temperature, seed, step, int(rounds[i]))
                            for i in range(x.shape[0])])
    k = np.where(bar, -np.inf, k)
    cls = np.argmax(k, 1)
    s = -np.sort(-k, 1)
    gap = s[:, 0] - s[:, 1] if k.shape[1] > 1 else np.full(k.shape[0], np.inf)
    return cls + 1, np.where(np.isfinite(gap), gap, np.inf)


def truncated_draw(x, bar, temperature, seed, step, top_k, top_p, row_offset=0, rounds=None):
    """truncation_twin.draw over the allowed classes (barred ones out of the top-k count, the masses and the maximum): the
    row is restricted to its allowed classes, truncated, and its draw mapped back.  Returns (tokens, the sets of tokens an
    ambiguous boundary may draw, gap)."""
    x = np.asarray(x, np.float32)
    R, V = x.shape
    if rounds is None:
        keys = sampling_twin.gumbel_keys(x, temperature, seed, step, row_offset)
    else:
        keys = np.concatenate([sampling_twin.gumbel_keys(x[i:i + 1], temperature, seed, step, int(rounds[i]))
                               for i in range(R)])
    tok, either, gap = np.zeros(R, np.int64), [], np.full(R, np.inf)
    for r in range(R):
        cls = np.flatnonzero(~bar[r])
        o, n, n_lo, n_hi = truncation_twin.kept(x[r, cls], temperature, top_k, top_p)
        kk = keys[r, cls][o]
        opts = set()
        for m in sorted({n, n_lo, n_hi} | set(range(min(n, n_lo, n_hi), max(n, n_lo, n_hi) + 1))):
            km = np.where(np.arange(len(o)) < m, kk, -np.inf)
            opts.add(int(cls[o[np.lexsort((o, -km))[0]]]) + 1)
        km = np.where(np.arange(len(o)) < n, kk, -np.inf)
        tok[r] = int(cls[o[np.lexsort((o, -km))[0]]]) + 1
        s = np.sort(km[:n])
        gap[r] = s[-1] - s[-2] if n > 1 else np.inf
        either.append(opts)
    return tok, either, gap


def probabilities(x_row, bar_row, temperature, top_k=0, top_p=1.0):
    """the distribution a constrained (truncated) draw samples: the (truncated) softmax over the allowed classes"""
    cls = np.flatnonzero(~bar_row)
    p = np.zeros(len(bar_row))
    p[cls] = truncation_twin.probabilities(np.asarray(x_row)[cls], temperature, top_k, top_p)
    return p


def obeys(tokens, rules, finished=True):
    """whether an answer's tokens between <START> and <END> (a beam's pads included: a pad breaks n-grams) obey the rules
    when the fallback never applied: at least min_words words when it finished, no n-gram twice, no banned word"""
    tokens = [int(t) for t in tokens]
    words = [t for t in tokens if t]
    if finished and len(words) < rules.min_words:
        return False
    if any(w in rules.banned for w in words):
        return False
    n = rules.no_repeat_ngram
    if n > 0:
        grams = [tuple(tokens[i:i + n]) for i in range(len(tokens) - n + 1) if 0 not in tokens[i:i + n]]
        if len(grams) != len(set(grams)):
            return False
    return True
