"""TEST INFRASTRUCTURE ONLY.  Host twin of the beam search's n-best lists (DESIGN §24), on top of host_diverse.merge_step:
merge_step moves the live beams, and this module keeps each group's list of finished hypotheses.

The rule.  A finished hypothesis of `length` tokens has l = length - 1 generated tokens and norm = score / lp(l), lp(l) =
math.pow((5 + l) / 6, alpha) (the C library's pow, as the engine's host table) and an IEEE fp64 division.  A group's list
holds the n best of every <END> candidate the search met, by (norm desc, step asc, q asc), q the candidate index of
host_diverse.  The pick is the best list head by (norm desc, group asc).  Lists are given as their ordered arrays: answer
(N, G, n, L), length (N, G, n) (0: never filled), score and norm (N, G, n)."""
import math

import numpy as np

from host_decode import HostStep, start_state
from host_diverse import merge_step


def lp_table(alpha, L):
    """lp(l) for l = 0 .. L-1 at the engine's alpha (a float32 widened to fp64)"""
    a = float(np.float32(alpha))
    return np.array([math.pow((5.0 + l) / 6.0, a) for l in range(L)], np.float64)


def end_candidates(stp, k, G, lam, end, topv, topi, scores, tokens):
    """The <END> candidates of one merge, per search n and group g: [(q, source column, s)], s the unpenalised fp64
    score.  `tokens` (N*k) are the merge's filled tokens (0: unfilled), which set the penalties of later groups."""
    N = scores.shape[0]
    w = k // G
    ne = 1 if stp == 1 else w
    lamd = float(np.float32(lam))
    out = [[[] for _ in range(G)] for _ in range(N)]
    for n in range(N):
        for g in range(G):
            earlier = [int(t) for t in tokens[n * k:n * k + g * w] if t != 0]
            for e in range(ne):
                col = g * w + e
                row = n * k + col
                ent = sorted(range(k), key=lambda p: (-(float(topv[row, p]) - lamd * earlier.count(int(topi[row, p]) + 1)), p))
                for j, p in enumerate(ent[:w]):
                    if int(topi[row, p]) + 1 == end:
                        out[n][g].append((e * w + j, col, float(scores[n, col]) + float(topv[row, p])))
    return out


def list_step(stp, L, end, lp, beams, cands, ans, length, score, norm):
    """Each list after one merge's candidates `cands` (end_candidates) enter it; new arrays.  An earlier entry precedes a
    new one at equal norm (an earlier step), and new ones are ordered by q."""
    ans, length, score, norm = ans.copy(), length.copy(), score.copy(), norm.copy()
    N, G, nb = length.shape
    div = 1.0 if lp is None else float(lp[stp])
    for n in range(N):
        for g in range(G):
            old = [(float(norm[n, g, i]), 0, i, ans[n, g, i].copy(), int(length[n, g, i]), float(score[n, g, i]))
                   for i in range(nb) if length[n, g, i] > 0]
            new = []
            for q, col, s in cands[n][g]:
                row = np.zeros(L, np.int32)
                row[:stp] = beams[n, col, :stp]
                row[stp] = end
                new.append((s / div, 1, q, row, stp + 1, s))
            keep = sorted(old + new, key=lambda t: (-t[0], t[1], t[2]))[:nb]
            ans[n, g], length[n, g], score[n, g], norm[n, g] = 0, 0, 0.0, 0.0
            for i, (x, _, _, row, ln, s) in enumerate(keep):
                ans[n, g, i], length[n, g, i], score[n, g, i], norm[n, g, i] = row, ln, s, x
    return ans, length, score, norm


def pick_lists(ans, length, score, norm):
    """Each search's pick: the best list head by (norm desc, group asc).  (answer (N, L), length (N), score (N), group
    (N), -1 and zeros where no group finished)."""
    N, G, _, L = ans.shape
    pa, pl, ps, pg = np.zeros((N, L), np.int32), np.zeros(N, np.int32), np.zeros(N, np.float64), np.full(N, -1, np.int64)
    for n in range(N):
        best = -1
        for g in range(G):
            if length[n, g, 0] > 0 and (best < 0 or norm[n, g, 0] > norm[n, best, 0]):
                best = g
        if best >= 0:
            pa[n], pl[n], ps[n], pg[n] = ans[n, best, 0], length[n, best, 0], score[n, best, 0], best
    return pa, pl, ps, pg


def nbest_merge_step(stp, k, G, lam, lp, L, end, topv, topi, scores, beams, ans, length, score, norm):
    """One merge with lists: merge_step's (scores, beams, tokens, parent) and the lists after the step."""
    N = scores.shape[0]
    z = np.zeros((N, G, L), np.int32)
    scores_o, beams_o, tokens, parent = merge_step(stp, k, G, lam, L, end, topv, topi, scores, beams, z,
                                                   np.zeros((N, G), np.int32), np.zeros((N, G)))[:4]
    cands = end_candidates(stp, k, G, lam, end, topv, topi, scores, tokens)
    return (scores_o, beams_o, tokens, parent) + list_step(stp, L, end, lp, beams, cands, ans, length, score, norm)


def empty_lists(N, G, nb, L):
    return (np.zeros((N, G, nb, L), np.int32), np.zeros((N, G, nb), np.int32), np.zeros((N, G, nb)),
            np.zeros((N, G, nb)))


def nbest_search(step, h, c, N, k, G, lam, alpha, nb, L, start, end):
    """host_diverse.diverse_search with lists: (answer (N, G, nb, L), length, score, norm (N, G, nb))."""
    lp = lp_table(alpha, L) if alpha != 0 else None
    beams = np.zeros((N, k, L), np.int32)
    beams[:, :, 0] = start
    scores = np.zeros((N, k), np.float64)
    lists = empty_lists(N, G, nb, L)
    tokens = np.full(N * k, start, np.int32)
    for stp in range(1, L):
        logp, out_h, out_c = step(tokens, h, c)
        top = np.argsort(-logp, axis=1, kind="stable")[:, :k]        # value desc, class asc
        topv = np.take_along_axis(logp, top, 1)
        scores, beams_n, tokens, parent, *lists = nbest_merge_step(stp, k, G, lam, lp, L, end, topv, top, scores, beams,
                                                                   *lists)
        beams = beams_n
        keep = parent < 0
        src = np.where(keep, 0, parent)
        h = [np.where(keep[:, None], a, o[src]) for a, o in zip(h, out_h)]
        c = [np.where(keep[:, None], a, o[src]) for a, o in zip(c, out_c)]
    return tuple(lists)


def host_nbest_beam_search(eng, encOut, k, G, lam, alpha, nb, L, start, end):
    """vd_gen_nbest_beam_search's search on the host, the decoder stepped through vd_gen_decoder_step at N * k rows."""
    N = encOut.shape[0]
    h, c = start_state(eng, encOut, k)
    with HostStep(eng, N * k) as step:
        return nbest_search(step, h, c, N, k, G, lam, alpha, nb, L, start, end)
