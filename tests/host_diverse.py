"""TEST INFRASTRUCTURE ONLY.  Host twin of diverse beam search (DESIGN §22): the merge rule of k_beam_merge as a pure numpy
step function, and a host search that drives a decoder step (host_decode.HostStep on the device, or any row-wise step) at
N * k rows exactly as host_decode.host_beam_search does, with the top k of every row taken from the same log-probability
bits.  G = 1 is the reference's merge (model.lua:529-569).

Candidate order.  Group g owns columns [g*w, (g+1)*w), w = k / G.  Its explored columns are all w (only its first at step
1); explored column e takes its w best top-k entries by (augmented desc, top-k position asc), augmented = (double)logp -
lam * n, n = the columns of groups < g filled at this step with the entry's token.  Candidate q = e * w + j is the j-th of
them; q orders the finished-hypothesis ties and the fill ties."""
import numpy as np

from host_decode import HostStep, start_state


def merge_step(stp, k, G, lam, L, end, topv, topi, scores, beams, ans, ans_len, ans_score, pick=False):
    """One merge of N searches.  topv / topi (N*k, k) float32 / int (0-based classes, a row's entries in (value desc,
    class asc) order), scores (N, k) float64, beams (N, k, L), ans (N, G, L), ans_len (N, G), ans_score (N, G).  Returns
    (scores, beams, tokens (N*k), parent (N*k), ans, ans_len, ans_score) as new arrays, followed with `pick` (the last
    step's merge) by the pick's answer (N, L), length (N) and score (N).  Positions of beams after stp are carried over
    unchanged; an unfilled column keeps its beam and score, writes a pad at stp and has parent -1 - row."""
    N = scores.shape[0]
    w = k // G
    ne = 1 if stp == 1 else w
    lamd = float(np.float32(lam))
    scores_o, beams_o = scores.copy(), beams.copy()
    ans, ans_len, ans_score = ans.copy(), ans_len.copy(), ans_score.copy()
    tokens = np.zeros(N * k, np.int32)
    parent = np.zeros(N * k, np.int32)
    for n in range(N):
        filled = []                                            # tokens of the filled columns of the groups so far
        for g in range(G):
            c0 = g * w
            cands = []                                         # (q, source column, token, s, a)
            for e in range(ne):
                col = c0 + e
                row = n * k + col
                ent = []
                for p in range(k):
                    tok = int(topi[row, p]) + 1
                    cnt = filled.count(tok)
                    ent.append((float(topv[row, p]) - lamd * cnt, p, tok, cnt))
                ent.sort(key=lambda t: (-t[0], t[1]))
                for j, (_, p, tok, cnt) in enumerate(ent[:w]):
                    s = float(scores[n, col]) + float(topv[row, p])
                    cands.append((e * w + j, col, tok, s, s - lamd * cnt if cnt else s))
            fin = [c for c in cands if c[2] == end]
            if fin:
                best = fin[0]
                for c in fin[1:]:
                    if c[3] > best[3]:
                        best = c
                if ans_len[n, g] == 0 or best[3] > ans_score[n, g]:
                    ans[n, g, :stp] = beams[n, best[1], :stp]
                    ans[n, g, stp] = end
                    ans_len[n, g], ans_score[n, g] = stp + 1, best[3]
            rest = sorted((c for c in cands if c[2] != end), key=lambda c: (-c[4], c[0]))[:w]
            for j in range(w):
                c, r = c0 + j, n * k + c0 + j
                if j < len(rest):
                    _, src, tok, s, _ = rest[j]
                    beams_o[n, c, :stp] = beams[n, src, :stp]
                    beams_o[n, c, stp] = tok
                    scores_o[n, c] = s
                    tokens[r], parent[r] = tok, n * k + src
                    filled.append(tok)
                else:
                    beams_o[n, c, stp] = 0
                    tokens[r], parent[r] = 0, -1 - r
    out = (scores_o, beams_o, tokens, parent, ans, ans_len, ans_score)
    if pick:
        out = out + pick_answers(ans, ans_len, ans_score)
    return out


def pick_index(length, score):
    """the group of the best finished hypothesis by (score desc, group asc), -1 when none"""
    best = -1
    for g in range(len(length)):
        if length[g] > 0 and (best < 0 or score[g] > score[best]):
            best = g
    return best


def pick_answers(ans, ans_len, ans_score):
    """each search's pick: (answer (N, L), length (N), score (N)), zeros where no group finished"""
    N, _, L = ans.shape
    pa, pl, ps = np.zeros((N, L), np.int32), np.zeros(N, np.int32), np.zeros(N, np.float64)
    for n in range(N):
        b = pick_index(ans_len[n], ans_score[n])
        if b >= 0:
            pa[n], pl[n], ps[n] = ans[n, b], ans_len[n, b], ans_score[n, b]
    return pa, pl, ps


def diverse_search(step, h, c, N, k, G, lam, L, start, end, stats=None):
    """The search on `step(tokens (N*k), h, c) -> (logp (N*k, V), h', c')` from the start state h, c (lists of (N*k, H)
    arrays).  Returns each group's (answer (N, G, L), length (N, G), score (N, G)).  `stats` counts columns left without a
    candidate ("stale"), pad tokens fed ("pad_rows") and the steps at which some group finished ("end_steps")."""
    beams = np.zeros((N, k, L), np.int32)
    beams[:, :, 0] = start
    scores = np.zeros((N, k), np.float64)
    ans, ans_len, ans_score = np.zeros((N, G, L), np.int32), np.zeros((N, G), np.int32), np.zeros((N, G), np.float64)
    tokens = np.full(N * k, start, np.int32)
    for stp in range(1, L):
        logp, out_h, out_c = step(tokens, h, c)
        top = np.argsort(-logp, axis=1, kind="stable")[:, :k]        # value desc, class asc
        topv = np.take_along_axis(logp, top, 1)
        if stats is not None:
            stats["pad_rows"] += int((tokens == 0).sum())
        before = ans_len.copy()
        scores, beams, tokens, parent, ans, ans_len, ans_score = merge_step(stp, k, G, lam, L, end, topv, top, scores, beams,
                                                                            ans, ans_len, ans_score)
        if stats is not None:
            stats["stale"] += int((parent < 0).sum())
            if (ans_len != before).any():
                stats["end_steps"].add(stp)
        keep = parent < 0
        src = np.where(keep, 0, parent)
        h = [np.where(keep[:, None], a, o[src]) for a, o in zip(h, out_h)]
        c = [np.where(keep[:, None], a, o[src]) for a, o in zip(c, out_c)]
    return ans, ans_len, ans_score


def host_diverse_beam_search(eng, encOut, k, G, lam, L, start, end, stats=None):
    """vd_gen_diverse_beam_search's search on the host for every round of the last encoder forward, the decoder stepped
    through vd_gen_decoder_step at N * k rows (host_decode.HostStep)."""
    N = encOut.shape[0]
    h, c = start_state(eng, encOut, k)
    with HostStep(eng, N * k) as step:
        return diverse_search(step, h, c, N, k, G, lam, L, start, end, stats)
