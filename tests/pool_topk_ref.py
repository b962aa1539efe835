"""TEST INFRASTRUCTURE ONLY.  numpy reference of the answer-pool top-k (DESIGN §18): per row the k best pool rows by
(score desc, pool index asc), the tie rule of utils.computeRanks / k_rank_rows and the top-k kernels."""
import numpy as np


def topk_rows(scores, k):
    """scores (rows, m) -> (index (rows, k) int32, value (rows, k) as scores' dtype)"""
    scores = np.asarray(scores)
    rows, m = scores.shape
    assert 1 <= k <= m
    idx = np.empty((rows, k), np.int32)
    for r in range(rows):
        s = scores[r]
        thr = np.partition(s, m - k)[m - k]              # the k-th largest value: every row of the answer is >= it
        cand = np.nonzero(s >= thr)[0]
        order = np.lexsort((cand, -s[cand]))            # score desc, then index asc
        idx[r] = cand[order[:k]]
    return idx, np.take_along_axis(scores, idx, 1)


def pool_topk(Q, E, k, chunk=128):
    """the k best rows of E (m, H) for every row of Q (rows, H), scores in float64"""
    Q = np.asarray(Q, np.float64)
    E = np.asarray(E, np.float64)
    out_i, out_v = [], []
    for r0 in range(0, Q.shape[0], chunk):
        i, v = topk_rows(Q[r0:r0 + chunk] @ E.T, k)
        out_i.append(i)
        out_v.append(v)
    return np.concatenate(out_i), np.concatenate(out_v)
