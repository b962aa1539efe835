"""TEST INFRASTRUCTURE ONLY.  numpy twin of truncated sampling (visdial_b200/csrc/common.cuh's TruncCfg rule, DESIGN §23),
on top of sampling_twin's Gumbel keys.  For row r at step t: y = float32(x) / float32(T) (the device's fp32 division);
order the classes by (y desc, class asc); keep the first K (all when K is 0 or >= V); of those, with m = max y,
w = float32 exp(y - m) and q = rint(w 2^32) as uint64, S = the kept q's sum and tau = ceil(P S) in float64, keep the
shortest prefix whose cumulative q reaches tau (all when P = 1); the token is 1 + the argmax over the kept classes of
sampling_twin.gumbel_keys (the untruncated draw's keys).

numpy's float32 exp can differ from CUDA's expf by an ulp or two, which can move the top-p boundary when a prefix's
cumulative mass lies within that distance of tau.  `kept` therefore also returns the prefix lengths for the prefix masses
scaled against the total by 1 -/+ 2^-20: a row whose two lengths differ is boundary-ambiguous, and a device
result may take either."""
import numpy as np

from sampling_twin import gumbel_keys

AMBIGUITY = 2.0 ** -20


def order(y) -> np.ndarray:
    """class indices by (y desc, class asc), for one row"""
    return np.lexsort((np.arange(y.shape[0]), -y))


def _prefix_len(cum, tau) -> int:
    """the shortest prefix (>= 1) whose cumulative mass reaches tau"""
    return int(min(np.searchsorted(cum, tau, side="left") + 1, cum.shape[0]))


def kept(x_row, temperature: float, top_k: int, top_p: float, eps: float = 0.0, ambiguity: float = AMBIGUITY):
    """(classes in order, n, n_lo, n_hi) for one row: the kept classes are the first n of the order; n_lo / n_hi are n
    for a prefix mass `ambiguity` heavier / lighter against the total (equal to n unless the row is boundary-ambiguous).
    eps > 0 (logits known only to within eps, as replayed ones are) also widens the top-k boundary to the classes whose y
    is within eps of the K-th's."""
    y = np.asarray(x_row, np.float32) / np.float32(temperature)
    V = y.shape[0]
    o = order(y)
    K = lo_k = hi_k = top_k if 1 <= top_k < V else V
    if K < V and eps > 0:
        yk = y[o[K - 1]]
        lo_k, hi_k = max(1, int((y > yk + eps).sum())), int((y >= yk - eps).sum())
    if top_p >= 1.0:
        return o, K, lo_k, hi_k

    def prefix(m, scale):
        w = np.exp(y[o[:m]] - y.max()).astype(np.float32)
        q = np.rint(w.astype(np.float64) * 2.0 ** 32).astype(np.uint64)
        tau = int(np.ceil(np.float64(np.float32(top_p)) * np.float64(int(q.sum()))))
        # the integer rule on the exact cumulative sums (< 2^53, so float64 holds them exactly)
        return _prefix_len(np.cumsum(q).astype(np.float64) * scale, tau)
    n = prefix(K, 1.0)
    return o, n, min(n, prefix(lo_k, 1 + ambiguity)), max(n, prefix(hi_k, 1 - ambiguity))


def draw(x, temperature: float, seed: int, step: int, top_k: int, top_p: float, row_offset: int = 0, rounds=None,
         eps: float = 0.0, ambiguity: float = AMBIGUITY):
    """the truncated draw of every row of x (rows, V): (1-based tokens, the set of tokens some boundary between the
    ambiguous ones draws (just the token unless the row is boundary-ambiguous), the gap between the two best kept keys,
    kept-set masks (rows, V) for the smallest and the largest boundary).  rounds (rows) replaces row_offset + r as row
    r's global round; eps and ambiguity as kept's."""
    x = np.asarray(x, np.float32)
    R, V = x.shape
    if rounds is None:
        keys = gumbel_keys(x, temperature, seed, step, row_offset)
    else:
        keys = np.concatenate([gumbel_keys(x[i:i + 1], temperature, seed, step, int(rounds[i])) for i in range(R)])
    tok, gap = np.zeros(R, np.int64), np.full(R, np.inf)
    either = []
    small, large = np.zeros((R, V), bool), np.zeros((R, V), bool)
    for r in range(R):
        o, n, n_lo, n_hi = kept(x[r], temperature, top_k, top_p, eps, ambiguity)
        lo, hi = min(n, n_lo, n_hi), max(n, n_lo, n_hi)
        small[r, o[:lo]] = True
        large[r, o[:hi]] = True
        k = keys[r, o]                                   # keys in the rule's order
        # the first maximum of each prefix in class terms: argmax over o[:m] with ties to the lower class
        kk = np.where(np.arange(V) < n, k, -np.inf)
        c = o[np.lexsort((o, -kk))[0]]
        tok[r] = c + 1
        s = np.sort(kk[:n])
        gap[r] = s[-1] - s[-2] if n > 1 else np.inf
        opts = set()
        for m in range(lo, hi + 1):
            km = np.where(np.arange(V) < m, k, -np.inf)
            opts.add(int(o[np.lexsort((o, -km))[0]]) + 1)
        either.append(opts)
    return tok, either, gap, small, large


def probabilities(x_row, temperature: float, top_k: int, top_p: float) -> np.ndarray:
    """the renormalised truncated softmax(x / T) of one row, float64 (the distribution the rule draws from)"""
    o, n, _, _ = kept(x_row, temperature, top_k, top_p)
    y = np.asarray(x_row, np.float64) / temperature
    p = np.zeros(y.shape[0])
    k = o[:n]
    p[k] = np.exp(y[k] - y[k].max())
    return p / p.sum()
