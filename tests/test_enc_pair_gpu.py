"""The persistent encoder LSTM pair of enc_lstm.cu (k_enc_pair_fwd, k_enc_pair_bwd<GS>) step by step against fp64 numpy, through
vd_test_kernel, at the shapes and edges that switch its code paths.

The weights are one pair of SeqLSTM (D+H, 4H) weights, gate blocks [i f o g], rounded to fp16 and laid out as the engine lays
them out (engine.cu lstm_pair_forward / lstm_pair_backward): W1h16 = Wh1^T [4H, H], W2cat16 = [Wx2 | Wh2]^T [4H, 2H],
Whb2_16 = Wh2 [H, 4H], B1cat16 = [Wx2 | Wh1] [H, 8H].

References are teacher-forced: step t is computed in fp64 from the operands the kernel itself read at that step (its fp16 h of
step t-1, its fp32 c of step t-1; in the BPTT its fp16 da of step t+1), so only the fp32 accumulation of exact fp16 products and
the fast activations remain, and the bounds can be error scales of a single step.  U = 2^-24; a contraction of K fp16 products
accumulated in fp32 and then added to an fp32 term is within (K + 8) U sum|terms| of the exact sum.  fsigmoid / ftanh
(__expf, __fdividef) are within ACT_ABS absolute.  The BPTT's cell-gradient carry is free-running in fp64, as the kernel keeps it
in registers: its error bound is propagated step by step (it grows at most linearly, |f| < 1).  Outputs the code computes from the
same float, and the masked rows' zeros, are compared with ==.

Every output starts as NaN with GUARD_ROWS NaN rows after its T R rows, which must come back untouched."""
import numpy as np
import pytest
import torch

from helpers import Buf, call, lstm_step_bwd_ref, lstm_step_fwd_ref, run, small_params, within
from visdial_b200 import Engine
from visdial_b200._lib import VD_E_STATE

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
TINY = 2.0 ** -149           # fp32's smallest subnormal: the absolute rounding of results that underflow (T = 300 decays that far)
ACT_ABS = 5e-7               # fsigmoid / ftanh of tc_ptx.cuh: __expf (2 + 1.16|x| ulp) and __fdividef, over |x| < 16
GUARD_ROWS = 3
F16_NAN = 0x7e00


# ---------------------------------------------------------------------------------------------- plumbing
class Dev:
    """x (rows, ...) on the device followed by GUARD_ROWS rows of NaN (fp32, or fp16 passed as uint16 bits) or 0 (ints)"""

    def __init__(self, eng, x):
        x = np.ascontiguousarray(x)
        self.n = x.shape[0]
        self.fill = {np.dtype(np.float32): np.nan, np.dtype(np.uint16): F16_NAN, np.dtype(np.int32): 0,
                     np.dtype(np.int64): 0}[x.dtype]
        img = np.full((self.n + GUARD_ROWS,) + x.shape[1:], self.fill, x.dtype)
        img[:self.n] = x
        self.buf = Buf(eng, img)

    def ptr(self, off=0):
        return self.buf.ptr(off)

    def get(self):
        img = self.buf.get()
        guard = img[self.n:]
        if img.dtype == np.float32:
            assert np.isnan(guard).all(), "a kernel wrote into the guard rows"
        else:
            assert (guard == self.fill).all(), "a kernel wrote into the guard rows"
        return img[:self.n]


class Pool:
    def __init__(self, eng):
        self.eng, self.bufs = eng, []

    def __call__(self, x):
        d = Dev(self.eng, x)
        self.bufs.append(d)
        return d

    def out(self, shape, half=False):
        return self(np.full(shape, F16_NAN, np.uint16) if half else np.full(shape, np.nan, np.float32))

    def free(self):
        for d in self.bufs:
            d.buf.free()
        self.bufs = []


@pytest.fixture(scope="module")
def eng():
    e = Engine(small_params("lf-ques", "disc"))
    e.profile(True)                       # launches counted under their launch-site names (test_launches_counted)
    yield e
    e.close()


@pytest.fixture
def pool(eng):
    p = Pool(eng)
    yield p
    p.free()


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def groups_of(R, H):
    """the launchers' CTA groups: min(row blocks, SMs / CTAs per group)"""
    RB = -(-R // 128)
    return max(1, min(RB, sm_count() // (3 * H // 32)))


def uneven_rows(H):
    """a row count whose 128-row blocks outnumber the CTA groups and are no multiple of them: CTAs walk 2 or 3 blocks"""
    g = max(1, sm_count() // (3 * H // 32))
    return 2 * g * 128 + 77                   # 2 g + 1 blocks, the last one partial


def f16(x):
    """fp16-rounded values (float64) and their bits"""
    h = np.asarray(x, np.float32).astype(np.float16)
    return h.astype(np.float64), h.view(np.uint16)


def half_of(bits):
    return np.asarray(bits).view(np.float16).astype(np.float64)


def shift_prev(X, T, R):
    """rows of step t-1 at step t, zero at t = 0"""
    Y = np.zeros_like(X)
    Y[R:] = X[:(T - 1) * R]
    return Y


def shift_next(X, T, R):
    """rows of step t+1 at step t, zero at t = T-1"""
    Y = np.zeros_like(X)
    Y[:(T - 1) * R] = X[R:]
    return Y


def engine_mask(T, R, seed):
    """time-major token ids as the engine feeds them, 0 = pad: right-aligned sequences (pads first) of random length,
    all-pad rows, pads in the middle of a sequence, and rows 0, 63, 64, 127, 128, R-1 masked at t = 0 or t = T-1 only"""
    rng = np.random.default_rng(seed)
    L = rng.integers(0, T + 1, R)
    L[np.arange(R) % 13 == 5] = 0
    ids = np.where(np.arange(T)[:, None] >= T - L[None, :], rng.integers(1, 1000, (T, R)), 0).astype(np.int32)
    if T > 2:
        mid = np.flatnonzero(np.arange(R) % 11 == 3)
        ids[:, mid] = rng.integers(1, 1000, (T, mid.size))
        ids[T // 2, mid] = 0
    for r, t in ((0, 0), (63, T - 1), (64, 0), (127, T - 1), (128, 0), (R - 1, T - 1)):
        if r < R:
            ids[:, r] = rng.integers(1, 1000, T)
            ids[t, r] = 0
    return ids


class Pair:
    """one pair of fp16-rounded SeqLSTM weights (fp64 values) and the engine's fp16 layouts (bits)"""

    def __init__(self, H, seed):
        rng = np.random.default_rng(seed)
        self.H = H
        self.Wh1, self.Wx2, self.Wh2 = (f16(rng.standard_normal((H, 4 * H)) / np.sqrt(H))[0] for _ in range(3))
        self.bias2 = np.asarray(0.5 * rng.standard_normal(4 * H), np.float32)
        self.W1h16 = f16(self.Wh1.T)[1]
        self.W2cat16 = f16(np.concatenate([self.Wx2, self.Wh2], 0).T)[1]
        self.Whb2_16 = f16(self.Wh2)[1]
        self.B1cat16 = f16(np.concatenate([self.Wx2, self.Wh1], 1))[1]


# ---------------------------------------------------------------------------------------------- forward
def run_forward(eng, pool, W, T, R, G1in, ids):
    H, TR = W.H, T * R
    o = dict(gates1=pool(G1in), c1=pool.out((TR, H)), h1=pool.out((TR, H)), h1_16=pool.out((TR, H), True),
             gates2=pool.out((TR, 4 * H)), c2=pool.out((TR, H)), h2=pool.out((TR, H)), h2_16=pool.out((TR, H), True))
    flags = pool(np.zeros(3 * (-(-R // 128)) * T, np.int32))
    run(eng, "enc_pair_forward",
        [pool(W.W1h16), pool(W.W2cat16), pool(W.bias2), pool(ids.reshape(-1)), o["gates1"], o["c1"], o["h1"], o["h1_16"],
         o["gates2"], o["c2"], o["h2"], o["h2_16"], flags], [T, R, H])
    return {k: v.get() for k, v in o.items()}


def cell_bounds(a, cp, c, dz):
    """error bounds of the activated gates, c and h of one step from the bound dz of the pre-activation"""
    H = a.shape[1] // 4
    i, f, o, g = a[:, :H], a[:, H:2 * H], a[:, 2 * H:3 * H], a[:, 3 * H:]
    ea = np.concatenate([a[:, :3 * H] * (1 - a[:, :3 * H]), 1 - g * g], 1) * dz + ACT_ABS
    ei, ef, eo, eg = ea[:, :H], ea[:, H:2 * H], ea[:, 2 * H:3 * H], ea[:, 3 * H:]
    ec = np.abs(cp) * ef + np.abs(g) * ei + np.abs(i) * eg + 3 * U * (np.abs(f * cp) + np.abs(i * g))
    tc = np.tanh(c)
    eh = eo * np.abs(tc) + np.abs(o) * (ec * (1 - tc * tc) + ACT_ABS) + 2 * U * np.abs(o * tc)
    return ea, ec, eh


def check_forward(W, T, R, G1in, ids, got, tag):
    """teacher-forced: step t from the kernel's own h*_16[t-1] and c*[t-1]; layer 2 from its own h1_16[t]"""
    H = W.H
    m = ids.reshape(-1) == 0
    G1 = np.asarray(G1in, np.float64).reshape(T * R, 4 * H)
    b2 = W.bias2.astype(np.float64)
    h1_16, h2_16 = half_of(got["h1_16"]), half_of(got["h2_16"])
    c1p, c2p = shift_prev(got["c1"].astype(np.float64), T, R), shift_prev(got["c2"].astype(np.float64), T, R)
    h1p, h2p = shift_prev(h1_16, T, R), shift_prev(h2_16, T, R)
    layers = (
        ("1", G1, h1p, W.Wh1, c1p, np.abs(G1) + np.abs(h1p) @ np.abs(W.Wh1)),
        ("2", h1_16 @ W.Wx2 + b2, h2p, W.Wh2, c2p, np.abs(h1_16) @ np.abs(W.Wx2) + np.abs(b2) + np.abs(h2p) @ np.abs(W.Wh2)),
    )
    for L, zx, hp, Wh, cp, S in layers:
        a, c, h = lstm_step_fwd_ref(zx, hp, Wh, cp, m)
        ea, ec, eh = cell_bounds(a, cp, c, (H + 8) * U * S)
        for name, ref, bound in (("gates", a, ea), ("c", c, ec), ("h", h, eh)):
            g = got[name + L]
            within(g, ref, bound, "%s %s%s" % (tag, name, L))
            assert (g[m] == 0).all(), (tag, name + L, "masked rows must be exact zeros")
        h16 = got["h%s_16" % L]
        assert (h16 == got["h" + L].astype(np.float16).view(np.uint16)).all(), (tag, "h%s_16 is not fp16(h%s)" % (L, L))


def fwd64(W, T, R, G1in, ids):
    """free-running fp64 forward of the pair (fp16-rounded weights, nothing else rounded): gates, c, h of both layers"""
    H = W.H
    m = ids.reshape(T, R) == 0
    G1 = np.asarray(G1in, np.float64).reshape(T, R, 4 * H)
    out = {k: np.zeros((T, R, 4 * H if k.startswith("gates") else H)) for k in ("gates1", "c1", "h1", "gates2", "c2", "h2")}
    for t in range(T):
        hp1, cp1 = (out["h1"][t - 1], out["c1"][t - 1]) if t else (None, None)
        out["gates1"][t], out["c1"][t], out["h1"][t] = lstm_step_fwd_ref(G1[t], hp1, W.Wh1, cp1, m[t])
        hp2, cp2 = (out["h2"][t - 1], out["c2"][t - 1]) if t else (None, None)
        zx2 = out["h1"][t] @ W.Wx2 + W.bias2.astype(np.float64)
        out["gates2"][t], out["c2"][t], out["h2"][t] = lstm_step_fwd_ref(zx2, hp2, W.Wh2, cp2, m[t])
    return {k: v.reshape(T * R, -1) for k, v in out.items()}


# shapes: KB = H/64 from 1 to 8, the unit split (H = 64, 192) and the gate split (others); R at the 64-row minimum (warpgroup 1's
# rows all invalid), around a block edge, the benched 320, and uneven_rows (several row blocks per CTA group); T = 1 (no
# recurrent contraction), 2, 20, 40 and the 300-token concatenated history of the lf encoders
CASES = [(64, 64, 20), (64, 127, 2), (64, "uneven", 20),
         (128, 128, 40), (128, 129, 1), (128, "uneven", 20),
         (192, 320, 20), (192, "uneven", 2), (192, 64, 40),
         (256, 64, 1), (256, 320, 20), (256, "uneven", 20),
         (384, 129, 40), (384, "uneven", 20),
         (512, 320, 40), (512, 64, 2), (512, "uneven", 20), (512, 128, 1), (512, 64, 300)]


def case_id(c):
    return "H%d-R%s-T%d" % c


def shape(c):
    H, R, T = c
    return H, uneven_rows(H) if R == "uneven" else R, T


def forward_inputs(H, R, T, seed):
    rng = np.random.default_rng(seed)
    return np.asarray(rng.standard_normal((T * R, 4 * H)), np.float32), engine_mask(T, R, seed)


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_forward(eng, pool, case):
    H, R, T = shape(case)
    if case[1] == "uneven":
        RB, g = -(-R // 128), groups_of(R, H)
        assert RB > g and (g == 1 or RB % g != 0), (RB, g)
    W = Pair(H, 11 + H)
    G1in, ids = forward_inputs(H, R, T, H + R + T)
    got = run_forward(eng, pool, W, T, R, G1in, ids)
    check_forward(W, T, R, G1in, ids, got, case_id(case))


# ---------------------------------------------------------------------------------------------- BPTT
LAST = ("dh_last1", "dc_last1", "dh_last2", "dc_last2")


def bwd_inputs(W, T, R, seed, present=LAST, factor=1.0):
    """saved activations of a free-running fp64 forward (fp32), the mask, and the present last-step gradients (R, H)"""
    H = W.H
    G1in, ids = forward_inputs(H, R, T, seed)
    fw = fwd64(W, T, R, G1in, ids)
    rng = np.random.default_rng(seed + 1)
    last = {k: np.asarray(rng.standard_normal((R, H)) * factor, np.float32) if k in present else None for k in LAST}
    return {k: np.asarray(fw[k], np.float32) for k in ("gates1", "c1", "gates2", "c2")}, ids, last, fw


def flag_ints(eng, pool, T, R, H):
    n = pool(np.zeros(1, np.int64))
    run(eng, "enc_pair_bwd_flag_ints", [n], [T, R, H])
    return int(n.get()[0])


def run_backward(eng, pool, W, T, R, saved, ids, last, gate_split):
    H, TR = W.H, T * R
    o = dict(da1=pool.out((TR, 4 * H)), da1_16=pool.out((TR, 4 * H), True), da2=pool.out((TR, 4 * H)),
             da2_16=pool.out((TR, 4 * H), True), scale=pool.out(2))
    flags = pool(np.zeros(flag_ints(eng, pool, T, R, H), np.int32))
    dh = [pool.out((TR, H)), pool.out((TR, H))] if gate_split else [None, None]
    run(eng, "enc_pair_backward",
        [pool(W.B1cat16), pool(W.Whb2_16), pool(ids.reshape(-1)), pool(saved["gates1"]), pool(saved["c1"]), pool(saved["gates2"]),
         pool(saved["c2"])] + [None if last[k] is None else pool(last[k]) for k in LAST] +
        [o["da1"], o["da1_16"], o["da2"], o["da2_16"], flags] + dh + [o["scale"]], [T, R, H])
    got = {k: v.get() for k, v in o.items()}
    got["s"] = float(got["scale"][0])
    return got


def layer_bwd_ref(gates, c, dh, edh, dc_last, m, T, R):
    """free-running fp64 SeqLSTM backward pointwise over the sequence with its error bound: dh (T R, H) is the full gradient
    wrt h_t (teacher-forced recurrent part + dh_last), edh its bound; the dc carry and its bound run step by step"""
    H = c.shape[1]
    da, eda = np.zeros((T * R, 4 * H)), np.zeros((T * R, 4 * H))
    dc = np.zeros((R, H)) if dc_last is None else np.asarray(dc_last, np.float64)
    edc = np.zeros((R, H))
    for t in reversed(range(T)):
        sl = slice(t * R, (t + 1) * R)
        a, ct = np.asarray(gates[sl], np.float64), np.asarray(c[sl], np.float64)
        cp = np.asarray(c[sl.start - R:sl.start], np.float64) if t else np.zeros((R, H))
        da[sl], dc_new = lstm_step_bwd_ref(a, cp, ct, dh[sl], dc, m[sl])
        i, f, o, g = a[:, :H], a[:, H:2 * H], a[:, 2 * H:3 * H], a[:, 3 * H:]
        tc = np.tanh(ct)
        dht, e_dh = np.abs(dh[sl]), edh[sl]
        d = np.abs(dc + dh[sl] * o * (1 - tc * tc))
        ed = edc + e_dh * o * (1 - tc * tc) + dht * o * 2 * np.abs(tc) * ACT_ABS + 3 * U * (np.abs(dc) + d) + 4 * TINY
        ea = np.concatenate([ed * np.abs(g * i * (1 - i)), ed * np.abs(cp * f * (1 - f)),
                             e_dh * np.abs(tc * o * (1 - o)) + dht * o * (1 - o) * ACT_ABS, ed * np.abs(i * (1 - g * g))], 1)
        eda[sl] = ea + 4 * U * np.abs(da[sl]) + 4 * TINY
        edc = ed * f + U * d * f
        edc[m[sl]] = 0
        dc = dc_new
    return da, eda


def bwd_teacher_ref(W, T, R, saved, ids, last, got):
    """teacher-forced BPTT reference: dh2_t = da2_16[t+1] Wh2^T (+ dh_last2), dh1_t = da2_16[t] Wx2^T + da1_16[t+1] Wh1^T
    (+ dh_last1), the fp16 da divided by the kernel's scale s"""
    H, s = W.H, got["s"]
    m = ids.reshape(-1) == 0
    A2, A1 = half_of(got["da2_16"]) / s, half_of(got["da1_16"]) / s
    A2n, A1n = shift_next(A2, T, R), shift_next(A1, T, R)
    out = {}
    for L, dh, S, K in (("2", A2n @ W.Wh2.T, np.abs(A2n) @ np.abs(W.Wh2.T), 4 * H),
                        ("1", A2 @ W.Wx2.T + A1n @ W.Wh1.T, np.abs(A2) @ np.abs(W.Wx2.T) + np.abs(A1n) @ np.abs(W.Wh1.T), 8 * H)):
        if last["dh_last" + L] is not None:
            dh[(T - 1) * R:] += last["dh_last" + L]
            S[(T - 1) * R:] += np.abs(last["dh_last" + L])
        out[L] = layer_bwd_ref(saved["gates" + L], saved["c" + L], dh, (K + 8) * U * S, last["dc_last" + L], m, T, R)
    return out


def check_backward(W, T, R, saved, ids, last, got, tag):
    m = ids.reshape(-1) == 0
    s = got["s"]
    assert s > 0 and np.log2(s) == np.round(np.log2(s)), (tag, "scale is not a power of two", s)
    assert got["scale"][1] == np.float32(1.0 / s)
    refs = bwd_teacher_ref(W, T, R, saved, ids, last, got)
    for L in ("1", "2"):
        da, da16 = got["da" + L], got["da%s_16" % L]
        within(da, refs[L][0], refs[L][1], "%s da%s" % (tag, L))
        assert (da[m] == 0).all() and (half_of(da16[m]) == 0).all(), (tag, "masked rows of da%s must be (signed) zeros" % L)
        want16 = np.clip(da * np.float32(s), -65504, 65504).astype(np.float16).view(np.uint16)
        assert (da16 == want16).all(), (tag, "da%s_16 is not fp16(s da%s)" % (L, L))
    return refs


def presence(k):
    return tuple(n for j, n in enumerate(LAST) if k >> j & 1)


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_backward(eng, pool, case):
    """the engine's split (gate split at H % 128 == 0); the last-step gradients the history pair (dh_last2) or the gen question
    pair (all four) passes, alternately"""
    H, R, T = shape(case)
    W = Pair(H, 11 + H)
    present = ("dh_last2",) if CASES.index(case) % 2 else LAST
    saved, ids, last, _ = bwd_inputs(W, T, R, H + R + T, present)
    got = run_backward(eng, pool, W, T, R, saved, ids, last, gate_split=H % 128 == 0)
    check_backward(W, T, R, saved, ids, last, got, case_id(case))


@pytest.mark.parametrize("H,R,T", [(256, 320, 20), (256, 129, 1), (512, "uneven", 20), (128, 64, 40)])
def test_backward_splits_agree(eng, pool, H, R, T):
    """the unit split at H % 128 == 0 (null dh1 / dh2), which the engine does not take there, against its own reference and
    against the gate split on the same inputs: layer 2's last step has no contraction and must be bit-identical; elsewhere the
    two differ by fp32 re-association, which an fp16 rounding of da may turn into one fp16 ulp (2^-11) fed to later steps"""
    R = uneven_rows(H) if R == "uneven" else R
    W = Pair(H, 5 + H)
    saved, ids, last, _ = bwd_inputs(W, T, R, 3 * H + R + T)
    gs = run_backward(eng, pool, W, T, R, saved, ids, last, gate_split=True)
    us = run_backward(eng, pool, W, T, R, saved, ids, last, gate_split=False)
    check_backward(W, T, R, saved, ids, last, us, "unit split")
    assert gs["s"] == us["s"]
    last_rows = slice((T - 1) * R, T * R)
    assert (gs["da2"][last_rows] == us["da2"][last_rows]).all()
    for L in ("1", "2"):
        a, b = gs["da" + L].reshape(T, -1), us["da" + L].reshape(T, -1)
        step_max = np.abs(a).max(1, keepdims=True)
        within(b, a, 2.0 ** -9 * step_max + 1e-30, "gate vs unit split, da" + L)


@pytest.mark.parametrize("k", range(16), ids=lambda k: "+".join(presence(k)) or "none")
def test_backward_last_inputs(eng, pool, k):
    """every presence pattern of dh_last1, dc_last1, dh_last2, dc_last2, on both splits"""
    H, R, T = 128, 129, 3
    W = Pair(H, 77)
    saved, ids, last, _ = bwd_inputs(W, T, R, 900 + k, presence(k))
    for gate_split in (True, False):
        got = run_backward(eng, pool, W, T, R, saved, ids, last, gate_split)
        check_backward(W, T, R, saved, ids, last, got, "%s gs=%d" % (presence(k), gate_split))
        if not presence(k):
            assert got["s"] == 1.0
            assert (got["da1"] == 0).all() and (got["da2"] == 0).all()


@pytest.mark.parametrize("gate_split", [True, False], ids=["gate-split", "unit-split"])
def test_gradient_scale_sweep(eng, pool, gate_split):
    """dh_last* / dc_last* times 1, 2^-10, 2^-20.  Powers of two are exact, so da / factor must stay within the factor-1 run's
    bound of the factor-1 run; with the BPTT's power-of-two scale the unit split is bit-identical across factors.  fp16 da must
    not hold zeros where the factor-1 run's does not."""
    H, R, T = 256, 129, 20
    W = Pair(H, 31)
    saved, ids, last, _ = bwd_inputs(W, T, R, 4321)
    base = run_backward(eng, pool, W, T, R, saved, ids, last, gate_split)
    refs = check_backward(W, T, R, saved, ids, last, base, "factor 1")
    for e in (10, 20):
        f = 2.0 ** -e
        got = run_backward(eng, pool, W, T, R, saved, ids, {k: v * np.float32(f) for k, v in last.items()}, gate_split)
        errs = {L: float(np.abs(got["da" + L] / f - base["da" + L]).max() / np.abs(base["da" + L]).max()) for L in ("1", "2")}
        print("scale sweep %s factor 2^-%d: s = 2^%d, max|da/f - da(f=1)| / max|da(f=1)| = %.3g (layer 1), %.3g (layer 2)"
              % ("gate split" if gate_split else "unit split", e, int(np.log2(got["s"])), errs["1"], errs["2"]))
        for L in ("1", "2"):
            # the gate split's red.add order changes from run to run, so an element within its bound of fp16's underflow
            # threshold may round to zero in one run and not in the other
            clear = np.abs(base["da" + L]) > 2 * refs[L][1] + 2.0 ** -24 / base["s"]
            lost = (got["da%s_16" % L] == 0) & (base["da%s_16" % L] != 0) & clear
            assert not lost.any(), ("factor 2^-%d" % e, "fp16 da%s flushed to zero in %d elements" % (L, lost.sum()))
            within(got["da" + L] / f, base["da" + L], 2 * refs[L][1], "factor 2^-%d da%s" % (e, L))
            if not gate_split:
                assert (got["da" + L] / f == base["da" + L]).all(), ("factor 2^-%d" % e, "unit split not bit-identical")


# ---------------------------------------------------------------------------------------------- end to end
@pytest.mark.parametrize("magnitude", ["unit", "b32"])
def test_free_running_pair(eng, pool, magnitude):
    """T = 20, H = 512, R = 320: the kernel's forward and BPTT over the whole sequence (the BPTT on the forward's outputs)
    against an fp64 forward and BPTT with nothing rounded but the weights.  F16-class bound: fp16 h and da carry a relative
    rounding of 2^-11 per step; the bound is 2^-7 of each step's largest reference value, per output.
    "unit": all four last-step gradients ~N(0, 1).  "b32": the history pair's dh_last2 alone, drawn at the magnitudes of the
    reference model's disc training step at B = 32 (max |dL/dh| ~8e-4, median ~1e-5): da there is ~1e-6, in the fp16 subnormal
    range unless the BPTT scales it."""
    H, R, T = 512, 320, 20
    W = Pair(H, 2024)
    G1in, ids = forward_inputs(H, R, T, 99)
    rng = np.random.default_rng(100)
    if magnitude == "unit":
        last = {k: np.asarray(rng.standard_normal((R, H)), np.float32) for k in LAST}
    else:
        x = np.exp(rng.standard_normal((R, H)) + np.log(1.1e-5)) * rng.choice([-1.0, 1.0], (R, H))
        last = {k: None for k in LAST}
        last["dh_last2"] = np.asarray(np.clip(x, -8e-4, 8e-4), np.float32)
    fw = run_forward(eng, pool, W, T, R, G1in, ids)
    ref = fwd64(W, T, R, G1in, ids)
    for k in ("gates1", "c1", "h1", "gates2", "c2", "h2"):
        a, b = fw[k].reshape(T, -1), ref[k].reshape(T, -1)
        within(a, b, 2.0 ** -7 * np.abs(b).max(1, keepdims=True), "free-running forward " + k)
    saved = {k: fw[k] for k in ("gates1", "c1", "gates2", "c2")}
    got = run_backward(eng, pool, W, T, R, saved, ids, last, gate_split=True)
    m = ids.reshape(-1) == 0
    z = np.zeros((T * R, H))
    dh2 = z.copy()
    dc2 = None if last["dc_last2"] is None else last["dc_last2"]
    dh1 = z.copy()
    if last["dh_last2"] is not None:
        dh2[(T - 1) * R:] = last["dh_last2"]
    if last["dh_last1"] is not None:
        dh1[(T - 1) * R:] = last["dh_last1"]
    # fp64 BPTT, layer 2 then layer 1, step by step with the recurrence in fp64
    da = {}
    for L, Wh, dh_ext, dcl in (("2", W.Wh2, dh2, dc2), ("1", W.Wh1, dh1, last["dc_last1"])):
        if L == "1":
            dh_ext = dh_ext + da["2"] @ W.Wx2.T
        g, c = saved["gates" + L], saved["c" + L]
        out = np.zeros((T * R, 4 * H))
        dc = np.zeros((R, H)) if dcl is None else np.asarray(dcl, np.float64)
        rec = np.zeros((R, H))
        for t in reversed(range(T)):
            sl = slice(t * R, (t + 1) * R)
            cp = c[sl.start - R:sl.start] if t else None
            out[sl], dc = lstm_step_bwd_ref(g[sl], cp, c[sl], dh_ext[sl] + rec, dc, m[sl])
            rec = out[sl] @ Wh.T
        da[L] = out
    for L in ("1", "2"):
        a, b = got["da" + L].reshape(T, -1), da[L].reshape(T, -1)
        print("free-running %s: da%s max error / step max = %.3g, s = 2^%d"
              % (magnitude, L, float((np.abs(a - b) / np.abs(b).max(1, keepdims=True)).max()), int(np.log2(got["s"]))))
    for L in ("1", "2"):
        a, b = got["da" + L].reshape(T, -1), da[L].reshape(T, -1)
        within(a, b, 2.0 ** -7 * np.abs(b).max(1, keepdims=True), "free-running BPTT da" + L)


# ---------------------------------------------------------------------------------------------- determinism, refusals, counts
def test_deterministic(eng, pool):
    """the forward and the unit-split BPTT have no atomics: two runs on the same inputs agree bit for bit"""
    H, R, T = 256, 320, 20
    W = Pair(H, 8)
    G1in, ids = forward_inputs(H, R, T, 8)
    a, b = (run_forward(eng, pool, W, T, R, G1in, ids) for _ in range(2))
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), k
    saved, ids, last, _ = bwd_inputs(W, T, R, 9)
    a, b = (run_backward(eng, pool, W, T, R, saved, ids, last, gate_split=False) for _ in range(2))
    for k in ("da1", "da2", "da1_16", "da2_16"):
        assert a[k].tobytes() == b[k].tobytes(), k


@pytest.mark.parametrize("H,R", [(96, 128), (576, 128), (64, 63)])
def test_refused_shape(eng, pool, H, R):
    """enc_pair_shape_ok: H % 64, H > 512, R < 64 come back as VD_E_STATE, and the next valid call still succeeds"""
    T = 2
    dummy = pool(np.zeros(64, np.float32))
    assert call(eng, "enc_pair_forward", [dummy] * 13, [T, R, H]) == VD_E_STATE
    assert call(eng, "enc_pair_backward", [dummy] * 19, [T, R, H]) == VD_E_STATE
    W = Pair(64, 3)
    G1in, ids = forward_inputs(64, 64, T, 3)
    check_forward(W, T, 64, G1in, ids, run_forward(eng, pool, W, T, 64, G1in, ids), "after refusal")


def test_launches_counted(eng):
    """runs last: vd_kernel_stats counts the kernels under their launch-site names"""
    for name in ("k_enc_pair_fwd", "k_enc_pair_bwd", "k_ep_pick_scale"):
        assert eng.kernel_stats(name)["launches"] > 0, name
