"""Whole SeqLSTM runs of the engine (Engine::lstm_forward / lstm_backward / lstm_pair_forward / lstm_pair_backward, routed by
route_lstm / route_lstm_pair) against the fp64 SeqLSTM of tests/seq_lstm_ref.py, through vd_test_kernel's seq_lstm and
seq_lstm_pair entries.  Each case asserts its route (info) against a Python mirror of the engine's predicates, then its outputs.

Checks and bounds.  U = 2^-24; S = the sum of the absolute terms of a pre-activation or a contraction, sum_k |a_k b_k|.
* Teacher-forced steps: step t is recomputed in fp64 from the state the device saved at t-1 (its h, c; fp16 h on Opt16), and in
  the BPTT from the device's da_{t+1}; the cell-gradient carry runs free and its bound is propagated step by step, as in
  test_enc_pair_gpu.py.  A pre-activation (K = D + H terms) or a recurrent gradient (K = 4H terms) is within
  fp32 (VD_MATH_FP32):   (K + 2) U S
  TF32 (tensor-core modes): (2^-9 + (K + 2) U) S       (both operands cut to a 10-bit mantissa: 2^-10 each, as in §7)
  and the activations add 5e-7 (the fast sigmoid / tanh of the step kernels).  Opt16's fp16 steps are held to
  test_lstm16_step_gpu.py's 4e-3 (1 + |ref|) in the forward; its BPTT reads fp16 Wh (2^-11 S) and tanh.approx (2^-10) and stores
  fp16(s da) (2^-11 relative, 2^-25 / s absolute).
* Weight, bias, input and embedding gradients are recomputed from the device's own operands (its saved h and da; on Opt16 its
  fp16 h and da16 / s), element by element, within the GEMM primitive bound of §7 scaled by that element's S: (K + 2) U S for
  fp32 accumulation (Opt16's fp16 weight gradient, whose operands are exact, and every reduction in VD_MATH_FP32), plus 2^-9 S
  where a tensor-core mode may run the contraction in TF32.  K is the whole accumulation chain (T R, plus V + 1 for the table).
* Free-running: the device's h / c / da against the fp64 reference run from the inputs alone.  VD_MATH_FP32 within 1e-5 of each
  step's largest value (fp32 re-association over 20 steps); TF32 and F16 within 3e-2 of it, a bound for wiring errors, which
  are O(0.1).
Every output starts as NaN between NaN guard bands, which must come back untouched; masked rows must be exact zeros.

The shadow-alignment clause of lstm_step_fwd_tc_ok / lstm_step_bwd_tc_ok (tma_ok) cannot fail on a layout segment: every segment
starts 128-byte aligned, D % 4 == 0 and H % 32 == 0.  test_tma_ok_holds_on_every_segment says so, and the Simt-both-ways case in
a tensor-core mode is H = 96 (H % 64 != 0)."""
import numpy as np
import pytest
import torch

import seq_lstm_ref as S
from helpers import Pool, run, small_params, within
from visdial_b200 import VD_MATH_F16, VD_MATH_FP32, VD_MATH_TF32, Engine, init_parameters
from visdial_b200 import engine as VE

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
TF32 = 2.0 ** -9
ACT = 5e-7
TINY = 2.0 ** -149           # fp32's smallest subnormal: the absolute rounding of results that underflow
SIMT, TC, OPT16, PAIR16 = 0, 1, 2, 3
FREE = {VD_MATH_FP32: 1e-5, VD_MATH_TF32: 3e-2, VD_MATH_F16: 3e-2}
MODES = {"fp32": VD_MATH_FP32, "tf32": VD_MATH_TF32, "f16": VD_MATH_F16}


def report(tag, what, err, bound):
    """largest error / bound, printed (pytest -s) for DESIGN §7"""
    r = float(np.max(np.abs(err) / np.maximum(bound, 1e-300))) if np.size(err) else 0.0
    print("RATIO %-28s %-10s %.3g" % (tag, what, r))


def close(got, ref, bound, tag, what):
    got = np.asarray(got, np.float64)
    ref = np.broadcast_to(np.asarray(ref, np.float64), got.shape)
    bound = np.broadcast_to(bound, got.shape)
    report(tag, what, got - ref, bound)
    within(got, ref, bound, "%s %s" % (tag, what))


# ---------------------------------------------------------------------------------------------- engines and plumbing
@pytest.fixture(scope="module")
def engines():
    d = {}
    yield d
    for e in d.values():
        e.close()


def engine(engines, E, H, V, mode):
    """lf-ques / disc at embedSize E, rnnHiddenSize H, vocabSize V: segments ques.lstm1 (E -> H), ques.lstm2 (H -> H),
    opt.lstm (E -> H); LSTM biases ~ N(0, 0.5^2) so that a dropped or doubled bias shows"""
    if (E, H, V) not in engines:
        p = small_params("lf-ques", "disc", embedSize=E, rnnHiddenSize=H, vocabSize=V)
        eng = Engine(p)
        flat = init_parameters(p, seed=E + H + V)
        segs = VE.layout(p)[0]
        rng = np.random.default_rng(H)
        for s in segs:
            if "lstm" in s.name and s.name.endswith(".bias"):
                flat[s.offset:s.offset + s.size] = rng.normal(0, 0.5, s.size)
        eng.set_parameters(flat)
        eng.p, eng.flat, eng.segs = p, flat, {s.name: (i, s) for i, s in enumerate(segs)}
        engines[(E, H, V)] = eng
    eng = engines[(E, H, V)]
    eng.set_math_mode(mode)
    eng.zero_grad()
    return eng


@pytest.fixture
def pool_of():
    pools = []

    def make(eng):
        pools.append(Pool(eng))
        return pools[-1]
    yield make
    for p in pools:
        p.free()


def params(eng, seg):
    """W (D + H, 4H), b (4H,), the embedding (V + 1, E) with its pad row zero (as refresh_shadows leaves it), D, H, offset"""
    i, s = eng.segs[seg + ".weight"]
    W = eng.flat[s.offset:s.offset + s.size].reshape(s.rows, s.cols).astype(np.float64)
    _, sb = eng.segs[seg + ".bias"]
    b = eng.flat[sb.offset:sb.offset + sb.size].astype(np.float64)
    _, se = eng.segs["wordEmbed.weight"]
    emb = eng.flat[se.offset:se.offset + se.size].reshape(se.rows, se.cols).astype(np.float64).copy()
    emb[0] = 0
    return W, b, emb, s.rows - s.cols // 4, s.cols // 4, s.offset


def grads(eng, seg):
    g = eng.get_gradients().astype(np.float64)
    out = {}
    for k, name in (("dW", seg + ".weight"), ("db", seg + ".bias"), ("dEmb", "wordEmbed.weight")):
        _, s = eng.segs[name]
        out[k] = g[s.offset:s.offset + s.size].reshape(s.rows, s.cols) if k != "db" else g[s.offset:s.offset + s.size]
    return out


def half(bits):
    return np.asarray(bits).view(np.float16).astype(np.float64)


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---------------------------------------------------------------------------------------------- the route mirror
def tma_ok(off, ld):
    return off % 4 == 0 and ld % 4 == 0          # W and its shadow are cudaMalloc'ed: 16-byte alignment is off % 4 == 0


def route(mode, R, H, D, off, gathered, has_h0):
    """Engine::route_lstm: {fwd, bwd, table_grad, wave_fwd, wave_bwd}"""
    if mode == VD_MATH_F16 and gathered and not has_h0 and H in (256, 512) and R >= 1024:        # lstm16_shape_ok
        return [OPT16, OPT16, 1, 0, 0]
    tc = mode != VD_MATH_FP32
    fwd = TC if tc and H % 64 == 0 and tma_ok(off + D, D + H) else SIMT                          # lstm_step_fwd_tc_ok
    bwd = TC if tc and H % 128 == 0 and tma_ok(off + D * 4 * H, 4 * H) else SIMT                 # lstm_step_bwd_tc_ok
    return [fwd, bwd, int(gathered and tc), 0, 0]


def route_pair(mode, R, H, D1, off1, off2):
    """Engine::route_lstm_pair; kWavefrontMinRows = 64"""
    if mode == VD_MATH_F16 and H % 64 == 0 and H <= 512 and R >= 64 and 3 * (H // 32) <= sms():   # enc_pair_shape_ok
        return [PAIR16, PAIR16, 0, 0, 0] * 2
    a, b = route(mode, R, H, D1, off1, False, False), route(mode, R, H, H, off2, False, False)
    wf, wb = int(b[0] == TC and R >= 64), int(a[1] == TC and b[1] == TC and R >= 64)
    return a[:3] + [wf, wb] + b[:3] + [wf, wb]


# ---------------------------------------------------------------------------------------------- inputs
def mask_ids(T, R, rng):
    """time-major ids, 0 = reset: ~10 % random zeros, rows 0, 127, 128, R-1 masked at the first / last step, row 1 always"""
    ids = np.where(rng.random((T, R)) < 0.1, 0, 1).astype(np.int32)
    for r, t in ((0, 0), (127, T - 1), (128, 0), (R - 1, T - 1)):
        if r < R:
            ids[t, r] = 0
    if R > 1:
        ids[:, 1] = 0
    return ids


def tokens(T, R, V, rng):
    """ids in [0, V]: ~15 % pad tokens, a quarter of the rows the last table row V (its dP row is large), the rest uniform"""
    tok = rng.integers(1, V + 1, (T, R))
    tok[rng.random((T, R)) < 0.25] = V
    tok[rng.random((T, R)) < 0.15] = 0
    return tok.astype(np.int32)


def run_seq(eng, pool, seg, T, R, x=None, tok=None, mask=None, h0=None, c0=None, dh_all=None, dh_last=None, dc_last=None,
            train=True, want=(), f16=False):
    """one seq_lstm call; want: any of dx, dh0, dc0, demb.  Returns the outputs (float64, time-major shapes) and info"""
    i, s = eng.segs[seg + ".weight"]
    H, D = s.cols // 4, s.rows - s.cols // 4
    V1, E = eng.p["vocabSize"] + 1, eng.p["embedSize"]
    dev = lambda a, dt=np.float32: None if a is None else pool(np.ascontiguousarray(a, dt).reshape(-1))
    hdt = np.uint16 if f16 else np.float32
    n = T if train else 1
    o = {"h": pool.out(n * R * H, hdt), "c": pool.out(n * R * H), "info": pool.out(5, np.int32)}
    if train:
        o.update(gates=pool.out(T * R * 4 * H, hdt), da=pool.out(T * R * 4 * H, hdt), scale=pool.out(2))
    sizes = {"dx": T * R * D, "dh0": R * H, "dc0": R * H, "demb": V1 * E}
    for k in want:
        o[k] = pool.out(sizes[k])
    ptrs = [dev(x), dev(tok, np.int32), dev(mask, np.int32), dev(h0), dev(c0), dev(dh_all), dev(dh_last), dev(dc_last)]
    ptrs += [o.get(k) for k in ("h", "c", "gates", "da", "dx", "dh0", "dc0", "demb", "scale", "info")]
    run(eng, "seq_lstm", ptrs, [i, T, R, int(train)])
    got = {k: v.get() for k, v in o.items()}
    for k in ("h", "gates", "da"):
        if k in got:
            got[k] = half(got[k]) if f16 else got[k].astype(np.float64)
    shapes = {"h": (n, R, H), "c": (n, R, H), "gates": (T, R, 4 * H), "da": (T, R, 4 * H), "dx": (T, R, D), "dh0": (R, H),
              "dc0": (R, H), "demb": (V1, E)}
    return {k: (np.asarray(v, np.float64).reshape(shapes[k]) if k in shapes else v) for k, v in got.items()}


# ---------------------------------------------------------------------------------------------- bounds
def cell_bounds(a, cp, c, dz, act):
    """bounds of the activated gates, c and h of one step from the bound dz of the pre-activation"""
    H = a.shape[-1] // 4
    i, f, o, g = a[..., :H], a[..., H:2 * H], a[..., 2 * H:3 * H], a[..., 3 * H:]
    ea = np.concatenate([a[..., :3 * H] * (1 - a[..., :3 * H]), 1 - g * g], -1) * dz + act
    ei, ef, eo, eg = ea[..., :H], ea[..., H:2 * H], ea[..., 2 * H:3 * H], ea[..., 3 * H:]
    ec = np.abs(cp) * ef + np.abs(g) * ei + np.abs(i) * eg + 3 * U * (np.abs(f * cp) + np.abs(i * g))
    tc = np.tanh(c)
    eh = eo * np.abs(tc) + np.abs(o) * (ec * (1 - tc * tc) + act) + 2 * U * np.abs(o * tc)
    return ea, ec, eh


def bptt_bound(gates, c, c0, mask, dh, e_dh, dc_last, act):
    """the teacher-forced BPTT's per-element bound on da and the bound of the free-running cell-gradient carry past step 0"""
    T, R, G = gates.shape
    H = G // 4
    eda = np.zeros_like(gates)
    dc = np.zeros((R, H)) if dc_last is None else np.asarray(dc_last, np.float64)
    edc = np.zeros((R, H))
    for t in reversed(range(T)):
        a, ct = gates[t], c[t]
        cp = c[t - 1] if t else (np.zeros((R, H)) if c0 is None else c0)
        i, f, o, g = a[:, :H], a[:, H:2 * H], a[:, 2 * H:3 * H], a[:, 3 * H:]
        tc = np.tanh(ct)
        d = dc + dh[t] * o * (1 - tc * tc)
        ed = edc + e_dh[t] * o * (1 - tc * tc) + np.abs(dh[t]) * o * 2 * np.abs(tc) * act + 3 * U * (np.abs(dc) + np.abs(d))
        eda[t] = np.concatenate([ed * np.abs(g * i * (1 - i)), ed * np.abs(cp * f * (1 - f)),
                                 e_dh[t] * np.abs(tc * o * (1 - o)) + np.abs(dh[t]) * o * (1 - o) * act,
                                 ed * np.abs(i * (1 - g * g))], 1) + TINY
        edc = ed * f + U * np.abs(d) * f
        dc = d * f
        if mask is not None:
            edc[mask[t]] = 0
            dc[mask[t]] = 0
            eda[t][mask[t]] = 0
    return eda, edc


def gemm_factor(mode, K, exact_operands=False):
    return (K + 2) * U + (TF32 if mode != VD_MATH_FP32 and not exact_operands else 0.0)


# ---------------------------------------------------------------------------------------------- one saved run, checked
def check_saved(tag, mode, rt, W, b, emb, x, tok, mask, h0, c0, dh_all, dh_last, dc_last, got, g, want, step_bounds=None):
    """teacher-forced forward, BPTT and gradients, then the free-running forward / BPTT"""
    T, R, H = got["c"].shape
    D, G = W.shape[0] - H, 4 * H
    opt16 = rt[0] == OPT16
    m = None if mask is None else mask == 0
    # forward
    ga, c, h, Sz = S.forward(W, b, x, m, h0, c0, tf=(got["h"], got["c"]))
    if opt16:
        for k, ref in (("gates", ga), ("c", c), ("h", h)):
            close(got[k], ref, 4e-3 * (1 + np.abs(ref)), tag, k)
    else:
        cp = np.concatenate([np.zeros((1, R, H)) if c0 is None else c0[None], got["c"][:-1]])
        ea, ec, eh = cell_bounds(ga, cp, c, gemm_factor(mode, D + H) * Sz, ACT)
        for k, ref, e in (("gates", ga, ea), ("c", c, ec), ("h", h, eh)):
            close(got[k], ref, e, tag, k)
    if m is not None:
        for k in ("gates", "c", "h"):
            assert (got[k][m] == 0).all(), (tag, k, "masked rows must be exact zeros")
    # BPTT from the device's saved gates / c and its da_{t+1}
    s = float(got["scale"][0]) if opt16 else 1.0
    if opt16:
        assert s > 0 and np.log2(s) == np.round(np.log2(s)) and got["scale"][1] == np.float32(1 / s), (tag, got["scale"])
    da_dev = got["da"] / s
    da, dh, Sdh, dc0 = S.backward(W, got["gates"], got["c"], c0, m, dh_all, dh_last, dc_last, tf_da=da_dev)
    if opt16:
        e_dh = (2.0 ** -11 + (G + 2) * U) * Sdh
        eda, _ = bptt_bound(got["gates"], got["c"], c0, m, dh, e_dh, dc_last, 2.0 ** -10)
        eda += 2.0 ** -11 * np.abs(da) + 2.0 ** -25 / s
    else:
        eda, edc = bptt_bound(got["gates"], got["c"], c0, m, dh, gemm_factor(mode, G) * Sdh, dc_last, ACT)
        eda += 4 * U * np.abs(da)
    close(da_dev, da, eda, tag, "da")
    if m is not None:
        assert (got["da"][m] == 0).all(), (tag, "masked rows of da must be zeros")
    if "dc0" in want:
        close(got["dc0"], dc0, edc, tag, "dc0")
    # gradients from the device's own operands
    TR = T * R
    wg = S.weight_grads(W, x, got["h"], da_dev, h0)
    close(g["dW"][D:], wg["dWh"][0], gemm_factor(mode, TR, exact_operands=opt16) * wg["dWh"][1], tag, "dWh")
    if "dh0" in want:
        close(got["dh0"], wg["dh0"][0], gemm_factor(mode, G) * wg["dh0"][1], tag, "dh0")
    if rt[2]:
        V1 = emb.shape[0]
        tg = S.table_grads(W, emb, tok, da_dev)
        f = gemm_factor(mode, TR + V1)
        close(g["dW"][:D], tg["dWx"][0], f * tg["dWx"][1], tag, "dWx")
        close(g["db"], tg["db"][0], (TR + V1 + 2) * U * tg["db"][1], tag, "db")
        close(got["demb"] if "demb" in want else g["dEmb"], tg["dEmb"][0], f * tg["dEmb"][1], tag, "dEmb")
        if "demb" in want:
            assert (g["dEmb"] == 0).all(), (tag, "demb_out set: dW(wordEmbed) must stay untouched")
    else:
        close(g["dW"][:D], wg["dWx"][0], gemm_factor(mode, TR) * wg["dWx"][1], tag, "dWx")
        close(g["db"], wg["db"][0], (TR + 2) * U * wg["db"][1], tag, "db")
        if "dx" in want:
            close(got["dx"], wg["dx"][0], gemm_factor(mode, G) * wg["dx"][1], tag, "dx")
        assert (g["dEmb"] == 0).all(), (tag, "a dense / fp32 run leaves dW(wordEmbed) alone")
    # free-running
    fga, fc, fh, _ = S.forward(W, b, x, m, h0, c0)
    fda = S.backward(W, fga, fc, c0, m, dh_all, dh_last, dc_last)[0]
    for k, ref in (("h", fh), ("c", fc), ("da", fda)):
        v = got[k] / (s if k == "da" else 1.0)
        stepmax = np.abs(ref).reshape(T, -1).max(1)[:, None, None]
        close(v, ref, FREE[mode] * stepmax + 1e-30, tag, "free " + k)


CASES = {
    # name: mode, E, H, V, seg, T, R, input, masked, h0, c0, dh (all / last / both / lastonly), want, f16 dh_last factor
    # ---- Simt (VD_MATH_FP32)
    "fp32-dense-T1": ("fp32", 36, 64, 40, "ques.lstm1", 1, 37, "dense", True, True, True, "all", ("dx", "dh0", "dc0")),
    "fp32-dense-T2-dh_all": ("fp32", 36, 64, 40, "ques.lstm2", 2, 53, "dense", False, False, False, "dh_all", ("dx",)),
    "fp32-dense-T3-last": ("fp32", 36, 64, 40, "ques.lstm1", 3, 129, "dense", True, True, True, "last", ("dx", "dh0", "dc0")),
    "fp32-dense-T20": ("fp32", 36, 64, 40, "ques.lstm2", 20, 70, "dense", True, True, True, "all", ("dx", "dh0", "dc0")),
    "fp32-gather-T20": ("fp32", 36, 64, 40, "opt.lstm", 20, 64, "gather", True, True, True, "all", ("dx", "dh0", "dc0")),
    "fp32-gather-T3-nomask": ("fp32", 36, 64, 40, "opt.lstm", 3, 33, "gather", False, False, False, "last", ("dx",)),
    # ---- Tc (TF32)
    "tf32-H128-dense": ("tf32", 300, 128, 40, "ques.lstm1", 20, 200, "dense", True, True, True, "all", ("dx", "dh0", "dc0")),
    "tf32-H64-dense": ("tf32", 300, 64, 40, "ques.lstm2", 5, 129, "dense", True, True, True, "all", ("dx", "dh0", "dc0")),
    "tf32-H96-dense": ("tf32", 300, 96, 40, "ques.lstm1", 3, 64, "dense", True, True, False, "last", ("dx", "dh0", "dc0")),
    "tf32-H512-table": ("tf32", 300, 512, 40, "opt.lstm", 20, 300, "gather", True, False, False, "last", ()),
    "tf32-H512-table-demb-h0": ("tf32", 300, 512, 40, "opt.lstm", 5, 200, "gather", False, True, True, "all", ("demb", "dh0", "dc0")),
    # ---- Opt16 (VD_MATH_F16)
    "f16-H256-R1024-T20": ("f16", 300, 256, 40, "opt.lstm", 20, 1024, "gather", False, False, True, "lastonly", ()),
    "f16-H512-R1101-mask-c0": ("f16", 300, 512, 40, "opt.lstm", 6, 1101, "gather", True, False, True, "lastonly", ()),
    "f16-H512-R1024-x2^-10": ("f16", 300, 512, 40, "opt.lstm", 6, 1024, "gather", False, False, False, "lastonly", (), 2.0 ** -10),
    "f16-H256-R1101-x2^-20": ("f16", 300, 256, 40, "opt.lstm", 6, 1101, "gather", True, False, False, "lastonly", (), 2.0 ** -20),
    "f16-H256-R1024-zero": ("f16", 300, 256, 40, "opt.lstm", 4, 1024, "gather", True, False, True, "lastonly", (), 0.0),
    "f16-H256-gather-h0": ("f16", 300, 256, 40, "opt.lstm", 3, 1024, "gather", True, True, True, "last", ("demb",)),
    "f16-H256-R1023": ("f16", 300, 256, 40, "opt.lstm", 3, 1023, "gather", True, False, False, "lastonly", ()),
}


def build_inputs(eng, c, rng):
    mode, E, H, V, seg, T, R, kind, masked, with_h0, with_c0, dhs = c[:12]
    W, b, emb, D, H, off = params(eng, seg)
    tok = tokens(T, R, V, rng) if kind == "gather" else None
    x = emb[tok] if tok is not None else rng.standard_normal((T, R, D)).astype(np.float32).astype(np.float64)
    mask = (tok if tok is not None else mask_ids(T, R, rng)) if masked else None
    f32 = lambda *s: rng.standard_normal(s).astype(np.float32).astype(np.float64)
    h0 = np.tanh(f32(R, H)).astype(np.float32).astype(np.float64) if with_h0 else None
    c0 = f32(R, H) if with_c0 else None
    factor = c[13] if len(c) > 13 else 1.0
    dh_all = f32(T, R, H) * 0.5 if dhs in ("all", "dh_all") else None
    dh_last = (f32(R, H) * factor).astype(np.float32).astype(np.float64) if dhs in ("all", "last", "lastonly") else None
    dc_last = f32(R, H) * 0.5 if dhs in ("all", "last") else None
    return W, b, emb, D, H, off, x, tok, mask, h0, c0, dh_all, dh_last, dc_last


@pytest.mark.parametrize("name", sorted(CASES))
def test_seq_lstm(engines, pool_of, name):
    c = CASES[name]
    mode = MODES[c[0]]
    eng = engine(engines, c[1], c[2], c[3], mode)
    pool = pool_of(eng)
    rng = np.random.default_rng(sum(map(ord, name)))
    W, b, emb, D, H, off, x, tok, mask, h0, c0, dh_all, dh_last, dc_last = build_inputs(eng, c, rng)
    T, R, want = c[5], c[6], c[12]
    rt = route(mode, R, H, D, off, tok is not None, h0 is not None)
    if name in ("f16-H256-gather-h0", "f16-H256-R1023"):
        assert rt[0] != OPT16                        # gathered with h0 / one row short of lstm16_shape_ok: not the fp16 route
    got = run_seq(eng, pool, c[4], T, R, x=None if tok is not None else x, tok=tok, mask=mask, h0=h0, c0=c0, dh_all=dh_all,
                  dh_last=dh_last, dc_last=dc_last, want=want, f16=rt[0] == OPT16)
    assert list(got["info"]) == rt, (name, list(got["info"]), rt)
    g = grads(eng, c[4])
    check_saved(name, mode, rt, W, b, emb, x, tok, mask, h0, c0, dh_all, dh_last, dc_last, got, g, want)
    if rt[0] == OPT16 and not np.any(dh_last):
        assert (got["da"] == 0).all() and (g["dW"] == 0).all() and (g["db"] == 0).all() and (g["dEmb"] == 0).all()


@pytest.mark.parametrize("name,T", [("fp32", 3), ("fp32", 4), ("tf32", 3), ("tf32", 4), ("f16", 5)])
def test_inference_run(engines, pool_of, name, T):
    """train = 0: h / c ping-pong between two slots (both parities of T); Opt16 keeps h_T in h32_last"""
    mode = MODES[name]
    E, H, R, seg = (36, 64, 129, "ques.lstm2") if name == "fp32" else (300, 128, 200, "ques.lstm1") if name == "tf32" \
        else (300, 256, 1101, "opt.lstm")
    eng = engine(engines, E, H, 40, mode)
    pool = pool_of(eng)
    rng = np.random.default_rng(T)
    W, b, emb, D, H, off = params(eng, seg)
    gathered = name == "f16"
    tok = tokens(T, R, 40, rng) if gathered else None
    x = emb[tok] if gathered else rng.standard_normal((T, R, D)).astype(np.float32).astype(np.float64)
    mask = tok if gathered else mask_ids(T, R, rng)
    h0 = None if gathered else np.tanh(rng.standard_normal((R, H))).astype(np.float32).astype(np.float64)
    c0 = rng.standard_normal((R, H)).astype(np.float32).astype(np.float64)
    rt = route(mode, R, H, D, off, gathered, h0 is not None)
    got = run_seq(eng, pool, seg, T, R, x=None if gathered else x, tok=tok, mask=mask, h0=h0, c0=c0, train=False)
    assert list(got["info"]) == rt, (list(got["info"]), rt)
    assert rt[0] == {"fp32": SIMT, "tf32": TC, "f16": OPT16}[name]
    _, fc, fh, _ = S.forward(W, b, x, mask == 0, h0, c0)
    for k, ref in (("h", fh[-1]), ("c", fc[-1])):
        close(got[k][0], ref, FREE[mode] * np.abs(ref).max(), "infer-%s-T%d" % (name, T), "free " + k)
    assert (eng.get_gradients() == 0).all(), "a forward-only run accumulates no gradient"


def test_tma_ok_holds_on_every_segment(engines):
    eng = engine(engines, 300, 96, 40, VD_MATH_TF32)
    for name, (_, s) in eng.segs.items():
        if name.endswith(".weight") and "lstm" in name:
            H = s.cols // 4
            D = s.rows - H
            assert tma_ok(s.offset + D, D + H) and tma_ok(s.offset + D * 4 * H, 4 * H), name


# ---------------------------------------------------------------------------------------------- gradient contract
def test_backward_accumulates_and_demb_is_overwritten(engines, pool_of):
    """two BPTTs without a zero_grad in between leave twice one run's dW and db; demb_out is overwritten, not accumulated,
    and dW(wordEmbed) stays untouched; without demb_out the embedding gradient accumulates into dW(wordEmbed)"""
    eng = engine(engines, 300, 512, 40, VD_MATH_TF32)
    pool = pool_of(eng)
    rng = np.random.default_rng(5)
    T, R = 4, 200
    tok = tokens(T, R, 40, rng)
    dh_last = rng.standard_normal((R, 512)).astype(np.float32)
    call = lambda want: run_seq(eng, pool, "opt.lstm", T, R, tok=tok, mask=tok, dh_last=dh_last, want=want)
    one = call(("demb",))
    g1 = grads(eng, "opt.lstm")
    two = call(("demb",))
    g2 = grads(eng, "opt.lstm")
    assert (g1["dEmb"] == 0).all() and (g2["dEmb"] == 0).all()
    for k in ("dW", "db"):
        within(g2[k], 2 * g1[k], 1e-5 * np.abs(g1[k]).max(), "second BPTT " + k)
    within(two["demb"], one["demb"], 1e-5 * np.abs(one["demb"]).max(), "demb_out overwritten")
    eng.zero_grad()
    call(())
    call(())
    g = grads(eng, "opt.lstm")
    within(g["dEmb"], 2 * one["demb"], 2e-5 * np.abs(one["demb"]).max(), "dW(wordEmbed) accumulates")


# ---------------------------------------------------------------------------------------------- stacked pairs
PAIRS = {
    # name: mode, H, T, R, last1 present
    "tf32-R32-serial-last1": ("tf32", 512, 5, 32, True),
    "tf32-R32-serial": ("tf32", 512, 3, 32, False),
    "tf32-R320-wave": ("tf32", 512, 20, 320, False),
    "tf32-R320-wave-last1": ("tf32", 512, 5, 320, True),
    "f16-pair16-tail-atb": ("f16", 512, 4, 64, True),           # T R - R = 192 < 256: the fp32 gemm_atb weight gradient
    "f16-pair16-tail-atb16": ("f16", 512, 6, 64, False),        # T R - R = 320: gemm_atb16 on h16 and x16
}


@pytest.mark.parametrize("name", sorted(PAIRS))
def test_seq_lstm_pair(engines, pool_of, name):
    """free-running fp64 two-layer forward and BPTT (the pair keeps no da to teacher-force on): h / c of both layers, dx1,
    both layers' weight and bias gradients, each within the free-running bound of its step or of its largest element"""
    c = PAIRS[name]
    mode = MODES[c[0]]
    H, T, R = c[1], c[2], c[3]
    eng = engine(engines, 300, H, 40, mode)
    pool = pool_of(eng)
    rng = np.random.default_rng(sum(map(ord, name)))
    W1, b1, _, D1, _, off1 = params(eng, "ques.lstm1")
    W2, b2, _, _, _, off2 = params(eng, "ques.lstm2")
    f32 = lambda *s: rng.standard_normal(s).astype(np.float32).astype(np.float64)
    x = f32(T, R, D1)
    mask = mask_ids(T, R, rng)
    m = mask == 0
    x[m] = 0
    last = {k: f32(R, H) for k in ("dh_last2", "dc_last2")}
    last.update({k: f32(R, H) if c[4] else None for k in ("dh_last1", "dc_last1")})
    rt = route_pair(mode, R, H, D1, off1, off2)
    dev = lambda a: None if a is None else pool(np.asarray(a, np.float32).reshape(-1))
    o = {k: pool.out(T * R * H) for k in ("h1", "c1", "h2", "c2")}
    o["dx1"], o["info"] = pool.out(T * R * D1), pool.out(10, np.int32)
    i1, i2 = eng.segs["ques.lstm1.weight"][0], eng.segs["ques.lstm2.weight"][0]
    run(eng, "seq_lstm_pair", [dev(x), pool(mask.reshape(-1))] + [dev(last[k]) for k in ("dh_last2", "dc_last2", "dh_last1",
                                                                                          "dc_last1")]
        + [o[k] for k in ("h1", "c1", "h2", "c2", "dx1", "info")], [i1, i2, T, R])
    got = {k: v.get().astype(np.float64) for k, v in o.items()}
    assert list(got["info"].astype(int)) == rt, (name, list(got["info"]), rt)
    g1, g2 = grads(eng, "ques.lstm1"), grads(eng, "ques.lstm2")
    # fp64 pair, free-running
    ga1, c1, h1, _ = S.forward(W1, b1, x, m)
    ga2, c2, h2, _ = S.forward(W2, b2, h1, m)
    da2, _, _, _ = S.backward(W2, ga2, c2, None, m, None, last["dh_last2"], last["dc_last2"])
    w2 = S.weight_grads(W2, h1, h2, da2)
    da1, _, _, _ = S.backward(W1, ga1, c1, None, m, w2["dx"][0], last["dh_last1"], last["dc_last1"])
    w1 = S.weight_grads(W1, x, h1, da1)
    tol = FREE[mode]
    for k, ref in (("h1", h1), ("c1", c1), ("h2", h2), ("c2", c2), ("dx1", w1["dx"][0])):
        stepmax = np.abs(ref).reshape(T, -1).max(1)[:, None]
        close(got[k].reshape(T, -1), ref.reshape(T, -1), tol * stepmax + 1e-30, name, k)
    for L, gg, w, D in (("1", g1, w1, D1), ("2", g2, w2, H)):
        for k, ref in (("dWx", w["dWx"][0]), ("dWh", w["dWh"][0])):
            close(gg["dW"][:D] if k == "dWx" else gg["dW"][D:], ref, tol * np.abs(ref).max(), name, k + L)
        close(gg["db"], w["db"][0], tol * np.abs(w["db"][0]).max(), name, "db" + L)
