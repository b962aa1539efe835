"""The fused vocabulary projections of gemm_tc.cu (vocab_lse_tc, vocab_dlogits_tc, vocab_sample_tc) and their finish kernels,
one by one through vd_test_kernel, against fp64 references on the same operands; plus nll_bwd_scaled and scale_copy, the
dense gen step's d-logits on the materialised route.

Operands are rounded to TF32 here (low 13 mantissa bits cleared), so the tensor cores' truncation or rounding leaves them
unchanged and every product a_k b_k is exact in fp32: the reference is x = A B^T + bias in fp64 on those operands, and the
only error of a device logit is its fp32 accumulation.  Rows come in three logit sets: O(1) logits; |x| of 30-60 with a
spread of about 60 (a row shift of +-45 on a reserved feature), where __expf's argument-dependent error matters; and rows
with one class 40 above the rest (a reserved feature per boosted class), where softmax is a onehot and the target's d-logit
cancels.  Masked and target-less rows carry logits near 100, so an unmasked exp(x) overflows.

Bounds are error scales, not observed errors.  U = 2^-24.
  - logit:  e_x = (K + 1) U (sum_k |a_k b_k| + |bias|), the K + 1 additions of the accumulation and the bias.  The in-wgmma
    fp32 accumulation needs no factor on top: on an H100 80GB HBM3 (700 W power limit) the largest error / e_x over every
    case below is 0.22 (tgt_logit and part_max at K = 36), 0.12 at the C3 shape.  The module prints each output's largest
    error / bound when it ends (pytest -s).
  - __expf(a) costs 2 + 1.173 |a| ulp (CUDA's documented bound; one ulp <= 2U relative), expf / logf a few ulp (ULP_FN).
  - A slice's sum of exponentials: the __expf of each term and of up to 8 rescales (arguments summing to at most the slice's
    spread R), the rounding of each argument (U R) and a 16-term chain: relative U (100 + 8 R), with margin.
  - Each further sum adds its chain length.
These bounds stay below about 5e-3 relative even for |x| near 100 at K = 512, while a slice dropped, counted twice or
never rescaled, a target one column off, a missing bias or a draw at the wrong Philox counter moves an output by 1e-2 or
more, or leaves NaN or a wrong class."""

import numpy as np
import pytest
import torch

import sampling_twin
from helpers import ISENT, Pool, _image, call, run, small_params, within
from visdial_b200 import VD_MATH_TF32, Engine
from visdial_b200._lib import VD_E_SHAPE, check

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
ULP_FN = 4 * U               # relative error of one expf / logf, with margin
TC_FACTOR = 1.0              # measured: the accumulation needs no factor on top of (K + 1) U sum |a b|
BOOST, SHIFT, HUGE = 40.0, 45.0, 2.25      # dominant class; row shift of the |x| ~ 30-60 set; masked rows at x ~ 100
GUMBEL_SPREAD = 20.2         # largest minus smallest Gumbel value of the rule (17.33 + 2.85)
SLICE = 64                   # columns per (row, slice) partial: 128-column tiles, two epilogue warps per row
SEED = 0x1234_5678_9ABC_DEF1  # both 32-bit words non-zero
DEV = torch.device("cuda")
RATIOS = {}                  # output -> largest err / bound seen (printed at the end of the module)


@pytest.fixture(scope="module")
def eng():
    e = Engine(small_params("lf-ques", "disc"))
    e.set_math_mode(VD_MATH_TF32)         # vd_gemm_tn's materialised logits of the cross-route tests
    e.profile(True)                       # launches counted under their launch-site names
    yield e
    e.close()
    if RATIOS:
        print("\nlargest error / bound per output:")
        for k in sorted(RATIOS):
            print("  %-40s %.3g" % (k, RATIOS[k]))


@pytest.fixture
def pool(eng):
    p = Pool(eng)
    yield p
    p.free()


# ---------------------------------------------------------------------------------------------- plumbing
def tf32(x):
    x = np.ascontiguousarray(x, np.float32)
    return (x.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def T(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV, torch.float64)


def nparts_of(N):
    return -(-N // 128) * 2


def vocab_tc_ok(M, N, K, offA, lda, offB, ldb):
    """mirror of gemm_tc.cu's vocab_tc_ok (device bases are 256-byte aligned: 16 bytes <=> offset % 4 == 0)"""
    return M >= 64 and N >= 256 and N % 4 == 0 and K >= 32 and offA % 4 == 0 and lda % 4 == 0 and offB % 4 == 0 and ldb % 4 == 0


def tc_run(eng, name, ptrs, ints, reals=()):
    """an accepted fused call is exactly one k_tc_gemm launch"""
    n0, k0 = eng.launch_count(), eng.kernel_stats("k_tc_gemm")["launches"]
    run(eng, name, ptrs, ints, reals)
    assert eng.launch_count() == n0 + 1 and eng.kernel_stats("k_tc_gemm")["launches"] == k0 + 1, name


def twithin(got, ref, bound, what):
    """|got - ref| <= bound on the GPU in fp64 (got finite); records the largest err / bound under `what`"""
    got = torch.as_tensor(got).to(DEV, torch.float64) if not torch.is_tensor(got) else got.to(torch.float64)
    assert bool(torch.isfinite(got).all()), (what, "non-finite output")
    err = (got - ref).abs()
    bound = torch.as_tensor(bound, dtype=torch.float64, device=DEV).expand_as(err)
    ratio = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, np.inf, 0.0))
    worst = float(ratio.max()) if ratio.numel() else 0.0
    for key in {what, what.split(" @")[0]}:
        RATIOS[key] = max(RATIOS.get(key, 0.0), worst)
    if worst > 1:
        i = np.unravel_index(int(torch.argmax(ratio)), tuple(err.shape))
        raise AssertionError("%s: %d elements out of bound, worst at %s: got %r ref %r bound %r"
                             % (what, int((ratio > 1).sum()), i, float(got[i]), float(ref[i]), float(bound[i])))


def boost_classes(N):
    """first / last quadruple of slices 0 and 3, the last valid column, the first quadruple of the last column tile"""
    return [1, 62, 194, 253, N - 1, (N - 1) // 128 * 128 + 2]


def operands(M, N, K, seed, bias=True, flat=0.0):
    """TF32 A (M, K), B (N, K), fp32 bias (N) or None; per row its set: 0 O(1), 1 |x| ~ 30-60, 2 one class BOOST above the
    rest (boost[m] = that class), 3 flat (A row 0: x = bias)"""
    rng = np.random.default_rng(seed)
    kind = rng.choice(4, M, p=[0.55 - flat, 0.25, 0.2, flat])
    A = rng.standard_normal((M, K))
    A[:, :7] = 0.0
    big, dom = kind == 1, kind == 2
    A[big, 7:] *= 5.0
    A[big, 0] = rng.choice([-1.0, 1.0], int(big.sum()))
    bdim = rng.integers(1, 7, M)
    A[dom, 7:] *= 0.1
    A[dom, bdim[dom]] = BOOST
    A[kind == 3] = 0.0
    B = rng.standard_normal((N, K)) * (1.5 / np.sqrt(K - 7))
    B[:, :7] = 0.0
    B[:, 0] = SHIFT
    bc = boost_classes(N)
    for d, c in enumerate(bc):
        B[c, d + 1] = 1.0
    b = f32(rng.standard_normal(N) * 0.3) if bias else None
    boost = np.where(dom, np.array(bc)[bdim - 1], -1)
    return tf32(A), tf32(B), b, kind, boost


def f32(x):
    return np.asarray(x, np.float32)


def reference(A, B, b):
    """x = A B^T + bias in fp64 and its error scale e_x, on the GPU"""
    A64, B64 = T(A), T(B)
    x = A64 @ B64.T
    s = A64.abs() @ B64.abs().T
    if b is not None:
        b64 = T(b)
        x += b64
        s += b64.abs()
    s *= TC_FACTOR * (A.shape[1] + 1) * U
    return x, s


def slices(t, N, fill):
    S = nparts_of(N)
    return torch.nn.functional.pad(t, (0, S * SLICE - N), value=fill).view(t.shape[0], S, SLICE)


def nonempty(N):
    return (torch.arange(nparts_of(N), device=DEV) * SLICE) < N


def lse_stats(x, ex, nparts):
    """fp64 row lse, softmax, and the bounds of the device's lse: `b` against the exact lse of x, `b_dev` against the exact
    lse of the device's own fp32 logits (the part without e_x)"""
    mx = x.max(1).values
    p = torch.exp(x - mx[:, None])
    ssum = p.sum(1)
    p /= ssum[:, None]
    lse = mx + torch.log(ssum)
    R = mx - x.min(1).values
    b_dev = U * (100 + 8 * R) + ULP_FN * (mx.abs() + (lse - mx).abs() + nparts + 4) + 2 * U * R
    return lse, p, (p * ex).sum(1) + b_dev, b_dev


def check_partials(pm, ps, x, ex, N, what):
    """part_max / part_sum of every (row, slice) against x: empty slices exactly (-inf, 0)"""
    ne = nonempty(N).cpu().numpy()
    assert (pm[:, ~ne] == -np.inf).all() and (ps[:, ~ne] == 0).all(), (what, "empty slices must be (-inf, 0)")
    xs, es = slices(x, N, -np.inf)[:, ne], slices(ex, N, 0.0)[:, ne]
    pm_t = T(pm[:, ne])
    twithin(pm_t, xs.max(-1).values, es.max(-1).values, "part_max @" + what)
    R = xs.max(-1).values - slices(x, N, np.inf)[:, ne].min(-1).values
    t = torch.exp(xs - pm_t[..., None])
    st = t.sum(-1)
    twithin(T(ps[:, ne]), st, (t * es).sum(-1) + st * U * (100 + 8 * R), "part_sum @" + what)


# ---------------------------------------------------------------------------------------------- vocab_lse_tc / dlogits
# (M, N, K, lda - K, A offset in floats, row scale): M 64 (the minimum), 127 / 129 (a ragged / one-row second row block),
# 200, 400 (a dense gen step, B numOptions), 840 (C1's rows), 6 700 (C3's training rows: every CTA walks ~32 tiles);
# N 256 (two whole tiles), 260 (a 4-column tail tile), 300, 320 (its second slice exactly empty), 324, 1 000 (C1),
# 10 000 (C2-C5, a 16-column tail); K 32, 36 (a partial k-block), 128, 512
CASES = [
    (64, 256, 32, 0, 0, "none"),
    (127, 260, 36, 4, 4, "neg_g"),
    (129, 300, 128, 0, 0, "ones"),
    (200, 320, 512, 4, 4, "none"),
    (840, 1000, 512, 0, 0, "neg_g"),
    (400, 10000, 512, 0, 0, "neg_g"),
    (6700, 10000, 512, 0, 0, "none"),
    (64, 324, 36, 0, 0, "ones"),
    (129, 10000, 32, 4, 4, "none"),
    (200, 256, 128, 4, 0, "neg_g"),
    (127, 1000, 36, 0, 0, "none"),
    (64, 10000, 128, 0, 4, "ones"),
    (840, 324, 32, 0, 0, "neg_g"),
    (400, 300, 512, 4, 4, "none"),
    (129, 320, 36, 0, 0, "neg_g"),
]


def case_inputs(M, N, K, seed):
    A, B, b, kind, boost = operands(M, N, K, seed)
    rng = np.random.default_rng(seed + 1)
    tgt = rng.integers(1, N + 1, M).astype(np.int32)
    dom = boost >= 0
    half = dom & (rng.random(M) < 0.5)
    tgt[half] = boost[half] + 1                                  # the target is the dominant class: its d-logit cancels
    tgt[rng.random(M) < 0.08] = 0
    ids = rng.integers(1, 50, M).astype(np.int32)
    ids[rng.random(M) < 0.08] = 0
    tail = (N - 1) // 128 * 128
    edge = [1, 64, 65, 128, 129, N, tail + 1, N - 2]             # columns 0, 63, 64, 127, 128, N - 1, inside the tail tile
    tgt[:len(edge)], ids[:len(edge)] = edge, 1
    keep = (ids != 0) & (tgt > 0)
    A[~keep, 0] = HUGE                                           # unkept rows: logits near 100, exp(x) without the lse = inf
    g = f32(rng.standard_normal(M) * 0.3)
    g[rng.random(M) < 0.15] = 0.0
    return A, B, b, tgt, ids, keep, -g


def dlogits_buf(pool, M, N, ldc, offC):
    return pool(_image(np.full((M, N), np.nan, np.float32), offC, ldc, rows_extra=2))


def dlogits_view(dev, M, N, ldc, offC, what):
    img = dev.get()
    assert np.isnan(img[:offC]).all(), (what, "wrote before C")
    full = img[offC:].reshape(M + 2, ldc)
    assert np.isnan(full[M:]).all(), (what, "wrote rows past M")
    assert np.isnan(full[:M, N:]).all(), (what, "wrote columns [N, ldc)")
    return full[:M, :N]


@pytest.mark.parametrize("M,N,K,pad,offA,scale_kind", CASES)
def test_vocab_lse_and_dlogits(eng, pool, M, N, K, pad, offA, scale_kind):
    i = CASES.index((M, N, K, pad, offA, scale_kind))
    A, B, b, tgt, ids, keep, neg_g = case_inputs(M, N, K, 100 + i)
    lda, S = K + pad, nparts_of(N)
    tag = "%dx%dx%d" % (M, N, K)
    dA, dB, db_, dt, di = pool(_image(A, offA, lda)), pool(B), pool(b), pool(tgt), pool(ids)
    # ---- forward partials, twice: bit-identical
    outs = []
    for _ in range(2):
        pm, ps, tl = pool.out((M, S)), pool.out((M, S)), pool.out(M)
        tc_run(eng, "vocab_lse_tc", [dA.ptr(offA), dB, db_, dt, pm, ps, tl], [M, N, K, lda, K])
        outs.append((pm.get(), ps.get(), tl.get()))
    for a, c in zip(outs[0], outs[1]):
        assert (a.view(np.uint32) == c.view(np.uint32)).all(), "vocab_lse_tc must repeat bit for bit"
    gpm, gps, gtl = outs[0]
    x, ex = reference(A, B, b)
    check_partials(gpm, gps, x, ex, N, tag)
    has = tgt > 0
    r = torch.arange(M, device=DEV)
    tcol = torch.as_tensor(np.maximum(tgt, 1) - 1, device=DEV, dtype=torch.long)
    h = torch.as_tensor(has, device=DEV)
    twithin(T(gtl[has]), x[r, tcol][h], ex[r, tcol][h], "tgt_logit @" + tag)
    assert np.isnan(gtl[~has]).all(), "rows without a target leave tgt_logit untouched"
    # ---- the training criterion's chain: lse and -(x_tgt - lse) on kept rows
    lse_ref, p, b_lse, b_dev = lse_stats(x, ex, S)
    lse_d, loss = pool.out(M), pool.out(M)
    run(eng, "vocab_lse_finish", [pm, ps, tl, dt, di, lse_d, loss], [S, 0, M], [-1.0])
    g_lse = lse_d.get()
    twithin(T(g_lse), lse_ref, b_lse, "lse @" + tag)
    gl, k = loss.get(), torch.as_tensor(keep, device=DEV)
    assert (gl[~keep] == 0).all(), "unkept rows: loss 0"
    ref = -(x[r, tcol] - lse_ref)
    twithin(T(gl[keep]), ref[k], (ex[r, tcol] + b_lse + 2 * U * ref.abs())[k], "criterion @" + tag)
    # ---- d-logits, teacher-forced on fp32(lse_ref): against fp64
    s = {"none": None, "ones": np.ones(M, np.float32), "neg_g": neg_g}[scale_kind]
    s64 = T(s) if s is not None else torch.ones(M, dtype=torch.float64, device=DEV)
    ds = pool(s) if s is not None else None
    ldc, offC = (N + 4, 4) if i % 2 else (N, 0)
    L = T(f32(lse_ref.cpu().numpy()))
    dL = pool(f32(L.cpu().numpy()))
    C1 = dlogits_buf(pool, M, N, ldc, offC)
    tc_run(eng, "vocab_dlogits_tc", [dA.ptr(offA), dB, db_, dt, di, dL, C1.ptr(offC), ds], [M, N, K, lda, K, ldc])
    got = dlogits_view(C1, M, N, ldc, offC, "teacher-forced")
    kf = k.to(torch.float64)[:, None]
    q = torch.exp(x - L[:, None])
    onehot = torch.zeros_like(q)
    onehot[r[h], tcol[h]] = 1.0
    d_ref = kf * s64[:, None] * (q - onehot)
    bound = kf * s64.abs()[:, None] * q * (ex + U * (5 + 3.35 * (x - L[:, None]).abs())) + 2 * U * d_ref.abs()
    del onehot
    twithin(T(got), d_ref, bound, "dlogits @" + tag)
    assert (got[~keep] == 0).all(), "masked rows and rows without a target: exactly 0"
    del d_ref, bound, q
    if M * N <= 4_000_000:
        C1b = dlogits_buf(pool, M, N, ldc, offC)
        tc_run(eng, "vocab_dlogits_tc", [dA.ptr(offA), dB, db_, dt, di, dL, C1b.ptr(offC), ds], [M, N, K, lda, K, ldc])
        assert (dlogits_view(C1b, M, N, ldc, offC, "repeat").view(np.uint32) == got.view(np.uint32)).all(), \
            "vocab_dlogits_tc must repeat bit for bit"
    if scale_kind == "ones":
        C0 = dlogits_buf(pool, M, N, ldc, offC)
        tc_run(eng, "vocab_dlogits_tc", [dA.ptr(offA), dB, db_, dt, di, dL, C0.ptr(offC), None], [M, N, K, lda, K, ldc])
        assert (dlogits_view(C0, M, N, ldc, offC, "null scale").view(np.uint32) == got.view(np.uint32)).all(), \
            "row_scale = 1 must give the unscaled bits"
    # ---- chained on the device's own lse: every kept row's d-logits sum to s (sum softmax - 1) = 0
    C2 = dlogits_buf(pool, M, N, ldc, offC)
    tc_run(eng, "vocab_dlogits_tc", [dA.ptr(offA), dB, db_, dt, di, lse_d, C2.ptr(offC), ds], [M, N, K, lda, K, ldc])
    got2 = T(dlogits_view(C2, M, N, ldc, offC, "chained"))
    a = (x - lse_ref[:, None]).abs()
    rb = s64.abs() * ((p * (U * a + 2 * U * (2 + 1.173 * a))).sum(1) + b_dev) + U * got2.abs().sum(1)
    twithin(got2.sum(1)[k], torch.zeros(int(keep.sum()), dtype=torch.float64, device=DEV), rb[k], "dlogit row sum @" + tag)
    assert bool((got2[~k] == 0).all())


def test_forward_chain_accumulates_over_time_steps(eng, pool):
    """gen_option_lhood / the dense gen step: vocab_lse_tc then vocab_lse_finish(sign +1, accumulate 1) for each time step
    t, on rows t Ro .. of one activation buffer, into one score buffer"""
    Ro, N, K, steps = 400, 10000, 512, 3
    A, B, b, tgt, ids, keep, _ = case_inputs(Ro * steps, N, K, 7)
    S = nparts_of(N)
    dA, dB, db_, dt, di = pool(A), pool(B), pool(b), pool(tgt), pool(ids)
    o0 = f32(np.random.default_rng(8).standard_normal(Ro))
    out = pool(o0)
    pm, ps, tl = pool.out((Ro, S)), pool.out((Ro, S)), pool.out(Ro)
    for t in range(steps):
        tc_run(eng, "vocab_lse_tc", [dA.ptr(t * Ro * K), dB, db_, dt.ptr(t * Ro), pm, ps, tl], [Ro, N, K, K, K])
        run(eng, "vocab_lse_finish", [pm, ps, tl, dt.ptr(t * Ro), di.ptr(t * Ro), None, out], [S, 1, Ro], [1.0])
    x, ex = reference(A, B, b)
    lse_ref, _, b_lse, _ = lse_stats(x, ex, S)
    r = torch.arange(Ro * steps, device=DEV)
    tcol = torch.as_tensor(np.maximum(tgt, 1) - 1, device=DEV, dtype=torch.long)
    k = torch.as_tensor(keep, device=DEV, dtype=torch.float64)
    term = (k * (x[r, tcol] - lse_ref)).view(steps, Ro)
    tb = (k * (ex[r, tcol] + b_lse + U * (x[r, tcol] - lse_ref).abs())).view(steps, Ro)
    ref = T(o0) + term.sum(0)
    twithin(T(out.get()), ref, tb.sum(0) + U * (steps + 1) * (T(o0).abs() + term.abs().sum(0)), "accumulated lhood")


# ---------------------------------------------------------------------------------------------- sampling
def twin_keys(x, temperature, seed, step, row_offset, row_stride):
    """fp64 twin keys x / T + g of the rows row_offset + r row_stride, and g"""
    V = x.shape[1]
    g = np.concatenate([sampling_twin.gumbel_of_words(sampling_twin.sample_words(seed, step, row_offset + r * row_stride, 1, V))
                        for r in range(x.shape[0])])
    return x / temperature + g, g


# (M, N, K, lda - K, A offset, T, row_offset, row_stride, step, bias)
SAMPLE_CASES = [
    (64, 256, 32, 0, 0, 1.0, 0, 1, 1, True),
    (129, 324, 36, 4, 4, 0.5, 17, 3, 5, True),
    (200, 10000, 128, 0, 0, 1.7, 17, 1, 5, True),
    (127, 1000, 512, 0, 0, 0.5, 0, 3, 1, False),
    (64, 10000, 512, 4, 4, 1.7, 17, 3, 1, False),
    (129, 260, 36, 0, 0, 1.0, 0, 1, 5, True),
]


@pytest.mark.parametrize("M,N,K,pad,offA,temp,roff,rstride,step,bias", SAMPLE_CASES)
def test_vocab_sample(eng, pool, M, N, K, pad, offA, temp, roff, rstride, step, bias):
    i = SAMPLE_CASES.index((M, N, K, pad, offA, temp, roff, rstride, step, bias))
    A, B, b, kind, boost = operands(M, N, K, 300 + i, bias=bias, flat=0.1)
    lda, S, L = K + pad, nparts_of(N), 6
    dA, dB, db_ = pool(_image(A, offA, lda)), pool(B), pool(b) if bias else None
    outs = []
    for _ in range(2):
        o = [pool.out((M, S)), pool.out((M, S)), pool.out((M, S)), pool.out((M, S), np.int32), pool.out((M, S))]
        tc_run(eng, "vocab_sample_tc", [dA.ptr(offA), dB, db_] + o, [M, N, K, lda, K, SEED, step, roff, rstride], [temp])
        outs.append(o)
    got = [d.get() for d in outs[0]]
    for a, d in zip(got, outs[1]):
        assert (a.view(np.uint32) == d.get().view(np.uint32)).all(), "vocab_sample_tc must repeat bit for bit"
    pm, ps, pk, pc, px = got
    # the statistics are vocab_lse_tc's, bit for bit
    lpm, lps, ltl = pool.out((M, S)), pool.out((M, S)), pool.out(M)
    tc_run(eng, "vocab_lse_tc", [dA.ptr(offA), dB, db_, pool(np.zeros(M, np.int32)), lpm, lps, ltl], [M, N, K, lda, K])
    assert (lpm.get().view(np.uint32) == pm.view(np.uint32)).all() and (lps.get().view(np.uint32) == ps.view(np.uint32)).all()
    xt, ext = reference(A, B, b)
    x, ex = xt.cpu().numpy(), ext.cpu().numpy()
    key, g = twin_keys(x, temp, SEED, step, roff, rstride)
    kb = ex / temp + 16 * U * (np.abs(x) / temp + np.abs(g) + 20)      # the device's fp32 key error
    ne = nonempty(N).cpu().numpy()
    assert (pk[:, ~ne] == -np.inf).all() and (pc[:, ~ne] == 0x7fffffff).all() and (px[:, ~ne].view(np.uint32) == 0).all(), \
        "empty slices: (-inf, 0x7fffffff, 0)"
    pad_to = S * SLICE
    ks = np.pad(key, ((0, 0), (0, pad_to - N)), constant_values=-np.inf).reshape(M, S, SLICE)[:, ne]
    kbs = np.pad(kb, ((0, 0), (0, pad_to - N))).reshape(M, S, SLICE)[:, ne].max(-1)
    win = ks.argmax(-1) + np.flatnonzero(ne)[None, :] * SLICE                 # ties to the lower class, as the device
    top2 = -np.partition(-ks, 1, axis=-1)[..., :2]
    exempt = (top2[..., 0] - top2[..., 1]) <= 2 * kbs
    c = pc[:, ne]
    assert ((c == win) | exempt).all(), "slice winner differs from the twin outside near-ties"
    assert exempt.mean() <= 0.03, exempt.mean()
    rr = np.arange(M)[:, None]
    twithin(T(pk[:, ne]), T(key[rr, c]), T(kb[rr, c]), "part_key @%dx%d" % (M, N))
    twithin(T(px[:, ne]), T(x[rr, c]), T(ex[rr, c]), "part_x @%dx%d" % (M, N))
    # ---- the finish: the row's winner, answer column `step` only, logp column step - 1 only
    tok, ans, lp = pool.out(M, np.int32), pool.out((M, L + 1), np.int32), pool.out((M, L))
    run(eng, "vocab_sample_finish", [pool(pm), pool(ps), pool(pk), pool(pc), pool(px), tok, ans, lp], [S, M, step, L])
    gt, ga, gl = tok.get(), ans.get(), lp.get()
    assert (ga[:, step] == gt).all() and (np.delete(ga, step, 1) == ISENT).all(), "answer column step only"
    assert np.isnan(np.delete(gl, step - 1, 1)).all(), "logp column step - 1 only"
    wr = key.argmax(1)
    t2 = -np.partition(-key, 1, axis=1)[:, :2]
    row_exempt = (t2[:, 0] - t2[:, 1]) <= 2 * kb.max(1)
    assert ((gt == wr + 1) | row_exempt).all() and row_exempt.mean() <= 0.05, row_exempt.mean()
    dom = boost >= 0
    rest = np.where(np.arange(N)[None, :] == boost[:, None], -np.inf, x).max(1)
    assert ((x[np.arange(M), boost] - rest)[dom] / temp > GUMBEL_SPREAD).all(), "the boost outweighs any Gumbel draw"
    assert (gt[dom] == boost[dom] + 1).all(), "a class 40 above the rest always wins, skipped quadruples or not"
    lse_ref, _, b_lse, _ = lse_stats(xt, ext, S)
    lse_ref, b_lse = lse_ref.cpu().numpy(), b_lse.cpu().numpy()
    ref = x[np.arange(M), gt - 1] - lse_ref
    within(gl[:, step - 1], ref, ex[np.arange(M), gt - 1] + b_lse + 2 * U * np.abs(ref), "sampled logp")
    tok2, ans2 = pool.out(M, np.int32), pool.out((M, L + 1), np.int32)
    run(eng, "vocab_sample_finish", [pool(pm), pool(ps), pool(pk), pool(pc), pool(px), tok2, ans2, None], [S, M, step, L])
    assert (tok2.get() == gt).all() and (ans2.get() == ga).all(), "a null logp changes nothing else"


def test_vocab_sample_finish_synthetic(eng, pool):
    rows, V, L, step = 300, 10000, 4, 2
    S = nparts_of(V)
    rng = np.random.default_rng(21)
    pm = f32(rng.standard_normal((rows, S)) * 5)
    ps = f32(rng.uniform(1, 100, (rows, S)))
    pk = f32(rng.standard_normal((rows, S)) * 3)
    pc = (np.arange(S)[None, :] * SLICE + rng.integers(0, SLICE, (rows, S))).astype(np.int32)
    px = f32(rng.standard_normal((rows, S)) * 4)
    # rows 0 / 1: two slices with equal best keys, the lower class in the later / the earlier slice
    pk[0, 3] = pk[0, 7] = pk[1, 3] = pk[1, 7] = 50.0
    pc[0, 3], pc[0, 7], pc[1, 3], pc[1, 7] = 300, 5, 200, 460
    # empty slices (-inf, 0, -inf, 0x7fffffff, 0): first, all but the last, last, and a few inside
    for r, sl in ((2, [0]), (3, list(range(S - 1))), (4, [S - 1]), (5, [0, 1, 57])):
        pm[r, sl], ps[r, sl], pk[r, sl], pc[r, sl], px[r, sl] = -np.inf, 0.0, -np.inf, 0x7fffffff, 0.0
    m64, s64 = pm.astype(np.float64), ps.astype(np.float64)
    mx = m64.max(1)
    lse = mx + np.log((s64 * np.exp(m64 - mx[:, None])).sum(1))
    order = np.lexsort((pc, -pk.astype(np.float64)), axis=1)[:, 0]
    r = np.arange(rows)
    tok, ans, lp = pool.out(rows, np.int32), pool.out((rows, L + 1), np.int32), pool.out((rows, L))
    run(eng, "vocab_sample_finish", [pool(pm), pool(ps), pool(pk), pool(pc), pool(px), tok, ans, lp], [S, rows, step, L])
    gt = tok.get()
    assert (gt == pc[r, order] + 1).all(), "winner by (key desc, class asc)"
    assert gt[0] == 6 and gt[1] == 201, "equal keys: the lower class wins"
    assert gt[3] == pc[3, S - 1] + 1 and np.isfinite(pk[r, order]).all(), "an empty slice never wins"
    assert (ans.get()[:, step] == gt).all()
    fin = np.isfinite(m64)
    lb = ULP_FN * (np.abs(mx) + np.abs(lse - mx) + S + 4) + 2 * U * np.where(fin, np.abs(m64 - mx[:, None]), 0).max(1)
    ref = px[r, order].astype(np.float64) - lse
    within(lp.get()[:, step - 1], ref, lb + U * np.abs(ref), "vocab_sample_finish logp")


# ---------------------------------------------------------------------------------------------- cross-route
@pytest.mark.parametrize("M,N,K,pad,offA", [(200, 10000, 128, 0, 0), (129, 324, 36, 4, 4)])
def test_fused_matches_materialised_route(eng, pool, M, N, K, pad, offA):
    """the same logits materialised by vd_gemm_tn in TF32 (the same k_tc_gemm<128> contraction, MODE_GENERIC epilogue) are
    the fused epilogues' logits bit for bit; lse, d-logits and draws then differ only by their reductions and exp"""
    A, B, b, tgt, ids, keep, neg_g = case_inputs(M, N, K, 500 + N)
    lda, S = K + pad, nparts_of(N)
    dA, dB, db_, dt, di, ds = pool(_image(A, offA, lda)), pool(B), pool(b), pool(tgt), pool(ids), pool(neg_g)
    Lm = pool.out((M, N))
    k0 = eng.kernel_stats("k_tc_gemm")["launches"]
    check(eng.lib.vd_gemm_tn(eng.h, M, N, K, dA.ptr(offA), lda, dB.ptr(), K, Lm.ptr(), N, 0.0, db_.ptr(), 0))
    assert eng.kernel_stats("k_tc_gemm")["launches"] == k0 + 1, "vd_gemm_tn took the tensor-core route"
    X = Lm.get()
    pm, ps, tl = pool.out((M, S)), pool.out((M, S)), pool.out(M)
    tc_run(eng, "vocab_lse_tc", [dA.ptr(offA), dB, db_, dt, pm, ps, tl], [M, N, K, lda, K])
    has = tgt > 0
    r = np.arange(M)
    assert (tl.get()[has].view(np.uint32) == X[r[has], tgt[has] - 1].view(np.uint32)).all(), "tgt_logit == materialised bits"
    xs = np.pad(X, ((0, 0), (0, S * SLICE - N)), constant_values=-np.inf).reshape(M, S, SLICE).max(-1)
    assert (pm.get().view(np.uint32) == f32(xs).view(np.uint32)).all(), "part_max == materialised bits"
    # lse + likelihood: fused chain against lhood_accumulate on the materialised logits
    x = T(X)
    _, p, _, b_dev = lse_stats(x, torch.zeros_like(x), S)
    rows_b = ULP_FN * (2 * x.abs().max(1).values + N / 128 + 24)
    o0 = f32(np.random.default_rng(3).standard_normal(M))
    fo, ro, lse_d = pool(o0), pool(o0), pool.out(M)
    run(eng, "vocab_lse_finish", [pm, ps, tl, dt, di, lse_d, fo], [S, 1, M], [1.0])
    run(eng, "lhood_accumulate", [Lm, dt, di, ro], [M, N])
    gf, gr = fo.get(), ro.get()
    assert (gf[~keep] == o0[~keep]).all() and (gr[~keep] == o0[~keep]).all()
    kk = torch.as_tensor(keep, device=DEV)
    twithin(T(gf[keep]), T(gr[keep]), (b_dev + rows_b)[kk] + 2 * U * T(np.abs(gf[keep]) + np.abs(gf - o0)[keep]),
            "fused vs rows lhood")
    # d-logits: fused against nll_bwd_scaled on the same lse (in place, as the engine calls it)
    C = pool.out((M, N))
    tc_run(eng, "vocab_dlogits_tc", [dA.ptr(offA), dB, db_, dt, di, lse_d, C, ds], [M, N, K, lda, K, N])
    Lw = pool(X)
    run(eng, "nll_bwd_scaled", [Lw, lse_d, dt, di, ds, Lw], [M, N])
    gd, gn = T(C.get()), T(Lw.get())
    l = T(lse_d.get())
    a = (x - l[:, None]).abs()
    q = torch.exp(x - l[:, None])
    sb = T(np.abs(neg_g))[:, None] * q * (2 * U * (2 + 1.173 * a) + ULP_FN + 2 * U * a) + 4 * U * gn.abs()
    twithin(gd, gn, sb, "fused vs rows dlogits")
    # draws: equal logits give equal keys, so the tokens agree everywhere
    tok, ans, lp = pool.out(M, np.int32), pool.out((M, 3), np.int32), pool.out((M, 2))
    o = [pool.out((M, S)), pool.out((M, S)), pool.out((M, S)), pool.out((M, S), np.int32), pool.out((M, S))]
    tc_run(eng, "vocab_sample_tc", [dA.ptr(offA), dB, db_] + o, [M, N, K, lda, K, SEED, 2, 5, 2], [0.8])
    run(eng, "vocab_sample_finish", o + [tok, ans, lp], [S, M, 2, 2])
    tok2, ans2, lp2 = pool.out(M, np.int32), pool.out((M, 3), np.int32), pool.out((M, 2))
    run(eng, "logsoftmax_sample_rows", [Lm, tok2, ans2, lp2], [M, N, 2, SEED, 2, 5, 2], [0.8])
    assert (tok.get() == tok2.get()).all(), "fused and materialised draws"
    g1, g2 = lp.get()[:, 1], lp2.get()[:, 1]
    twithin(T(g1), T(g2), b_dev + rows_b + 2 * U * T(np.abs(g2)), "fused vs rows sampled logp")


# ---------------------------------------------------------------------------------------------- materialised helpers
@pytest.mark.parametrize("V", [40, 257, 10000])
def test_nll_bwd_scaled_and_scale_copy(eng, pool, V):
    rows = 200
    rng = np.random.default_rng(V + 9)
    x = f32(rng.standard_normal((rows, V)) * 3)
    x[:10] += 50.0
    tgt = rng.integers(1, V + 1, rows).astype(np.int32)
    tgt[:3] = [0, V, 1]
    tgt[rng.random(rows) < 0.1] = 0
    ids = rng.integers(1, 9, rows).astype(np.int32)
    ids[rng.random(rows) < 0.1] = 0
    keep = (ids != 0) & (tgt > 0)
    s = f32(rng.standard_normal(rows))
    s[::7] = 0.0
    s[1] = -2.5
    x64 = x.astype(np.float64)
    mx = x64.max(1)
    L = f32(mx + np.log(np.exp(x64 - mx[:, None]).sum(1))).astype(np.float64)
    q = np.exp(x64 - L[:, None])
    onehot = np.arange(V)[None, :] == (tgt - 1)[:, None]
    ref = np.where(keep[:, None], s[:, None] * (q - onehot), 0)
    bound = np.abs(s)[:, None] * q * (ULP_FN + U * np.abs(x64 - L[:, None])) + 2 * U * np.abs(ref)
    dx, dL, dt, di, dsc = pool(x), pool(f32(L)), pool(tgt), pool(ids), pool(s)
    out = pool.out((rows, V))
    run(eng, "nll_bwd_scaled", [dx, dL, dt, di, dsc, out], [rows, V])
    got = out.get()
    within(got, ref, bound, "nll_bwd_scaled")
    assert (got[~keep] == 0).all() and (got[keep & (s == 0)] == 0).all()
    run(eng, "nll_bwd_scaled", [dx, dL, dt, di, dsc, dx], [rows, V])            # in place, as the engine calls it
    assert (dx.get().view(np.uint32) == got.view(np.uint32)).all(), "in place == out of place"
    for alpha in (-1.0, 0.37, 0.0):
        n = rows * V - 3
        dst = pool.out(n)
        run(eng, "scale_copy", [dst, pool(x.reshape(-1)[:n])], [n], [alpha])
        assert (dst.get() == np.float32(alpha) * x.reshape(-1)[:n]).all(), ("scale_copy", alpha)


# ---------------------------------------------------------------------------------------------- refusals
def test_refusals(eng, pool):
    """each shape vocab_tc_ok refuses comes back as VD_E_SHAPE with nothing launched and nothing written; a valid call right
    after works"""
    A, B = pool(np.zeros((80, 40), np.float32)), pool(np.zeros((300, 40), np.float32))
    bias = pool(np.zeros(300, np.float32))
    tgt, ids, lse = pool(np.ones(80, np.int32)), pool(np.ones(80, np.int32)), pool(np.zeros(80, np.float32))
    base = dict(M=64, N=256, K=32, offA=0, lda=32, offB=0, ldb=32, offC=0, ldc=256)
    assert vocab_tc_ok(*(base[k] for k in ("M", "N", "K", "offA", "lda", "offB", "ldb")))

    def launch(name, c):
        o = [pool.out(80 * 6) for _ in range(3)] + [pool.out(80 * 6, np.int32), pool.out(80 * 6), pool.out(81 * 300)]
        ints = [c["M"], c["N"], c["K"], c["lda"], c["ldb"]]
        a, b = A.ptr(c["offA"]), B.ptr(c["offB"])
        if name == "vocab_lse_tc":
            rc = call(eng, name, [a, b, bias, tgt, o[0], o[1], o[2]], ints)
        elif name == "vocab_sample_tc":
            rc = call(eng, name, [a, b, bias, o[0], o[1], o[2], o[3], o[4]], ints + [SEED, 1, 0, 1], [1.0])
        else:
            rc = call(eng, name, [a, b, bias, tgt, ids, lse, o[5].ptr(c["offC"]), None], ints + [c["ldc"]])
        return rc, o

    shapes = [dict(M=63), dict(N=252), dict(N=258), dict(K=31), dict(offA=1), dict(offB=1), dict(lda=34), dict(ldb=34),
              dict(offC=1), dict(ldc=258)]
    for kw in shapes:
        c = dict(base, **kw)
        for name in ("vocab_lse_tc", "vocab_sample_tc", "vocab_dlogits_tc"):
            if name != "vocab_dlogits_tc" and ("offC" in kw or "ldc" in kw):
                continue
            assert not (vocab_tc_ok(*(c[k] for k in ("M", "N", "K", "offA", "lda", "offB", "ldb")))
                        and c["offC"] % 4 == 0 and c["ldc"] % 4 == 0)
            n0 = eng.launch_count()
            rc, o = launch(name, c)
            assert rc == VD_E_SHAPE and eng.launch_count() == n0, (name, kw, rc)
            for d in o:
                v = d.get()
                assert (np.isnan(v) if v.dtype == np.float32 else v == ISENT).all(), (name, kw, "a refused call wrote")
            n0 = eng.launch_count()
            rc, _ = launch(name, base)
            check(rc)
            assert eng.launch_count() == n0 + 1, (name, kw)
