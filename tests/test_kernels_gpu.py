"""The engine's pointwise, attention, criterion and decoding kernels one by one, through vd_test_kernel, against fp64 numpy
references written from the contracts in visdial_b200/csrc/kernels.cuh.

Shapes mix the product sizes (H = 512, P = 196, Cm = 512, K = 100, V = 10 000, 640 000 option tokens) with the edges that
change a kernel's code path (column slices, unrolled-loop remainders, accumulator counts, KMAX instances, shared-memory
opt-in).  Every output lives in a buffer with NaN (or sentinel) guard bands: nothing outside the output may change, and
where the contract says "out =" the output starts as NaN and the inputs sit between NaN guards, so a read of a poisoned
element shows as a non-finite result.  "+=" outputs start from non-zero values, so an overwrite fails.

Tolerances are error scales, not observed errors.  U = 2^-24 is fp32's unit roundoff.  A sum computed in fp32 along a
chain of at most n additions is within n U sum|terms| of the exact sum (first order); each bound below names its chain.
exp / log / tanh cost a few ulp each (CUDA's expf, logf, tanhf: <= 2 ulp), and tanh_e, the SAN kernels' exp-based tanh,
carries an absolute error of about 1e-7 (TANH_E_ABS).  A softmax turns an absolute error d of its inputs into a relative
error of at most 2 d of its outputs.  Outputs the code calls bit-identical, integer outputs and pure data movement are
compared with ==."""

import numpy as np
import pytest
import torch

import dense_oracle
import sampling_twin
from helpers import ISENT, Pool, call, run, small_params, within
from oracle import philox
from oracle import visdial_oracle as O
from visdial_b200 import Engine
from visdial_b200._lib import VD_E_BADARG, check

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
TANH_E_ABS = 3e-7            # tanh_e: __expf (2 ulp near 0, i.e. ~2.4e-7 absolute on 1 - e) and __fdividef
ULP_FN = 4 * U               # relative error of one expf / logf / tanhf, with margin
SEED, ITER = 0x1234_5678_9ABC, 7


# ---------------------------------------------------------------------------------------------- plumbing
@pytest.fixture(scope="module")
def eng():
    e = Engine(small_params("lf-ques", "disc"))
    e.profile(True)                       # every launch counted under its launch-site name (test_every_kernel_was_launched)
    yield e
    e.close()


@pytest.fixture
def pool(eng):
    p = Pool(eng)
    yield p
    p.free()


def f32(x):
    return np.asarray(x, np.float32)


def dropout_setup(eng, p):
    eng.set_training(1)
    eng.set_dropout_seed(SEED, ITER)
    return p


def keep_factors(site, n, p):
    if p == 0:
        return np.ones(n)
    return philox.keep_mask(SEED, ITER, site, n, p).astype(np.float64) / (1 - p)


# ---------------------------------------------------------------------------------------------- history attention
def _smem_ok(R, H, nfloats):
    return nfloats * 4 <= 227 * 1024


def mn_fwd_ref(q, h):
    S = np.einsum("bic,bjc->bij", q, h)
    Sa = np.einsum("bic,bjc->bij", np.abs(q), np.abs(h))
    R = q.shape[1]
    mask = np.triu(np.ones((R, R), bool), 1)
    Sm = np.where(mask, -9999999.0, S)
    P = np.exp(Sm - Sm.max(-1, keepdims=True))
    P /= P.sum(-1, keepdims=True)
    return S, Sa, P


@pytest.mark.parametrize("B,R,H", [(320, 10, 512), (1, 1, 32), (320, 10, 1024), (1, 32, 512), (320, 32, 32), (1, 10, 32),
                                   (1, 32, 1024)])
def test_mn_attention(eng, pool, B, R, H):
    rng = np.random.default_rng(B * 1000 + R * 10 + H)
    s = (4.0 / H) ** 0.25
    q, h = f32(rng.standard_normal((B, R, H)) * s), f32(rng.standard_normal((B, R, H)) * s)
    dA = f32(rng.standard_normal((B, R, H)))
    q64, h64, dA64 = q.astype(np.float64), h.astype(np.float64), dA.astype(np.float64)
    fwd_fits, bwd_fits = _smem_ok(R, H, 2 * R * H + R * R), _smem_ok(R, H, 3 * R * H + 2 * R * R)
    dq_, dh_ = pool(q), pool(h)
    probs, hatt = pool.out((B, R, R)), pool.out((B, R, H))
    S, Sa, P = mn_fwd_ref(q64, h64)
    n0 = eng.launch_count()
    rc = call(eng, "mn_attention_fwd", [dq_, dh_, probs, hatt], [B, R, H])
    if not fwd_fits:
        assert rc == -3 and eng.launch_count() == n0, rc
    else:
        check(rc)
        gp, gh = probs.get(), hatt.get()
        mask = np.triu(np.ones((R, R), bool), 1)
        assert (gp[:, mask] == 0).all(), "masked probabilities must be exactly 0"
        dS = U * (H / 32 + 8) * Sa                                   # lane chains of H/32 products, 5 shuffle levels
        bp = P * (2 * dS.max(-1, keepdims=True) + ULP_FN * (R + 4))
        within(gp, P, bp, "mn probs")
        assert np.abs(gp.sum(-1) - 1).max() <= (bp.sum(-1) + U * R).max()
        ref = np.einsum("bij,bjc->bic", P, h64)
        within(gh, ref, np.einsum("bij,bjc->bic", bp, np.abs(h64)) + U * (R + 2) * np.einsum("bij,bjc->bic", P, np.abs(h64)),
               "mn hAtt")
    P32 = f32(P)
    dp_, ddA = pool(P32), pool(dA)
    dq, dh = pool.out((B, R, H)), pool.out((B, R, H))
    n0 = eng.launch_count()
    rc = call(eng, "mn_attention_bwd", [dq_, dh_, dp_, ddA, dq, dh], [B, R, H])
    if not bwd_fits:
        # the launcher's opt-in for more than 227 KB of shared memory fails; the kernel is never launched
        assert rc == -3 and eng.launch_count() == n0, rc
        run(eng, "reduce_sum", [pool(f32([1.0])), pool.out(1)], [1], [1.0])   # the refusal left no stale error behind
        return
    check(rc)
    Pw = P32.astype(np.float64)
    # manual backward at the fp32 probabilities (signed and all-absolute evaluation)
    def bwd(q, h, P, dA, ab):
        dS = np.einsum("bic,bjc->bij", dA, h) * (P > 0 if not ab else 1)
        dot = (P * dS).sum(-1, keepdims=True)
        dSp = P * (dS + dot if ab else dS - dot)
        return (np.einsum("bij,bjc->bic", dSp, h), np.einsum("bij,bic->bjc", dSp, q) + np.einsum("bij,bic->bjc", P, dA))
    rq, rh = bwd(q64, h64, Pw, dA64, False)
    aq, ah = bwd(np.abs(q64), np.abs(h64), Pw, np.abs(dA64), True)
    chain = U * (H / 32 + 2 * R + 12)
    within(dq.get(), rq, chain * aq, "mn dq")
    within(dh.get(), rh, chain * ah, "mn dh")
    if B == 1 and H == 32:
        # the manual backward is autograd's at fp64 probabilities
        qt, ht = torch.tensor(q64, requires_grad=True), torch.tensor(h64, requires_grad=True)
        mask = torch.triu(torch.ones(R, R, dtype=torch.bool), 1)
        Pt = O.mask_softmax(torch.einsum("bic,bjc->bij", qt, ht), mask.expand(B, R, R))
        (torch.einsum("bij,bjc->bic", Pt, ht) * torch.tensor(dA64)).sum().backward()
        tq, th = bwd(q64, h64, Pt.detach().numpy(), dA64, False)
        assert np.allclose(qt.grad.numpy(), tq, rtol=0, atol=1e-9) and np.allclose(ht.grad.numpy(), th, rtol=0, atol=1e-9)


def hrea_ref(sq, sh, Hs):
    B, R = sq.shape
    v = sq[:, :, None] + sh[:, None, :]
    v = np.where(np.triu(np.ones((R, R), bool), 1)[None], 0.0, v)
    v = np.where(v == 0, -np.inf, v)                                  # ReplaceZero(-inf)
    P = np.exp(v - v.max(-1, keepdims=True))
    P /= P.sum(-1, keepdims=True)
    return P, np.einsum("bij,bjc->bic", P, Hs)


@pytest.mark.parametrize("B,R,H", [(320, 10, 512), (1, 1, 32), (320, 10, 1024), (1, 32, 512), (320, 32, 32), (1, 32, 1024)])
def test_hrea_attention(eng, pool, B, R, H):
    rng = np.random.default_rng(B * 1000 + R * 10 + H + 1)
    sq, sh = f32(rng.standard_normal((B, R)) * 2), f32(rng.standard_normal((B, R)) * 2)
    Hs, dA = f32(rng.standard_normal((B, R, H))), f32(rng.standard_normal((B, R, H)))
    for b in range(0, B, 3):                                          # sq_i + sh_j exactly 0 on some j < i
        if R > 2:
            i = 1 + b % (R - 1)
            sh[b, (b // 3) % i] = -sq[b, i]
    sq64, sh64, Hs64, dA64 = (x.astype(np.float64) for x in (sq, sh, Hs, dA))
    P, att = hrea_ref(sq64, sh64, Hs64)
    d = [pool(sq), pool(sh), pool(Hs)]
    probs, gatt = pool.out((B, R, R)), pool.out((B, R, H))
    fwd_fits, bwd_fits = _smem_ok(R, H, R * H + R * R), _smem_ok(R, H, 2 * R * H + 2 * R * R)
    assert fwd_fits
    run(eng, "hrea_attention_fwd", d + [probs, gatt], [B, R, H])
    gp = probs.get()
    assert (gp[P == 0] == 0).all(), "masked and replaced-zero probabilities must be exactly 0"
    dv = U * 2 * (np.abs(sq64)[:, :, None] + np.abs(sh64)[:, None, :])
    bp = P * (2 * dv.max(-1, keepdims=True) + ULP_FN * (R + 4))
    within(gp, P, bp, "hrea probs")
    within(gatt.get(), att, np.einsum("bij,bjc->bic", bp, np.abs(Hs64)) + U * (R + 2) * np.einsum("bij,bjc->bic", P, np.abs(Hs64)),
           "hrea att")
    P32 = f32(P)
    dsq, dsh, dHs = pool.out((B, R)), pool.out((B, R)), pool.out((B, R, H))
    n0 = eng.launch_count()
    rc = call(eng, "hrea_attention_bwd", d + [pool(P32), pool(dA), dsq, dsh, dHs], [B, R, H])
    if not bwd_fits:
        assert rc == -3 and eng.launch_count() == n0, rc
        return
    check(rc)
    Pw = P32.astype(np.float64)

    def bwd(Hs, dA, ab):
        dS = np.einsum("bic,bjc->bij", dA, Hs)
        dot = (Pw * dS).sum(-1, keepdims=True)
        dSp = Pw * (dS + dot if ab else dS - dot)
        return dSp.sum(2), dSp.sum(1), np.einsum("bij,bic->bjc", Pw, dA)
    r = bwd(Hs64, dA64, False)
    a = bwd(np.abs(Hs64), np.abs(dA64), True)
    chain = U * (H / 32 + 2 * R + 12)
    for got, ref, ab, nm in zip((dsq, dsh, dHs), r, a, ("dsq", "dsh", "dHs")):
        within(got.get(), ref, chain * ab, "hrea " + nm)
    if B == 1 and R == 32 and H == 512:
        # against fp64 autograd of the forward (the oracle's MaskFuture + ReplaceZero ops)
        t = [torch.tensor(x, requires_grad=True) for x in (sq64, sh64, Hs64)]
        v = O.replace_zero(O.mask_future(t[0][:, :, None] + t[1][:, None, :]), float("-inf"))
        (torch.einsum("bij,bjc->bic", torch.softmax(v, -1), t[2]) * torch.tensor(dA64)).sum().backward()
        rt = bwd(Hs64, dA64, False)                                  # at fp32 probabilities: differs by O(U)
        for g, ref in zip(t, rt):
            assert np.abs(g.grad.numpy() - ref).max() <= 1e-5 * max(1.0, np.abs(ref).max())


def test_hrea_refuses_more_than_32_rounds(eng, pool):
    B, R, H = 1, 33, 32
    n0 = eng.launch_count()
    rc = call(eng, "hrea_attention_fwd", [pool(np.zeros((B, R), np.float32)), pool(np.zeros((B, R), np.float32)),
                                          pool(np.zeros((B, R, H), np.float32)), pool.out((B, R, R)), pool.out((B, R, H))],
              [B, R, H])
    assert rc < 0 and eng.launch_count() == n0


# ---------------------------------------------------------------------------------------------- SAN
SAN_CASES = [  # (B, R, P, H, Cm, p)
    (8, 8, 196, 512, 512, 0.5),        # the benched sizes (N = 64), CS = 4
    (8, 8, 9, 32, 16, 0.0),            # the small configs: remainder loop only, CS = 1
    (1, 1, 1, 32, 508, 0.5),
    (8, 8, 197, 300, 516, 0.0),        # C4 = 129 over 4 slices; odd float4 column count per half
    (1, 1, 196, 512, 1024, 0.5),
    (8, 8, 197, 300, 508, 0.5),
    (1, 1, 9, 512, 16, 0.0),
]


@pytest.mark.parametrize("B,R,P,H,Cm,p", SAN_CASES)
def test_san(eng, pool, B, R, P, H, Cm, p):
    N = B * R
    rng = np.random.default_rng(N * 7 + P * 3 + H + Cm)
    dropout_setup(eng, p)
    site_t, site_s = 3, 11
    # expand + dropout: img_tr[n] = t[n / R] * f
    t = f32(np.tanh(rng.standard_normal((B, P, H))))
    img_tr = pool.out((N, P, H))
    dt = pool(t)
    run(eng, "san_expand_dropout", [img_tr, dt], [B, R, P, H, site_t], [p])
    ft = keep_factors(site_t, N * P * H, p).reshape(N, P, H)
    ref_img = np.repeat(t.astype(np.float64), R, axis=0) * ft
    g_img = img_tr.get()
    assert (g_img == f32(ref_img)).all(), "san_expand_dropout"
    # scores: s[n,p] = sum_c w_c f tanh(ic + qc) + b
    ic, qc = f32(rng.standard_normal((N, P, Cm))), f32(rng.standard_normal((N, Cm)))
    w, b = f32(rng.standard_normal(Cm) / np.sqrt(Cm) * 4), f32([0.25])
    dic_, dqc_, dw_, db_ = pool(ic), pool(qc), pool(w), pool(b)
    s = pool.out((N, P))
    run(eng, "san_score_fwd", [dic_, dqc_, dw_, db_, s], [N, P, Cm, site_s], [p])
    fs = keep_factors(site_s, N * P * Cm, p).reshape(N, P, Cm)
    y = np.tanh(ic.astype(np.float64) + qc.astype(np.float64)[:, None, :])
    wf = w.astype(np.float64) * fs
    ref_s = (wf * y).sum(-1) + 0.25
    within(s.get(), ref_s, np.abs(wf).sum(-1) * (TANH_E_ABS + 2 * U) + U * (Cm / 32 + 10) * (np.abs(wf * y).sum(-1) + 0.25),
           "san_score_fwd")
    # softmax + attention: u_out = softmax(s) . img_tr + u_in
    s_in = f32(rng.standard_normal((N, P)) * 2)
    u_in = f32(rng.standard_normal((N, H)))
    p_out, u_out = pool.out((N, P)), pool.out((N, H))
    run(eng, "san_softmax_att_fwd", [pool(s_in), p_out, img_tr, pool(u_in), u_out], [N, P, H])
    s64 = s_in.astype(np.float64)
    pr = np.exp(s64 - s64.max(1, keepdims=True))
    pr /= pr.sum(1, keepdims=True)
    bp = pr * (2 * U * np.abs(s64).max(1, keepdims=True) * 2 + ULP_FN * (P / 256 + 12))
    within(p_out.get(), pr, bp, "san softmax p")
    img64 = g_img.astype(np.float64)
    ref_u = np.einsum("np,nph->nh", pr, img64) + u_in
    within(u_out.get(), ref_u, np.einsum("np,nph->nh", bp, np.abs(img64))
           + U * (P + 72) * (np.einsum("np,nph->nh", pr, np.abs(img64)) + np.abs(u_in)), "san u_out")
    # attention backward: dp = du . img_tr, ds = p (dp - sum p dp), dimg_tr = p du
    du = f32(rng.standard_normal((N, H)))
    p32 = f32(pr)
    ds, dimg = pool.out((N, P)), pool.out((N, P, H))
    run(eng, "san_att_bwd", [pool(du), pool(p32), img_tr, ds, dimg], [N, P, H])
    pw, du64 = p32.astype(np.float64), du.astype(np.float64)
    dp = np.einsum("nph,nh->np", img64, du64)
    dpa = np.einsum("nph,nh->np", np.abs(img64), np.abs(du64))
    ref_ds = pw * (dp - (pw * dp).sum(1, keepdims=True))
    within(ds.get(), ref_ds, U * (H / 32 + P / 512 + 16) * pw * (dpa + (pw * dpa).sum(1, keepdims=True)), "san ds")
    ref_di = pw[:, :, None] * du64[:, None, :]
    within(dimg.get(), ref_di, U * np.abs(ref_di), "san dimg_tr")
    # score backward (CS = 4 from Cm = 512): dic, dqc = sum_p dic, dw += sum ds f y, db += sum ds
    dsv = f32(rng.standard_normal((N, P)) + 0.5)                     # mean 0.5: db = sum ds is far from zero
    w0, b0 = f32(rng.standard_normal(Cm)), f32([3.0])
    dicb, dqcb = pool.out((N, P, Cm)), pool.out((N, Cm))
    dwb, dbb = pool(w0), pool(b0)
    args = [pool(dsv), dic_, dqc_, dw_, dicb, dqcb, dwb, dbb]
    run(eng, "san_score_bwd", args, [N, P, Cm, site_s], [p])
    g_dic, g_dqc, g_dw, g_db = dicb.get(), dqcb.get(), dwb.get(), dbb.get()
    ds64 = dsv.astype(np.float64)[:, :, None]
    gfac = ds64 * fs
    ref_dic = gfac * w.astype(np.float64) * (1 - y * y)
    e_dic = np.abs(gfac * w.astype(np.float64)) * (2 * TANH_E_ABS + 8 * U)
    within(g_dic, ref_dic, e_dic + U * np.abs(ref_dic), "san dic")
    within(g_dqc, ref_dic.sum(1), e_dic.sum(1) + U * (P + 68) * np.abs(ref_dic).sum(1), "san dqc")
    tw = gfac * y
    within(g_dw, w0 + tw.sum((0, 1)), (np.abs(gfac) * (TANH_E_ABS + 2 * U)).sum((0, 1))
           + U * (P + N + 70) * (np.abs(tw).sum((0, 1)) + np.abs(w0)), "san dw")
    within(g_db, 3.0 + dsv.astype(np.float64).sum(), U * (P + N + 4) * (np.abs(dsv).sum() + 3.0), "san db")
    # dqc (and dic) are written once, in a fixed order: a second run repeats them bit for bit
    dicb2, dqcb2 = pool.out((N, P, Cm)), pool.out((N, Cm))
    run(eng, "san_score_bwd", [args[0], dic_, dqc_, dw_, dicb2, dqcb2, dwb, dbb], [N, P, Cm, site_s], [p])
    assert (dqcb2.get() == g_dqc).all() and (dicb2.get() == g_dic).all(), "dqc / dic must repeat bit for bit"
    # collapse: dt_pre[b] = sum_r dimg_tr[b R + r] f * (1 - t^2)
    dtp = pool.out((B, P, H))
    run(eng, "san_collapse_bwd", [dimg, dt, dtp], [B, R, P, H, site_t], [p])
    gdi = dimg.get().astype(np.float64) * ft
    sr = gdi.reshape(B, R, P, H).sum(1)
    t64 = t.astype(np.float64)
    ref_dt = sr * (1 - t64 * t64)
    within(dtp.get(), ref_dt, U * (R + 4) * np.abs(gdi).reshape(B, R, P, H).sum(1) * (1 + t64 * t64), "san dt_pre")
    eng.set_training(0)


# ---------------------------------------------------------------------------------------------- option scores, criteria
@pytest.mark.parametrize("N,K,H", [(320, 100, 512), (320, 1, 32), (64, 7, 32), (64, 129, 512), (320, 129, 32), (3, 100, 32)])
def test_disc_scores(eng, pool, N, K, H):
    rng = np.random.default_rng(N + K * 10 + H)
    feat, enc = f32(rng.standard_normal((N, K, H))), f32(rng.standard_normal((N, H)))
    ds = f32(rng.standard_normal((N, K)))
    f64, e64 = feat.astype(np.float64), enc.astype(np.float64)
    sc = pool.out((N, K))
    dfe, den = pool(feat), pool(enc)
    run(eng, "disc_scores_fwd", [dfe, den, sc], [N, K, H])
    within(sc.get(), np.einsum("nkh,nh->nk", f64, e64), U * (H / 32 + 8) * np.einsum("nkh,nh->nk", np.abs(f64), np.abs(e64)),
           "disc scores")
    dfeat, denc = pool.out((N, K, H)), pool.out((N, H))
    run(eng, "disc_scores_bwd", [pool(ds), dfe, den, dfeat, denc], [N, K, H])
    d64 = ds.astype(np.float64)
    rf = d64[:, :, None] * e64[:, None, :]
    within(dfeat.get(), rf, U * np.abs(rf), "disc dfeat")
    within(denc.get(), np.einsum("nk,nkh->nh", d64, f64), U * (K + 2) * np.einsum("nk,nkh->nh", np.abs(d64), np.abs(f64)),
           "disc dencOut")


def _lse_bound(s):
    """error scale of an fp32 log-sum-exp of rows s (max shift, exp of s - max, strided + block sums, log)"""
    K = s.shape[1]
    return ULP_FN * (2 * np.abs(s).max(1) + K / 128 + 24)


@pytest.mark.parametrize("N,K", [(320, 100), (64, 1), (64, 7), (320, 129), (5, 300)])
def test_xent(eng, pool, N, K):
    rng = np.random.default_rng(N * 3 + K)
    s = f32(rng.standard_normal((N, K)) * 5 + 80 * rng.choice([-1, 1], (N, 1)))   # ~80: exp without the max shift overflows
    gt = rng.integers(1, K + 1, N).astype(np.int32)
    s64 = s.astype(np.float64)
    mx = s64.max(1)
    lse = mx + np.log(np.exp(s64 - mx[:, None]).sum(1))
    loss = pool.out(N)
    ds_, dg = pool(s), pool(gt)
    run(eng, "xent_fwd", [ds_, dg, loss], [N, K])
    within(loss.get(), lse - s64[np.arange(N), gt - 1], _lse_bound(s64) + 2 * U * np.abs(s64[np.arange(N), gt - 1]), "xent loss")
    ref_loss = torch.nn.functional.cross_entropy(torch.tensor(s64), torch.tensor(gt - 1, dtype=torch.long), reduction="none")
    assert np.allclose(ref_loss.numpy(), lse - s64[np.arange(N), gt - 1], rtol=0, atol=1e-9)
    dsc = pool.out((N, K))
    run(eng, "xent_bwd", [ds_, dg, dsc], [N, K])
    pr = np.exp(s64 - lse[:, None])
    ref = (pr - np.eye(K)[gt - 1]) / N
    within(dsc.get(), ref, (pr * _lse_bound(s64)[:, None] + 2 * U) / N, "xent dscores")


@pytest.mark.parametrize("N,K", [(32, 100), (64, 1), (64, 7), (320, 129), (5, 300)])
def test_soft_xent(eng, pool, N, K):
    rng = np.random.default_rng(N * 5 + K)
    s = f32(rng.standard_normal((N, K)) * 5 + 80)
    rel = f32(rng.choice([0.0, 0.0, 0.5, 1.0], (N, K)))
    rel[:, 0] = 1.0                                                     # positive row sums, zeros elsewhere
    s64, r64 = s.astype(np.float64), rel.astype(np.float64)
    rs = r64.sum(1)
    mx = s64.max(1)
    lse = mx + np.log(np.exp(s64 - mx[:, None]).sum(1))
    ref_loss = lse - (r64 * s64).sum(1) / rs
    pr = np.exp(s64 - lse[:, None])
    ref_d = (pr - r64 / rs[:, None]) / N
    # pinned to the dense step's reference (torch cross-entropy with probability targets, autograd)
    st = torch.tensor(s64, requires_grad=True)
    L = dense_oracle.soft_xent(st, torch.tensor(r64))
    L.backward()
    assert abs(L.item() - ref_loss.mean()) <= 1e-9 * abs(ref_loss.mean()) + 1e-12
    assert np.abs(st.grad.numpy() - ref_d).max() <= 1e-12
    outs = []
    for _ in range(2):
        loss, dsc = pool.out(N), pool.out((N, K))
        run(eng, "soft_xent", [pool(s), pool(rel), loss, dsc], [N, K])
        outs.append((loss.get(), dsc.get()))
    dot_b = U * (K / 128 + 12) * (r64 * np.abs(s64)).sum(1) / rs
    within(outs[0][0], ref_loss, _lse_bound(s64) + dot_b + 2 * U * np.abs(ref_loss), "soft_xent loss")
    within(outs[0][1], ref_d, (pr * _lse_bound(s64)[:, None] + U * (K / 128 + 12) * r64 / rs[:, None] + 2 * U) / N,
           "soft_xent dscores")
    assert (outs[0][0] == outs[1][0]).all() and (outs[0][1] == outs[1][1]).all(), "soft_xent must repeat bit for bit"


@pytest.mark.parametrize("n", [1, 1023, 1025, 10 ** 6])
def test_reduce_sum(eng, pool, n):
    rng = np.random.default_rng(n)
    x = f32(rng.standard_normal(n) + 0.25)
    out = pool.out(1)
    run(eng, "reduce_sum", [pool(x), out], [n], [0.5])
    ref = 0.5 * x.astype(np.float64).sum()
    within(out.get(), np.array([ref]), 0.5 * U * (n / 1024 + 14) * np.abs(x).sum() + U * abs(ref), "reduce_sum")


# ---------------------------------------------------------------------------------------------- ranks
def rank_ref(s):
    """rank[k] = 1 + #{j: s_j > s_k or (s_j == s_k and j < k)} (ties to the lower index; -0.0 == +0.0)"""
    K = s.shape[1]
    a, b = s[:, None, :], s[:, :, None]                                # a: s_j, b: s_k
    lower = np.arange(K)[None, :] < np.arange(K)[:, None]              # [k, j]: j < k
    return 1 + ((a > b) | ((a == b) & lower[None])).sum(2)


def test_rank_rows(eng, pool):
    N, K = 320, 100
    rng = np.random.default_rng(5)
    s = f32(rng.integers(-20, 20, (N, K)) * 0.5)                       # many exact duplicates
    s[1] = 3.0                                                          # a row all equal
    s[2, ::2], s[2, 1::2] = 0.0, -0.0                                   # +0.0 / -0.0 ties
    s[3] = rng.standard_normal(K)
    s[4, 50], s[4, 7] = 1e9, 1e9
    gt = rng.integers(1, K + 1, N).astype(np.int32)
    ref = rank_ref(s)
    assert (ref == O.compute_ranks(torch.tensor(s), None).numpy()).all()
    full, gtr = pool.out((N, K), np.int32), pool.out(N, np.int32)
    ds = pool(s)
    run(eng, "rank_rows", [ds, None, full], [N, K])
    run(eng, "rank_rows", [ds, pool(gt), gtr], [N, K])
    g = full.get()
    assert (g == ref).all(), "full ranks"
    assert (np.sort(g, 1) == np.arange(1, K + 1)).all(), "full ranks are a permutation of 1..K"
    assert (gtr.get() == ref[np.arange(N), gt - 1]).all(), "ground-truth ranks"


# ---------------------------------------------------------------------------------------------- vocabulary rows
def _logits(rng, rows, V):
    x = f32(rng.standard_normal((rows, V)) * 3)
    if V >= 768:
        x[0, [5, 261, 517]] = x[0].max() + 1                            # duplicate maxima in three threads' columns
        x[1, 300::256] = 9.0                                            # duplicates in one thread's columns
        x[2, 1] = x[2, 257] = x[2, 513] = x[2, 2] = x[2].max() + 0.5
    for r in range(3, min(rows, 40)):                                   # a run of exact duplicates per row
        x[r, r::7] = 5.5
    return x


def _lsm_ref(x):
    x = x.astype(np.float64)
    mx = x.max(1, keepdims=True)
    return x - mx - np.log(np.exp(x - mx).sum(1, keepdims=True))


@pytest.mark.parametrize("V", [40, 257, 10000])
def test_logsoftmax_nll_lhood(eng, pool, V):
    rows = 200
    rng = np.random.default_rng(V)
    x = _logits(rng, rows, V)
    ids = rng.integers(0, 3, rows).astype(np.int32)                     # one third masked rows
    tgt = rng.integers(0, V + 1, rows).astype(np.int32)                 # target 0 = no loss term
    tgt[:4] = 0
    keep = (ids != 0) & (tgt > 0)
    ref = _lsm_ref(x)
    bound = _lse_bound(x.astype(np.float64))[:, None] + U * np.abs(ref)
    lx = pool(x)
    di, dt = pool(ids), pool(tgt)
    run(eng, "logsoftmax_rows", [lx, di], [rows, V])
    lp = lx.get()
    assert (lp[ids == 0] == 0).all(), "masked rows are all zero"
    within(lp[ids != 0], ref[ids != 0], bound[ids != 0], "logsoftmax_rows")
    lp_all = pool(x)
    run(eng, "logsoftmax_rows", [lp_all, None], [rows, V])
    within(lp_all.get(), ref, bound, "logsoftmax_rows without mask")
    # nll on the fp32 log-probabilities: exact selections / one expf
    loss = pool.out(rows)
    run(eng, "nll_fwd", [lx, dt, di, loss], [rows, V])
    r = np.arange(rows)
    assert (loss.get() == np.where(keep, -lp[r, np.maximum(tgt, 1) - 1], 0)).all(), "nll_fwd"
    dl = pool.out((rows, V))
    run(eng, "nll_bwd", [lx, dt, di, dl], [rows, V])
    e = np.exp(lp.astype(np.float64))
    ref_d = np.where(keep[:, None], e - (np.arange(V)[None] == (tgt - 1)[:, None]), 0)
    within(dl.get(), ref_d, ULP_FN * e + U, "nll_bwd")
    # likelihood from raw logits, accumulated
    lh0 = f32(rng.standard_normal(rows))
    lh = pool(lh0)
    run(eng, "lhood_accumulate", [pool(x), dt, di, lh], [rows, V])
    add = np.where(keep, ref[r, np.maximum(tgt, 1) - 1], 0)
    within(lh.get(), lh0 + add, np.where(keep, bound[r, np.maximum(tgt, 1) - 1], 0) + U * np.abs(lh0 + add), "lhood_accumulate")
    ref_lh = O.compute_lhood(torch.tensor(np.where(keep, tgt, 0)[None], dtype=torch.long), torch.tensor(np.where(ids[:, None] != 0, ref, 0)[None]))
    assert np.allclose(ref_lh.numpy().reshape(-1), add, rtol=0, atol=1e-9)


def test_vocab_lse_finish(eng, pool):
    rows, V = 300, 10000
    npd = pool(np.zeros(1, np.int32), ISENT)
    run(eng, "vocab_lse_nparts", [npd], [V])
    nparts = int(npd.get()[0])
    assert nparts >= 2
    rng = np.random.default_rng(11)
    pm = f32(rng.standard_normal((rows, nparts)) * 5)
    ps = f32(rng.uniform(1, 100, (rows, nparts)))
    tl = f32(rng.standard_normal(rows) * 5)
    tgt = rng.integers(0, 5, rows).astype(np.int32)
    ids = rng.integers(0, 3, rows).astype(np.int32)
    keep = (ids != 0) & (tgt > 0)
    m64, s64 = pm.astype(np.float64), ps.astype(np.float64)
    mx = m64.max(1)
    lse = mx + np.log((s64 * np.exp(m64 - mx[:, None])).sum(1))
    lb = ULP_FN * (np.abs(mx) + np.abs(lse - mx) + nparts + 4) + U * np.abs(m64 - mx[:, None]).max(1) * 2
    for acc in (0, 1):
        o0 = f32(rng.standard_normal(rows))
        lse_o = pool.out(rows)
        out = pool(o0) if acc else pool.out(rows)
        run(eng, "vocab_lse_finish", [pool(pm), pool(ps), pool(tl), pool(tgt), pool(ids), lse_o, out], [nparts, acc, rows], [-1.0])
        within(lse_o.get(), lse, lb, "vocab_lse_finish lse")
        v = np.where(keep, -(tl - lse), 0)
        ref = v + (o0 if acc else 0)
        within(out.get(), ref, np.where(keep, lb + U * np.abs(tl - lse), 0) + U * np.abs(ref), "vocab_lse_finish out")


TOPK_CASES = [(V, k) for V in (40, 257, 10000) for k in (1, 4, 5, 8, 9, 16, 17, 32) if k <= V]


@pytest.mark.parametrize("V,k", TOPK_CASES)
def test_logsoftmax_topk(eng, pool, V, k):
    rows = 64
    rng = np.random.default_rng(V * 40 + k)
    x = _logits(rng, rows, V)
    if V >= 256 * 32:
        for r, t in ((4, 0), (5, 77), (6, 255)):                       # the k best all in thread t's columns c = t mod 256
            x[r, t + 256 * np.arange(k)] = 20.0 + np.arange(k)[::-1] * 0.25
        x[7, 3 + 256 * np.arange(k)] = 20.0                             # ... and all equal there
    ids = np.ones(rows, np.int32)
    ids[8:12] = 0
    lx = pool(x)
    lsm = pool(x)
    run(eng, "logsoftmax_rows", [lsm, pool(ids)], [rows, V])
    L = lsm.get()
    tv, ti = pool.out((rows, k)), pool.out((rows, k), np.int32)
    run(eng, "logsoftmax_topk_rows", [lx, pool(ids), tv, ti], [rows, V, k])
    order = np.lexsort((np.broadcast_to(np.arange(V), L.shape), -L.astype(np.float64)), axis=1)[:, :k]
    gi, gv = ti.get(), tv.get()
    assert (gi == order).all(), "top-k classes: value descending, class ascending"
    assert (gv.view(np.uint32) == np.take_along_axis(L, order, 1).view(np.uint32)).all(), "top-k values == logsoftmax_rows bits"


def test_logsoftmax_topk_refusals(eng, pool):
    x = pool(np.zeros((2, 40), np.float32))
    for V, k in ((40, 33), (8, 9), (40, 0)):
        n0 = eng.launch_count()
        rc = call(eng, "logsoftmax_topk_rows", [x, None, pool.out((2, 33)), pool.out((2, 33), np.int32)], [2, V, k])
        assert rc == VD_E_BADARG and eng.launch_count() == n0, (V, k, rc)


@pytest.mark.parametrize("V,T,stride", [(40, 1.0, 1), (257, 0.7, 1), (10000, 1.0, 1), (10000, 1.3, 3)])
def test_logsoftmax_sample(eng, pool, V, T, stride):
    rows, L, step, off, seed = 96, 5, 3, 17, 0xDEADBEEF12
    rng = np.random.default_rng(V + int(T * 10))
    x = f32(rng.standard_normal((rows, V)) * 2)
    x[:8, :] = 0.0                                                      # flat rows: the Gumbel draw alone decides
    lx = pool(x)
    lsm = pool(x)
    run(eng, "logsoftmax_rows", [lsm, None], [rows, V])
    Lb = lsm.get()
    tok, ans, lp = pool.out(rows, np.int32), pool.out((rows, L + 1), np.int32), pool.out((rows, L))
    run(eng, "logsoftmax_sample_rows", [lx, tok, ans, lp], [rows, V, L, seed, step, off, stride], [T])
    gt, ga, gl = tok.get(), ans.get(), lp.get()
    assert (ga[:, step] == gt).all() and (np.delete(ga, step, 1) == ISENT).all(), "answer column step only"
    assert np.isnan(np.delete(gl, step - 1, 1)).all(), "logp column step - 1 only"
    assert (gl[:, step - 1].view(np.uint32) == Lb[np.arange(rows), gt - 1].view(np.uint32)).all(), "logp == logsoftmax_rows bits"
    checked = 0
    for r in range(rows):
        cls, gap = sampling_twin.draw(x[r:r + 1], T, seed, step, off + r * stride)
        thr = 16 * U * (np.abs(x[r]).max() / T + 20)                    # the device's fp32 key error
        if gap[0] > thr:
            checked += 1
            assert gt[r] == cls[0], (r, gt[r], cls[0], gap[0])
    assert checked >= 0.9 * rows


# ---------------------------------------------------------------------------------------------- embedding, token grouping
def _ids(rng, rows, nv):
    ids = rng.integers(1, nv, rows).astype(np.int32)
    ids[rng.random(rows) < 0.5] = 0                                     # ~50 % pads
    ids[rng.random(rows) < 0.1] = min(3, nv - 1)                        # one heavy hitter
    return ids


@pytest.mark.parametrize("rows,E,ldx,p", [(1, 12, 12, 0.0), (31, 1024, 1028, 0.5), (33, 300, 304, 0.0), (640000, 12, 16, 0.5),
                                          (5000, 300, 300, 0.5)])
def test_embedding(eng, pool, rows, E, ldx, p):
    nv = 41
    rng = np.random.default_rng(rows + E)
    dropout_setup(eng, p)
    site = 9
    emb = f32(rng.standard_normal((nv, E)))
    ids = _ids(rng, rows, nv)
    out = pool.out((rows, E))
    run(eng, "embed_rows", [out, pool(emb), pool(ids)], [rows, E, site], [p])
    fac = keep_factors(site, rows * E, p).reshape(rows, E)
    ref = np.where(ids[:, None] != 0, emb.astype(np.float64)[ids], 0) * fac
    assert (out.get() == f32(ref)).all(), "embed_rows"
    dx = f32(rng.standard_normal((rows, ldx)))
    d0 = f32(rng.standard_normal((nv, E)))
    demb = pool(d0)
    run(eng, "embed_scatter_add", [demb, pool(dx), pool(ids)], [ldx, rows, E, site], [p])
    terms = torch.tensor(dx[:, :E].astype(np.float64) * fac)
    it = torch.tensor(ids, dtype=torch.long)
    ref = torch.tensor(d0.astype(np.float64)).index_add_(0, it, terms).numpy()
    absum = torch.zeros(nv, E, dtype=torch.float64).index_add_(0, it, terms.abs()).numpy()
    cnt = np.bincount(ids, minlength=nv)[:, None]
    within(demb.get(), ref, U * (cnt + 34) * (absum + np.abs(d0)), "embed_scatter_add")
    eng.set_training(0)


def test_embed_scatter_add_refuses_wide_rows(eng, pool):
    n0 = eng.launch_count()
    rc = call(eng, "embed_scatter_add", [pool(np.zeros((2, 1028), np.float32)), pool(np.zeros((1, 1028), np.float32)),
                                         pool(np.ones(1, np.int32))], [1028, 1, 1028, 0], [0.0])
    assert rc < 0 and eng.launch_count() == n0


def _group(eng, pool, ids, nv):
    n = ids.size
    perm, st = pool.out(n, np.int32), pool.out(n, np.int32)
    scratch = pool.out(3 * nv, np.int32)
    run(eng, "group_rows_by_token", [pool(ids), scratch, perm, st], [n, nv])
    scratch.get()
    return perm, st


@pytest.mark.parametrize("n,nv,kind", [(640000, 10000, "mixed"), (640000, 40, "mixed"), (640000, 1025, "mixed"),
                                       (640000, 1025, "pad"), (640000, 1025, "one"), (1, 40, "mixed"), (31, 40, "one"),
                                       (33, 2000, "mixed")])
def test_group_rows_by_token(eng, pool, n, nv, kind):
    rng = np.random.default_rng(n + nv)
    ids = {"mixed": lambda: _ids(rng, n, nv), "pad": lambda: np.zeros(n, np.int32),
           "one": lambda: np.full(n, nv - 1, np.int32)}[kind]()
    perm, st = _group(eng, pool, ids, nv)
    gp, gs = perm.get(), st.get()
    assert (np.sort(gp) == np.arange(n)).all(), "perm is a permutation"
    assert (np.diff(gs) >= 0).all(), "sorted_tok is non-decreasing"
    assert (gs == ids[gp]).all(), "each token's group is exactly its rows"


@pytest.mark.parametrize("ncols", [4, 1020, 2048, 2052])
def test_segsum_rows(eng, pool, ncols):
    n, nv, ldx = 20000, 40, ncols + 8
    rng = np.random.default_rng(ncols)
    ids = _ids(rng, n, nv)
    perm, st = _group(eng, pool, ids, nv)
    X = f32(rng.standard_normal((n, ldx)))
    o0 = f32(rng.standard_normal((nv, ncols)))
    out = pool(o0)
    run(eng, "segsum_rows", [pool(X), perm, st, out], [ldx, n, ncols])
    it = torch.tensor(ids, dtype=torch.long)
    x64 = torch.tensor(X[:, :ncols].astype(np.float64))
    ref = torch.tensor(o0.astype(np.float64)).index_add_(0, it, x64).numpy()
    absum = torch.zeros(nv, ncols, dtype=torch.float64).index_add_(0, it, x64.abs()).numpy()
    cnt = np.bincount(ids, minlength=nv)[:, None]
    within(out.get(), ref, U * (cnt / 64 + 66) * (absum + np.abs(o0)), "segsum_rows")    # <= 64 rows per block, then one red per block


@pytest.mark.parametrize("ncols,scaled", [(8, True), (1016, False), (2048, True), (2056, True)])
def test_segsum_rows16(eng, pool, ncols, scaled):
    n, nv, ldx = 20000, 40, ncols + 8
    rng = np.random.default_rng(ncols + 1)
    ids = _ids(rng, n, nv)
    perm, st = _group(eng, pool, ids, nv)
    X = rng.standard_normal((n, ldx)).astype(np.float16)
    o0 = f32(rng.standard_normal((nv, ncols)))
    out = pool(o0)
    sc = pool(f32([0.25])) if scaled else None
    run(eng, "segsum_rows16", [pool(X.view(np.uint16)), perm, st, out, sc], [ldx, n, ncols])
    s = 0.25 if scaled else 1.0
    it = torch.tensor(ids, dtype=torch.long)
    x64 = torch.tensor(X[:, :ncols].astype(np.float64))
    sums = torch.zeros(nv, ncols, dtype=torch.float64).index_add_(0, it, x64).numpy()
    absum = torch.zeros(nv, ncols, dtype=torch.float64).index_add_(0, it, x64.abs()).numpy()
    cnt = np.bincount(ids, minlength=nv)[:, None]
    ref = o0 + s * sums
    within(out.get(), ref, U * (cnt / 64 + 66) * (s * absum + np.abs(o0)), "segsum_rows16")


def test_cvt_f32_to_f16(eng, pool):
    rows, cols, lds, ldd = 300, 36, 40, 44
    rng = np.random.default_rng(3)
    X = f32(rng.standard_normal((rows, cols)) * np.exp2(rng.integers(-30, 18, (rows, cols))))
    X[0, :12] = [np.inf, -np.inf, np.nan, 65504, 65519.996, 65520, -65520, 1e6, 2 ** -24, 2 ** -25, 3 * 2 ** -26, -0.0]
    X[1, :4] = [1 + 2 ** -11, 1 + 3 * 2 ** -11, 2 ** -14 * (1 - 2 ** -10), 6e-8]    # ties to even, subnormal edges
    src = np.full((rows, lds), np.nan, np.float32)
    src[:, :cols] = X
    dst = pool(np.full((rows, ldd), 0x7e00, np.uint16), 0x7e00)
    run(eng, "cvt_f32_to_f16", [dst, pool(src)], [ldd, lds, rows, cols])
    g = dst.get()
    assert (g[:, cols:] == 0x7e00).all(), "padding columns untouched"
    # round to nearest even (numpy's conversion), saturating at +-65504: the kernel's cvt.rn.satfinite
    ref = np.clip(X, -65504, 65504).astype(np.float16)
    gh = g[:, :cols].view(np.float16)
    nan = np.isnan(X)
    assert np.isnan(gh[nan]).all()
    assert (gh[~nan].view(np.uint16) == ref[~nan].view(np.uint16)).all(), "fp16 conversion"


def test_pick_grad_scale(eng, pool):
    def expect(x):
        a = np.abs(x[~np.isnan(x)]).max() if (~np.isnan(x)).any() else 0.0    # fmaxf skips NaN
        if not (a > 0 and np.isfinite(a)):
            return 1.0
        e = np.frexp(np.float32(a))[1]
        return float(2.0 ** np.clip(10 - e, -60, 60))
    rng = np.random.default_rng(4)
    cases = [np.zeros(8), rng.standard_normal(4000) * 3, np.r_[np.ones(7), 512.0], np.r_[np.zeros(7), 1023.99],
             np.r_[np.zeros(7), 1024.0], np.r_[np.ones(3), np.inf], np.r_[np.full(3, 1e-30), 0.0], np.r_[1e30, np.zeros(3)],
             np.r_[np.full(3, 1e-40), 0.0], np.r_[-700.0, np.zeros(3)], rng.standard_normal(1 << 20) * 1e-5]
    for x in cases:
        x = f32(x)
        bits, sc = pool.out(1, np.int32), pool.out(2)
        run(eng, "pick_grad_scale", [pool(x), bits, sc], [x.size])
        s = expect(x)
        assert (sc.get() == f32([s, 1.0 / s])).all(), (x[:4], sc.get(), s)
        if s != 1.0:
            assert 2 ** 9 <= np.abs(x).max() * s < 2 ** 10 or abs(np.log2(s)) == 60


# ---------------------------------------------------------------------------------------------- small helpers
@pytest.mark.parametrize("rows,cols,ldx,off", [(1000, 512, 512, 0), (1000, 13, 16, 0), (300, 64, 66, 0), (513, 64, 64, 1),
                                               (3, 4, 4, 0)])
def test_colsum_add(eng, pool, rows, cols, ldx, off):
    rng = np.random.default_rng(rows + cols + off)
    X = f32(rng.standard_normal((rows, ldx)))
    img = np.concatenate([np.full(off, np.nan, np.float32), X.reshape(-1)])
    o0 = f32(rng.standard_normal(cols))
    out = pool(o0)
    run(eng, "colsum_add", [out, pool(img).ptr(off)], [rows, cols, ldx])
    x64 = X[:, :cols].astype(np.float64)
    within(out.get(), o0 + x64.sum(0), U * (min(rows, 256) + rows / 256 + 12) * (np.abs(x64).sum(0) + np.abs(o0)), "colsum_add")


@pytest.mark.parametrize("rows,H", [(320, 512), (33, 32), (1, 300)])
def test_rowdot(eng, pool, rows, H):
    rng = np.random.default_rng(rows + H)
    x, w, b = f32(rng.standard_normal((rows, H))), f32(rng.standard_normal(H)), f32([0.5])
    x64, w64 = x.astype(np.float64), w.astype(np.float64)
    out = pool.out(rows)
    dx_, dw_, db_ = pool(x), pool(w), pool(b)
    run(eng, "rowdot_fwd", [out, dx_, dw_, db_], [rows, H])
    within(out.get(), x64 @ w64 + 0.5, U * (H / 32 + 8) * (np.abs(x64) @ np.abs(w64) + 0.5), "rowdot_fwd")
    ds = f32(rng.standard_normal(rows))
    d64 = ds.astype(np.float64)
    for acc in (0, 1):
        dx0 = f32(rng.standard_normal((rows, H)))
        dxb = pool(dx0) if acc else pool.out((rows, H))
        w0, b0 = f32(rng.standard_normal(H)), f32([1.5])
        dwb, dbb = pool(w0), pool(b0)
        run(eng, "rowdot_bwd", [pool(ds), dx_, dw_, dxb, dwb, dbb], [acc, rows, H])
        rdx = d64[:, None] * w64[None] + (dx0 if acc else 0)
        within(dxb.get(), rdx, 2 * U * np.abs(rdx) + U * np.abs(d64[:, None] * w64[None]), "rowdot dx")
        within(dwb.get(), w0 + d64 @ x64, U * (32 + rows / 32 + 4) * (np.abs(d64) @ np.abs(x64) + np.abs(w0)), "rowdot dw")
        within(dbb.get(), 1.5 + d64.sum(), U * (32 + rows / 32 + 4) * (np.abs(d64).sum() + 1.5), "rowdot db")


def test_repeat_and_sum_rows(eng, pool):
    B, R, cols, lds = 7, 10, 37, 41
    rng = np.random.default_rng(8)
    src = f32(rng.standard_normal((B, lds)))
    dst = pool.out((B * R, cols))
    run(eng, "repeat_rows", [dst, pool(src)], [B, R, cols, lds])
    assert (dst.get() == np.repeat(src[:, :cols], R, 0)).all()
    dst2 = pool.out((B * R, lds))
    run(eng, "repeat_rows", [dst2, pool(src)], [B, R, lds, -1])
    assert (dst2.get() == np.repeat(src, R, 0)).all()
    x = f32(rng.standard_normal((B * R, cols)))
    out = pool.out((B, cols))
    run(eng, "sum_repeated_rows", [out, pool(x)], [B, R, cols])
    x64 = x.astype(np.float64).reshape(B, R, cols)
    within(out.get(), x64.sum(1), U * (R + 1) * np.abs(x64).sum(1), "sum_repeated_rows")


def test_masktime(eng, pool):
    T, N, E, I, ldx, off = 6, 50, 12, 8, 24, 3
    rng = np.random.default_rng(9)
    ids = rng.integers(0, 3, (T, N)).astype(np.int32)
    wemb, img = f32(rng.standard_normal((T, N, E))), f32(rng.standard_normal((N, I)))
    out = pool.out((T, N, E + I))
    run(eng, "masktime_concat_fwd", [out, pool(wemb), pool(img), pool(ids)], [T, N, E, I])
    ref_img = O.mask_time(torch.tensor(ids), torch.tensor(img)).numpy()
    assert (out.get() == np.concatenate([wemb, ref_img], -1)).all(), "masktime_concat_fwd"
    dx = f32(rng.standard_normal((T, N, ldx)))
    dimg = pool.out((N, I))
    run(eng, "masktime_bwd", [pool(dx), pool(ids), dimg], [ldx, off, T, N, I])
    t = dx[:, :, off:off + I].astype(np.float64) * (ids != 0)[:, :, None]
    within(dimg.get(), t.sum(0), U * (T + 1) * np.abs(t).sum(0), "masktime_bwd")


def test_id_transposes_and_round_rows(eng, pool):
    B, R, K, T, H = 6, 10, 7, 5, 33
    rng = np.random.default_rng(10)
    src = rng.integers(0, 50, (B * R, T)).astype(np.int32)
    dst = pool.out((T, B * R), np.int32)
    run(eng, "transpose_ids", [pool(src), dst], [B * R, T])
    assert (dst.get() == src.T).all()
    opts = rng.integers(0, 50, (B * R * K, T)).astype(np.int32)
    rnd = rng.integers(0, R, B).astype(np.int32)
    dst = pool.out((T, B * K), np.int32)
    run(eng, "transpose_ids_rounds", [pool(opts), pool(rnd), dst], [B, R, K, T])
    sel = opts.reshape(B, R, K, T)[np.arange(B), rnd].reshape(B * K, T)
    assert (dst.get() == sel.T).all()
    rows = f32(rng.standard_normal((B * R, H)))
    g = pool.out((B, H))
    run(eng, "gather_round_rows", [pool(rows), pool(rnd), g], [B, R, H])
    assert (g.get() == rows.reshape(B, R, H)[np.arange(B), rnd]).all()
    small = f32(rng.standard_normal((B, H)))
    sc = pool.out((B * R, H))
    run(eng, "scatter_round_rows", [pool(small), pool(rnd), sc], [B, R, H])
    ref = np.zeros((B, R, H), np.float32)
    ref[np.arange(B), rnd] = small
    assert (sc.get() == ref.reshape(B * R, H)).all()


def test_clamp_adam(eng, pool):
    n = 4096
    rng = np.random.default_rng(12)
    gs = np.float32(0.5)
    dW = f32(rng.standard_normal(n) * 12)
    edges = f32([10.0, -10.0, np.nextafter(np.float32(10), np.float32(0)), np.nextafter(np.float32(10), np.float32(20)),
                 -np.nextafter(np.float32(10), np.float32(0)), -np.nextafter(np.float32(10), np.float32(20)), 0.0, 1e30])
    dW[:edges.size] = edges                                             # g = dW * 0.5 at +-5 exactly, just inside, just outside
    W, m, v = f32(rng.standard_normal(n)), f32(rng.standard_normal(n) * 0.1), f32(rng.uniform(0, 0.5, n))
    step, b1, b2, eps = 1e-3, 0.9, 0.999, 1e-8
    bufs = [pool(W), pool(dW), pool(m), pool(v)]
    run(eng, "clamp_adam", bufs, [n], [step, b1, b2, eps, float(gs)])
    gW, gdW, gm, gv = (b.get() for b in bufs)
    g32 = np.clip(dW * gs, f32(-5), f32(5))                             # one fp32 product, then the clamp: exact
    assert (gdW == g32).all(), "clamped gradient"
    assert (np.abs(g32[:6]) == 5).sum() == 4 and (np.abs(g32[[2, 4]]) < 5).all()
    g, W64, m64, v64 = (x.astype(np.float64) for x in (g32, W, m, v))
    B1, B2 = float(np.float32(b1)), float(np.float32(b2))
    rm = B1 * m64 + (1 - B1) * g
    rv = B2 * v64 + (1 - B2) * g * g
    within(gm, rm, 3 * U * (B1 * np.abs(m64) + (1 - B1) * np.abs(g)), "adam m")
    within(gv, rv, 4 * U * (B2 * v64 + (1 - B2) * g * g), "adam v")
    tmp = np.sqrt(rv) + float(np.float32(eps))
    rW = W64 - float(np.float32(step)) * rm / tmp
    ratio = np.abs(rm / tmp)
    within(gW, rW, U * np.abs(rW) + float(np.float32(step)) * ratio * 12 * U + U * np.abs(W64), "adam W")
    # the oracle's step (model.lua:96-99, optim_updates.lua:62-91) is the same formula
    st = {"m": torch.tensor(m64), "v": torch.tensor(v64), "t": 0}
    Wt, dWt = torch.tensor(W64), torch.tensor(g)
    lr = float(np.float32(step)) * (1 - B1) / np.sqrt(1 - B2)          # the oracle's bias-corrected step at t = 1
    O.clamp_adam(Wt, dWt, st, lr, beta1=B1, beta2=B2, eps=float(np.float32(eps)))
    assert np.abs(Wt.numpy() - rW).max() <= 1e-12 and np.abs(st["m"].numpy() - rm).max() <= 1e-15


def test_unknown_name_and_wrong_counts(eng, pool):
    x = pool(np.zeros(4, np.float32))
    assert call(eng, "no_such_kernel", [x]) == VD_E_BADARG
    assert call(eng, "reduce_sum", [x], [4], [1.0]) == VD_E_BADARG
    assert call(eng, "reduce_sum", [x, x], [4, 1], [1.0]) == VD_E_BADARG
    assert call(eng, "reduce_sum", [x, x], [4], []) == VD_E_BADARG
    run(eng, "reduce_sum", [x, pool.out(1)], [4], [1.0])


# launch-site names (check_launch) of every launcher the tests above call
LAUNCH_NAMES = [
    "mn_attention_fwd", "mn_attention_bwd", "hrea_attention_fwd", "hrea_attention_bwd",
    "k_san_expand_dropout", "k_san_score_fwd", "san_softmax_att_fwd", "san_att_bwd", "san_score_bwd", "k_san_collapse_bwd",
    "k_disc_scores_fwd", "disc_scores_bwd", "xent_fwd", "xent_bwd", "soft_xent", "reduce_sum", "rank_rows",
    "logsoftmax_rows", "lhood_accumulate", "k_nll_fwd", "k_nll_bwd", "k_vocab_lse_finish", "k_logsoftmax_topk_rows",
    "k_logsoftmax_sample_rows", "k_embed_rows", "embed_scatter_add", "k_tok_hist", "k_tok_scan", "k_tok_fill",
    "k_segsum_rows", "k_cvt16", "k_amax", "k_pick_scale", "k_segsum16", "colsum_add", "k_rowdot_fwd", "rowdot_bwd",
    "k_repeat_rows", "k_sum_repeated_rows", "k_masktime_concat_fwd", "k_masktime_bwd", "k_transpose_ids",
    "k_transpose_ids_rounds", "k_round_rows", "k_clamp_adam",
]


def test_every_kernel_was_launched(eng):
    """runs last: every launcher of the families above ran at least once through vd_test_kernel"""
    missing = [n for n in LAUNCH_NAMES if eng.kernel_stats(n)["launches"] == 0]
    assert not missing, missing
