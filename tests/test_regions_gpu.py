"""Region features on the GPU (DESIGN §26): the masked SAN kernels one by one, the resident corpus's counts and pad rows,
the training step and evaluation of both attention encoders against the region oracle in every math mode, pad invariance,
equivalence to a smaller layout, dialog pools, and the commands end to end on a region features file."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import region_oracle
from helpers import Pool, run, seg_slices, small_batch, small_params, torch_batch, torch_params
from oracle import philox
from visdial_b200 import VD_MATH_F16, VD_MATH_FP32, VD_MATH_TF32, Batch, Engine, init_parameters
from visdial_b200._lib import VD_E_BADARG, VD_E_STATE, VdError, check
from visdial_b200.synthetic import make_batch, make_corpus, write_region_features

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEED, ITER = 77, 3


@pytest.fixture(scope="module")
def eng():
    e = Engine(small_params("lf-ques", "disc"))
    yield e
    e.close()


@pytest.fixture
def pool(eng):
    p = Pool(eng)
    yield p
    p.free()


def f32(x):
    return np.asarray(x, np.float32)


def keep(site, n, p):
    return philox.keep_mask(SEED, ITER, site, n, p).astype(np.float64) / (1 - p)


def rel_close(got, ref, what, tol=2e-5):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    assert np.isfinite(got).all(), what
    scale = max(1.0, float(np.abs(ref).max()))
    assert float(np.abs(got - ref).max()) <= tol * scale, (what, float(np.abs(got - ref).max()), scale)


# ---------------------------------------------------------------------------------------------- kernels
KERNEL_CASES = [(P, H) for P in (36, 100, 196) for H in (64, 512)]


def _counts(rng, B, P):
    c = rng.integers(1, P + 1, size=B).astype(np.int32)
    c[0], c[-1] = 1, P
    return c


@pytest.mark.parametrize("P,H", KERNEL_CASES)
def test_masked_san_kernels(eng, pool, P, H):
    B, R, Cm, p = 3, 2, 64 if H == 64 else 512, 0.5
    N = B * R
    rng = np.random.default_rng(P * 31 + H)
    eng.set_training(1)
    eng.set_dropout_seed(SEED, ITER)
    cnt = _counts(rng, B, P)
    row_c = np.repeat(cnt, R)
    valid = np.arange(P)[None, :] < row_c[:, None]                  # (N, P)
    dcnt = pool(cnt)
    site_s, site_t = 11, 3

    # score forward: valid positions as the unmasked formula, pads 0
    ic, qc = f32(rng.standard_normal((N, P, Cm))), f32(rng.standard_normal((N, Cm)))
    w, b = f32(rng.standard_normal(Cm) / np.sqrt(Cm)), f32([0.25])
    ic_nan = ic.copy()
    ic_nan[~valid] = np.nan
    dic_, dqc_, dw_, db_ = pool(ic_nan), pool(qc), pool(w), pool(b)
    s = pool.out((N, P))
    run(eng, "san_score_fwd_masked", [dic_, dqc_, dw_, db_, s, dcnt], [N, P, Cm, site_s, R], [p])
    fs = keep(site_s, N * P * Cm, p).reshape(N, P, Cm)
    y = np.tanh(ic.astype(np.float64) + qc.astype(np.float64)[:, None, :])
    ref_s = (w * fs * y).sum(-1) + 0.25
    gs = s.get()
    assert (gs[~valid] == 0).all(), "pad scores are 0"
    rel_close(gs[valid], ref_s[valid], "san_score_fwd_masked", 1e-5)

    # softmax + attention: softmax over the valid positions, p = 0 at pads; pad rows of img_tr hold NaN and are never read
    s_in = f32(rng.standard_normal((N, P)) * 2)
    img = f32(rng.standard_normal((N, P, H)))
    img_nan = img.copy()
    img_nan[~valid] = np.nan
    s_nan = s_in.copy()
    s_nan[~valid] = np.nan
    u_in = f32(rng.standard_normal((N, H)))
    dimg = pool(img_nan)
    p_out, u_out = pool.out((N, P)), pool.out((N, H))
    run(eng, "san_softmax_att_fwd_masked", [pool(s_nan), p_out, dimg, pool(u_in), u_out, dcnt], [N, P, H, R])
    s64 = np.where(valid, s_in.astype(np.float64), -np.inf)
    pr = np.exp(s64 - s64.max(1, keepdims=True))
    pr /= pr.sum(1, keepdims=True)
    gp = p_out.get()
    assert (gp[~valid] == 0).all(), "pad probabilities are exactly 0"
    rel_close(gp, pr, "masked softmax p", 1e-5)
    rel_close(u_out.get(), np.einsum("np,nph->nh", pr, np.where(valid[:, :, None], img, 0.0)) + u_in, "masked u_out", 2e-5)

    # attention backward: ds and dimg_tr rows of pads are exact zeros
    du = f32(rng.standard_normal((N, H)))
    p32 = f32(pr)
    ds, dimg_tr = pool.out((N, P)), pool.out((N, P, H))
    run(eng, "san_att_bwd_masked", [pool(du), pool(p32), dimg, ds, dimg_tr, dcnt], [N, P, H, R])
    img0 = np.where(valid[:, :, None], img, 0.0)
    dp = np.einsum("nph,nh->np", img0, du.astype(np.float64))
    pw = p32.astype(np.float64)
    ref_ds = pw * (dp - (pw * dp).sum(1, keepdims=True))
    g_ds, g_di = ds.get(), dimg_tr.get()
    assert (g_ds[~valid] == 0).all() and (g_di[~valid] == 0).all(), "pad ds / dimg_tr rows are exact zeros"
    rel_close(g_ds, ref_ds, "masked ds", 2e-5)
    rel_close(g_di, pw[:, :, None] * du[:, None, :], "masked dimg_tr", 1e-6)

    # score backward: dic pad rows zero, dqc / dw / db summed over the valid positions only
    dsv = f32(rng.standard_normal((N, P)) + 0.5)
    dsv_nan = dsv.copy()
    dsv_nan[~valid] = np.nan
    w0, b0 = f32(rng.standard_normal(Cm)), f32([3.0])
    dicb, dqcb, dwb, dbb = pool.out((N, P, Cm)), pool.out((N, Cm)), pool(w0), pool(b0)
    run(eng, "san_score_bwd_masked", [pool(dsv_nan), dic_, dqc_, dw_, dicb, dqcb, dwb, dbb, dcnt], [N, P, Cm, site_s, R], [p])
    gfac = np.where(valid, dsv, 0.0)[:, :, None] * fs
    ref_dic = gfac * w * (1 - y * y)
    g_dic = dicb.get()
    assert (g_dic[~valid] == 0).all(), "pad dic rows are exact zeros"
    rel_close(g_dic, ref_dic, "masked dic", 1e-5)
    rel_close(dqcb.get(), ref_dic.sum(1), "masked dqc", 2e-5)
    rel_close(dwb.get(), w0 + (gfac * y).sum((0, 1)), "masked dw", 2e-5)
    rel_close(dbb.get(), 3.0 + np.where(valid, dsv, 0.0).sum(), "masked db", 2e-5)

    # collapse: per-dialog counts, pad positions 0
    t = f32(np.tanh(rng.standard_normal((B, P, H))))
    dtp = pool.out((B, P, H))
    run(eng, "san_collapse_bwd_masked", [dimg_tr, pool(t), dtp, dcnt], [B, R, P, H, site_t], [p])
    ft = keep(site_t, N * P * H, p).reshape(N, P, H)
    ref_dt = (g_di.astype(np.float64) * ft).reshape(B, R, P, H).sum(1) * (1 - t.astype(np.float64) ** 2)
    g_dt = dtp.get()
    bvalid = np.arange(P)[None, :] < cnt[:, None]
    assert (g_dt[~bvalid] == 0).all(), "pad dt_pre rows are exact zeros"
    rel_close(g_dt, ref_dt, "masked collapse", 1e-5)


@pytest.mark.parametrize("P,H", KERNEL_CASES)
def test_masked_kernels_with_every_count_at_P_are_the_unmasked_kernels(eng, pool, P, H):
    B, R, Cm, p = 2, 2, 64 if H == 64 else 512, 0.5
    N = B * R
    rng = np.random.default_rng(P + H)
    eng.set_training(1)
    eng.set_dropout_seed(SEED, ITER)
    dcnt = pool(np.full(B, P, np.int32))
    ic, qc = pool(f32(rng.standard_normal((N, P, Cm)))), pool(f32(rng.standard_normal((N, Cm))))
    w, b = pool(f32(rng.standard_normal(Cm) / 8)), pool(f32([0.5]))
    img, s_in, u_in = pool(f32(rng.standard_normal((N, P, H)))), pool(f32(rng.standard_normal((N, P)))), \
        pool(f32(rng.standard_normal((N, H))))
    du, dsv, t = pool(f32(rng.standard_normal((N, H)))), pool(f32(rng.standard_normal((N, P)))), \
        pool(f32(np.tanh(rng.standard_normal((B, P, H)))))
    outs = {}
    for masked in (False, True):
        sfx, extra_p, extra_i = ("_masked", [dcnt], [R]) if masked else ("", [], [])
        s, pr, uo = pool.out((N, P)), pool.out((N, P)), pool.out((N, H))
        ds, di = pool.out((N, P)), pool.out((N, P, H))
        dic, dqc, dw, db = pool.out((N, P, Cm)), pool.out((N, Cm)), pool(np.zeros(Cm, np.float32)), pool(np.zeros(1, np.float32))
        dt = pool.out((B, P, H))
        run(eng, "san_score_fwd" + sfx, [ic, qc, w, b, s] + extra_p, [N, P, Cm, 5] + extra_i, [p])
        run(eng, "san_softmax_att_fwd" + sfx, [s_in, pr, img, u_in, uo] + extra_p, [N, P, H] + extra_i)
        run(eng, "san_att_bwd" + sfx, [du, pr, img, ds, di] + extra_p, [N, P, H] + extra_i)
        run(eng, "san_score_bwd" + sfx, [dsv, ic, qc, w, dic, dqc, dw, db] + extra_p, [N, P, Cm, 5] + extra_i, [p])
        run(eng, "san_collapse_bwd" + sfx, [di, t, dt] + extra_p, [B, R, P, H, 3], [p])
        outs[masked] = [x.get() for x in (s, pr, uo, ds, di, dic, dqc, dt)]
    for a, b_ in zip(outs[False], outs[True]):
        assert np.array_equal(a, b_), "MASK with every count = P must be the unmasked kernel bit for bit"


# ---------------------------------------------------------------------------------------------- engine
def region_params(enc, dec, P, **kw):
    return small_params(enc, dec, imgRegions=P, imgFeatureSize=16, **kw)


ENGINE_CASES = [(enc, dec, mode) for enc in ("mn-att-ques-im-hist", "lf-att-ques-im-hist") for dec in ("disc", "gen")
                for mode in (VD_MATH_FP32, VD_MATH_TF32, VD_MATH_F16)]


def _engine(p, flat, mode, train=True):
    e = Engine(p)
    e.set_math_mode(mode)
    e.set_parameters(flat)
    e.set_training(1 if train else 0)
    e.set_dropout_seed(SEED, ITER)
    e.zero_grad()
    return e


def _step(e, nb):
    e.zero_grad()
    loss = e.forward_backward(Batch(nb))
    return loss, e.get_gradients()


# the dropout seed and iteration of tests/test_parity_gpu.py, whose grid comparison these bounds are
PARITY_SEED, PARITY_ITER = 11, 3


@pytest.mark.parametrize("enc,dec,mode", ENGINE_CASES)
def test_training_step_and_ranks_against_the_region_oracle(enc, dec, mode):
    """test_parity_gpu's training comparison (sizes, batch, dropout seed, FP32 bounds) on 9 region rows with counts"""
    p = small_params(enc, dec, imgRegions=9)
    flat = init_parameters(p, seed=3)
    nb = small_batch(p)
    assert nb["img_count"].min() == 1 and nb["img_count"].max() == 9
    e = _engine(p, flat, mode)
    e.set_dropout_seed(PARITY_SEED, PARITY_ITER)
    loss, grads = _step(e, nb)
    with region_oracle.regions() as O:
        ref = O.forward_backward(O.Ctx(train=True, mask_fn=philox.make_mask_fn(PARITY_SEED, PARITY_ITER)), p,
                                 torch_params(p, flat), torch_batch(nb))
    tol = 1e-4 if mode == VD_MATH_FP32 else 5e-3
    assert abs(loss - ref["loss"]) <= tol * max(1.0, abs(ref["loss"])), (loss, ref["loss"])
    # FP32: test_parity_gpu's bounds for the grid (atol 2e-5, rtol 2e-4 of the segment's largest gradient)
    atol, rtol = (2e-5, 2e-4) if mode == VD_MATH_FP32 else (2e-5, 3e-2)
    for name, sl in seg_slices(p).items():
        r = ref["grads"][name].numpy().ravel()
        err = float(np.abs(grads[sl] - r).max())
        assert err <= atol + rtol * float(np.abs(r).max()), (name, mode, err, float(np.abs(r).max()))
    if dec == "disc":
        e.set_training(0)
        ranks = e.retrieve(Batch(nb), use_gt=True)
        with region_oracle.regions() as O:
            ref_r = O.retrieve_batch(O.Ctx(train=False), p, torch_params(p, flat), torch_batch(nb), use_gt=True)
        if mode == VD_MATH_FP32:
            assert np.array_equal(np.asarray(ranks).ravel(), np.asarray(ref_r).ravel())
    e.close()


@pytest.mark.parametrize("enc,dec,mode", ENGINE_CASES)
def test_eval_forward_and_ranks_against_the_region_oracle(enc, dec, mode):
    p = region_params(enc, dec, 12)
    flat = init_parameters(p, seed=5)
    nb = small_batch(p, B=4, seed=9)
    e = _engine(p, flat, mode, train=False)
    enc_out = e.encoder_forward(Batch(nb)).numpy()
    loss = e.forward_backward(Batch(nb), only_forward=True)
    with region_oracle.regions() as O:
        ref = O.forward_backward(O.Ctx(train=False), p, torch_params(p, flat), torch_batch(nb), only_forward=True)
    tol = 2e-5 if mode == VD_MATH_FP32 else 5e-3
    assert float(np.abs(enc_out - ref["encOut"].numpy()).max()) <= tol, mode
    assert abs(loss - ref["loss"]) <= (1e-4 if mode == VD_MATH_FP32 else 5e-3) * max(1.0, abs(ref["loss"]))
    if dec == "disc" and mode == VD_MATH_FP32:
        ranks = e.retrieve(Batch(nb), use_gt=False)
        with region_oracle.regions() as O:
            ref_r = O.retrieve_batch(O.Ctx(train=False), p, torch_params(p, flat), torch_batch(nb), use_gt=False)
        assert np.array_equal(np.asarray(ranks).ravel(), np.asarray(ref_r).ravel())
    e.close()


@pytest.mark.parametrize("enc,dec,mode", ENGINE_CASES)
def test_pad_rows_do_not_matter(enc, dec, mode):
    p = region_params(enc, dec, 12)
    flat = init_parameters(p, seed=6)
    nb = small_batch(p, B=4, seed=10)
    pad = np.arange(12)[None, :] >= nb["img_count"][:, None]
    e = _engine(p, flat, mode)
    base = _step(e, nb)
    for v in (1e3, -1e3):
        other = dict(nb)
        other["img_feat"] = nb["img_feat"].copy()
        other["img_feat"][pad] = v
        got = _step(e, other)
        assert got[0] == base[0], ("pad values changed the loss", v)
        for name, sl in seg_slices(p).items():
            # Exact: the SAN's weight gradients, among them those of the two GEMMs over all N*P rows (san.img, the hops'
            # img_common), where a pad value would leak first.  The rest agree to rounding only, because two runs of one
            # step do not repeat them bit for bit: biases (k_colsum_add), the embedding table (k_embed_scatter_add), the
            # score's dw, db (k_san_score_bwd) are summed with atomics, and the LSTM weight gradients in some routes too.
            if not (name.startswith("san.") and name.endswith(".weight") and ".score." not in name):
                scale = max(float(np.abs(base[1][sl]).max()), 1e-30)
                assert float(np.abs(got[1][sl] - base[1][sl]).max()) <= 1e-5 * scale, ("pad values changed", name, v)
            else:
                assert np.array_equal(got[1][sl], base[1][sl]), ("pad values changed", name, v)
    e.close()


@pytest.mark.parametrize("enc", ["mn-att-ques-im-hist", "lf-att-ques-im-hist"])
def test_regions_without_counts_step_as_the_grid(enc):
    """imgRegions = S*S without counts runs the grid's kernels on the same rows: the same step as the grid engine"""
    g = small_params(enc, "disc")
    r = dict(g, imgRegions=g["imgSpatialSize"] ** 2)
    flat = init_parameters(g, seed=3)
    nb = small_batch(g, B=4, seed=7)
    rb = dict(nb, img_feat=np.ascontiguousarray(nb["img_feat"].reshape(4, r["imgRegions"], -1)))
    out = []
    for p, b in ((g, nb), (r, rb)):
        e = _engine(p, flat, VD_MATH_FP32)
        out.append(_step(e, b))
        e.close()
    assert out[0][0] == out[1][0]
    for name, sl in seg_slices(g).items():
        scale = max(float(np.abs(out[0][1][sl]).max()), 1e-30)
        assert float(np.abs(out[0][1][sl] - out[1][1][sl]).max()) <= 1e-6 * scale, name


@pytest.mark.parametrize("enc,dec", [("mn-att-ques-im-hist", "disc"), ("lf-att-ques-im-hist", "gen")])
def test_pads_behave_as_if_removed(enc, dec):
    """P = 12 with counts against the same images laid out at P = max count, dropout off (eval-mode masks)"""
    p = region_params(enc, dec, 12, dropout=0.0)
    flat = init_parameters(p, seed=7)
    nb = small_batch(p, B=4, seed=11)
    nb["img_count"] = np.minimum(nb["img_count"], 7).astype(np.int32)
    nb["img_count"][0] = 7
    small = dict(nb, img_feat=np.ascontiguousarray(nb["img_feat"][:, :7]))
    p7 = dict(p, imgRegions=7)
    out = []
    for pp, b in ((p, nb), (p7, small)):
        e = _engine(pp, flat, VD_MATH_FP32, train=False)
        loss = e.forward_backward(Batch(b), only_forward=True)
        out.append((loss, e.encoder_forward(Batch(b)).numpy()))
        e.close()
    assert abs(out[0][0] - out[1][0]) <= 1e-5 * max(1.0, abs(out[1][0]))
    np.testing.assert_allclose(out[0][1], out[1][1], rtol=1e-5, atol=1e-6)


def test_counts_are_refused_outside_their_range_and_on_a_grid_engine():
    p = region_params("mn-att-ques-im-hist", "disc", 12)
    e = _engine(p, init_parameters(p, seed=1), VD_MATH_FP32)
    nb = make_batch(p, 3, seed=2)
    for bad in (0, 13):
        b = dict(nb, img_count=np.array([3, bad, 4], np.int32))
        with pytest.raises(VdError) as ex:
            e.forward_backward(Batch(b))
        assert ex.value.code == VD_E_BADARG
    e.close()
    g = small_params("mn-att-ques-im-hist", "disc")
    eg = _engine(g, init_parameters(g, seed=1), VD_MATH_FP32)
    gb = make_batch(g, 2, seed=3)
    with pytest.raises(VdError):
        eg.forward_backward(Batch(dict(gb, img_count=np.array([1, 1], np.int32))))
    eg.close()


# ---------------------------------------------------------------------------------------------- corpus
def _corpus(p, raw):
    from visdial_b200.dataloader import Corpus
    from visdial_b200.engine import derive_flags
    e = Engine(p)
    opt = derive_flags(dict(p))
    return e, Corpus(e, raw, opt, p["vocabSize"] - 1, p["vocabSize"])


def test_corpus_batches_carry_counts_and_zero_pad_rows():
    p = region_params("mn-att-ques-im-hist", "disc", 10, vocabSize=40, numOptions=100)
    raw = make_corpus(p, 12, 40, seed=3, max_ques_len=8, max_ans_len=6, max_cap_len=14)
    images, counts = raw["images"].copy(), raw["num_boxes"].copy()
    e, c = _corpus(p, raw)
    inds = np.array([3, 0, 7, 11, 1], np.int64)
    b = c.get_batch(inds, 0)
    pos = raw["img_pos"][inds]
    assert np.array_equal(b["img_count"], counts[pos])
    want = images[pos].copy()
    want[np.arange(10)[None, :] >= counts[pos][:, None]] = 0.0
    assert np.array_equal(b["img_feat"], want), "gathered rows: the stored rows, pad rows zeroed"
    stored = c.read("img_fv").reshape(images.shape)
    assert (stored[np.arange(10)[None, :] >= counts[:, None]] == 0).all()
    # counts are set once per corpus: the pad rows they zeroed are gone
    with pytest.raises(VdError) as ex:
        check(e.lib.vd_corpus_region_counts(c.h, counts.ctypes.data, len(counts)))
    assert ex.value.code == VD_E_STATE
    c.close()
    e.close()


def test_refused_counts_leave_the_corpus_as_it_was():
    p = region_params("mn-att-ques-im-hist", "disc", 10, vocabSize=40, numOptions=100)
    raw = make_corpus(p, 12, 40, seed=3, max_ques_len=8, max_ans_len=6, max_cap_len=14)
    images, counts = raw["images"].copy(), raw.pop("num_boxes")
    e, c = _corpus(p, raw)
    inds = np.array([3, 0, 7], np.int64)
    for v in (0, 11):
        bad = counts.copy()
        bad[2] = v
        with pytest.raises(VdError) as ex:
            check(e.lib.vd_corpus_region_counts(c.h, bad.ctypes.data, len(bad)))
        assert ex.value.code == VD_E_BADARG
        assert np.array_equal(c.read("img_fv").reshape(images.shape), images), "a refused call changes no row"
        assert "img_count" not in c.get_batch(inds, 0).keys(), "nor sets counts"
    check(e.lib.vd_corpus_region_counts(c.h, counts.ctypes.data, len(counts)))
    assert np.array_equal(c.get_batch(inds, 0)["img_count"], counts[raw["img_pos"][inds]])
    c.close()
    e.close()


def test_corpus_batch_steps_like_the_host_batch():
    p = region_params("lf-att-ques-im-hist", "disc", 10, vocabSize=40, numOptions=100)
    raw = make_corpus(p, 12, 40, seed=4, max_ques_len=8, max_ans_len=6, max_cap_len=14, ques_len_cap=5, ans_len_cap=4)
    e, c = _corpus(p, raw)
    e.set_math_mode(VD_MATH_FP32)
    e.set_parameters(init_parameters(p, seed=2))
    e.set_training(0)
    b = c.get_batch(np.array([0, 1, 2, 5], np.int64), 0)
    host = Batch(b.numpy())
    l1 = e.forward_backward(b, only_forward=True)
    l2 = e.forward_backward(host, only_forward=True)
    assert l1 == l2
    c.close()
    e.close()


# ---------------------------------------------------------------------------------------------- generation and pools
def test_beam_search_with_mixed_counts_matches_the_oracle():
    p = region_params("mn-att-ques-im-hist", "gen", 12, vocabSize=30)
    flat = init_parameters(p, seed=8)
    nb = make_batch(p, 3, seed=12)
    V, R = p["vocabSize"], p["maxQuesCount"]
    e = _engine(p, flat, VD_MATH_FP32, train=False)
    e.encoder_forward(Batch(nb))
    ans, length, _ = e.gen_beam_search(3, 8, V - 1, V)
    e.close()
    P = torch_params(p, flat)
    with region_oracle.regions() as O:
        for b in range(nb["ques_fwd"].shape[0]):
            one = {k: v[b:b + 1] for k, v in nb.items() if k in ("ques_fwd", "hist", "img_feat", "img_count")}
            ref = O.generate_answers(O.Ctx(train=False), p, P, torch_batch(one), V - 1, V, beam_size=3, beam_len=8,
                                     strict=False)
            for r in range(R):
                n = b * R + r
                if ref[r] is None:
                    assert length[n] == 0, n
                    continue
                L = int(ref[r]["length"])
                assert length[n] == L, (n, length[n], L)
                assert [int(x) for x in ans[n, :L]] == [int(x) for x in np.asarray(ref[r]["answer"]).ravel()[:L]], n


def test_dialog_pool_slots_with_different_counts_answer_as_whole_dialogs():
    p = region_params("mn-att-ques-im-hist", "gen", 12, vocabSize=30)
    flat = init_parameters(p, seed=9)
    nb = make_batch(p, 3, seed=13)
    assert len(set(nb["img_count"].tolist())) > 1
    V, R = p["vocabSize"], p["maxQuesCount"]
    Tq = nb["ques_fwd"].shape[2]
    W = max(nb["hist"].shape[2], Tq) + 20
    e = _engine(p, flat, VD_MATH_FP32, train=False)
    w_ans, w_len, _, _ = e.gen_dialog_beam_search(Batch(nb), 3, 8, V - 1, V, W, 6)
    w_ans, w_len = np.asarray(w_ans).reshape(3, R, -1), np.asarray(w_len).reshape(3, R)
    e.dialog_open(3, Tq, W, 6)
    join = {k: nb[k] for k in ("ques_fwd", "hist", "img_feat", "img_count")}
    slots = np.asarray(e.dialog_join(Batch(join)))
    order = [2, 0, 1]                                    # ask the slots in another order than they joined
    for r in range(R):
        a, length, _ = e.dialog_ask_beam_slots(slots[order], nb["ques_fwd"][order, r], 3, 8, V - 1, V)
        for i, d in enumerate(order):
            assert length[i] == w_len[d, r] and np.array_equal(np.asarray(a)[i], w_ans[d, r]), (r, d)
    e.close()


def test_sampling_with_mixed_counts_matches_the_oracle():
    """FP32 sampling on a batch of mixed counts against oracle.generate_answers' sampling branch drawing with the device's
    rule (sampling_twin): every token equal up to the first step whose two best keys are too close to order in fp32"""
    import sampling_twin
    p = region_params("mn-att-ques-im-hist", "gen", 12, vocabSize=30)
    flat = init_parameters(p, seed=8)
    nb = make_batch(p, 3, seed=14)
    assert len(set(nb["img_count"].tolist())) > 1
    V, L = p["vocabSize"], 8
    e = _engine(p, flat, VD_MATH_FP32, train=False)
    e.encoder_forward(Batch(nb))
    ans, _ = e.gen_sample(L, V - 1, 1.0, 123)
    e.close()
    with region_oracle.regions():
        ref, _, gaps = sampling_twin.generate_answers_sample(p, torch_params(p, flat), torch_batch(nb), V - 1, L, 1.0, 123)
    compared = 0
    for n in range(ref.shape[0]):
        for t in range(1, L + 1):
            if gaps[n, t - 1] < 1e-4:
                break
            assert int(ans[n, t]) == int(ref[n, t]), (n, t)
            compared += 1
    assert compared >= ref.shape[0] * L // 2, compared


def test_resumed_conversation_equals_one_asked_round_by_round():
    """vd_dialog_join_rounds keeps each slot's count: a conversation resumed at round r answers as one asked r times"""
    p = region_params("mn-att-ques-im-hist", "gen", 12, vocabSize=30)
    flat = init_parameters(p, seed=10)
    nb = make_batch(p, 3, seed=15)
    assert len(set(nb["img_count"].tolist())) > 1
    V, R = p["vocabSize"], p["maxQuesCount"]
    Tq = nb["ques_fwd"].shape[2]
    W = max(nb["hist"].shape[2], Tq) + 20
    rounds = np.array([3, 0, 5], np.int32)
    join = {k: nb[k] for k in ("ques_fwd", "hist", "img_feat", "img_count")}
    e = _engine(p, flat, VD_MATH_FP32, train=False)
    # asked round by round; the answers given become the resumed conversations' transcripts
    e.dialog_open(3, Tq, W, 6)
    slots = np.asarray(e.dialog_join(Batch(join)))
    Ta = 8
    answers = np.zeros((3, R, Ta), np.int32)
    asked = {}
    for r in range(R):
        a, length, _ = e.dialog_ask_beam_slots(slots, nb["ques_fwd"][:, r], 3, 8, V - 1, V)
        for d in range(3):
            words = [int(w) for w in np.asarray(a)[d, 1:int(length[d]) - 1]] if length[d] else []
            answers[d, r, :len(words[:Ta])] = words[:Ta]
            asked[(d, r)] = (np.asarray(a)[d].copy(), int(length[d]))
    # resumed at `rounds`, then asked the remaining rounds
    e.dialog_open(3, Tq, W, 6)
    e.dialog_join_rounds(Batch(join), rounds, answers, np.array([2, 0, 1], np.int32))
    slot_of = {0: 2, 1: 0, 2: 1}
    for r in range(R):
        live = [d for d in range(3) if rounds[d] <= r]
        if not live:
            continue
        a, length, _ = e.dialog_ask_beam_slots(np.array([slot_of[d] for d in live]), nb["ques_fwd"][live, r], 3, 8, V - 1, V)
        for i, d in enumerate(live):
            assert int(length[i]) == asked[(d, r)][1] and np.array_equal(np.asarray(a)[i], asked[(d, r)][0]), (d, r)
    e.close()


# ---------------------------------------------------------------------------------------------- commands
V = 40


def _write(d, enc, dec, P):
    from visdial_b200 import h5lite
    p = region_params(enc, dec, P, vocabSize=V, numOptions=100)
    w2i = {"w%d" % i: i for i in range(1, V - 2)}
    w2i["?"] = V - 2                                          # a typed question ends in '?' (utils.question_words)
    ques, imgs, info = {}, {}, {"word2ind": w2i}
    for i, (split, n) in enumerate({"train": 40, "val": 9}.items()):
        raw = make_corpus(p, n, 40, seed=21 + i, max_ques_len=8, max_ans_len=6, max_cap_len=14,
                          ques_len_cap=5 if "lf" in enc else None, ans_len_cap=4 if "lf" in enc else None)
        imgs[split] = (raw.pop("images"), raw.pop("num_boxes"))
        ques.update({k + "_" + split: np.asarray(v, np.uint32) for k, v in raw.items()})
        info["unique_img_" + split] = ["COCO_%s2014_%012d.jpg" % (split, 1000 * i + j) for j in range(n)]
    h5lite.write(os.path.join(d, "visdial_data.h5"), ques)
    write_region_features(os.path.join(d, "data_img.h5"), imgs)
    with open(os.path.join(d, "visdial_params.json"), "w") as f:
        json.dump(info, f)
    flags = ["-inputJson", os.path.join(d, "visdial_params.json"), "-inputQues", os.path.join(d, "visdial_data.h5"),
             "-inputImg", os.path.join(d, "data_img.h5")]
    sizes = ["-encoder", enc, "-decoder", dec] + [x for k in ("embedSize", "rnnHiddenSize", "imgFeatureSize",
                                                             "imgEmbedSize", "commonEmbeddingSize") for x in ("-" + k, str(p[k]))]
    return flags, sizes


def _run(mod, *args, ok=True, stdin=None):
    r = subprocess.run([sys.executable, "-m", "visdial_b200." + mod] + [str(a) for a in args], cwd=ROOT, input=stdin,
                       capture_output=True, text=True, timeout=1200)
    if ok:
        assert r.returncode == 0, (r.stdout[-3000:], r.stderr[-3000:])
    return r


@pytest.mark.parametrize("enc,dec", [("mn-att-ques-im-hist", "disc"), ("lf-att-ques-im-hist", "gen")])
def test_commands_on_a_region_features_file(tmp_path, enc, dec):
    flags, sizes = _write(str(tmp_path), enc, dec, 10)
    save = tmp_path / "ck"
    _run("train", *flags, *sizes, "-numEpochs", 1, "-batchSize", 8, "-savePath", save, "-math", "fp32")
    cks = sorted(save.rglob("*.t7"))
    assert cks, list(save.rglob("*"))
    ck = str(cks[-1])
    from visdial_b200.checkpoint import load_checkpoint
    assert load_checkpoint(ck)["modelParams"]["imgRegions"] == 10
    ranks = tmp_path / "ranks.json"
    _run("evaluate", *flags, "-loadPath", ck, "-useGt", "-batchSize", 4, "-saveRanks", "-saveRankPath", ranks, "-math", "fp32")
    assert ranks.exists()
    gen = tmp_path / "gen"
    extra = ["-sampleWords", 1] if dec == "gen" else []      # a sampled answer always exists; a beam may reach no <END>
    _run("generate", *flags, "-loadPath", ck, "-maxThreads", 3, "-resultPath", gen, "-math", "fp32", *extra)
    data = json.load(open(str(gen / "results.json")))["data"]
    assert len(data) == 3 and all(len(d["dialog"]) == 10 for d in data)
    assert all(isinstance(x["answer"], str) and isinstance(x["question"], str) for d in data for x in d["dialog"])
    # chat -serve 1: two conversations on images of the split, each with its own region count
    ids = [1000, 1001]
    lines = [{"id": "a", "image_id": ids[0], "question": "w1 w2"}, {"id": "b", "image_id": ids[1], "question": "w3"},
             {"id": "a", "question": "w4 w5 w6"}]
    r = _run("chat", *flags, "-loadPath", ck, "-math", "fp32", "-serve", 1, "-capacity", 2, *extra,
             stdin="".join(json.dumps(x) + "\n" for x in lines))
    out = [json.loads(x) for x in r.stdout.splitlines() if x.startswith("{")]
    got = [(o["id"], o["round"]) for o in out if "answer" in o]
    assert sorted(got) == [("a", 0), ("a", 1), ("b", 0)], out
    assert not [o for o in out if "error" in o], out
    # a region file for a model whose imgFeatureSize differs is refused with a message
    bad = _run("train", *flags, *[x if x != "16" else "24" for x in sizes], "-numEpochs", 1, "-savePath", tmp_path / "bad",
               ok=False)
    assert bad.returncode != 0 and "imgFeatureSize" in (bad.stdout + bad.stderr)
