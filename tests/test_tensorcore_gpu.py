"""Tensor-core (wgmma / TF32) path against fp64 numpy and against the oracle.

Stated tolerance for TF32 operands (10-bit mantissa, unit round-off 2^-11, fp32 accumulate): a K-term
contraction of O(1) terms: the tensor core TRUNCATES fp32 operands to TF32 (relative error < 2^-10 per operand),
so a K-term contraction of unit-variance operands has rms error ~ 1e-3 * sqrt(K); the tests bound the rms error
by 1.5e-3 * sqrt(K) and the max error by 8e-3 * sqrt(K) (GEMM primitives) and use rtol 3e-2 on whole-graph
losses / gradients after 20-40 recurrent steps.  Integer outputs (ranks) are compared exactly on rows whose
oracle score gaps exceed the TF32 noise."""
import ctypes as C

import numpy as np
import pytest
import torch

from helpers import full_params, seg_slices, small_params, torch_batch, torch_params
from oracle import philox
from oracle import visdial_oracle as O
from visdial_b200 import VD_MATH_F16, VD_MATH_FP32, VD_MATH_TF32, Batch, Engine, init_parameters
from visdial_b200._lib import check
from visdial_b200.synthetic import make_batch

pytestmark = pytest.mark.gpu


class Dev:
    def __init__(self, eng, arr):
        self.eng, self.shape, self.nbytes = eng, arr.shape, arr.nbytes
        p = C.c_void_p()
        check(eng.lib.vd_device_alloc(eng.h, C.byref(p), arr.nbytes))
        self.p = p
        a = np.ascontiguousarray(arr, dtype=np.float32)
        check(eng.lib.vd_memcpy_h2d(eng.h, p, a.ctypes.data, a.nbytes))

    def get(self):
        out = np.empty(self.shape, dtype=np.float32)
        check(self.eng.lib.vd_memcpy_d2h(self.eng.h, out.ctypes.data, self.p, out.nbytes))
        return out

    def free(self):
        check(self.eng.lib.vd_device_free(self.eng.h, self.p))


@pytest.fixture(scope="module")
def eng():
    e = Engine(small_params("lf-ques", "disc"))
    yield e
    e.close()


def _tn(eng, mode, A, B, Cin, beta, bias, act):
    eng.set_math_mode(mode)
    M, K = A.shape
    N = B.shape[0]
    dA, dB, dC = Dev(eng, A), Dev(eng, B), Dev(eng, Cin)
    dbias = Dev(eng, bias) if bias is not None else None
    check(eng.lib.vd_gemm_tn(eng.h, M, N, K, dA.p, K, dB.p, K, dC.p, N, beta, dbias.p if dbias else None, act))
    out = dC.get()
    for d in (dA, dB, dC) + ((dbias,) if dbias else ()):
        d.free()
    return out


TN_SHAPES = [(128, 128, 32), (128, 256, 64), (256, 128, 512), (300, 2048, 300), (1000, 512, 2048), (77, 300, 512),
             (4096, 2048, 512), (129, 520, 812), (3200, 512, 512)]


@pytest.mark.parametrize("M,N,K", TN_SHAPES)
def test_gemm_tn_tf32_vs_fp64(eng, M, N, K):
    rng = np.random.default_rng(M * 7 + N * 3 + K)
    A = rng.standard_normal((M, K)).astype(np.float32)
    B = rng.standard_normal((N, K)).astype(np.float32)
    ref = A.astype(np.float64) @ B.astype(np.float64).T
    got = _tn(eng, VD_MATH_TF32, A, B, np.zeros((M, N), np.float32), 0.0, None, 0)
    err = np.abs(got - ref).max()
    rms = float(np.sqrt(np.mean((got - ref) ** 2)))
    assert err < 8e-3 * np.sqrt(K) and rms < 1.5e-3 * np.sqrt(K), (err, rms)
    assert err > 0 or K < 8                      # it really ran in reduced precision, not a silent fp32 fallback
    got32 = _tn(eng, VD_MATH_FP32, A, B, np.zeros((M, N), np.float32), 0.0, None, 0)
    assert np.abs(got32 - ref).max() < 2e-5 * np.sqrt(K) * 4


def test_gemm_tn_epilogue_bias_beta_tanh(eng):
    rng = np.random.default_rng(5)
    M, N, K = 200, 384, 96
    A = rng.standard_normal((M, K)).astype(np.float32) * 0.2
    B = rng.standard_normal((N, K)).astype(np.float32) * 0.2
    C0 = rng.standard_normal((M, N)).astype(np.float32)
    bias = rng.standard_normal(N).astype(np.float32)
    ref = np.tanh(1.0 * C0 + bias[None, :] + A.astype(np.float64) @ B.astype(np.float64).T)
    for mode, tol in ((VD_MATH_TF32, 1e-2), (VD_MATH_FP32, 2e-5)):
        got = _tn(eng, mode, A, B, C0.copy(), 1.0, bias, 1)
        assert np.abs(got - ref).max() < tol


ATB_SHAPES = [(128, 128, 256), (300, 2048, 4000), (512, 2048, 6400), (512, 512, 333), (64, 300, 1000), (2048, 812, 2560)]


@pytest.mark.parametrize("M,N,K", ATB_SHAPES)
def test_gemm_atb_vs_fp64(eng, M, N, K):
    rng = np.random.default_rng(M + N + K)
    A = rng.standard_normal((K, M)).astype(np.float32)
    B = rng.standard_normal((K, N)).astype(np.float32)
    C0 = rng.standard_normal((M, N)).astype(np.float32)
    ref = C0 + A.astype(np.float64).T @ B.astype(np.float64)
    for mode, tol in ((VD_MATH_TF32, 8e-3 * np.sqrt(K)), (VD_MATH_FP32, 1e-4 * np.sqrt(K))):
        eng.set_math_mode(mode)
        dA, dB, dC = Dev(eng, A), Dev(eng, B), Dev(eng, C0)
        check(eng.lib.vd_gemm_atb(eng.h, M, N, K, dA.p, M, dB.p, N, dC.p, N))
        got = dC.get()
        for d in (dA, dB, dC):
            d.free()
        assert np.abs(got - ref).max() < tol, mode


@pytest.mark.parametrize("M,N,K,inv", [(128, 256, 64, 1.0), (512, 2048, 6400, 0.25), (512, 2048, 333, 1.0), (256, 1024, 70000, 2.0 ** -7)])
def test_gemm_atb16_vs_fp64(eng, M, N, K, inv):
    """VD_MATH_F16 weight-gradient primitive (both operands MN-major fp16, kind::f16, fp32 accumulate, split-K): exact
    products of the fp16-rounded operands, so only the fp32 accumulation order separates it from fp64."""
    rng = np.random.default_rng(M + N + K)
    A = rng.standard_normal((K, M)).astype(np.float16).astype(np.float32)
    B = rng.standard_normal((K, N)).astype(np.float16).astype(np.float32)
    C0 = rng.standard_normal((M, N)).astype(np.float32)
    ref = C0 + inv * (A.astype(np.float64).T @ B.astype(np.float64))
    dA, dB, dC = Dev(eng, A), Dev(eng, B), Dev(eng, C0)
    check(eng.lib.vd_gemm_atb16(eng.h, M, N, K, dA.p, M, dB.p, N, dC.p, N, inv))
    got = dC.get()
    for d in (dA, dB, dC):
        d.free()
    assert np.abs(got - ref).max() < 2e-6 * K * inv + 1e-5, float(np.abs(got - ref).max())


def _rel(a, b):
    a = np.asarray(a, np.float64).ravel()
    b = np.asarray(b, np.float64).ravel()
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


@pytest.mark.parametrize("enc,dec", [("mn-att-ques-im-hist", "disc"), ("lf-ques", "gen"), ("hrea-ques-im-hist", "gen"),
                                     ("lf-ques-im-hist", "disc")])
def test_tf32_graph_matches_oracle_mid_size(enc, dec):
    """H=128 so that the fused wgmma LSTM kernels (H % 128 == 0) are the ones that run."""
    p = small_params(enc, dec, rnnHiddenSize=128, embedSize=64, vocabSize=200, numOptions=10, commonEmbeddingSize=64,
                     imgFeatureSize=64 if "att" in enc else 256, imgSpatialSize=4, imgEmbedSize=32)
    flat = init_parameters(p, seed=3)
    nb = make_batch(p, 13, seed=7, max_ques_len=9, max_ans_len=6, max_cap_len=12, max_hist_len=14, max_hist_concat=40,
                    empty_round_every=4)
    eng = Engine(p)
    eng.set_math_mode(VD_MATH_TF32)
    eng.set_parameters(flat)
    eng.set_training(1)
    eng.set_dropout_seed(11, 3)
    eng.zero_grad()
    loss = eng.forward_backward(Batch(nb))
    g = eng.get_gradients()
    psite = {O.SITE_FUSION: p["dropout"]}
    ref = O.forward_backward(O.Ctx(train=True, mask_fn=philox.make_mask_fn(11, 3, psite), structure="batched"), p,
                             torch_params(p, flat), torch_batch(nb))
    assert abs(loss - ref["loss"]) < 5e-3 * max(1.0, abs(ref["loss"])), (loss, ref["loss"])
    for name, s in seg_slices(p).items():
        r = ref["grads"][name].numpy().ravel()
        if np.abs(r).max() < 1e-7:
            continue
        assert _rel(g[s], r) < 3e-2, name
    eng.close()


def test_tf32_headline_shapes_and_rank_exactness():
    p = full_params("mn-att-ques-im-hist", "disc")
    flat = init_parameters(p, seed=3)
    nb = make_batch(p, 2, seed=5)
    eng = Engine(p)
    eng.set_math_mode(VD_MATH_TF32)
    eng.set_parameters(flat)
    eng.set_training(1)
    eng.set_dropout_seed(11, 3)
    eng.zero_grad()
    loss = eng.forward_backward(Batch(nb))
    g = eng.get_gradients()
    P = torch_params(p, flat)
    tb = torch_batch(nb)
    ref = O.forward_backward(O.Ctx(train=True, mask_fn=philox.make_mask_fn(11, 3), structure="batched"), p, P, tb)
    assert abs(loss - ref["loss"]) < 5e-3 * max(1.0, abs(ref["loss"])), (loss, ref["loss"])
    # san.hop1.score.bias has a mathematically zero gradient (softmax shift invariance): skip ~0 segments
    worst = max(_rel(g[s], ref["grads"][n].numpy()) for n, s in seg_slices(p).items()
                if float(ref["grads"][n].abs().max()) > 1e-6)
    assert worst < 2e-2, worst
    # Scores within the stated TF32 tolerance; ranks and argmax bit-exact wherever the oracle's gap to every other
    # option exceeds twice the measured score deviation (inside that band a rank flip is legitimate rounding).
    ranks = eng.retrieve(Batch(nb), use_gt=False)
    eng.set_training(0)
    b = Batch(nb)
    eng.encoder_forward(b)
    got_sc = eng.decoder_forward(b).numpy()
    ev = O.forward_backward(O.Ctx(structure="batched"), p, P, tb, only_forward=True)
    sc = ev["decOut"].numpy()
    dev = float(np.abs(got_sc - sc).max())
    assert dev < 5e-3 * max(1.0, float(np.abs(sc).max())), dev
    ref_r = O.compute_ranks(ev["decOut"]).numpy()
    gap = np.abs(sc[:, :, None] - sc[:, None, :]) + np.eye(100)[None] * 1e9
    safe = gap.min(2) > 2 * dev                   # (N,100): options whose score is isolated
    assert safe.mean() > 0.2, (safe.mean(), dev)
    assert np.array_equal(ranks[safe], ref_r[safe])
    srt = np.sort(sc, 1)
    top_ok = (srt[:, -1] - srt[:, -2]) > 2 * dev
    assert top_ok.any()
    assert np.array_equal((ranks == 1).argmax(1)[top_ok], sc.argmax(1)[top_ok])
    eng.close()


def test_tf32_cta_pair_kernels_match_oracle():
    """B=5 dialogs -> 5000 option sequences: enough 128-row tiles (forward 40 x 16, backward 40 x 4 = 160 >= 132 SMs) for
    the SM-filling TF32 step kernels of the option LSTM (k_tc_gemm<128, LSTM_FWD / LSTM_BWD>) to be the ones that run,
    forward and backward.  (The name is historical: these tiles used to run on CTA pairs.)"""
    p = full_params("mn-att-ques-im-hist", "disc")
    flat = init_parameters(p, seed=3)
    nb = make_batch(p, 5, seed=9)
    eng = Engine(p)
    eng.set_math_mode(VD_MATH_TF32)
    eng.set_parameters(flat)
    eng.set_training(1)
    eng.set_dropout_seed(11, 3)
    eng.zero_grad()
    loss = eng.forward_backward(Batch(nb))
    g = eng.get_gradients()
    ref = O.forward_backward(O.Ctx(train=True, mask_fn=philox.make_mask_fn(11, 3), structure="batched"), p,
                             torch_params(p, flat), torch_batch(nb))
    assert abs(loss - ref["loss"]) < 5e-3 * max(1.0, abs(ref["loss"])), (loss, ref["loss"])
    for name in ("opt.lstm.weight", "opt.lstm.bias", "wordEmbed.weight", "ques.lstm1.weight", "san.out.weight"):
        s = seg_slices(p)[name]
        assert _rel(g[s], ref["grads"][name].numpy()) < 2e-2, name
    eng.close()


@pytest.mark.parametrize("mode", [VD_MATH_TF32, VD_MATH_FP32])
def test_option_stream_overlap_is_only_a_schedule(mode):
    """vd_set_option_overlap: the option LSTM on its own stream (SM budget, balanced grids, private embedding-gradient
    buffer) must give the loss, gradients, Adam state and ranks of the one-timeline order.  Only the order of the
    atomic gradient additions differs, so the comparison is at re-association level."""
    p = full_params("mn-att-ques-im-hist", "disc")
    flat = init_parameters(p, seed=5)
    nb = make_batch(p, 4, seed=21)
    out = []
    for overlap in (True, False):
        eng = Engine(p)
        eng.set_math_mode(mode)
        eng.set_option_overlap(overlap, 16)
        eng.set_parameters(flat)
        eng.set_training(1)
        eng.set_dropout_seed(11, 3)
        eng.zero_grad()
        b = Batch(nb)
        ranks = eng.retrieve(b, use_gt=True)               # forward only: no atomics anywhere -> must be identical
        loss = eng.forward_backward(b)
        g = eng.get_gradients()
        eng.clamp_adam_step(1e-3)
        w = eng.get_parameters()
        out.append((loss, g, w, ranks))
        eng.close()
    (l1, g1, w1, r1), (l0, g0, w0, r0) = out
    assert abs(l1 - l0) <= 1e-6 * max(1.0, abs(l0))
    gmax = float(np.abs(g0).max())
    # fp32 re-association only: the pad row of the embedding gradient alone is a sum over ~4e4 rows whose order the
    # counting sort's atomics pick anew on every run (a segment whose true gradient is 0 holds only that noise)
    for name, s in seg_slices(p).items():
        assert float(np.abs(g1[s] - g0[s]).max()) <= 1e-4 * float(np.abs(g0[s]).max()) + 1e-7 * gmax, name
    # one Adam step moves a weight by at most lr; elements with |g| ~ eps turn gradient noise into a fraction of lr
    assert float(np.abs(w1 - w0).max()) <= 2.1e-3
    assert float(np.abs(w1 - w0).mean()) <= 2e-6
    assert np.array_equal(r1, r0)


@pytest.mark.parametrize("enc,dec,B", [("hrea-ques-im-hist", "gen", 2), ("lf-ques-im-hist", "disc", 2), ("lf-ques", "gen", 4)])
def test_tf32_other_configs_at_reference_layer_sizes(enc, dec, B):
    """BASELINE configs 1-3 at the reference's real layer sizes (E=300, H=512, fc7 4096, V=10000 / 1000)."""
    p = full_params(enc, dec, vocabSize=1000 if enc == "lf-ques" else 10000)
    flat = init_parameters(p, seed=3)
    nb = make_batch(p, B, seed=5, max_hist_concat=80)
    eng = Engine(p)
    eng.set_math_mode(VD_MATH_TF32)
    eng.set_parameters(flat)
    eng.set_training(1)
    eng.set_dropout_seed(11, 3)
    eng.zero_grad()
    loss = eng.forward_backward(Batch(nb))
    g = eng.get_gradients()
    psite = {O.SITE_FUSION: p["dropout"]}
    ref = O.forward_backward(O.Ctx(train=True, mask_fn=philox.make_mask_fn(11, 3, psite), structure="batched"), p,
                             torch_params(p, flat), torch_batch(nb))
    assert abs(loss - ref["loss"]) < 5e-3 * max(1.0, abs(ref["loss"])), (loss, ref["loss"])
    for name, s in seg_slices(p).items():
        r = ref["grads"][name].numpy().ravel()
        if np.abs(r).max() < 1e-6:
            continue
        assert _rel(g[s], r) < 3e-2, name
    eng.close()


@pytest.mark.parametrize("B,T0", [(2, None), (11, None)])
def test_f16_option_lstm_matches_oracle(B, T0):
    """VD_MATH_F16: H = 256 and 100 options so that the option LSTM (B*10*100 >= 1024 rows) takes the fp16 CTA-pair kernels
    (first step, recurrent steps, BPTT steps, MN-major weight gradient, fp16 segmented embedding gradient)."""
    p = small_params("mn-att-ques-im-hist", "disc", rnnHiddenSize=256, embedSize=64, vocabSize=300, numOptions=100,
                     commonEmbeddingSize=64, imgFeatureSize=64, imgSpatialSize=4, imgEmbedSize=32)
    flat = init_parameters(p, seed=3)
    nb = make_batch(p, B, seed=7, max_ques_len=9, max_ans_len=6, max_cap_len=12, max_hist_len=14, empty_round_every=4)
    P, tb = torch_params(p, flat), torch_batch(nb)
    ref = O.forward_backward(O.Ctx(train=True, mask_fn=philox.make_mask_fn(11, 3), structure="batched"), p, P, tb)
    ev = O.forward_backward(O.Ctx(structure="batched"), p, P, tb, only_forward=True)
    res = {}
    for mode in (VD_MATH_TF32, VD_MATH_F16):
        eng = Engine(p)
        eng.set_math_mode(mode)
        eng.set_parameters(flat)
        eng.set_training(1)
        eng.set_dropout_seed(11, 3)
        eng.zero_grad()
        loss = eng.forward_backward(Batch(nb))
        g = eng.get_gradients()
        eng.set_training(0)
        b = Batch(nb)
        eng.encoder_forward(b)
        sc = eng.decoder_forward(b).numpy()
        eng.close()
        res[mode] = (loss, g, sc)
    for mode in (VD_MATH_TF32, VD_MATH_F16):
        loss, g, sc = res[mode]
        assert abs(loss - ref["loss"]) < 5e-3 * max(1.0, abs(ref["loss"])), (mode, loss, ref["loss"])
        dev = float(np.abs(sc - ev["decOut"].numpy()).max())
        assert dev < 5e-3 * max(1.0, float(ev["decOut"].abs().max())), (mode, dev)
        for name, s in seg_slices(p).items():
            r = ref["grads"][name].numpy().ravel()
            if np.abs(r).max() < 1e-7:
                continue
            assert _rel(g[s], r) < 3e-2, (mode, name, _rel(g[s], r))
    # the fp16 option LSTM is in the TF32 error class: its deviation from the oracle stays within 2x the TF32 path's
    for name in ("opt.lstm.weight", "opt.lstm.bias", "wordEmbed.weight"):
        s = seg_slices(p)[name]
        r = ref["grads"][name].numpy().ravel()
        assert _rel(res[VD_MATH_F16][1][s], r) < 2.0 * _rel(res[VD_MATH_TF32][1][s], r) + 1e-3, name


@pytest.mark.parametrize("enc", ["lf-ques", "hrea-ques-im-hist"])
def test_fused_vocab_softmax_matches_oracle_and_unfused(enc):
    """gen decoder, tensor-core mode: vd_forward_backward keeps the (rows, V) logits on chip (projection epilogue = online
    softmax statistics + target logit; backward = projection recomputed with softmax - onehot in the epilogue).  Same loss and
    gradients as the oracle (TF32 tolerance) and as the materialising module-level path of the same mode (1e-4: both TF32)."""
    p = small_params(enc, "gen", rnnHiddenSize=128, embedSize=64, vocabSize=300, imgFeatureSize=256, imgEmbedSize=32)
    flat = init_parameters(p, seed=3)
    nb = make_batch(p, 13, seed=7, max_ques_len=9, max_ans_len=6, max_cap_len=12, max_hist_len=14, empty_round_every=4)
    ref = O.forward_backward(O.Ctx(train=True, mask_fn=philox.make_mask_fn(11, 3), structure="batched"), p, torch_params(p, flat),
                             torch_batch(nb))
    out = {}
    for fused in (True, False):
        eng = Engine(p)
        eng.set_math_mode(VD_MATH_TF32)
        eng.set_parameters(flat)
        eng.set_training(1)
        eng.set_dropout_seed(11, 3)
        eng.zero_grad()
        b = Batch(nb)
        if fused:
            loss = eng.forward_backward(b)                       # one crossing: decOut is never handed out
        else:                                                    # module-level calls: decOut materialised (LogSoftMax output)
            eng.encoder_forward(b); eng.forward_connect(); eng.decoder_forward(b)
            loss = eng.criterion_forward(b)
            eng.criterion_backward(b); eng.decoder_backward(b)
            eng.encoder_backward(b, eng.backward_connect(b))
        out[fused] = (loss, eng.get_gradients())
        eng.close()
    lf, gf = out[True]
    lu, gu = out[False]
    assert abs(lf - ref["loss"]) < 5e-3 * abs(ref["loss"]), (lf, ref["loss"])
    assert abs(lf - lu) < 2e-4 * abs(lu), (lf, lu)
    for name, s in seg_slices(p).items():
        r = ref["grads"][name].numpy().ravel()
        if np.abs(r).max() < 1e-7:
            continue
        assert _rel(gf[s], r) < 3e-2, name
        assert _rel(gf[s], gu[s]) < 2e-3, name


def test_fused_vocab_gen_retrieval_ranks():
    """gen retrieval (model.lua:392-420, utils.computeLhood): the option likelihoods come from the fused projection epilogue in the
    tensor-core mode; ranks agree with the oracle wherever its likelihood gaps exceed the TF32 noise, and with fp32 mode mostly."""
    p = small_params("lf-ques", "gen", rnnHiddenSize=128, embedSize=64, vocabSize=300, numOptions=10)
    flat = init_parameters(p, seed=3)
    nb = make_batch(p, 7, seed=9, max_ques_len=9, max_ans_len=6, gen_eval=True)
    ref = O.retrieve_batch(O.Ctx(), p, torch_params(p, flat), torch_batch(nb), use_gt=False).numpy()
    got = {}
    for mode in (VD_MATH_TF32, VD_MATH_FP32):
        eng = Engine(p)
        eng.set_math_mode(mode)
        eng.set_parameters(flat)
        got[mode] = eng.retrieve(Batch(nb), use_gt=False)
        eng.close()
    assert np.array_equal(got[VD_MATH_FP32], ref)
    assert (got[VD_MATH_TF32] == ref).mean() > 0.9
    assert np.array_equal(np.sort(got[VD_MATH_TF32], 1), np.sort(ref, 1))


@pytest.mark.parametrize("enc", ["mn-att-ques-im-hist", "hrea-ques-im-hist"])
def test_persistent_encoder_walks_several_row_blocks(enc):
    """52 dialogs = 520 encoder rows = 5 row blocks of 128 (the last one partial) on the 3 CTA groups of the persistent encoder LSTM
    kernels (enc_lstm.cu): every CTA walks several row blocks in turn, with its barrier phases, flag counters and register state carried
    across them.  F16 mode against the engine's own fp32 mode on one training step (dropout on), loss and per-segment gradients."""
    p = full_params(enc, "disc")
    flat = init_parameters(p, seed=5)
    nb = make_batch(p, 52, seed=9)
    out = {}
    for mode in (VD_MATH_FP32, VD_MATH_F16):
        eng = Engine(p)
        eng.set_math_mode(mode)
        eng.set_parameters(flat)
        eng.set_training(1)
        eng.set_dropout_seed(3, 1)
        eng.zero_grad()
        loss = eng.forward_backward(Batch(nb))
        out[mode] = (loss, eng.get_gradients().astype(np.float64))
        eng.close()
    (l0, g0), (l1, g1) = out[VD_MATH_FP32], out[VD_MATH_F16]
    assert abs(l1 - l0) < 5e-3 * abs(l0), (l0, l1)
    for name, s in seg_slices(p).items():
        m = float(np.abs(g0[s]).max())
        if m < 1e-9:
            continue
        assert float(np.abs(g1[s] - g0[s]).max()) < 3e-2 * m, name
