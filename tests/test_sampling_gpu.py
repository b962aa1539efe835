"""Model:generateAnswers' sampling on the device (vd_gen_sample, model.lua:581-602) against the rule's numpy twin
(tests/sampling_twin.py).  Each draw is pinned, not only exercised: with the vocabulary projection's weight zeroed the logits
are the bias in every math mode, so every token must be the twin's Gumbel argmax; with real weights the sampled tokens are
replayed through vd_gen_decoder_step with explicit state (what the host sampler did), which checks the initial state, the
feed-back of the samples and both routes (fused projection epilogue / materialised logits).  A device draw may differ from
the float64 twin only where the row's two best keys are closer than 1e-5 (float32 rounding of the keys)."""
import numpy as np
import pytest
from scipy import stats

from helpers import small_batch, small_params
from host_decode import HostStep, start_state
from sampling_twin import draw
from visdial_b200 import VD_MATH_F16, VD_MATH_FP32, VD_MATH_TF32, init_parameters
from visdial_b200 import _lib
from visdial_b200.engine import Batch, Engine, split_parameters

pytestmark = pytest.mark.gpu

MODES = [VD_MATH_FP32, VD_MATH_TF32, VD_MATH_F16]
MODE_IDS = ["fp32", "tf32", "f16"]
# per-step launches (DESIGN §14): the embedding, 3 per LSTM layer (x-projection, recurrent GEMM, pointwise), the vocabulary
# projection and the draw in FP32; 2 per LSTM layer when the layer step takes the fused wgmma kernel (H % 64 == 0), on
# either sampling route (projection + k_logsoftmax_sample_rows, or the MODE_SAMPLE projection + its finish kernel)
STEP_LAUNCHES_FP32 = 9
STEP_LAUNCHES_TC = 7
NEAR_TIE = 1e-5
SEED = (3 << 32) | 77           # both key words in use

# small: the row route in every mode (rows < 64, V < 256); tc: the fused route in the tensor-core modes
SIZES = {"small": dict(V=9, H=32, E=12, D=3), "tc": dict(V=256, H=128, E=64, D=8)}


def _engine(enc, mode, V, H, E, bias=None, seed=5):
    params = small_params(enc, "gen", vocabSize=V, rnnHiddenSize=H, embedSize=E)
    eng = Engine(params)
    eng.set_math_mode(mode)
    eng.set_training(0)
    flat = init_parameters(params, seed=seed)
    if bias is not None:                          # logits = bias on every row whatever the decoder state
        sp = split_parameters(params, flat)
        sp["dec.out.weight"][:] = 0
        sp["dec.out.bias"][:] = bias
    eng.set_parameters(flat)
    return params, eng


def _forward(eng, params, D, seed=7):
    return eng.encoder_forward(Batch(small_batch(params, B=D, seed=seed))).numpy()


def _bias(V, spread, seed=0):
    return (np.random.default_rng(seed).normal(size=V) * spread).astype(np.float32)


def _check_draws(got_tokens, want_tokens, gaps):
    """tokens equal wherever the twin's top-two key gap is >= NEAR_TIE; returns the number of excluded near-ties"""
    ok = gaps >= NEAR_TIE
    bad = np.nonzero(ok & (got_tokens != want_tokens))
    assert bad[0].size == 0, (bad, got_tokens[bad], want_tokens[bad], gaps[bad])
    return int((~ok).sum())


@pytest.mark.parametrize("size", sorted(SIZES))
@pytest.mark.parametrize("mode", MODES, ids=MODE_IDS)
def test_rule_and_counter_layout_exact(mode, size):
    s = SIZES[size]
    V, L, T, r0 = s["V"], 4, 0.8, 13
    bias = _bias(V, 1.5)
    params, eng = _engine("lf-ques", mode, V, s["H"], s["E"], bias=bias)
    _forward(eng, params, s["D"])
    ans, logp = eng.gen_sample(L, V - 1, T, SEED, r0)
    N = ans.shape[0]
    assert ans.shape == (N, L + 1) and logp.shape == (N, L) and N == 10 * s["D"]
    assert (ans[:, 0] == V - 1).all()
    X = np.repeat(bias.astype(np.float64)[None], N, 0)
    lse = np.log(np.exp(bias.astype(np.float64) - bias.max()).sum()) + bias.max()
    excluded = 0
    for t in range(1, L + 1):
        want, gap = draw(X, T, SEED, t, r0)
        excluded += _check_draws(ans[:, t], want, gap)
        np.testing.assert_allclose(logp[:, t - 1], bias[ans[:, t] - 1].astype(np.float64) - lse, rtol=0, atol=1e-5)
    assert excluded <= N * L // 100, excluded
    eng.close()


def _chisquare(counts, p):
    """chi-square p-value with the classes of expected count < 5 pooled into one bin"""
    e = p * counts.sum()
    small = e < 5
    if small.any():
        counts = np.append(counts[~small], counts[small].sum())
        e = np.append(e[~small], e[small].sum())
    return stats.chisquare(counts, e)[1]


@pytest.mark.parametrize("route", ["rows", "fused"])
def test_distribution(route):
    """>= 10 000 draws (every row and step a fresh draw from softmax(bias / T)) for two temperatures"""
    if route == "rows":
        V, H, E, D, L, mode, spread = 9, 32, 12, 20, 50, VD_MATH_FP32, 1.0
    else:
        V, H, E, D, L, mode, spread = 256, 128, 64, 8, 125, VD_MATH_TF32, 0.3
    bias = _bias(V, spread, seed=1)
    params, eng = _engine("lf-ques", mode, V, H, E, bias=bias)
    _forward(eng, params, D)
    for T in (0.6, 1.5):
        ans, _ = eng.gen_sample(L, V - 1, T, 1234, 0)
        assert ans[:, 1:].size >= 10000
        counts = np.bincount(ans[:, 1:].reshape(-1) - 1, minlength=V).astype(np.float64)
        x = bias.astype(np.float64) / T
        p = np.exp(x - x.max())
        p /= p.sum()
        pval = _chisquare(counts, p)
        assert pval > 1e-4, (T, pval)
    eng.close()


def replay(eng, encOut, tokens):
    """the sampled tokens (N, L + 1) fed back through vd_gen_decoder_step with explicit state, as the host sampler stepped
    the decoder: model.lua:581-588 with decoderConnect (gen.lua:63-68).  Returns the (N, V) log-probabilities of every step."""
    h, c = start_state(eng, encOut)                                             # forwardConnect, gen.lua:30-42
    out = []
    with HostStep(eng, encOut.shape[0]) as step:
        for t in range(tokens.shape[1] - 1):
            lp, h, c = step(tokens[:, t], h, c)
            out.append(lp.astype(np.float64))
    return out


@pytest.mark.parametrize("size", sorted(SIZES))
@pytest.mark.parametrize("mode", MODES, ids=MODE_IDS)
@pytest.mark.parametrize("enc", ["lf-ques", "mn-att-ques-im-hist"])
def test_state_chaining_against_the_step_decoder(enc, mode, size):
    s = SIZES[size]
    V, L, T, r0 = s["V"], 8, 0.9, 21
    params, eng = _engine(enc, mode, V, s["H"], s["E"])
    encOut = _forward(eng, params, s["D"])
    ans, logp = eng.gen_sample(L, V - 1, T, SEED, r0)
    lps = replay(eng, encOut, ans)
    N = ans.shape[0]
    tol = 1e-5 if mode == VD_MATH_FP32 else 1e-4
    excluded = 0
    for t in range(1, L + 1):
        np.testing.assert_allclose(logp[:, t - 1], lps[t - 1][np.arange(N), ans[:, t] - 1], rtol=0, atol=tol)
        want, gap = draw(lps[t - 1], T, SEED, t, r0)
        excluded += _check_draws(ans[:, t], want, gap)
    assert excluded <= N * L // 100, excluded
    assert len(np.unique(ans[:, 1:])) > 1
    eng.close()


# ---- Model.generateAnswers over the device dataloader ------------------------------------------------------------
def _model_and_loader(enc, n, seed=77):
    from visdial_b200.dataloader import Dataloader
    from visdial_b200.model import Model
    from visdial_b200.synthetic import make_corpus
    params = small_params(enc, "gen", vocabSize=9)
    raw = make_corpus(params, n, 40, seed=seed, max_ques_len=8, max_ans_len=6, max_cap_len=14)
    model = Model(dict(params, batchSize=1), seed=3)
    model.engine.set_math_mode(VD_MATH_FP32)
    model.engine.set_parameters(init_parameters(params, seed=3))
    opt = dict(params, useHistory="hist" in enc, concatHistory=False, useIm="im" in enc, maxHistoryLen=60, imgNorm=1)
    dl = Dataloader(model.engine).initialize(opt, ["val"], {"val": raw})
    return params, model, dl


def test_dialogs_per_call_gives_the_per_dialog_entries():
    params, model, dl = _model_and_loader("hrea-ques-im-hist", 12)
    R, V = params["maxQuesCount"], params["vocabSize"]
    p = {"sampleWords": 1, "temperature": 1.3, "beamLen": 8, "maxThreads": 12, "seed": 99}
    one = model.generateAnswers(dl, "val", dict(p, dialogsPerCall=1))
    five = model.generateAnswers(dl, "val", dict(p, dialogsPerCall=5))       # batches of 5, 5 and 2
    assert len(one) == len(five) == 12
    differ = 0
    for conv, (a, b) in enumerate(zip(one, five)):
        assert a["image_id"] == b["image_id"] and len(a["dialog"]) == len(b["dialog"]) == R
        rows = [it for it, (x, y) in enumerate(zip(a["dialog"], b["dialog"])) if x["answer"] != y["answer"]]
        for x, y in zip(a["dialog"], b["dialog"]):
            assert x["question"] == y["question"] and len(x["answer"]) == len(y["answer"]) == 9
        if not rows:
            continue
        # a row may differ only from a draw that was a near-tie: replay the one-dialog answers for this dialog
        differ += len(rows)
        model.wrapper.evaluate()
        encOut = model.forwardBackward(dl.getIndexData(np.array([conv]), model.params, "val"), True, True).numpy()
        toks = np.array([d["answer"] for d in a["dialog"]], np.int32)
        lps = replay(model.engine, encOut, toks)
        model.wrapper.training()
        for it in rows:
            t = next(c for c in range(1, 9) if a["dialog"][it]["answer"][c] != b["dialog"][it]["answer"][c])
            _, gap = draw(lps[t - 1][it:it + 1], 1.3, 99, t, conv * R + it)
            assert gap[0] < NEAR_TIE, (conv, it, t, gap)
    assert differ <= 2, differ
    assert all(1 <= tok <= V for d in one for r in d["dialog"] for tok in r["answer"])
    dl.close(); model.engine.close()


@pytest.mark.parametrize("mode,V,H,D,per_step", [(VD_MATH_FP32, 9, 32, 2, STEP_LAUNCHES_FP32),
                                                 (VD_MATH_TF32, 9, 128, 2, STEP_LAUNCHES_TC),
                                                 (VD_MATH_TF32, 256, 128, 8, STEP_LAUNCHES_TC)],
                         ids=["fp32", "tc_rows", "tc_fused"])
def test_launch_count_is_linear_in_beam_len(mode, V, H, D, per_step):
    params, eng = _engine("lf-ques", mode, V, H, 12 if H == 32 else 64)
    _forward(eng, params, D)
    counts = {}
    for L in (2, 7):
        eng.profile_reset()
        eng.gen_sample(L, V - 1, 1.0, 5, 0)
        counts[L] = eng.launch_count()
    assert counts[7] - counts[2] == per_step * 5, counts
    eng.close()


def test_refusals():
    V = 9
    ans, lp = np.zeros(4096, np.int32), np.zeros(4096, np.float32)

    def call(eng, L=5, start=V - 1, T=1.0, r0=0, answer=True, logp=True):
        return eng.lib.vd_gen_sample(eng.h, L, start, T, 7, r0, ans.ctypes.data if answer else None,
                                     lp.ctypes.data if logp else None)

    disc = Engine(small_params("lf-ques", "disc", vocabSize=V))
    assert call(disc) == _lib.VD_E_STATE
    disc.close()
    params, eng = _engine("lf-ques", VD_MATH_FP32, V, 32, 12)
    assert call(eng) == _lib.VD_E_STATE                                       # no encoder forward yet
    with pytest.raises(_lib.VdError):
        eng.gen_sample(5, V - 1, 1.0, 7)
    _forward(eng, params, 2)
    bad = [dict(L=0), dict(L=-1), dict(T=0.0), dict(T=-1.0), dict(T=float("inf")), dict(T=float("nan")), dict(r0=-1),
           dict(start=0), dict(start=V + 1), dict(answer=False)]
    for kw in bad:
        assert call(eng, **kw) == _lib.VD_E_BADARG, kw
    assert call(eng, logp=False) == _lib.VD_OK
    assert call(eng, L=1, start=V, T=1e-3, r0=1 << 40) == _lib.VD_OK
    eng.close()
