"""Truncated sampling on the device (DESIGN §23): k_truncated_sample_rows alone against the rule's numpy twin
(tests/truncation_twin.py) and the untruncated sampler, then whole calls (vd_gen_truncated_sample,
vd_gen_dialog_truncated_sample, vd_dialog_ask_truncated_slots), their route and launches, their refusals, and the generate /
chat options.  Where the twin's float32 exp or a replay's logits can move a boundary or a near-tie, a test accepts either
result and counts the rows, as test_sampling_gpu.py counts key gaps below 1e-5."""
import json
import subprocess
import sys

import numpy as np
import pytest
import torch

import truncation_twin as tt
from dialog_history import next_row, right_aligned, row_words, sample_words
from helpers import Buf, run, small_batch, small_params
from test_dialog_generation_gpu import MAX_ANS, ROOT, _width
from test_dialog_pool_gpu import _W, _drive
from test_sampling_gpu import SIZES, STEP_LAUNCHES_FP32, STEP_LAUNCHES_TC, _engine, _forward, _model_and_loader, replay
from visdial_b200 import VD_MATH_F16, VD_MATH_FP32, VD_MATH_TF32
from visdial_b200 import _lib
from visdial_b200.engine import Batch, Engine
from visdial_b200.model import truncates

pytestmark = pytest.mark.gpu

MODES = [VD_MATH_FP32, VD_MATH_TF32, VD_MATH_F16]
MODE_IDS = ["fp32", "tf32", "f16"]
NEAR_TIE = 1e-5
SEED = (3 << 32) | 77


# ---- the kernel alone ---------------------------------------------------------------------------------------------
def _rows(kind, rows, V, seed):
    rng = np.random.default_rng(seed)
    if kind == "random":
        return (rng.normal(size=(rows, V)) * 2.0).astype(np.float32)
    if kind == "ties":                                   # a handful of distinct values: ties at every boundary
        return rng.integers(-2, 3, size=(rows, V)).astype(np.float32)
    x = np.zeros((rows, V), np.float32)                  # "equal": equal masses, -0 beside +0
    x[:, 1::3] = -0.0
    return x


def _kernel(eng, name, x, extra_ints, reals, L=2, step=2, r0=5, stride=3, rounds=None):
    rows, V = x.shape
    bufs = [Buf(eng, x), Buf(eng, np.zeros(rows, np.int32)), Buf(eng, np.zeros((rows, L + 1), np.int32)),
            Buf(eng, np.zeros((rows, L), np.float32))]
    ptrs = bufs + ([None if rounds is None else Buf(eng, np.asarray(rounds, np.int64))] if name == "truncated_sample_rows" else [])
    run(eng, name, ptrs, [rows, V, L, SEED, step, r0, stride] + extra_ints, reals)
    out = bufs[1].get(), bufs[2].get(), bufs[3].get()
    for b in ptrs:
        if b is not None:
            b.free()
    assert (out[1][:, step] == out[0]).all()
    return out[0], out[2][:, step - 1]


def _logsoftmax(eng, x):
    b = Buf(eng, x)
    run(eng, "logsoftmax_rows", [b, None], list(x.shape))
    out = b.get()
    b.free()
    return out


@pytest.fixture(scope="module")
def eng():
    e = Engine(small_params("lf-ques", "gen"))
    yield e
    e.close()


CASES = [(1, 1.0), (3, 1.0), (0, 0.5), (0, 0.9), (50, 0.9), (2, 0.3), (0, 1e-6)]


@pytest.mark.parametrize("V", [5, 9, 37, 257, 10000])
@pytest.mark.parametrize("kind", ["random", "ties", "equal"])
def test_kernel_against_the_twin(eng, V, kind):
    rows, T, step, r0, stride = 48, 0.8, 2, 5, 3
    x = _rows(kind, rows, V, seed=V)
    rounds = r0 + np.arange(rows) * stride
    lsm = _logsoftmax(eng, x)
    free_tok, free_lp = _kernel(eng, "logsoftmax_sample_rows", x, [], [T])
    excluded = ambiguous = 0
    for k, p in CASES + [(V, 1.0), (0, 1.0), (V - 1, 0.999)]:
        tok, lp = _kernel(eng, "truncated_sample_rows", x, [k], [T, p])
        want, either, gap, small, large = tt.draw(x, T, SEED, step, k, p, rounds=rounds)
        r = np.arange(rows)
        # logp: the untruncated LogSoftMax's bits at the drawn token
        assert np.array_equal(lp.view(np.int32), lsm[r, tok - 1].view(np.int32)), (k, p)
        if not truncates(k, p, V):                      # the untruncated kernel bit for bit
            assert np.array_equal(tok, free_tok) and np.array_equal(lp.view(np.int32), free_lp.view(np.int32)), (k, p)
        # every token kept; the coupling with the untruncated draw on the same logits
        assert large[r, tok - 1].all(), (k, p)
        inside = small[r, free_tok - 1]
        assert np.array_equal(tok[inside], free_tok[inside]), (k, p)
        # the twin's draw, except at a near-tie of the keys or an ambiguous boundary
        for i in np.nonzero(tok != want)[0]:
            if len(either[i]) > 1 and tok[i] in either[i]:
                ambiguous += 1
            else:
                assert gap[i] < NEAR_TIE, (k, p, i, tok[i], want[i], gap[i])
                excluded += 1
        # row_round draws what the affine rule draws
        tok2, lp2 = _kernel(eng, "truncated_sample_rows", x, [k], [T, p], r0=0, stride=0, rounds=rounds)
        assert np.array_equal(tok, tok2) and np.array_equal(lp.view(np.int32), lp2.view(np.int32))
    assert excluded + ambiguous <= max(2, rows * len(CASES) // 50), (excluded, ambiguous)


def test_kernel_refuses_what_it_cannot_take(eng):
    x = np.zeros((2, 8), np.float32)
    for k, p in ((-1, 1.0), (0, 0.0), (0, 1.5), (0, float("nan"))):
        with pytest.raises(_lib.VdError) as e:
            _kernel(eng, "truncated_sample_rows", x, [k], [1.0, p])
        assert e.value.code == _lib.VD_E_BADARG
    with pytest.raises(_lib.VdError) as e:
        _kernel(eng, "truncated_sample_rows", np.zeros((1, 49153), np.float32), [5], [1.0, 1.0])
    assert e.value.code == _lib.VD_E_BADARG
    _kernel(eng, "truncated_sample_rows", np.zeros((1, 49152), np.float32), [5], [1.0, 0.5])


# ---- whole calls --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("size", sorted(SIZES))
@pytest.mark.parametrize("mode", MODES, ids=MODE_IDS)
def test_inactive_truncation_is_gen_sample(mode, size):
    s = SIZES[size]
    V, L, T, r0 = s["V"], 6, 0.9, 13
    params, eng = _engine("mn-att-ques-im-hist", mode, s["V"], s["H"], s["E"])
    _forward(eng, params, s["D"])
    ans, logp = eng.gen_sample(L, V - 1, T, SEED, r0)
    for k, p in ((0, 1.0), (V, 1.0), (V + 5, 1.0)):
        a, lp = eng.gen_truncated_sample(L, V - 1, T, SEED, r0, k, p)
        assert np.array_equal(a, ans) and np.array_equal(lp.view(np.int32), logp.view(np.int32)), (k, p)
    eng.close()


TRUNC = {"small": [(3, 1.0), (0, 0.7), (4, 0.8)], "tc": [(20, 1.0), (0, 0.9), (50, 0.9)]}


@pytest.mark.parametrize("size", sorted(SIZES))
@pytest.mark.parametrize("mode", MODES, ids=MODE_IDS)
@pytest.mark.parametrize("enc", ["lf-ques", "mn-att-ques-im-hist"])
def test_active_truncation_against_the_replayed_decoder(enc, mode, size):
    s = SIZES[size]
    V, L, T, r0 = s["V"], 8, 0.9, 21
    params, eng = _engine(enc, mode, V, s["H"], s["E"])
    encOut = _forward(eng, params, s["D"])
    tol = 1e-5 if mode == VD_MATH_FP32 else 1e-4
    eps = 4 * tol / T                                    # replayed y are the device's to within this
    for k, p in TRUNC[size]:
        ans, logp = eng.gen_truncated_sample(L, V - 1, T, SEED, r0, k, p)
        lps = replay(eng, encOut, ans)
        N = ans.shape[0]
        r = np.arange(N)
        excluded = 0
        for t in range(1, L + 1):
            np.testing.assert_allclose(logp[:, t - 1], lps[t - 1][r, ans[:, t] - 1], rtol=0, atol=tol)
            want, either, gap, _, large = tt.draw(lps[t - 1], T, SEED, t, k, p, row_offset=r0, eps=eps, ambiguity=eps)
            assert large[r, ans[:, t] - 1].all(), (k, p, t)
            off = np.nonzero(ans[:, t] != want)[0]
            for i in off:
                assert len(either[i]) > 1 or gap[i] < 2 * eps, (k, p, t, i, gap[i])
            excluded += off.size
        assert excluded <= max(2, N * L // 50), (k, p, excluded)
        assert len(np.unique(ans[:, 1:])) > 1 or k == 1
    eng.close()


def test_dialogs_per_call_gives_the_per_dialog_draws():
    params, model, dl = _model_and_loader("hrea-ques-im-hist", 12)
    p = {"sampleWords": 1, "temperature": 1.3, "beamLen": 8, "maxThreads": 12, "seed": 99, "topK": 4, "topP": 0.9}
    one = model.generateAnswers(dl, "val", dict(p, dialogsPerCall=1))
    five = model.generateAnswers(dl, "val", dict(p, dialogsPerCall=5))
    differ = sum(x["answer"] != y["answer"] for a, b in zip(one, five) for x, y in zip(a["dialog"], b["dialog"]))
    assert differ <= 2, differ                          # only a near-tie draw may differ (test_sampling_gpu.py)
    plain = model.generateAnswers(dl, "val", dict(p, topK=0, topP=1.0, dialogsPerCall=5))
    assert plain != five
    dl.close(); model.engine.close()


@pytest.mark.parametrize("mode,V,H,D,per_step", [(VD_MATH_FP32, 9, 32, 2, STEP_LAUNCHES_FP32),
                                                 (VD_MATH_TF32, 9, 128, 2, STEP_LAUNCHES_TC),
                                                 (VD_MATH_TF32, 256, 128, 8, STEP_LAUNCHES_TC)],
                         ids=["fp32", "tc_rows", "tc_fused"])
def test_launches_per_step_are_the_rows_routes(mode, V, H, D, per_step):
    params, eng = _engine("lf-ques", mode, V, H, 12 if H == 32 else 64)
    _forward(eng, params, D)
    counts = {}
    for L in (2, 7):
        eng.profile_reset()
        eng.gen_truncated_sample(L, V - 1, 1.0, 5, 0, 3, 0.9)
        counts[L] = eng.launch_count()
    assert counts[7] - counts[2] == per_step * 5, counts
    eng.close()


def test_refusals_leave_the_engine_usable():
    V = 9
    ans, lp = np.zeros(4096, np.int32), np.zeros(4096, np.float32)

    def call(eng, k, p, L=5):
        return eng.lib.vd_gen_truncated_sample(eng.h, L, V - 1, 1.0, 7, 0, k, p, ans.ctypes.data, lp.ctypes.data)

    bad = [(-1, 1.0), (-5, 0.5), (0, 0.0), (0, -0.5), (0, 1.5), (0, float("nan")), (0, float("inf"))]
    disc = Engine(small_params("lf-ques", "disc", vocabSize=V))
    assert call(disc, 3, 0.9) == _lib.VD_E_STATE
    disc.close()
    params, eng = _engine("hrea-ques-im-hist", VD_MATH_FP32, V, 32, 12)
    assert call(eng, 3, 0.9) == _lib.VD_E_STATE                                # no encoder forward yet
    nb = small_batch(params, B=3, seed=7)
    eng.encoder_forward(Batch(nb))
    for k, p in bad:
        assert call(eng, k, p) == _lib.VD_E_BADARG, (k, p)
        assert call(eng, k, p, L=0) == _lib.VD_E_BADARG
    assert call(eng, 3, 0.9) == _lib.VD_OK
    W = _W(params, nb)
    for k, p in bad:
        with pytest.raises(_lib.VdError) as e:
            eng.gen_dialog_truncated_sample(Batch(nb), 5, V - 1, V, 1.0, 7, 0, W, MAX_ANS, k, p)
        assert e.value.code == _lib.VD_E_BADARG, (k, p)
    Tq = nb["ques_fwd"].shape[2]

    def open_pool():
        eng.dialog_open(3, Tq, W, MAX_ANS)
        return eng.dialog_join(Batch({x: np.ascontiguousarray(nb[x]) for x in ("ques_fwd", "hist", "img_feat") if x in nb}))

    want = eng.dialog_ask_truncated_slots(open_pool(), nb["ques_fwd"][:, 0], 5, V - 1, V, 1.0, 7, 0, 3, 0.9)
    sl = open_pool()
    rounds = eng.dialog_slots().copy()
    for k, p in bad:
        with pytest.raises(_lib.VdError) as e:
            eng.dialog_ask_truncated_slots(sl, nb["ques_fwd"][:, 0], 5, V - 1, V, 1.0, 7, 0, k, p)
        assert e.value.code == _lib.VD_E_BADARG, (k, p)
        assert np.array_equal(eng.dialog_slots(), rounds)
    got = eng.dialog_ask_truncated_slots(sl, nb["ques_fwd"][:, 0], 5, V - 1, V, 1.0, 7, 0, 3, 0.9)
    for g, w in zip(got, want):
        assert np.array_equal(g, w)
    eng.close()
    # a vocabulary whose row does not fit the shared-memory stage: refused when truncation is active only
    big = 49153
    params, eng = _engine("lf-ques", VD_MATH_FP32, big, 32, 12)
    _forward(eng, params, 1)
    with pytest.raises(_lib.VdError) as e:
        eng.gen_truncated_sample(3, big - 1, 1.0, 7, 0, 5, 1.0)
    assert e.value.code == _lib.VD_E_BADARG
    a, _ = eng.gen_truncated_sample(3, big - 1, 1.0, 7, 0, 0, 1.0)
    assert np.array_equal(a, eng.gen_sample(3, big - 1, 1.0, 7, 0)[0])
    eng.close()


# ---- dialogs and pools (FP32) -------------------------------------------------------------------------------------
@pytest.mark.parametrize("enc", ["lf-ques-hist", "hre-ques-hist", "hrea-ques-im-hist", "mn-att-ques-im-hist"])
def test_fp32_dialogs_append_the_truncated_samples(enc):
    V, L, T, r0, k, p = 256, 8, 0.9, 21, 20, 0.9
    params, eng = _engine(enc, VD_MATH_FP32, V, 128, 64, bias=None)
    nb = small_batch(params, B=4, seed=7)
    B, R = nb["ques_fwd"].shape[:2]
    W = _width(params, nb)
    ans, logp, hist = eng.gen_dialog_truncated_sample(Batch(nb), L, V - 1, V, T, SEED, r0, W, MAX_ANS, k, p)
    a = ans.reshape(B, R, L + 1)
    want = np.zeros_like(hist)
    for b in range(B):
        want[b, 0] = right_aligned(row_words(nb["hist"][b, 0]), W)
        for r in range(R - 1):
            want[b, r + 1] = next_row(want[b, r], row_words(nb["ques_fwd"][b, r]), sample_words(a[b, r], V),
                                      params["concatHistory"], V, W, MAX_ANS)
    assert np.array_equal(hist, want)
    for r in range(R):                                   # round r: the single-call draw on the history it read
        h = hist.copy()
        h[:, r + 1:] = 0
        eng.encoder_forward(Batch(dict(nb, hist=h)))
        ra, rl = eng.gen_truncated_sample(L, V - 1, T, SEED, r0, k, p)
        rows = np.arange(B) * R + r
        assert np.array_equal(ra[rows], ans[rows]) and np.array_equal(rl[rows], logp[rows]), r
    eng.close()


@pytest.mark.parametrize("enc", ["lf-ques-hist", "hrea-ques-im-hist", "mn-att-ques-im-hist"])
def test_fp32_mixed_round_asks_equal_the_dialog_rows(enc):
    V, L, T, r0, k, p = 256, 8, 0.9, 21, 20, 0.9
    params, eng = _engine(enc, VD_MATH_FP32, V, 128, 64)
    D = 6
    nb = small_batch(params, B=D, seed=7)
    R = nb["ques_fwd"].shape[1]
    W = _W(params, nb)
    ans, logp, _ = eng.gen_dialog_truncated_sample(Batch(nb), L, V - 1, V, T, SEED, r0, W, MAX_ANS, k, p)
    got, _ = _drive(eng, nb, 3, W, lambda sl, q: eng.dialog_ask_truncated_slots(sl, q, L, V - 1, V, T, SEED, r0, k, p),
                    seed=3, draw_base=[d * R for d in range(D)])
    for d in range(D):
        for r, (x, lp) in enumerate(got[d]):
            assert np.array_equal(x, ans[d * R + r]) and np.array_equal(lp, logp[d * R + r]), (d, r)
    eng.close()


# ---- commands -----------------------------------------------------------------------------------------------------
from test_dialog_generation_gpu import command_files  # noqa: E402,F401  (the generate command's corpus and checkpoint)


def _cmd(module, *args, stdin=None):
    r = subprocess.run([sys.executable, "-m", module] + [str(a) for a in args], cwd=ROOT, input=stdin, capture_output=True,
                       text=True, timeout=1200)
    assert r.returncode == 0, (r.stdout[-3000:], r.stderr[-3000:])
    return r.stdout


def test_generate_and_chat_commands(command_files, tmp_path):
    flags, fo, ckp = command_files
    common = [*flags, "-loadPath", ckp, "-maxThreads", 4, "-math", "fp32", "-beamLen", 20, "-sampleWords", 1]
    _cmd("visdial_b200.generate", *common, "-resultPath", tmp_path / "plain")
    plain = (tmp_path / "plain" / "results.json").read_bytes()
    _cmd("visdial_b200.generate", *common, "-resultPath", tmp_path / "plain", "-topK", 0, "-topP", 1)
    assert (tmp_path / "plain" / "results.json").read_bytes() == plain and b"topK" not in plain
    # top-k 1 and a tiny top-p both draw every step's argmax, whatever the temperature
    _cmd("visdial_b200.generate", *common, "-resultPath", tmp_path / "k1", "-topK", 1, "-temperature", 0.7)
    _cmd("visdial_b200.generate", *common, "-resultPath", tmp_path / "p0", "-topP", 1e-7, "-temperature", 1.6,
         "-history", "generated")
    k1, p0 = (json.load(open(str(tmp_path / d / "results.json"))) for d in ("k1", "p0"))
    assert k1["opts"]["topK"] == 1 and p0["opts"]["topP"] == 1e-7
    assert k1["data"] != json.loads(plain)["data"]
    _cmd("visdial_b200.generate", *common, "-resultPath", tmp_path / "k1h", "-topK", 1, "-history", "generated")
    assert json.load(open(str(tmp_path / "k1h" / "results.json")))["data"] == p0["data"]
    if torch.cuda.device_count() >= 2:
        _cmd("visdial_b200.generate", *common, "-resultPath", tmp_path / "p1", "-topP", 0.9)
        _cmd("visdial_b200.generate", *common, "-resultPath", tmp_path / "p2", "-topP", 0.9, "-gpus", 2)
        assert (tmp_path / "p1" / "results.json").read_bytes() == (tmp_path / "p2" / "results.json").read_bytes()
    lines = "".join(json.dumps({"id": "u", "image_id": k1["data"][0]["image_id"], "question": q}) + "\n"
                    for q in ([1, 2, 3], [4, 5]))                      # token ids: the corpus's words are synthetic
    out = [json.loads(x) for x in _cmd("visdial_b200.chat", *common, "-serve", 1, "-capacity", 2, "-topP", 0.9,
                                       stdin=lines).splitlines() if x.startswith("{")]
    answers = [o for o in out if "answer" in o]
    assert len(answers) == 2 and all(o["answer"] is not None for o in answers)
