"""Dialogs generated on the model's own answers (vd_gen_dialog_beam_search / vd_gen_dialog_sample, DESIGN §17) against a
host loop: for each round r, the batch rebuilt with the host history rule (tests/dialog_history.py) at width W, the encoder
forward through vd_encoder_forward, and tests/host_decode.py's search on round r's rows only.  The host side runs the same
kernels at the same row counts, so answers, lengths and fp64 scores must agree bit for bit, and the history rows the
device fed its encoder must be the host rule's."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from dialog_history import beam_words, next_row, right_aligned, row_words, sample_words
from helpers import small_batch, small_params
from host_decode import HostStep, host_beam_search, start_state
from sampling_twin import draw
from visdial_b200 import VD_MATH_F16, VD_MATH_FP32, VD_MATH_TF32, init_parameters
from visdial_b200 import _lib
from visdial_b200.engine import Batch, Engine, split_parameters

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENCODERS = ["lf-ques-hist", "hre-ques-im-hist", "hrea-ques-im-hist", "mn-ques-hist", "mn-att-ques-im-hist"]
MODES = [VD_MATH_FP32, VD_MATH_TF32, VD_MATH_F16]
MODE_IDS = ["fp32", "tf32", "f16"]
SIZES = {"small": dict(V=9, H=32, E=12, D=3, k=3, L=8, end_bias=1.0),
         "tc": dict(V=256, H=128, E=64, D=8, k=5, L=12, end_bias=4.0)}
MAX_ANS = 5                      # small_batch's answer width
SEED = (3 << 32) | 77
NEAR_TIE = 1e-5


def _engine(enc, mode, V, H, E, end_bias, dec="gen", seed=5):
    params = small_params(enc, dec, vocabSize=V, rnnHiddenSize=H, embedSize=E)
    eng = Engine(params)
    eng.set_math_mode(mode)
    eng.set_training(0)
    flat = init_parameters(params, seed=seed)
    if dec == "gen":
        split_parameters(params, flat)["dec.out.bias"][V - 1] += end_bias      # <END> = class V-1: varied lengths
    eng.set_parameters(flat)
    return params, eng


def _width(params, nb):
    """W: the concatenated history's batch width, or question + answer width for per-round history"""
    return 30 if params["concatHistory"] else nb["ques_fwd"].shape[2] + MAX_ANS


class _RoundView:
    """The engine as tests/host_decode.py sees it for round r: forwardConnect's start state of rows b*R + r only."""

    class _Rows:
        def __init__(self, a):
            self.a = a

        def numpy(self):
            return self.a

    def __init__(self, eng, r):
        self.eng, self.r, self.R = eng, r, eng.params["maxQuesCount"]

    def __getattr__(self, name):
        return getattr(self.eng, name)

    def encoder_rnn_state(self, level, rows):
        h, c = self.eng.encoder_rnn_state(level, rows * self.R)
        if h is None:
            return None, None
        return self._Rows(h.numpy()[self.r::self.R]), self._Rows(c.numpy()[self.r::self.R])


def _host_rounds(eng, params, nb, W, mal, search, answer_words):
    """The dialog loop on the host.  search(view, encOut of round r's rows, r) -> that round's outputs (B rows each);
    answer_words(outputs, b) -> the words written into the history.  Returns (outputs stacked to (B*R, ...), history)."""
    B, R = nb["ques_fwd"].shape[:2]
    end = params["vocabSize"]
    hist = np.zeros((B, R, W), np.int32)
    for b in range(B):
        hist[b, 0] = right_aligned(row_words(nb["hist"][b, 0]), W)
    outs = []
    for r in range(R):
        encOut = eng.encoder_forward(Batch(dict(nb, hist=hist.copy()))).numpy()
        out = search(_RoundView(eng, r), encOut[r::R], r)
        outs.append(out)
        if r + 1 < R:
            for b in range(B):
                hist[b, r + 1] = next_row(hist[b, r], row_words(nb["ques_fwd"][b, r]), answer_words(out, b),
                                          params["concatHistory"], end, W, mal)
    stacked = [np.stack([o[i] for o in outs], 1).reshape((B * R,) + outs[0][i].shape[1:]) for i in range(len(outs[0]))]
    return stacked, hist


def host_dialog_beam(eng, params, nb, k, L, W, mal):
    V = params["vocabSize"]
    return _host_rounds(eng, params, nb, W, mal, lambda view, enc, r: host_beam_search(view, enc, k, L, V - 1, V),
                        lambda out, b: beam_words(out[0][b], out[1][b]))


def _compare_beam(eng, params, nb, k, L, W, mal=MAX_ANS):
    V = params["vocabSize"]
    got = eng.gen_dialog_beam_search(Batch(nb), k, L, V - 1, V, W, mal)
    (ans, length, score), hist = host_dialog_beam(eng, params, nb, k, L, W, mal)
    for g, w, name in zip(got, (ans, length, score, hist), ("answer", "length", "score", "history")):
        assert g.shape == w.shape and np.array_equal(g, w), name
    return got


@pytest.mark.parametrize("size", sorted(SIZES))
@pytest.mark.parametrize("mode", MODES, ids=MODE_IDS)
@pytest.mark.parametrize("enc", ENCODERS)
def test_device_loop_matches_host_loop(enc, mode, size):
    s = SIZES[size]
    params, eng = _engine(enc, mode, s["V"], s["H"], s["E"], s["end_bias"])
    nb = small_batch(params, B=s["D"], seed=7)
    ans, length, score, hist = _compare_beam(eng, params, nb, s["k"], s["L"], _width(params, nb))
    assert (length > 0).any()
    # generated answers did reach the history: it is not the dataset's
    assert not np.array_equal(hist[:, 1:, -nb["hist"].shape[2]:], nb["hist"][:, 1:])
    eng.close()


@pytest.mark.parametrize("k,L", [(1, 8), (2, 2)], ids=["beam1", "len2"])
def test_edges_match_host_loop(k, L):
    params, eng = _engine("hrea-ques-im-hist", VD_MATH_FP32, 9, 32, 12, 0.0)
    nb = small_batch(params, B=3, seed=7)
    nb["ques_fwd"][1, 3] = 0                                  # a question of pads mid-dialog
    ans, length, score, hist = _compare_beam(eng, params, nb, k, L, _width(params, nb))
    assert not hist[1, 4:].any()                              # no Q, no A, and rightAlign's break
    if L == 2:                                                # rounds where no beam finished fed an empty answer back
        assert (length == 0).any()
    eng.close()


def test_concat_edges_and_answer_cut():
    params, eng = _engine("lf-ques-hist", VD_MATH_FP32, 9, 32, 12, 1.0)
    nb = small_batch(params, B=3, seed=7)
    nb["ques_fwd"][1, 3] = 0
    nb["hist"] = np.ascontiguousarray(nb["hist"][:, :, -18:])                        # a batch cut to Th = W = 18
    ans, length, score, hist = _compare_beam(eng, params, nb, 3, 10, 18, mal=2)   # rows overflow W
    assert hist[1, 4, -1] == 9 and (length > 0).any() and (np.count_nonzero(hist, -1) == 18).any()
    eng.close()


@pytest.mark.parametrize("mode", [VD_MATH_FP32, VD_MATH_F16], ids=["fp32", "f16"])
@pytest.mark.parametrize("enc", ["lf-ques-hist", "hrea-ques-im-hist", "mn-att-ques-im-hist"])
def test_sampling_matches_host_loop(enc, mode):
    """The device's samples replayed round by round: each round's history rebuilt from the device's earlier answers must
    be what the device fed its encoder, and each draw the twin's at the round's global index."""
    V, L, T, r0 = 256, 8, 0.9, 21
    params, eng = _engine(enc, mode, V, 128, 64, 2.0)
    nb = small_batch(params, B=4, seed=7)
    B, R = nb["ques_fwd"].shape[:2]
    W = _width(params, nb)
    ans, logp, hist = eng.gen_dialog_sample(Batch(nb), L, V - 1, V, T, SEED, r0, W, MAX_ANS)
    assert ans.shape == (B * R, L + 1) and (ans[:, 0] == V - 1).all()
    a = ans.reshape(B, R, L + 1)
    tol = 1e-5 if mode == VD_MATH_FP32 else 1e-4
    excluded = 0

    def replay(view, encOut, r):
        nonlocal excluded
        h, c = start_state(view, encOut)
        with HostStep(view, B) as step:
            for t in range(1, L + 1):
                lp, h, c = step(a[:, r, t - 1], h, c)
                lp = lp.astype(np.float64)
                np.testing.assert_allclose(logp.reshape(B, R, L)[:, r, t - 1], lp[np.arange(B), a[:, r, t] - 1],
                                           rtol=0, atol=tol)
                for b in range(B):                            # global round (r0 + b R + r)
                    want, gap = draw(lp[b:b + 1], T, SEED, t, r0 + b * R + r)
                    if gap[0] >= NEAR_TIE:
                        assert a[b, r, t] == want[0], (b, r, t)
                    else:
                        excluded += 1
        return (a[:, r],)

    _, want_hist = _host_rounds(eng, params, nb, W, MAX_ANS, replay, lambda out, b: sample_words(out[0][b], V))
    assert np.array_equal(hist, want_hist)
    assert excluded <= B * R * L // 100, excluded
    eng.close()


def test_refusals():
    V = 9
    ans, length, score = np.zeros(4096, np.int32), np.zeros(512, np.int32), np.zeros(512, np.float64)

    def call(eng, nb, W, mal=MAX_ANS):
        return eng.lib.vd_gen_dialog_beam_search(eng.h, Batch(nb).c, 3, 5, V - 1, V, W, mal, ans.ctypes.data,
                                                 length.ctypes.data, score.ctypes.data, None)

    disc_params, disc = _engine("hrea-ques-im-hist", VD_MATH_FP32, V, 32, 12, 0.0, dec="disc")
    nb = small_batch(disc_params, B=2)
    assert call(disc, nb, _width(disc_params, nb)) == _lib.VD_E_STATE
    disc.close()
    params, eng = _engine("lf-ques", VD_MATH_FP32, V, 32, 12, 0.0)
    nb = dict(small_batch(params, B=2), hist=np.ones((2, 10, 4), np.int32))
    assert call(eng, nb, 8) == _lib.VD_E_STATE
    with pytest.raises(_lib.VdError):
        eng.gen_dialog_sample(Batch(nb), 5, V - 1, V, 1.0, 1, 0, 8, MAX_ANS)
    eng.close()
    params, eng = _engine("hrea-ques-im-hist", VD_MATH_FP32, V, 32, 12, 0.0)
    nb = small_batch(params, B=2)
    Th = nb["hist"].shape[2]
    assert call(eng, nb, Th - 1) == _lib.VD_E_BADARG
    assert call(eng, nb, Th, mal=0) == _lib.VD_E_BADARG
    assert call(eng, nb, Th) == _lib.VD_OK
    eng.close()


def test_launch_count_is_linear_in_beam_len_and_independent_of_batch():
    params, eng = _engine("hrea-ques-im-hist", VD_MATH_FP32, 9, 32, 12, 1.0)
    counts = {}
    for B in (1, 8):
        nb = small_batch(params, B=B, seed=7)
        nb = dict(nb, ques_fwd=nb["ques_fwd"][:, :, -6:], hist=np.pad(nb["hist"], ((0, 0), (0, 0), (9 - nb["hist"].shape[2], 0))))
        for L in (2, 7):
            eng.profile_reset()
            eng.gen_dialog_beam_search(Batch(nb), 3, L, 8, 9, 11, MAX_ANS)
            counts[(B, L)] = eng.launch_count()
    R, STEP_LAUNCHES_FP32 = 10, 14                            # test_beam_search_gpu.py's per-step count
    assert counts[(1, 7)] - counts[(1, 2)] == R * 5 * STEP_LAUNCHES_FP32, counts
    assert counts[(1, 2)] == counts[(8, 2)] and counts[(1, 7)] == counts[(8, 7)], counts
    eng.close()


# ---- Model.generateAnswers and the generate command ---------------------------------------------------------------
def _model_and_loader(enc, n, seed=77):
    from visdial_b200.dataloader import Dataloader
    from visdial_b200.model import Model
    from visdial_b200.synthetic import make_corpus
    params = small_params(enc, "gen", vocabSize=9)
    concat = "lf" in enc
    raw = make_corpus(params, n, 40, seed=seed, max_ques_len=8, max_ans_len=6, max_cap_len=14,
                      ques_len_cap=5 if concat else None, ans_len_cap=4 if concat else None)
    model = Model(dict(params, batchSize=1), seed=3)
    model.engine.set_math_mode(VD_MATH_FP32)
    model.engine.set_parameters(init_parameters(params, seed=3))
    opt = dict(params, useHistory=True, concatHistory=concat, useIm="im" in enc, maxHistoryLen=60, imgNorm=1)
    return model, Dataloader(model.engine).initialize(opt, ["val"], {"val": raw})


@pytest.mark.parametrize("sample", [0, 1], ids=["beam", "sample"])
@pytest.mark.parametrize("enc", ["hrea-ques-im-hist", "lf-ques-im-hist"])
def test_dialogs_per_call_gives_the_same_entries(enc, sample):
    model, dl = _model_and_loader(enc, 12)
    p = {"beamSize": 4, "beamLen": 8, "maxThreads": 12, "history": "generated", "sampleWords": sample, "temperature": 0.8}
    one = model.generateAnswers(dl, "val", dict(p, dialogsPerCall=1), strict=False)
    eight = model.generateAnswers(dl, "val", dict(p, dialogsPerCall=8), strict=False)   # calls of 8 and 4 dialogs
    gt = model.generateAnswers(dl, "val", dict(p, dialogsPerCall=1, history="gt"), strict=False)
    assert len(one) == len(eight) == 12
    for a, b in zip(one, eight):
        assert a["image_id"] == b["image_id"]
        for x, y in zip(a["dialog"], b["dialog"]):
            assert (x is None) == (y is None)
            if x is not None:
                assert x["question"] == y["question"] and x["answer"] == y["answer"]
                if not sample:
                    assert x["length"] == y["length"] and abs(x["score"] - y["score"]) < 1e-5
    # round 0 reads only the caption: the same answer on either history
    first = [(a["dialog"][0] or {}).get("answer") for a in one]
    assert first == [(a["dialog"][0] or {}).get("answer") for a in gt]
    with pytest.raises(ValueError):
        model.generateAnswers(dl, "val", dict(p, history="model"))
    dl.close(); model.engine.close()


def _run(*args):
    r = subprocess.run([sys.executable, "-m", "visdial_b200.generate"] + [str(a) for a in args], cwd=ROOT,
                       capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, (r.stdout[-3000:], r.stderr[-3000:])


@pytest.fixture(scope="module")
def command_files(tmp_path_factory):
    from test_cli_gpu import _params, write_files
    from visdial_b200.model import Model
    d = tmp_path_factory.mktemp("dialog_cli")
    flags, fo = write_files(str(d), "hrea-ques-im-hist", "gen")
    p = _params("hrea-ques-im-hist", "gen")
    m = Model(p, seed=1234)
    w = init_parameters(p, seed=5)
    split_parameters(p, w)["dec.out.bias"][p["vocabSize"] - 1] += 3.0     # every round's beam reaches <END> (strict)
    m.engine.set_parameters(w)
    ckp = str(d / "model.t7")
    m.save(ckp, final=True)
    m.engine.close()
    return flags, fo, ckp


@pytest.mark.parametrize("sample", [0, 1], ids=["beam", "sample"])
def test_generate_command_with_generated_history(command_files, tmp_path, sample):
    from test_cli_gpu import _model, _texts
    from visdial_b200.checkpoint import load_checkpoint
    flags, fo, ckp = command_files
    _run(*flags, "-loadPath", ckp, "-resultPath", tmp_path / "vis", "-maxThreads", 6, "-sampleWords", sample,
         "-temperature", 0.7, "-beamLen", 20, "-math", "fp32", "-history", "generated", "-dialogsPerCall", 3)
    res = json.load(open(str(tmp_path / "vis" / "results.json")))
    assert res["opts"]["history"] == "generated"
    ck = load_checkpoint(ckp)
    m, dl = _model(ck["modelParams"], fo, "val", ck)
    answers = m.generateAnswers(dl, "val", {"maxThreads": 6, "sampleWords": sample, "temperature": 0.7, "beamSize": 5,
                                            "beamLen": 20, "history": "generated", "dialogsPerCall": 3})
    want = _texts(answers, dl.ind2word)
    dl.close(); m.engine.close()
    assert res["data"] == want and len(want) == 6 and all(len(a["dialog"]) == 10 for a in want)


def test_generate_command_two_gpus_writes_the_one_gpu_file(command_files, tmp_path):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    flags, fo, ckp = command_files
    for sample in (0, 1):
        outs = []
        for n in (1, 2):
            res = tmp_path / ("gen%d_%d" % (sample, n))
            _run(*flags, "-loadPath", ckp, "-resultPath", res, "-maxThreads", 5, "-sampleWords", sample, "-math", "fp32",
                 "-history", "generated", "-gpus", n)
            outs.append((res / "results.json").read_bytes())
        assert outs[0] == outs[1], sample
