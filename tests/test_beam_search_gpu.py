"""Model:generateAnswers' beam search on the device (vd_gen_beam_search, model.lua:472-579) against the host reference
(tests/host_decode.py): the decoder stepped through vd_gen_decoder_step with the same kernels at the same row count, the
top k and the candidate merge on the host.  The two walk the same hypotheses, so answers, lengths and fp64 scores must
agree bit for bit."""
import numpy as np
import pytest

from helpers import small_batch, small_params
from host_decode import host_beam_search
from visdial_b200 import VD_MATH_F16, VD_MATH_FP32, VD_MATH_TF32, init_parameters
from visdial_b200 import _lib
from visdial_b200.engine import Batch, Engine, split_parameters

pytestmark = pytest.mark.gpu

# per-step launches of the search in the FP32 math mode (DESIGN §14): 4 state gathers, the embedding, 3 per LSTM layer
# (x-projection, recurrent GEMM, pointwise), the vocabulary projection, the fused log-softmax + top-k and the merge
STEP_LAUNCHES_FP32 = 14


def _engine(enc, mode, V, H, E, end_bias, seed=5):
    params = small_params(enc, "gen", vocabSize=V, rnnHiddenSize=H, embedSize=E)
    eng = Engine(params)
    eng.set_math_mode(mode)
    eng.set_training(0)
    flat = init_parameters(params, seed=seed)
    split_parameters(params, flat)["dec.out.bias"][V - 1] += end_bias      # <END> = class V-1: beams finish at varied steps
    eng.set_parameters(flat)
    return params, eng


def _forward(eng, params, D, seed=7):
    return eng.encoder_forward(Batch(small_batch(params, B=D, seed=seed))).numpy()


SIZES = {"small": dict(V=9, H=32, E=12, D=3, k=3, L=8, end_bias=1.0),
         "tc": dict(V=256, H=128, E=64, D=8, k=5, L=20, end_bias=4.0)}


@pytest.mark.parametrize("size", sorted(SIZES))
@pytest.mark.parametrize("mode", [VD_MATH_FP32, VD_MATH_TF32, VD_MATH_F16], ids=["fp32", "tf32", "f16"])
@pytest.mark.parametrize("enc", ["lf-ques", "hrea-ques-im-hist", "mn-att-ques-im-hist", "lf-att-ques-im-hist"])
def test_device_search_matches_host_search(enc, mode, size):
    s = SIZES[size]
    V, k, L = s["V"], s["k"], s["L"]
    params, eng = _engine(enc, mode, V, s["H"], s["E"], s["end_bias"])
    encOut = _forward(eng, params, s["D"])
    stats = {"stale": 0, "pad_rows": 0, "end_steps": set()}
    want = host_beam_search(eng, encOut, k, L, V - 1, V, stats)
    got = eng.gen_beam_search(k, L, V - 1, V)
    for g, w, name in zip(got, want, ("answer", "length", "score")):
        assert g.shape == w.shape and np.array_equal(g, w), name
    # the quirks were exercised: columns without a candidate, pad tokens fed on, hypotheses finishing at several steps
    assert stats["stale"] > 0 and stats["pad_rows"] > 0 and len(stats["end_steps"]) > 1, stats
    assert (want[1] > 0).any()
    eng.close()


@pytest.mark.parametrize("enc", ["lf-ques", "mn-att-ques-im-hist"])
@pytest.mark.parametrize("k,L", [(1, 8), (9, 6), (3, 2)], ids=["beam1", "beam_eq_V", "len2"])
def test_device_search_edges_match_host_search(enc, k, L):
    params, eng = _engine(enc, VD_MATH_FP32, 9, 32, 12, 1.0)
    encOut = _forward(eng, params, 2)
    want = host_beam_search(eng, encOut, k, L, 8, 9)
    got = eng.gen_beam_search(k, L, 8, 9)
    for g, w, name in zip(got, want, ("answer", "length", "score")):
        assert np.array_equal(g, w), name
    eng.close()


def test_launch_count_is_linear_in_beam_len():
    params, eng = _engine("lf-ques", VD_MATH_FP32, 9, 32, 12, 1.0)
    _forward(eng, params, 2)
    counts = {}
    for L in (2, 7):
        eng.profile_reset()
        eng.gen_beam_search(3, L, 8, 9)
        counts[L] = eng.launch_count()
    assert counts[7] - counts[2] == STEP_LAUNCHES_FP32 * 5, counts
    eng.close()


def test_refusals():
    V = 9
    ans, length, score = np.zeros(4096, np.int32), np.zeros(512, np.int32), np.zeros(512, np.float64)

    def call(eng, k, L):
        return eng.lib.vd_gen_beam_search(eng.h, k, L, V - 1, V, ans.ctypes.data, length.ctypes.data, score.ctypes.data)

    disc = Engine(small_params("lf-ques", "disc", vocabSize=V))
    assert call(disc, 3, 5) == _lib.VD_E_STATE
    disc.close()
    params, eng = _engine("lf-ques", VD_MATH_FP32, V, 32, 12, 0.0)
    assert call(eng, 3, 5) == _lib.VD_E_STATE                                 # no encoder forward yet
    with pytest.raises(_lib.VdError):
        eng.gen_beam_search(3, 5, V - 1, V)
    _forward(eng, params, 2)
    for k, L in ((0, 5), (33, 5), (V + 1, 5), (3, 1)):
        assert call(eng, k, L) == _lib.VD_E_BADARG, (k, L)
    assert call(eng, V, 2) == _lib.VD_OK
    eng.close()


# ---- Model.generateAnswers over the device dataloader ------------------------------------------------------------
def _model_and_loader(enc, n, seed=77):
    from oracle import dataloader_oracle as D
    from visdial_b200.dataloader import Dataloader
    from visdial_b200.model import Model
    from visdial_b200.synthetic import make_corpus
    params = small_params(enc, "gen", vocabSize=9)
    concat = "lf" in enc and "hist" in enc
    raw = make_corpus(params, n, 40, seed=seed, max_ques_len=8, max_ans_len=6, max_cap_len=14,
                      ques_len_cap=5 if concat else None, ans_len_cap=4 if concat else None)
    V = params["vocabSize"]
    orc = D.DataloaderOracle(raw, use_history="hist" in enc, concat_history=concat, use_im="im" in enc, start=V - 1, end=V,
                             img_norm=True, att="att" in enc)
    model = Model(dict(params, batchSize=1), seed=3)
    model.engine.set_math_mode(VD_MATH_FP32)
    flat = init_parameters(params, seed=3)
    model.engine.set_parameters(flat)
    opt = dict(params, useHistory="hist" in enc, concatHistory=concat, useIm="im" in enc, maxHistoryLen=60, imgNorm=1)
    dl = Dataloader(model.engine).initialize(opt, ["val"], {"val": raw})
    return params, flat, orc, model, dl


@pytest.mark.parametrize("enc", ["hrea-ques-im-hist", "mn-att-ques-im-hist"])
def test_batched_call_matches_oracle_per_dialog(enc):
    """Each dialog of a 6-dialog call against oracle.generate_answers on that dialog alone (the rule of
    test_dataloader_gpu.py::test_generate_answers_matches_oracle)."""
    import torch
    from helpers import torch_batch, torch_params
    from oracle import visdial_oracle as O
    params, flat, orc, model, dl = _model_and_loader(enc, 12)
    V = params["vocabSize"]
    got = model.generateAnswers(dl, "val", {"beamSize": 3, "beamLen": 6, "maxThreads": 6, "dialogsPerCall": 6}, strict=False)
    assert len(got) == 6
    P = torch_params(params, flat)
    for conv in range(6):
        with torch.no_grad():
            want = O.generate_answers(O.Ctx(), params, P, torch_batch(orc.get_index_data(np.array([conv]))), V - 1, V,
                                      beam_size=3, beam_len=6, strict=False)
        assert len(got[conv]["dialog"]) == len(want) == 10
        for g, w in zip(got[conv]["dialog"], want):
            assert (g is None) == (w is None)
            if g is not None:
                assert g["length"] == w["length"] and abs(g["score"] - w["score"]) < 1e-4
                # a winner that passed through a stale beam column took a top-k over an all-zero row: which of the tied
                # tokens it picked is implementation-defined (torch.topk vs the pinned tie rule)
                if 0 not in w["answer"][1:w["length"]].tolist():
                    assert g["answer"] == w["answer"].tolist()
    dl.close(); model.engine.close()


def test_dialogs_per_call_gives_the_per_dialog_entries():
    params, flat, orc, model, dl = _model_and_loader("hrea-ques-im-hist", 12)
    p = {"beamSize": 4, "beamLen": 8, "maxThreads": 12}
    one = model.generateAnswers(dl, "val", dict(p, dialogsPerCall=1), strict=False)
    five = model.generateAnswers(dl, "val", dict(p, dialogsPerCall=5), strict=False)      # batches of 5, 5 and 2
    assert len(one) == len(five) == 12
    found = 0
    for a, b in zip(one, five):
        assert a["image_id"] == b["image_id"] and len(a["dialog"]) == len(b["dialog"])
        for x, y in zip(a["dialog"], b["dialog"]):
            assert (x is None) == (y is None)
            if x is None:
                continue
            found += 1
            assert x["question"] == y["question"] and x["answer"] == y["answer"] and x["length"] == y["length"]
            assert abs(x["score"] - y["score"]) < 1e-5
    assert found > 0
    dl.close(); model.engine.close()
