"""n-best lists with length normalisation on the device (vd_gen_nbest_beam_search and its dialog / pool forms, DESIGN §24)
against the host twin (tests/host_nbest.py): the merge kernel alone through vd_test_kernel, whole searches stepped
through vd_gen_decoder_step at the same row count (answers, lengths, fp64 scores and norms bit for bit), the reductions to
the plain and diverse searches, launches, dialogs on the picks, pool asks, refusals and the commands."""
import json

import numpy as np
import pytest

from dialog_history import beam_words, next_row, right_aligned, row_words
from helpers import ISENT, Pool, call, check, small_batch, small_params
from host_nbest import empty_lists, host_nbest_beam_search, lp_table, nbest_merge_step, pick_lists
from test_dialog_generation_gpu import MAX_ANS, _engine, _width
from test_dialog_pool_gpu import _W, _drive
from test_dialog_session_gpu import _AskView
from test_diverse_beam_gpu import F64_GUARD, LAM, MODE_IDS, MODES, SIZES, _cmd, _forward, _tables
from visdial_b200 import VD_MATH_FP32
from visdial_b200 import _lib
from visdial_b200.engine import Batch, Engine

pytestmark = pytest.mark.gpu

ALPHA, NB = 0.7, 5


# ---- the merge kernel alone ---------------------------------------------------------------------------------------
def _ordered(ans, length, score, norm, ord_):
    """a list's slots read in list order (positions past the filled ones: zeros)"""
    N, G, nb, L = ans.shape
    out = [np.zeros_like(ans), np.zeros_like(length), np.zeros_like(score), np.zeros_like(score)]
    for n in range(N):
        for g in range(G):
            m = int((length[n, g] > 0).sum())
            assert (length[n, g, :m] > 0).all()                  # slots fill in order
            for i in range(m):
                s = int(ord_[n, g, i]) if ord_ is not None else i
                out[0][n, g, i], out[1][n, g, i], out[2][n, g, i] = ans[n, g, s], length[n, g, s], score[n, g, s]
                out[3][n, g, i] = norm[n, g, s] if norm is not None else score[n, g, s]
    return out


@pytest.mark.parametrize("k,G", [(6, 1), (6, 2), (8, 2), (32, 1), (32, 32)])
@pytest.mark.parametrize("nb", [1, 2, 5, 32])
def test_merge_kernel_matches_twin_and_plain_merge(k, G, nb):
    """every step of a search on random tables (the first, the middle ones and the last): the lists (through the slot
    order, and at the last step the ordered outputs and the pick) against the twin; beams, scores, tokens and parents
    against the twin and the beam_merge hook"""
    N, L, V = 5, 6, max(12, k + 3)
    eng = Engine(small_params("lf-ques", "gen", vocabSize=V))
    evicted = 0
    for alpha in (0.0, ALPHA, 2.0):
        rng = np.random.default_rng(1000 * k + 10 * G + nb + int(10 * alpha))
        lp = lp_table(alpha, L) if alpha else None
        pool = Pool(eng)
        many, normed = nb > 1, nb > 1 or lp is not None
        st = dict(a=pool(np.zeros((N, G, nb, L), np.int32), ISENT), al=pool(np.zeros((N, G, nb), np.int32), ISENT),
                  asc=pool(np.zeros((N, G, nb)), F64_GUARD),
                  nrm=pool(np.zeros((N, G, nb)), F64_GUARD) if normed else None,
                  ord=pool(np.zeros((N, G, nb), np.int32), ISENT) if many else None,
                  lp=pool(lp, F64_GUARD) if lp is not None else None)
        plain = dict(a=pool(np.zeros((N, G, L), np.int32), ISENT), al=pool(np.zeros((N, G), np.int32), ISENT),
                     asc=pool(np.zeros((N, G)), F64_GUARD))
        beams = np.zeros((N, k, L), np.int32)
        beams[:, :, 0] = V - 1
        scores = np.zeros((N, k))
        lists = empty_lists(N, G, nb, L)
        for stp in range(1, L):
            last = stp == L - 1
            topv, topi = _tables(rng, N, k, V, V, stp)
            want = nbest_merge_step(stp, k, G, LAM, lp, L, V, topv, topi, scores, beams, *lists)
            outs = {}
            for name in ("nbest", "plain"):
                d = dict(tv=pool(topv), ti=pool(topi), si=pool(scores, F64_GUARD), so=pool(np.full((N, k), F64_GUARD), F64_GUARD),
                         bi=pool(beams), bo=pool(beams.copy(), ISENT), tok=pool.out(N * k, np.int32),
                         par=pool.out(N * k, np.int32))
                s = st if name == "nbest" else plain
                picks = [pool.out((N, L), np.int32), pool.out(N, np.int32), pool(np.full(N, F64_GUARD), F64_GUARD)] if last \
                    else [None, None, None]
                ptrs = [d["tv"], d["ti"], d["si"], d["so"], d["bi"], d["bo"], d["tok"], d["par"], s["a"], s["al"], s["asc"]] + picks
                if name == "nbest":
                    o = [pool.out((N, G, nb, L), np.int32), pool.out((N, G, nb), np.int32),
                         pool(np.full((N, G, nb), F64_GUARD), F64_GUARD), pool(np.full((N, G, nb), F64_GUARD), F64_GUARD)] \
                        if many else [None] * 4
                    check(call(eng, "beam_merge_nbest", ptrs + [s["lp"], s["nrm"], s["ord"]] + o, [N, stp, k, G, L, V, nb],
                               [LAM]))
                    d["outs"] = o
                else:
                    check(call(eng, "beam_merge", ptrs, [N, stp, k, G, L, V], [LAM]))
                d["picks"] = picks
                outs[name] = d
            for x, w, nm in zip(("so", "bo", "tok", "par"), want[:4], ("scores", "beams", "tokens", "parent")):
                g1, g2 = outs["nbest"][x].get().reshape(np.shape(w)), outs["plain"][x].get().reshape(np.shape(w))
                assert np.array_equal(g1, w) and np.array_equal(g2, w), (nm, alpha, stp)
            slots = _ordered(st["a"].get(), st["al"].get(), st["asc"].get(), st["nrm"].get() if normed else None,
                             st["ord"].get() if many else None)
            for g_, w, nm in zip(slots, want[4:], ("ans", "len", "score", "norm")):
                assert np.array_equal(g_, w), (nm, alpha, stp)
            if last:
                if many:
                    for g_, w, nm in zip(outs["nbest"]["outs"], want[4:], ("out_ans", "out_len", "out_score", "out_norm")):
                        assert np.array_equal(g_.get(), w), (nm, alpha)
                for g_, w, nm in zip(outs["nbest"]["picks"], pick_lists(*want[4:])[:3], ("pick_ans", "pick_len", "pick_score")):
                    assert np.array_equal(g_.get().reshape(np.shape(w)), w), (nm, alpha)
            evicted += int((want[5] > 0).all(axis=2).sum())
            scores, beams, lists = want[0], want[1], want[4:]
        assert (lists[1] > 0).any()
        pool.free()
    if nb <= 2:
        assert evicted > 0                                      # full lists met more candidates
    eng.close()


# ---- whole searches -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("size", sorted(SIZES))
@pytest.mark.parametrize("mode", MODES, ids=MODE_IDS)
@pytest.mark.parametrize("enc", ["lf-ques", "hrea-ques-im-hist", "mn-att-ques-im-hist", "lf-att-ques-im-hist"])
def test_device_search_matches_host_twin(enc, mode, size):
    s = SIZES[size]
    V, k, G, L = s["V"], s["k"], s["G"], s["L"]
    params, eng = _engine(enc, mode, V, s["H"], s["E"], s["end_bias"])
    encOut = _forward(eng, params, s["D"])
    want = host_nbest_beam_search(eng, encOut, k, G, LAM, ALPHA, NB, L, V - 1, V)
    got = eng.gen_nbest_beam_search(k, G, LAM, ALPHA, NB, L, V - 1, V)
    for g, w, name in zip(got, want, ("answer", "length", "score", "norm")):
        assert g.shape == w.shape and np.array_equal(g, w), name
    assert (want[1][:, :, 1] > 0).any() and not np.array_equal(want[2], want[3])
    eng.close()


@pytest.mark.parametrize("mode", MODES, ids=MODE_IDS)
def test_reductions_to_the_plain_and_diverse_searches(mode):
    s = SIZES["tc"]
    params, eng = _engine("hrea-ques-im-hist", mode, s["V"], s["H"], s["E"], s["end_bias"])
    _forward(eng, params, s["D"])
    V, L = s["V"], s["L"]
    for k in (1, 5, 10):
        a, n, sc = eng.gen_beam_search(k, L, V - 1, V)
        na, nn, ns, nx = eng.gen_nbest_beam_search(k, 1, LAM, 0.0, 1, L, V - 1, V)
        assert np.array_equal(na[:, 0, 0], a) and np.array_equal(nn[:, 0, 0], n) and np.array_equal(ns[:, 0, 0], sc), k
        assert np.array_equal(nx[:, 0, 0], sc)
    da, dn, ds = eng.gen_diverse_beam_search(s["k"], s["G"], LAM, L, V - 1, V)
    na, nn, ns, _ = eng.gen_nbest_beam_search(s["k"], s["G"], LAM, 0.0, 1, L, V - 1, V)
    assert np.array_equal(na[:, :, 0], da) and np.array_equal(nn[:, :, 0], dn) and np.array_equal(ns[:, :, 0], ds)
    eng.close()


def test_launches_per_call_are_the_beam_searchs():
    params, eng = _engine("lf-ques", VD_MATH_FP32, 9, 32, 12, 1.0)
    _forward(eng, params, 2)
    counts = {}
    for name, fn in (("beam", lambda L: eng.gen_beam_search(6, L, 8, 9)),
                     ("nbest", lambda L: eng.gen_nbest_beam_search(6, 3, LAM, ALPHA, NB, L, 8, 9)),
                     ("one", lambda L: eng.gen_nbest_beam_search(6, 1, 0.0, 2.0, 32, L, 8, 9))):
        for L in (2, 7):
            eng.profile_reset()
            fn(L)
            counts[name, L] = eng.launch_count()
    for L in (2, 7):
        assert counts["nbest", L] == counts["beam", L] == counts["one", L], counts
    eng.close()


# ---- dialogs on the picks -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("enc", ["lf-ques-hist", "lf-ques-im-hist", "lf-att-ques-im-hist", "hre-ques-hist", "hrea-ques-im-hist",
                                 "mn-ques-hist", "mn-att-ques-im-hist"])
def test_fp32_dialogs_append_the_picks(enc):
    s = SIZES["small"]
    V, k, G, L = s["V"], s["k"], s["G"], s["L"]
    params, eng = _engine(enc, VD_MATH_FP32, V, s["H"], s["E"], s["end_bias"])
    nb = small_batch(params, B=s["D"], seed=7)
    B, R = nb["ques_fwd"].shape[:2]
    W = _width(params, nb)
    ans, length, score, norm, hist = eng.gen_dialog_nbest_beam_search(Batch(nb), k, G, LAM, ALPHA, 3, L, V - 1, V, W, MAX_ANS)
    assert ans.shape == (B * R, G, 3, L) and length.shape == score.shape == norm.shape == (B * R, G, 3)
    pa, pl, _, _ = pick_lists(ans, length, score, norm)
    want = np.zeros_like(hist)
    for b in range(B):
        want[b, 0] = right_aligned(row_words(nb["hist"][b, 0]), W)
        for r in range(R - 1):
            want[b, r + 1] = next_row(want[b, r], row_words(nb["ques_fwd"][b, r]), beam_words(pa[b * R + r], pl[b * R + r]),
                                      params["concatHistory"], V, W, MAX_ANS)
    assert np.array_equal(hist, want)
    for r in range(R):
        h = hist.copy()
        h[:, r + 1:] = 0                                        # what round r's encoder read
        eng.encoder_forward(Batch(dict(nb, hist=h)))
        got = eng.gen_nbest_beam_search(k, G, LAM, ALPHA, 3, L, V - 1, V)
        rows = np.arange(B) * R + r
        for g, w in zip(got, (ans, length, score, norm)):
            assert np.array_equal(g[rows], w[rows]), r
    assert (length[:, :, 1] > 0).any()
    eng.close()


# ---- pools --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("enc", ["lf-ques-im-hist", "hrea-ques-im-hist", "mn-att-ques-im-hist"])
def test_fp32_mixed_round_asks_equal_the_dialog_rows(enc):
    s = SIZES["small"]
    V, k, G, L = s["V"], s["k"], s["G"], s["L"]
    params, eng = _engine(enc, VD_MATH_FP32, V, s["H"], s["E"], s["end_bias"])
    D = 6
    nb = small_batch(params, B=D, seed=7)
    R = nb["ques_fwd"].shape[1]
    W = _W(params, nb)
    want = eng.gen_dialog_nbest_beam_search(Batch(nb), k, G, LAM, ALPHA, NB, L, V - 1, V, W, MAX_ANS)[:4]
    got, _ = _drive(eng, nb, 3, W, lambda sl, q: eng.dialog_ask_nbest_slots(sl, q, k, G, LAM, ALPHA, NB, L, V - 1, V), seed=5)
    for d in range(D):
        for r, res in enumerate(got[d]):
            for g, w in zip(res, want):
                assert np.array_equal(g, w[d * R + r]), (d, r)
    eng.close()


def test_tensor_core_asks_equal_the_host_twin_from_their_state():
    from visdial_b200 import VD_MATH_F16
    s = SIZES["tc"]
    V, k, G, L = s["V"], s["k"], s["G"], 12
    params, eng = _engine("hrea-ques-im-hist", VD_MATH_F16, V, s["H"], s["E"], s["end_bias"])
    nb = small_batch(params, B=6, seed=7)
    W = _W(params, nb)
    n_asks = [0]

    def ask(sl, q):
        got = eng.dialog_ask_nbest_slots(sl, q, k, G, LAM, ALPHA, NB, L, V - 1, V)
        want = host_nbest_beam_search(_AskView(eng), eng.dialog_encoding().numpy(), k, G, LAM, ALPHA, NB, L, V - 1, V)
        for g, w in zip(got, want):
            assert np.array_equal(g, w)
        n_asks[0] += 1
        return got

    _drive(eng, nb, 3, W, ask, seed=11)
    assert n_asks[0] > 0
    eng.close()


def test_refusals_leave_the_engine_and_the_pool_unchanged():
    V = 9
    a, n, sc, nx = (np.zeros(1 << 16, np.int32), np.zeros(1 << 12, np.int32), np.zeros(1 << 12), np.zeros(1 << 12))

    def search(eng, k, G, alpha, nbest, L=5):
        return eng.lib.vd_gen_nbest_beam_search(eng.h, k, G, LAM, alpha, nbest, L, V - 1, V, a.ctypes.data, n.ctypes.data,
                                                sc.ctypes.data, nx.ctypes.data)

    bad = [(6, 3, ALPHA, 0), (6, 3, ALPHA, 33), (6, 3, ALPHA, -1), (6, 3, -0.5, 2), (6, 3, float("nan"), 2),
           (6, 3, float("inf"), 2), (6, 4, ALPHA, 2), (0, 1, 0.0, 1), (33, 1, 0.0, 1)]
    disc = Engine(small_params("lf-ques", "disc", vocabSize=V))
    assert search(disc, 6, 3, ALPHA, 2) == _lib.VD_E_STATE
    disc.close()
    params, eng = _engine("hrea-ques-im-hist", VD_MATH_FP32, V, 32, 12, 1.0)
    assert search(eng, 6, 3, ALPHA, 2) == _lib.VD_E_STATE                      # no encoder forward yet
    nb = small_batch(params, B=3, seed=7)
    eng.encoder_forward(Batch(nb))
    for k, G, alpha, nbest in bad:
        assert search(eng, k, G, alpha, nbest) == _lib.VD_E_BADARG, (k, G, alpha, nbest)
    assert search(eng, 6, 3, ALPHA, 2) == _lib.VD_OK
    W = _W(params, nb)
    for k, G, alpha, nbest in bad:
        with pytest.raises(_lib.VdError) as e:
            eng.gen_dialog_nbest_beam_search(Batch(nb), k, G, LAM, alpha, nbest, 5, V - 1, V, W, MAX_ANS)
        assert e.value.code == _lib.VD_E_BADARG, (k, G, alpha, nbest)
    Tq = nb["ques_fwd"].shape[2]

    def open_pool():
        eng.dialog_open(3, Tq, W, MAX_ANS)
        return eng.dialog_join(Batch({x: np.ascontiguousarray(nb[x]) for x in ("ques_fwd", "hist", "img_feat") if x in nb}))

    want = eng.dialog_ask_nbest_slots(open_pool(), nb["ques_fwd"][:, 0], 6, 3, LAM, ALPHA, 2, 5, V - 1, V)
    sl = open_pool()
    rounds = eng.dialog_slots().copy()
    for k, G, alpha, nbest in bad:
        with pytest.raises(_lib.VdError) as e:
            eng.dialog_ask_nbest_slots(sl, nb["ques_fwd"][:, 0], k, G, LAM, alpha, nbest, 5, V - 1, V)
        assert e.value.code == _lib.VD_E_BADARG, (k, G, alpha, nbest)
        assert np.array_equal(eng.dialog_slots(), rounds)
    got = eng.dialog_ask_nbest_slots(sl, nb["ques_fwd"][:, 0], 6, 3, LAM, ALPHA, 2, 5, V - 1, V)
    for g, w in zip(got, want):
        assert np.array_equal(g, w)
    eng.close()


# ---- commands -----------------------------------------------------------------------------------------------------
from test_dialog_generation_gpu import command_files  # noqa: E402,F401  (the generate command's corpus and checkpoint)


def test_generate_and_chat_commands(command_files, tmp_path):
    flags, fo, ckp = command_files
    common = [*flags, "-loadPath", ckp, "-maxThreads", 3, "-math", "fp32", "-beamLen", 20]
    _cmd("visdial_b200.generate", *common, "-resultPath", tmp_path / "plain")
    plain = (tmp_path / "plain" / "results.json").read_bytes()
    _cmd("visdial_b200.generate", *common, "-resultPath", tmp_path / "plain", "-nBest", 1, "-lengthPenalty", 0)
    assert (tmp_path / "plain" / "results.json").read_bytes() == plain
    assert b"nBest" not in plain and b"lengthPenalty" not in plain and b'"nbest"' not in plain
    _cmd("visdial_b200.generate", *common, "-resultPath", tmp_path / "nb", "-nBest", 5)
    res = json.load(open(str(tmp_path / "nb" / "results.json")))
    assert res["opts"]["nBest"] == 5
    five = 0
    for d in res["data"]:
        for t in d["dialog"]:
            assert 1 <= len(t["nbest"]) <= 5 and t["nbest"][0] == t["answer"]
            five += len(t["nbest"]) == 5
    assert five > 0
    lines = "".join(json.dumps({"id": "u", "image_id": res["data"][0]["image_id"], "question": q}) + "\n"
                    for q in ([1, 2, 3], [4, 5]))                      # token ids: the corpus's words are synthetic
    out = [json.loads(x) for x in _cmd("visdial_b200.chat", *common, "-serve", 1, "-capacity", 2, "-nBest", 3,
                                       "-lengthPenalty", 0.7, stdin=lines).splitlines() if x.startswith("{")]
    answers = [o for o in out if "answer" in o]
    assert len(answers) == 2
    for o in answers:
        if o["answer"] is not None:
            nbl = o["nbest"]
            assert 1 <= len(nbl) <= 3 and nbl[0]["answer"] == o["answer"] and nbl[0]["score"] == o["score"]
            assert nbl[0]["normScore"] == o["normScore"]
            assert all(a["normScore"] >= b["normScore"] for a, b in zip(nbl, nbl[1:]))
