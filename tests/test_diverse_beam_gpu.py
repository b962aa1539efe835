"""Diverse beam search on the device (vd_gen_diverse_beam_search and its dialog / pool forms, DESIGN §22) against the host
twin (tests/host_diverse.py): the merge kernel alone through vd_test_kernel, whole searches stepped through
vd_gen_decoder_step at the same row count (answers, lengths and fp64 scores bit for bit), the G = 1 and no-penalty
invariants, dialogs on the picks, pool asks, launches, refusals and the commands."""
import json
import subprocess
import sys

import numpy as np
import pytest

from dialog_history import beam_words, next_row, right_aligned, row_words
from helpers import ISENT, Pool, call, check, small_batch, small_params
from host_diverse import host_diverse_beam_search, merge_step, pick_answers
from test_dialog_generation_gpu import MAX_ANS, ROOT, _engine, _width
from test_dialog_pool_gpu import _W, _drive
from test_dialog_session_gpu import _AskView
from visdial_b200 import VD_MATH_F16, VD_MATH_FP32, VD_MATH_TF32
from visdial_b200 import _lib
from visdial_b200.engine import Batch, Engine

pytestmark = pytest.mark.gpu

MODES = [VD_MATH_FP32, VD_MATH_TF32, VD_MATH_F16]
MODE_IDS = ["fp32", "tf32", "f16"]
# test_beam_search_gpu.py's two sizes, with a beam that splits into groups
SIZES = {"small": dict(V=9, H=32, E=12, D=3, k=6, G=3, L=8, end_bias=1.0),
         "tc": dict(V=256, H=128, E=64, D=8, k=10, G=5, L=20, end_bias=4.0)}
LAM = 0.5
F64_GUARD = -7.25                # float64 buffers: a guard value no kernel writes


# ---- the merge kernel alone ---------------------------------------------------------------------------------------
def _tables(rng, N, k, V, end, stp):
    """top-k tables as the decoder's are (value desc, class asc) with values on a coarse grid (ties in the augmented and
    fp64 scores across columns and groups), <END> likely in the explored sets, and pad rows (all zero)"""
    x = np.round(rng.normal(0.0, 1.0, (N * k, V)), 1).astype(np.float32)
    x[:, end - 1] += 1.2
    logp = (x - np.log(np.exp(x.astype(np.float64)).sum(1, keepdims=True))).astype(np.float32)
    logp[rng.random(N * k) < 0.15] = 0.0
    top = np.argsort(-logp, axis=1, kind="stable")[:, :k]
    return np.take_along_axis(logp, top, 1), top.astype(np.int32)


def _merge_case(rng, N, k, G, L, stp, V):
    topv, topi = _tables(rng, N, k, V, V, stp)
    beams = np.zeros((N, k, L), np.int32)
    beams[:, :, 0] = V - 1
    beams[:, :, 1:stp] = rng.integers(0, V - 1, (N, k, stp - 1))
    beams[:, :, stp + 1:] = rng.integers(1, V, (N, k, L - stp - 1))      # never read: carried over unchanged
    scores = np.round(rng.normal(-2.0, 0.5, (N, k)), 1)
    scores[:, 1::2] = scores[:, ::2][:, :scores[:, 1::2].shape[1]]            # equal column scores
    ans = np.zeros((N, G, L), np.int32)
    ans_len = np.where(rng.random((N, G)) < 0.3, 2, 0).astype(np.int32)
    ans_score = np.where(ans_len > 0, -2.5, 0.0)
    ans[:, :, 0] = np.where(ans_len > 0, V - 1, 0)
    ans[:, :, 1] = np.where(ans_len > 0, V, 0)
    return topv, topi, scores, beams, ans, ans_len, ans_score


@pytest.mark.parametrize("k,G", [(6, 1), (6, 2), (6, 6), (8, 2), (32, 2), (32, 32)])
@pytest.mark.parametrize("stp", [1, 3, 5], ids=["step1", "step3", "last"])
def test_merge_kernel_matches_step_function(k, G, stp):
    N, L, V = 7, 6, max(12, k + 3)
    rng = np.random.default_rng(1000 * k + 10 * G + stp)
    eng = Engine(small_params("lf-ques", "gen", vocabSize=V))
    pool = Pool(eng)
    stale = ends = 0
    for lam in (0.0, LAM, 3.0):
        topv, topi, scores, beams, ans, ans_len, ans_score = _merge_case(rng, N, k, G, L, stp, V)
        last = stp == L - 1
        want = merge_step(stp, k, G, lam, L, V, topv, topi, scores, beams, ans, ans_len, ans_score, pick=last)
        d = dict(tv=pool(topv), ti=pool(topi), si=pool(scores, F64_GUARD), so=pool(np.full((N, k), F64_GUARD), F64_GUARD),
                 bi=pool(beams), bo=pool(beams.copy(), ISENT), tok=pool.out(N * k, np.int32), par=pool.out(N * k, np.int32),
                 a=pool(ans, ISENT), al=pool(ans_len, ISENT), asc=pool(ans_score, F64_GUARD))
        picks = [pool.out((N, L), np.int32), pool.out(N, np.int32), pool(np.full(N, F64_GUARD), F64_GUARD)] if last else \
            [None, None, None]
        check(call(eng, "beam_merge", [d["tv"], d["ti"], d["si"], d["so"], d["bi"], d["bo"], d["tok"], d["par"], d["a"],
                                       d["al"], d["asc"]] + picks, [N, stp, k, G, L, V], [lam]))
        got = [d[x].get() for x in ("so", "bo", "tok", "par", "a", "al", "asc")] + [p.get() for p in picks if p is not None]
        names = ("scores", "beams", "tokens", "parent", "ans", "ans_len", "ans_score", "pick_ans", "pick_len", "pick_score")
        assert len(got) == len(want)
        for g, w, name in zip(got, want, names):
            assert np.array_equal(g.reshape(np.shape(w)), w), (name, lam)
        stale += int((want[3] < 0).sum())
        ends += int((want[5] != ans_len).sum())
        pool.free()
    assert ends > 0                                         # finished <END> candidates were met
    if stp == 1 or G == k:                                  # so were columns left unfilled (one explored column, or w = 1)
        assert stale > 0
    eng.close()


# ---- whole searches -----------------------------------------------------------------------------------------------
def _forward(eng, params, D, seed=7):
    return eng.encoder_forward(Batch(small_batch(params, B=D, seed=seed))).numpy()


@pytest.mark.parametrize("size", sorted(SIZES))
@pytest.mark.parametrize("mode", MODES, ids=MODE_IDS)
@pytest.mark.parametrize("enc", ["lf-ques", "hrea-ques-im-hist", "mn-att-ques-im-hist", "lf-att-ques-im-hist"])
def test_device_search_matches_host_twin(enc, mode, size):
    s = SIZES[size]
    V, k, G, L = s["V"], s["k"], s["G"], s["L"]
    params, eng = _engine(enc, mode, V, s["H"], s["E"], s["end_bias"])
    encOut = _forward(eng, params, s["D"])
    stats = {"stale": 0, "pad_rows": 0, "end_steps": set()}
    want = host_diverse_beam_search(eng, encOut, k, G, LAM, L, V - 1, V, stats)
    got = eng.gen_diverse_beam_search(k, G, LAM, L, V - 1, V)
    for g, w, name in zip(got, want, ("answer", "length", "score")):
        assert g.shape == w.shape and np.array_equal(g, w), name
    assert stats["stale"] > 0 and stats["pad_rows"] > 0 and len(stats["end_steps"]) > 1, stats
    assert (want[1] > 0).any()
    plain = eng.gen_diverse_beam_search(k, G, 0.0, L, V - 1, V)
    assert not np.array_equal(plain[0], got[0])                 # the penalty changed some group's answer
    eng.close()


@pytest.mark.parametrize("mode", MODES, ids=MODE_IDS)
def test_one_group_is_the_beam_search(mode):
    s = SIZES["tc"]
    params, eng = _engine("hrea-ques-im-hist", mode, s["V"], s["H"], s["E"], s["end_bias"])
    _forward(eng, params, s["D"])
    V = s["V"]
    for k in (1, 5, 10):
        a, n, sc = eng.gen_beam_search(k, s["L"], V - 1, V)
        ga, gn, gs = eng.gen_diverse_beam_search(k, 1, LAM, s["L"], V - 1, V)
        assert np.array_equal(ga[:, 0], a) and np.array_equal(gn[:, 0], n) and np.array_equal(gs[:, 0], sc), k
    eng.close()


@pytest.mark.parametrize("size", sorted(SIZES))
def test_fp32_no_penalty_makes_every_group_a_width_w_search(size):
    s = SIZES[size]
    V, k, G, L = s["V"], s["k"], s["G"], s["L"]
    params, eng = _engine("mn-att-ques-im-hist", VD_MATH_FP32, V, s["H"], s["E"], s["end_bias"])
    _forward(eng, params, s["D"])
    a, n, sc = eng.gen_beam_search(k // G, L, V - 1, V)
    ga, gn, gs = eng.gen_diverse_beam_search(k, G, 0.0, L, V - 1, V)
    for g in range(G):
        assert np.array_equal(ga[:, g], a) and np.array_equal(gn[:, g], n) and np.array_equal(gs[:, g], sc), g
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
    ans, length, score, hist = eng.gen_dialog_diverse_beam_search(Batch(nb), k, G, LAM, L, V - 1, V, W, MAX_ANS)
    assert ans.shape == (B * R, G, L) and length.shape == score.shape == (B * R, G)
    pa, pl, _ = pick_answers(ans, length, score)
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
        ra, rn, rs = eng.gen_diverse_beam_search(k, G, LAM, L, V - 1, V)
        rows = np.arange(B) * R + r
        assert np.array_equal(ra[rows], ans[rows]) and np.array_equal(rn[rows], length[rows]) and \
            np.array_equal(rs[rows], score[rows]), r
    assert (length > 0).any()
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
    ans, length, score, _ = eng.gen_dialog_diverse_beam_search(Batch(nb), k, G, LAM, L, V - 1, V, W, MAX_ANS)
    got, _ = _drive(eng, nb, 3, W, lambda sl, q: eng.dialog_ask_diverse_slots(sl, q, k, G, LAM, L, V - 1, V), seed=5)
    for d in range(D):
        for r, (a, n, sc) in enumerate(got[d]):
            i = d * R + r
            assert np.array_equal(a, ans[i]) and np.array_equal(n, length[i]) and np.array_equal(sc, score[i]), (d, r)
    one, _ = _drive(eng, nb, 3, W, lambda sl, q: eng.dialog_ask_diverse_slots(sl, q, k, 1, LAM, L, V - 1, V), seed=5)
    beam, _ = _drive(eng, nb, 3, W, lambda sl, q: eng.dialog_ask_beam_slots(sl, q, k, L, V - 1, V), seed=5)
    for d in range(D):
        assert len(one[d]) == len(beam[d])
        for (a, n, sc), (ba, bn, bs) in zip(one[d], beam[d]):
            assert np.array_equal(a[0], ba) and n[0] == bn and sc[0] == bs, d
    eng.close()


@pytest.mark.parametrize("mode", [VD_MATH_TF32, VD_MATH_F16], ids=["tf32", "f16"])
def test_tensor_core_asks_equal_the_host_twin_from_their_state(mode):
    s = SIZES["tc"]
    V, k, G, L = s["V"], s["k"], s["G"], 12
    params, eng = _engine("hrea-ques-im-hist", mode, V, s["H"], s["E"], s["end_bias"])
    nb = small_batch(params, B=6, seed=7)
    W = _W(params, nb)
    n_asks = [0]

    def ask(sl, q):
        a, n, sc = eng.dialog_ask_diverse_slots(sl, q, k, G, LAM, L, V - 1, V)
        wa, wn, ws = host_diverse_beam_search(_AskView(eng), eng.dialog_encoding().numpy(), k, G, LAM, L, V - 1, V)
        assert np.array_equal(a, wa) and np.array_equal(n, wn) and np.array_equal(sc, ws)
        n_asks[0] += 1
        return a, n, sc

    _drive(eng, nb, 3, W, ask, seed=11)
    assert n_asks[0] > 0
    eng.close()


# ---- launches and refusals ----------------------------------------------------------------------------------------
def test_launches_per_step_are_the_beam_searchs():
    params, eng = _engine("lf-ques", VD_MATH_FP32, 9, 32, 12, 1.0)
    _forward(eng, params, 2)
    counts = {}
    for name, fn in (("beam", lambda L: eng.gen_beam_search(6, L, 8, 9)),
                     ("diverse", lambda L: eng.gen_diverse_beam_search(6, 3, LAM, L, 8, 9))):
        for L in (2, 7):
            eng.profile_reset()
            fn(L)
            counts[name, L] = eng.launch_count()
    assert counts["diverse", 7] - counts["diverse", 2] == counts["beam", 7] - counts["beam", 2], counts
    assert 0 <= counts["diverse", 2] - counts["beam", 2] <= 1, counts
    eng.close()


def test_refusals_leave_the_engine_usable():
    V = 9
    a, n, sc = np.zeros(1 << 14, np.int32), np.zeros(1 << 10, np.int32), np.zeros(1 << 10, np.float64)

    def search(eng, k, G, lam, L=5):
        return eng.lib.vd_gen_diverse_beam_search(eng.h, k, G, lam, L, V - 1, V, a.ctypes.data, n.ctypes.data, sc.ctypes.data)

    bad = [(6, 0, LAM), (6, -1, LAM), (6, 4, LAM), (6, 3, -0.5), (6, 3, float("nan")), (6, 3, float("inf")), (0, 1, 0.0),
           (33, 1, 0.0), (V + 1, 1, 0.0)]
    disc = Engine(small_params("lf-ques", "disc", vocabSize=V))
    assert search(disc, 6, 3, LAM) == _lib.VD_E_STATE
    disc.close()
    params, eng = _engine("hrea-ques-im-hist", VD_MATH_FP32, V, 32, 12, 1.0)
    assert search(eng, 6, 3, LAM) == _lib.VD_E_STATE                           # no encoder forward yet
    nb = small_batch(params, B=3, seed=7)
    eng.encoder_forward(Batch(nb))
    for k, G, lam in bad:
        assert search(eng, k, G, lam) == _lib.VD_E_BADARG, (k, G, lam)
        assert search(eng, k, G, lam, L=1) == _lib.VD_E_BADARG
    assert search(eng, 6, 3, LAM) == _lib.VD_OK
    W = _W(params, nb)
    for k, G, lam in bad:
        with pytest.raises(_lib.VdError) as e:
            eng.gen_dialog_diverse_beam_search(Batch(nb), k, G, lam, 5, V - 1, V, W, MAX_ANS)
        assert e.value.code == _lib.VD_E_BADARG, (k, G, lam)
    # a pool: a refused ask changes no slot's round, and the next ask answers as in a pool that never saw it
    Tq = nb["ques_fwd"].shape[2]

    def open_pool():
        eng.dialog_open(3, Tq, W, MAX_ANS)
        return eng.dialog_join(Batch({x: np.ascontiguousarray(nb[x]) for x in ("ques_fwd", "hist", "img_feat") if x in nb}))

    want = eng.dialog_ask_diverse_slots(open_pool(), nb["ques_fwd"][:, 0], 6, 3, LAM, 5, V - 1, V)
    sl = open_pool()
    rounds = eng.dialog_slots().copy()
    for k, G, lam in bad:
        with pytest.raises(_lib.VdError) as e:
            eng.dialog_ask_diverse_slots(sl, nb["ques_fwd"][:, 0], k, G, lam, 5, V - 1, V)
        assert e.value.code == _lib.VD_E_BADARG, (k, G, lam)
        assert np.array_equal(eng.dialog_slots(), rounds)
    got = eng.dialog_ask_diverse_slots(sl, nb["ques_fwd"][:, 0], 6, 3, LAM, 5, V - 1, V)
    for g, w in zip(got, want):
        assert np.array_equal(g, w)
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
    common = [*flags, "-loadPath", ckp, "-maxThreads", 3, "-math", "fp32", "-beamLen", 20]
    _cmd("visdial_b200.generate", *common, "-resultPath", tmp_path / "plain")
    plain = (tmp_path / "plain" / "results.json").read_bytes()
    _cmd("visdial_b200.generate", *common, "-resultPath", tmp_path / "plain", "-beamGroups", 1, "-diversity", 2.0)
    assert (tmp_path / "plain" / "results.json").read_bytes() == plain
    assert b"beamGroups" not in plain and b'"answers"' not in plain
    _cmd("visdial_b200.generate", *common, "-resultPath", tmp_path / "dbs", "-beamGroups", 5, "-beamSize", 10)
    res = json.load(open(str(tmp_path / "dbs" / "results.json")))
    assert res["opts"]["beamGroups"] == 5
    five = 0
    for d in res["data"]:
        for t in d["dialog"]:
            assert 1 <= len(t["answers"]) <= 5 and t["answers"][0] == t["answer"]
            five += len(t["answers"]) == 5
    assert five > 0
    lines = "".join(json.dumps({"id": "u", "image_id": res["data"][0]["image_id"], "question": q}) + "\n"
                    for q in ([1, 2, 3], [4, 5]))                      # token ids: the corpus's words are synthetic
    out = [json.loads(x) for x in _cmd("visdial_b200.chat", *common, "-serve", 1, "-capacity", 2, "-beamGroups", 5,
                                       "-beamSize", 10, stdin=lines).splitlines() if x.startswith("{")]
    answers = [o for o in out if "answer" in o]
    assert len(answers) == 2
    for o in answers:
        if o["answer"] is not None:
            alt = o["alternatives"]
            assert 1 <= len(alt) <= 5 and alt[0]["answer"] == o["answer"] and alt[0]["score"] == o["score"]
            assert all(a["score"] >= b["score"] for a, b in zip(alt, alt[1:]))
