"""The answer rules on the device (vd_set_answer_rules, DESIGN §25) against the numpy twin (tests/answer_rules_twin.py): the
top-k, merge and sampling kernels alone through vd_test_kernel, whole beam searches stepped through vd_gen_decoder_step
(bit for bit), sampled calls replayed through it, setting and clearing, launches, dialogs, refusals and the commands."""
import json

import numpy as np
import pytest

import answer_rules_twin as art
from helpers import Buf, call, run, small_batch
from test_diverse_beam_gpu import LAM, MODE_IDS, MODES, SIZES, _cmd, _forward
from test_dialog_generation_gpu import MAX_ANS, _engine, _width
from test_sampling_gpu import replay
from visdial_b200 import VD_MATH_FP32, _lib
from visdial_b200.engine import Batch, Engine
from visdial_b200.model import history_answer

pytestmark = pytest.mark.gpu

SEED = (5 << 32) | 91
ALPHA, NB = 0.7, 5


def _hist(rng, rows, L, V, start):
    """row histories with repeats (few distinct words) and pads"""
    h = rng.integers(1, min(V, 4) + 1, (rows, L)).astype(np.int32)
    h[:, 0] = start
    h[rng.random((rows, L)) < 0.1] = 0
    h[:, 0] = start
    return h


def _rule_ints(r, ld, end):
    return [ld, end, r.min_words, r.no_repeat_ngram, len(r.banned)]


def _logsoftmax(eng, x, mask=None):
    b = Buf(eng, x)
    m = Buf(eng, mask) if mask is not None else None
    run(eng, "logsoftmax_rows", [b, m], list(x.shape))
    out = b.get()
    b.free()
    if m is not None:
        m.free()
    return out


@pytest.fixture(scope="module")
def eng():
    from helpers import small_params
    e = Engine(small_params("lf-ques", "gen"))
    yield e
    e.close()


def _rule_sets(V):
    end = V
    ban = sorted({1, min(3, V - 1)} - {end})
    return [art.Rules(min_words=3, no_repeat_ngram=2, banned=ban), art.Rules(no_repeat_ngram=1),
            art.Rules(min_words=2, no_repeat_ngram=3)]


# ---- the kernels alone --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V", [5, 37, 257, 10000])
def test_topk_kernel_matches_twin(eng, V):
    rng = np.random.default_rng(V)
    L, rows, end = 8, 24, V
    for k in [kk for kk in (1, 5, 10, 32) if kk <= V]:
        for rules in _rule_sets(V):
            bn = Buf(eng, np.asarray(rules.banned or [0], np.int32))
            short = 0
            for stp in range(1, L):
                x = (rng.normal(size=(rows, V)) * 2).astype(np.float32)
                hist = _hist(rng, rows, L, V, V - 1)
                mask = hist[:, stp - 1].copy()
                mask[::5] = 0                                      # pad rows
                ref = _logsoftmax(eng, x, mask)
                bar = art.barred_rows(hist, stp, V, end, rules)
                tv, ti = art.topk(ref, bar, k)
                bufs = [Buf(eng, x), Buf(eng, mask), Buf(eng, np.zeros((rows, k), np.float32)),
                        Buf(eng, np.zeros((rows, k), np.int32)), Buf(eng, hist)]
                run(eng, "logsoftmax_topk_rows_rules", bufs + [bn if rules.banned else None],
                    [rows, V, k, stp] + _rule_ints(rules, L, end))
                gv, gi = bufs[2].get(), bufs[3].get()
                assert np.array_equal(gi, ti), (V, k, stp)
                assert np.array_equal(gv.view(np.uint32), tv.view(np.uint32)), (V, k, stp)   # logsoftmax_rows' bits
                short += int((gi < 0).any())
                for b in bufs:
                    b.free()
            bn.free()
            if V == 5 and k == 5:
                assert short > 0                                   # rows with fewer than k allowed classes


def _merge(eng, name, stp, k, G, L, end, topv, topi, scores, beams):
    N = scores.shape[0]
    bufs = [Buf(eng, topv), Buf(eng, topi), Buf(eng, scores), Buf(eng, np.zeros_like(scores)), Buf(eng, beams),
            Buf(eng, beams.copy()), Buf(eng, np.zeros(N * k, np.int32)), Buf(eng, np.zeros(N * k, np.int32)),
            Buf(eng, np.zeros((N, G, L), np.int32)), Buf(eng, np.zeros((N, G), np.int32)), Buf(eng, np.zeros((N, G)))]
    run(eng, name, bufs + [None] * (3 + (7 if name != "beam_merge" else 0)),
        [N, stp, k, G, L, end] + ([1] if name != "beam_merge" else []), [LAM])
    out = [bufs[i].get() for i in (3, 5, 6, 7, 8, 9, 10)]      # scores, beams, tokens, parent, ans, len, score out
    for b in bufs:
        b.free()
    return out


@pytest.mark.parametrize("k,G", [(6, 1), (6, 2), (8, 2), (32, 1)])
def test_merge_kernel_skips_empty_entries(eng, k, G):
    rng = np.random.default_rng(k * 10 + G)
    N, V, L = 4, 40, 6
    end = V
    for stp in range(1, L):
        beams = rng.integers(1, V, (N, k, L)).astype(np.int32)
        beams[:, :, 0] = V - 1
        scores = np.round(rng.normal(size=(N, k)), 1)
        x = np.round(rng.normal(size=(N * k, V)), 1).astype(np.float32)
        logp = (x - np.log(np.exp(x.astype(np.float64)).sum(1, keepdims=True))).astype(np.float32)
        for frac in (0.0, 0.9):                                    # no -inf entries, then many
            bar = rng.random((N * k, V)) < frac
            bar[:, end - 1] = False
            tv, ti = art.topk(logp, bar, k)
            got = _merge(eng, "beam_merge_rules", stp, k, G, L, end, tv, ti, scores, beams)
            z = art.empty_lists(N, G, 1, L)
            want = art.rules_merge_step(stp, k, G, LAM, None, L, end, tv, ti, scores, beams, *z)
            assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
            assert np.array_equal(got[2], want[2]) and np.array_equal(got[3], want[3])
            assert np.array_equal(got[4].reshape(N, G, 1, L), want[4]) and np.array_equal(got[5].reshape(N, G, 1), want[5])
            assert np.isfinite(got[0]).all() and (got[1][:, :, stp] >= 0).all()
            if frac == 0.0:
                plain = _merge(eng, "beam_merge", stp, k, G, L, end, tv, ti, scores, beams)
                for a, b in zip(plain, got):
                    assert np.array_equal(a, b)


def _sample(eng, name, x, hist, stp, rules, end, extra_ints=(), reals=(1.0,)):
    rows, V = x.shape
    L = hist.shape[1] - 1
    ans = hist.copy()
    bufs = [Buf(eng, x), Buf(eng, np.zeros(rows, np.int32)), Buf(eng, ans), Buf(eng, np.zeros((rows, L), np.float32))]
    bn = Buf(eng, np.asarray(rules.banned, np.int32)) if rules.banned else None
    hb = bufs[2]
    if name.endswith("_rules"):
        ints = [rows, V, L, SEED, stp, 3, 1] + list(extra_ints) + _rule_ints(rules, L + 1, end)
        run(eng, name, bufs + [None, hb, bn], ints, reals)
    else:
        run(eng, name, bufs + ([None] if name == "truncated_sample_rows" else []), [rows, V, L, SEED, stp, 3, 1] + list(extra_ints),
            reals)
    tok, lp = bufs[1].get(), bufs[3].get()[:, stp - 1]
    for b in bufs + ([bn] if bn else []):
        b.free()
    return tok, lp


@pytest.mark.parametrize("V", [5, 37, 257, 10000])
def test_sampling_kernels_match_twin(eng, V):
    rng = np.random.default_rng(V + 1)
    L, rows, end, T = 8, 64, V, 1.0
    near, total = 0, 0
    for rules in _rule_sets(V):
        for stp in range(1, L + 1):
            x = (rng.normal(size=(rows, V)) * 2).astype(np.float32)
            hist = np.zeros((rows, L + 1), np.int32)
            hist[:, :stp] = _hist(rng, rows, stp, V, V - 1)
            hist[:, 1:stp][hist[:, 1:stp] == 0] = 2               # sampled answers have no pads
            bar = art.barred_rows(hist, stp, V, end, rules)
            ref = _logsoftmax(eng, x)
            tok, lp = _sample(eng, "logsoftmax_sample_rows_rules", x, hist, stp, rules, end)
            want, gap = art.sample_draw(x, bar, T, SEED, stp, 3)
            ok = tok == want
            near += int((~ok).sum())
            assert (gap[~ok] < 1e-4).all(), (V, stp)
            assert not bar[np.arange(rows), tok - 1].any()
            assert np.array_equal(lp.view(np.uint32), ref[np.arange(rows), tok - 1].view(np.uint32))
            free, _ = _sample(eng, "logsoftmax_sample_rows", x, hist, stp, art.Rules(), end)
            keep = ~bar[np.arange(rows), free - 1]
            assert np.array_equal(tok[keep], free[keep])           # coupled to the rule-free draw
            for top_k, top_p in ((3, 1.0), (0, 0.9), (5, 0.8)):
                tt, tlp = _sample(eng, "truncated_sample_rows_rules", x, hist, stp, rules, end, [top_k], (T, top_p))
                wt, either, tgap = art.truncated_draw(x, bar, T, SEED, stp, top_k, top_p, 3)
                bad = [r for r in range(rows) if tt[r] != wt[r] and not (tt[r] in either[r] or tgap[r] < 1e-4)]
                assert not bad, (V, stp, top_k, top_p, bad[:5])
                near += int((tt != wt).sum())
                assert not bar[np.arange(rows), tt - 1].any()
                assert np.array_equal(tlp.view(np.uint32), ref[np.arange(rows), tt - 1].view(np.uint32))
            total += rows * 4
    assert near < total // 100


def test_all_barred_rows_draw_end(eng):
    V, L, rows = 37, 6, 8
    rules = art.Rules(min_words=4, banned=list(range(1, V)))
    x = np.random.default_rng(0).normal(size=(rows, V)).astype(np.float32)
    hist = np.zeros((rows, L + 1), np.int32)
    hist[:, 0] = V - 1
    for name, ex, re in (("logsoftmax_sample_rows_rules", [], (1.0,)), ("truncated_sample_rows_rules", [2], (1.0, 0.5))):
        tok, _ = _sample(eng, name, x, hist, 2, rules, V, ex, re)
        assert (tok == V).all()


# ---- whole calls --------------------------------------------------------------------------------------------------
RULES = art.Rules(min_words=2, no_repeat_ngram=2, banned=[3])


def _set(eng, r):
    eng.set_answer_rules(r.min_words, r.no_repeat_ngram, r.banned)


@pytest.mark.parametrize("size", sorted(SIZES))
@pytest.mark.parametrize("mode", MODES, ids=MODE_IDS)
@pytest.mark.parametrize("enc", ["lf-ques", "hrea-ques-im-hist"])
def test_beam_searches_match_twin(enc, mode, size):
    s = SIZES[size]
    V, k, G, L = s["V"], s["k"], s["G"], s["L"]
    params, eng = _engine(enc, mode, V, s["H"], s["E"], s["end_bias"])
    encOut = _forward(eng, params, s["D"])
    free = [eng.gen_beam_search(k, L, V - 1, V), eng.gen_diverse_beam_search(k, 2, LAM, L, V - 1, V),
            eng.gen_nbest_beam_search(k, 1, LAM, ALPHA, NB, L, V - 1, V)]
    rules = RULES if V > 9 else art.Rules(min_words=2, no_repeat_ngram=3)
    _set(eng, rules)
    got = [eng.gen_beam_search(k, L, V - 1, V), eng.gen_diverse_beam_search(k, 2, LAM, L, V - 1, V),
           eng.gen_nbest_beam_search(k, 1, LAM, ALPHA, NB, L, V - 1, V)]
    want = [art.host_rules_beam_search(eng, encOut, k, 1, 0.0, 0.0, 1, L, V - 1, V, rules),
            art.host_rules_beam_search(eng, encOut, k, 2, LAM, 0.0, 1, L, V - 1, V, rules),
            art.host_rules_beam_search(eng, encOut, k, 1, LAM, ALPHA, NB, L, V - 1, V, rules)]
    assert np.array_equal(got[0][0], want[0][0][:, 0, 0]) and np.array_equal(got[0][1], want[0][1][:, 0, 0])
    assert np.array_equal(got[0][2], want[0][2][:, 0, 0])
    for i in range(3):
        assert np.array_equal(got[1][i], want[1][i][:, :, 0]), i
        assert np.array_equal(got[2][i], want[2][i]), i
    assert np.array_equal(got[2][3], want[2][3])
    if V > 9:                                                      # the fallback cannot apply: every answer obeys
        for a, n in zip(got[2][0].reshape(-1, L), got[2][1].ravel()):
            if n > 0:
                assert art.obeys(a[1:n - 1], rules)
        assert not np.array_equal(got[0][0], free[0][0])
    eng.set_answer_rules()
    again = [eng.gen_beam_search(k, L, V - 1, V), eng.gen_diverse_beam_search(k, 2, LAM, L, V - 1, V),
             eng.gen_nbest_beam_search(k, 1, LAM, ALPHA, NB, L, V - 1, V)]
    for f, a in zip(free, again):
        for x, y in zip(f, a):
            assert np.array_equal(x, y)
    eng.close()


@pytest.mark.parametrize("mode", MODES, ids=MODE_IDS)
@pytest.mark.parametrize("enc", ["lf-ques", "mn-att-ques-im-hist"])
def test_sampled_calls_replay_to_the_twin(enc, mode):
    s = SIZES["tc"]
    V, L, T = s["V"], 10, 0.9
    params, eng = _engine(enc, mode, V, s["H"], s["E"], s["end_bias"])
    encOut = _forward(eng, params, s["D"])
    rows = encOut.shape[0]
    _set(eng, RULES)
    for trunc in ((0, 1.0), (0, 0.9)):
        if trunc == (0, 1.0):
            ans, logp = eng.gen_sample(L, V - 1, T, SEED, 4)
        else:
            ans, logp = eng.gen_truncated_sample(L, V - 1, T, SEED, 4, *trunc)
        lps = replay(eng, encOut, ans)
        bad = 0
        for t in range(1, L + 1):
            bar = art.barred_rows(ans, t, V, V, RULES)
            assert not bar[np.arange(rows), ans[:, t] - 1].any()
            if trunc == (0, 1.0):
                want, gap = art.sample_draw(lps[t - 1], bar, T, SEED, t, 4)
                bad += int(((ans[:, t] != want) & (gap > 1e-3)).sum())
            else:
                want, either, gap = art.truncated_draw(lps[t - 1], bar, T, SEED, t, *trunc, row_offset=4)
                bad += sum(1 for r in range(rows) if ans[r, t] != want[r] and ans[r, t] not in either[r] and gap[r] > 1e-3)
        assert bad <= rows * L // 50, bad
        for r in range(rows):
            w = history_answer(ans[r, 1:], V)
            assert art.obeys(w, RULES, finished=len(w) < L)
    eng.set_answer_rules()
    eng.close()


def test_launches_per_step_are_the_rule_free_calls():
    s = SIZES["tc"]
    params, eng = _engine("lf-ques", VD_MATH_FP32, s["V"], s["H"], s["E"], s["end_bias"])
    _forward(eng, params, 2)
    V = s["V"]
    counts = {}
    for ruled in (False, True):
        if ruled:
            _set(eng, RULES)
        for L in (4, 9):
            for name, fn in (("beam", lambda: eng.gen_beam_search(6, L, V - 1, V)),
                             ("sample", lambda: eng.gen_sample(L, V - 1, 1.0, SEED, 0)),
                             ("trunc", lambda: eng.gen_truncated_sample(L, V - 1, 1.0, SEED, 0, 5, 1.0))):
                eng.profile_reset()
                fn()
                counts[name, L, ruled] = eng.launch_count()
    for name in ("beam", "sample", "trunc"):
        assert counts[name, 9, True] - counts[name, 4, True] == counts[name, 9, False] - counts[name, 4, False], counts
    eng.close()


def test_refusals_keep_the_rules():
    s = SIZES["tc"]
    V = s["V"]
    params, eng = _engine("lf-ques", VD_MATH_FP32, V, s["H"], s["E"], s["end_bias"])
    _forward(eng, params, 2)
    _set(eng, RULES)
    ruled = eng.gen_beam_search(5, 12, V - 1, V)
    for bad in (dict(min_words=-1), dict(no_repeat_ngram=-1), dict(banned=[0]), dict(banned=[V + 1]),
                dict(banned=list(range(1, 1026)))):
        with pytest.raises(_lib.VdError) as e:
            eng.set_answer_rules(**bad)
        assert e.value.code == _lib.VD_E_BADARG
    r = _lib.vd_answer_rules(0, 0, 2, None)
    assert eng.lib.vd_set_answer_rules(eng.h, r) == _lib.VD_E_BADARG
    for a, b in zip(ruled, eng.gen_beam_search(5, 12, V - 1, V)):
        assert np.array_equal(a, b)                                # the old rules stand
    eng.set_answer_rules(min_words=11)
    with pytest.raises(_lib.VdError):
        eng.gen_beam_search(5, 12, V - 1, V)                       # min_words > L - 2
    eng.gen_sample(12, V - 1, 1.0, SEED)                           # sampling allows L - 1
    eng.set_answer_rules(banned=[V])
    with pytest.raises(_lib.VdError):
        eng.gen_beam_search(5, 12, V - 1, V)                       # <END> banned
    eng.set_answer_rules()
    eng.close()


# ---- dialogs and pools --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("enc", ["lf-ques-hist", "hre-ques-hist", "hrea-ques-im-hist", "mn-att-ques-im-hist"])
def test_fp32_dialogs_and_pool_asks_obey_and_agree(enc):
    V = 64
    params, eng = _engine(enc, VD_MATH_FP32, V, 32, 16, 2.0)
    nb = small_batch(params, B=2, seed=3)
    W = _width(params, nb)
    L = 10
    _set(eng, RULES)
    ans, length, score, hist = eng.gen_dialog_beam_search(Batch(nb), 4, L, V - 1, V, W, MAX_ANS)
    R = params["maxQuesCount"]
    for a, n in zip(ans.reshape(-1, L), length.ravel()):
        if n > 0:
            assert art.obeys(a[1:n - 1], RULES)
    # the same rounds asked one at a time through a session: the same answers
    eng.dialog_begin(Batch(nb), W, MAX_ANS)
    q = np.asarray(nb["ques_fwd"])
    eng.set_answer_rules(banned=[V])                               # refused: the session's round and next ask stay
    with pytest.raises(_lib.VdError):
        eng.dialog_ask_beam_slots([0, 1], q[:, 0], 4, L, V - 1, V)
    assert eng.dialog_round()[0] == 0
    _set(eng, RULES)
    for r in range(R):
        a2, n2, s2 = eng.dialog_ask_beam_slots(list(range(q.shape[0])), q[:, r], 4, L, V - 1, V)
        a1 = ans.reshape(q.shape[0], R, L)[:, r]
        assert np.array_equal(a2, a1) and np.array_equal(n2, length.reshape(q.shape[0], R)[:, r]), r
    eng.set_answer_rules()
    eng.dialog_end()
    eng.close()


# ---- commands -----------------------------------------------------------------------------------------------------
from test_dialog_generation_gpu import command_files  # noqa: E402,F401  (the generate command's corpus and checkpoint)


def test_generate_and_chat_commands(command_files, tmp_path):
    flags, fo, ckp = command_files
    common = [*flags, "-loadPath", ckp, "-maxThreads", 3, "-math", "fp32", "-beamLen", 20]
    _cmd("visdial_b200.generate", *common, "-resultPath", tmp_path / "plain")
    plain = (tmp_path / "plain" / "results.json").read_bytes()
    _cmd("visdial_b200.generate", *common, "-resultPath", tmp_path / "plain", "-minWords", 0, "-noRepeatNgram", 0)
    assert (tmp_path / "plain" / "results.json").read_bytes() == plain
    assert b"minWords" not in plain and b"bannedWords" not in plain
    rules = ["-minWords", 2, "-noRepeatNgram", 2, "-bannedWords", "w1"]   # the corpus's words are w1 .. w<V-2>
    for extra in ([], ["-sampleWords", 1, "-topP", 0.9]):
        _cmd("visdial_b200.generate", *common, *rules, *extra, "-resultPath", tmp_path / "ruled")
        res = json.load(open(str(tmp_path / "ruled" / "results.json")))
        assert res["opts"]["minWords"] == 2 and res["opts"]["bannedWords"] == "w1"
        for d in res["data"]:
            for t in d["dialog"]:
                words = t["answer"].split()
                assert "w1" not in words
                grams = [tuple(words[i:i + 2]) for i in range(len(words) - 1)]
                assert len(grams) == len(set(grams)), t["answer"]
                if not extra:
                    assert len(words) >= 2, t["answer"]
    res = json.load(open(str(tmp_path / "plain" / "results.json")))
    lines = "".join(json.dumps({"id": "u", "image_id": res["data"][0]["image_id"], "question": q}) + "\n"
                    for q in ([1, 2, 3], [4, 5]))
    out = [json.loads(x) for x in _cmd("visdial_b200.chat", *common, "-serve", 1, "-capacity", 2, *rules,
                                       stdin=lines).splitlines() if x.startswith("{")]
    assert len([o for o in out if "answer" in o]) == 2
