"""Resuming conversations in a dialog pool (vd_dialog_join_rounds, DESIGN §21): a conversation joined at round r with the
rounds it already had must continue exactly as the original conversation would have.  In VD_MATH_FP32 that is bit for bit:
history rows, answers, lengths, fp64 scores and encodings; in the tensor-core modes the answers are host_decode's search
from the ask's own state and the encodings are within §7's bound of vd_encoder_forward.  The prefill kernel is checked
against the append kernel it shares its row rule with, and against the host rule."""
import numpy as np
import pytest

from dialog_history import next_row, row_words
from helpers import Pool, call, check, small_batch, small_params, within
from host_decode import host_beam_search
from test_dialog_generation_gpu import MAX_ANS, SEED, _engine, _width
from test_dialog_pool_gpu import _code, _rows
from test_dialog_session_gpu import SIZES, _AskView, _pool_engine
from visdial_b200 import VD_MATH_F16, VD_MATH_FP32, VD_MATH_TF32
from visdial_b200 import _lib
from visdial_b200.engine import Batch, Engine
from visdial_b200.model import history_answer

pytestmark = pytest.mark.gpu

HIST_ENCODERS = ["lf-ques-hist", "hre-ques-hist", "hre-ques-im-hist", "hrea-ques-im-hist", "mn-ques-hist",
                 "mn-ques-im-hist", "mn-att-ques-im-hist"]


def _W(params, nb):
    return _width(params, nb) if params["useHistory"] else 0


def _answers(words, R):
    """(D, R, Ta) left-aligned rows of the answer word lists {d: [round j's words]}"""
    D = len(words)
    Ta = max([1] + [len(w) for d in range(D) for w in words[d]])
    a = np.zeros((D, R, Ta), np.int32)
    for d in range(D):
        for j, w in enumerate(words[d]):
            a[d, j, :len(w)] = w
    return a


# ---- the prefill kernel -----------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def keng():
    e = Engine(small_params("lf-ques", "disc"))
    e.profile(True)
    yield e
    e.close()


@pytest.mark.parametrize("concat", [0, 1], ids=["per_round", "concat"])
@pytest.mark.parametrize("C,R,W", [(6, 10, 11), (5, 10, 24), (4, 4, 7)])
def test_hist_prefill_equals_sequential_appends(keng, concat, C, R, W):
    """k_hist_prefill's rows 1..r_i, one launch, equal r_i sequential k_hist_append launches (==) and the host rule:
    empty and pad-only answers, <END> mid-row, questions of pads, rows that overflow W, r = 0 and R-1, guard bands."""
    rng = np.random.default_rng(C * 10 + R + W + concat)
    Tq, Ta, V, mal = 5, 7, 40, 4
    end = V
    n = C - 1                                             # one slot stays free
    slot = rng.permutation(C)[:n].astype(np.int32)
    rounds = rng.integers(0, R, n).astype(np.int32)
    rounds[0], rounds[-1] = 0, R - 1
    base = np.zeros((C, R, W), np.int32)                 # row 0: a caption; rows above: whatever a join wrote (pads)
    for c in range(C):
        L = int(rng.integers(0 if c == 1 else 1, W + 1))
        base[c, 0, W - L:] = rng.integers(1, V - 1, L)
    ques = np.zeros((n, R, Tq), np.int32)
    ans = np.zeros((n, R, Ta), np.int32)
    for i in range(n):
        for j in range(R):
            ql = 0 if rng.random() < 0.15 else int(rng.integers(1, Tq + 1))
            ques[i, j, Tq - ql:] = rng.integers(1, V - 1, ql)
            kind = rng.random()
            if kind < 0.15:
                continue                                  # empty answer
            al = int(rng.integers(1, Ta + 1))
            ans[i, j, :al] = rng.integers(1, V - 1, al)
            if kind < 0.3:
                ans[i, j, al // 2] = end                  # <END> mid-row
            elif kind < 0.45:
                ans[i, j, ::2] = 0                        # pads between words are not words
    order = np.argsort(-rounds, kind="stable")
    cnt = np.asarray([(rounds > j).sum() for j in range(R)], np.int32)
    row0 = np.concatenate([[0], np.cumsum(cnt)[:-1]]).astype(np.int32)
    P = int(cnt.sum())
    q = np.zeros((max(P, 1), Tq), np.int32)
    for i, d in enumerate(order):
        for j in range(rounds[d]):
            q[row0[j] + i] = ques[d, j]
    pool = Pool(keng)
    try:
        hd = pool(base)
        n0 = keng.launch_count()
        check(call(keng, "hist_prefill", [hd, pool(slot[order]), pool(rounds[order]), pool(row0), pool(q), pool(ans[order])],
                   [n, R, W, Tq, Ta, end, mal, concat]))
        assert keng.launch_count() == n0 + 1
        got = hd.get()
        want = base.copy()
        for d in range(n):
            one = pool(base[slot[d]][None].copy())
            for j in range(rounds[d]):
                check(call(keng, "hist_append_slots", [one, pool(ques[d]), pool(ans[d, j][None]), None, None, None],
                           [1, R, W, j, Tq, Ta, Ta, end, mal, concat]))
            want[slot[d]] = one.get()[0]
            h = base[slot[d]].copy()                      # the host rule
            for j in range(rounds[d]):
                h[j + 1] = next_row(h[j], row_words(ques[d, j]), history_answer(ans[d, j], end), bool(concat), end, W, mal)
            assert np.array_equal(want[slot[d]], h), d
        assert np.array_equal(got, want)
    finally:
        pool.free()


# ---- a resumed conversation continues as the original -----------------------------------------------------------------
def _original(eng, nb, W, ask, words_of, stop):
    """Pool A: dialog d joins at round 0 and is asked all R rounds, grouped by round.  Returns each dialog's per-round
    results, the answer words its history took, and its history when it reached round stop[d]."""
    D, R, Tq = nb["ques_fwd"].shape
    eng.dialog_open(D, Tq, W, MAX_ANS)
    slots = eng.dialog_join(Batch(nb), np.arange(D) * R).tolist()
    res, words, hist = {d: [] for d in range(D)}, {d: [] for d in range(D)}, {}
    for t in range(R):
        for d in range(D):
            if stop[d] == t and W:
                hist[d] = eng.dialog_slot_history([slots[d]], W)[0]
        out = ask(slots, nb["ques_fwd"][:, t])
        for d in range(D):
            res[d].append(tuple(x[d] for x in out))
            if t < stop[d]:
                words[d].append(words_of(out, d))
    return res, words, hist


def _resumed(eng, nb, other, W, ask, stop, words, draw=True):
    """Pool B: two other conversations join and are asked first; then nb's dialogs resume in non-lowest slots at stop[d]
    from A's questions and answers, and everyone is asked on, grouped by round.  Returns the results of rounds >= stop[d]
    and each dialog's history just after the resume."""
    D, R, Tq = nb["ques_fwd"].shape
    C = D + 4
    eng.dialog_open(C, Tq, W, MAX_ANS)
    live = eng.dialog_join(Batch(_rows(other, [0, 1]))).tolist()
    ask(live, other["ques_fwd"][[0, 1], 0])
    slots = list(range(C - 1, C - 1 - D, -1))
    rounds = np.asarray([stop[d] for d in range(D)], np.int32)
    eng.dialog_join_rounds(Batch(nb), rounds, _answers(words, R) if W else None, slots,
                           np.arange(D) * R if draw else None)
    assert [int(eng.dialog_slots()[s]) for s in slots] == rounds.tolist()
    hist = {d: eng.dialog_slot_history([slots[d]], W)[0] for d in range(D)} if W else {}
    res = {d: [] for d in range(D)}
    for t in range(R):
        pick = [d for d in range(D) if stop[d] <= t]
        sl = [slots[d] for d in pick]
        q = nb["ques_fwd"][pick, t]
        if t + 1 < R:                                      # the others share the asks
            sl, q = live + sl, np.concatenate([other["ques_fwd"][[0, 1], t + 1], q])
        if not sl:
            continue
        out = ask(sl, q)
        off = len(sl) - len(pick)
        for i, d in enumerate(pick):
            res[d].append(tuple(x[off + i] for x in out))
    return res, hist


def _stops(D, R):
    return {d: [0, 1, R // 2, R - 1, 3, R - 2][d % 6] for d in range(D)}


def _same(a, b):
    return len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b))


def _check_resume(eng, nb, other, W, ask, words_of, draw=True):
    D, R = nb["ques_fwd"].shape[:2]
    stop = _stops(D, R)
    want, words, want_hist = _original(eng, nb, W, ask, words_of, stop)
    got, hist = _resumed(eng, nb, other, W, ask, stop, words, draw)
    for d in range(D):
        if W:
            assert np.array_equal(hist[d], want_hist[d]), d
        assert len(got[d]) == R - stop[d]
        for i, g in enumerate(got[d]):
            assert _same(g, want[d][stop[d] + i]), (d, stop[d] + i)


@pytest.mark.parametrize("size", sorted(SIZES))
@pytest.mark.parametrize("enc", HIST_ENCODERS)
def test_fp32_resume_equals_the_original(enc, size):
    s = SIZES[size]
    params, eng = _engine(enc, VD_MATH_FP32, s["V"], s["H"], s["E"], s["end_bias"])
    nb = small_batch(params, B=6, seed=7)
    other = small_batch(params, B=2, seed=11)
    k, L, V = s["k"], s["L"], s["V"]

    def ask(slots, q):
        a, n, sc = eng.dialog_ask_beam_slots(slots, q, k, L, V - 1, V)
        return a, n, sc, eng.dialog_encoding().numpy()

    _check_resume(eng, nb, other, _W(params, nb), ask, lambda out, d: history_answer(out[0][d], V, out[1][d]))
    eng.close()


@pytest.mark.parametrize("enc", ["lf-ques-hist", "hrea-ques-im-hist", "mn-att-ques-im-hist"])
def test_fp32_resumed_sampling_and_pool_asks(enc):
    V, L, T, r0 = 256, 8, 0.9, 21
    params, eng = _engine(enc, VD_MATH_FP32, V, 128, 64, 2.0)
    nb = small_batch(params, B=6, seed=7)
    other = small_batch(params, B=2, seed=11)
    _check_resume(eng, nb, other, _W(params, nb),
                  lambda slots, q: eng.dialog_ask_sample_slots(slots, q, L, V - 1, V, T, SEED, r0),
                  lambda out, d: history_answer(out[0][d, 1:], V))
    eng.close()
    params, eng, nb = _pool_engine(enc, VD_MATH_FP32, B=6)
    other = small_batch(params, B=2, seed=11)
    rng = np.random.default_rng(5)                         # _pool_engine's pool rows
    prow = rng.integers(1, 65, (300, MAX_ANS)).astype(np.int32)
    prow[::7, 3:] = 0
    _check_resume(eng, nb, other, _W(params, nb), lambda slots, q: eng.dialog_ask_pool_slots(slots, q, 3),
                  lambda out, d: history_answer(prow[out[0][d, 0]], params["vocabSize"]), draw=False)
    eng.close()


# ---- ground truth ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dec", ["gen", "disc"])
@pytest.mark.parametrize("enc", HIST_ENCODERS + ["lf-ques", "lf-ques-im"])
def test_fp32_ground_truth_resume(enc, dec):
    """Dataset dialogs resumed at round r on their ground-truth answers: the rebuilt rows are the batch's history rows,
    and asking question r answers as the ground-truth forward's row (b, r) does."""
    if dec == "gen":
        params, eng = _engine(enc, VD_MATH_FP32, 64, 64, 32, 2.0)
        nb = small_batch(params, B=6, seed=7)
    else:
        params, eng, nb = _pool_engine(enc, VD_MATH_FP32, B=6)
    D, R, Tq = nb["ques_fwd"].shape
    V = params["vocabSize"]
    W = nb["hist"].shape[2] if params["useHistory"] else 0    # the dataset's width: its rows are cut as the rule cuts
    ds = [0, 2, 4]                                         # small_batch's odd dialogs have an empty last round
    rounds = np.asarray([1, R // 2, R - 1], np.int32)
    enc_full = eng.encoder_forward(Batch(nb)).numpy().reshape(D, R, -1)
    if dec == "gen":
        wa, wn, ws = eng.gen_beam_search(3, 10, V - 1, V)
    else:
        wi, wsc = eng.answer_pool_retrieve(Batch(nb), 3)
    eng.dialog_open(5, Tq, W, MAX_ANS)
    slots = [4, 1, 3]
    sub = _rows(nb, ds)
    words = {i: [history_answer(nb["answer_out"][d, j], V) for j in range(rounds[i])] for i, d in enumerate(ds)}
    eng.dialog_join_rounds(Batch(sub), rounds, _answers(words, R) if W else None, slots)
    if W:
        h = eng.dialog_slot_history(slots, W)
        for i, d in enumerate(ds):
            want = np.zeros((R, W), np.int32)
            want[:rounds[i] + 1] = nb["hist"][d, :rounds[i] + 1]
            assert np.array_equal(h[i], want), d
    q = np.stack([nb["ques_fwd"][d, rounds[i]] for i, d in enumerate(ds)])
    if dec == "gen":
        a, n, sc = eng.dialog_ask_beam_slots(slots, q, 3, 10, V - 1, V)
    else:
        ti, tsc = eng.dialog_ask_pool_slots(slots, q, 3)
    got = eng.dialog_encoding().numpy()
    for i, d in enumerate(ds):
        row = d * R + rounds[i]
        assert np.array_equal(got[i], enc_full[d, rounds[i]]), d
        if dec == "gen":
            assert np.array_equal(a[i], wa[row]) and n[i] == wn[row] and sc[i] == ws[row], d
        else:
            assert np.array_equal(ti[i], wi[row]) and np.array_equal(tsc[i], wsc[row]), d
    eng.close()


# ---- tensor-core modes --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", [VD_MATH_TF32, VD_MATH_F16], ids=["tf32", "f16"])
@pytest.mark.parametrize("enc", ["lf-ques-hist", "hre-ques-im-hist", "hrea-ques-im-hist", "mn-att-ques-im-hist"])
def test_tensor_core_resume(enc, mode):
    """Each ask after a resume answers as host_beam_search from its own state, bit for bit; each encoding is within 5e-3
    of vd_encoder_forward on the conversation's own history rebuilt as a batch."""
    s = SIZES["tc"]
    params, eng = _engine(enc, mode, s["V"], s["H"], s["E"], s["end_bias"])
    nb = small_batch(params, B=4, seed=7)
    D, R, Tq = nb["ques_fwd"].shape
    W, k, L, V = _W(params, nb), s["k"], s["L"], s["V"]
    rng = np.random.default_rng(3)
    words = {d: [list(rng.integers(1, V - 1, int(rng.integers(0, MAX_ANS + 2)))) for _ in range(R)] for d in range(D)}
    stop = np.asarray([0, 2, R // 2, R - 1][:D], np.int32)
    eng.dialog_open(D, Tq, W, MAX_ANS)
    eng.dialog_join_rounds(Batch(nb), stop, _answers(words, R), list(range(D)))
    encs = {d: {} for d in range(D)}
    for t in range(R):
        pick = [d for d in range(D) if stop[d] <= t]
        a, n, sc = eng.dialog_ask_beam_slots(pick, nb["ques_fwd"][pick, t], k, L, V - 1, V)
        rows = eng.dialog_encoding().numpy()
        wa, wn, ws = host_beam_search(_AskView(eng), rows, k, L, V - 1, V)
        assert np.array_equal(a, wa) and np.array_equal(n, wn) and np.array_equal(sc, ws), t
        for i, d in enumerate(pick):
            encs[d][t] = rows[i]
    hist = eng.dialog_slot_history(list(range(D)), W)
    for d in range(D):
        full = eng.encoder_forward(Batch(dict(_rows(nb, [d]), hist=hist[d][None].copy()))).numpy().reshape(R, -1)
        for t, e in encs[d].items():
            within(e, full[t], 5e-3, "dialog %d round %d" % (d, t))
    eng.close()


# ---- reopen --------------------------------------------------------------------------------------------------------------
def test_reopen_keeps_every_conversation_in_its_slot(command_files):
    """DialogPool.reopen after vd_set_parameters: with the same weights the next asks equal (==) those of a pool that
    never reopened and the slot ids hold; with new weights they equal a fresh pool resumed from the same transcripts."""
    from test_cli_gpu import _model
    from visdial_b200 import init_parameters
    from visdial_b200.checkpoint import load_checkpoint
    _, fo, ckp = command_files
    ck = load_checkpoint(ckp)
    m1, dl1 = _model(ck["modelParams"], fo, "val", ck)
    m2, dl2 = _model(ck["modelParams"], fo, "val", ck)
    R = m1.params["maxQuesCount"]
    ques = np.asarray(dl1.getIndexData(np.arange(3), m1.params, "val")["ques_fwd"])
    params = {"beamSize": 3, "beamLen": 12}

    def drive(pool, slots, t0, t1):
        return [{s: e and e["answer"] for s, e in pool.ask({s: ques[i, t] for i, s in enumerate(slots)}).items()}
                for t in range(t0, t1)]

    def opened(m, dl):
        p = m.openDialogPool(dl, "val", 6, params)
        p.join([3])                                        # slot 0 stays at round 0
        s = p.join([0, 1, 2])
        drive(p, s, 0, 3)
        return p, s

    a, sa = opened(m1, dl1)
    want = drive(a, sa, 3, R)
    b, sb = opened(m2, dl2)
    m2.engine.set_parameters(m2.engine.get_parameters())
    assert _code(b.ask, {sb[0]: ques[0, 3]}) == _lib.VD_E_STATE          # stale until reopened
    b.reopen()
    assert sb == sa and [b.round(s) for s in sb] == [3, 3, 3] and b.round(0) == 0
    assert drive(b, sb, 3, R) == want
    flat = init_parameters(m2.params, seed=99)             # new weights
    b, sb = opened(m2, dl2)
    trans = {s: list(zip(b.convs[s]["ques"], b.convs[s]["ans"])) for s in sb}
    m2.engine.set_parameters(flat)
    b.reopen()
    got = drive(b, sb, 3, R)
    m1.engine.set_parameters(flat)
    f = m1.openDialogPool(dl1, "val", 6, params)
    f.join([3])
    assert [f.resume(i, trans[s]) for i, s in enumerate(sb)] == sb
    assert drive(f, sb, 3, R) == got
    for m, dl in ((m1, dl1), (m2, dl2)):
        dl.close()
        m.engine.close()


# ---- work and refusals ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("enc", ["lf-ques-im-hist", "hre-ques-hist", "hrea-ques-im-hist", "mn-att-ques-im-hist"])
def test_resume_work(enc):
    """At fixed r_max the launches do not depend on n; the LSTM FLOP classes are P = sum r_i rows' worth (a full forward
    of the same dialogs does n*R); mn runs no question pair."""
    params, eng = _engine(enc, VD_MATH_FP32, 9, 32, 12, 1.0)
    nb = small_batch(params, B=6, seed=7)
    R, Tq = nb["ques_fwd"].shape[1:]
    W = _W(params, nb)
    words = {d: [[1, 2]] * R for d in range(6)}
    eng.profile(True)
    lstm = ("lstm_step", "lstm_step_small", "lstm_step_first")

    def measure(ds, rounds):
        eng.dialog_open(6, Tq, W, MAX_ANS)
        eng.profile_reset()
        n0 = eng.launch_count()
        eng.dialog_join_rounds(Batch(_rows(nb, ds)), np.asarray(rounds, np.int32), _answers({i: words[d] for i, d in
                                                                                              enumerate(ds)}, R), ds)
        return eng.launch_count() - n0, sum(eng.kernel_stats(c)["flops"] for c in lstm)

    l1, f1 = measure([0, 1], [4, 2])
    l2, f2 = measure([0, 1, 2, 3, 4], [4, 1, 3, 2, 4])
    assert l1 == l2, (l1, l2)
    if enc.startswith("lf"):
        assert f1 == f2 == 0
    else:
        assert f1 > 0 and f2 / f1 == pytest.approx(14 / 6), (f1, f2)
        eng.profile_reset()
        eng.encoder_forward(Batch(_rows(nb, [0, 1])))
        full = sum(eng.kernel_stats(c)["flops"] for c in lstm)
        if enc.startswith("mn"):                           # the history pair only
            assert f1 < full * 6 / (2 * R)
    eng.close()


def test_refusals_change_nothing():
    V = 9
    params, eng = _engine("hrea-ques-im-hist", VD_MATH_FP32, V, 32, 12, 1.0)
    nb = small_batch(params, B=4, seed=7)
    R, Tq = nb["ques_fwd"].shape[1:]
    W = _width(params, nb)
    ans = _answers({0: [[1, 2]] * R, 1: [[3]] * R}, R)
    sub = Batch(_rows(nb, [0, 1]))

    def jr(rounds=(2, 3), a=ans, slots=(2, 3), b=sub, Ta=None):
        a2 = a if Ta is None else a[:, :, :Ta]
        return eng.dialog_join_rounds(b, np.asarray(rounds, np.int32), a2, list(slots))

    assert _code(jr) == _lib.VD_E_STATE                                                 # no pool
    eng.dialog_open(4, Tq, W, MAX_ANS)
    live = eng.dialog_join(Batch(_rows(nb, [2, 3]))).tolist()
    assert live == [0, 1]

    def next_asks():
        return eng.dialog_ask_beam_slots(live, nb["ques_fwd"][[2, 3], int(eng.dialog_slots()[0])], 3, 6, 8, 9)

    before = (eng.dialog_slots().copy(), eng.dialog_slot_history(live, W))
    bad = np.array(ans)
    bad[0, 1, 0] = V + 1
    badq = dict(_rows(nb, [0, 1]))
    badq["ques_fwd"] = badq["ques_fwd"].copy()
    badq["ques_fwd"][1, 0, -1] = -1
    wide = dict(_rows(nb, [0, 1]))
    wide["ques_fwd"] = np.zeros((2, R, Tq + 1), np.int32)
    for fn, code in ((lambda: jr(slots=(1, 3)), _lib.VD_E_STATE),                      # an occupied slot
                     (lambda: jr(rounds=(2, R)), _lib.VD_E_BADARG),
                     (lambda: jr(rounds=(-1, 2)), _lib.VD_E_BADARG),
                     (lambda: jr(slots=(2, 4)), _lib.VD_E_BADARG),                     # outside [0, C)
                     (lambda: jr(slots=(2, 2)), _lib.VD_E_BADARG),                     # named twice
                     (lambda: jr(Ta=0), _lib.VD_E_BADARG),
                     (lambda: jr(a=bad), _lib.VD_E_BADARG),                            # an answer token
                     (lambda: jr(b=Batch(badq)), _lib.VD_E_BADARG),                    # a question token
                     (lambda: eng.dialog_join_rounds(sub, np.asarray([2, 3], np.int32), None, [2, 3]), _lib.VD_E_BADARG),
                     (lambda: jr(b=Batch(wide)), _lib.VD_E_SHAPE)):
        assert _code(fn) == code
        assert np.array_equal(eng.dialog_slots(), before[0])
    narrow = dict(_rows(nb, [0, 1]))
    narrow["hist"] = np.zeros((2, R, W + 1), np.int32)
    assert _code(lambda: jr(b=Batch(narrow))) == _lib.VD_E_BADARG                    # hist_width < b->Th
    want = next_asks()
    eng.dialog_open(4, Tq, W, MAX_ANS)
    assert eng.dialog_join(Batch(_rows(nb, [2, 3]))).tolist() == live
    assert _same(next_asks(), want) and np.array_equal(eng.dialog_slot_history(live, W)[:, 0], before[1][:, 0])
    eng.set_parameters(eng.get_parameters())
    assert _code(jr) == _lib.VD_E_STATE                                                 # a stale pool
    eng.close()


# ---- the serve command -----------------------------------------------------------------------------------------------
from test_dialog_generation_gpu import command_files  # noqa: E402,F401


def test_serve_history_answers_as_generate(command_files, tmp_path):
    """A join line whose history holds a dataset dialog's ground-truth rounds 0..r-1 (questions as token ids, answers as
    text) is answered at round r as generate answers it on the dataset's history."""
    import json
    import subprocess
    import sys

    from test_cli_gpu import _model
    from test_dialog_generation_gpu import ROOT
    from visdial_b200.chat import _image_index
    from visdial_b200.checkpoint import load_checkpoint
    from visdial_b200.utils import idToWords
    flags, fo, ckp = command_files
    ck = load_checkpoint(ckp)
    m, dl = _model(ck["modelParams"], fo, "val", ck)
    inds = [0, 6, 7]                                       # the corpus's dialogs 1-5 hold its empty rounds
    ids = [list(_image_index(dl, "val"))[i] for i in inds]
    b = dl.getIndexData(np.asarray(inds), m.params, "val")
    ques, aout = np.asarray(b["ques_fwd"]), np.asarray(b["answer_out"])
    R = ques.shape[1]
    table = m.generateAnswers(dl, "val", {"maxThreads": 8, "beamSize": 5, "beamLen": 20})
    gt = [table[i] for i in inds]
    end = dl.word2ind["<END>"]
    lines, want = [], {}
    for d, (i, r) in enumerate(zip(ids, [1, R // 2, R - 1])):
        hist = [[[int(t) for t in ques[d, j] if t], idToWords(history_answer(aout[d, j], end), dl.ind2word).strip()]
                for j in range(r)]
        lines.append({"id": "u%d" % d, "image_id": i, "history": hist, "question": [int(t) for t in ques[d, r] if t]})
        want["u%d" % d] = (r, idToWords(gt[d]["dialog"][r]["answer"], dl.ind2word).strip())
    lines += [{"id": "u0", "history": [], "question": [1]},                            # an open id
              {"id": "x", "image_id": ids[0], "history": [["a"]]},                    # malformed
              {"id": "y", "image_id": ids[0], "history": [[[1], "w1"]] * R}]           # R rounds
    dl.close(); m.engine.close()
    r = subprocess.run([sys.executable, "-m", "visdial_b200.chat"] + [str(a) for a in flags] +
                       ["-loadPath", ckp, "-math", "fp32", "-beamLen", "20", "-serve", "1", "-capacity", "4"],
                       cwd=ROOT, input="".join(json.dumps(x) + "\n" for x in lines), capture_output=True, text=True,
                       timeout=1200)
    assert r.returncode == 0, r.stderr[-3000:]
    out = [json.loads(x) for x in r.stdout.splitlines() if x.startswith("{")]
    assert sorted(o["id"] for o in out if "error" in o) == ["u0", "x", "y"]
    got = {o["id"]: (o["round"], o["answer"]) for o in out if "answer" in o}
    assert got == want
