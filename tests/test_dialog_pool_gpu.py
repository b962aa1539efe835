"""Dialog pools (vd_dialog_open / join / ask_*_slots / leave, DESIGN §20): conversations that join, are asked and leave on
their own, each at its own round, several rounds in one ask.  Fed the same questions, a conversation must answer as a
one-dialog vd_dialog_begin session does, whichever conversations share its asks, whichever slot it holds and whenever it
joined: bit for bit in VD_MATH_FP32; in the tensor-core modes each ask's answers are host_decode's search from the ask's
own state, bit for bit, and its encoding is within §7's bound of vd_encoder_forward on the conversation's own history."""
import numpy as np
import pytest

from helpers import Pool, call, check, small_batch, small_params, within
from host_decode import host_beam_search
from test_dialog_generation_gpu import MAX_ANS, SEED, _engine, _width
from test_dialog_session_gpu import SIZES, _AskView, _pool_engine
from visdial_b200 import VD_MATH_F16, VD_MATH_FP32, VD_MATH_TF32
from visdial_b200 import _lib
from visdial_b200.engine import Batch, Engine

pytestmark = pytest.mark.gpu

ALL_ENCODERS = ["lf-ques", "lf-ques-im", "lf-ques-hist", "lf-ques-im-hist", "lf-att-ques-im-hist", "hre-ques-hist",
                "hre-ques-im-hist", "hrea-ques-im-hist", "mn-ques-hist", "mn-ques-im-hist", "mn-att-ques-im-hist"]


def _rows(nb, ds):
    return {k: np.ascontiguousarray(nb[k][ds]) for k in ("ques_fwd", "hist", "img_feat") if k in nb}


def _W(params, nb):
    return _width(params, nb) if params["useHistory"] else 0


def _code(fn, *a):
    try:
        fn(*a)
    except _lib.VdError as e:
        return e.code
    return _lib.VD_OK


def _drive(eng, nb, C, W, ask, seed, draw_base=None):
    """A seeded schedule over nb's D dialogs in a pool of capacity C < D: joins while slots are free, asks of random
    subsets in random row order (so one ask mixes rounds), some conversations leaving before their last round, and slots
    reused after a leave.  Returns each dialog's ask results in order and its history rows when it left."""
    D, R, Tq = nb["ques_fwd"].shape
    rng = np.random.default_rng(seed)
    eng.dialog_open(C, Tq, W, MAX_ANS)
    waiting, live = list(range(D)), {}
    got, hist = {d: [] for d in range(D)}, {}
    stop = {d: R if rng.random() < 0.7 else int(rng.integers(1, R)) for d in range(D)}
    mixed = reused = False
    used = set()
    while waiting or live:
        free = C - len(live)
        if waiting and free and (not live or rng.random() < 0.4):
            ds = waiting[:int(rng.integers(1, min(free, len(waiting)) + 1))]
            waiting = waiting[len(ds):]
            base = None if draw_base is None else np.asarray([draw_base[d] for d in ds])
            slots = eng.dialog_join(Batch(_rows(nb, ds)), base).tolist()
            reused |= bool(used & set(slots))
            used |= set(slots)
            live.update(zip(slots, ds))
            continue
        occupied = sorted(live)
        pick = [s for s in occupied if rng.random() < 0.6] or [occupied[int(rng.integers(len(occupied)))]]
        pick = [pick[i] for i in rng.permutation(len(pick))]
        rounds = eng.dialog_slots()
        assert all(rounds[s] == len(got[live[s]]) for s in occupied)
        mixed |= len({int(rounds[s]) for s in pick}) > 1
        q = np.stack([nb["ques_fwd"][live[s], rounds[s]] for s in pick])
        res = ask(pick, q)
        for i, s in enumerate(pick):
            d = live[s]
            got[d].append(tuple(x[i] for x in res))
            if len(got[d]) == stop[d]:
                if W:
                    hist[d] = eng.dialog_slot_history([s], W)[0]
                eng.dialog_leave([s])
                del live[s]
                assert eng.dialog_slots()[s] == -1
    assert mixed and reused
    return got, hist


def _single(eng, nb, d, W, ask_lockstep):
    """dialog d alone in a vd_dialog_begin session, asked its R questions: each ask's results and the history after it"""
    R = nb["ques_fwd"].shape[1]
    eng.dialog_begin(Batch(_rows(nb, [d])), W, MAX_ANS)
    res, hists = [], []
    for r in range(R):
        out = ask_lockstep(nb["ques_fwd"][[d], r])
        res.append(tuple(x[0] for x in out))
        hists.append(eng.dialog_history(W)[0] if W else None)
    return res, hists


def _same(a, b):
    return len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize("size", sorted(SIZES))
@pytest.mark.parametrize("enc", ALL_ENCODERS)
def test_fp32_mixed_rounds_equal_one_dialog_sessions(enc, size):
    s = SIZES[size]
    params, eng = _engine(enc, VD_MATH_FP32, s["V"], s["H"], s["E"], s["end_bias"])
    D = s["D"] + 2
    nb = small_batch(params, B=D, seed=7)
    R = nb["ques_fwd"].shape[1]
    W, k, L, V = _W(params, nb), s["k"], s["L"], s["V"]
    got, hist = _drive(eng, nb, max(2, D // 3), W,
                       lambda slots, q: eng.dialog_ask_beam_slots(slots, q, k, L, V - 1, V), seed=D)
    want = {d: _single(eng, nb, d, W, lambda q: eng.dialog_ask_beam(q, k, L, V - 1, V)) for d in range(D)}
    for d in range(D):
        n = len(got[d])
        for r in range(n):
            assert _same(got[d][r], want[d][0][r]), (d, r)
        if W:
            assert np.array_equal(hist[d], want[d][1][n - 1] * (np.arange(R) <= min(n, R - 1))[:, None]), d
    if params["useHistory"]:                       # the dataset's questions: vd_gen_dialog_beam_search's rows
        ans, length, score, _ = eng.gen_dialog_beam_search(Batch(nb), k, L, V - 1, V, W, MAX_ANS)
        for d in range(D):
            for r, (a, n, sc) in enumerate(want[d][0]):
                i = d * R + r
                assert np.array_equal(a, ans[i]) and n == length[i] and sc == score[i], (d, r)
    eng.close()


@pytest.mark.parametrize("enc", ["lf-ques-hist", "hrea-ques-im-hist", "mn-att-ques-im-hist"])
def test_fp32_mixed_rounds_sampling_equals_dialog_sample(enc):
    V, L, T, r0 = 256, 8, 0.9, 21
    params, eng = _engine(enc, VD_MATH_FP32, V, 128, 64, 2.0)
    D = 6
    nb = small_batch(params, B=D, seed=7)
    R = nb["ques_fwd"].shape[1]
    W = _W(params, nb)
    ans, logp, _ = eng.gen_dialog_sample(Batch(nb), L, V - 1, V, T, SEED, r0, W, MAX_ANS)
    got, _ = _drive(eng, nb, 3, W, lambda slots, q: eng.dialog_ask_sample_slots(slots, q, L, V - 1, V, T, SEED, r0), seed=3,
                    draw_base=[d * R for d in range(D)])
    for d in range(D):
        for r, (a, lp) in enumerate(got[d]):
            assert np.array_equal(a, ans[d * R + r]) and np.array_equal(lp, logp[d * R + r]), (d, r)
    eng.close()


@pytest.mark.parametrize("enc", ["lf-ques-im-hist", "hrea-ques-im-hist", "mn-att-ques-im-hist"])
def test_fp32_mixed_rounds_pool_equals_answer_pool_dialog(enc):
    params, eng, nb = _pool_engine(enc, VD_MATH_FP32, B=6)
    R = nb["ques_fwd"].shape[1]
    W = _W(params, nb)
    idx, score, _ = eng.answer_pool_dialog(Batch(nb), 3, W, MAX_ANS)
    got, _ = _drive(eng, nb, 3, W, lambda slots, q: eng.dialog_ask_pool_slots(slots, q, 3), seed=5)
    for d in range(6):
        for r, (i, s) in enumerate(got[d]):
            assert np.array_equal(i, idx[d * R + r]) and np.array_equal(s, score[d * R + r]), (d, r)
    eng.close()


@pytest.mark.parametrize("mode", [VD_MATH_TF32, VD_MATH_F16], ids=["tf32", "f16"])
@pytest.mark.parametrize("enc", ["lf-ques-hist", "hre-ques-im-hist", "hrea-ques-im-hist", "mn-att-ques-im-hist"])
def test_tensor_core_mixed_rounds(enc, mode):
    """Each mixed-round ask's answers are host_beam_search's from the ask's own state; each row's encoding is within
    5e-3 of vd_encoder_forward on its conversation's own history rebuilt as a batch."""
    s = SIZES["tc"]
    params, eng = _engine(enc, mode, s["V"], s["H"], s["E"], s["end_bias"])
    D = 6
    nb = small_batch(params, B=D, seed=7)
    R = nb["ques_fwd"].shape[1]
    W, k, L, V = _W(params, nb), s["k"], s["L"], s["V"]

    def ask(slots, q):
        a, n, sc = eng.dialog_ask_beam_slots(slots, q, k, L, V - 1, V)
        enc_rows = eng.dialog_encoding().numpy()
        wa, wn, ws = host_beam_search(_AskView(eng), enc_rows, k, L, V - 1, V)
        assert np.array_equal(a, wa) and np.array_equal(n, wn) and np.array_equal(sc, ws)
        return a, n, sc, enc_rows

    got, hist = _drive(eng, nb, 3, W, ask, seed=11)
    checked = 0
    for d in range(D):
        if len(got[d]) < R:
            continue
        full = eng.encoder_forward(Batch(dict(_rows(nb, [d]), hist=hist[d][None].copy()))).numpy().reshape(R, -1)
        for r in range(R):
            within(got[d][r][3], full[r], 5e-3, "dialog %d round %d" % (d, r))
        checked += 1
    assert checked
    eng.close()


@pytest.mark.parametrize("enc", ["lf-ques-im-hist", "hre-ques-hist", "hrea-ques-im-hist", "mn-att-ques-im-hist"])
def test_launches_and_lstm_work_do_not_depend_on_the_mix_of_rounds(enc):
    """An ask's launch count depends on n and on whether a row is at round 0 or R-1, not on the other rounds; its LSTM
    FLOP classes are n rows of one round."""
    params, eng = _engine(enc, VD_MATH_FP32, 9, 32, 12, 1.0)
    nb = small_batch(params, B=6, seed=7)
    R, Tq = nb["ques_fwd"].shape[1:]
    W = _W(params, nb)
    eng.profile(True)
    eng.dialog_open(6, Tq, W, MAX_ANS)
    slots = eng.dialog_join(Batch(nb))
    eng.dialog_ask_beam_slots(slots[:1], nb["ques_fwd"][:1, 0], 3, 6, 8, 9)   # rounds (1, 0, 0, 0, 0, 0)
    for _ in range(3):
        eng.dialog_ask_beam_slots(slots[1:2], nb["ques_fwd"][:1, 0], 3, 6, 8, 9)   # slot 1 at round 3
    eng.dialog_ask_beam_slots(slots[2:3], nb["ques_fwd"][:1, 0], 3, 6, 8, 9)   # slot 2 at round 1

    def measure(sl):
        q = nb["ques_fwd"][:len(sl), 1]
        eng.profile_reset()
        n0 = eng.launch_count()
        eng.dialog_ask_beam_slots(sl, q, 3, 6, 8, 9)
        return eng.launch_count() - n0, sum(eng.kernel_stats(c)["flops"] for c in ("lstm_step", "lstm_step_small",
                                                                                   "lstm_step_first"))
    a = measure([slots[0], slots[1]])            # rounds 1 and 3
    b = measure([slots[2], slots[0]])            # rounds 1 and 2
    assert a == b, (a, b)
    eng.close()


def test_refusals_and_isolation():
    V = 9
    params, eng = _engine("hrea-ques-im-hist", VD_MATH_FP32, V, 32, 12, 1.0)
    nb = small_batch(params, B=4, seed=7)
    other = small_batch(params, B=5, seed=11)
    R, Tq = nb["ques_fwd"].shape[1:]
    W = _width(params, nb)
    q = nb["ques_fwd"][:2, 0]

    def ask(sl, qq=None):
        return eng.dialog_ask_beam_slots(sl, q if qq is None else qq, 3, 6, 8, 9)

    assert _code(ask, [0, 1]) == _lib.VD_E_STATE                                          # no session
    assert _code(eng.dialog_open, 0, Tq, W, MAX_ANS) == _lib.VD_E_SHAPE
    assert _code(eng.dialog_open, 3, Tq, Tq - 1, MAX_ANS) == _lib.VD_E_BADARG
    eng.dialog_open(3, Tq, W, MAX_ANS)
    assert _code(eng.dialog_join, Batch(nb)) == _lib.VD_E_STATE                             # 4 dialogs, 3 slots
    assert (eng.dialog_slots() == -1).all()
    slots = eng.dialog_join(Batch(_rows(nb, [0, 1])))
    assert slots.tolist() == [0, 1]
    assert _code(ask, [0, 2]) == _lib.VD_E_STATE                                          # slot 2 is free
    assert _code(ask, [0, 0]) == _lib.VD_E_BADARG                                         # named twice
    assert _code(ask, [0, 3]) == _lib.VD_E_BADARG                                         # outside [0, C)
    assert _code(eng.dialog_ask_beam_slots, [], q[:0], 3, 6, 8, 9) == _lib.VD_E_BADARG    # n < 1
    assert _code(ask, [0, 1], np.zeros((2, Tq + 1), np.int32)) == _lib.VD_E_SHAPE
    assert _code(ask, [0, 1], np.full((2, Tq), V + 1, np.int32)) == _lib.VD_E_BADARG
    assert _code(eng.dialog_ask_pool_slots, [0, 1], q, 1) == _lib.VD_E_STATE              # gen: no pool answerer
    assert _code(eng.dialog_leave, [2]) == _lib.VD_E_STATE
    assert _code(eng.dialog_round) == _lib.VD_E_STATE                                     # not every slot occupied
    assert eng.dialog_slots().tolist() == [0, 0, -1]                                      # nothing changed

    def session(interleave):
        eng.dialog_open(3, Tq, W, MAX_ANS)
        sl = eng.dialog_join(Batch(_rows(nb, [0, 1])))
        out = []
        for r in range(R):
            if interleave:                                # a refused ask, then other work: the next answers are unchanged
                assert _code(ask, sl[:1], nb["ques_fwd"][:1, 0] * 0 + V + 1) == _lib.VD_E_BADARG
                eng.encoder_forward(Batch(other))
                eng.gen_beam_search(2, 5, 8, 9)
            out.append(ask(sl, nb["ques_fwd"][:2, r]))
        assert _code(ask, sl[:1], nb["ques_fwd"][:1, 0]) == _lib.VD_E_STATE               # had R asks
        return out, eng.dialog_slot_history(sl, W)

    want, want_hist = session(False)
    got, hist = session(True)
    assert all(_same(g, w) for g, w in zip(got, want)) and np.array_equal(hist, want_hist)
    eng.set_parameters(eng.get_parameters())                                              # stale until reopened
    assert _code(ask, [0, 1]) == _lib.VD_E_STATE
    assert _code(eng.dialog_join, Batch(_rows(nb, [2]))) == _lib.VD_E_STATE
    eng.close()


# ---- the per-row kernels one by one ----------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def keng():
    e = Engine(small_params("lf-ques", "disc"))
    e.profile(True)
    yield e
    e.close()


@pytest.mark.parametrize("C,R,H", [(6, 10, 512), (5, 10, 32), (4, 32, 64)])
def test_per_row_attention(keng, C, R, H):
    """Row i reads facts 0..r_i of slot s_i only: equal (==) to the range kernel's row r_i of that slot, and to fp64, with
    NaN in every cache row it must not read (later rounds, free slots) and in the guard bands."""
    rng = np.random.default_rng(C * 100 + R + H)
    sc = (4.0 / H) ** 0.25
    facts = (rng.standard_normal((C, R, H)) * sc).astype(np.float32)
    shc = (rng.standard_normal((C, R)) * 2).astype(np.float32)
    slot = np.asarray([s for s in rng.permutation(C)[:C - 1]], np.int32)      # one slot stays free
    rnd = rng.integers(0, R, slot.size).astype(np.int32)
    rnd[0], rnd[-1] = 0, R - 1
    n = slot.size
    q = (rng.standard_normal((n, H)) * sc).astype(np.float32)
    sq = (rng.standard_normal(n) * 2).astype(np.float32)
    fn, sn = np.full_like(facts, np.nan), np.full_like(shc, np.nan)
    for i in range(n):
        fn[slot[i], :rnd[i] + 1] = facts[slot[i], :rnd[i] + 1]
        sn[slot[i], :rnd[i] + 1] = shc[slot[i], :rnd[i] + 1]
    pool = Pool(keng)
    try:
        for name, args, rng_name, rng_args in (
                ("mn", lambda o, p: [pool(q), pool(fn), p, o, pool(slot), pool(rnd)], "mn_attention_rows_fwd",
                 lambda i, o, p: [pool(q[i:i + 1]), pool(facts[slot[i]][None]), p, o]),
                ("hrea", lambda o, p: [pool(sq), pool(sn), pool(fn), p, o, pool(slot), pool(rnd)], "hrea_attention_rows_fwd",
                 lambda i, o, p: [pool(sq[i:i + 1]), pool(shc[slot[i]][None]), pool(facts[slot[i]][None]), p, o])):
            probs, out = pool.out((n, 1, R)), pool.out((n, H))
            n0 = keng.launch_count()
            check(call(keng, name + "_attention_slots_fwd", args(out, probs), [n, R, H, R * H]))
            assert keng.launch_count() == n0 + 1
            got = out.get()
            for i in range(n):
                p1, o1 = pool.out((1, 1, R)), pool.out((1, H))
                check(call(keng, rng_name, rng_args(i, o1, p1), [1, R, H, int(rnd[i]), int(rnd[i]) + 1, R * H]))
                assert np.array_equal(got[i], o1.get()[0]), (name, i)
                f64 = facts[slot[i], :rnd[i] + 1].astype(np.float64)
                if name == "mn":
                    v = f64 @ q[i].astype(np.float64)
                else:
                    v = sq[i] + shc[slot[i], :rnd[i] + 1].astype(np.float64)
                P = np.exp(v - v.max())
                P /= P.sum()
                within(got[i], P @ f64, 1e-5 * (1 + np.abs(f64).max()), "%s row %d" % (name, i))
            assert not np.isnan(probs.get()[:, 0]).any()
    finally:
        pool.free()


def test_per_row_cache_write_append_gather_and_scatter(keng):
    C, R, H, Tq, W, P = 5, 10, 48, 6, 14, 20
    rng = np.random.default_rng(9)
    slot = np.asarray([3, 0, 4], np.int32)
    rnd = np.asarray([2, 0, R - 1], np.int32)
    n = slot.size
    pool = Pool(keng)
    try:
        # cache write: facts and sh at (slot, round), the state rows at slot, one launch
        facts0, shc0 = rng.standard_normal((C, R, H)).astype(np.float32), rng.standard_normal((C, R)).astype(np.float32)
        sth0, stc0 = rng.standard_normal((C, H)).astype(np.float32), rng.standard_normal((C, H)).astype(np.float32)
        h3, sh = rng.standard_normal((n, H)).astype(np.float32), rng.standard_normal(n).astype(np.float32)
        hn, cn = rng.standard_normal((n, H)).astype(np.float32), rng.standard_normal((n, H)).astype(np.float32)
        f, s, th, tc = pool(facts0), pool(shc0), pool(sth0), pool(stc0)
        n0 = keng.launch_count()
        check(call(keng, "dialog_cache_write_slots", [f, s, pool(h3), pool(sh), pool(slot), pool(rnd), th, tc, pool(hn), pool(cn)],
                   [n, R, H]))
        assert keng.launch_count() == n0 + 1
        wf, ws, wh, wc = facts0.copy(), shc0.copy(), sth0.copy(), stc0.copy()
        wf[slot, rnd], ws[slot, rnd], wh[slot], wc[slot] = h3, sh, hn, cn
        assert np.array_equal(f.get(), wf) and np.array_equal(s.get(), ws)
        assert np.array_equal(th.get(), wh) and np.array_equal(tc.get(), wc)

        # the ask gather: questions into the cache and time-major ids, history rows, image product, state (zeros at round 0)
        q = rng.integers(0, 50, (n, Tq)).astype(np.int32)
        ques0 = rng.integers(0, 50, (C, R, Tq)).astype(np.int32)
        hist = rng.integers(0, 50, (C, R, W)).astype(np.int32)
        img = rng.standard_normal((C, P)).astype(np.float32)
        qc = pool(ques0)
        ids_q, ids_h = pool.out((Tq, n), np.int32), pool.out((W, n), np.int32)
        io, ho, co = pool.out((n, P)), pool.out((n, H)), pool.out((n, H))
        n0 = keng.launch_count()
        check(call(keng, "dialog_gather", [pool(slot), pool(rnd), pool(q), qc, ids_q, pool(hist), ids_h, pool(img), io,
                                           pool(sth0), pool(stc0), ho, co], [n, R, Tq, W, P, H]))
        assert keng.launch_count() == n0 + 1
        wq = ques0.copy()
        wq[slot, rnd] = q
        first = (rnd == 0)[:, None]
        assert np.array_equal(qc.get(), wq) and np.array_equal(ids_q.get(), q.T)
        assert np.array_equal(ids_h.get(), hist[slot, rnd].T) and np.array_equal(io.get(), img[slot])
        assert np.array_equal(ho.get(), np.where(first, 0, sth0[slot])) and np.array_equal(co.get(), np.where(first, 0, stc0[slot]))

        # the join's scatter of image products into slots
        dst = pool(img)
        src = rng.standard_normal((2, P)).astype(np.float32)
        check(call(keng, "scatter_rows", [dst, pool(src), pool(np.asarray([4, 1], np.int32))], [2, P]))
        wi = img.copy()
        wi[[4, 1]] = src
        assert np.array_equal(dst.get(), wi)

        # the per-row append: row r_i + 1 of slot s_i, nothing at round R-1, against the lockstep form on one dialog
        Wh = 16
        base = np.zeros((C, R, Wh), np.int32)
        for c in range(C):
            for r in range(R):
                base[c, r, Wh - 3:] = [c + 1, r + 1, 7]
        ques = rng.integers(1, 9, (C, R, Tq)).astype(np.int32)
        ans = rng.integers(1, 9, (n, 8)).astype(np.int32)
        hd = pool(base)
        n0 = keng.launch_count()
        check(call(keng, "hist_append_slots", [hd, pool(ques), pool(ans), None, pool(slot), pool(rnd)],
                   [n, R, Wh, 0, Tq, 8, 8, 9, 5, 1]))
        assert keng.launch_count() == n0 + 1
        got = hd.get()
        want = base.copy()
        for i in range(n):
            if rnd[i] == R - 1:
                continue
            one = pool(base[slot[i]][None].copy())
            qq = np.zeros((1, R, Tq), np.int32)
            qq[0, rnd[i]] = ques[slot[i], rnd[i]]
            check(call(keng, "hist_append_slots", [one, pool(qq), pool(ans[i:i + 1]), None, None, None],
                       [1, R, Wh, int(rnd[i]), Tq, 8, 8, 9, 5, 1]))
            want[slot[i]] = one.get()[0]
        assert np.array_equal(got, want)
    finally:
        pool.free()


def test_per_row_draw_rounds_equal_the_affine_rule(keng):
    """SampleCfg::row_round fed row_offset + r * row_stride draws what the affine rule draws, on both sampling routes."""
    rows, V, L, seed, step, off, stride = 100, 1000, 4, SEED, 3, 17, 10
    rng = np.random.default_rng(4)
    logits = (rng.standard_normal((rows, V)) * 3).astype(np.float32)
    drawn = (off + np.arange(rows) * stride).astype(np.int64)
    pool = Pool(keng)
    try:
        outs = []
        for name, extra in (("logsoftmax_sample_rows", []), ("logsoftmax_sample_rows_drawn", [pool(drawn, 0)])):
            tok, ans, lp = pool.out((rows,), np.int32), pool(np.zeros((rows, L + 1), np.int32)), pool.out((rows, L))
            check(call(keng, name, [pool(logits), tok, ans, lp] + extra, [rows, V, L, seed, step, off, stride], [0.8]))
            outs.append((tok.get(), ans.get(), lp.get()))
        assert all(np.array_equal(a, b, equal_nan=True) for a, b in zip(*outs))
        # the fused tensor-core epilogue: A (rows, K) x B (V, K)
        K = 64
        A = rng.standard_normal((rows, K)).astype(np.float32)
        Bm = (rng.standard_normal((V, K)) / 8).astype(np.float32)
        bias = rng.standard_normal(V).astype(np.float32)
        npart = pool(np.zeros(1, np.int32))
        check(call(keng, "vocab_lse_nparts", [npart], [V]))
        nparts = int(npart.get()[0])
        outs = []
        for name, extra in (("vocab_sample_tc", []), ("vocab_sample_tc_drawn", [pool(drawn, 0)])):
            parts = [pool.out((rows, nparts)) for _ in range(3)] + [pool.out((rows, nparts), np.int32), pool.out((rows, nparts))]
            check(call(keng, name, [pool(A), pool(Bm), pool(bias)] + parts + extra, [rows, V, K, K, K, seed, step, off, stride],
                       [0.8]))
            outs.append([p.get() for p in parts])
        assert all(np.array_equal(a, b, equal_nan=True) for a, b in zip(*outs))
    finally:
        pool.free()


# ---- the serve command -----------------------------------------------------------------------------------------------
from test_dialog_generation_gpu import command_files  # noqa: E402,F401  (the generate command's corpus and checkpoint)


def test_serve_answers_as_chat_questions(command_files, tmp_path):
    """Interleaved conversations piped into chat -serve 1 get the answers chat -questions gives each of them; refused
    lines and the automatic leave after maxQuesCount answers produce the specified lines."""
    import json
    import subprocess
    import sys

    from test_cli_gpu import _model
    from test_dialog_generation_gpu import ROOT
    from visdial_b200.checkpoint import load_checkpoint
    flags, fo, ckp = command_files
    n = 3
    common = [*flags, "-loadPath", ckp, "-maxThreads", n, "-math", "fp32", "-beamLen", 20]
    ck = load_checkpoint(ckp)
    m, dl = _model(ck["modelParams"], fo, "val", ck)
    from visdial_b200.chat import _image_index
    ids = list(_image_index(dl, "val"))[:n]
    ques = np.asarray(dl.getIndexData(np.arange(n), m.params, "val")["ques_fwd"])
    R = ques.shape[1]
    dl.close(); m.engine.close()
    asked = {str(i): [[int(t) for t in row if t] for row in ques[d]] for d, i in enumerate(ids)}
    qfile = tmp_path / "q.json"
    qfile.write_text(json.dumps(asked))
    r = subprocess.run([sys.executable, "-m", "visdial_b200.chat"] + [str(a) for a in common] +
                       ["-resultPath", str(tmp_path / "chat"), "-questions", str(qfile)], cwd=ROOT, capture_output=True,
                       text=True, timeout=1200)
    assert r.returncode == 0, r.stderr[-3000:]
    want = {str(d["image_id"]): d["dialog"] for d in json.load(open(str(tmp_path / "chat" / "results.json")))["data"]}
    lines = [{"id": "x", "question": "hello"},                                  # unknown id, no image: refused
             {"id": "y", "image_id": -5, "question": "hi"}]                     # unknown image: refused
    rng = np.random.default_rng(2)
    left = {i: list(asked[str(i)]) for i in ids}
    first = set()
    while any(left.values()):                                                   # interleaved, several per conversation
        i = [j for j in ids if left[j]][int(rng.integers(len([j for j in ids if left[j]])))]
        obj = {"id": "u%d" % i, "question": left[i].pop(0)}
        if i not in first:
            obj["image_id"] = i
            first.add(i)
        lines.append(obj)
    lines.insert(len(lines) - (len(lines) - 2) // 2, {"id": "z", "image_id": ids[0], "question": "hi"})   # the pool is full
    lines.append({"id": "v", "leave": True})                                     # never joined: unknown
    r = subprocess.run([sys.executable, "-m", "visdial_b200.chat"] + [str(a) for a in common] + ["-serve", "1", "-capacity", str(n)],
                       cwd=ROOT, input="".join(json.dumps(x) + "\n" for x in lines), capture_output=True, text=True,
                       timeout=1200)
    assert r.returncode == 0, r.stderr[-3000:]
    out = [json.loads(x) for x in r.stdout.splitlines() if x.startswith("{")]
    errors = [o for o in out if "error" in o]
    assert [o["id"] for o in errors] == ["x", "y", "z", "v"], errors
    assert "full" in errors[2]["error"] and "unknown id" in errors[3]["error"]
    got = {}
    for o in out:
        if "answer" in o:
            got.setdefault(o["id"], []).append(o)
    for i in ids:
        conv = got["u%d" % i]
        assert [o["answer"] for o in conv] == [x["answer"].strip() for x in want[str(i)]], i
        assert [o["round"] for o in conv] == list(range(R))
        assert conv[-1].get("done") is True and all("done" not in o for o in conv[:-1])
