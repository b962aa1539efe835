"""Dialog sessions (vd_dialog_*, DESIGN §19): B dialogs asked one round at a time, each ask encoding only the new round over
the session's cached facts, image products and dialog-LSTM state.  Fed the batch's own questions, a session must give what
vd_gen_dialog_beam_search / vd_gen_dialog_sample / vd_answer_pool_dialog give on that batch: bit for bit in VD_MATH_FP32,
and in the tensor-core modes each round's encoding within §7's bound of vd_encoder_forward on the session's own history,
with the session's history rows the history rule applied to its own answers."""
import numpy as np
import pytest

from dialog_history import beam_words, next_row, right_aligned, row_words
from helpers import Pool, call, check, small_batch, small_params, within
from host_decode import host_beam_search
from test_dialog_generation_gpu import MAX_ANS, SEED, _engine, _width
from visdial_b200 import VD_MATH_F16, VD_MATH_FP32, VD_MATH_TF32
from visdial_b200 import _lib
from visdial_b200.engine import Batch, Engine

pytestmark = pytest.mark.gpu

ENCODERS = ["lf-ques-hist", "hre-ques-hist", "hre-ques-im-hist", "hrea-ques-im-hist", "mn-ques-hist", "mn-ques-im-hist",
            "mn-att-ques-im-hist"]
SIZES = {"small": dict(V=9, H=32, E=12, D=3, k=3, L=8, end_bias=1.0),
         "tc": dict(V=256, H=128, E=64, D=8, k=5, L=12, end_bias=4.0)}
U = 2.0 ** -24


def _session_beam(eng, nb, W, k, L, V, mal=MAX_ANS):
    """Opens a session on nb and asks its own questions round by round; returns the (B*R, ...) outputs like
    vd_gen_dialog_beam_search's, the history and each round's encoding."""
    B, R = nb["ques_fwd"].shape[:2]
    eng.dialog_begin(Batch(nb), W, mal)
    outs, encs = [], []
    for r in range(R):
        assert eng.dialog_round() == (r, B)
        outs.append(eng.dialog_ask_beam(nb["ques_fwd"][:, r], k, L, V - 1, V))
        encs.append(eng.dialog_encoding().numpy())
    hist = eng.dialog_history(W)
    stacked = [np.stack([o[i] for o in outs], 1).reshape((B * R,) + outs[0][i].shape[1:]) for i in range(3)]
    return stacked, hist, encs


@pytest.mark.parametrize("size", sorted(SIZES))
@pytest.mark.parametrize("enc", ENCODERS)
def test_fp32_session_equals_dialog_beam_search(enc, size):
    s = SIZES[size]
    params, eng = _engine(enc, VD_MATH_FP32, s["V"], s["H"], s["E"], s["end_bias"])
    nb = small_batch(params, B=s["D"], seed=7)
    W = _width(params, nb)
    want = eng.gen_dialog_beam_search(Batch(nb), s["k"], s["L"], s["V"] - 1, s["V"], W, MAX_ANS)
    got, hist, _ = _session_beam(eng, nb, W, s["k"], s["L"], s["V"])
    for g, w, name in zip(got + [hist], want, ("answer", "length", "score", "history")):
        assert g.shape == w.shape and np.array_equal(g, w), name
    assert (want[1] > 0).any()
    with pytest.raises(_lib.VdError) as e:                    # full: an eleventh ask is refused
        eng.dialog_ask_beam(nb["ques_fwd"][:, 0], s["k"], s["L"], s["V"] - 1, s["V"])
    assert e.value.code == _lib.VD_E_STATE
    eng.close()


def test_fp32_session_pad_question_and_short_rows():
    """A question of pads mid-dialog writes no Q or A (and empties later rows); questions asked narrower than the batch's
    width are right-aligned into it."""
    params, eng = _engine("hrea-ques-im-hist", VD_MATH_FP32, 9, 32, 12, 0.0)
    nb = small_batch(params, B=3, seed=7)
    nb["ques_fwd"][1, 3] = 0
    W = _width(params, nb)
    want = eng.gen_dialog_beam_search(Batch(nb), 2, 8, 8, 9, W, MAX_ANS)
    B, R, Tq = nb["ques_fwd"].shape
    eng.dialog_begin(Batch(nb), W, MAX_ANS)
    outs = []
    for r in range(R):
        q = nb["ques_fwd"][:, r]
        n = max(1, int(np.count_nonzero(q, 1).max()))
        outs.append(eng.dialog_ask_beam(q[:, Tq - n:], 2, 8, 8, 9))           # only the words' columns
    for i, name in enumerate(("answer", "length", "score")):
        got = np.stack([o[i] for o in outs], 1).reshape(want[i].shape)
        assert np.array_equal(got, want[i]), name
    assert np.array_equal(eng.dialog_history(W), want[3]) and not want[3][1, 4:].any()
    eng.close()


@pytest.mark.parametrize("enc", ["lf-ques-hist", "hrea-ques-im-hist", "mn-att-ques-im-hist"])
def test_fp32_session_equals_dialog_sample(enc):
    V, L, T, r0 = 256, 8, 0.9, 21
    params, eng = _engine(enc, VD_MATH_FP32, V, 128, 64, 2.0)
    nb = small_batch(params, B=4, seed=7)
    B, R = nb["ques_fwd"].shape[:2]
    W = _width(params, nb)
    ans, logp, hist = eng.gen_dialog_sample(Batch(nb), L, V - 1, V, T, SEED, r0, W, MAX_ANS)
    eng.dialog_begin(Batch(nb), W, MAX_ANS)
    for r in range(R):
        a, lp = eng.dialog_ask_sample(nb["ques_fwd"][:, r], L, V - 1, V, T, SEED, r0)
        assert np.array_equal(a, ans.reshape(B, R, L + 1)[:, r]), r
        assert np.array_equal(lp, logp.reshape(B, R, L)[:, r]), r
    assert np.array_equal(eng.dialog_history(W), hist)
    eng.close()


def _pool_engine(enc, mode, B=4, m=300, w=MAX_ANS):
    params, eng = _engine(enc, mode, 64, 64, 32, 0.0, dec="disc")
    rng = np.random.default_rng(5)
    pool = rng.integers(1, 65, (m, w)).astype(np.int32)
    pool[::7, 3:] = 0
    eng.answer_pool_encode(pool)
    return params, eng, small_batch(params, B=B, seed=7)


@pytest.mark.parametrize("enc", ["lf-ques-im-hist", "hrea-ques-im-hist", "mn-att-ques-im-hist"])
def test_fp32_session_equals_answer_pool_dialog(enc):
    params, eng, nb = _pool_engine(enc, VD_MATH_FP32)
    B, R = nb["ques_fwd"].shape[:2]
    W = _width(params, nb)
    idx, score, hist = eng.answer_pool_dialog(Batch(nb), 3, W, MAX_ANS)
    eng.dialog_begin(Batch(nb), W, MAX_ANS)
    for r in range(R):
        i, s = eng.dialog_ask_pool(nb["ques_fwd"][:, r], 3)
        assert np.array_equal(i, idx.reshape(B, R, 3)[:, r]) and np.array_equal(s, score.reshape(B, R, 3)[:, r]), r
    assert np.array_equal(eng.dialog_history(W), hist)
    eng.close()


@pytest.mark.parametrize("mode", [VD_MATH_FP32, VD_MATH_TF32, VD_MATH_F16], ids=["fp32", "tf32", "f16"])
@pytest.mark.parametrize("enc", ["lf-ques", "lf-ques-im"])
def test_encoders_without_history(enc, mode):
    """No history: round r's encoding is vd_encoder_forward's row r of the batch (FP32 bitwise)."""
    params, eng = _engine(enc, mode, 256, 128, 64, 2.0)
    nb = small_batch(params, B=5, seed=7)
    B, R = nb["ques_fwd"].shape[:2]
    full = eng.encoder_forward(Batch(nb)).numpy().reshape(B, R, -1)
    eng.dialog_begin(Batch(nb), 0, 0)
    for r in range(R):
        eng.dialog_ask_beam(nb["ques_fwd"][:, r], 3, 6, 255, 256)
        e = eng.dialog_encoding().numpy()
        if mode == VD_MATH_FP32:
            assert np.array_equal(e, full[:, r]), r
        else:
            within(e, full[:, r], 5e-3, "round %d encoding" % r)
    eng.close()


class _AskView:
    """The engine as tests/host_decode.py sees it after an ask: forwardConnect's start state is the ask's own
    (vd_dialog_rnn_state, and vd_dialog_encoding as encOut)."""

    class _Rows:
        def __init__(self, a):
            self.a = a

        def numpy(self):
            return self.a

    def __init__(self, eng):
        self.eng = eng
        self.state = [tuple(None if t is None else t.numpy() for t in eng.dialog_rnn_state(level)) for level in range(2)]

    def __getattr__(self, name):
        return getattr(self.eng, name)

    def encoder_rnn_state(self, level, rows):
        h, c = self.state[level]
        if h is None:
            return None, None
        assert h.shape[0] == rows
        return self._Rows(h), self._Rows(c)


@pytest.mark.parametrize("size", sorted(SIZES))
@pytest.mark.parametrize("mode", [VD_MATH_TF32, VD_MATH_F16], ids=["tf32", "f16"])
@pytest.mark.parametrize("enc", ENCODERS)
def test_tensor_core_session(enc, mode, size):
    """Each round's answers equal host_decode.host_beam_search started from the ask's own state (encoding and
    question-LSTM state), bit for bit; each round's encoding is within §7's bound of vd_encoder_forward on the session's
    own history rebuilt as a batch; the history rows are the history rule applied to the session's answers."""
    s = SIZES[size]
    params, eng = _engine(enc, mode, s["V"], s["H"], s["E"], s["end_bias"])
    nb = small_batch(params, B=s["D"], seed=7)
    B, R = nb["ques_fwd"].shape[:2]
    W, V, k, L = _width(params, nb), s["V"], s["k"], s["L"]
    eng.dialog_begin(Batch(nb), W, MAX_ANS)
    ans, length, encs = [], [], []
    for r in range(R):
        a, n, sc = eng.dialog_ask_beam(nb["ques_fwd"][:, r], k, L, V - 1, V)
        enc_r = eng.dialog_encoding().numpy()
        wa, wn, ws = host_beam_search(_AskView(eng), enc_r, k, L, V - 1, V)
        assert np.array_equal(a, wa) and np.array_equal(n, wn) and np.array_equal(sc, ws), r
        ans.append(a); length.append(n); encs.append(enc_r)
    assert (np.stack(length) > 0).any()
    hist = eng.dialog_history(W)
    full = eng.encoder_forward(Batch(dict(nb, hist=hist.copy()))).numpy().reshape(B, R, -1)
    for r in range(R):
        within(encs[r], full[:, r], 5e-3, "round %d encoding" % r)
    want = np.zeros_like(hist)
    for b in range(B):
        want[b, 0] = right_aligned(row_words(nb["hist"][b, 0]), W)
        for r in range(R - 1):
            want[b, r + 1] = next_row(want[b, r], row_words(nb["ques_fwd"][b, r]), beam_words(ans[r][b], length[r][b]),
                                      params["concatHistory"], V, W, MAX_ANS)
    assert np.array_equal(hist, want)
    eng.close()


@pytest.mark.parametrize("enc", ["lf-ques-im-hist", "hrea-ques-im-hist", "mn-att-ques-im-hist"])
def test_launches_per_ask_do_not_grow_with_the_round(enc):
    params, eng = _engine(enc, VD_MATH_FP32, 9, 32, 12, 1.0)
    eng.profile(True)
    nb = small_batch(params, B=4, seed=7)
    eng.dialog_begin(Batch(nb), _width(params, nb), MAX_ANS)
    counts = []
    for r in range(nb["ques_fwd"].shape[1]):
        n0 = eng.launch_count()
        eng.dialog_ask_beam(nb["ques_fwd"][:, r], 3, 6, 8, 9)
        counts.append(eng.launch_count() - n0)
    # Round 0 of the dialog LSTM has no state to continue (the full forward's step 0 has none either): hre / hrea skip
    # its recurrent contraction there.  The last round appends nothing (there is no row R): one launch fewer.
    first = 1 if params["encoder"].startswith("hre") else 0
    assert len(set(counts[1:-1])) == 1 and counts[0] == counts[1] - first and counts[-1] == counts[1] - 1, counts
    eng.close()


LSTM_CLASSES = ("lstm_step", "lstm_step_small", "lstm_step_first")


@pytest.mark.parametrize("enc", ["lf-ques-im-hist", "hre-ques-hist", "hrea-ques-im-hist", "mn-att-ques-im-hist"])
def test_lstm_work_per_ask_is_one_round(enc):
    """The LSTM FLOP classes of an ask (disc: no decoder LSTM) are the same at every round and are 1/R of a full encoder
    forward's on the same batch: B question rows and B history rows per ask (and one dialog-LSTM step), not B*(r+1)."""
    params, eng, nb = _pool_engine(enc, VD_MATH_FP32, B=4)
    enc_nb = {k: v for k, v in nb.items() if k in ("ques_fwd", "hist", "img_feat")}     # no option LSTM in the forward
    B, R = nb["ques_fwd"].shape[:2]

    def lstm_flops():
        return sum(eng.kernel_stats(c)["flops"] for c in LSTM_CLASSES)

    W = _width(params, nb)
    eng.profile(True)
    eng.dialog_begin(Batch(nb), W, MAX_ANS)
    per_ask = []
    for r in range(R):
        eng.profile_reset()
        eng.dialog_ask_pool(nb["ques_fwd"][:, r], 1)
        per_ask.append(lstm_flops())
    eng.profile_reset()
    eng.encoder_forward(Batch(dict(enc_nb, hist=eng.dialog_history(W))))       # the same rows, all rounds at once
    full = lstm_flops()
    assert full > 0 and len(set(per_ask)) == 1 and per_ask[0] * R == full, (per_ask, full)
    eng.close()


@pytest.mark.parametrize("enc,dec", [("mn-att-ques-im-hist", "gen"), ("hrea-ques-im-hist", "disc")])
def test_other_calls_between_asks_leave_the_session_intact(enc, dec):
    """vd_encoder_forward, vd_gen_beam_search (gen) and vd_retrieve, vd_answer_pool_retrieve (disc) between two asks leave
    every later answer and the history as an uninterrupted session's."""
    if dec == "gen":
        params, eng = _engine(enc, VD_MATH_FP32, 9, 32, 12, 1.0)
        nb = small_batch(params, B=3, seed=7)

        def ask(q):
            return eng.dialog_ask_beam(q, 3, 8, 8, 9)
    else:
        params, eng, nb = _pool_engine(enc, VD_MATH_FP32, B=3)

        def ask(q):
            return eng.dialog_ask_pool(q, 3)
    other = small_batch(params, B=5, seed=11)
    W = _width(params, nb)
    R = nb["ques_fwd"].shape[1]

    def session(interleave):
        eng.dialog_begin(Batch(nb), W, MAX_ANS)
        got = []
        for r in range(R):
            got.append(ask(nb["ques_fwd"][:, r]))
            if interleave:
                eng.encoder_forward(Batch(other))
                if dec == "gen":
                    eng.gen_beam_search(2, 5, 8, 9)
                else:
                    eng.retrieve(Batch(other), use_gt=False)
                    eng.answer_pool_retrieve(Batch(other), 2)
        return got, eng.dialog_history(W)

    want, want_hist = session(False)
    got, hist = session(True)
    for g, w in zip(got, want):
        for x, y in zip(g, w):
            assert np.array_equal(x, y)
    assert np.array_equal(hist, want_hist)
    eng.close()


def test_refusals():
    V = 9
    params, eng = _engine("hrea-ques-im-hist", VD_MATH_FP32, V, 32, 12, 1.0)
    nb = small_batch(params, B=2, seed=7)
    W, Th, Tq = _width(params, nb), nb["hist"].shape[2], nb["ques_fwd"].shape[2]
    q = nb["ques_fwd"][:, 0]

    def code(fn, *a):
        try:
            fn(*a)
        except _lib.VdError as e:
            return e.code
        return _lib.VD_OK

    assert code(eng.dialog_ask_beam, q, 3, 6, 8, 9) == _lib.VD_E_STATE                     # no session
    assert code(eng.dialog_begin, Batch(nb), Th - 1, MAX_ANS) == _lib.VD_E_BADARG
    assert code(eng.dialog_begin, Batch(nb), W, 0) == _lib.VD_E_BADARG
    eng.dialog_begin(Batch(nb), W, MAX_ANS)
    assert code(eng.dialog_ask_pool, q, 1) == _lib.VD_E_STATE                               # gen: no pool answerer
    assert code(eng.dialog_ask_beam, np.zeros((2, Tq + 1), np.int32), 3, 6, 8, 9) == _lib.VD_E_SHAPE
    assert code(eng.dialog_ask_beam, np.full((2, Tq), V + 1, np.int32), 3, 6, 8, 9) == _lib.VD_E_BADARG
    assert code(eng.dialog_ask_beam, q, 33, 6, 8, 9) == _lib.VD_E_BADARG
    assert code(eng.dialog_ask_beam, q, 3, 6, 0, 9) == _lib.VD_E_BADARG
    assert eng.dialog_round() == (0, 2)                                                     # nothing changed
    eng.dialog_ask_beam(q, 3, 6, 8, 9)
    assert eng.dialog_round() == (1, 2)
    eng.set_math_mode(VD_MATH_FP32)                                                         # stale: refused until begin
    assert code(eng.dialog_ask_beam, nb["ques_fwd"][:, 1], 3, 6, 8, 9) == _lib.VD_E_STATE
    eng.dialog_begin(Batch(nb), W, MAX_ANS)
    eng.dialog_ask_beam(q, 3, 6, 8, 9)
    eng.set_parameters(eng.get_parameters())
    assert code(eng.dialog_ask_beam, nb["ques_fwd"][:, 1], 3, 6, 8, 9) == _lib.VD_E_STATE
    eng.dialog_begin(Batch(nb), W, MAX_ANS)
    with pytest.raises(ValueError):                                                         # B rows, no more, no fewer
        eng.dialog_ask_beam(nb["ques_fwd"][:1, 0], 3, 6, 8, 9)
    assert eng.dialog_round() == (0, 2)
    eng.dialog_end()
    assert code(eng.dialog_round) == _lib.VD_E_STATE
    eng.close()
    params, eng, nb = _pool_engine("hrea-ques-im-hist", VD_MATH_FP32, B=2)
    eng.dialog_begin(Batch(nb), _width(params, nb), MAX_ANS)
    assert code(eng.dialog_ask_beam, q, 3, 6, 8, 9) == _lib.VD_E_STATE                     # disc: no search
    eng.set_math_mode(VD_MATH_FP32)                                                         # stale pool and session
    assert code(eng.dialog_ask_pool, nb["ques_fwd"][:, 0], 1) == _lib.VD_E_STATE
    eng.close()


# ---- the round-range kernels, against fp64 and against the full-range kernel's rows ----------------------------------
@pytest.fixture(scope="module")
def keng():
    e = Engine(small_params("lf-ques", "disc"))
    e.profile(True)
    yield e
    e.close()


@pytest.mark.parametrize("B,R,H", [(8, 10, 512), (3, 10, 32), (2, 32, 64)])
def test_round_range_attention(keng, B, R, H):
    rng = np.random.default_rng(B * 100 + R + H)
    s = (4.0 / H) ** 0.25
    q = (rng.standard_normal((B, R, H)) * s).astype(np.float32)
    h = (rng.standard_normal((B, R, H)) * s).astype(np.float32)
    sq = (rng.standard_normal((B, R)) * 2).astype(np.float32)
    sh = (rng.standard_normal((B, R)) * 2).astype(np.float32)
    pool = Pool(keng)
    try:
        fp, fo = pool.out((B, R, R)), pool.out((B, R, H))
        check(call(keng, "mn_attention_fwd", [pool(q), pool(h), fp, fo], [B, R, H]))
        full_mn = fo.get()
        hp, ho = pool.out((B, R, R)), pool.out((B, R, H))
        check(call(keng, "hrea_attention_fwd", [pool(sq), pool(sh), pool(h), hp, ho], [B, R, H]))
        full_hrea = ho.get()
        for r in sorted({0, R // 2, R - 1}):
            hc = h.copy()
            hc[:, r + 1:] = np.nan                            # facts not cached yet: never read
            shc = sh.copy()
            shc[:, r + 1:] = np.nan
            h64 = h.astype(np.float64)
            probs, out = pool.out((B, 1, R)), pool.out((B, H))
            n0 = keng.launch_count()
            check(call(keng, "mn_attention_rows_fwd", [pool(np.ascontiguousarray(q[:, r])), pool(hc), probs, out],
                       [B, R, H, r, r + 1, R * H]))
            assert keng.launch_count() == n0 + 1
            got = out.get()
            assert np.array_equal(got, full_mn[:, r]), "mn row %d differs from the full kernel's" % r
            S = np.einsum("bc,bjc->bj", q[:, r].astype(np.float64), h64[:, :r + 1])
            P = np.exp(S - S.max(-1, keepdims=True))
            P /= P.sum(-1, keepdims=True)
            ref = np.einsum("bj,bjc->bc", P, h64[:, :r + 1])
            Sa = np.einsum("bc,bjc->bj", np.abs(q[:, r]).astype(np.float64), np.abs(h64[:, :r + 1]))
            bp = P * (2 * U * (H / 32 + 8) * Sa.max(-1, keepdims=True) + 8 * U * (R + 4))
            within(got, ref, np.einsum("bj,bjc->bc", bp, np.abs(h64[:, :r + 1])) + U * (R + 2) * np.abs(ref) + 1e-6,
                   "mn rows r=%d" % r)
            assert not probs.get()[:, 0, r + 1:].any()
            probs, out = pool.out((B, 1, R)), pool.out((B, H))
            check(call(keng, "hrea_attention_rows_fwd", [pool(np.ascontiguousarray(sq[:, r])), pool(shc), pool(hc), probs, out],
                       [B, R, H, r, r + 1, R * H]))
            got = out.get()
            assert np.array_equal(got, full_hrea[:, r]), "hrea row %d differs from the full kernel's" % r
            v = sq[:, r, None].astype(np.float64) + sh[:, :r + 1].astype(np.float64)
            P = np.exp(v - v.max(-1, keepdims=True))
            P /= P.sum(-1, keepdims=True)
            ref = np.einsum("bj,bjc->bc", P, h64[:, :r + 1])
            within(got, ref, 1e-5 * (1 + np.abs(h64).max()), "hrea rows r=%d" % r)
        assert call(keng, "mn_attention_rows_fwd", [pool(q[:, 0]), pool(h), pool.out((B, 1, R)), pool.out((B, H))],
                    [B, R, H, 2, 1, R * H]) == _lib.VD_E_BADARG
    finally:
        pool.free()


@pytest.mark.parametrize("hrea", [False, True])
def test_dialog_cache_write(keng, hrea):
    B, R, H = 5, 10, 96
    rng = np.random.default_rng(3)
    facts0 = rng.standard_normal((B, R, H)).astype(np.float32)
    sh0 = rng.standard_normal((B, R)).astype(np.float32)
    pool = Pool(keng)
    try:
        for r in (0, 4, R - 1):
            h3 = rng.standard_normal((B, H)).astype(np.float32)
            sh = rng.standard_normal(B).astype(np.float32)
            f, s = pool(facts0), pool(sh0)
            n0 = keng.launch_count()
            check(call(keng, "dialog_cache_write", [f, s if hrea else None, pool(h3), pool(sh) if hrea else None],
                       [B, R, H, r]))
            assert keng.launch_count() == n0 + 1                                  # one launch for every piece
            want_f, want_s = facts0.copy(), sh0.copy()
            want_f[:, r] = h3
            if hrea:
                want_s[:, r] = sh
            assert np.array_equal(f.get(), want_f) and np.array_equal(s.get(), want_s)
    finally:
        pool.free()


# ---- the chat command ------------------------------------------------------------------------------------------------
from test_dialog_generation_gpu import command_files  # noqa: E402,F401  (the generate command's corpus and checkpoint)


def test_chat_command_answers_as_generate_with_generated_history(command_files, tmp_path):
    """chat -questions fed the dataset's questions (as token ids) writes generate -history generated's results, and the
    text Model.openDialogs(...).ask returns."""
    import json
    import subprocess
    import sys

    from test_cli_gpu import _model
    from test_dialog_generation_gpu import ROOT
    from visdial_b200.checkpoint import load_checkpoint
    from visdial_b200.utils import idToWords
    flags, fo, ckp = command_files
    n = 3
    common = [*flags, "-loadPath", ckp, "-maxThreads", n, "-math", "fp32", "-beamLen", 20]

    def run(module, *args):
        r = subprocess.run([sys.executable, "-m", module] + [str(a) for a in common + list(args)], cwd=ROOT,
                           capture_output=True, text=True, timeout=1200)
        assert r.returncode == 0, (r.stdout[-3000:], r.stderr[-3000:])

    run("visdial_b200.generate", "-resultPath", tmp_path / "gen", "-history", "generated")
    gen = json.load(open(str(tmp_path / "gen" / "results.json")))["data"]
    ck = load_checkpoint(ckp)
    m, dl = _model(ck["modelParams"], fo, "val", ck)
    ques = np.asarray(dl.getIndexData(np.arange(n), m.params, "val")["ques_fwd"])
    asked = {str(g["image_id"]): [[int(t) for t in row if t] for row in ques[d]] for d, g in enumerate(gen)}
    qfile = tmp_path / "q.json"
    qfile.write_text(json.dumps(asked))
    session = m.openDialogs(dl, "val", range(n), {"beamSize": 5, "beamLen": 20})
    direct = [[] for _ in range(n)]
    for r in range(ques.shape[1]):
        for d, e in enumerate(session.ask([asked[str(g["image_id"])][r] for g in gen])):
            direct[d].append({"question": idToWords(e["question"], dl.ind2word), "answer": idToWords(e["answer"], dl.ind2word)})
    session.close()
    dl.close(); m.engine.close()
    run("visdial_b200.chat", "-resultPath", tmp_path / "chat", "-questions", qfile)
    chat = json.load(open(str(tmp_path / "chat" / "results.json")))
    assert [c["dialog"] for c in chat["data"]] == direct
    assert chat["data"] == gen
