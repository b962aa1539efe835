"""Answer-pool retrieval (vd_answer_pool_*, DESIGN §18): the fused score + top-k kernels on both routes against the numpy
reference (tests/pool_topk_ref.py) on small-integer operands, which TF32 and fp32 both score exactly; the pool encoding
against the oracle's fp64 SeqLSTM; the pool scores against the 100-option path; the model-level top-k against fp64;
refusals; and the dialog loop on retrieved answers against a host loop."""
import ctypes as C

import numpy as np
import pytest
import torch

from dialog_history import right_aligned, row_words, next_row
from helpers import Buf, call, run, seg_slices, small_batch, small_params
from oracle import visdial_oracle as O
from pool_topk_ref import pool_topk, topk_rows
from visdial_b200 import VD_MATH_F16, VD_MATH_FP32, VD_MATH_TF32, init_parameters
from visdial_b200 import _lib
from visdial_b200.engine import Batch, Engine

pytestmark = pytest.mark.gpu

MODES = [VD_MATH_FP32, VD_MATH_TF32, VD_MATH_F16]
MODE_IDS = ["fp32", "tf32", "f16"]
# bound on a disc score against fp64 (DESIGN §18): §7's per-element bounds (FP32 2e-5, tensor-core modes 5e-3) on the pool
# embedding carried through the dot product, i.e. times sum_h |encOut[n, h]| (at least 1)
SCORE_TOL = {VD_MATH_FP32: 2e-5, VD_MATH_TF32: 5e-3, VD_MATH_F16: 5e-3}
GUARD = 64


def _disc_engine(enc="mn-att-ques-im-hist", mode=VD_MATH_FP32, seed=5, **kw):
    params = small_params(enc, "disc", **kw)
    eng = Engine(params)
    eng.set_math_mode(mode)
    eng.set_training(0)
    flat = init_parameters(params, seed=seed)
    eng.set_parameters(flat)
    return params, eng, flat


def _pool_tokens(rng, m, w, V):
    """left-aligned rows of 1..w words, zero-padded, as opt_list stores them"""
    tok = np.zeros((m, w), np.int32)
    lens = rng.integers(1, w + 1, m)
    for j in range(m):
        tok[j, :lens[j]] = rng.integers(1, V + 1, lens[j])
    return tok


# ---- 1. kernel exactness -------------------------------------------------------------------------------------------
M_CASES = [1, 63, 64, 65, 127, 128, 129, 1000, 100003]
ROW_CASES = [1, 10, 127, 128, 129, 1280]
K_CASES = [1, 4, 5, 8, 16, 32]


def _topk_call(eng, Q, E, k, ldq):
    rows, H = Q.shape
    m = E.shape[0]
    qimg = np.full((GUARD + rows * ldq + GUARD), np.nan, np.float32)
    qimg[GUARD:GUARD + rows * ldq].reshape(rows, ldq)[:, :H] = Q
    eimg = np.full((m + 2) * H, np.nan, np.float32)        # two NaN rows after the pool: never scored
    eimg[:m * H] = E.ravel()
    qb, eb = Buf(eng, qimg), Buf(eng, eimg)
    vb = Buf(eng, np.full(GUARD + rows * k + GUARD, np.nan, np.float32))
    ib = Buf(eng, np.full(GUARD + rows * k + GUARD, -7, np.int32))
    run(eng, "answer_pool_topk", [qb.ptr(GUARD), eb, vb.ptr(GUARD), ib.ptr(GUARD)], [rows, ldq, m, H, k])
    v, i = vb.get(), ib.get()
    for b in (qb, eb, vb, ib):
        b.free()
    assert np.isnan(v[:GUARD]).all() and np.isnan(v[GUARD + rows * k:]).all(), "stray write into the score guard bands"
    assert (i[:GUARD] == -7).all() and (i[GUARD + rows * k:] == -7).all(), "stray write into the index guard bands"
    return i[GUARD:GUARD + rows * k].reshape(rows, k), v[GUARD:GUARD + rows * k].reshape(rows, k)


@pytest.fixture(scope="module")
def kernel_engine():
    params, eng, _ = _disc_engine(rnnHiddenSize=64)
    yield eng
    eng.close()


CASES = [(m, rows, K_CASES[(a + b) % len(K_CASES)]) for a, m in enumerate(M_CASES) for b, rows in enumerate(ROW_CASES)
         if not (m == 100003 and rows == 1280)] + [(100003, 1280, 32), (100003, 129, 1)]


@pytest.mark.parametrize("route", ["tc", "simt"])
@pytest.mark.parametrize("m,rows,k", CASES)
def test_topk_exact(kernel_engine, m, rows, k, route):
    eng = kernel_engine
    k = min(k, m)
    H = 64
    rng = np.random.default_rng(m * 7 + rows * 131 + k)
    Q = rng.integers(-2, 3, (rows, H)).astype(np.float32)      # small integers: every dot product is exact
    E = rng.integers(-2, 3, (m, H)).astype(np.float32)
    eng.set_math_mode(VD_MATH_TF32 if route == "tc" else VD_MATH_FP32)
    eng.profile(True)
    eng.profile_reset()
    i, v = _topk_call(eng, Q, E, k, H + 4)
    assert eng.kernel_stats("pool_topk" if route == "tc" else "pool_topk_simt")["launches"] == 1
    assert eng.kernel_stats("pool_topk_simt" if route == "tc" else "pool_topk")["launches"] == 0
    assert eng.kernel_stats("pool_topk_rows")["launches"] == 1
    eng.profile(False)
    ri, rv = pool_topk(Q, E, k)
    assert np.array_equal(i, ri), "indices"
    assert np.array_equal(v.astype(np.float64), rv), "scores"
    i2, v2 = _topk_call(eng, Q, E, k, H + 4)                   # run to run: bit-identical
    assert np.array_equal(i, i2) and np.array_equal(v.view(np.int32), v2.view(np.int32))


@pytest.mark.parametrize("route", ["tc", "simt"])
def test_topk_all_ties(kernel_engine, route):
    """every score equal: the answer is the k lowest pool indices, across every tile, chunk and slot"""
    eng = kernel_engine
    eng.set_math_mode(VD_MATH_TF32 if route == "tc" else VD_MATH_FP32)
    Q = np.ones((129, 64), np.float32)
    E = np.ones((5000, 64), np.float32)
    i, v = _topk_call(eng, Q, E, 32, 64)
    assert (i == np.arange(32)[None]).all() and (v == 64).all()


# ---- 2. pool encoding against the oracle -------------------------------------------------------------------------
ENC_TOL = {VD_MATH_FP32: 2e-5, VD_MATH_TF32: 3e-3, VD_MATH_F16: 1e-2}


@pytest.mark.parametrize("mode", MODES, ids=MODE_IDS)
def test_pool_encoding(mode):
    params, eng, flat = _disc_engine(mode=mode, vocabSize=60, embedSize=32, rnnHiddenSize=256)
    rng = np.random.default_rng(3)
    m, w = 1100, 6                                              # >= 1 024 rows: the fp16 route runs in F16
    tok = _pool_tokens(rng, m, w, params["vocabSize"])
    eng.profile(True)
    eng.answer_pool_encode(tok)
    assert eng.kernel_stats("pool_encode")["launches"] == 1
    # the option LSTM's route: the fp16 step kernels in F16 (1 100 rows in one chunk), fp32 operands otherwise
    assert (eng.kernel_stats("k_lstm16")["launches"] > 0) == (mode == VD_MATH_F16)
    got = eng.answer_pool().numpy()
    sl = seg_slices(params)
    E_, H = params["embedSize"], params["rnnHiddenSize"]
    emb = flat[sl["wordEmbed.weight"]].reshape(-1, E_).astype(np.float64)
    emb[0] = 0
    W = torch.from_numpy(flat[sl["opt.lstm.weight"]].reshape(E_ + H, 4 * H).astype(np.float64))
    b = torch.from_numpy(flat[sl["opt.lstm.bias"]].astype(np.float64))
    x = torch.from_numpy(emb[tok.T])                            # (T, m, E), no maskzero (disc.lua:4-5)
    out, _ = O.seq_lstm(x, W, b)
    ref = out[-1].numpy()
    err = np.abs(got - ref).max()
    assert err <= ENC_TOL[mode], err
    eng.close()


# ---- 3. consistency with the 100-option path ---------------------------------------------------------------------
def _batch_pool(nb):
    """the distinct option rows of a disc batch, in first-seen order, and each option's pool index"""
    opts = nb["options"]
    flat = opts.reshape(-1, opts.shape[-1])
    uniq, first, inv = np.unique(flat, axis=0, return_index=True, return_inverse=True)
    order = np.argsort(first)
    rank = np.empty_like(order)
    rank[order] = np.arange(len(order))
    return uniq[order].astype(np.int32), rank[inv.ravel()].reshape(opts.shape[:-1])


@pytest.mark.parametrize("mode", MODES, ids=MODE_IDS)
def test_pool_scores_match_option_scores(mode):
    params, eng, _ = _disc_engine(mode=mode, rnnHiddenSize=256, embedSize=32, vocabSize=60)
    nb = small_batch(params, B=4, seed=11)
    pool, where = _batch_pool(nb)
    eng.answer_pool_encode(pool)
    emb = eng.answer_pool().numpy().astype(np.float64)
    enc = eng.encoder_forward(Batch(nb)).numpy().astype(np.float64)
    scores = eng.decoder_forward(Batch(nb)).numpy().astype(np.float64)
    N, K = scores.shape
    mine = np.einsum("nh,nkh->nk", enc, emb[where.reshape(N, K)])
    tol = SCORE_TOL[mode] * np.abs(enc).sum(1, keepdims=True).clip(min=1.0)
    assert (np.abs(mine - scores) <= tol).all(), float(np.abs(mine - scores).max())
    idx, sc = eng.answer_pool_retrieve(Batch(nb), 1)
    assert (sc[:, 0] >= scores.max(1) - tol[:, 0]).all()
    eng.close()


# ---- 4. model-level top-k against fp64 ---------------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES, ids=MODE_IDS)
def test_retrieve_against_fp64(mode):
    params, eng, _ = _disc_engine(mode=mode, rnnHiddenSize=128, embedSize=32, vocabSize=60)
    rng = np.random.default_rng(5)
    tok = _pool_tokens(rng, 3000, 5, params["vocabSize"])
    dup = [7, 1500, 2999]
    tok = np.concatenate([tok, tok[dup]])                       # rows 3000.. duplicate rows 7, 1500, 2999
    eng.answer_pool_encode(tok)
    emb = eng.answer_pool().numpy().astype(np.float64)
    nb = small_batch(params, B=6, seed=3)
    k = 8
    idx, sc = eng.answer_pool_retrieve(Batch(nb), k)
    enc = eng.encoder_forward(Batch(nb)).numpy().astype(np.float64)
    s64 = enc @ emb.T
    bound = SCORE_TOL[mode] * np.abs(enc).sum(1).clip(min=1.0)
    N = s64.shape[0]
    assert idx.shape == (N, k) and (idx >= 0).all() and (idx < len(tok)).all()
    assert (np.abs(sc - np.take_along_axis(s64, idx, 1)) <= bound[:, None]).all()
    for n in range(N):                                          # order: (returned score desc, index asc), exactly
        for j in range(k - 1):
            assert sc[n, j] > sc[n, j + 1] or (sc[n, j] == sc[n, j + 1] and idx[n, j] < idx[n, j + 1])
    ri, rv = topk_rows(s64, k + 1)
    near = 0
    for n in range(N):
        if abs(rv[n, k - 1] - rv[n, k]) <= 2 * bound[n]:
            near += 1
            continue
        assert set(idx[n]) == set(ri[n, :k]), n
    print("rows with a near tie at the k-th place: %d of %d" % (near, N))
    for n in range(N):
        for a, b in zip(dup, range(3000, 3003)):
            row = list(idx[n])
            if b in row:
                assert a in row and row.index(b) == row.index(a) + 1 and sc[n, row.index(a)] == sc[n, row.index(b)]
    eng.close()


# ---- 5. refusals -------------------------------------------------------------------------------------------------
def _code(fn):
    with pytest.raises(_lib.VdError) as e:
        fn()
    return e.value.code


def test_refusals():
    params, eng, flat = _disc_engine(rnnHiddenSize=64)
    V = params["vocabSize"]
    nb = small_batch(params, B=2, seed=1)
    tok = _pool_tokens(np.random.default_rng(0), 20, 4, V)
    assert _code(lambda: eng.answer_pool_retrieve(Batch(nb), 1)) == _lib.VD_E_STATE          # no pool
    assert _code(lambda: eng.answer_pool()) == _lib.VD_E_STATE
    for bad in (V + 1, -1):
        t = tok.copy()
        t[3, 1] = bad
        assert _code(lambda: eng.answer_pool_encode(t)) == _lib.VD_E_BADARG
    assert _code(lambda: eng.answer_pool_encode(np.zeros((3, 0), np.int32))) == _lib.VD_E_BADARG
    assert _code(lambda: eng.answer_pool_encode(np.zeros((0, 4), np.int32))) == _lib.VD_E_BADARG
    eng.answer_pool_encode(tok)
    for k in (0, 21, 33):
        assert _code(lambda: eng.answer_pool_retrieve(Batch(nb), k)) == _lib.VD_E_BADARG
    eng.answer_pool_retrieve(Batch(nb), 20)
    stale = [lambda: eng.set_parameters(flat), lambda: eng.set_math_mode(VD_MATH_TF32),
             lambda: (eng.zero_grad(), eng.clamp_adam_step(1e-3))]
    for act in stale:
        eng.answer_pool_encode(tok)
        eng.answer_pool_retrieve(Batch(nb), 1)
        act()
        assert _code(lambda: eng.answer_pool_retrieve(Batch(nb), 1)) == _lib.VD_E_STATE
    eng.close()
    gparams = small_params("mn-att-ques-im-hist", "gen")
    geng = Engine(gparams)
    assert _code(lambda: geng.answer_pool_encode(tok)) == _lib.VD_E_STATE
    assert _code(lambda: geng.answer_pool_retrieve(Batch(small_batch(gparams, B=2)), 1)) == _lib.VD_E_STATE
    geng.close()
    params, eng, _ = _disc_engine(enc="lf-ques-im")                                           # no history
    eng.answer_pool_encode(tok)
    nb = small_batch(params, B=2)
    assert _code(lambda: eng.answer_pool_dialog(Batch(nb), 1, 20, 5)) == _lib.VD_E_STATE
    eng.close()


# ---- 6. dialog loop against a host loop --------------------------------------------------------------------------
ENCODERS = ["lf-ques-hist", "hre-ques-im-hist", "hrea-ques-im-hist", "mn-ques-hist", "mn-att-ques-im-hist"]
MAX_ANS = 5


def _pool_words(row, end):
    out = []
    for t in row:
        if t == end:
            break
        if t != 0:
            out.append(int(t))
    return out


def _host_dialog(eng, params, nb, pool, k, W, mal):
    B, R = nb["ques_fwd"].shape[:2]
    end = params["vocabSize"]
    hist = np.zeros((B, R, W), np.int32)
    for b in range(B):
        hist[b, 0] = right_aligned(row_words(nb["hist"][b, 0]), W)
    idx = np.zeros((B, R, k), np.int32)
    sc = np.zeros((B, R, k), np.float32)
    for r in range(R):
        i, s = eng.answer_pool_retrieve(Batch(dict(nb, hist=hist.copy())), k)
        idx[:, r], sc[:, r] = i.reshape(B, R, k)[:, r], s.reshape(B, R, k)[:, r]
        if r + 1 < R:
            for b in range(B):
                hist[b, r + 1] = next_row(hist[b, r], row_words(nb["ques_fwd"][b, r]), _pool_words(pool[idx[b, r, 0]], end),
                                          params["concatHistory"], end, W, mal)
    return idx.reshape(B * R, k), sc.reshape(B * R, k), hist


@pytest.mark.parametrize("mode", MODES, ids=MODE_IDS)
@pytest.mark.parametrize("enc", ENCODERS)
def test_dialog_matches_host_loop(enc, mode):
    params, eng, _ = _disc_engine(enc=enc, mode=mode, vocabSize=30, rnnHiddenSize=64, embedSize=16)
    nb = small_batch(params, B=5, seed=7)
    pool = _pool_tokens(np.random.default_rng(2), 300, MAX_ANS, params["vocabSize"])
    eng.answer_pool_encode(pool)
    W = 30 if params["concatHistory"] else nb["ques_fwd"].shape[2] + MAX_ANS
    got = eng.answer_pool_dialog(Batch(nb), 3, W, MAX_ANS)
    want = _host_dialog(eng, params, nb, pool, 3, W, MAX_ANS)
    for g, w, name in zip(got, want, ("index", "score", "history")):
        assert g.shape == w.shape and np.array_equal(g, w), name
    assert not np.array_equal(got[2][:, 1:, -nb["hist"].shape[2]:], nb["hist"][:, 1:])
    eng.close()


def test_dialog_per_call_invariance():
    params, eng, _ = _disc_engine(enc="hre-ques-im-hist", mode=VD_MATH_FP32)
    nb = small_batch(params, B=8, seed=9)
    pool = _pool_tokens(np.random.default_rng(4), 100, MAX_ANS, params["vocabSize"])
    eng.answer_pool_encode(pool)
    W = nb["ques_fwd"].shape[2] + MAX_ANS
    whole = eng.answer_pool_dialog(Batch(nb), 2, W, MAX_ANS)
    R = params["maxQuesCount"]
    for b in range(8):
        one = eng.answer_pool_dialog(Batch({key: v[b:b + 1] if v.shape[0] == 8 else v[b * R:(b + 1) * R]
                                            for key, v in nb.items()}), 2, W, MAX_ANS)
        assert np.array_equal(one[0], whole[0][b * R:(b + 1) * R]) and np.array_equal(one[2][0], whole[2][b])
        assert np.array_equal(one[1].view(np.int32), whole[1][b * R:(b + 1) * R].view(np.int32))
    eng.close()


# ---- 7. the generate command on a disc checkpoint ------------------------------------------------------------------
def _run(*args):
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "visdial_b200.generate"] + [str(a) for a in args], cwd=root,
                       capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, (r.stdout[-3000:], r.stderr[-3000:])


@pytest.fixture(scope="module")
def disc_command_files(tmp_path_factory):
    from test_cli_gpu import _params, write_files
    from visdial_b200.model import Model
    d = tmp_path_factory.mktemp("pool_cli")
    flags, fo = write_files(str(d), "hrea-ques-im-hist", "disc")
    p = _params("hrea-ques-im-hist", "disc")
    m = Model(p, seed=1234)
    m.engine.set_parameters(init_parameters(p, seed=5))
    ckp = str(d / "model.t7")
    m.save(ckp, final=True)
    m.engine.close()
    return flags, fo, ckp


@pytest.mark.parametrize("history", ["gt", "generated"])
def test_generate_command_disc(disc_command_files, tmp_path, history):
    import json
    from test_cli_gpu import _model, _texts
    from visdial_b200.checkpoint import load_checkpoint
    flags, fo, ckp = disc_command_files
    _run(*flags, "-loadPath", ckp, "-resultPath", tmp_path / "vis", "-maxThreads", 6, "-math", "fp32", "-history", history,
         "-dialogsPerCall", 3)
    res = json.load(open(str(tmp_path / "vis" / "results.json")))
    assert res["opts"]["history"] == history
    ck = load_checkpoint(ckp)
    m, dl = _model(ck["modelParams"], fo, "val", ck)
    answers = m.retrieveAnswers(dl, "val", {"maxThreads": 6, "history": history, "dialogsPerCall": 3})
    pool = dl.answerPool("val")
    want = _texts(answers, dl.ind2word)
    for a in answers:                                     # each answer is its pool row's words, best first in topK
        for x in a["dialog"]:
            assert x["answer"] == [int(t) for t in pool[x["index"]] if t != 0] and x["topK"][0]["index"] == x["index"]
    with pytest.raises(ValueError):
        m.generateAnswers(dl, "val", {"maxThreads": 1})   # generateAnswers keeps refusing disc models (model.lua:434-437)
    dl.close(); m.engine.close()
    assert res["data"] == want and len(want) == 6 and all(len(a["dialog"]) == 10 for a in want)


def test_generate_command_disc_two_gpus_writes_the_one_gpu_file(disc_command_files, tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    flags, fo, ckp = disc_command_files
    for history in ("gt", "generated"):
        outs = []
        for n in (1, 2):
            res = tmp_path / ("gen_%s_%d" % (history, n))
            _run(*flags, "-loadPath", ckp, "-resultPath", res, "-maxThreads", 5, "-math", "fp32", "-history", history,
                 "-gpus", n)
            outs.append((res / "results.json").read_bytes())
        assert outs[0] == outs[1], history
