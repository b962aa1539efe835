"""Deterministic training (vd_set_deterministic, DESIGN §27): the gradient reductions' routes without float atomics, one by
one against fp64 and bit for bit across launches and SM budgets; whole training steps bit for bit across fresh engines,
option overlap and SM reserves, in every math mode; the accuracy bounds of the default routes; the default's kernel list
after the mode is turned off again; and the train / finetune commands' checkpoints byte for byte."""
import ctypes as C
import hashlib
import os
import shutil

import numpy as np
import pytest
import torch

from test_dense_gpu import data  # noqa: F401  (the finetune command's data files and checkpoint)
from helpers import run, seg_slices, small_batch, small_params, torch_batch, torch_params
from oracle import philox
from oracle import visdial_oracle as O
from visdial_b200 import VD_MATH_F16, VD_MATH_FP32, VD_MATH_TF32, Batch, Engine, init_parameters
from visdial_b200.synthetic import make_batch

pytestmark = pytest.mark.gpu

MODES = {"fp32": VD_MATH_FP32, "tf32": VD_MATH_TF32, "f16": VD_MATH_F16}
BUDGETS = (132, 116, 92)
DET_KERNELS = ("k_slot_reduce", "k_tsort_hist", "k_tsort_fill", "k_segsum_det", "k_segsum_det_join")


def _ptr(t, off=0):
    return None if t is None else C.c_void_p(t.data_ptr() + t.element_size() * off)


@pytest.fixture(scope="module")
def eng():
    e = Engine(small_params("lf-ques", "disc", vocabSize=300))
    e.set_deterministic(True)
    yield e
    e.close()


def _budgets():
    n = torch.cuda.get_device_properties(0).multi_processor_count
    return [b for b in BUDGETS if b <= n]


# ---- 1. the routes, kernel by kernel ------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["tf32", "fp32"])
@pytest.mark.parametrize("M,N,K", [(512, 2048, 20000), (300, 1200, 4097), (33, 70, 6001), (128, 128, 64)])
def test_gemm_atb(eng, mode, M, N, K):
    """Engine::gemm_atb's deterministic route (k_tc_atb / k_gemm_atb into slots, then k_slot_reduce): C += A^T B against fp64
    with test_gemm_gpu's bound, and the same bits under every SM budget."""
    eng.set_math_mode(MODES[mode])
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N + K)
    A = torch.randn(K, M, device="cuda", generator=g)
    B = torch.randn(K, N, device="cuda", generator=g)
    if mode == "tf32":                    # TF32-exact operands: only the accumulation order separates the result from fp64
        A = (A.view(torch.int32) & ~0x1FFF).view(torch.float32)
        B = (B.view(torch.int32) & ~0x1FFF).view(torch.float32)
    C0 = torch.randn(M, N, device="cuda", generator=g)
    ref = C0.double() + A.double().T @ B.double()
    bound = (K + 40) * 2.0 ** -24 * (A.double().abs().T @ B.double().abs()) + 2.0 ** -24 * C0.double().abs()
    outs = []
    for b in _budgets() + [_budgets()[0]]:
        Cm = C0.clone()
        run(eng, "gemm_atb", [_ptr(A), None, _ptr(B), _ptr(Cm)], [M, N, K, M, N, N, b])
        torch.cuda.synchronize()
        outs.append(Cm)
    assert bool(((outs[0].double() - ref).abs() <= bound).all()), float((outs[0].double() - ref).abs().max())
    for o in outs[1:]:
        assert torch.equal(o, outs[0])


@pytest.mark.parametrize("M,N,K", [(512, 2048, 608000), (256, 1024, 30000), (64, 192, 4160), (128, 256, 64)])
def test_gemm_atb16(eng, M, N, K):
    """k_atb16's deterministic route (the chunk plan from the shape, partial tiles into k-range slots): against fp64 with
    test_atb16_streamk_gpu's bound (below the C4 option dWh shape, whose fp64 product is not formed here) and the same bits
    on every CTA count, including the C4 option dWh (512 x 2048, K = 608 000)."""
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    A = torch.randn(K, M, device="cuda", generator=g).half()
    B = torch.randn(K, N, device="cuda", generator=g).half()
    C0 = torch.randn(M, N, device="cuda", generator=g)
    inv = 0.5
    sc = torch.tensor([inv], device="cuda")
    outs = []
    for b in _budgets() + [_budgets()[0]]:
        Cm = C0.clone()
        run(eng, "gemm_atb16", [_ptr(A), _ptr(B), _ptr(Cm), _ptr(sc)], [M, N, K, M, N, N, b, 1, 1])
        torch.cuda.synchronize()
        outs.append(Cm)
    for o in outs[1:]:
        assert torch.equal(o, outs[0])
    if K <= 65536:
        ref = C0.double() + inv * (A.double().T @ B.double())
        err = float((outs[0].double() - ref).abs().max())
        assert err < 2e-6 * K * inv + 1e-5, err


def _stable_groups(ids, nv):
    perm = np.argsort(ids, kind="stable").astype(np.int32)
    return perm, ids[perm]


@pytest.mark.parametrize("n", [1, 31, 2048, 2049, 70001])
def test_group_rows_by_token_is_stable(eng, n):
    rng = np.random.default_rng(n)
    nv = 301
    ids = rng.integers(0, nv, n).astype(np.int32)
    ids[: n // 2] = 0                       # a long run of pads spans many sort blocks
    d_ids = torch.from_numpy(ids).cuda()
    scratch = torch.zeros(3 * nv, dtype=torch.int32, device="cuda")
    perm = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    stok = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    run(eng, "group_rows_by_token", [_ptr(d_ids), _ptr(scratch), _ptr(perm), _ptr(stok)], [n, nv])
    rp, rt = _stable_groups(ids, nv)
    assert np.array_equal(perm.cpu().numpy(), rp) and np.array_equal(stok.cpu().numpy(), rt)


@pytest.mark.parametrize("n,ncols", [(1, 4), (255, 64), (257, 2048), (9000, 300), (70001, 128)])
@pytest.mark.parametrize("half", [False, True])
def test_segsum_rows(eng, n, ncols, half):
    """segsum_rows / segsum_rows16's deterministic route: out[tok] += scale * (sum of the token's rows in sorted order),
    tokens spanning several blocks included; against fp64, and the same bits twice."""
    if half and ncols % 8:
        pytest.skip("segsum_rows16 takes multiples of 8 columns")
    rng = np.random.default_rng(n + ncols)
    nv = 301
    ids = rng.integers(0, nv, n).astype(np.int32)
    ids[: n // 3] = 7
    perm, stok = _stable_groups(ids, nv)
    X = torch.randn(n, ncols, device="cuda")
    if half:
        X = X.half()
    inv = torch.tensor([0.25], device="cuda")
    out0 = torch.randn(nv, ncols, device="cuda")
    ref = out0.double().clone()
    ref.index_add_(0, torch.from_numpy(ids).long().cuda(), X.double() * (0.25 if half else 1.0))
    outs = []
    for _ in range(2):
        o = out0.clone()
        dp, dt = torch.from_numpy(perm).cuda(), torch.from_numpy(stok).cuda()
        if half:
            run(eng, "segsum_rows16", [_ptr(X), _ptr(dp), _ptr(dt), _ptr(o), _ptr(inv)], [ncols, n, ncols])
        else:
            run(eng, "segsum_rows", [_ptr(X), _ptr(dp), _ptr(dt), _ptr(o)], [ncols, n, ncols])
        outs.append(o)
    assert torch.equal(outs[0], outs[1])
    cnt = np.bincount(ids, minlength=nv).max()
    err = float((outs[0].double() - ref).abs().max())
    assert err < (cnt + 2) * 2.0 ** -23 * float(ref.abs().max() + 1) * 4, err


@pytest.mark.parametrize("rows,E,ldx", [(1, 12, 12), (3000, 300, 600), (12800, 64, 64)])
def test_embed_scatter_add(eng, rows, E, ldx):
    """embed_scatter_add's deterministic route (stable sort + ordered segmented sum) with dropout factors, against fp64."""
    nv = 301
    rng = np.random.default_rng(rows)
    ids = rng.integers(0, nv, rows).astype(np.int32)
    ids[::3] = 0
    dx = torch.randn(rows, ldx, device="cuda")
    demb0 = torch.randn(nv, E, device="cuda")
    eng.set_training(1)
    eng.set_dropout_seed(11, 3)
    outs = []
    for _ in range(2):
        o = demb0.clone()
        run(eng, "embed_scatter_add", [_ptr(o), _ptr(dx), _ptr(torch.from_numpy(ids).cuda())], [ldx, rows, E, 0], [0.0])
        outs.append(o)
    assert torch.equal(outs[0], outs[1])
    ref = demb0.double().clone()
    ref.index_add_(0, torch.from_numpy(ids).long().cuda(), dx[:, :E].double())
    assert float((outs[0].double() - ref).abs().max()) < 1e-4 * max(1.0, float(ref.abs().max())) * np.sqrt(rows)
    # with dropout p = 0.5: the two launches agree bit for bit
    outs = []
    for _ in range(2):
        o = demb0.clone()
        run(eng, "embed_scatter_add", [_ptr(o), _ptr(dx), _ptr(torch.from_numpy(ids).cuda())], [ldx, rows, E, 1], [0.5])
        outs.append(o)
    assert torch.equal(outs[0], outs[1])
    eng.set_training(0)


@pytest.mark.parametrize("rows,cols", [(1, 3), (1000, 2048), (777, 301)])
def test_colsum_and_rowdot(eng, rows, cols):
    X = torch.randn(rows, cols, device="cuda")
    out0 = torch.randn(cols, device="cuda")
    outs = []
    for _ in range(2):
        o = out0.clone()
        run(eng, "colsum_add", [_ptr(o), _ptr(X)], [rows, cols, cols])
        outs.append(o)
    assert torch.equal(outs[0], outs[1])
    ref = out0.double() + X.double().sum(0)
    assert float((outs[0].double() - ref).abs().max()) < (rows + 2) * 2.0 ** -24 * float(X.double().abs().sum(0).max() + 1)
    ds = torch.randn(rows, device="cuda")
    w = torch.randn(cols, device="cuda")
    res = []
    for _ in range(2):
        dx = torch.zeros(rows, cols, device="cuda")
        dw = out0.clone()
        db = torch.zeros(1, device="cuda")
        run(eng, "rowdot_bwd", [_ptr(ds), _ptr(X), _ptr(w), _ptr(dx), _ptr(dw), _ptr(db)], [0, rows, cols])
        res.append((dw, db))
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])
    ref = out0.double() + (ds.double()[:, None] * X.double()).sum(0)
    bound = (rows + 2) * 2.0 ** -24 * float((ds.double().abs()[:, None] * X.double().abs()).sum(0).max() + 1)
    assert float((res[0][0].double() - ref).abs().max()) < bound
    assert abs(float(res[0][1]) - float(ds.double().sum())) < (rows + 2) * 2.0 ** -24 * float(ds.abs().sum() + 1)


# ---- 2. whole steps -------------------------------------------------------------------------------------------------------
STEP_CASES = [("lf-ques", {}), ("hre-ques-im-hist", {}), ("hrea-ques-im-hist", {}), ("mn-att-ques-im-hist", {}),
              ("mn-att-ques-im-hist", {"imgRegions": 5})]


def _params(enc, dec, extra):
    # H = 256 and 13 dialogs x 10 options: the fp16 option LSTM, the persistent encoder pair (with its gate split at
    # H % 128 == 0) and the stream-K weight gradient all engage in VD_MATH_F16
    return small_params(enc, dec, rnnHiddenSize=256, embedSize=64, vocabSize=200, numOptions=10, commonEmbeddingSize=64,
                        imgFeatureSize=64, imgSpatialSize=4, imgEmbedSize=32, **extra)


def _digest(eng):
    W = eng.get_parameters()
    m, v, _ = eng.optim_state()
    return tuple(hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest() for a in (W, m, v))


def _train(p, mode, overlap=True, reserve=16, steps=3, kind="plain"):
    flat = init_parameters(p, seed=3)
    eng = Engine(p)
    eng.set_math_mode(mode)
    eng.set_option_overlap(overlap, reserve)
    eng.set_deterministic(True)
    eng.set_parameters(flat)
    eng.set_training(1)
    losses = []
    B = 13
    for it in range(steps):
        nb = make_batch(p, B, seed=7 + it, max_ques_len=9, max_ans_len=6, max_cap_len=12, max_hist_len=14, empty_round_every=4,
                        gen_eval=kind == "dense_gen")
        eng.set_dropout_seed(11, it + 1)
        eng.zero_grad()
        if kind == "plain":
            loss = eng.forward_backward(Batch(nb))
        else:
            rng = np.random.default_rng(it)
            rounds = rng.integers(0, p["maxQuesCount"], B).astype(np.int32)
            rel = rng.random((B, p["numOptions"])).astype(np.float32)
            f = eng.forward_backward_dense if kind == "dense" else eng.forward_backward_dense_gen
            loss = f(Batch(nb), rounds, rel)
        losses.append(np.float32(loss).tobytes())
        eng.clamp_adam_step(1e-3)
    d = (tuple(losses),) + _digest(eng)
    eng.close()
    return d


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("dec", ["disc", "gen"])
@pytest.mark.parametrize("enc,extra", STEP_CASES)
def test_steps_repeat_bit_for_bit(enc, extra, dec, mode):
    p = _params(enc, dec, extra)
    a = _train(p, MODES[mode])
    assert _train(p, MODES[mode]) == a, "two fresh engines"
    assert _train(p, MODES[mode], overlap=False) == a, "option overlap off"
    assert _train(p, MODES[mode], reserve=0) == a, "reserve 0"


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("dec", ["disc", "gen"])
def test_dense_steps_repeat_bit_for_bit(dec, mode):
    p = _params("hre-ques-im-hist", dec, {})
    kind = "dense" if dec == "disc" else "dense_gen"
    a = _train(p, MODES[mode], kind=kind)
    assert _train(p, MODES[mode], kind=kind) == a
    assert _train(p, MODES[mode], overlap=False, kind=kind) == a
    assert _train(p, MODES[mode], reserve=0, kind=kind) == a


# ---- 3. accuracy: the default routes' bounds --------------------------------------------------------------------------------
@pytest.mark.parametrize("enc,dec", [("lf-ques", "gen"), ("hre-ques-im-hist", "disc"), ("hrea-ques-im-hist", "gen"),
                                     ("mn-att-ques-im-hist", "disc")])
def test_parity_with_the_oracle_fp32(enc, dec):
    """test_parity_gpu's training-step bounds against the oracle, in deterministic mode"""
    from test_parity_gpu import ITER, SEED, _compare_grads, _run_engine
    p = small_params(enc, dec)
    flat = init_parameters(p, seed=3)
    nb = small_batch(p, B=3)
    eng = _run_engine(p, flat, nb, VD_MATH_FP32, 1)
    eng.set_deterministic(True)
    loss = eng.forward_backward(Batch(nb))
    g = eng.get_gradients()
    eng.close()
    ref = O.forward_backward(O.Ctx(train=True, mask_fn=philox.make_mask_fn(SEED, ITER, {O.SITE_FUSION: p["dropout"]})), p,
                             torch_params(p, flat), torch_batch(nb))
    assert abs(loss - ref["loss"]) <= 1e-4 * max(1.0, abs(ref["loss"])), (loss, ref["loss"])
    _compare_grads(p, g, ref["grads"], 2e-5, 2e-4)


@pytest.mark.parametrize("mode", [VD_MATH_FP32, VD_MATH_TF32, VD_MATH_F16])
def test_c4_b32_fixture(mode):
    """test_c4_b32_gpu's training-step bounds against tests/golden/c4_b32__*.npz at B = 32, in deterministic mode"""
    from test_c4_b32_gpu import FIX, TOL, _setup
    fx, tol = np.load(FIX), TOL[mode]
    p, nb, eng = _setup(fx, mode)
    eng.set_deterministic(True)
    eng.set_training(1)
    eng.set_dropout_seed(int(fx["drop_seed"]), int(fx["drop_iter"]))
    eng.zero_grad()
    loss = eng.forward_backward(Batch(nb))
    g = eng.get_gradients().astype(np.float64)
    eng.close()
    ref_loss = float(fx["train_loss"])
    assert abs(loss - ref_loss) < tol["loss"] * abs(ref_loss), (loss, ref_loss)
    stride = int(fx["stride"])
    sample, ref, idx = g[::stride], fx["grad_sample"], np.arange(0, g.size, stride)
    sl = seg_slices(p)
    for name, amax, nrm in zip(fx["seg_names"], fx["seg_absmax"], fx["seg_norm"]):
        if amax < 1e-9:
            continue
        s = sl[str(name)]
        m = (idx >= s.start) & (idx < s.stop)
        if m.any():
            assert float(np.abs(sample[m] - ref[m]).max() / amax) < tol["grad"], name
        assert abs(float(np.sqrt((g[s] ** 2).sum())) - nrm) / nrm < tol["norm"], name


# ---- 4. off is off ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", list(MODES))
def test_off_is_the_default(mode):
    p = _params("mn-att-ques-im-hist", "disc", {})
    nb = make_batch(p, 13, seed=7, max_ques_len=9, max_ans_len=6, max_cap_len=12, max_hist_len=14, empty_round_every=4)
    counts = []
    for toggle in (False, True):
        eng = Engine(p)
        eng.set_math_mode(MODES[mode])
        eng.set_parameters(init_parameters(p, seed=3))
        eng.set_training(1)
        if toggle:
            eng.set_deterministic(True)
            eng.zero_grad()
            eng.forward_backward(Batch(nb))
            eng.set_deterministic(False)
        eng.zero_grad()
        eng.profile(True)
        eng.profile_reset()
        n0 = eng.launch_count()
        eng.forward_backward(Batch(nb))
        counts.append((eng.launch_count() - n0, [eng.kernel_stats(k)["launches"] for k in DET_KERNELS],
                       eng.kernel_stats("k_atb16")["launches"], eng.kernel_stats("embed_scatter_add")["launches"]))
        eng.close()
    assert counts[0] == counts[1], counts
    assert counts[0][1] == [0] * len(DET_KERNELS)


# ---- 5. the commands ----------------------------------------------------------------------------------------------------------
def _twice(run, mod, save, *args):
    got = []
    for _ in range(2):
        run(mod, *args, "-savePath", save)
        got.append({f: open(os.path.join(save, f), "rb").read() for f in sorted(os.listdir(save))})
        shutil.rmtree(save)
    assert got[0] and got[0] == got[1], mod


def test_train_checkpoints_are_byte_identical(tmp_path):
    import test_cli_gpu as T
    enc, dec = "hre-ques-im-hist", "disc"
    d = tmp_path / "data"
    d.mkdir()
    flags, _ = T.write_files(str(d), enc, dec)
    p = T._params(enc, dec)
    _twice(T._run, "train", tmp_path / "run", *T._size_flags(p), *flags, "-batchSize", 4, "-numEpochs", 1, "-saveIter", 1,
           "-math", "f16", "-deterministic", 1)


def test_finetune_checkpoints_are_byte_identical(data, tmp_path):
    import test_dense_gpu as D
    _, flags, ann, ck = data
    _twice(D._run, "finetune", tmp_path / "run", *flags, "-loadPath", ck, "-denseAnnotations", ann["train"], "-numEpochs", 1,
           "-saveIter", 1, "-batchSize", 4, "-math", "tf32", "-deterministic", 1)


# ---- 6. two GPUs --------------------------------------------------------------------------------------------------------------
def test_refused_with_a_communicator():
    """One GPU only: vd_set_deterministic(e, 1) with world > 1 and vd_comm_init(world > 1) on a deterministic engine are
    refused with VD_E_STATE (needs no second GPU: the refusal comes before any NCCL call)."""
    e = Engine(small_params("lf-ques", "disc"))
    e.set_deterministic(True)
    idb = (C.c_uint8 * 128)()
    rc = e.lib.vd_comm_init(e.h, idb, 0, 2)
    assert rc == -6, rc
    e.set_deterministic(False)
    e.close()
