"""The gen dense fine-tuning step (vd_forward_backward_dense_gen) against its fp64 reference (tests/dense_gen_oracle.py) in
the three math modes, its agreement with vd_gen_option_lhood, its decoder row counts, the d-logit chunking, repeatability,
refusals, the 2-GPU equivalence, and finetune_gen -> evaluate -> ndcg end to end."""
import ctypes as C
import json
import math
import os
import re

import numpy as np
import pytest
import torch

from dense_gen_oracle import forward_backward_dense_gen as dense_gen_ref
from dense_oracle import soft_xent
from helpers import Buf, run, seg_slices, small_batch, small_params, torch_batch, torch_params
from oracle import philox
from oracle import visdial_oracle as O
from test_dense_gpu import SEED, ITER, _free_port, _ndcg_numpy, _rel, _run, _targets
from test_dense_gpu import data  # noqa: F401  (the synthetic files gen_data adds a gen checkpoint to)
from visdial_b200 import VD_MATH_F16, VD_MATH_FP32, VD_MATH_TF32, Batch, Engine, VdError, init_parameters
from visdial_b200._lib import VD_E_BADARG, VD_E_SHAPE, VD_E_STATE
from visdial_b200.synthetic import make_batch

pytestmark = pytest.mark.gpu

ENCODERS = ("lf-ques", "hre-ques-im-hist", "hrea-ques-im-hist", "mn-att-ques-im-hist")
# TF32 / F16: B*K >= 64 option rows and V >= 256, V % 4 == 0: the fused vocabulary route.  FP32: the rows route.
MID = dict(rnnHiddenSize=128, embedSize=64, vocabSize=300, numOptions=10, commonEmbeddingSize=64, imgSpatialSize=4,
           imgEmbedSize=32)
F16 = dict(rnnHiddenSize=256, embedSize=64, vocabSize=300, numOptions=100, commonEmbeddingSize=64, imgFeatureSize=64,
           imgSpatialSize=4, imgEmbedSize=32)


def _case(enc, mode):
    if mode == VD_MATH_FP32:
        p = small_params(enc, "gen", vocabSize=300)
        nb = small_batch(p, B=3, gen_eval=True)
    else:
        p = small_params(enc, "gen", imgFeatureSize=64 if "att" in enc else 256, **MID) if mode == VD_MATH_TF32 else \
            small_params(enc, "gen", **F16)
        nb = make_batch(p, 13 if mode == VD_MATH_TF32 else 11, seed=7, max_ques_len=9, max_ans_len=6, max_cap_len=12,
                        max_hist_len=14, max_hist_concat=40, empty_round_every=2, gen_eval=True)
    return p, nb


def _edge_targets(p, nb):
    """_targets, then: dialog 1 annotated on its last round, which make_batch leaves empty (empty_round_every = 2) and
    whose options are made all-pad as the dataloader pads missing rounds; dialog 0's annotated round gets an empty option
    (<START> -> <END>, no word) and an all-pad option."""
    B, R, K = nb["ques_fwd"].shape[0], p["maxQuesCount"], p["numOptions"]
    rounds, rel = _targets(p, B)
    rounds[1] = R - 1
    assert not nb["ques_fwd"][1, R - 1].any()
    for key in ("option_in", "option_out"):
        nb[key][1, R - 1] = 0
        nb[key][0, rounds[0], 1] = 0
        nb[key][0, rounds[0], 2] = 0
    nb["option_in"][0, rounds[0], 1, 0] = p["vocabSize"] - 1
    nb["option_out"][0, rounds[0], 1, 0] = p["vocabSize"]
    rel[0, 1] = max(rel[0, 1], 0.5)
    return rounds, rel


def _engine(p, flat, mode, training=1):
    eng = Engine(p)
    eng.set_math_mode(mode)
    eng.set_parameters(flat)
    eng.set_training(training)
    eng.set_dropout_seed(SEED, ITER)
    eng.zero_grad()
    return eng


def _scores(eng, B, K):
    out = Buf(eng, np.zeros(B * K, np.float32))
    run(eng, "dense_scores", [out], [B * K])
    s = out.get().reshape(B, K)
    out.free()
    return s


@pytest.mark.parametrize("mode", [VD_MATH_FP32, VD_MATH_TF32, VD_MATH_F16], ids=["fp32", "tf32", "f16"])
@pytest.mark.parametrize("enc", ENCODERS)
def test_dense_gen_step_matches_reference(enc, mode):
    """Loss, the (B, K) scores and every parameter segment's gradient, dropout on, at test_dense_gpu's tolerances."""
    p, nb = _case(enc, mode)
    rounds, rel = _edge_targets(p, nb)
    flat = init_parameters(p, seed=3)
    B, K = len(rounds), p["numOptions"]
    eng = _engine(p, flat, mode)
    loss = eng.forward_backward_dense_gen(Batch(nb), rounds, rel)
    scores = _scores(eng, B, K)
    g = eng.get_gradients()
    eng.close()
    ctx = O.Ctx(train=True, mask_fn=philox.make_mask_fn(SEED, ITER, {O.SITE_FUSION: p["dropout"]}), structure="batched")
    ref = dense_gen_ref(ctx, p, torch_params(p, flat), torch_batch(nb), rounds, rel)
    rs = ref["scores"].numpy()
    assert (scores[1] == 0).all() and scores[0, 2] == 0 and rs[0, 1] != 0     # all-pad rows score 0, the empty option not
    if mode == VD_MATH_FP32:
        assert abs(loss - ref["loss"]) <= 1e-4 * max(1.0, abs(ref["loss"])), (loss, ref["loss"])
        assert float(np.abs(scores - rs).max()) <= 1e-4 * max(1.0, float(np.abs(rs).max()))
    else:
        assert abs(loss - ref["loss"]) < 5e-3 * max(1.0, abs(ref["loss"])), (loss, ref["loss"])
        assert float(np.abs(scores - rs).max()) < 5e-3 * max(1.0, float(np.abs(rs).max()))
    for name, s in seg_slices(p).items():
        r = ref["grads"][name].numpy().ravel()
        if mode == VD_MATH_FP32:
            scale = max(float(np.abs(r).max()), 1e-30)
            err = float(np.abs(g[s] - r).max())
            assert err <= 2e-5 + 2e-4 * scale, (name, err, scale)
        elif np.abs(r).max() >= 1e-7:
            assert _rel(g[s], r) < 3e-2, (name, _rel(g[s], r))


def _option_lhood(eng, nb, B, R, K):
    b = Batch(nb)
    assert eng.lib.vd_encoder_forward(eng.h, C.byref(b.c), None) == 0
    ptr = C.c_void_p()
    assert eng.lib.vd_gen_option_lhood(eng.h, C.byref(b.c), C.byref(ptr)) == 0
    out = np.empty(B * R * K, np.float32)
    assert eng.lib.vd_memcpy_d2h(eng.h, out.ctypes.data, ptr, out.nbytes) == 0
    return out.reshape(B, R, K)


@pytest.mark.parametrize("mode", [VD_MATH_FP32, VD_MATH_TF32], ids=["fp32", "tf32"])
@pytest.mark.parametrize("enc", ["hre-ques-im-hist", "mn-att-ques-im-hist"])
def test_scores_are_the_option_lhood_evaluate_ranks_by(enc, mode):
    """Dropout off: the step's scores are vd_gen_option_lhood's rows of the annotated rounds, and its loss is the soft
    cross-entropy of those rows."""
    p, nb = _case(enc, mode)
    rounds, rel = _edge_targets(p, nb)
    B, R, K = len(rounds), p["maxQuesCount"], p["numOptions"]
    eng = _engine(p, init_parameters(p, seed=3), mode, training=2)
    loss = eng.forward_backward_dense_gen(Batch(nb), rounds, rel)
    scores = _scores(eng, B, K)
    eng.set_training(0)
    lh = _option_lhood(eng, nb, B, R, K)[np.arange(B), rounds]
    eng.close()
    tol = 1e-5 if mode == VD_MATH_FP32 else 2e-3
    assert float(np.abs(scores - lh).max()) <= tol * max(1.0, float(np.abs(lh).max()))
    want = float(soft_xent(torch.tensor(lh, dtype=torch.float64), torch.tensor(rel, dtype=torch.float64)))
    assert loss == pytest.approx(want, rel=tol, abs=tol)


def test_decoder_runs_on_the_selected_rows_only():
    """Profiling counts (not timings): the decoder LSTM step classes and the two vocabulary passes do B * numOptions
    rows of work per time step.  B * K >= 4096 rows put the decoder steps in the lstm_step classes, apart from the
    encoder's 320-row steps."""
    p = small_params("hre-ques-im-hist", "gen", rnnHiddenSize=64, embedSize=32, vocabSize=256, numOptions=100,
                     imgFeatureSize=64, imgEmbedSize=32)
    B, K, H, V = 41, p["numOptions"], p["rnnHiddenSize"], p["vocabSize"]
    nb = make_batch(p, B, seed=7, max_ques_len=6, max_ans_len=4, max_cap_len=8, max_hist_len=9, gen_eval=True)
    To = nb["option_in"].shape[-1]
    rounds, rel = _targets(p, B)
    eng = _engine(p, init_parameters(p, seed=3), VD_MATH_TF32)
    eng.profile(True)
    eng.profile_reset()
    eng.forward_backward_dense_gen(Batch(nb), rounds, rel)
    eng.synchronize()
    st = {k: eng.kernel_stats(k)["flops"] for k in ("lstm_step", "lstm_step_bwd", "vocab_lse", "vocab_dlogits")}
    eng.close()
    rows = B * K
    per_step = 2.0 * rows * 4 * H * H                          # the recurrent contraction of B*K rows, H-wide input of layer 2
    assert st["lstm_step"] == 2 * To * per_step                # both layers start from a state: every step is recurrent
    assert st["lstm_step_bwd"] == 2 * (To - 1) * per_step
    assert st["vocab_lse"] == To * 2.0 * rows * V * H
    assert st["vocab_dlogits"] == To * 2.0 * rows * V * H


def _fp32_step(eng, nb, rounds, rel, chunk_bytes):
    run(eng, "dense_gen_chunk_bytes", [], [chunk_bytes])
    eng.zero_grad()
    eng.set_dropout_seed(SEED, ITER)
    loss = eng.forward_backward_dense_gen(Batch(nb), rounds, rel)
    return loss, _scores(eng, len(rounds), eng.params["numOptions"]), eng.get_gradients()


def test_chunking_and_repetition():
    """FP32: one time step of d-logits per chunk against every step at once, and a repeated step.  Loss and scores bit
    for bit; dW to re-association level (the weight-, bias- and embedding-gradient kernels accumulate with atomics, and
    dec.out's dW / db add up per chunk)."""
    p, nb = _case("lf-ques", VD_MATH_FP32)
    rounds, rel = _edge_targets(p, nb)
    eng = _engine(p, init_parameters(p, seed=3), VD_MATH_FP32)
    step = 4 * len(rounds) * p["numOptions"] * p["vocabSize"]
    runs = [_fp32_step(eng, nb, rounds, rel, c) for c in (step, 1 << 40, 1 << 40, 0)]
    eng.close()
    (l0, s0, g0) = runs[0]
    for l1, s1, g1 in runs[1:]:
        assert l1 == l0 and (s1 == s0).all()
        for name, s in seg_slices(p).items():
            assert float(np.abs(g1[s] - g0[s]).max()) <= 1e-6 * float(np.abs(g0[s]).max()) + 1e-12, name


def test_refusals_keep_the_engine_usable():
    p, nb = _case("lf-ques", VD_MATH_FP32)
    rounds, rel = _targets(p, 3)
    disc = Engine(small_params("lf-ques", "disc"))
    with pytest.raises(VdError) as e:
        disc.forward_backward_dense_gen(Batch(small_batch(small_params("lf-ques", "disc"), B=3)), rounds,
                                        np.ones((3, 7), np.float32))
    assert e.value.code == VD_E_STATE
    disc.close()
    eng = _engine(p, init_parameters(p, seed=3), VD_MATH_FP32)
    good = eng.forward_backward_dense_gen(Batch(nb), rounds, rel)
    no_opts = {k: v for k, v in nb.items() if k not in ("option_in", "option_out")}
    with pytest.raises(VdError) as e:
        eng.forward_backward_dense_gen(Batch(no_opts), rounds, rel)
    assert e.value.code == VD_E_SHAPE
    bad = [(np.array([0, -1, 2]), rel), (np.array([0, 10, 2]), rel)]
    for v in (-0.25, np.nan, np.inf):
        x = rel.copy()
        x[1, 3] = v
        bad.append((rounds, x))
    x = rel.copy()
    x[2] = 0
    bad.append((rounds, x))
    for r, x in bad:
        with pytest.raises(VdError) as e:
            eng.forward_backward_dense_gen(Batch(nb), r, x)
        assert e.value.code == VD_E_BADARG, (r, x)
    b = Batch(nb)
    loss = C.c_float()
    ok_r = np.ascontiguousarray(rounds, np.int32)
    ok_x = np.ascontiguousarray(rel, np.float32)
    for args in ((None, ok_r.ctypes.data, ok_x.ctypes.data), (C.byref(b.c), None, ok_x.ctypes.data),
                 (C.byref(b.c), ok_r.ctypes.data, None)):
        assert eng.lib.vd_forward_backward_dense_gen(eng.h, *args, C.byref(loss)) == VD_E_BADARG
    eng.zero_grad()
    assert eng.forward_backward_dense_gen(Batch(nb), rounds, rel) == good
    eng.close()


# ---- two GPUs -----------------------------------------------------------------------------------------------------------
def _mg_case(mode, gpuid):
    kw = F16 if mode != VD_MATH_FP32 else {}
    p = small_params("hre-ques-im-hist", "gen", gpuid=gpuid, **kw)
    nb = small_batch(p, B=4, seed=3, gen_eval=True)
    return p, nb, _targets(p, 4)


def _mg_worker(rank, world, port, mode, out):
    import torch.distributed as dist
    from visdial_b200 import dist as vdist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    p, full, (rounds, rel) = _mg_case(mode, rank)
    lo, hi = vdist.shard_range(4, rank, world)
    eng = _engine(p, init_parameters(p, seed=3), mode, training=2)
    vdist.attach_engine(eng, rank, world)
    eng.zero_grad()
    loss = eng.forward_backward_dense_gen(Batch(vdist.shard_batch(full, rank, world, p["maxQuesCount"])), rounds[lo:hi],
                                          rel[lo:hi])
    eng.clamp_adam_step(1e-3)
    w, g = eng.get_parameters(), eng.get_gradients()
    losses = vdist.gather_ranks(np.asarray([loss], dtype=np.float64), rank, world)
    if rank == 0:
        out.put((w, g, losses))
    eng.close()
    dist.destroy_process_group()


@pytest.mark.parametrize("mode", [VD_MATH_FP32, VD_MATH_TF32], ids=["fp32", "tf32"])
def test_two_gpus_match_one(mode):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_mg_worker, args=(r, 2, port, mode, q)) for r in range(2)]
    for pr in procs:
        pr.start()
    w2, g2, losses = q.get(timeout=300)
    for pr in procs:
        pr.join(timeout=60)
        assert pr.exitcode == 0
    p, full, (rounds, rel) = _mg_case(mode, 0)
    eng = _engine(p, init_parameters(p, seed=3), mode, training=2)
    loss1 = eng.forward_backward_dense_gen(Batch(full), rounds, rel)
    eng.clamp_adam_step(1e-3)
    w1, g1 = eng.get_parameters(), eng.get_gradients()
    eng.close()
    assert float(np.mean(losses)) == pytest.approx(loss1, rel=1e-5)
    scale = max(float(np.abs(g1).max()), 1e-30)
    tol = 1e-5 if mode == VD_MATH_FP32 else 5e-3
    assert float(np.abs(g2 - g1).max()) < tol * scale + 1e-7
    if mode == VD_MATH_FP32:
        assert float(np.abs(w2 - w1).max()) < 0.02 * 1e-3


# ---- commands -----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gen_data(data):
    """test_dense_gpu's synthetic files (its `data` fixture) with a gen checkpoint."""
    from visdial_b200 import Model
    d, flags, ann, _ = data
    p = small_params("lf-ques", "gen", vocabSize=40, numOptions=100, numEpochs=2, saveIter=1, batchSize=4)
    m = Model(p, seed=1234)
    ck = str(d / "gen.t7")
    m.save(ck, final=True)
    m.engine.close()
    return d, flags, ann, ck


def test_finetune_gen_evaluate_ndcg(gen_data, tmp_path):
    from visdial_b200.checkpoint import load_checkpoint
    d, flags, ann, ck = gen_data
    save = tmp_path / "run"
    r = _run("finetune_gen", *flags, "-loadPath", ck, "-denseAnnotations", ann["train"], "-numEpochs", 2, "-saveIter", 1,
             "-batchSize", 4, "-math", "fp32", "-savePath", save)
    n_ann = 24 - 2 - 1
    per_epoch = math.ceil(n_ann / 4)
    assert "\n%d iter per epoch." % per_epoch in r.stdout and "%d annotated rounds" % n_ann in r.stdout
    assert sorted(os.listdir(save)) == ["model_epoch_1.t7", "model_epoch_2.t7", "model_final.t7"]
    assert load_checkpoint(str(save / "model_epoch_1.t7"))["optims"]["t"] == per_epoch
    w0, w1 = load_checkpoint(ck)["modelW"], load_checkpoint(str(save / "model_final.t7"))["modelW"]
    assert np.abs(w1 - w0).max() > 0
    ranks = tmp_path / "ranks.json"
    _run("evaluate", *flags, "-loadPath", save / "model_final.t7", "-split", "val", "-saveRanks", "-saveRankPath", ranks,
         "-math", "fp32")
    r = _run("ndcg", "-ranks", ranks, "-denseAnnotations", ann["val"])
    want, n = _ndcg_numpy(json.load(open(ranks)), ann["val"])
    got = float(re.search(r"^NDCG: (\S+)$", r.stdout, re.M).group(1))
    assert got == float("%f" % want) and "Rounds scored: %d" % n in r.stdout


def test_finetune_gen_two_gpus(gen_data, tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    d, flags, ann, ck = gen_data
    save = tmp_path / "run2"
    r = _run("finetune_gen", *flags, "-loadPath", ck, "-denseAnnotations", ann["train"], "-numEpochs", 1, "-saveIter", 1,
             "-batchSize", 2, "-math", "fp32", "-savePath", save, "-gpus", 2)
    assert "weights identical on 2 ranks" in r.stdout
    assert "model_final.t7" in os.listdir(save)
