"""The dense fine-tuning step (vd_forward_backward_dense) against its CPU reference (tests/dense_oracle.py) in the three
math modes at test_parity_gpu / test_tensorcore_gpu's tolerances, its option-LSTM row count, repeatability, refusals, the
2-GPU equivalence, and the finetune -> evaluate -> ndcg commands end to end."""
import ctypes as C
import json
import math
import os
import re
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

from dense_oracle import forward_backward_dense as dense_ref
from helpers import seg_slices, small_batch, small_params, torch_batch, torch_params
from oracle import philox
from oracle import visdial_oracle as O
from visdial_b200 import VD_MATH_F16, VD_MATH_FP32, VD_MATH_TF32, Batch, Engine, VdError, init_parameters
from visdial_b200._lib import VD_E_BADARG, VD_E_STATE
from visdial_b200.synthetic import make_batch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEED, ITER = 11, 3
ENCODERS = ("lf-ques", "hre-ques-im-hist", "hrea-ques-im-hist", "mn-att-ques-im-hist")
MID = dict(rnnHiddenSize=128, embedSize=64, vocabSize=200, numOptions=10, commonEmbeddingSize=64, imgSpatialSize=4,
           imgEmbedSize=32)
F16 = dict(rnnHiddenSize=256, embedSize=64, vocabSize=300, numOptions=100, commonEmbeddingSize=64, imgFeatureSize=64,
           imgSpatialSize=4, imgEmbedSize=32)


def _case(enc, mode):
    """(params, batch) at the sizes test_parity_gpu (fp32) and test_tensorcore_gpu (TF32 mid-size; F16 with >= 1024 option
    rows for the selected rounds, so that the fp16 option-LSTM kernels run) hold the standard step to."""
    if mode == VD_MATH_FP32:
        p = small_params(enc, "disc", vocabSize=300)
        return p, small_batch(p, B=3)
    if mode == VD_MATH_TF32:
        p = small_params(enc, "disc", imgFeatureSize=64 if "att" in enc else 256, **MID)
        B = 13
    else:
        p = small_params(enc, "disc", **F16)
        B = 11
    return p, make_batch(p, B, seed=7, max_ques_len=9, max_ans_len=6, max_cap_len=12, max_hist_len=14, max_hist_concat=40,
                         empty_round_every=4)


def _targets(p, B, seed=5):
    rng = np.random.default_rng(seed)
    rounds = rng.integers(0, p["maxQuesCount"], size=B).astype(np.int32)
    rel = rng.choice([0.0, 0.0, 0.0, 0.5, 1.0], size=(B, p["numOptions"])).astype(np.float32)
    rel[:, 0] = np.maximum(rel[:, 0], 0.5)                 # positive row sums
    return rounds, rel


def _engine(p, flat, mode, training=1):
    eng = Engine(p)
    eng.set_math_mode(mode)
    eng.set_parameters(flat)
    eng.set_training(training)
    eng.set_dropout_seed(SEED, ITER)
    eng.zero_grad()
    return eng


def _rel(a, b):
    a = np.asarray(a, np.float64).ravel()
    b = np.asarray(b, np.float64).ravel()
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


@pytest.mark.parametrize("mode", [VD_MATH_FP32, VD_MATH_TF32, VD_MATH_F16], ids=["fp32", "tf32", "f16"])
@pytest.mark.parametrize("enc", ENCODERS)
def test_dense_step_matches_reference(enc, mode):
    """Loss and every parameter segment's gradient, dropout on; and exact zeros wherever only unselected rounds feed the
    standard step's gradient (dEnc is zero on those rounds, the option LSTM never sees them)."""
    p, nb = _case(enc, mode)
    flat = init_parameters(p, seed=3)
    B = nb["ques_fwd"].shape[0]
    rounds, rel = _targets(p, B)
    eng = _engine(p, flat, mode)
    loss = eng.forward_backward_dense(Batch(nb), rounds, rel)
    g = eng.get_gradients()
    eng.close()
    psite = {O.SITE_FUSION: p["dropout"]}
    ctx = lambda: O.Ctx(train=True, mask_fn=philox.make_mask_fn(SEED, ITER, psite), structure="batched")
    P, tb = torch_params(p, flat), torch_batch(nb)
    ref = dense_ref(ctx(), p, P, tb, rounds, rel)
    std = O.forward_backward(ctx(), p, P, tb)
    if mode == VD_MATH_FP32:                                 # test_parity_gpu: fp32 re-association only
        assert abs(loss - ref["loss"]) <= 1e-4 * max(1.0, abs(ref["loss"])), (loss, ref["loss"])
    else:                                                    # test_tensorcore_gpu: 10-bit-mantissa operands
        assert abs(loss - ref["loss"]) < 5e-3 * max(1.0, abs(ref["loss"])), (loss, ref["loss"])
    only_unselected = 0
    std_max = max(float(v.abs().max()) for v in std["grads"].values())
    for name, s in seg_slices(p).items():
        r = ref["grads"][name].numpy().ravel()
        if mode == VD_MATH_FP32:
            scale = max(float(np.abs(r).max()), 1e-30)
            err = float(np.abs(g[s] - r).max())
            assert err <= 2e-5 + 2e-4 * scale, (name, err, scale)
        elif np.abs(r).max() >= 1e-7:
            assert _rel(g[s], r) < 3e-2, (name, _rel(g[s], r))
        # (a gradient that is zero up to rounding in both steps, like a bias under a softmax's shift invariance, is not one)
        zero = (r == 0) & (np.abs(std["grads"][name].numpy().ravel()) > 1e-6 * std_max)
        only_unselected += int(zero.sum())
        assert not g[s][zero].any(), (name, int(zero.sum()), float(np.abs(g[s][zero]).max()))
    if mode == VD_MATH_FP32:
        assert only_unselected > 0                           # the words of unselected rounds only (V = 300)


def test_option_lstm_runs_on_the_selected_rows_only():
    """Profiling counts (not timings): the fp16 option-LSTM step class does B * numOptions rows of work per step, the
    standard step N * numOptions."""
    p = small_params("mn-att-ques-im-hist", "disc", **F16)
    B, K, H = 11, p["numOptions"], p["rnnHiddenSize"]
    nb = make_batch(p, B, seed=7, max_ques_len=9, max_ans_len=6, max_cap_len=12, max_hist_len=14, empty_round_every=4)
    To = nb["options"].shape[2]
    rounds, rel = _targets(p, B)
    eng = _engine(p, init_parameters(p, seed=3), VD_MATH_F16)
    eng.profile(True)
    flops = {}
    for what in ("standard", "dense"):
        eng.profile_reset()
        eng.zero_grad()
        if what == "standard":
            eng.forward_backward(Batch(nb))
        else:
            eng.forward_backward_dense(Batch(nb), rounds, rel)
        eng.synchronize()
        flops[what] = (eng.kernel_stats("lstm_step")["flops"], eng.kernel_stats("lstm_step_bwd")["flops"])
    eng.close()
    per_step = 2.0 * B * K * 4 * H * H                       # the recurrent contraction of B*K rows
    assert flops["dense"] == ((To - 1) * per_step, (To - 1) * per_step)
    R = p["maxQuesCount"]
    assert flops["standard"] == ((To - 1) * R * per_step, (To - 1) * R * per_step)


def test_repeated_fp32_steps_agree():
    """Two fp32 dense steps from the same state: the loss (forward, gather, disc scores, soft cross-entropy with its
    fixed-order reductions) bit for bit; dW to re-association level, because the existing weight- and embedding-gradient
    kernels accumulate with atomics."""
    p, nb = _case("mn-att-ques-im-hist", VD_MATH_FP32)
    flat = init_parameters(p, seed=3)
    rounds, rel = _targets(p, 3)
    eng = _engine(p, flat, VD_MATH_FP32)
    out = []
    for _ in range(2):
        eng.zero_grad()
        eng.set_dropout_seed(SEED, ITER)
        out.append((eng.forward_backward_dense(Batch(nb), rounds, rel), eng.get_gradients()))
    eng.close()
    (l0, g0), (l1, g1) = out
    assert l0 == l1
    for name, s in seg_slices(p).items():
        assert float(np.abs(g1[s] - g0[s]).max()) <= 1e-6 * float(np.abs(g0[s]).max()) + 1e-12, name


def test_refusals_keep_the_engine_usable():
    p, nb = _case("lf-ques", VD_MATH_FP32)
    flat = init_parameters(p, seed=3)
    rounds, rel = _targets(p, 3)
    gen = Engine(small_params("lf-ques", "gen"))
    with pytest.raises(VdError) as e:
        gen.forward_backward_dense(Batch(small_batch(small_params("lf-ques", "gen"), B=3)), rounds, np.ones((3, 7), np.float32))
    assert e.value.code == VD_E_STATE
    gen.close()
    eng = _engine(p, flat, VD_MATH_FP32)
    good = eng.forward_backward_dense(Batch(nb), rounds, rel)
    bad = []
    for r, x in ((np.array([0, -1, 2]), rel), (np.array([0, 10, 2]), rel)):
        bad.append((r, x))
    for v in (-0.25, np.nan, np.inf):
        x = rel.copy()
        x[1, 3] = v
        bad.append((rounds, x))
    x = rel.copy()
    x[2] = 0
    bad.append((rounds, x))
    for r, x in bad:
        with pytest.raises(VdError) as e:
            eng.forward_backward_dense(Batch(nb), r, x)
        assert e.value.code == VD_E_BADARG, (r, x)
    b = Batch(nb)
    loss = C.c_float()
    ok_r = np.ascontiguousarray(rounds, np.int32)
    ok_x = np.ascontiguousarray(rel, np.float32)
    for args in ((None, ok_r.ctypes.data, ok_x.ctypes.data), (C.byref(b.c), None, ok_x.ctypes.data),
                 (C.byref(b.c), ok_r.ctypes.data, None)):
        assert eng.lib.vd_forward_backward_dense(eng.h, *args, C.byref(loss)) == VD_E_BADARG
    eng.zero_grad()
    assert eng.forward_backward_dense(Batch(nb), rounds, rel) == good
    eng.close()


# ---- two GPUs -----------------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


BIG = dict(rnnHiddenSize=256, embedSize=64, vocabSize=300, numOptions=100, commonEmbeddingSize=64, imgFeatureSize=64,
           imgSpatialSize=4, imgEmbedSize=32)


def _mg_case(mode, gpuid):
    p = small_params("mn-att-ques-im-hist", "disc", gpuid=gpuid, **(BIG if mode != VD_MATH_FP32 else {}))
    nb = small_batch(p, B=4, seed=3)
    return p, nb, _targets(p, 4)


def _mg_worker(rank, world, port, mode, out):
    import torch.distributed as dist
    from visdial_b200 import dist as vdist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    p, full, (rounds, rel) = _mg_case(mode, rank)
    lo, hi = vdist.shard_range(4, rank, world)
    eng = _engine(p, init_parameters(p, seed=3), mode, training=2)   # dropout off: masks are indexed per local shard
    vdist.attach_engine(eng, rank, world)
    eng.zero_grad()
    loss = eng.forward_backward_dense(Batch(vdist.shard_batch(full, rank, world, p["maxQuesCount"])), rounds[lo:hi], rel[lo:hi])
    eng.clamp_adam_step(1e-3)
    w, g = eng.get_parameters(), eng.get_gradients()
    losses = vdist.gather_ranks(np.asarray([loss], dtype=np.float64), rank, world)
    if rank == 0:
        out.put((w, g, losses))
    eng.close()
    dist.destroy_process_group()


@pytest.mark.parametrize("mode", [VD_MATH_FP32, VD_MATH_TF32], ids=["fp32", "tf32"])
def test_two_gpus_match_one(mode):
    """2 ranks x B/2 against 1 x B: one dense step and Adam, test_multigpu_gpu's tolerances."""
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
    loss1 = eng.forward_backward_dense(Batch(full), rounds, rel)
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
V = 40
SPLITS = {"train": 24, "val": 13}


def _params():
    return small_params("lf-ques", "disc", vocabSize=V, numOptions=100, numEpochs=2, saveIter=1, batchSize=4)


@pytest.fixture(scope="module")
def data(tmp_path_factory):
    """visdial_params.json / visdial_data.h5 (lf-ques: no image file), dense annotations of both splits, a disc
    checkpoint.  Returns (directory, the -input* flags, the annotation files, the checkpoint)."""
    from visdial_b200 import Model, h5lite
    from visdial_b200.synthetic import make_corpus
    d = tmp_path_factory.mktemp("dense")
    p = _params()
    ques, info, ann = {}, {"word2ind": {"w%d" % i: i for i in range(1, V - 1)}}, {}
    rng = np.random.default_rng(4)
    for i, (split, n) in enumerate(SPLITS.items()):
        raw = make_corpus(p, n, 40, seed=11 + i, max_ques_len=8, max_ans_len=6, max_cap_len=14)
        ques.update({k + "_" + split: np.asarray(v, np.uint32) for k, v in raw.items()})
        info["unique_img_" + split] = ["COCO_%s2014_%012d.jpg" % (split, 1000 * i + j) for j in range(n)]
        entries = []
        for j in range(n - 2 if split == "train" else n):
            rel = rng.choice([0.0, 0.0, 0.5, 1.0], size=100)
            if split == "train" and j == 3:
                rel[:] = 0.0                                       # skipped
            else:
                rel[rng.integers(0, 100)] = 1.0
            entries.append({"image_id": 1000 * i + j, "round_id": int(rng.integers(1, int(raw["num_rounds"][j]) + 1)),
                            ("relevance" if split == "train" else "gt_relevance"): rel.tolist()})
        ann[split] = str(d / ("%s_dense.json" % split))
        with open(ann[split], "w") as f:
            json.dump(entries, f)
    h5lite.write(str(d / "visdial_data.h5"), ques)
    with open(str(d / "visdial_params.json"), "w") as f:
        json.dump(info, f)
    m = Model(p, seed=1234)
    ck = str(d / "disc.t7")
    m.save(ck, final=True)
    m.engine.close()
    flags = ["-inputJson", str(d / "visdial_params.json"), "-inputQues", str(d / "visdial_data.h5")]
    return d, flags, ann, ck


def _run(mod, *args):
    r = subprocess.run([sys.executable, "-m", "visdial_b200." + mod] + [str(a) for a in args], cwd=ROOT,
                       capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, (r.stdout[-3000:], r.stderr[-3000:])
    return r


def _ndcg_numpy(table, ann_path):
    """NDCG restated from the challenge's definition, independently of visdial_b200.dense."""
    ranks = {(e["image_id"], e["round_id"]): e["ranks"] for e in table}
    vals = []
    for e in json.load(open(ann_path)):
        rel = np.asarray(e["gt_relevance"], np.float64)
        if rel.sum() == 0:
            continue
        order = np.argsort(ranks[(e["image_id"], e["round_id"])])
        k = int((rel != 0).sum())
        disc = np.log2(np.arange(k) + 2.0)
        vals.append((rel[order][:k] / disc).sum() / (np.sort(rel)[::-1][:k] / disc).sum())
    return float(np.mean(vals)), len(vals)


def test_finetune_evaluate_ndcg(data, tmp_path):
    from visdial_b200.checkpoint import load_checkpoint
    d, flags, ann, ck = data
    save = tmp_path / "run"
    r = _run("finetune", *flags, "-loadPath", ck, "-denseAnnotations", ann["train"], "-numEpochs", 2, "-saveIter", 1,
             "-batchSize", 4, "-math", "fp32", "-savePath", save)
    n_ann = SPLITS["train"] - 2 - 1
    per_epoch = math.ceil(n_ann / 4)
    assert "\n%d iter per epoch." % per_epoch in r.stdout and "1 annotated entries with all relevances 0 skipped" in r.stdout
    assert "%d annotated rounds" % n_ann in r.stdout
    assert sorted(os.listdir(save)) == ["model_epoch_1.t7", "model_epoch_2.t7", "model_final.t7"]
    ck1 = load_checkpoint(str(save / "model_epoch_1.t7"))
    assert ck1["optims"]["t"] == per_epoch
    w0, w1 = load_checkpoint(ck)["modelW"], load_checkpoint(str(save / "model_final.t7"))["modelW"]
    assert np.abs(w1 - w0).max() > 0
    ranks = tmp_path / "ranks.json"
    _run("evaluate", *flags, "-loadPath", save / "model_final.t7", "-saveRanks", "-saveRankPath", ranks, "-math", "fp32")
    r = _run("ndcg", "-ranks", ranks, "-denseAnnotations", ann["val"])
    want, n = _ndcg_numpy(json.load(open(ranks)), ann["val"])
    got = float(re.search(r"^NDCG: (\S+)$", r.stdout, re.M).group(1))
    assert got == float("%f" % want) and "Rounds scored: %d" % n in r.stdout


def test_finetune_two_gpus(data, tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    d, flags, ann, ck = data
    save = tmp_path / "run2"
    r = _run("finetune", *flags, "-loadPath", ck, "-denseAnnotations", ann["train"], "-numEpochs", 1, "-saveIter", 1,
             "-batchSize", 2, "-math", "fp32", "-savePath", save, "-gpus", 2)
    assert "weights identical on 2 ranks" in r.stdout
    assert "model_final.t7" in os.listdir(save)
