"""Dense relevance annotations, NDCG, the ndcg and finetune commands' host side, and the soft-target loss of the dense
fine-tuning reference.  No GPU."""
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from dense_oracle import soft_xent
from visdial_b200 import cli, dense, t7
from visdial_b200.finetune import finetune_opts

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K = 5


def _write(path, obj):
    with open(path, "w") as f:
        json.dump(obj, f)
    return str(path)


def _entry(iid, rid, rel, key="gt_relevance"):
    return {"image_id": iid, "round_id": rid, key: rel}


# ---- reader ------------------------------------------------------------------------------------------------------------
def test_reader_accepts_both_keys_and_maps_images_through_the_split(tmp_path):
    imgs = ["COCO_train2014_%012d.jpg" % i for i in (7, 1003, 42)]
    p = _write(tmp_path / "a.json", [_entry(42, 3, [0, 1, 0.5, 0, 0]), _entry(7, 10, [1, 0, 0, 0, 0], key="relevance")])
    d = dense.read(p, K, unique_img=imgs, num_rounds=[10, 10, 10])
    assert d.dialog.tolist() == [2, 0] and d.round_id.tolist() == [3, 10] and d.image_id.tolist() == [42, 7]
    assert d.relevance.dtype == np.float32 and d.relevance[0].tolist() == [0, 1, 0.5, 0, 0]
    assert d.skipped == 0 and len(d) == 2
    assert dense.read(p, K).dialog is None                             # without a split: keyed by (image_id, round_id)


def test_reader_skips_and_counts_zero_sum_entries(tmp_path):
    p = _write(tmp_path / "a.json", [_entry(1, 1, [0] * K), _entry(2, 2, [0, 0, 1, 0, 0]), _entry(3, 1, [0.0] * K)])
    d = dense.read(p, K)
    assert d.skipped == 2 and len(d) == 1 and d.image_id.tolist() == [2]


@pytest.mark.parametrize("entries,what", [
    ([_entry(99, 1, [1] * K)], "image not in the split"),
    ([_entry(1, 5, [0, 1, 0, 0, 0])], "duplicate"),
    ([_entry(1, 0, [1] * K)], "round_id outside 1..10"),
    ([_entry(2, 9, [1] * K)], "round_id outside 1..8"),                # dialog 2 has 8 rounds
    ([_entry(1, 1, [1] * (K + 1))], "6 relevances, numOptions is 5"),
    ([_entry(1, 1, [1, -0.5, 0, 0, 0])], "finite and >= 0"),
    ([_entry(1, 1, [1, float("nan"), 0, 0, 0])], "finite and >= 0"),
    ([_entry(1, 1, [1, float("inf"), 0, 0, 0])], "finite and >= 0"),
    ([{"image_id": 1, "round_id": 1}], "gt_relevance or relevance"),
])
def test_reader_refusals_name_the_entry(tmp_path, entries, what):
    p = _write(tmp_path / "a.json", [_entry(1, 5, [0, 0, 0, 1, 0])] + entries)
    with pytest.raises(ValueError) as e:
        dense.read(p, K, unique_img=["img_0001.jpg", "x_0002.jpg"], num_rounds=[10, 8])
    msg = str(e.value)
    assert what in msg and "entry 1 " in msg and "image_id %r" % entries[-1]["image_id"] in msg, msg


# ---- NDCG --------------------------------------------------------------------------------------------------------------
def _ranks_of(order):
    """1-based rank of every option from the predicted order (best first)."""
    r = np.empty(len(order), np.int64)
    r[np.asarray(order)] = np.arange(1, len(order) + 1)
    return r


def test_ndcg_perfect_and_reversed_orderings():
    rel = np.array([[1.0, 0.5, 0.0, 0.0, 0.25]])
    best = _ranks_of(np.argsort(-rel[0], kind="stable"))
    assert dense.ndcg(best[None], rel) == pytest.approx(1.0, abs=1e-15)
    # reversed: options in order 3, 2, 4, 1, 0 (the worst first); k = 3 nonzero relevances, so 3 positions count
    rev = _ranks_of([3, 2, 4, 1, 0])
    dcg = 0.0 / math.log2(2) + 0.0 / math.log2(3) + 0.25 / math.log2(4)
    idcg = 1.0 / math.log2(2) + 0.5 / math.log2(3) + 0.25 / math.log2(4)
    assert dense.ndcg(rev[None], rel) == pytest.approx(dcg / idcg, rel=1e-12)


def test_ndcg_counts_only_nonzero_relevances_and_averages_rounds():
    rel = np.array([[0.0, 1.0, 0.0, 0.0, 0.0], [0.5, 0.5, 0.0, 0.0, 0.0]])
    r0 = _ranks_of([0, 1, 2, 3, 4])              # the one relevant option at position 2, but only k = 1 position counts
    r1 = _ranks_of([1, 2, 0, 3, 4])              # k = 2: positions 1 and 2, the second holds a zero
    want1 = (0.5 / math.log2(2)) / (0.5 / math.log2(2) + 0.5 / math.log2(3))
    assert dense.ndcg(r0[None], rel[:1]) == 0.0
    assert dense.ndcg(np.stack([r0, r1]), rel) == pytest.approx((0.0 + want1) / 2, rel=1e-12)


def test_tied_relevances_give_one_idcg_in_either_order():
    rel = np.array([[0.5, 0.0, 0.5, 1.0, 0.0]])
    a, b = _ranks_of([3, 0, 2, 1, 4]), _ranks_of([3, 2, 0, 4, 1])
    assert dense.ndcg(a[None], rel) == dense.ndcg(b[None], rel) == pytest.approx(1.0, abs=1e-15)


# ---- ndcg command ------------------------------------------------------------------------------------------------------
def _ndcg_cmd(*args):
    return subprocess.run([sys.executable, "-m", "visdial_b200.ndcg"] + [str(a) for a in args], cwd=ROOT,
                          capture_output=True, text=True, timeout=120)


def test_ndcg_command_prints_the_value_and_refuses_missing_rounds(tmp_path):
    rng = np.random.default_rng(0)
    ann, table, rels, ranks = [], [], [], []
    for iid in range(6):
        rel = rng.choice([0.0, 0.0, 0.5, 1.0], size=100)
        rel[iid] = 1.0
        ann.append(_entry(iid + 1000, 1 + iid % 10, rel.tolist()))
        for rid in range(1, 11):                                       # every round, as evaluate -saveRanks writes them
            r = _ranks_of(rng.permutation(100))
            table.append({"image_id": iid + 1000, "round_id": rid, "ranks": r.tolist()})
            if rid == 1 + iid % 10:
                rels.append(rel)
                ranks.append(r)
    ann.append(_entry(2000, 4, [0.0] * 100))                           # all zero: skipped, not looked up
    a = _write(tmp_path / "ann.json", ann)
    r = _ndcg_cmd("-ranks", _write(tmp_path / "ranks.json", table), "-denseAnnotations", a)
    assert r.returncode == 0, r.stderr
    want = dense.ndcg(np.stack(ranks), np.stack(rels))
    assert "NDCG: %f\n" % want in r.stdout and "Rounds scored: 6\n" in r.stdout and "1 annotated entries" in r.stdout
    missing = [e for e in table if not (e["image_id"] == 1003 and e["round_id"] == 4)]
    r = _ndcg_cmd("-ranks", _write(tmp_path / "short.json", missing), "-denseAnnotations", a)
    assert r.returncode != 0 and "NDCG" not in r.stdout
    assert "(image_id 1003, round_id 4) is missing" in r.stderr


def test_ndcg_command_does_not_load_the_engine(tmp_path):
    a = _write(tmp_path / "ann.json", [_entry(1, 1, [1.0, 0.5])])
    rk = _write(tmp_path / "r.json", [{"image_id": 1, "round_id": 1, "ranks": [2, 1]}])
    code = ("import sys, runpy; sys.argv = ['ndcg', '-ranks', %r, '-denseAnnotations', %r]\n"
            "try:\n    runpy.run_module('visdial_b200.ndcg', run_name='__main__')\n"
            "except SystemExit as e:\n    assert e.code == 0\n"
            "assert 'libvisdial_b200' not in open('/proc/self/maps').read()\n"
            "import visdial_b200._lib as L; assert L._lib is None\n") % (rk, a)
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    assert "NDCG: %f" % ((0.5 + 1.0 / math.log2(3)) / (1.0 + 0.5 / math.log2(3))) in r.stdout


# ---- finetune command --------------------------------------------------------------------------------------------------
def test_finetune_options_are_train_options_plus_the_annotations():
    assert [o[0] for o in cli.FINETUNE_OPTIONS[:-1]] == [o[0] for o in cli.TRAIN_OPTIONS]
    o = finetune_opts(["-encoder", "mn-att-ques-im-hist", "-decoder", "disc", "-savePath", "run/"])
    assert o["denseAnnotations"] == "data/visdial_1.0_train_dense_sample.json"
    assert o["inputImg"] == "data/data_img_pool5.h5" and o["imgNorm"] == 0 and o["gpus"] == 1 and o["savePath"] == "run/"
    o = finetune_opts(["-denseAnnotations", "x.json", "-batchSize", "8", "-gpus", "2"])
    assert o["denseAnnotations"] == "x.json" and o["batchSize"] == 8 and o["gpus"] == 2
    assert o["savePath"].startswith("checkpoints/model-") and o["savePath"].endswith("-lf-ques-hist-gen/")


def test_finetune_refuses_a_gen_model_before_any_gpu_work(tmp_path):
    ck = str(tmp_path / "gen.t7")
    t7.save(ck, {"modelW": np.zeros(4, np.float32), "modelParams": {"encoder": "lf-ques", "decoder": "gen"}})
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    for args in (["-loadPath", ck, "-decoder", "disc"], ["-decoder", "gen"]):
        r = subprocess.run([sys.executable, "-m", "visdial_b200.finetune"] + args + ["-savePath", str(tmp_path / "run")],
                           cwd=ROOT, capture_output=True, text=True, timeout=120, env=env)
        assert r.returncode != 0 and "needs a disc model" in r.stderr, r.stderr
    assert not (tmp_path / "run").exists()


# ---- the reference's soft loss -----------------------------------------------------------------------------------------
def test_soft_loss_and_gradient_against_fp64_and_finite_differences():
    rng = np.random.default_rng(3)
    B, Ko = 4, 9
    s = rng.standard_normal((B, Ko)) * 3
    rel = rng.choice([0.0, 0.5, 1.0], size=(B, Ko))
    rel[:, 0] = 1.0
    p = rel / rel.sum(1, keepdims=True)
    lse = s.max(1) + np.log(np.exp(s - s.max(1, keepdims=True)).sum(1))
    want = float(np.mean(lse - (p * s).sum(1)))
    sm = np.exp(s - lse[:, None])
    want_grad = (sm - p) / B
    st = torch.tensor(s, dtype=torch.float64, requires_grad=True)
    loss = soft_xent(st, torch.tensor(rel, dtype=torch.float64))
    loss.backward()
    assert float(loss) == pytest.approx(want, rel=1e-13)
    np.testing.assert_allclose(st.grad.numpy(), want_grad, rtol=1e-12, atol=1e-15)
    eps = 1e-6
    fd = np.zeros_like(s)
    for i in range(B):
        for k in range(Ko):
            for sgn in (1, -1):
                t = s.copy()
                t[i, k] += sgn * eps
                fd[i, k] += sgn * float(soft_xent(torch.tensor(t), torch.tensor(rel))) / (2 * eps)
    np.testing.assert_allclose(fd, want_grad, rtol=1e-6, atol=1e-9)
    # an unnormalised relevance row gives the loss of its normalised targets
    assert float(soft_xent(st.detach(), torch.tensor(rel * 7.0))) == pytest.approx(want, rel=1e-13)
