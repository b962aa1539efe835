"""The finetune_gen command's host side and the gen dense step's fp64 reference (tests/dense_gen_oracle.py).  No GPU."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from dense_gen_oracle import forward_backward_dense_gen as dense_gen_ref
from helpers import seg_slices, small_batch, small_params, torch_batch, torch_params
from oracle import visdial_oracle as O
from visdial_b200 import cli, init_parameters, t7
from visdial_b200.finetune_gen import finetune_gen_opts

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_options_are_finetunes():
    o = finetune_gen_opts(["-loadPath", "gen.t7", "-savePath", "run/"])
    assert {n for n, _, _ in cli.FINETUNE_OPTIONS} <= set(o)
    for name, default, _ in cli.FINETUNE_OPTIONS:
        if name not in ("loadPath", "savePath"):
            assert o[name] == default or name == "inputImg", name
    assert o["loadPath"] == "gen.t7" and o["savePath"] == "run/" and o["gpus"] == 1
    o = finetune_gen_opts(["-denseAnnotations", "x.json", "-batchSize", "8", "-gpus", "2", "-math", "fp32"])
    assert o["denseAnnotations"] == "x.json" and o["batchSize"] == 8 and o["gpus"] == 2 and o["math"] == "fp32"
    with pytest.raises(SystemExit):
        finetune_gen_opts(["-noSuchOption", "1"])


def test_refuses_a_disc_model_before_any_gpu_work(tmp_path):
    ck = str(tmp_path / "disc.t7")
    t7.save(ck, {"modelW": np.zeros(4, np.float32), "modelParams": {"encoder": "lf-ques", "decoder": "disc"}})
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    for args in (["-loadPath", ck, "-decoder", "gen"], ["-decoder", "disc"]):
        r = subprocess.run([sys.executable, "-m", "visdial_b200.finetune_gen"] + args + ["-savePath", str(tmp_path / "run")],
                           cwd=ROOT, capture_output=True, text=True, timeout=120, env=env)
        assert r.returncode != 0 and "visdial_b200.finetune " in r.stderr and "'disc' decoder" in r.stderr, r.stderr
    assert not (tmp_path / "run").exists()


@pytest.mark.parametrize("enc", ["lf-ques", "mn-att-ques-im-hist"])
def test_reference_gradient_matches_finite_differences(enc):
    """d loss / d theta of the score-level loss (fp64, dropout off) against central differences, for entries of the
    decoder's projection and both LSTM layers, the word embedding, and an encoder weight reached only through the
    annotated round's initial decoder state."""
    p = small_params(enc, "gen", vocabSize=30, embedSize=8, rnnHiddenSize=32, numOptions=5, imgEmbedSize=8,
                     commonEmbeddingSize=8)
    nb = small_batch(p, B=2, gen_eval=True)
    rounds = np.array([1, p["maxQuesCount"] - 1], np.int32)
    rel = np.array([[0, 1, 0.5, 0, 0], [0.25, 0, 0, 1, 0]], np.float32)
    flat = init_parameters(p, seed=3).astype(np.float64)
    tb = {k: (v.double() if v.is_floating_point() else v) for k, v in torch_batch(nb).items()}
    P = torch_params(p, flat, dtype=torch.float64)
    ref = dense_gen_ref(O.Ctx(train=False, structure="batched"), p, P, tb, rounds, rel)
    assert ref["scores"].shape == (2, p["numOptions"]) and np.isfinite(ref["loss"])
    segs = seg_slices(p)
    names = ["dec.out.weight", "dec.out.bias", "dec.lstm1.weight", "dec.lstm2.weight", "wordEmbed.weight"]
    names.append("ques.lstm1.weight" if "ques.lstm1.weight" in segs else [n for n in segs if n.startswith("ques")][0])
    rng = np.random.default_rng(0)
    eps = 1e-6

    def loss_at(f):
        Q = torch_params(p, f.astype(np.float32), dtype=torch.float64)
        for k in Q:                                               # keep the fp64 perturbation (torch_params goes via float32)
            s = segs[k]
            Q[k] = torch.from_numpy(f[s].reshape(Q[k].shape).copy())
        return dense_gen_ref(O.Ctx(train=False, structure="batched"), p, Q, tb, rounds, rel)["loss"]

    checked = 0
    for name in names:
        s = segs[name]
        g = ref["grads"][name].numpy().ravel()
        # the largest entries (those the loss depends on) and a random one
        for i in list(np.argsort(-np.abs(g))[:2]) + [int(rng.integers(0, g.size))]:
            f = flat.copy()
            f[s.start + i] += eps
            up = loss_at(f)
            f[s.start + i] -= 2 * eps
            fd = (up - loss_at(f)) / (2 * eps)
            assert abs(fd - g[i]) <= 1e-6 + 1e-5 * abs(g[i]), (name, int(i), fd, float(g[i]))
            checked += int(g[i] != 0)
    assert checked >= len(names)
