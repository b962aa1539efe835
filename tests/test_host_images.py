"""Host placement of image features (DESIGN §29) without a GPU: the placement rule on the sizes users run, the look-ahead
draws against a plain generator, and the refusal of a multi-GPU run whose pinned copies would not fit in host memory."""
import numpy as np
import pytest

from visdial_b200 import cli
from visdial_b200 import dataloader as DL
from visdial_b200.dataloader import Dataloader, image_placement

H100 = 81559 << 20                                   # what an H100 80GB HBM3 reports as its total memory
POOL5, FC7, BOX = 512 * 14 * 14 * 4, 4096 * 4, 2048 * 4


def _on_host(sizes, B, dev=H100):
    return [h for h, _ in image_placement(sizes, B, dev)]


def test_placement():
    # VisDial v0.9 pool5: train (82 783 images) and val (40 504) at the default batchSize, and train alone at the bench's B
    assert _on_host([82783 * POOL5, 40504 * POOL5], 40) == [False, False]
    assert _on_host([82783 * POOL5], 32) == [False]
    assert _on_host([82783 * FC7, 40504 * FC7], 40) == [False, False]
    # VisDial v1.0 with 36 fixed detector boxes: train (123 287 images) and val (2 064)
    assert _on_host([123287 * 36 * BOX, 2064 * 36 * BOX], 40) == [False, False]
    # the adaptive 100-box file: 101 GB of train goes to the host, val still fits beside the engine
    assert _on_host([123287 * 100 * BOX, 2064 * 100 * BOX], 40) == [True, False]
    # an evaluation at a large batch keeps a split that takes less than half the device
    assert _on_host([40504 * POOL5], 256) == [False]
    # a split placed on the device counts against the next one's budget
    place = image_placement([30 << 30, 30 << 30], 40, H100)
    assert [h for h, _ in place] == [False, True] and place[1][1] == place[0][1] - (30 << 30)
    # a budget of 0 bytes sends every split to the host; imgDeviceBytes is never 0 (0 is "no limit")
    assert image_placement([16, 16], 4, 0) == [(True, 1), (True, 1)]


class _FakeCorpus:
    def __init__(self, n):
        self.numThreads, self.images_on_host = n, True
        self.prefetched, self.got = [], []

    def get_batch(self, inds, mode, with_num_rounds=False):
        self.got.append(np.array(inds))
        return np.array(inds)

    def prefetch(self, inds):
        self.prefetched.append(np.array(inds))


class _FakeDense:
    def __init__(self, n):
        self.dialog = np.arange(n)[::-1].copy()
        self.round_id = np.ones(n, np.int64)
        self.relevance = np.zeros((n, 3), np.float32)

    def __len__(self):
        return len(self.dialog)


def test_look_ahead_draws_what_a_plain_generator_draws():
    dl = Dataloader(None, seed=3)
    train, val = _FakeCorpus(50), _FakeCorpus(20)
    dl.corpus = {"train": train, "val": val}
    dl.numThreads = {"train": 50, "val": 20}
    dl.part = {"train": (0, 50), "val": (0, 20)}
    dense_a, dense_b = _FakeDense(17), _FakeDense(23)
    plain = np.random.default_rng(3)
    p = {"batchSize": 4, "decoder": "disc"}
    seq = ["train", "train", ("dense", dense_a), "train", ("train", 6), ("train", 6), "val", ("train", 6),
           ("dense", dense_a), ("dense", dense_a), ("dense", dense_b), "val", "train", "train"]
    for step in seq:
        if step == "val":                      # a validation walk draws nothing and leaves the look-ahead in place
            start = 0
            while start < 20:
                _, start = dl.getTestBatch(start, p, "val")
            continue
        if isinstance(step, tuple) and step[0] == "dense":
            batch, _, _ = dl.getDenseTrainBatch(p, step[1])
            assert batch.tolist() == step[1].dialog[plain.integers(0, len(step[1]), size=4)].tolist(), step
            continue
        size = step[1] if isinstance(step, tuple) else None
        got = dl.getTrainBatch(p, size)
        assert got.tolist() == plain.integers(0, 50, size=size or 4).tolist(), step
    # every training and dense draw prefetches the draw after it; every val batch but the last prefetches the next one
    assert len(train.prefetched) == len(seq) - 2
    assert [b.tolist() for b in val.prefetched] == [list(range(s, min(s + 4, 20))) for s in (4, 8, 12, 16)] * 2


def _features_file(tmp_path, n, shape):
    from visdial_b200 import h5lite
    path = str(tmp_path / "img.h5")
    h5lite.write(path, {"images_train": np.zeros((n,) + shape, np.float32)})
    return path


def test_multi_gpu_runs_that_would_not_fit_in_host_memory_are_refused(tmp_path, monkeypatch, capsys):
    path = _features_file(tmp_path, 10, (2, 3, 3))             # 720 bytes of features
    monkeypatch.setattr(DL, "device_memory", lambda gpuid: 0)  # none of it fits on the device
    monkeypatch.setattr(DL, "host_memory", lambda: 1500)
    opt = {"useIm": True, "inputImg": path, "batchSize": 4, "gpuid": 0}
    assert cli.host_memory_problem(opt, ["train"], 2, 0) is None          # 2 x 720 <= 1500
    problem = cli.host_memory_problem(opt, ["train"], 3, 0)
    assert problem and "3 GPUs" in problem
    assert cli.host_memory_problem(dict(opt, useIm=False), ["train"], 3, 0) is None
    monkeypatch.setattr(DL, "device_memory", lambda gpuid: 1 << 40)     # it fits on the device: nothing is pinned
    assert cli.host_memory_problem(opt, ["train"], 3, 0) is None
    # the commands refuse it before any GPU work: cli.build exits 2 before it creates the engine
    monkeypatch.setattr(DL, "device_memory", lambda gpuid: 0)
    with pytest.raises(SystemExit) as e:
        cli.build({"encoder": "mn-att-ques-im-hist", "decoder": "disc", "imgFeatureSize": 2}, opt, 0, 3, ["train"])
    assert e.value.code == 2 and "pinned host memory" in capsys.readouterr().err
