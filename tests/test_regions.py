"""Region features without a GPU (DESIGN §26): the h5 layout, the commands' imgRegions and refusals, the dataloader's
refusal of a region file for a non-att encoder, the host-side parameter checks, and the masked SAN restatement in fp64
against the unmasked SAN on the compacted layout and against central differences."""
import ctypes as C

import numpy as np
import pytest
import torch

import region_oracle
from helpers import small_params, torch_batch, torch_params
from oracle import visdial_oracle as O
from visdial_b200 import _lib, cli, engine as E, h5lite
from visdial_b200.synthetic import make_batch, make_corpus, region_features, write_region_features


def test_h5lite_round_trips_region_features_and_counts(tmp_path):
    rng = np.random.default_rng(0)
    feats, counts = region_features(rng, 6, 10, 8)
    fixed, none = region_features(rng, 3, 36, 4, adaptive=False)
    assert none is None and counts[0] == 10 and counts[1] == 1 and counts.min() >= 1 and counts.max() <= 10
    path = str(tmp_path / "img.h5")
    write_region_features(path, {"train": (feats, counts), "val": (fixed, None)})
    got = h5lite.read(path)
    assert set(got) == {"images_train", "num_boxes_train", "images_val"}
    assert got["images_train"].shape == (6, 10, 8) and np.array_equal(got["images_train"], feats)
    assert got["num_boxes_train"].dtype.kind == "i" and np.array_equal(got["num_boxes_train"], counts)
    assert np.array_equal(got["images_val"], fixed)
    from visdial_b200.dataloader import image_regions, read_num_boxes
    assert image_regions(path, "train") == (10, 8) and image_regions(path, "val") == (36, 4)
    assert read_num_boxes(path, "val") is None and np.array_equal(read_num_boxes(path, "train"), counts)


def test_h5lite_shapes_reads_headers_only(tmp_path):
    path = str(tmp_path / "img.h5")
    a = np.arange(2 * 5 * 4, dtype=np.float32).reshape(2, 5, 4)
    h5lite.write(path, {"images_train": a, "num_boxes_train": np.array([5, 2], np.int32)}, chunks={"images_train": (1, 5, 4)},
                 gzip=True)
    assert h5lite.shapes(path) == {"images_train": (2, 5, 4), "num_boxes_train": (2,)}
    with pytest.raises(h5lite.H5Error):
        h5lite.shapes(path, ["images_val"])


def test_cli_refuses_splits_with_different_region_layouts(tmp_path):
    reg = str(tmp_path / "reg.h5")
    rng = np.random.default_rng(3)
    write_region_features(reg, {"train": region_features(rng, 3, 36, 8, adaptive=False),
                                "val": region_features(rng, 3, 100, 8)})
    with pytest.raises(ValueError, match="different image features"):
        cli.set_image_regions({"encoder": "mn-att-ques-im-hist", "imgFeatureSize": 8}, {"useIm": True, "inputImg": reg},
                              ["train", "val"])


@pytest.mark.parametrize("enc", ["mn-att-ques-im-hist", "lf-att-ques-im-hist"])
def test_restatement_without_counts_is_the_oracles_encoder(enc):
    """region_oracle with img_count None on the grid's S*S rows equals the oracle's own encoder, training mode included"""
    from oracle import philox
    p = small_params(enc, "disc")
    flat = E.init_parameters(p, seed=5)
    nb = make_batch(p, 3, seed=9)
    S, Cf = p["imgSpatialSize"], p["imgFeatureSize"]
    ctx = lambda: O.Ctx(train=True, mask_fn=philox.make_mask_fn(77, 3))
    ref = O.forward_backward(ctx(), p, torch_params(p, flat), torch_batch(nb))
    rb = dict(nb, img_feat=nb["img_feat"].reshape(3, S * S, Cf))
    with region_oracle.regions():
        got = O.forward_backward(ctx(), dict(p, imgRegions=S * S), torch_params(p, flat), torch_batch(rb))
    assert got["loss"] == ref["loss"]
    for k in ref["grads"]:
        assert torch.allclose(got["grads"][k], ref["grads"][k], rtol=1e-5, atol=1e-7), k


def _grid_file(path):
    h5lite.write(path, {"images_train": np.zeros((2, 8, 3, 3), np.float32)})


@pytest.mark.parametrize("enc", ["mn-att-ques-im-hist", "lf-att-ques-im-hist"])
def test_cli_sets_img_regions_from_the_features_file(tmp_path, enc):
    reg = str(tmp_path / "reg.h5")
    write_region_features(reg, {"train": region_features(np.random.default_rng(1), 4, 12, 16)})
    opt = {"useIm": True, "inputImg": reg}
    mp = cli.set_image_regions({"encoder": enc, "imgFeatureSize": 16}, opt, ["train"])
    assert mp["imgRegions"] == 12
    grid = str(tmp_path / "grid.h5")
    _grid_file(grid)
    mp = cli.set_image_regions({"encoder": enc, "imgFeatureSize": 8, "imgRegions": 12}, dict(opt, inputImg=grid), ["train"])
    assert "imgRegions" not in mp, "a grid run records the modelParams it recorded before"
    with pytest.raises(ValueError, match="imgFeatureSize"):
        cli.set_image_regions({"encoder": enc, "imgFeatureSize": 2048}, opt, ["train"])


def test_cli_refuses_a_region_file_for_a_non_att_encoder(tmp_path):
    reg = str(tmp_path / "reg.h5")
    write_region_features(reg, {"val": region_features(np.random.default_rng(2), 3, 5, 4)})
    with pytest.raises(ValueError, match="att encoders"):
        cli.set_image_regions({"encoder": "hrea-ques-im-hist", "imgFeatureSize": 4}, {"useIm": True, "inputImg": reg}, ["val"])


def test_dataloader_refuses_a_region_file_for_a_non_att_encoder():
    from visdial_b200.dataloader import Corpus
    p = small_params("lf-ques-im-hist", "disc", vocabSize=40, numOptions=100)
    raw = make_corpus(p, 8, 40, seed=1, max_ques_len=6, max_ans_len=5, max_cap_len=12)
    raw["images"] = np.zeros((8, 5, 24), np.float32)
    with pytest.raises(ValueError, match="att encoders"):
        Corpus(None, raw, E.derive_flags(dict(p)), 38, 39)


def test_img_regions_is_host_checked_and_leaves_the_layout_alone():
    lib = _lib.load()
    n = C.c_int64()
    bad = E.to_c_params(small_params("hrea-ques-im-hist", "gen", imgRegions=36))
    assert lib.vd_layout_count(C.byref(bad), None, C.byref(n)) == -1 and b"att encoders" in lib.vd_last_error()
    grid = small_params("mn-att-ques-im-hist", "disc")
    segs, total = E.layout(grid)
    segs_r, total_r = E.layout(dict(grid, imgRegions=100))
    assert total == total_r and [(s.name, s.rows, s.cols) for s in segs] == [(s.name, s.rows, s.cols) for s in segs_r]
    assert C.sizeof(_lib.vd_batch) == _lib.vd_batch.img_count.offset + 8


def _region_setup(enc, P=9, B=3, seed=4):
    p = small_params(enc, "disc", imgRegions=P, imgFeatureSize=8)
    flat = E.init_parameters(p, seed=seed)
    nb = make_batch(p, B, seed=seed)
    return p, torch_params(p, flat, torch.float64), nb


@pytest.mark.parametrize("enc", ["mn-att-ques-im-hist", "lf-att-ques-im-hist"])
def test_masked_san_equals_the_unmasked_san_on_the_compacted_layout(enc):
    p, P64, nb = _region_setup(enc)
    tb = {k: (v.double() if v.is_floating_point() else v) for k, v in torch_batch(nb).items()}
    with region_oracle.regions():
        masked = O.forward_backward(O.Ctx(train=False), p, P64, tb, only_forward=True)["encOut"]
    R = p["maxQuesCount"]
    for b, c in enumerate(nb["img_count"]):
        one = {k: v[b:b + 1] for k, v in tb.items() if k in ("ques_fwd", "hist", "img_feat", "answer_ind", "options")}
        one["options"] = tb["options"][b * R:(b + 1) * R]
        one["answer_ind"] = tb["answer_ind"][b * R:(b + 1) * R]
        one["img_feat"] = one["img_feat"][:, :int(c)]
        with region_oracle.regions():
            ref = O.forward_backward(O.Ctx(train=False), dict(p, imgRegions=int(c)), P64, one, only_forward=True)["encOut"]
        assert torch.allclose(masked[b * R:(b + 1) * R], ref, rtol=1e-12, atol=1e-13), (b, int(c))


@pytest.mark.parametrize("enc", ["mn-att-ques-im-hist", "lf-att-ques-im-hist"])
def test_masked_san_gradients_against_central_differences(enc):
    p, P64, nb = _region_setup(enc, P=7, B=2, seed=5)
    tb = {k: (v.double() if v.is_floating_point() else v) for k, v in torch_batch(nb).items()}
    ctx = O.Ctx(train=False)
    with region_oracle.regions():
        grads = O.forward_backward(ctx, p, P64, tb)["grads"]
        rng = np.random.default_rng(0)
        for name in [k for k in P64 if k.startswith("san.")]:
            flat = P64[name].view(-1)
            for i in rng.choice(flat.numel(), size=min(3, flat.numel()), replace=False):
                h = 1e-6
                old = float(flat[i])
                flat[i] = old + h
                lp = O.forward_backward(ctx, p, P64, tb, only_forward=True)["loss"]
                flat[i] = old - h
                lm = O.forward_backward(ctx, p, P64, tb, only_forward=True)["loss"]
                flat[i] = old
                fd = (lp - lm) / (2 * h)
                g = float(grads[name].view(-1)[i])
                assert abs(g - fd) <= 1e-6 + 1e-5 * abs(fd), (name, int(i), g, fd)
