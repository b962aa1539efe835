"""The train / evaluate / generate commands' host side: option defaults restated from the reference scripts, the flags
opts.lua derives, utils.idToWords, h5lite's memory-mapped reads and the one-process-per-rank launch.  No GPU."""
import re
import time

import numpy as np
import pytest

from visdial_b200 import cli, h5lite
from visdial_b200.utils import idToWords

# opts.lua:6-40
TRAIN_DEFAULTS = dict(
    inputImg="data/data_img.h5", inputQues="data/visdial_data.h5", inputJson="data/visdial_params.json",   # :6-8
    savePath="checkpoints/", saveIter=2,                                                                   # :9-10
    encoder="lf-ques-hist", decoder="gen", imgNorm=1,                                                      # :13-15
    imgEmbedSize=300, imgFeatureSize=4096, imgSpatialSize=14, embedSize=300, rnnHiddenSize=512,            # :18-22
    maxHistoryLen=60, numLayers=2, commonEmbeddingSize=512, numAttentionLayers=1,                          # :23-26
    loadPath="",                                                                                           # :28
    batchSize=40, learningRate=1e-3, weightInit="xavier", dropout=0.5, numEpochs=100, LRateDecay=10,       # :31-36
    lrDecayRate=0.9997592083, minLRate=5e-5, gpuid=0, backend="cudnn",                                     # :37-40
)
# evaluate.lua:15-30
EVALUATE_DEFAULTS = dict(
    inputImg="data/data_img.h5", inputQues="data/visdial_data.h5", inputJson="data/visdial_params.json",   # :16-18
    loadPath="checkpoints/model.t7", split="val", useGt=False,                                             # :20-22
    batchSize=30, gpuid=0, backend="cudnn",                                                                # :25-27
    saveRanks=False, saveRankPath="logs/ranks.json",                                                       # :29-30
)
# generate.lua:15-30
GENERATE_DEFAULTS = dict(
    inputImg="data/data_img.h5", inputQues="data/visdial_data.h5", inputJson="data/visdial_params.json",   # :16-18
    loadPath="checkpoints/model.t7", resultPath="vis/results",                                             # :20-21
    beamSize=5, beamLen=20, sampleWords=0, temperature=1.0, maxThreads=50, gpuid=0, backend="cudnn",       # :24-30
)
RUN_DEFAULTS = dict(gpus=1, math="tf32")


@pytest.mark.parametrize("options,want,extra", [
    (cli.TRAIN_OPTIONS, TRAIN_DEFAULTS, {}),
    (cli.EVALUATE_OPTIONS, EVALUATE_DEFAULTS, {}),
    (cli.GENERATE_OPTIONS, GENERATE_DEFAULTS, {"dialogsPerCall": 1}),
], ids=["train", "evaluate", "generate"])
def test_defaults_are_the_reference_scripts(options, want, extra):
    got = cli.parse(options, [])
    assert got == dict(want, **extra, **RUN_DEFAULTS)
    for k, v in got.items():
        assert type(v) is type(dict(want, **extra, **RUN_DEFAULTS)[k]), k


def test_flags_parse_like_torch_cmdline():
    o = cli.parse(cli.EVALUATE_OPTIONS, ["-useGt", "-saveRanks", "-batchSize", "7", "-split", "test", "-gpus", "2",
                                         "-math", "fp32"])
    assert o["useGt"] is True and o["saveRanks"] is True and o["batchSize"] == 7 and o["split"] == "test"
    assert o["gpus"] == 2 and o["math"] == "fp32"
    g = cli.parse(cli.GENERATE_OPTIONS, ["-temperature", "0.5", "-sampleWords", "1", "-dialogsPerCall", "4"])
    assert g["temperature"] == 0.5 and g["sampleWords"] == 1 and g["dialogsPerCall"] == 4
    for bad in (["-gpuid", "-1"], ["-gpus", "0"], ["-math", "bf16"], ["-batchSiz", "3"]):
        with pytest.raises(SystemExit):
            cli.parse(cli.TRAIN_OPTIONS, bad)


def test_train_derived_flags():
    """opts.lua:44-67."""
    now = time.struct_time((2017, 3, 9, 14, 5, 7, 3, 68, 0))
    o = cli.train_opts(["-encoder", "hre-ques-hist", "-decoder", "disc"], now=now)
    assert o["savePath"] == "checkpoints/model-3-9-2017-14:5:7-hre-ques-hist-disc/"          # :44-52
    assert (o["useHistory"], o["useIm"], o["concatHistory"]) == (True, False, False)          # :55-59
    assert o["inputImg"] == "data/data_img.h5" and o["imgNorm"] == 1
    o = cli.train_opts(["-encoder", "lf-ques-im"])
    assert (o["useHistory"], o["useIm"], o["concatHistory"]) == (False, True, True)
    assert re.fullmatch(r"checkpoints/model-\d+-\d+-\d+-\d+:\d+:\d+-lf-ques-im-gen/", o["savePath"])
    o = cli.train_opts(["-encoder", "mn-att-ques-im-hist", "-imgNorm", "1"])                  # :62-67
    assert o["inputImg"] == "data/data_img_pool5.h5" and o["imgNorm"] == 0
    o = cli.train_opts(["-encoder", "mn-att-ques-im-hist", "-inputImg", "x.h5", "-savePath", "run/"])
    assert o["inputImg"] == "x.h5" and o["imgNorm"] == 0 and o["savePath"] == "run/"
    assert "gpus" not in cli.model_params(o) and "math" not in cli.model_params(o)


def test_checkpoint_model_params_reach_the_dataloader_options():
    """evaluate.lua:61-75: the model's encoder / decoder / imgNorm replace the command's, the flags follow the encoder."""
    opt = cli.parse(cli.GENERATE_OPTIONS, [])
    ck = {"modelParams": {"encoder": "lf-ques-hist", "decoder": "gen", "imgNorm": 1, "batchSize": 40, "gpuid": 3}}
    mp = cli.adopt_checkpoint_model(opt, ck, batchSize=5)
    assert mp["batchSize"] == 5 and mp["gpuid"] == 3 and ck["modelParams"]["batchSize"] == 40
    assert (opt["encoder"], opt["useHistory"], opt["concatHistory"], opt["useIm"]) == ("lf-ques-hist", True, True, False)


W = {1: "a", 2: "b", 3: "c", 8: "<START>", 9: "<END>"}


@pytest.mark.parametrize("ids,text", [
    ([1, 2, 3], " a b c"),                      # a leading space before every word
    ([0, 0, 1, 0, 2], " a b"),                  # pads skipped (right-aligned questions)
    ([8, 1, 2, 9], " <START> a b <END>"),      # <START> kept, <END> kept
    ([8, 1, 9, 2, 3], " <START> a <END>"),     # stop after <END>
    ([8, 2, 9, 0, 0], " <START> b <END>"),     # pads after <END>
    ([8, 9, 0, 1], " <START> <END>"),
    ([0, 0], ""),
    ([], ""),
])
def test_id_to_words(ids, text):
    """utils.lua:48-63."""
    assert idToWords(ids, W) == text
    assert idToWords(np.asarray(ids, dtype=np.int32), W) == text


def _datasets():
    rng = np.random.default_rng(2)
    return {"ques_val": rng.integers(0, 9000, size=(5, 10, 7)).astype(np.uint32),
            "images_val": rng.standard_normal((5, 4, 3, 3)).astype(np.float32),
            "d64": rng.standard_normal(6), "i64": np.arange(-3, 3, dtype=np.int64).reshape(2, 3)}


def test_h5lite_maps_contiguous_datasets_read_only(tmp_path):
    data = _datasets()
    path = str(tmp_path / "m.h5")
    h5lite.write(path, data)
    out = h5lite.read(path)
    for k, v in data.items():
        a = out[k]
        assert isinstance(a, np.memmap) and not a.flags.writeable, k
        assert a.dtype == v.dtype and a.shape == v.shape and np.array_equal(a, v), k
        with pytest.raises(ValueError):
            a[(0,) * a.ndim] = 1


@pytest.mark.parametrize("gzip", [False, True], ids=["chunked", "deflated"])
def test_h5lite_decodes_chunked_datasets(tmp_path, gzip):
    data = _datasets()
    path = str(tmp_path / "c.h5")
    h5lite.write(path, data, chunks={"ques_val": (2, 4, 7), "images_val": (3, 4, 3, 3)}, gzip=gzip)
    out = h5lite.read(path)
    for k in ("ques_val", "images_val"):
        assert not isinstance(out[k], np.memmap) and out[k].flags.writeable, k
        assert out[k].dtype == data[k].dtype and np.array_equal(out[k], data[k]), k
    assert isinstance(out["d64"], np.memmap)


def test_h5lite_decodes_big_endian_datasets(tmp_path):
    a = np.array([[1, -2, 300000], [7, 8, -9]], dtype=np.int32)
    path = str(tmp_path / "be.h5")
    h5lite.write(path, {"x": a})
    b = bytearray(open(path, "rb").read())
    i = b.index(a.astype("<i4").tobytes())
    b[i:i + a.nbytes] = a.astype(">i4").tobytes()
    import struct
    j = b.index(struct.pack("<BBBBI", 0x10, 0x08, 0, 0, 4))
    b[j + 1] |= 1                                                          # the datatype's byte-order bit
    open(path, "wb").write(bytes(b))
    out = h5lite.read(path)["x"]
    assert not isinstance(out, np.memmap) and out.dtype == np.int32 and out.dtype.isnative
    assert np.array_equal(out, a)


def test_h5lite_refuses_an_empty_file(tmp_path):
    p = tmp_path / "e.h5"
    p.write_bytes(b"")
    with pytest.raises(h5lite.H5Error):
        h5lite.read(str(p))


def _plumbing_rank(opt, rank, world):
    """A stand-in for a command's per-rank work in cli.launch: a share of `n` dialogs, gathered and written by rank 0."""
    from visdial_b200 import dist as vdist
    from visdial_b200.dataloader import eval_partition
    if rank == opt.get("fail_rank"):
        raise RuntimeError("rank %d fails" % rank)
    lo, hi = eval_partition(opt["n"], rank, world)
    table = vdist.gather_objects([{"rank": rank, "dialog": i} for i in range(lo, hi)], world)
    loss = vdist.mean_over_ranks(float(rank), world)
    if rank == 0:
        cli.write_json(opt["out"], {"table": table, "loss": loss})


def test_launch_gathers_every_rank_in_order_and_stops_on_a_failed_rank(tmp_path):
    """-gpus N: one spawned process per rank with a gloo group; rank 0 writes the rank-ordered gather.  When a rank fails the
    others (waiting for it in the next collective) are stopped, the exit code is non-zero and nothing is written."""
    import json
    out = tmp_path / "o.json"
    assert cli.launch("test_cli_host", "_plumbing_rank", {"gpus": 3, "n": 7, "out": str(out)}) == 0
    got = json.load(open(out))
    assert [e["dialog"] for e in got["table"]] == list(range(7))
    assert [e["rank"] for e in got["table"]] == [0, 0, 0, 1, 1, 2, 2] and got["loss"] == 1.0
    out = tmp_path / "two.json"
    assert cli.launch("test_cli_host", "_plumbing_rank", {"gpus": 3, "n": 2, "out": str(out)}) == 0   # an empty share
    assert [e["dialog"] for e in json.load(open(out))["table"]] == [0, 1]
    out = tmp_path / "f.json"
    t = time.time()
    assert cli.launch("test_cli_host", "_plumbing_rank", {"gpus": 3, "n": 7, "out": str(out), "fail_rank": 2}) != 0
    assert not out.exists() and time.time() - t < 120
