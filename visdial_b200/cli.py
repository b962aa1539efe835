"""What the train / evaluate / generate commands share (train.lua + opts.lua, evaluate.lua, generate.lua): option tables
with the reference's flag spellings and defaults, parsed the way torch.CmdLine parses them (`-name value`; a boolean option
given alone flips its default), the checkpoint hand-over, the engine set-up and the one-process-per-GPU launch."""
from __future__ import annotations

import json
import os
import socket
import sys
import time

from .engine import derive_flags

# opts.lua:6-40
TRAIN_OPTIONS = [
    ("inputImg", "data/data_img.h5", "HDF5 file with image features"),
    ("inputQues", "data/visdial_data.h5", "HDF5 file with preprocessed questions"),
    ("inputJson", "data/visdial_params.json", "JSON file with info and vocab"),
    ("savePath", "checkpoints/", "Path to save checkpoints"),
    ("saveIter", 2, "Save model checkpoint after every saveIter epochs"),
    ("encoder", "lf-ques-hist", "Name of the encoder to use"),
    ("decoder", "gen", "Name of the decoder to use (gen/disc)"),
    ("imgNorm", 1, "normalize the image feature. 1=yes, 0=no"),
    ("imgEmbedSize", 300, "Size of the multimodal embedding"),
    ("imgFeatureSize", 4096, "Channel size of the image feature"),
    ("imgSpatialSize", 14, "Spatial size of image features (for attention-based encoders)."),
    ("embedSize", 300, "Size of input word embeddings"),
    ("rnnHiddenSize", 512, "Size of the LSTM state"),
    ("maxHistoryLen", 60, "Maximum history to consider when using concatenated QA pairs"),
    ("numLayers", 2, "Number of layers in LSTM"),
    ("commonEmbeddingSize", 512, "Common embedding size in MN-ATT-QIH"),
    ("numAttentionLayers", 1, "No. of attention hops in MN-ATT-QIH"),
    ("loadPath", "", "Checkpoint path to load from"),
    ("batchSize", 40, "Batch size (number of threads) (Adjust base on GPU memory)"),
    ("learningRate", 1e-3, "Learning rate"),
    ("weightInit", "xavier", "Weight initialization strategy: xavier|heuristic|kaiming (accepted, no effect)"),
    ("dropout", 0.5, "Dropout"),
    ("numEpochs", 100, "Epochs"),
    ("LRateDecay", 10, "After lr_decay epochs lr reduces to 0.1*lr"),
    ("lrDecayRate", 0.9997592083, "Decay for learning rate"),
    ("minLRate", 5e-5, "Minimum learning rate"),
    ("gpuid", 0, "GPU id to use"),
    ("backend", "cudnn", "nn|cudnn (accepted, no effect)"),
]

# the finetune command: train's options and the dense relevance annotations of the train split
FINETUNE_OPTIONS = TRAIN_OPTIONS + [
    ("denseAnnotations", "data/visdial_1.0_train_dense_sample.json", "VisDial v1.0 dense relevance annotations (train split)"),
]

# evaluate.lua:15-30
EVALUATE_OPTIONS = [
    ("inputImg", "data/data_img.h5", "h5file path with image feature"),
    ("inputQues", "data/visdial_data.h5", "h5file file with preprocessed questions"),
    ("inputJson", "data/visdial_params.json", "json path with info and vocab"),
    ("loadPath", "checkpoints/model.t7", "path to saved model"),
    ("split", "val", "split to evaluate on"),
    ("useGt", False, "whether to use ground truth for retrieving ranks"),
    ("batchSize", 30, "Batch size (number of threads) (Adjust base on GRAM)"),
    ("gpuid", 0, "GPU id to use"),
    ("backend", "cudnn", "nn|cudnn (accepted, no effect)"),
    ("saveRanks", False, "Whether to save ranks or not"),
    ("saveRankPath", "logs/ranks.json", ""),
]

# generate.lua:15-30
GENERATE_OPTIONS = [
    ("inputImg", "data/data_img.h5", "h5file path with image feature"),
    ("inputQues", "data/visdial_data.h5", "h5file file with preprocessed questions"),
    ("inputJson", "data/visdial_params.json", "json path with info and vocab"),
    ("loadPath", "checkpoints/model.t7", "path to saved model"),
    ("resultPath", "vis/results", "path to save generated results"),
    ("beamSize", 5, "Beam size"),
    ("beamLen", 20, "Beam length"),
    ("sampleWords", 0, "Whether to sample"),
    ("temperature", 1.0, "Sampling temperature"),
    ("maxThreads", 50, "Max threads"),
    ("gpuid", 0, "GPU id to use"),
    ("backend", "cudnn", "nn|cudnn (accepted, no effect)"),
    ("dialogsPerCall", 1, "Dialogs per encoder forward and device search call (1 = the reference's per-dialog loop)"),
]
# the generate command's table: generate.lua's options above, and which history each round is answered with
HISTORY_MODES = ("gt", "generated")
GENERATE_COMMAND_OPTIONS = GENERATE_OPTIONS + [
    ("history", "gt", "History each round is answered with: gt (the dataset's) | generated (the dialog's own answers)"),
]

# options of every command that the reference does not have: how the run is spread over GPUs and which math it uses
MATH_MODES = ("fp32", "tf32", "f16")
RUN_OPTIONS = [
    ("gpus", 1, "Number of GPUs (one process each, on gpuid .. gpuid+gpus-1)"),
    ("math", "tf32", "Tensor-core math mode: fp32 (rank-exact evaluation) | tf32 | f16"),
]

SEED = 1234                                                   # torch.manualSeed(1234), train.lua:12 / evaluate.lua:41


def parse(options, argv=None, prog=None) -> dict:
    """torch.CmdLine:parse over `options` + RUN_OPTIONS: `-name value`, the value taking the type of the default; a
    boolean option given alone flips its default.  Unknown options, bad values and -h exit like an argument parser."""
    table = options + RUN_OPTIONS
    defaults = {n: d for n, d, _ in table}
    prog = prog or os.path.basename(sys.argv[0])

    def fail(msg):
        print("%s: error: %s (see -h)" % (prog, msg), file=sys.stderr)
        raise SystemExit(2)

    args = list(sys.argv[1:] if argv is None else argv)
    opt = dict(defaults)
    i = 0
    while i < len(args):
        a = args[i]
        if a in ("-h", "--help"):
            print("usage: %s [options]" % prog)
            for n, d, h in table:
                print("  -%-22s %s [%s]" % (n, h, d))
            raise SystemExit(0)
        name = a[1:] if a.startswith("-") else None
        if name not in defaults:
            fail("unknown option %r" % a)
        d = defaults[name]
        if isinstance(d, bool):
            opt[name] = not d
            i += 1
            continue
        if i + 1 >= len(args):
            fail("%s needs a value" % a)
        try:
            opt[name] = type(d)(args[i + 1])
        except ValueError:
            fail("%s takes a %s, not %r" % (a, type(d).__name__, args[i + 1]))
        i += 2
    if opt["math"] not in MATH_MODES:
        fail("-math is one of %s" % "|".join(MATH_MODES))
    if "history" in opt and opt["history"] not in HISTORY_MODES:
        fail("-history is one of %s" % "|".join(HISTORY_MODES))
    if opt["gpus"] < 1:
        fail("-gpus must be at least 1")
    if opt["gpuid"] < 0:
        fail("-gpuid must be >= 0: visdial_b200 has no CPU path")
    return opt


def train_opts(argv=None, now=None, options=TRAIN_OPTIONS, prog="python -m visdial_b200.train") -> dict:
    """opts.lua:42-67: parsed options, the time-stamped default savePath and the flags derived from the encoder name."""
    opt = parse(options, argv, prog)
    if opt["savePath"] == "checkpoints/":                                           # :44-52
        t = now or time.localtime()
        opt["savePath"] = "checkpoints/model-%d-%d-%d-%d:%d:%d-%s-%s/" % (
            t.tm_mon, t.tm_mday, t.tm_year, t.tm_hour, t.tm_min, t.tm_sec, opt["encoder"], opt["decoder"])
    derive_flags(opt)                                                               # :55-59,66
    if "att" in opt["encoder"] and opt["inputImg"] == "data/data_img.h5":           # :62-65 (conv features)
        opt["inputImg"] = "data/data_img_pool5.h5"
    return opt


def model_params(opt: dict) -> dict:
    """`modelParams = opt` (train.lua:27) without the options that only say how the run is launched."""
    run_only = {n for n, _, _ in RUN_OPTIONS}
    return {k: v for k, v in opt.items() if k not in run_only}


def adopt_checkpoint_model(opt: dict, ck: dict, **overrides) -> dict:
    """train.lua:35-41 / evaluate.lua:61-75 / generate.lua:56-67: the checkpoint's modelParams with `overrides`, and the
    model's encoder / decoder / imgNorm (and the flags they imply) copied into `opt` for the dataloader.  The flags are
    derived for every command (generate.lua:63-67 omits concatHistory, which would feed a late-fusion model unconcatenated
    history)."""
    mp = dict(ck["modelParams"])
    mp.update(overrides)
    opt["imgNorm"], opt["encoder"], opt["decoder"] = mp.get("imgNorm", 1), mp["encoder"], mp["decoder"]
    derive_flags(opt)
    if mp.get("maxHistoryLen") is not None:
        opt["maxHistoryLen"] = mp["maxHistoryLen"]
    return mp


def vocab_size(opt: dict) -> int:
    """dataloader.lua:17-22: the json's words plus <START> and <END>."""
    with open(opt["inputJson"]) as f:
        return len(json.load(f)["word2ind"]) + 2


def build(mp: dict, opt: dict, rank: int, world: int, subsets, ck=None):
    """Model on GPU gpuid + rank in the requested math mode (with the checkpoint's weights and learning rate when `ck` is
    given), and its device dataloader over `subsets` read from opt's files.  Returns (model, dataloader)."""
    from . import VD_MATH_F16, VD_MATH_FP32, VD_MATH_TF32
    from .checkpoint import restore
    from .dataloader import Dataloader
    from .model import Model
    mp = dict(mp, gpuid=opt["gpuid"] + rank)
    model = Model(mp, seed=SEED)
    model.engine.set_math_mode({"fp32": VD_MATH_FP32, "tf32": VD_MATH_TF32, "f16": VD_MATH_F16}[opt["math"]])
    if ck is not None:
        restore(model, ck)
    dl = Dataloader(model.engine, seed=SEED, rank=rank, world=world).initialize_from_files(opt, subsets)
    for k in ("vocabSize", "maxQuesCount", "numOptions"):
        if getattr(dl, k) != model.params[k]:
            raise ValueError("the data has %s = %d, the model %d" % (k, getattr(dl, k), model.params[k]))
    return model, dl


def write_json(path: str, obj):
    """utils.writeJSON, written to a temporary name first so that a failed run leaves no partial file."""
    d = os.path.dirname(path)
    if d:
        os.makedirs(d, exist_ok=True)
    tmp = path + ".tmp%d" % os.getpid()
    with open(tmp, "w") as f:
        json.dump(obj, f)
    os.replace(tmp, path)


# ------------------------------------------------------------------------------------------------ several GPUs
def _free_port() -> int:
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _rank_main(module: str, fn: str, opt: dict, rank: int, world: int, port: int):
    import importlib

    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)      # out-of-band only: ids, losses, result gathers
    try:
        getattr(importlib.import_module(module), fn)(opt, rank, world)
    finally:
        dist.destroy_process_group()


def launch(module: str, fn: str, opt: dict) -> int:
    """Run `module.fn(opt, rank, world)`: in this process for -gpus 1, else in one spawned process per GPU.  If a rank
    fails, the others are stopped (they would wait for it in the next collective) and its exit code is returned."""
    world = int(opt["gpus"])
    if world == 1:
        import importlib
        getattr(importlib.import_module(module), fn)(opt, 0, 1)
        return 0
    import multiprocessing as mp
    ctx = mp.get_context("spawn")
    port = _free_port()
    procs = [ctx.Process(target=_rank_main, args=(module, fn, opt, r, world, port)) for r in range(world)]
    for p in procs:
        p.start()
    code = 0
    try:
        while any(p.exitcode is None for p in procs):
            failed = [p.exitcode for p in procs if p.exitcode not in (None, 0)]
            if failed:
                code = failed[0]
                break
            time.sleep(0.2)
        code = code or next((p.exitcode for p in procs if p.exitcode), 0)
    finally:
        for p in procs:
            if p.exitcode is None:
                p.terminate()
        for p in procs:
            p.join()
    return code


def run(module: str, fn: str, opt: dict):
    sys.exit(launch(module, fn, opt))
