"""What the train / evaluate / generate commands share (train.lua + opts.lua, evaluate.lua, generate.lua): option tables
with the reference's flag spellings and defaults, parsed the way torch.CmdLine parses them (`-name value`; a boolean option
given alone flips its default), the checkpoint hand-over, the engine set-up and the one-process-per-GPU launch."""
from __future__ import annotations

import json
import math
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
# diverse beam search (DESIGN §22): several distinct answers per question from one search
DIVERSE_OPTIONS = [
    ("beamGroups", 1, "Diverse beam search: groups the beam is split into (1 = plain beam search; must divide beamSize)"),
    ("diversity", 0.5, "Diverse beam search: penalty per earlier group's column that chose the same token"),
]
# n-best lists (DESIGN §24): the beam search keeps each group's nBest best finished answers, ranked by length-normalised score
NBEST_OPTIONS = [
    ("lengthPenalty", 0.0, "Beam search: rank finished answers by score / ((5 + l) / 6)^lengthPenalty, l their tokens (0 = by score)"),
    ("nBest", 1, "Beam search: finished answers each group keeps and reports, best first (1 to 32)"),
]
# truncated sampling (DESIGN §23): -sampleWords 1 draws from the top-k / top-p prefix of each step's distribution
TRUNCATION_OPTIONS = [
    ("topK", 0, "Sampling: draw from the topK most likely words only (0 = all)"),
    ("topP", 1.0, "Sampling: draw from the fewest most likely words holding topP of the probability (1 = all)"),
]
# answer rules (DESIGN §25): words barred from every beam-search or sampling step of a gen model's answers
ANSWER_RULE_OPTIONS = [
    ("minWords", 0, "Answers: <END> is barred until the answer has minWords words"),
    ("noRepeatNgram", 0, "Answers: no n-gram of this many words occurs twice in an answer (0 = off)"),
    ("bannedWords", "", "Answers: comma-separated words never generated (e.g. UNK)"),
]
# the generate command's table: generate.lua's options above, diverse beam search, n-best lists, truncated sampling, answer
# rules, and which history each round is answered with
HISTORY_MODES = ("gt", "generated")
GENERATE_COMMAND_OPTIONS = GENERATE_OPTIONS + DIVERSE_OPTIONS + NBEST_OPTIONS + TRUNCATION_OPTIONS + ANSWER_RULE_OPTIONS + [
    ("history", "gt", "History each round is answered with: gt (the dataset's) | generated (the dialog's own answers)"),
]

# the chat command: generate's options, diverse beam search, n-best lists, truncated sampling, answer rules, and which images
# are talked about with which questions
CHAT_OPTIONS = GENERATE_OPTIONS + DIVERSE_OPTIONS + NBEST_OPTIONS + TRUNCATION_OPTIONS + ANSWER_RULE_OPTIONS + [
    ("split", "val", "Split the images and captions come from"),
    ("imageIds", "", "Comma-separated COCO image ids of the split (default: the -questions file's, else its first image)"),
    ("questions", "", "JSON {image_id: [question, ...]}: ask these and write results.json; else read stdin, one per line"),
    ("serve", 0, "1: serve many conversations from JSON lines on stdin, each answer a JSON line on stdout (DESIGN §20)"),
    ("capacity", 128, "-serve: how many conversations the dialog pool holds at once"),
]

# options of every command that the reference does not have: how the run is spread over GPUs and which math it uses
MATH_MODES = ("fp32", "tf32", "f16")
RUN_OPTIONS = [
    ("gpus", 1, "Number of GPUs (one process each, on gpuid .. gpuid+gpus-1)"),
    ("math", "tf32", "Tensor-core math mode: fp32 (rank-exact evaluation) | tf32 | f16"),
    ("deterministic", 0, "1: training steps repeat bit for bit (gradient sums in a fixed order, one GPU; DESIGN §27) | 0"),
]

# validation while training (DESIGN §28), parsed with train's, finetune's and finetune_gen's tables
VALIDATION_OPTIONS = [
    ("valIter", 0, "Rank the val split every valIter epochs, log val_log.json and keep model_best.t7 (0 = never)"),
    ("valDenseAnnotations", "", "VisDial v1.0 val dense relevance annotations: the validations also compute NDCG, the "
                                "selection metric (else MRR)"),
    ("valPatience", 0, "Stop after valPatience validations in a row without a better selection metric (0 = never)"),
]

SEED = 1234                                                   # torch.manualSeed(1234), train.lua:12 / evaluate.lua:41


def usage_error(prog: str, msg: str):
    """Exit 2 with `msg`, as an argument parser refuses a command line."""
    print("%s: error: %s (see -h)" % (prog, msg), file=sys.stderr)
    raise SystemExit(2)


def parse(options, argv=None, prog=None) -> dict:
    """torch.CmdLine:parse over `options` + RUN_OPTIONS: `-name value`, the value taking the type of the default; a
    boolean option given alone flips its default.  Unknown options, bad values and -h exit like an argument parser."""
    table = options + RUN_OPTIONS
    defaults = {n: d for n, d, _ in table}
    prog = prog or os.path.basename(sys.argv[0])

    def fail(msg):
        usage_error(prog, msg)

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
    if "beamGroups" in opt:
        if opt["beamGroups"] < 1 or opt["beamSize"] % opt["beamGroups"] != 0:
            fail("-beamGroups must be at least 1 and divide -beamSize")
        if not math.isfinite(opt["diversity"]) or opt["diversity"] < 0:
            fail("-diversity must be finite and >= 0")
    if "nBest" in opt:
        if not math.isfinite(opt["lengthPenalty"]) or opt["lengthPenalty"] < 0:
            fail("-lengthPenalty must be finite and >= 0")
        if not 1 <= opt["nBest"] <= 32:
            fail("-nBest must be in [1, 32]")
        if opt["lengthPenalty"] == 0 and opt["nBest"] == 1:   # options that change nothing leave the run's options as they were
            del opt["lengthPenalty"], opt["nBest"]
    if "topK" in opt:
        if opt["topK"] < 0:
            fail("-topK must be >= 0")
        if not (0.0 < opt["topP"] <= 1.0):
            fail("-topP must be in (0, 1]")
        if not truncated_sampling(opt):         # options that change nothing leave the run's options as they were
            del opt["topK"], opt["topP"]
    if "minWords" in opt:
        if opt["minWords"] < 0 or opt["noRepeatNgram"] < 0:
            fail("-minWords and -noRepeatNgram must be >= 0")
        if not answer_rules_active(opt):        # options that change nothing leave the run's options as they were
            del opt["minWords"], opt["noRepeatNgram"], opt["bannedWords"]
    if "valIter" in opt:
        if opt["valIter"] < 0 or opt["valPatience"] < 0:
            fail("-valIter and -valPatience must be >= 0")
        if opt["valIter"] == 0 and opt["valPatience"] > 0:
            fail("-valPatience needs -valIter")
        if opt["valIter"] == 0 and opt["valDenseAnnotations"]:
            fail("-valDenseAnnotations needs -valIter")
        for n, d, _ in VALIDATION_OPTIONS:      # the defaults change nothing: the run's options stay as they were
            if opt[n] == d:
                del opt[n]
    if opt["gpus"] < 1:
        fail("-gpus must be at least 1")
    if opt["deterministic"] not in (0, 1):
        fail("-deterministic is 0 or 1")
    if opt["deterministic"] == 1 and opt["gpus"] != 1:
        fail("-deterministic 1 runs on one GPU (-gpus 1)")
    if opt["deterministic"] == 0:               # the default changes nothing: the run's options stay as they were
        del opt["deterministic"]
    if opt["gpuid"] < 0:
        fail("-gpuid must be >= 0: visdial_b200 has no CPU path")
    return opt


def train_opts(argv=None, now=None, options=TRAIN_OPTIONS, prog="python -m visdial_b200.train") -> dict:
    """opts.lua:42-67: parsed options, the time-stamped default savePath and the flags derived from the encoder name.
    `options` are parsed with VALIDATION_OPTIONS; a validating run's files are checked here (validation_data_problem)."""
    opt = parse(options + VALIDATION_OPTIONS, argv, prog)
    if opt["savePath"] == "checkpoints/":                                           # :44-52
        t = now or time.localtime()
        opt["savePath"] = "checkpoints/model-%d-%d-%d-%d:%d:%d-%s-%s/" % (
            t.tm_mon, t.tm_mday, t.tm_year, t.tm_hour, t.tm_min, t.tm_sec, opt["encoder"], opt["decoder"])
    derive_flags(opt)                                                               # :55-59,66
    if "att" in opt["encoder"] and opt["inputImg"] == "data/data_img.h5":           # :62-65 (conv features)
        opt["inputImg"] = "data/data_img_pool5.h5"
    if opt.get("valIter"):
        problem = validation_data_problem(opt)
        if problem:
            usage_error(prog, problem)
    return opt


def validation_data_problem(opt: dict):
    """Why -valIter cannot run on opt's files, or None: the question file needs the val split, the json its
    unique_img_val, and a -valDenseAnnotations file must read against them (visdial_b200.dense.read).  Host reads only (the
    h5 headers, num_rounds_val, the json), so that a bad file is refused before any GPU work."""
    from . import dense, h5lite
    try:
        shapes = h5lite.shapes(opt["inputQues"])
    except (OSError, h5lite.H5Error) as e:
        return "-valIter: cannot read %s (%s)" % (opt["inputQues"], e)
    if "opt_val" not in shapes or "ans_index_val" not in shapes:
        return "-valIter: %s has no val split (opt_val, ans_index_val)" % opt["inputQues"]
    try:
        with open(opt["inputJson"]) as f:
            unique_img = json.load(f).get("unique_img_val")
    except (OSError, ValueError) as e:
        return "-valIter: cannot read %s (%s)" % (opt["inputJson"], e)
    if unique_img is None or len(unique_img) != shapes["opt_val"][0]:
        return "-valIter: %s needs unique_img_val, one entry per val dialog of %s" % (opt["inputJson"], opt["inputQues"])
    if not opt.get("valDenseAnnotations"):
        return None
    num_rounds = h5lite.read(opt["inputQues"], ["num_rounds_val"])["num_rounds_val"] if "num_rounds_val" in shapes else None
    try:
        ann = dense.read(opt["valDenseAnnotations"], int(shapes["opt_val"][2]), unique_img=unique_img, num_rounds=num_rounds)
    except (OSError, ValueError) as e:
        return "-valDenseAnnotations: %s" % (e.args[0] if e.args else e)
    if len(ann) == 0:
        return "-valDenseAnnotations: %s has no usable annotated round" % opt["valDenseAnnotations"]
    return None


def truncated_sampling(opt: dict) -> bool:
    """-sampleWords 1 with a truncating -topK (> 0) or -topP (< 1)"""
    return opt.get("sampleWords", 0) == 1 and (opt.get("topK", 0) > 0 or opt.get("topP", 1.0) < 1.0)


def banned_words(opt: dict) -> list:
    """-bannedWords as a list of words (empty entries dropped)"""
    return [w.strip() for w in opt.get("bannedWords", "").split(",") if w.strip()]


def answer_rules_active(opt: dict) -> bool:
    """-minWords > 0, -noRepeatNgram > 0 or a -bannedWords word"""
    return opt.get("minWords", 0) > 0 or opt.get("noRepeatNgram", 0) > 0 or bool(banned_words(opt))


def answer_rule_params(opt: dict) -> dict:
    """the answer rules as generateAnswers / DialogPool params (none when inactive)"""
    if not answer_rules_active(opt):
        return {}
    return {"minWords": opt.get("minWords", 0), "noRepeatNgram": opt.get("noRepeatNgram", 0), "bannedWords": banned_words(opt)}


def written_opts(opt: dict) -> dict:
    """The options a results.json records: the diverse beam search options only when they change the search
    (-beamGroups > 1), the n-best options only when one differs from its default (-lengthPenalty 0, -nBest 1), and the
    truncation options only when they truncate a sampling run (-sampleWords 1 with -topK > 0 or -topP < 1), so that every
    run without them writes the file it wrote before they existed.  The answer rules likewise, only when active."""
    plain = opt.get("beamGroups", 1) == 1
    unruled = not answer_rules_active(opt)
    untruncated = not truncated_sampling(opt)
    unlisted = all(opt.get(n, d) == d for n, d, _ in NBEST_OPTIONS)
    return {k: v for k, v in opt.items()
            if not (plain and k in ("beamGroups", "diversity")) and not (untruncated and k in ("topK", "topP"))
            and not (unlisted and k in ("lengthPenalty", "nBest"))
            and not (unruled and k in ("minWords", "noRepeatNgram", "bannedWords"))}


def model_params(opt: dict) -> dict:
    """`modelParams = opt` (train.lua:27) without the options that only say how the run is launched or validated."""
    run_only = {n for n, _, _ in RUN_OPTIONS + VALIDATION_OPTIONS}
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


def set_image_regions(mp: dict, opt: dict, subsets):
    """imgRegions from the image features file (DESIGN §26): P when its images_<split> is a 3-D (numImages, P, C) region
    file, and no entry for a grid or fc7 file, so that those runs record the modelParams they recorded before.  A region
    file needs an att encoder and imgFeatureSize = C."""
    from .dataloader import image_regions
    mp.pop("imgRegions", None)
    if not opt.get("useIm") or not subsets:
        return mp
    found = {s: image_regions(opt["inputImg"], s) for s in subsets}
    if len(set(found.values())) > 1:
        raise ValueError("the splits of %s hold different image features (%s); one run needs one layout (regions, "
                         "channels)" % (opt["inputImg"], ", ".join("%s: %s" % kv for kv in sorted(found.items()))))
    P, C = found[subsets[0]]
    if P == 0:
        return mp
    if "att" not in mp["encoder"]:
        raise ValueError("%s holds region features, which only the att encoders read, not %s"
                         % (opt["inputImg"], mp["encoder"]))
    if int(mp.get("imgFeatureSize", 4096)) != C:
        raise ValueError("%s holds region features of %d channels but the model has imgFeatureSize = %d (pass "
                         "-imgFeatureSize %d to train on it)" % (opt["inputImg"], C, int(mp.get("imgFeatureSize", 4096)), C))
    mp["imgRegions"] = P
    return mp


def host_memory_problem(opt: dict, subsets, world: int, gpuid: int):
    """Why the image features this run keeps in pinned host memory (dataloader.image_placement; one copy per rank) would
    not fit in the host's physical memory, or None.  Reads the features file's headers only."""
    from .dataloader import device_memory, host_memory, image_placement, split_image_bytes
    if not opt.get("useIm") or not subsets:
        return None
    sizes = split_image_bytes(opt["inputImg"], subsets)
    place = image_placement(sizes, int(opt.get("batchSize", 40)), device_memory(gpuid))
    pinned = sum(b for b, (on_host, _) in zip(sizes, place) if on_host)
    if pinned == 0 or world * pinned <= host_memory():
        return None
    return ("the image features of %s do not fit on the GPU and take %.1f GB of pinned host memory per GPU: %d GPUs "
            "need %.1f GB, more than the host's %.1f GB" % (opt["inputImg"], pinned / 1e9, world, world * pinned / 1e9,
                                                            host_memory() / 1e9))


def build(mp: dict, opt: dict, rank: int, world: int, subsets, ck=None):
    """Model on GPU gpuid + rank in the requested math mode (with the checkpoint's weights and learning rate when `ck` is
    given), and its device dataloader over `subsets` read from opt's files.  Returns (model, dataloader)."""
    from . import VD_MATH_F16, VD_MATH_FP32, VD_MATH_TF32
    from .checkpoint import restore
    from .dataloader import Dataloader
    from .model import Model
    mp = dict(mp, gpuid=opt["gpuid"] + rank)
    set_image_regions(mp, opt, subsets)
    problem = host_memory_problem(opt, subsets, world, mp["gpuid"])
    if problem:
        usage_error(os.path.basename(sys.argv[0]), problem)
    model = Model(mp, seed=SEED)
    model.engine.set_math_mode({"fp32": VD_MATH_FP32, "tf32": VD_MATH_TF32, "f16": VD_MATH_F16}[opt["math"]])
    if opt.get("deterministic", 0):
        model.engine.set_deterministic(True)
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
