"""`python -m visdial_b200.train -encoder ... -decoder ...`: train.lua on the engine.

Options and defaults are those of opts.lua:6-40 (see visdial_b200.cli).  Every `saveIter` epochs it writes
`<savePath>/model_epoch_N.t7` = {modelW, optims, modelParams}, at the end `<savePath>/model_final.t7` (float weights, no
optims); every 100 iterations it prints `[date][Epoch:..][Iter:..][Loss:..][lr:..]`.  `-loadPath` continues from a
checkpoint's weights and learning rate with fresh Adam moments, as train.lua:78-81 does.

`-gpus N` trains data-parallel on GPUs gpuid .. gpuid+N-1: each rank draws its own `batchSize` dialogs per iteration, the
gradients are all-reduced inside the engine's Adam step (NCCL), an epoch is ceil(numTrainThreads / (N * batchSize))
iterations, the printed loss is the mean of the ranks' running losses, and only rank 0 writes files.

`-valIter N` also ranks the val split every N epochs (visdial_b200.validation, DESIGN §28): `<savePath>/val_log.json`, a
`[Val]` line, `<savePath>/model_best.t7` at each strict improvement of the selection metric, and with `-valPatience P` an
early stop after P validations without one (model_final.t7 is written as at the normal end)."""
from __future__ import annotations

import hashlib
import math
import os
import time

from . import cli


def standard_iteration(model, dl, opt, say):
    """train's iteration and epoch: Model.trainIteration, over the training split's dialogs.  Returns (the iteration
    function, the number of items an epoch covers)."""
    return (lambda: model.trainIteration(dl)), model.params["numTrainThreads"]


def main(opt: dict, rank: int = 0, world: int = 1, iteration=standard_iteration):
    """`iteration(model, dataloader, opt, say)` gives the loop its step and epoch size (standard_iteration: train's)."""
    from . import dist as vdist
    from .checkpoint import load_checkpoint
    say = (lambda *a: print(*a, flush=True)) if rank == 0 else (lambda *a: None)
    say(opt)                                                                        # train.lua:9
    ck = None
    if opt["loadPath"]:                                                             # :32-42
        ck = load_checkpoint(opt["loadPath"])
        mp = cli.adopt_checkpoint_model(opt, ck, gpuid=opt["gpuid"], batchSize=opt["batchSize"])
    else:
        mp = cli.model_params(opt)                                                  # :27
    mp["vocabSize"] = cli.vocab_size(opt)                                           # :55-59 (the dataloader's count)
    validating = opt.get("valIter", 0) > 0                                          # the val split is read for it only
    model, dl = cli.build(mp, opt, rank, world, ["train", "val"] if validating else ["train"], ck)   # :47-48,76-81
    vdist.attach_engine(model.engine, rank, world)
    p = model.params
    # (numValThreads is not recorded: the val split is loaded only to validate, and the checkpoints' modelParams are
    # those of a run without it)
    p.update({k: getattr(dl, k) for k in ("numTrainThreads", "numTestThreads", "vocabSize",
                                          "maxQuesCount", "maxQuesLen", "maxAnsLen") if hasattr(dl, k)})
    if validating:                              # the dataloader's widths are its last split's: record the train split's
        p.update(maxQuesLen=int(dl.corpus["train"].desc.maxQuesLen), maxAnsLen=int(dl.corpus["train"].desc.maxAnsLen))
    p["gpuid"] = opt["gpuid"]
    savePath = opt["savePath"]                                                      # :62-65
    if rank == 0:
        os.makedirs(savePath, exist_ok=True)
    step, epoch_items = iteration(model, dl, opt, say)
    validate = None
    if validating:
        from .validation import Validator
        validate = Validator(model, dl, opt, rank, world, say)
    numIterPerEpoch = p["numIterPerEpoch"] = math.ceil(epoch_items / (world * p["batchSize"]))   # :68-69
    say("\n%d iter per epoch." % numIterPerEpoch)
    say("Training..")
    saveEvery = int(p["saveIter"]) * numIterPerEpoch
    valEvery = int(opt.get("valIter", 0)) * numIterPerEpoch
    for it in range(1, int(p["numEpochs"]) * numIterPerEpoch + 1):                  # :90-117
        step()
        if saveEvery > 0 and it % saveEvery == 0 and rank == 0:
            model.save(os.path.join(savePath, "model_epoch_%d.t7" % (it // numIterPerEpoch)))
        if it % 100 == 0:
            loss = vdist.mean_over_ranks(model.runningLoss, world) if world > 1 else model.runningLoss
            say("[%s][Epoch:%.02f][Iter:%d][Loss:%.05f][lr:%f]" % (time.strftime("%c"), it / numIterPerEpoch, it, loss,
                                                                   model.optims["learningRate"]))
        if valEvery > 0 and it % valEvery == 0 and validate(it, it // numIterPerEpoch):
            break
    if validate is not None:
        validate.report_best()
    if world > 1:
        # every rank applied the same all-reduced gradient: a rank whose weights differ from rank 0's would mean that the
        # final checkpoint does not describe what was trained, so it is not written
        digests = vdist.gather_objects([hashlib.sha256(model.engine.get_parameters().tobytes()).hexdigest()], world)
        if len(set(digests)) != 1:
            raise RuntimeError("the ranks' weights differ after training: %s" % digests)
        say("weights identical on %d ranks" % world)
    if rank == 0:
        model.save(os.path.join(savePath, "model_final.t7"), final=True)           # :120-121
    dl.close()
    model.engine.close()


if __name__ == "__main__":
    cli.run("visdial_b200.train", "main", cli.train_opts())
