"""`python -m visdial_b200.evaluate -loadPath ...`: evaluate.lua on the engine.

Options and defaults are those of evaluate.lua:15-30 (see visdial_b200.cli).  With `-useGt` it ranks the ground-truth
answer of every round and prints utils.processRanks (R@1/5/10, median and mean rank, MRR); without it, it computes the
full 100-option rank lists (the last round only on `-split test`, the EvalAI format).  `-saveRanks` writes the
{image_id, round_id, ranks} list as JSON to `saveRankPath`.

`-gpus N` ranks a contiguous share of the split on each of GPUs gpuid .. gpuid+N-1; rank 0 gathers the shares in rank
order, so what it prints and writes is what one GPU computes (exactly so in `-math fp32`)."""
from __future__ import annotations

import numpy as np

from . import cli


def rank_share(model, dl, split: str, use_gt: bool):
    """This rank's part of the evaluation: (ground-truth ranks (dialogs, rounds) or None, the {image_id, round_id, ranks}
    table).  A rank whose share of the split is empty (more GPUs than dialogs) contributes nothing."""
    if dl.numThreads[split] == 0:
        return (np.zeros((0, model.params["maxQuesCount"]), np.int32) if use_gt else None), []
    if not use_gt:
        return None, model.predict(dl, split)                                       # :100-101
    ranks = model.retrieve(dl, split)                                               # :98-99 (model.lua:142-189)
    # Model.retrieve(as_table=True) builds this table from the same matrix; the command needs both the matrix (the metrics
    # are computed once over every rank's share) and the table, so it calls the table step itself
    return ranks, model._round_table(dl, split, ranks, last_round_only=False)


def main(opt: dict, rank: int = 0, world: int = 1):
    from . import dist as vdist
    from .checkpoint import load_checkpoint
    from .utils import processRanks
    say = (lambda *a: print(*a, flush=True)) if rank == 0 else (lambda *a: None)
    split = opt["split"]
    if opt["useGt"] and split == "test":                                            # evaluate.lua:34-37
        say("Warning: No ground truth avaiilable in test split, changing useGt to false.")
        opt["useGt"] = False
    say(opt)
    ck = load_checkpoint(opt["loadPath"])                                           # :58-68
    mp = cli.adopt_checkpoint_model(opt, ck, batchSize=opt["batchSize"], useGt=opt["useGt"])
    model, dl = cli.build(mp, opt, rank, world, [split], ck)                        # :80-91
    say("Evaluating..")
    ranks, table = rank_share(model, dl, split, opt["useGt"])
    if world > 1:
        table = vdist.gather_objects(table, world)
        if ranks is not None:
            ranks = vdist.gather_ranks(ranks, rank, world)
    if ranks is not None and rank == 0:
        processRanks(ranks)
    if opt["saveRanks"] and rank == 0:                                              # :104-107
        say("Writing ranks to %s" % opt["saveRankPath"])
        cli.write_json(opt["saveRankPath"], table)
    dl.close()
    model.engine.close()


if __name__ == "__main__":
    cli.run("visdial_b200.evaluate", "main", cli.parse(cli.EVALUATE_OPTIONS, prog="python -m visdial_b200.evaluate"))
