"""`python -m visdial_b200.finetune_gen -loadPath <gen checkpoint> -denseAnnotations <file> ...`: fine-tune a generative
model on VisDial v1.0's dense relevance annotations (DESIGN §16).

Options are finetune's (visdial_b200.cli.FINETUNE_OPTIONS).  Each iteration draws `batchSize` annotated dialogs per rank
and takes one step of the soft-target cross-entropy between each dialog's normalised relevances and the log-likelihoods
of its annotated round's options under the decoder (vd_forward_backward_dense_gen) -- the scores `evaluate` ranks gen
models by, so the step optimises the ranking `ndcg` scores.  The epoch, `-loadPath`, checkpoints, log lines, `-gpus N`
and the weight check across ranks are finetune's.  A discriminative model is refused before any GPU work: its command
is visdial_b200.finetune."""
from __future__ import annotations

from . import cli, finetune, train


def dense_gen_iteration(model, dl, opt, say):
    """train.main's iteration hook: Model.trainIterationDenseGen over the annotated dialogs of the train split."""
    ann = finetune.read_annotations(model, dl, opt, say)
    return (lambda: model.trainIterationDenseGen(dl, ann)), len(ann)


def refuse_disc(opt: dict):
    """This command fine-tunes the gen decoder: say so before an engine is created."""
    decoder = opt["decoder"]
    if opt["loadPath"]:
        from .checkpoint import load_checkpoint
        decoder = load_checkpoint(opt["loadPath"])["modelParams"]["decoder"]
    if decoder != "gen":
        raise SystemExit("finetune_gen: this command fine-tunes gen models, this one has the %r decoder; "
                         "use python -m visdial_b200.finetune for disc models" % decoder)


def main(opt: dict, rank: int = 0, world: int = 1):
    refuse_disc(opt)
    train.main(opt, rank, world, iteration=dense_gen_iteration)


def finetune_gen_opts(argv=None):
    return cli.train_opts(argv, options=cli.FINETUNE_OPTIONS, prog="python -m visdial_b200.finetune_gen")


if __name__ == "__main__":
    opt = finetune_gen_opts()
    refuse_disc(opt)
    cli.run("visdial_b200.finetune_gen", "main", opt)
