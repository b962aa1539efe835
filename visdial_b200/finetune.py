"""`python -m visdial_b200.finetune -loadPath <disc checkpoint> -denseAnnotations <file> ...`: fine-tune a discriminative
model on VisDial v1.0's dense relevance annotations, the standard way to raise NDCG.

Options are train's (visdial_b200.cli.TRAIN_OPTIONS) plus `denseAnnotations` (default
data/visdial_1.0_train_dense_sample.json).  Each iteration draws `batchSize` annotated dialogs per rank and takes one step
of the soft-target cross-entropy between the disc scores of each dialog's annotated round and its normalised relevances
(vd_forward_backward_dense: the option LSTM runs on those rounds only).  An epoch is ceil(numAnnotated / (gpus *
batchSize)) iterations.  `-loadPath`, checkpoints, log lines, `-gpus N` and the weight check across ranks are train's.
A generative model is refused before any GPU work."""
from __future__ import annotations

from . import cli, train


def read_annotations(model, dl, opt, say):
    """opt's denseAnnotations read against the train split, with the counts finetune prints."""
    from . import dense
    K = model.params["numOptions"]
    ann = dense.read(opt["denseAnnotations"], K, unique_img=dl.unique_img_train,
                     num_rounds=getattr(dl, "train_num_rounds", None))
    if ann.skipped:
        say("%d annotated entries with all relevances 0 skipped" % ann.skipped)
    if len(ann) == 0:
        raise ValueError("%s has no usable annotated round" % opt["denseAnnotations"])
    say("%d annotated rounds" % len(ann))
    return ann


def dense_iteration(model, dl, opt, say):
    """train.main's iteration hook: Model.trainIterationDense over the annotated dialogs of the train split."""
    ann = read_annotations(model, dl, opt, say)
    return (lambda: model.trainIterationDense(dl, ann)), len(ann)


def refuse_gen(opt: dict):
    """The dense step exists for the disc decoder only: say so before an engine is created."""
    decoder = opt["decoder"]
    if opt["loadPath"]:
        from .checkpoint import load_checkpoint
        decoder = load_checkpoint(opt["loadPath"])["modelParams"]["decoder"]
    if decoder != "disc":
        raise SystemExit("finetune: dense fine-tuning needs a disc model, this one has the %r decoder" % decoder)


def main(opt: dict, rank: int = 0, world: int = 1):
    refuse_gen(opt)
    train.main(opt, rank, world, iteration=dense_iteration)


def finetune_opts(argv=None):
    return cli.train_opts(argv, options=cli.FINETUNE_OPTIONS, prog="python -m visdial_b200.finetune")


if __name__ == "__main__":
    opt = finetune_opts()
    refuse_gen(opt)
    cli.run("visdial_b200.finetune", "main", opt)
