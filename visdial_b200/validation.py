"""Validation while training (DESIGN §28): `-valIter N` ranks the val split every N epochs inside train, finetune and
finetune_gen.

One eval-mode pass over this rank's share of val computes every round's full option rank list (what `evaluate` without
`-useGt` writes); the ground-truth rank of a round is the entry of its answer in that list, so the pass also gives what
`evaluate -useGt` ranks, and the annotated rounds' lists give the NDCG `ndcg` computes.  Rank 0 gathers the shares in rank
order, prints one `[Val]` line, rewrites `<savePath>/val_log.json`, writes `<savePath>/model_best.t7` when the selection
metric (NDCG with -valDenseAnnotations, else MRR) improves strictly, and decides whether the run stops
(`-valPatience`); the decision reaches every rank over the gloo group.  The pass only reads the weights: the training
RNG, the iteration and dropout seed, the optimiser state, the learning rate and the running loss are left as they were."""
from __future__ import annotations

import os
import time

import numpy as np

from . import cli
from . import dense as vdense
from .utils import processRanks

METRIC_NAMES = {"meanRR": "MRR", "ndcg": "NDCG"}


class Selection:
    """The best-so-far bookkeeping of a run's validations.  A value strictly above the best so far is an improvement (a
    tie is not); with patience P > 0, `stop` holds once P validations in a row brought none."""

    def __init__(self, patience: int = 0):
        self.patience = int(patience)
        self.best = None
        self.best_epoch = None
        self.since_best = 0

    def record(self, epoch: int, value: float) -> bool:
        """Takes one validation's selection metric; True when it is the new best."""
        if self.best is None or value > self.best:
            self.best, self.best_epoch, self.since_best = value, epoch, 0
            return True
        self.since_best += 1
        return False

    @property
    def stop(self) -> bool:
        return self.patience > 0 and self.since_best >= self.patience


def gt_ranks(full: np.ndarray, answer_index: np.ndarray) -> np.ndarray:
    """The ground-truth rank of every round, (dialogs, rounds), from the full rank lists (dialogs, rounds, numOptions) and
    the 1-based answer indices (dialogs, rounds): what vd_retrieve with use_gt computes from the same scores."""
    idx = np.asarray(answer_index, np.int64)[..., None] - 1
    return np.take_along_axis(full, idx, axis=2)[..., 0]


def annotated_rows(full: np.ndarray, first: int, ann) -> tuple:
    """The annotated rounds that fall in a share of the split starting at dialog `first`: (their positions in `ann`,
    their rank lists (M, numOptions))."""
    sel = np.nonzero((ann.dialog >= first) & (ann.dialog < first + len(full)))[0]
    return sel, full[ann.dialog[sel] - first, ann.round_id[sel] - 1]


def metrics(gt: np.ndarray, dense_ranks=None, relevance=None) -> dict:
    """utils.processRanks of the ground-truth ranks (r@1, r@5, r@10, medianR, meanR, meanRR) and, given the annotated
    rounds' rank lists in annotation order with their relevances, the NDCG of dense.score_ranks as "ndcg"."""
    out = processRanks(gt, verbose=False)
    if relevance is not None:
        out["ndcg"] = vdense.ndcg(dense_ranks, relevance)
    return out


class Validator:
    """train.main's validation: `validator(it, epoch)` runs one pass and returns whether training stops there.  Built
    before the first training step, so that the val dense annotations are read against the split up front."""

    def __init__(self, model, dl, opt: dict, rank: int, world: int, say):
        self.model, self.dl, self.rank, self.world, self.say = model, dl, rank, world, say
        lo, hi = dl.part["val"]
        self.first = lo
        self.answer_index = dl.corpus["val"].raw["ans_index"][lo:hi]
        if (self.answer_index < 1).any():
            raise ValueError("ans_index_val has rounds without a ground-truth answer (index 0)")
        self.ann = None
        if opt.get("valDenseAnnotations"):
            self.ann = vdense.read(opt["valDenseAnnotations"], model.params["numOptions"], unique_img=dl.unique_img_val,
                                   num_rounds=getattr(dl, "val_num_rounds", None))
        self.metric = "ndcg" if self.ann is not None else "meanRR"
        self.selection = Selection(opt.get("valPatience", 0))
        self.log = []
        self.log_path = os.path.join(opt["savePath"], "val_log.json")
        self.best_path = os.path.join(opt["savePath"], "model_best.t7")

    def rank_lists(self) -> np.ndarray:
        """This rank's share of val: every round's full rank list, (dialogs, rounds, numOptions), in one eval-mode pass
        of the training batch size (Model._rank_walk switches the engine to evaluate mode and back).

        Every encoder forward zeroes the word embedding's pad row in W (LookupTableMaskZero), which an Adam step may have
        moved since; the row is put back afterwards, so that the pass leaves W, and the checkpoints written after it, bit
        for bit as they were."""
        from ._lib import check
        p, eng = self.model.params, self.model.engine
        R, K = p["maxQuesCount"], p["numOptions"]
        w, _ = eng.param_buffers()
        pad = np.empty(int(p["embedSize"]), np.float32)
        check(eng.lib.vd_memcpy_d2h(eng.h, pad.ctypes.data, w, pad.nbytes))
        try:
            parts = [r.reshape(-1, R, K) for r in self.model._rank_walk(self.dl, "val", False)]
        finally:
            eng.upload(w, pad)
        return np.concatenate(parts, 0) if parts else np.zeros((0, R, K), np.int32)

    def __call__(self, it: int, epoch: int) -> bool:
        from . import dist as vdist
        t0 = time.perf_counter()
        full = self.rank_lists()
        gt = gt_ranks(full, self.answer_index)
        pos = rows = None
        if self.ann is not None:
            pos, rows = annotated_rows(full, self.first, self.ann)
        if self.world > 1:
            gt = vdist.gather_ranks(gt, self.rank, self.world)
            if self.ann is not None:
                shares = vdist.gather_objects([(pos, rows)], self.world)
                pos = np.concatenate([s[0] for s in shares])
                rows = np.concatenate([s[1] for s in shares])
        stop = False
        if self.rank == 0:
            relevance = None
            if self.ann is not None:
                rows = rows[np.argsort(pos, kind="stable")]              # annotation order, as dense.score_ranks sums
                relevance = self.ann.relevance
            m = metrics(gt, rows, relevance)
            entry = dict({"epoch": epoch, "iter": it}, **m, seconds=time.perf_counter() - t0)
            self.log.append(entry)
            self.say("[%s][Epoch:%d][Val] R@1 %.5f R@5 %.5f R@10 %.5f MeanR %.5f MRR %.5f%s" % (
                time.strftime("%c"), epoch, m["r@1"], m["r@5"], m["r@10"], m["meanR"], m["meanRR"],
                " NDCG %.5f" % m["ndcg"] if "ndcg" in m else ""))
            cli.write_json(self.log_path, self.log)
            if self.selection.record(epoch, m[self.metric]):
                self.model.save(self.best_path)
            stop = self.selection.stop
            if stop:
                self.say("Stopping early: %s has not improved for %d validations" % (
                    METRIC_NAMES[self.metric], self.selection.since_best))
        if self.world > 1:
            stop = vdist.broadcast_object(stop, self.rank)
        return stop

    def report_best(self):
        if self.selection.best_epoch is not None:
            self.say("Best validation: epoch %d (%s %.5f), %s" % (self.selection.best_epoch, METRIC_NAMES[self.metric],
                                                                  self.selection.best, self.best_path))
