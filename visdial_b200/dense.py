"""VisDial v1.0 dense relevance annotations and the NDCG metric (host only: no GPU, no engine).

An annotation file is a JSON list of entries {image_id, round_id, gt_relevance | relevance}: one annotated round per dialog
(round_id 1-based), with a relevance in [0, 1] for each of the numOptions answer options.  The val file
(visdial_1.0_val_dense_annotations.json) uses `gt_relevance`, the train sample (visdial_1.0_train_dense_sample.json)
`relevance`; both keys are accepted (written from the published challenge code, not checked against the real files)."""
from __future__ import annotations

import json
from typing import Optional, Sequence

import numpy as np

from .utils import image_id


class DenseAnnotations:
    """The usable entries of one annotation file, in file order: image_id (M,), 1-based round_id (M,), relevance (M, K)
    float32, and, when read against a split's image table, `dialog` (M,) = the 0-based dialog index of each entry.
    `skipped` counts the entries whose relevances sum to 0 (NDCG 0/0, soft target undefined)."""

    def __init__(self, image_ids, round_ids, relevance, dialog, skipped):
        self.image_id = np.asarray(image_ids, dtype=np.int64)
        self.round_id = np.asarray(round_ids, dtype=np.int64)
        self.relevance = relevance
        self.dialog = dialog
        self.skipped = skipped

    def __len__(self):
        return len(self.round_id)


def read(path: str, num_options: int, unique_img: Optional[Sequence] = None,
         num_rounds: Optional[Sequence[int]] = None) -> DenseAnnotations:
    """Reads and checks an annotation file.  With `unique_img` (the split's `unique_img_<split>` of visdial_params.json)
    every image is mapped to its dialog index and its round checked against that dialog's `num_rounds` (all of
    maxQuesCount = 10 when None).  Raises ValueError naming the entry for an unknown image, a duplicate (image, round), a
    round outside 1..num_rounds, a relevance list that is not numOptions long, or a negative or non-finite relevance."""
    with open(path) as f:
        entries = json.load(f)
    if not isinstance(entries, list):
        raise ValueError("%s: a dense annotation file is a JSON list of entries" % path)
    index = {image_id(x): i for i, x in enumerate(unique_img)} if unique_img is not None else None
    seen = set()
    iids, rids, rels, dialogs, skipped = [], [], [], [], 0
    for n, e in enumerate(entries):
        where = "%s: entry %d (image_id %r, round_id %r)" % (path, n, e.get("image_id"), e.get("round_id"))
        rel = e.get("gt_relevance", e.get("relevance"))
        if rel is None or "image_id" not in e or "round_id" not in e:
            raise ValueError("%s: needs image_id, round_id and gt_relevance or relevance" % where)
        iid, rid = image_id(e["image_id"]), int(e["round_id"])
        if (iid, rid) in seen:
            raise ValueError("%s: duplicate of an earlier entry" % where)
        seen.add((iid, rid))
        d = None
        if index is not None:
            if iid not in index:
                raise ValueError("%s: image not in the split" % where)
            d = index[iid]
        n_rounds = int(num_rounds[d]) if (num_rounds is not None and d is not None) else 10
        if not 1 <= rid <= n_rounds:
            raise ValueError("%s: round_id outside 1..%d" % (where, n_rounds))
        r = np.asarray(rel, dtype=np.float64)
        if r.shape != (num_options,):
            raise ValueError("%s: %d relevances, numOptions is %d" % (where, r.size, num_options))
        if not np.isfinite(r).all() or (r < 0).any():
            raise ValueError("%s: relevances must be finite and >= 0" % where)
        if r.sum() == 0:
            skipped += 1
            continue
        iids.append(iid)
        rids.append(rid)
        rels.append(r.astype(np.float32))
        dialogs.append(d)
    relevance = np.stack(rels) if rels else np.zeros((0, num_options), np.float32)
    dialog = np.asarray(dialogs, dtype=np.int64) if index is not None else None
    return DenseAnnotations(iids, rids, relevance, dialog, skipped)


def ndcg(ranks: np.ndarray, relevance: np.ndarray) -> float:
    """Mean NDCG of rounds (M, K) as the VisDial v1.0 challenge defines it: k = the number of options with a nonzero
    relevance, DCG = sum_{i<k} rel[option at predicted position i] / log2(i + 2) with positions from the 1-based ranks
    (rank 1 first), IDCG = the same sum over the relevances sorted in descending order."""
    ranks = np.asarray(ranks, dtype=np.int64)
    rel = np.asarray(relevance, dtype=np.float64)
    M, K = rel.shape
    if M == 0:
        raise ValueError("no annotated rounds to score")
    disc = 1.0 / np.log2(np.arange(K, dtype=np.float64) + 2.0)
    k = (rel != 0).sum(1)
    keep = np.arange(K)[None, :] < k[:, None]
    predicted = np.take_along_axis(rel, np.argsort(ranks, axis=1, kind="stable"), axis=1)
    ideal = -np.sort(-rel, axis=1)
    dcg = (predicted * disc * keep).sum(1)
    idcg = (ideal * disc * keep).sum(1)
    return float((dcg / idcg).mean())


def score_ranks(table, dense: DenseAnnotations) -> float:
    """NDCG of a {image_id, round_id, ranks} table (what `evaluate -saveRanks` writes) on the annotated rounds.  Raises
    KeyError for an annotated round the table lacks and ValueError for a rank list that is not a permutation of 1..K."""
    K = dense.relevance.shape[1]
    by_round = {(image_id(e["image_id"]), int(e["round_id"])): e["ranks"] for e in table}
    ranks = np.empty((len(dense), K), dtype=np.int64)
    for i, key in enumerate(zip(dense.image_id.tolist(), dense.round_id.tolist())):
        if key not in by_round:
            raise KeyError("annotated round (image_id %d, round_id %d) is missing from the ranks" % key)
        r = np.asarray(by_round[key], dtype=np.int64)
        if r.shape != (K,) or not np.array_equal(np.sort(r), np.arange(1, K + 1)):
            raise ValueError("ranks of (image_id %d, round_id %d) are not a permutation of 1..%d" % (key + (K,)))
        ranks[i] = r
    return ndcg(ranks, dense.relevance)
