"""`python -m visdial_b200.ndcg -ranks logs/ranks.json -denseAnnotations <file>`: NDCG of a ranks file on the VisDial v1.0
dense relevance annotations, the leaderboard's metric (what EvalAI computes from the same file).

The ranks file is the {image_id, round_id, ranks} list `evaluate -split val -saveRanks` writes (without -useGt: every round,
100 ranks each).  Prints the NDCG and the number of annotated rounds scored; exits non-zero, printing no result, when an
annotated round is missing from the ranks file.  Host arithmetic only: it needs no GPU."""
from __future__ import annotations

import argparse
import json
import sys

from . import dense


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(prog="python -m visdial_b200.ndcg")
    ap.add_argument("-ranks", default="logs/ranks.json", help="ranks file written by evaluate -saveRanks")
    ap.add_argument("-denseAnnotations", default="data/visdial_1.0_val_dense_annotations.json",
                    help="dense relevance annotations (gt_relevance or relevance per entry)")
    opt = ap.parse_args(argv)
    with open(opt.ranks) as f:
        table = json.load(f)
    K = len(table[0]["ranks"]) if table else 100
    try:
        ann = dense.read(opt.denseAnnotations, K)
        value = dense.score_ranks(table, ann)
    except (KeyError, ValueError) as e:
        print("ndcg: %s" % (e.args[0] if e.args else e), file=sys.stderr)
        return 1
    if ann.skipped:
        print("%d annotated entries with all relevances 0 skipped" % ann.skipped)
    print("NDCG: %f" % value)
    print("Rounds scored: %d" % len(ann))
    return 0


if __name__ == "__main__":
    sys.exit(main())
