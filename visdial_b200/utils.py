"""utils.lua counterparts that stay on the host."""
import numpy as np


def idToWords(vector, ind2word) -> str:
    """utils.lua:48-63: every non-pad id becomes ' ' + its word (so the text starts with a space); <START> is kept, and
    the walk stops after the first <END>."""
    sentence = ""
    nextWord = None
    for wordId in vector:
        wordId = int(wordId)
        if wordId > 0:
            nextWord = ind2word[wordId]
            sentence += " " + nextWord
        if nextWord == "<END>":
            break
    return sentence


def image_id(x):
    """dataloader.lua:42-44: `tonumber(string.match(name, '000%d+'))` on the json image names; ints pass through."""
    if isinstance(x, (int, np.integer)):
        return int(x)
    import re
    mt = re.search(r"000\d+", str(x))
    return int(mt.group(0)) if mt else x


def processRanks(ranks, verbose=True):
    """utils.lua:131-160: R@1/5/10, median, mean rank, MRR."""
    r = np.asarray(ranks, dtype=np.float64).reshape(-1)
    n = r.size
    out = {"r@1": float((r <= 1).sum()) / n, "r@5": float((r <= 5).sum()) / n, "r@10": float((r <= 10).sum()) / n,
           "medianR": float(np.median(r)), "meanR": float(r.mean()), "meanRR": float((1.0 / r).mean())}
    if verbose:
        print("\tNo. questions: %d" % n)
        for k in ("r@1", "r@5", "r@10", "medianR", "meanR", "meanRR"):
            print("\t%s: %f" % (k, out[k]))
    return out
