"""utils.lua counterparts that stay on the host."""
import re

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


_PUNCT = re.compile(r"([?!.,;:()\[\]{}\"`])")
_CONTRACTION = re.compile(r"(?<=\w)(n't|'s|'re|'ve|'ll|'d|'m)\b")


def question_words(text: str) -> list:
    """A typed question as prepro.py's `word_tokenize(q + '?')` splits the dataset's questions, on the cases that matter
    for them: lower case; punctuation split off; the Treebank contractions n't 's 're 've 'll 'd 'm split from their word
    ("can't" -> "ca n't"); exactly one trailing '?' (one the user typed is not doubled)."""
    t = text.strip().lower()
    while t.endswith("?"):
        t = t[:-1].rstrip()
    t = _CONTRACTION.sub(r" \1", _PUNCT.sub(r" \1 ", t))
    return t.split() + ["?"]


def question_ids(question, word2ind: dict, width: int) -> np.ndarray:
    """One question row as a batch's ques_fwd holds it: (width,) int32, right-aligned, zero-padded.  `question` is text
    (question_words; words missing from word2ind become UNK) or a list of token ids; either is cut to its first `width`
    tokens, as prepro.py cuts questions to maxQuesLen."""
    if isinstance(question, str):
        unk = word2ind.get("UNK")
        ids = []
        for w in question_words(question):
            if w not in word2ind and unk is None:
                raise ValueError("%r is not in the vocabulary, which has no UNK" % w)
            ids.append(word2ind.get(w, unk))
    else:
        ids = [int(t) for t in question if int(t) != 0]
    ids = ids[:width]
    row = np.zeros(width, np.int32)
    if ids:
        row[width - len(ids):] = ids
    return row


def answer_ids(answer, word2ind: dict, width: int) -> np.ndarray:
    """One answer row as the corpus's `ans` holds it: (width,) int32, left-aligned, zero-padded.  `answer` is text,
    split by question_words' rules without the trailing '?' (words missing from word2ind become UNK; unverified against
    nltk), or a list of token ids (pads dropped); either is cut to its first `width` tokens, as prepro.py cuts answers to
    maxAnsLen."""
    if isinstance(answer, str):
        unk = word2ind.get("UNK")
        ids = []
        for w in question_words(answer)[:-1]:
            if w not in word2ind and unk is None:
                raise ValueError("%r is not in the vocabulary, which has no UNK" % w)
            ids.append(word2ind.get(w, unk))
    else:
        ids = [int(t) for t in answer if int(t) != 0]
    ids = ids[:width]
    row = np.zeros(width, np.int32)
    row[:len(ids)] = ids
    return row


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
