"""TEST INFRASTRUCTURE ONLY.  Host restatement of the history that vd_gen_dialog_beam_search / vd_gen_dialog_sample feed the
encoder (DESIGN §17): round 0 is the batch's round-0 row, and round r's question and answer are written into row r+1 by
dataloader.lua:202-278's rule — Q ++ A right-aligned, or row r ++ <END> ++ Q ++ A for the concatenated history — with the
answer cut to max_ans_len words, no answer after a question of pads, the rightmost W words of every row kept, and an empty
row r leaving row r+1 empty (utils.lua:20-22's `break`)."""
import numpy as np


def row_words(row) -> list:
    """the words of a right-aligned row: its trailing non-pad tokens"""
    row = [int(t) for t in row]
    n = 0
    while n < len(row) and row[len(row) - 1 - n] != 0:
        n += 1
    return row[len(row) - n:]


def beam_words(answer, length) -> list:
    """A of a beam: the non-pad words between <START> and <END> of the best finished hypothesis (none: length 0)"""
    return [int(t) for t in answer[1:max(int(length) - 1, 1)] if t != 0] if length > 0 else []


def sample_words(answer, end) -> list:
    """A of a sample (answer row with column 0 = <START>): the words before the first <END>"""
    out = []
    for t in answer[1:]:
        if t == end:
            break
        if t != 0:
            out.append(int(t))
    return out


def right_aligned(words, W) -> np.ndarray:
    out = np.zeros(W, np.int32)
    words = list(words)[-W:] if W > 0 else []
    if words:
        out[W - len(words):] = words
    return out


def next_row(prev, q_words, a_words, concat: bool, end: int, W: int, max_ans_len: int) -> np.ndarray:
    """row r+1 from row r, round r's question words and answer words"""
    p = row_words(prev)
    if not p:
        return np.zeros(W, np.int32)
    a = list(a_words)[:max_ans_len] if q_words else []
    return right_aligned((p + [end] if concat else []) + list(q_words) + a, W)


def dialog_history(row0, ques, answers, concat: bool, end: int, W: int, max_ans_len: int) -> np.ndarray:
    """(R, W) history of one dialog: row0 its round-0 row, ques (R, Tq) right-aligned questions, answers R word lists
    (the last one is never written)"""
    R = len(ques)
    h = np.zeros((R, W), np.int32)
    h[0] = right_aligned(row_words(row0), W)
    for r in range(R - 1):
        h[r + 1] = next_row(h[r], row_words(ques[r]), answers[r], concat, end, W, max_ans_len)
    return h
