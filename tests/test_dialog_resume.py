"""Resuming conversations without a device (DESIGN §21): serve_step's join lines with a history, the answer tokenizer, and
the transcript bookkeeping DialogPool.reopen replays."""
import numpy as np
import pytest

from visdial_b200 import chat
from visdial_b200.model import history_answer, transcript_arrays
from visdial_b200.utils import answer_ids


def _step(lines, convs, queues, free, images=(1, 2, 3), R=4):
    return chat.serve_step(lines, convs, queues, free, set(images), R)


def test_serve_join_with_history():
    convs, queues = {}, {}
    h = [["is it red?", "yes"], [[5, 6], [7]]]
    joins, leaves, errors, asks = _step([{"id": "a", "image_id": 1, "history": h, "question": "q2"},
                                         {"id": "b", "image_id": 2, "question": "p0"},
                                         {"id": "c", "image_id": 3, "history": [], "question": "r0"}], convs, queues, 4)
    assert joins == [("a", 1, h), ("b", 2), ("c", 3, [])] and leaves == [] and errors == []
    assert asks == [("a", "q2"), ("b", "p0"), ("c", "r0")]


def test_serve_history_refusals_change_nothing():
    convs, queues = {"a": 0}, {"a": ["pending"]}
    lines = [{"id": "a", "history": [["q", "a"]], "question": "x"},          # an open id
             {"id": "b", "image_id": 1, "history": [["q", "a"]] * 4},      # R rounds
             {"id": "c", "image_id": 1, "history": [["q"]]},               # malformed
             {"id": "d", "image_id": 1, "history": "q a"},
             {"id": "e", "image_id": 1, "history": [[[1, "x"], "a"]]},
             {"id": "f", "image_id": 1, "history": [[True, "a"]]}]
    joins, leaves, errors, asks = _step(lines, convs, queues, 3)
    assert joins == [] and leaves == [] and [e[0] for e in errors] == ["a", "b", "c", "d", "e", "f"]
    assert "first line" in errors[0][1] and "4 rounds" in errors[1][1]
    assert convs == {"a": 0} and asks == [("a", "pending")]


def test_serve_history_join_and_leave_in_one_step():
    convs, queues = {"a": 0}, {}
    lines = [{"id": "a", "leave": True}, {"id": "b", "image_id": 2, "history": [["q", "a"]], "question": "n"},
             {"id": "c", "image_id": 3, "history": [["q", "a"]]}, {"id": "c", "leave": True}]
    joins, leaves, errors, asks = _step(lines, convs, queues, 1)
    assert leaves == [0] and joins == [("b", 2, [["q", "a"]])] and errors == []
    assert asks == [("b", "n")] and set(convs) == {"b"}


def test_answer_ids():
    w2i = {"yes": 1, "it": 2, "is": 3, "n't": 4, "ca": 5, ",": 6, "UNK": 7, "?": 8, "red": 9}
    assert answer_ids("Yes, it is", w2i, 5).tolist() == [1, 6, 2, 3, 0]
    assert answer_ids("it isn't red?", w2i, 6).tolist() == [2, 3, 4, 9, 0, 0]   # no trailing '?'
    assert answer_ids("it is purple", w2i, 3).tolist() == [2, 3, 7]
    assert answer_ids("yes it is red", w2i, 2).tolist() == [1, 2]                 # cut to maxAnsLen
    assert answer_ids([0, 9, 0, 1], w2i, 3).tolist() == [9, 1, 0]
    assert answer_ids("", w2i, 2).tolist() == [0, 0]
    with pytest.raises(ValueError):
        answer_ids("purple", {"red": 1}, 2)


def test_transcript_bookkeeping():
    end = 20
    assert history_answer(np.asarray([19, 4, 0, 5, 20, 0]), end, 5) == [4, 5]          # beam: between <START> and <END>
    assert history_answer(np.asarray([19, 4, 20, 0]), end, 0) == []                   # no finished hypothesis
    assert history_answer(np.asarray([4, 0, 5, 20, 7]), end) == [4, 5]                # sample / pool / corpus rows
    q0, q1 = np.asarray([0, 3, 4], np.int32), np.asarray([5, 6, 7], np.int32)
    rounds, ques, ans = transcript_arrays([([q0, q1], [[1, 2, 3], []]), ([], [])], 4, 3)
    assert rounds.tolist() == [2, 0] and ques.shape == (2, 4, 3) and ans.shape == (2, 4, 3)
    assert ques[0, 0].tolist() == [0, 3, 4] and ques[0, 1].tolist() == [5, 6, 7] and not ques[0, 2:].any() and not ques[1].any()
    assert ans[0, 0].tolist() == [1, 2, 3] and not ans[0, 1:].any() and not ans[1].any()
    assert transcript_arrays([([], [])], 4, 3)[2].shape == (1, 4, 1)
    with pytest.raises(ValueError):
        transcript_arrays([([q0] * 4, [[1]] * 4)], 4, 3)                               # R rounds: nothing left to ask
    with pytest.raises(ValueError):
        transcript_arrays([([q0], [])], 4, 3)
