"""CPU side of dialog sessions (DESIGN §19): the question tokenizer on hand cases, and the chat command's options."""
import numpy as np
import pytest

from visdial_b200 import cli
from visdial_b200.chat import parse
from visdial_b200.utils import question_ids, question_words

W2I = {"is": 1, "it": 2, "?": 3, "UNK": 4, "ca": 5, "n't": 6, "dog": 7, "'s": 8, ",": 9, "red": 10, "do": 11}


@pytest.mark.parametrize("text,words", [
    ("Is it red", ["is", "it", "red", "?"]),
    ("is it red?", ["is", "it", "red", "?"]),                    # a typed '?' is not doubled
    ("is it red ??", ["is", "it", "red", "?"]),
    ("  IS IT RED?  ", ["is", "it", "red", "?"]),
    ("can't you see, the dog's tail", ["ca", "n't", "you", "see", ",", "the", "dog", "'s", "tail", "?"]),
    ("don't they're we've you'll i'd i'm", ["do", "n't", "they", "'re", "we", "'ve", "you", "'ll", "i", "'d", "i", "'m", "?"]),
    ("what (color) is it.", ["what", "(", "color", ")", "is", "it", ".", "?"]),
    ("", ["?"]),
])
def test_question_words(text, words):
    assert question_words(text) == words


def test_question_ids_unk_alignment_and_cut():
    assert question_ids("is it blue", W2I, 6).tolist() == [0, 0, 1, 2, 4, 3]          # UNK, right-aligned
    assert question_ids("can't the dog", W2I, 8).tolist() == [0, 0, 0, 5, 6, 4, 7, 3]
    assert question_ids("is it very red", W2I, 3).tolist() == [1, 2, 4]                # the first maxQuesLen tokens
    assert question_ids([0, 0, 7, 2], W2I, 3).tolist() == [0, 7, 2]                    # token ids: pads dropped, re-aligned
    assert question_ids([], W2I, 3).tolist() == [0, 0, 0]
    assert question_ids("is it", W2I, 4).dtype == np.int32
    with pytest.raises(ValueError):
        question_ids("is it blue", {k: v for k, v in W2I.items() if k != "UNK"}, 5)


def test_chat_options():
    opt = parse(["-loadPath", "m.t7", "-split", "test", "-imageIds", "3,5", "-questions", "q.json", "-beamSize", "3"])
    assert opt["split"] == "test" and opt["imageIds"] == "3,5" and opt["questions"] == "q.json" and opt["beamSize"] == 3
    defaults = parse([])
    for name, default, _ in cli.GENERATE_OPTIONS:                                      # generate's options and defaults
        assert defaults[name] == default, name
    assert defaults["split"] == "val" and defaults["questions"] == "" and defaults["gpus"] == 1
    with pytest.raises(SystemExit) as e:
        parse(["-gpus", "2"])
    assert e.value.code == 2
    with pytest.raises(SystemExit):
        parse(["-history", "generated"])                                               # not a chat option
