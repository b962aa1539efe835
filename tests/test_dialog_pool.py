"""The chat command's serve loop without a device (chat.serve_step, DESIGN §20): joins and leaves in arrival order, the
refused lines, and one ask of every conversation with a pending question, its oldest."""
from visdial_b200 import chat, cli


def _step(lines, convs, queues, free, images=(1, 2, 3)):
    return chat.serve_step(lines, convs, queues, free, set(images))


def test_first_line_joins_and_later_questions_wait():
    convs, queues = {}, {}
    joins, leaves, errors, asks = _step([{"id": "a", "image_id": 1, "question": "q1"}, {"id": "a", "question": "q2"},
                                         {"id": "b", "image_id": 2, "question": "p1"}], convs, queues, 4)
    assert joins == [("a", 1), ("b", 2)] and leaves == [] and errors == []
    assert asks == [("a", "q1"), ("b", "p1")] and queues == {"a": ["q2"]}
    convs.update(a=0, b=1)
    joins, leaves, errors, asks = _step([], convs, queues, 2)
    assert (joins, leaves, errors, asks) == ([], [], [], [("a", "q2")]) and queues == {}


def test_refused_lines():
    convs, queues = {"a": 0}, {}
    lines = [{"id": "x", "question": "q"},                      # unknown id without an image
             {"id": "y", "image_id": 9, "question": "q"},       # unknown image
             {"id": "z", "image_id": 1},                        # joins the last free slot, no question yet
             {"id": "w", "image_id": 2, "question": "q"},       # the pool is full
             {"id": "v", "leave": True},                        # unknown id
             {"question": "no id"}]
    joins, leaves, errors, asks = _step(lines, convs, queues, 1)
    assert joins == [("z", 1)] and asks == [] and leaves == []
    assert [e[0] for e in errors] == ["x", "y", "w", "v", None]
    assert "unknown id" in errors[0][1] and "image" in errors[1][1] and "full" in errors[2][1]


def test_joins_and_leaves_apply_in_arrival_order():
    convs, queues = {"a": 0, "b": 1}, {"a": ["old"]}
    # a full pool: c's first join is refused, a's leave frees the slot c's second join takes, and d finds the pool full
    lines = [{"id": "c", "image_id": 3, "question": "too early"}, {"id": "a", "leave": True},
             {"id": "c", "image_id": 3, "question": "c1"}, {"id": "d", "image_id": 1}]
    joins, leaves, errors, asks = _step(lines, convs, queues, 0)
    assert [e[0] for e in errors] == ["c", "d"] and all("full" in e[1] for e in errors)
    assert leaves == [0] and joins == [("c", 3)]
    assert asks == [("c", "c1")] and "a" not in convs and queues == {}
    # joined and left within one step: it never reaches the device, and its slot is free again
    convs, queues = {}, {}
    joins, leaves, errors, asks = _step([{"id": "e", "image_id": 1, "question": "q"}, {"id": "e", "leave": True},
                                         {"id": "f", "image_id": 2, "question": "r"}], convs, queues, 1)
    assert joins == [("f", 2)] and leaves == [] and errors == [] and asks == [("f", "r")]


def test_chat_options():
    names = [o[0] for o in cli.CHAT_OPTIONS]
    assert "serve" in names and "capacity" in names
    opt = chat.parse(["-serve", "1", "-capacity", "16"])
    assert opt["serve"] == 1 and opt["capacity"] == 16
    assert chat.parse([])["capacity"] == 128 and chat.parse([])["serve"] == 0
