"""`python -m visdial_b200.chat -loadPath ...`: talk to a model about an image, one question at a time (DESIGN §19).

Reads the model and data as `generate` does and opens a dialog session (Model.openDialogs) on the chosen images of
`-split`: their features and captions; each question is answered before the next is asked, and the model's own answers
become the history the next question is answered with.  Gen models answer with generate's beam search (`-beamSize`,
`-beamLen`; diverse with `-beamGroups` > 1 and `-diversity`, DESIGN §22; n-best lists ranked by length-normalised score
with `-nBest` and `-lengthPenalty`, DESIGN §24) or, with `-sampleWords 1`, by sampling
(truncated to the top `-topK` words and the top `-topP` of the probability, DESIGN §23); disc models with the best answer
of the split's answer pool.

With `-questions file.json` ({image_id: [question, ...]}, at most maxQuesCount per image; a question is text or a list of
token ids) every image of the file (or of `-imageIds`) is asked its questions, round by round, and
`<resultPath>/results.json` is written in generate's {opts, data} layout, which the visualiser in vis/ shows.  Without
it the command talks about one image (the first of `-imageIds`, else the split's first): it reads one question per line
from stdin and prints each answer.  One GPU only.

With `-serve 1` it serves many conversations at once from a dialog pool of `-capacity` slots (Model.openDialogPool,
DESIGN §20), reading JSON lines on stdin and writing JSON lines on stdout:
  in:  {"id": "u1", "image_id": 185565, "question": "is it sunny?"}   (the first line of an id joins it, with its image)
       {"id": "u2", "image_id": 185565, "history": [["is it sunny?", "yes"]], "question": "any people?"}
            (a first line may carry the rounds the conversation already had: it joins at round len(history); DESIGN §21)
       {"id": "u1", "leave": true}
  out: {"id", "round", "question", "answer", ...} for each answer (with -beamGroups > 1 also "alternatives": every group's
       finished answer as {"answer", "score"}, best first, the first being "answer"; with -nBest or -lengthPenalty also
       "normScore", and with -nBest > 1 "nbest": every group's finished answers as {"answer", "score", "normScore"}, best
       first, the first being "answer"); {"id", "error"} for a refused line (an unknown image, a
       full pool, an unknown id, a malformed history, one of maxQuesCount rounds or more, or one for an open id).  A
       conversation that has had maxQuesCount answers is left, its last answer with "done": true.
The server reads every line available without blocking, applies its joins and leaves in arrival order, then asks every
conversation with a pending question its oldest one, all in one device call (serve_step)."""
from __future__ import annotations

import json
import os
import select
import sys

from . import cli


def _image_index(dl, split: str) -> dict:
    img = getattr(dl, "unique_img_" + split, None)
    if img is None:
        raise ValueError("the data has no image ids for split %r" % split)
    from .utils import image_id
    return {image_id(x): i for i, x in enumerate(img)}


def _history_ok(h) -> bool:
    """a join line's "history": a list of [question, answer] pairs, each text or a list of token ids"""
    def turn(x):
        return isinstance(x, str) or (isinstance(x, list) and all(isinstance(t, int) and not isinstance(t, bool) for t in x))
    return isinstance(h, list) and all(isinstance(p, (list, tuple)) and len(p) == 2 and turn(p[0]) and turn(p[1]) for p in h)


def serve_step(lines, convs: dict, queues: dict, free: int, images, max_rounds: int = 10) -> tuple:
    """One step of the serve loop, without the device.  lines: the JSON objects read since the last ask, in arrival order;
    convs: the open conversations' ids (each mapped to its slot; None for one joined in this step); queues: {id: [pending
    question, ...]}; free: the free slots; images: the image ids conversations may join with; max_rounds: maxQuesCount.
    Updates convs and queues and returns (joins: the new conversations to join, (id, image_id), or (id, image_id,
    history) for a join line with a "history" of earlier rounds; leaves [slot] the slots to free; errors [(id, message)];
    asks [(id, question)]: each conversation with a pending question, with its oldest).  A line whose history is
    malformed, has max_rounds rounds or more, or names an open id is refused and changes nothing."""
    joins, leaves, errors = [], [], []
    for obj in lines:
        cid = obj.get("id") if isinstance(obj, dict) else None
        if cid is None:
            errors.append((None, "a line needs an id"))
            continue
        if "history" in obj:
            h = obj["history"]
            if cid in convs:
                errors.append((cid, "a history only comes with a conversation's first line"))
                continue
            if not _history_ok(h):
                errors.append((cid, "a history is a list of [question, answer] pairs"))
                continue
            if len(h) >= max_rounds:
                errors.append((cid, "a history of %d rounds or more leaves nothing to ask" % max_rounds))
                continue
        if obj.get("leave"):
            if cid not in convs:
                errors.append((cid, "unknown id"))
                continue
            if convs[cid] is None:                         # joined in this step: it never reaches the device
                joins = [j for j in joins if j[0] != cid]
            else:
                leaves.append(convs[cid])
            del convs[cid]
            queues.pop(cid, None)
            free += 1
            continue
        if cid not in convs:
            if "image_id" not in obj:
                errors.append((cid, "unknown id"))
                continue
            if obj["image_id"] not in images:
                errors.append((cid, "unknown image %r" % (obj["image_id"],)))
                continue
            if free < 1:
                errors.append((cid, "the pool is full"))
                continue
            free -= 1
            convs[cid] = None
            joins.append((cid, obj["image_id"], [list(p) for p in obj["history"]]) if "history" in obj else
                         (cid, obj["image_id"]))
        if obj.get("question") is not None:
            queues.setdefault(cid, []).append(obj["question"])
    asks = [(cid, q.pop(0)) for cid, q in queues.items() if q]
    for cid in [c for c, q in queues.items() if not q]:
        del queues[cid]
    return joins, leaves, errors, asks


class _Lines:
    """stdin's complete lines: read(block) returns those available now, waiting for the first one only when `block`"""

    def __init__(self, fd):
        self.fd, self.buf, self.eof = fd, b"", False

    def read(self, block: bool) -> list:
        while not self.eof:
            ready = b"\n" in self.buf and not select.select([self.fd], [], [], 0)[0]
            if ready or (not block and not select.select([self.fd], [], [], 0)[0]):
                break
            chunk = os.read(self.fd, 1 << 16)
            if not chunk:
                self.eof = True
            self.buf += chunk
        parts = self.buf.split(b"\n")
        self.buf = b"" if self.eof else parts.pop()
        return [p.decode() for p in parts if p.strip()]


def serve(model, dl, split: str, index: dict, params: dict, capacity: int, out=sys.stdout):
    """The -serve loop: JSON lines on stdin, answers as JSON lines on `out`, until stdin ends and nothing is pending."""
    from ._lib import VdError
    from .model import ranked_groups
    from .utils import idToWords
    pool = model.openDialogPool(dl, split, capacity, params)
    R = model.params["maxQuesCount"]
    convs, queues, free = {}, {}, capacity
    src = _Lines(sys.stdin.fileno())

    def emit(obj):
        out.write(json.dumps(obj) + "\n")
        out.flush()

    try:
        while True:
            raw = src.read(block=not queues)
            if not raw and not queues and src.eof:
                break
            objs = []
            for line in raw:
                try:
                    objs.append(json.loads(line))
                except ValueError:
                    objs.append({"id": None})
            joins, leaves, errors, asks = serve_step(objs, convs, queues, free, index, R)
            for cid, msg in errors:
                emit({"id": cid, "error": msg})
            if leaves:
                pool.leave(leaves)
            fresh = [j for j in joins if len(j) == 2]
            if fresh:
                for (cid, _), s in zip(fresh, pool.join([index[img] for _, img in fresh])):
                    convs[cid] = s
            for cid, img, history in (j for j in joins if len(j) == 3):    # joins at round len(history)
                try:
                    convs[cid] = pool.resume(index[img], history)
                except (ValueError, VdError) as e:                          # a word outside the vocabulary, a bad token id
                    del convs[cid]
                    queues.pop(cid, None)
                    emit({"id": cid, "error": str(e)})
            asks = [(cid, q) for cid, q in asks if cid in convs]
            free = capacity - len(convs)
            if not asks:
                continue
            got = pool.ask({convs[cid]: q for cid, q in asks})
            done = []
            for cid, q in asks:
                s = convs[cid]
                e = got[s]
                r = pool.round(s)
                line = {"id": cid, "round": r - 1, "question": idToWords(e["question"], dl.ind2word) if e else None,
                        "answer": idToWords(e["answer"], dl.ind2word).strip() if e else None}
                if e and "score" in e:
                    line["score"] = e["score"]
                if e and "normScore" in e:
                    line["normScore"] = e["normScore"]
                if e and "nbest" in e:
                    line["nbest"] = [{"answer": idToWords(x["answer"], dl.ind2word).strip(), "score": x["score"],
                                      "normScore": x["normScore"]} for x in e["nbest"]]
                if e and "groups" in e:
                    line["alternatives"] = [{"answer": idToWords(g["answer"], dl.ind2word).strip(), "score": g["score"]}
                                            for g in ranked_groups(e)]
                if r == R:
                    line["done"] = True
                    done.append(cid)
                emit(line)
            if done:
                pool.leave([convs.pop(c) for c in done])
                for c in done:
                    queues.pop(c, None)
                free = capacity - len(convs)
    finally:
        pool.close()


def parse(argv=None) -> dict:
    """CHAT_OPTIONS parsed as the other commands parse theirs; -gpus other than 1 is refused."""
    opt = cli.parse(cli.CHAT_OPTIONS, argv, prog="python -m visdial_b200.chat")
    if opt["gpus"] != 1:
        print("python -m visdial_b200.chat: error: chat runs on one GPU: -gpus must be 1 (see -h)", file=sys.stderr)
        raise SystemExit(2)
    return opt


def main(opt: dict, rank: int = 0, world: int = 1):
    from .checkpoint import load_checkpoint
    from .utils import idToWords
    ck = load_checkpoint(opt["loadPath"])
    mp = cli.adopt_checkpoint_model(opt, ck)
    split = opt["split"]
    model, dl = cli.build(mp, opt, 0, 1, [split], ck)
    try:
        index = _image_index(dl, split)
        asked = None
        if opt["questions"]:
            with open(opt["questions"]) as f:
                asked = {int(k): v for k, v in json.load(f).items()}
        ids = [int(x) for x in opt["imageIds"].split(",") if x.strip()] if opt["imageIds"] else \
            (list(asked) if asked is not None else [next(iter(index))])
        missing = [i for i in ids if i not in index]
        if missing:
            raise SystemExit("image ids not in split %s: %s" % (split, missing))
        params = {k: opt[k] for k in ("beamSize", "beamLen", "sampleWords", "temperature", "beamGroups", "diversity")}
        params.update({k: opt[k] for k in ("lengthPenalty", "nBest") if k in opt})
        if model.params["decoder"] == "gen":         # a disc pool's topK is its retrieval list: the truncation is gen's
            params.update({k: opt[k] for k in ("topK", "topP") if k in opt})
            params.update(cli.answer_rule_params(opt))
        R = model.params["maxQuesCount"]
        if opt["serve"]:
            serve(model, dl, split, index, params, opt["capacity"])
            return
        if asked is None:
            session = model.openDialogs(dl, split, [index[ids[0]]], params)
            if session.caption is not None:
                print("image %d: %s" % (ids[0], idToWords(session.caption[0], dl.ind2word).strip()), flush=True)
            for line in sys.stdin:
                if not line.strip():
                    continue
                e = session.ask([line.strip()])[0]
                print(idToWords(e["answer"], dl.ind2word).strip() if e else "(no answer within -beamLen)", flush=True)
                if session.round == R:
                    break
            session.close()
            return
        qs = [asked.get(i, []) for i in ids]
        if any(len(q) > R for q in qs):
            raise SystemExit("at most %d questions per image" % R)
        session = model.openDialogs(dl, split, [index[i] for i in ids], params)
        dialogs = [[] for _ in ids]
        for r in range(max(len(q) for q in qs)):
            # a dialog whose questions ran out is asked pads: it writes nothing into its history
            out = session.ask([q[r] if r < len(q) else [] for q in qs])
            for d, e in enumerate(out):
                if r < len(qs[d]):
                    if e is None:
                        raise SystemExit("no beam reached <END> within -beamLen (image %d, round %d)" % (ids[d], r))
                    dialogs[d].append({"question": idToWords(e["question"], dl.ind2word),
                                       "answer": idToWords(e["answer"], dl.ind2word)})
        session.close()
        path = os.path.join(opt["resultPath"], "results.json")
        cli.write_json(path, {"opts": cli.written_opts(opt), "data": [{"image_id": i, "dialog": d} for i, d in zip(ids, dialogs)]})
        print("Writing the results to " + path, flush=True)
    finally:
        dl.close()
        model.engine.close()


if __name__ == "__main__":
    cli.run("visdial_b200.chat", "main", parse())
