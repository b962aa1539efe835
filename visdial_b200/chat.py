"""`python -m visdial_b200.chat -loadPath ...`: talk to a model about an image, one question at a time (DESIGN §19).

Reads the model and data as `generate` does and opens a dialog session (Model.openDialogs) on the chosen images of
`-split`: their features and captions; each question is answered before the next is asked, and the model's own answers
become the history the next question is answered with.  Gen models answer with generate's beam search (`-beamSize`,
`-beamLen`) or, with `-sampleWords 1`, by sampling; disc models with the best answer of the split's answer pool.

With `-questions file.json` ({image_id: [question, ...]}, at most maxQuesCount per image; a question is text or a list of
token ids) every image of the file (or of `-imageIds`) is asked its questions, round by round, and
`<resultPath>/results.json` is written in generate's {opts, data} layout, which the visualiser in vis/ shows.  Without
it the command talks about one image (the first of `-imageIds`, else the split's first): it reads one question per line
from stdin and prints each answer.  One GPU only."""
from __future__ import annotations

import json
import os
import sys

from . import cli


def _image_index(dl, split: str) -> dict:
    img = getattr(dl, "unique_img_" + split, None)
    if img is None:
        raise ValueError("the data has no image ids for split %r" % split)
    from .utils import image_id
    return {image_id(x): i for i, x in enumerate(img)}


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
        params = {k: opt[k] for k in ("beamSize", "beamLen", "sampleWords", "temperature")}
        R = model.params["maxQuesCount"]
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
        cli.write_json(path, {"opts": opt, "data": [{"image_id": i, "dialog": d} for i, d in zip(ids, dialogs)]})
        print("Writing the results to " + path, flush=True)
    finally:
        dl.close()
        model.engine.close()


if __name__ == "__main__":
    cli.run("visdial_b200.chat", "main", parse())
