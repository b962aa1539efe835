"""`python -m visdial_b200.generate -loadPath ...`: generate.lua on the engine.

Options and defaults are those of generate.lua:15-30 (see visdial_b200.cli): beam search (beamSize 5, beamLen 20) or,
with `-sampleWords 1`, sampling at `temperature`, over the first `maxThreads` dialogs of the val split.  Writes
`<resultPath>/results.json` = {opts, data}, data = [{image_id, dialog: [{question, answer}]}] with the text of
utils.idToWords, which is what vis/static/main.js shows.  A round where no beam reaches <END> stops the command before
anything is written (the reference dies there too, model.lua:575).  `-dialogsPerCall D` searches D dialogs per device
call; 1 (the default) is the reference's per-dialog loop.  `-history generated` answers every round with the dialog's own
earlier answers in its history instead of the dataset's (`-history gt`, the default and the reference's behaviour; DESIGN
§17); it combines with `-sampleWords`, `-dialogsPerCall` and `-gpus`.  `-beamGroups G` (> 1, dividing `-beamSize`) runs
diverse beam search with penalty `-diversity` (DESIGN §22): each round's answer is the best group's, and the round also
lists `"answers"`, the text of every group that finished an answer, best first (the first is the round's answer).
`-nBest n` keeps each group's n best finished answers and the round also lists `"nbest"`, their text best first (the
first is the round's answer); `-lengthPenalty a` ranks finished answers by score / ((5 + l) / 6)^a, l their tokens
(DESIGN §24).  results.json records the two only when they differ from their defaults (1 and 0).
`-topK K` and `-topP P` truncate `-sampleWords 1`'s draws to the K most likely words and then to the fewest of those
holding P of the probability (DESIGN §23); they combine with `-history`, `-dialogsPerCall` and `-gpus`, and
results.json records them only when they truncate.  `-minWords m`, `-noRepeatNgram n` and `-bannedWords w1,w2` are the
answer rules (DESIGN §25): no answer ends before m words, repeats an n-gram or uses a banned word, in beam search and
sampling alike; results.json records them only when one is set.  A disc checkpoint answers every round with the
best answer of the split's answer pool (Model.retrieveAnswers, DESIGN §18); the beam and sampling options do not apply
to it, and its answer text is the pool row's words.

`-gpus N` splits those first `maxThreads` dialogs into contiguous shares over GPUs gpuid .. gpuid+N-1 and rank 0 writes
them in order; with per-dialog calls the file is the one a single GPU writes."""
from __future__ import annotations

import os

from . import cli


def rank_share(model, dl, opt: dict) -> list:
    """This rank's share of the first `maxThreads` val dialogs as results.json entries (an empty list when the share is
    empty): generateAnswers' token lists turned into utils.idToWords text."""
    from .model import ranked_groups
    from .utils import idToWords
    dl.restrict("val", max(0, opt["maxThreads"]))                                   # model.lua:455 over the ranks
    sampleParams = {k: opt[k] for k in ("beamSize", "beamLen", "sampleWords", "temperature", "dialogsPerCall")}   # :88-94
    sampleParams["history"] = opt.get("history", "gt")
    sampleParams.update({k: opt[k] for k in ("beamGroups", "diversity", "lengthPenalty", "nBest", "topK", "topP") if k in opt})
    sampleParams.update(cli.answer_rule_params(opt))
    if model.params["decoder"] == "disc":
        # a disc model answers by retrieval from the split's answer pool (DESIGN §18); model.lua:434-437 stops here
        answers = model.retrieveAnswers(dl, "val", {k: sampleParams[k] for k in ("dialogsPerCall", "history")})
    else:
        answers = model.generateAnswers(dl, "val", sampleParams)                    # :96
    words = dl.ind2word

    def turn(r):
        t = {"question": idToWords(r["question"], words), "answer": idToWords(r["answer"], words)}
        if "groups" in r:
            t["answers"] = [idToWords(g["answer"], words) for g in ranked_groups(r)]
        if "nbest" in r:
            t["nbest"] = [idToWords(x["answer"], words) for x in r["nbest"]]
        return t
    return [{"image_id": a["image_id"], "dialog": [turn(r) for r in a["dialog"]]} for a in answers]


def main(opt: dict, rank: int = 0, world: int = 1):
    from . import dist as vdist
    from .checkpoint import load_checkpoint
    say = (lambda *a: print(*a, flush=True)) if rank == 0 else (lambda *a: None)
    say(opt)
    ck = load_checkpoint(opt["loadPath"])                                           # generate.lua:53-60
    mp = cli.adopt_checkpoint_model(opt, ck)
    model, dl = cli.build(mp, opt, rank, world, ["val"], ck)                        # :72-83
    data = rank_share(model, dl, opt)
    if world > 1:
        data = vdist.gather_objects(data, world)
    if rank == 0:
        # the file says what was generated, not how the run was spread over GPUs: 1- and N-GPU runs write the same bytes
        opts = {k: v for k, v in cli.written_opts(opt).items() if k != "gpus"}
        path = os.path.join(opt["resultPath"], "results.json")                      # :97-103
        cli.write_json(path, {"opts": opts, "data": data})
        say("Writing the results to " + path)
    dl.close()
    model.engine.close()


if __name__ == "__main__":
    cli.run("visdial_b200.generate", "main", cli.parse(cli.GENERATE_COMMAND_OPTIONS, prog="python -m visdial_b200.generate"))
