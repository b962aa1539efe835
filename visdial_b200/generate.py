"""`python -m visdial_b200.generate -loadPath ...`: generate.lua on the engine.

Options and defaults are those of generate.lua:15-30 (see visdial_b200.cli): beam search (beamSize 5, beamLen 20) or,
with `-sampleWords 1`, sampling at `temperature`, over the first `maxThreads` dialogs of the val split.  Writes
`<resultPath>/results.json` = {opts, data}, data = [{image_id, dialog: [{question, answer}]}] with the text of
utils.idToWords, which is what vis/static/main.js shows.  A round where no beam reaches <END> stops the command before
anything is written (the reference dies there too, model.lua:575).  `-dialogsPerCall D` searches D dialogs per device
call; 1 (the default) is the reference's per-dialog loop.  `-history generated` answers every round with the dialog's own
earlier answers in its history instead of the dataset's (`-history gt`, the default and the reference's behaviour; DESIGN
§17); it combines with `-sampleWords`, `-dialogsPerCall` and `-gpus`.

`-gpus N` splits those first `maxThreads` dialogs into contiguous shares over GPUs gpuid .. gpuid+N-1 and rank 0 writes
them in order; with per-dialog calls the file is the one a single GPU writes."""
from __future__ import annotations

import os

from . import cli


def rank_share(model, dl, opt: dict) -> list:
    """This rank's share of the first `maxThreads` val dialogs as results.json entries (an empty list when the share is
    empty): generateAnswers' token lists turned into utils.idToWords text."""
    from .utils import idToWords
    dl.restrict("val", max(0, opt["maxThreads"]))                                   # model.lua:455 over the ranks
    sampleParams = {k: opt[k] for k in ("beamSize", "beamLen", "sampleWords", "temperature", "dialogsPerCall")}   # :88-94
    sampleParams["history"] = opt.get("history", "gt")
    answers = model.generateAnswers(dl, "val", sampleParams)                        # :96
    words = dl.ind2word
    return [{"image_id": a["image_id"],
             "dialog": [{"question": idToWords(r["question"], words), "answer": idToWords(r["answer"], words)}
                        for r in a["dialog"]]} for a in answers]


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
        opts = {k: v for k, v in opt.items() if k != "gpus"}
        path = os.path.join(opt["resultPath"], "results.json")                      # :97-103
        cli.write_json(path, {"opts": opts, "data": data})
        say("Writing the results to " + path)
    dl.close()
    model.engine.close()


if __name__ == "__main__":
    cli.run("visdial_b200.generate", "main", cli.parse(cli.GENERATE_COMMAND_OPTIONS, prog="python -m visdial_b200.generate"))
