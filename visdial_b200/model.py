"""Mirror of the reference's `Model` class (/root/reference/model.lua:8-430) over the C engine.
Same method names, argument meaning and call order as the Lua original, so that the parity tests
read like the reference's own driver code.  `generateAnswers` (beam search / sampling, model.lua:432-613) runs the beam
search and the sampling entirely on the device (vd_gen_beam_search, vd_gen_sample)."""
from __future__ import annotations

import numpy as np

from . import decoders, encoders
from .engine import Batch, DEFAULT_PARAMS, derive_flags
from .modules import Criterion, Sequential
from .cli import HISTORY_MODES
from .utils import image_id as _image_id


def _as_batch(b):
    """getTestBatch returns (batch, nextStartId) in the reference (dataloader.lua:375); accept either form."""
    if isinstance(b, tuple):
        b = b[0]
    return b if isinstance(b, Batch) else Batch(b)


def _question_width(dataloader, dtype, inds, convId, Tq, ques_len):
    """The `question` columns of dialog convId in a batch of the dialogs `inds` (padded to Tq): a one-dialog batch keeps
    the rightmost (its longest question) columns (dataloader.lua:380-384), so a wider batch keeps that many too.  Returns
    (width, the split's ques_length array, loaded at the first multi-dialog batch)."""
    if len(inds) == 1:
        return Tq, ques_len
    if ques_len is None:
        ques_len = dataloader.corpus[dtype].raw["ques_length"]
    return int(ques_len[dataloader.part[dtype][0] + convId].max()), ques_len


def _num_tokens(batch) -> int:
    """answerOut:gt(0):sum() (model.lua:78); device batches carry it from the host length table."""
    n = getattr(batch, "num_answer_tokens", None)
    return int(n) if n is not None else int((batch["answer_out"] > 0).sum())


class Model:
    def __init__(self, params: dict, seed: int = 1234):                  # model.lua:11-62
        p = dict(DEFAULT_PARAMS)
        p.update(params)
        self.params = derive_flags(p)
        encoder = encoders.load(p["encoder"])                             # :19-20
        decoder = decoders.load(p["decoder"])                             # :22-23
        enc = encoder.model(p)                                            # :25
        dec = decoder.model(p, enc)                                       # :26
        self.forwardConnect = decoder.forwardConnect                      # :28-29
        self.backwardConnect = decoder.backwardConnect
        self.decoderConnect = getattr(decoder, "decoderConnect", None)
        self.criterion = Criterion(p["decoder"])                          # :32-39
        self.wrapper = Sequential(enc, dec, p, seed)                      # :42 (weight-init.lua is a no-op here)
        if p["gpuid"] < 0:
            raise ValueError("visdial_b200 has no CPU path: gpuid must be >= 0")
        self.wrapper.cuda()                                               # :48-51
        self.criterion.engine = self.wrapper.engine
        self.encoder = self.wrapper.get(1)                                # :53-54
        self.decoder = self.wrapper.get(2)
        self.wrapperW, self.wrapperdW = self.wrapper.getParameters()      # :55
        self.wrapper.training()                                           # :57
        self.optims = {"learningRate": p["learningRate"]}                 # :60-61
        self.runningLoss = 0.0                                            # global `runningLoss`, train.lua:89
        self.engine = self.wrapper.engine
        self.iteration = 0

    # ---------------------------------------------------------------------------------------------
    def trainIteration(self, dataloader):                                 # model.lua:66-106
        self.wrapper.zeroGradParameters()                                 # :68
        batch = dataloader.getTrainBatch(self.params)                     # :71
        if not isinstance(batch, Batch):
            batch = Batch(batch)
        self.iteration += 1
        self.engine.set_dropout_seed(self.params.get("seed", 1234), self.iteration)
        curLoss = self.forwardBackward(batch)                             # :74
        if self.params["decoder"] == "gen":                               # :76-85
            numTokens = _num_tokens(batch)
            cur = curLoss / max(numTokens, 1)
        else:                                                             # :86-93
            cur = curLoss
        self._finish_iteration(cur)
        return curLoss

    def trainIterationDense(self, dataloader, dense):
        """trainIteration with the dense fine-tuning step (vd_forward_backward_dense) in place of the standard one: a batch
        of annotated dialogs of `dense` (visdial_b200.dense), the soft-target cross-entropy on their annotated rounds."""
        if self.params["decoder"] != "disc":
            raise ValueError("dense fine-tuning needs a disc model")
        self.wrapper.zeroGradParameters()
        batch, rounds, relevance = dataloader.getDenseTrainBatch(self.params, dense)
        self.iteration += 1
        self.engine.set_dropout_seed(self.params.get("seed", 1234), self.iteration)
        curLoss = self.engine.forward_backward_dense(batch, rounds, relevance)
        self._finish_iteration(curLoss)
        return curLoss

    def _finish_iteration(self, cur):
        self.runningLoss = 0.95 * self.runningLoss + 0.05 * cur if self.runningLoss > 0 else cur
        # model.lua:96-99 clamp(-5,5) + adam, fused with the gradient all-reduce when world > 1
        self.engine.clamp_adam_step(self.optims["learningRate"])
        if self.optims["learningRate"] > self.params["minLRate"]:          # :102-105
            self.optims["learningRate"] *= self.params["lrDecayRate"]

    def forwardBackward(self, batch, onlyForward=False, encOutOnly=False):   # model.lua:249-342
        if not isinstance(batch, Batch):
            batch = Batch(batch)
        # :252-294 (time-major views, image repeat, MN mask) are index arithmetic inside the engine
        encOut = self.encoder.forward(batch)                               # :297
        seqLen = batch.c.Tq
        self.decoder._last_batch = batch
        self.forwardConnect(self.encoder, self.decoder, encOut, seqLen)    # :300
        if encOutOnly:
            return encOut                                                  # :302
        if self.params["decoder"] == "gen":
            # decOut only travels on to the criterion here: let the engine keep the (rows, V) log-probabilities on chip
            self.engine.set_lazy_decout(True)
            try:
                decOut = self.decoder.forward(batch)                       # :313
            finally:
                self.engine.set_lazy_decout(False)
            curLoss = self.criterion.forward(decOut, batch)                # :314
            if not onlyForward:
                gradCriterionOut = self.criterion.backward(decOut, batch)  # :318
                self.decoder.backward(batch, gradCriterionOut)             # :319
                gradDecOut = self.backwardConnect(self.encoder, self.decoder)   # :322
                self.encoder.backward(batch, gradDecOut)                   # :323
        else:
            decOut = self.decoder.forward(batch)                           # :329
            curLoss = self.criterion.forward(decOut, batch)                # :330
            if not onlyForward:
                gradCriterionOut = self.criterion.backward(decOut, batch)  # :334
                t = self.decoder.backward(batch, gradCriterionOut)         # :335
                self.encoder.backward(batch, t[1])                         # :337 (t[2] in Lua)
        return curLoss

    def retrieveBatch(self, batch):                                        # model.lua:344-430
        if not isinstance(batch, Batch):
            batch = Batch(batch)
        return self.engine.retrieve(batch, use_gt=bool(self.params.get("useGt", True)))

    # ---------------------------------------------------------------------------------------------
    def evaluate(self, dataloader, dtype="val"):                           # model.lua:109-139
        self.wrapper.evaluate()
        curLoss, numTokens, n = 0.0, 0, 0
        numThreads = dataloader.numThreads[dtype]
        for startId in range(0, numThreads, self.params["batchSize"]):
            batch = _as_batch(dataloader.getTestBatch(startId, self.params, dtype))
            curLoss += self.forwardBackward(batch, True)
            if self.params["decoder"] == "gen":
                numTokens += _num_tokens(batch)
            n += 1
        self.wrapper.training()
        # :133 divides the summed loss by the answer-token count; for disc (a mean criterion per batch, no token count in
        # the disc batch table) the mean over batches is the comparable figure
        return curLoss / max(numTokens, 1) if self.params["decoder"] == "gen" else curLoss / max(n, 1)

    def _rank_walk(self, dataloader, dtype, use_gt):
        """The getTestBatch loop shared by retrieve / predict (model.lua:153-166, :208-221)."""
        self.wrapper.evaluate()
        out = []
        numThreads = dataloader.numThreads[dtype]
        for startId in range(0, numThreads, self.params["batchSize"]):
            batch = _as_batch(dataloader.getTestBatch(startId, self.params, dtype))
            out.append(self.engine.retrieve(batch, use_gt=use_gt))
        self.wrapper.training()
        return out

    def _round_table(self, dataloader, dtype, ranks, last_round_only):
        """model.lua:175-185 / :227-243: one {image_id, round_id, ranks} entry per (dialog, round)."""
        img = getattr(dataloader, "unique_img_" + dtype, None)
        nr = getattr(dataloader, dtype + "_num_rounds", None)
        first = dataloader.part[dtype][0] if dtype in getattr(dataloader, "part", {}) else 0
        table = []
        for i in range(ranks.shape[0]):
            n_i = int(nr[first + i]) if nr is not None else ranks.shape[1]
            iid = _image_id(img[first + i]) if img is not None else first + i
            rounds = [n_i] if last_round_only else range(1, n_i + 1)
            for j in rounds:
                r = ranks[i, j - 1]
                table.append({"image_id": iid, "round_id": int(j), "ranks": r.tolist() if np.ndim(r) else int(r)})
        return table

    def retrieve(self, dataloader, dtype="val", as_table=False, verbose=False):   # model.lua:142-189
        """Ground-truth ranks of a split, (numThreads, maxQuesCount).  `as_table=True` returns what the reference returns:
        the {image_id, round_id, ranks} list, after printing utils.processRanks of the matrix."""
        use_gt = bool(self.params.get("useGt", True))
        ranks = np.concatenate([r.reshape(-1, self.params["maxQuesCount"]) for r in self._rank_walk(dataloader, dtype, use_gt)], 0)
        if not as_table:
            return ranks
        from .utils import processRanks
        processRanks(ranks, verbose=verbose)                                       # :170
        return self._round_table(dataloader, dtype, ranks, last_round_only=False)

    def predict(self, dataloader, dtype="val"):                                   # model.lua:191-246
        """Full 100-option rank lists (evaluate.lua's EvalAI dump): every round of a val dialog, the last round of a test one."""
        K = int(self.params.get("numOptions", 100))
        ranks = np.concatenate([r.reshape(-1, self.params["maxQuesCount"], K) for r in self._rank_walk(dataloader, dtype, False)], 0)
        return self._round_table(dataloader, dtype, ranks, last_round_only=(dtype == "test"))

    # ---- beam search / sampling (model.lua:432-613, generate.lua) ---------------------------------------------
    def generateAnswers(self, dataloader, dtype="val", params=None, strict=True):
        """Model:generateAnswers.  Beam search (the default) and sampling (`sampleWords = 1`) run entirely on the device
        through vd_gen_beam_search / vd_gen_sample, for `params.dialogsPerCall` dialogs (default 1) per encoder forward and
        engine call: every round of those dialogs is searched or sampled at once.  One dialog per call gives exactly the
        per-dialog trimming and kernel shapes of the reference's loop; more dialogs per call run wider kernels (in the
        tensor-core math modes their rounding can differ from per-dialog runs).  The draws of a sampled round depend only on
        (seed, its global round index, the step): each call passes the index of its first round in the split (this rank's
        offset included), so the samples do not depend on dialogsPerCall or on how the split is sharded over ranks, only on
        the logits.  Returns the reference's answerTable with token-id lists (and text when the dataloader carries
        ind2word).  `strict=False` yields None for a round where no beam reached <END> (the reference indexes nil there,
        model.lua:575).

        `history`: "gt" (the default, the reference's behaviour) answers every round with the dataset's history;
        "generated" runs each dialog on its own answers (vd_gen_dialog_beam_search / vd_gen_dialog_sample, DESIGN §17):
        round r's history holds the answers generated for rounds < r.  Encoders without history have nothing to feed back
        and answer as with "gt"."""
        if self.params["decoder"] == "disc":                                            # :434-437
            raise ValueError("Sampling/beam search only for generative model")
        params = params or {}
        history = params.get("history", "gt")
        if history not in HISTORY_MODES:
            raise ValueError("history is one of %s, not %r" % ("|".join(HISTORY_MODES), history))
        generated = history == "generated" and bool(self.params.get("useHistory"))
        if generated:
            # the width the dataloader sizes history rows for (dataloader.lua:217-225, getIndexData's cut :387-392)
            maxAnsLen = dataloader.maxAnsLen
            histWidth = dataloader.maxHistoryLen if dataloader.concatHistory else \
                min(dataloader.maxQuesLen + maxAnsLen, dataloader.maxHistoryLen)
        sampleWords = bool(params.get("sampleWords", 0) == 1)                           # :443
        temperature, seed = float(params.get("temperature", 1.0)), int(params.get("seed", 1234))
        beamSize, beamLen = int(params.get("beamSize", 5)), int(params.get("beamLen", 20))
        startToken, endToken = dataloader.word2ind["<START>"], dataloader.word2ind["<END>"]   # :453-454
        numThreads = int(params.get("maxThreads") or dataloader.numThreads[dtype])      # :455
        dialogsPerCall = max(1, int(params.get("dialogsPerCall", 1)))
        ind2word = getattr(dataloader, "ind2word", None)
        words = (lambda ids: " ".join(ind2word.get(int(t), "<UNK>") for t in ids if int(t) > 0)) if ind2word else None
        img = getattr(dataloader, "unique_img_" + dtype, None)
        # getIndexData hands out this rank's slice of the split: the image list and the sampled rounds' global indices
        # count from the slice's first dialog
        offset = dataloader.part[dtype][0] if hasattr(dataloader, "part") and dtype in getattr(dataloader, "part", {}) else 0

        def entry(q, answer, **scored):
            e = {"question": q.tolist(), "answer": answer.tolist(), **scored}
            if words:
                e["question_text"], e["answer_text"] = words(q), words(answer)
            return e

        answerTable = []
        ques_len = None
        for first in range(0, numThreads, dialogsPerCall):
            inds = np.arange(first, min(numThreads, first + dialogsPerCall))
            self.wrapper.evaluate()                                                     # :460
            batch = dataloader.getIndexData(inds, self.params, dtype)                   # :462-463
            rowOffset = (offset + first) * self.params["maxQuesCount"]
            if generated:
                if sampleWords:
                    answer, _, _ = self.engine.gen_dialog_sample(batch, beamLen, startToken, endToken, temperature, seed,
                                                                 rowOffset, histWidth, maxAnsLen)
                else:
                    answer, length, score, _ = self.engine.gen_dialog_beam_search(batch, beamSize, beamLen, startToken,
                                                                                  endToken, histWidth, maxAnsLen)
            else:
                self.forwardBackward(batch, True, True)                                 # :467
                if sampleWords:                                                         # :582-594
                    answer, _ = self.engine.gen_sample(beamLen, startToken, temperature, seed, rowOffset)
                else:                                                                   # :472-579
                    answer, length, score = self.engine.gen_beam_search(beamSize, beamLen, startToken, endToken)
            if not sampleWords:
                length, score = length.reshape(len(inds), -1), score.reshape(len(inds), -1)
            ques = batch["ques_fwd"]                                                    # (D, maxQuesCount, Tq)
            Tq = ques.shape[2]
            answer = answer.reshape(len(inds), -1, answer.shape[1])
            self.wrapper.training()                                                     # :605
            for d, convId in enumerate(inds):
                w, ques_len = _question_width(dataloader, dtype, inds, convId, Tq, ques_len)
                threadAnswers = []
                for it in range(ques.shape[1]):
                    q, a = ques[d, it, Tq - w:], answer[d, it]
                    if sampleWords:
                        threadAnswers.append(entry(q, a))
                    elif length[d, it] > 0:
                        threadAnswers.append(entry(q, a, score=float(score[d, it]), length=int(length[d, it])))
                    elif strict:
                        raise IndexError("no beam reached <END> within beamLen (model.lua:575 indexes nil here)")
                    else:
                        threadAnswers.append(None)
                gid = offset + int(convId)
                answerTable.append({"image_id": _image_id(img[gid]) if img is not None else gid,
                                    "dialog": threadAnswers})                           # :606
        return answerTable

    # ---- checkpoints (train.lua:33-34,78-80,99-102,120-121; evaluate.lua:58-91) -------------------------------
    def save(self, path: str, final: bool = False):
        """torch.save(path, {modelW, optims, modelParams}) — `final` = the model_final.t7 form (float weights, no optims)."""
        from .checkpoint import save_checkpoint
        save_checkpoint(self, path, final)

    def load(self, path: str, permutation=None, restore_adam_state: bool = False):
        """wrapperW:copy(savedModel.modelW); optims.learningRate = savedModel.optims.learningRate."""
        from .checkpoint import load_checkpoint, restore
        ck = load_checkpoint(path, permutation)
        restore(self, ck, restore_adam_state)
        return ck
