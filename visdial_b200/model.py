"""Mirror of the reference's `Model` class (/root/reference/model.lua:8-430) over the C engine.
Same method names, argument meaning and call order as the Lua original, so that the parity tests
read like the reference's own driver code.  `generateAnswers` (beam search / sampling, model.lua:432-613) runs the beam
search and the sampling entirely on the device (vd_gen_beam_search, vd_gen_sample)."""
from __future__ import annotations

import contextlib

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

    def trainIterationDenseGen(self, dataloader, dense):
        """trainIterationDense for gen models (vd_forward_backward_dense_gen): the scores of the annotated round's options
        are their log-likelihoods under the decoder, the ones evaluate ranks gen models by."""
        if self.params["decoder"] != "gen":
            raise ValueError("trainIterationDenseGen needs a gen model")
        self.wrapper.zeroGradParameters()
        batch, rounds, relevance = dataloader.getDenseTrainBatch(self.params, dense)
        self.iteration += 1
        self.engine.set_dropout_seed(self.params.get("seed", 1234), self.iteration)
        curLoss = self.engine.forward_backward_dense_gen(batch, rounds, relevance)
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
        and answer as with "gt".

        `beamGroups` G > 1 (default 1) runs diverse beam search (vd_gen_diverse_beam_search, DESIGN §22): the beamSize
        columns in G groups, each group's candidates penalised by `diversity` (default 0.5) per column of an earlier group
        that chose the same token at that step.  Each round's answer / score / length are then the pick (the best group by
        score, the lower group on ties; what the "generated" history takes), and "groups" lists the G groups' entries
        (None for a group that finished no hypothesis).  `strict` raises only when every group is empty.

        `lengthPenalty` alpha (default 0) and `nBest` n (default 1) keep each group's n best finished hypotheses by norm =
        score / ((5 + l) / 6)^alpha, l = length - 1 (vd_gen_nbest_beam_search / vd_gen_dialog_nbest_beam_search, DESIGN
        §24).  At the defaults the calls are the ones above.  Otherwise each round's answer / score / length are the pick's
        (the best group head by normScore, the lower group on ties), every entry carries "normScore", "groups" (G > 1)
        lists the group heads, and with n > 1 "nbest" lists every finished hypothesis of every group by (normScore desc,
        group asc, list position asc).  Sampling ignores both.

        With `sampleWords`, `topK` K (default 0, off) and `topP` P (default 1, off) truncate every draw (DESIGN §23): to the
        first K classes by (logit desc, class asc), then to the shortest prefix of those holding P of their softmax mass
        (vd_gen_truncated_sample / vd_gen_dialog_truncated_sample).  When neither truncates (K = 0 or K >= vocabSize, and
        P = 1) the calls are the untruncated ones.  Beam search ignores both.

        `minWords` (default 0), `noRepeatNgram` (default 0, off) and `bannedWords` (a list of words, default none) are the
        answer rules (vd_set_answer_rules, DESIGN §25), in beam search and sampling alike: no answer ends before minWords
        words, repeats a noRepeatNgram-gram or uses a banned word.  They are set for this call's engine calls only; at their
        defaults nothing is set.  An unknown banned word raises ValueError."""
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
        groups, diversity = int(params.get("beamGroups", 1)), float(params.get("diversity", 0.5))
        diverse = groups > 1 and not sampleWords
        lengthPenalty, nBest = float(params.get("lengthPenalty", 0.0)), int(params.get("nBest", 1))
        listed = not sampleWords and (lengthPenalty != 0.0 or nBest != 1)
        topK, topP = int(params.get("topK", 0)), float(params.get("topP", 1.0))
        truncated = sampleWords and truncates(topK, topP, self.params["vocabSize"])
        startToken, endToken = dataloader.word2ind["<START>"], dataloader.word2ind["<END>"]   # :453-454
        rules = answer_rules(params, dataloader.word2ind)
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
            with rules_set(self.engine, rules):
                if generated:
                    if truncated:
                        answer, _, _ = self.engine.gen_dialog_truncated_sample(batch, beamLen, startToken, endToken, temperature,
                                                                               seed, rowOffset, histWidth, maxAnsLen, topK, topP)
                    elif sampleWords:
                        answer, _, _ = self.engine.gen_dialog_sample(batch, beamLen, startToken, endToken, temperature, seed,
                                                                     rowOffset, histWidth, maxAnsLen)
                    elif listed:
                        answer, length, score, norm, _ = self.engine.gen_dialog_nbest_beam_search(
                            batch, beamSize, groups, diversity, lengthPenalty, nBest, beamLen, startToken, endToken, histWidth,
                            maxAnsLen)
                    elif diverse:
                        answer, length, score, _ = self.engine.gen_dialog_diverse_beam_search(
                            batch, beamSize, groups, diversity, beamLen, startToken, endToken, histWidth, maxAnsLen)
                    else:
                        answer, length, score, _ = self.engine.gen_dialog_beam_search(batch, beamSize, beamLen, startToken,
                                                                                      endToken, histWidth, maxAnsLen)
                else:
                    self.forwardBackward(batch, True, True)                                 # :467
                    if truncated:
                        answer, _ = self.engine.gen_truncated_sample(beamLen, startToken, temperature, seed, rowOffset, topK, topP)
                    elif sampleWords:                                                       # :582-594
                        answer, _ = self.engine.gen_sample(beamLen, startToken, temperature, seed, rowOffset)
                    elif listed:
                        answer, length, score, norm = self.engine.gen_nbest_beam_search(beamSize, groups, diversity, lengthPenalty,
                                                                                        nBest, beamLen, startToken, endToken)
                    elif diverse:
                        answer, length, score = self.engine.gen_diverse_beam_search(beamSize, groups, diversity, beamLen,
                                                                                    startToken, endToken)
                    else:                                                                   # :472-579
                        answer, length, score = self.engine.gen_beam_search(beamSize, beamLen, startToken, endToken)
            R = self.params["maxQuesCount"]
            if listed:
                answer, length = answer.reshape(len(inds), R, groups, nBest, -1), length.reshape(len(inds), R, groups, nBest)
                score, norm = score.reshape(length.shape), norm.reshape(length.shape)
            elif not sampleWords:
                length, score = length.reshape(len(inds), R, -1), score.reshape(len(inds), R, -1)
            ques = batch["ques_fwd"]                                                    # (D, maxQuesCount, Tq)
            Tq = ques.shape[2]
            if not listed:
                answer = answer.reshape(len(inds), R, -1, answer.shape[-1])
            self.wrapper.training()                                                     # :605
            for d, convId in enumerate(inds):
                w, ques_len = _question_width(dataloader, dtype, inds, convId, Tq, ques_len)
                threadAnswers = []
                for it in range(ques.shape[1]):
                    q = ques[d, it, Tq - w:]
                    if sampleWords:
                        threadAnswers.append(entry(q, answer[d, it, 0]))
                        continue
                    if listed:
                        e = listed_entry(answer[d, it], length[d, it], score[d, it], norm[d, it],
                                         lambda a, **sc: entry(q, a, **sc))
                        if e is None and strict:
                            raise IndexError("no beam reached <END> within beamLen (model.lua:575 indexes nil here)")
                        threadAnswers.append(e)
                        continue
                    gs = [entry(q, answer[d, it, g], score=float(score[d, it, g]), length=int(length[d, it, g]))
                          if length[d, it, g] > 0 else None for g in range(length.shape[2])]
                    best = pick_group(length[d, it], score[d, it])
                    if best >= 0:
                        threadAnswers.append(dict(gs[best], groups=gs) if diverse else gs[best])
                    elif strict:
                        raise IndexError("no beam reached <END> within beamLen (model.lua:575 indexes nil here)")
                    else:
                        threadAnswers.append(None)
                gid = offset + int(convId)
                answerTable.append({"image_id": _image_id(img[gid]) if img is not None else gid,
                                    "dialog": threadAnswers})                           # :606
        return answerTable

    def retrieveAnswers(self, dataloader, dtype="val", params=None):
        """What a disc model answers (DESIGN §18): every round of the first `maxThreads` dialogs of split `dtype` answered
        by retrieval from the split's answer pool (opt_list_<dtype>).  The pool is encoded once per call
        (vd_answer_pool_encode); then `dialogsPerCall` dialogs (default 1) per engine call retrieve their `topK` (default 1)
        best pool rows by (score desc, pool index asc): vd_answer_pool_retrieve on the dataset's history (`history` "gt",
        the default), or vd_answer_pool_dialog on the answers retrieved for the dialog's earlier rounds ("generated";
        encoders without history answer as with "gt").  Returns generateAnswers' answerTable: per round the question, the
        top-1 pool row's tokens as `answer` (its non-pad words, no <START>), its 0-based pool `index` and `score`, and the
        `topK` list of {index, score, answer}; with text when the dataloader carries ind2word."""
        if self.params["decoder"] != "disc":
            raise ValueError("retrieveAnswers answers with the disc decoder; gen models use generateAnswers")
        params = params or {}
        history = params.get("history", "gt")
        if history not in HISTORY_MODES:
            raise ValueError("history is one of %s, not %r" % ("|".join(HISTORY_MODES), history))
        generated = history == "generated" and bool(self.params.get("useHistory"))
        maxAnsLen = dataloader.maxAnsLen
        if generated:
            histWidth = dataloader.maxHistoryLen if dataloader.concatHistory else \
                min(dataloader.maxQuesLen + maxAnsLen, dataloader.maxHistoryLen)
        topK = int(params.get("topK", 1))
        numThreads = int(params.get("maxThreads") or dataloader.numThreads[dtype])
        dialogsPerCall = max(1, int(params.get("dialogsPerCall", 1)))
        pool = dataloader.answerPool(dtype)
        self.engine.answer_pool_encode(pool)
        ind2word = getattr(dataloader, "ind2word", None)
        words = (lambda ids: " ".join(ind2word.get(int(t), "<UNK>") for t in ids if int(t) > 0)) if ind2word else None
        img = getattr(dataloader, "unique_img_" + dtype, None)
        offset = dataloader.part[dtype][0] if hasattr(dataloader, "part") and dtype in getattr(dataloader, "part", {}) else 0

        def answer_of(j):
            return np.array([t for t in pool[j] if t != 0], dtype=pool.dtype)

        def entry(q, idx, sc):
            a = answer_of(int(idx[0]))
            e = {"question": q.tolist(), "answer": a.tolist(), "index": int(idx[0]), "score": float(sc[0]),
                 "topK": [{"index": int(i), "score": float(v), "answer": answer_of(int(i)).tolist()} for i, v in zip(idx, sc)]}
            if words:
                e["question_text"], e["answer_text"] = words(q), words(a)
            return e

        answerTable = []
        ques_len = None
        R = self.params["maxQuesCount"]
        for first in range(0, numThreads, dialogsPerCall):
            inds = np.arange(first, min(numThreads, first + dialogsPerCall))
            batch = dataloader.getIndexData(inds, self.params, dtype)
            if generated:
                index, score, _ = self.engine.answer_pool_dialog(batch, topK, histWidth, maxAnsLen)
            else:
                index, score = self.engine.answer_pool_retrieve(batch, topK)
            index, score = index.reshape(len(inds), R, topK), score.reshape(len(inds), R, topK)
            ques = batch["ques_fwd"]
            Tq = ques.shape[2]
            for d, convId in enumerate(inds):
                w, ques_len = _question_width(dataloader, dtype, inds, convId, Tq, ques_len)
                gid = offset + int(convId)
                answerTable.append({"image_id": _image_id(img[gid]) if img is not None else gid,
                                    "dialog": [entry(ques[d, it, Tq - w:], index[d, it], score[d, it])
                                               for it in range(ques.shape[1])]})
        return answerTable

    def openDialogs(self, dataloader, dtype="val", inds=(0,), params=None) -> "DialogSession":
        """A dialog session (DESIGN §19) on dialogs `inds` (0-based) of split `dtype`: their images and captions, and
        questions asked one round at a time with DialogSession.ask.  `params` are generateAnswers' beamSize / beamLen /
        sampleWords / temperature / topK / topP for gen models, retrieveAnswers' topK for disc ones."""
        return DialogSession(self, dataloader, dtype, inds, params or {})

    def openDialogPool(self, dataloader, dtype="val", capacity=128, params=None) -> "DialogPool":
        """A dialog pool (DESIGN §20) of `capacity` conversations on the images and captions of split `dtype`: they join
        (DialogPool.join), are asked (DialogPool.ask) and leave on their own, each at its own round.  `params` as
        openDialogs'."""
        return DialogPool(self, dataloader, dtype, params or {}, capacity=capacity)

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


def answer_rules(params: dict, word2ind: dict):
    """The answer rules of `params` (DESIGN §25) as Engine.set_answer_rules' (min_words, no_repeat_ngram, banned ids):
    `minWords` (default 0), `noRepeatNgram` (default 0, off) and `bannedWords` (words, mapped through word2ind).  None when
    all three are at their defaults.  Raises ValueError for a banned word the vocabulary does not have."""
    minWords, noRepeat = int(params.get("minWords", 0)), int(params.get("noRepeatNgram", 0))
    words = list(params.get("bannedWords", ()) or ())
    unknown = [w for w in words if w not in word2ind]
    if unknown:
        raise ValueError("bannedWords not in the vocabulary: %s" % ", ".join(map(str, unknown)))
    if minWords == 0 and noRepeat == 0 and not words:
        return None
    return minWords, noRepeat, [int(word2ind[w]) for w in words]


@contextlib.contextmanager
def rules_set(engine, rules):
    """`rules` (answer_rules' value) on `engine` for the calls inside, cleared after them even when one raises, so that they
    never reach another caller of the engine; None sets nothing."""
    if rules is None:
        yield
        return
    engine.set_answer_rules(*rules)
    try:
        yield
    finally:
        engine.set_answer_rules()


def truncates(topK: int, topP: float, V: int) -> bool:
    """whether top-k / top-p truncation changes a draw over V classes (DESIGN §23): 1 <= topK < V or topP < 1"""
    return 1 <= topK < V or topP < 1.0


def pick_group(length, score) -> int:
    """A diverse search's pick (DESIGN §22): the group of the best finished hypothesis by (score desc, group asc), -1 when
    no group finished one."""
    best = -1
    for g in range(len(length)):
        if length[g] > 0 and (best < 0 or score[g] > score[best]):
            best = g
    return best


def ranked_groups(entry) -> list:
    """The finished groups of a diverse entry ("groups"), best first by (score desc, group asc), or by (normScore desc,
    group asc) when the entries carry one (DESIGN §24): the pick is the first."""
    done = [e for e in entry.get("groups", [entry]) if e is not None]
    return sorted(done, key=lambda e: -e.get("normScore", e["score"]))


def listed_entry(answer, length, score, norm, make):
    """A round's entry from its n-best lists (DESIGN §24): answer (G, n, L), length / score / norm (G, n).  `make(answer,
    score=, length=, normScore=)` builds one hypothesis' entry.  Returns the pick's entry (the best group head by
    (normScore desc, group asc)) with "groups" (the G heads, None for a group that finished nothing) when G > 1 and
    "nbest" (every finished hypothesis by (normScore desc, group asc, list position asc)) when n > 1; None when no group
    finished a hypothesis."""
    G, n = length.shape
    lists = [[make(answer[g, i], score=float(score[g, i]), length=int(length[g, i]), normScore=float(norm[g, i]))
              for i in range(n) if length[g, i] > 0] for g in range(G)]
    best = pick_group(length[:, 0], norm[:, 0])
    if best < 0:
        return None
    e = dict(lists[best][0])
    if G > 1:
        e["groups"] = [x[0] if x else None for x in lists]
    if n > 1:
        ranked = sorted(((x["normScore"], g, i) for g, xs in enumerate(lists) for i, x in enumerate(xs)),
                        key=lambda t: (-t[0], t[1], t[2]))
        e["nbest"] = [lists[g][i] for _, g, i in ranked]
    return e


def history_answer(row, end: int, length=None) -> list:
    """The words of an answer as the history rule reads them (DESIGN §17).  With `length`: a beam hypothesis (<START>
    first) of that many tokens, its words between <START> and <END>, none when length is 0.  Without: the words before
    the first <END> of `row` (a sample row without its <START> column, a pool row or a corpus answer).  Pads are not
    words."""
    if length is not None:
        return [int(t) for t in row[1:max(int(length) - 1, 1)] if t != 0] if length > 0 else []
    out = []
    for t in row:
        if int(t) == end:
            break
        if int(t) != 0:
            out.append(int(t))
    return out


def transcript_arrays(transcripts, R: int, width: int):
    """What vd_dialog_join_rounds reads for conversations given as transcripts, each a pair (question rows (width,)
    right-aligned, answer word lists) of equal length r < R: rounds (B), ques_fwd (B, R, width) and answers (B, R, Ta)
    left-aligned and zero-padded, Ta the longest answer (at least 1)."""
    B = len(transcripts)
    rounds = np.asarray([len(q) for q, _ in transcripts], np.int32)
    if any(len(q) != len(a) for q, a in transcripts) or (rounds >= R).any():
        raise ValueError("a transcript has one answer per question and fewer than maxQuesCount rounds")
    Ta = max([1] + [len(w) for _, a in transcripts for w in a])
    ques = np.zeros((B, R, width), np.int32)
    ans = np.zeros((B, R, Ta), np.int32)
    for i, (q, a) in enumerate(transcripts):
        for j in range(len(q)):
            ques[i, j] = q[j]
            ans[i, j, :len(a[j])] = a[j]
    return rounds, ques, ans


class DialogPool:
    """Conversations about the dataset's images that join, are asked and leave on their own, each at its own round
    (vd_dialog_open / join / ask_*_slots / leave, DESIGN §20).  A conversation is one dataset dialog's image and caption,
    asked its questions one at a time; the history rule, the widths and the answers are generateAnswers' /
    retrieveAnswers' with `history = "generated"`, and a sampled conversation draws as generateAnswers does for that
    dialog.  Fed the same questions, a conversation's answers do not depend on the others asked with it.
    The pool keeps each conversation's transcript (its dialog index, draw base, questions and the answers it was given or
    gave), so that conversations can join at any round (join with rounds, resume; DESIGN §21) and a pool can be reopened
    with every conversation in its own slot after a weight or math-mode change (reopen)."""

    def __init__(self, model, dataloader, dtype, params, capacity=None):
        self.model, self.dl, self.eng, self.dtype = model, dataloader, model.engine, dtype
        self.R = model.params["maxQuesCount"]
        self.disc = model.params["decoder"] == "disc"
        self.sampleWords = int(params.get("sampleWords", 0)) == 1
        self.temperature, self.seed = float(params.get("temperature", 1.0)), int(params.get("seed", 1234))
        self.beamSize, self.beamLen = int(params.get("beamSize", 5)), int(params.get("beamLen", 20))
        self.groups, self.diversity = int(params.get("beamGroups", 1)), float(params.get("diversity", 0.5))
        self.lengthPenalty, self.nBest = float(params.get("lengthPenalty", 0.0)), int(params.get("nBest", 1))
        # topK: a disc model's retrieval list length (default 1); a gen model's top-k truncation of sampling asks (default
        # 0, off), with topP (DESIGN §23)
        self.topK = int(params.get("topK", 1 if self.disc else 0))
        self.topP = float(params.get("topP", 1.0))
        self.truncated = not self.disc and self.sampleWords and truncates(self.topK, self.topP, model.params["vocabSize"])
        # the answer rules (DESIGN §25) of this pool's asks, set around each ask only; a disc pool retrieves without them
        self.rules = None if self.disc else answer_rules(params, dataloader.word2ind)
        self.start, self.end = dataloader.word2ind["<START>"], dataloader.word2ind["<END>"]
        self.width = dataloader.maxQuesLen
        self.maxAnsLen = dataloader.maxAnsLen
        self.histWidth = 0
        if model.params.get("useHistory"):
            self.histWidth = dataloader.maxHistoryLen if dataloader.concatHistory else \
                min(dataloader.maxQuesLen + self.maxAnsLen, dataloader.maxHistoryLen)
        self.offset = dataloader.part[dtype][0] if hasattr(dataloader, "part") and dtype in getattr(dataloader, "part", {}) \
            else 0
        self.rowOffset = 0                   # sampling: a slot draws as global round draw_base + its round
        self.words = getattr(dataloader, "ind2word", None)
        self.convs = {}                      # slot -> {"ind", "base", "ques": [rows], "ans": [word lists]}
        if self.disc:
            self.pool = dataloader.answerPool(dtype)
            self.eng.answer_pool_encode(self.pool)
        self.capacity = capacity
        if capacity is not None:
            self.eng.dialog_open(int(capacity), self.width, self.histWidth, self.maxAnsLen)

    def _batch(self, inds, gt=False) -> dict:
        """what a join reads of dialogs `inds`: images and round-0 history rows; questions are asked at the full width.
        gt: also the dialogs' own questions (right-aligned into the full width) and answers (corpus rows)."""
        batch = self.dl.getIndexData(np.asarray(inds, dtype=np.int64), self.model.params, self.dtype)
        host = {"ques_fwd": np.zeros((len(inds), self.R, self.width), np.int32)}
        for k in ("hist", "img_feat", "img_count"):
            if k in batch:
                host[k] = np.ascontiguousarray(batch[k])
        if gt:
            q = np.asarray(batch["ques_fwd"])
            host["ques_fwd"][:, :, self.width - q.shape[2]:] = q
            host["answer_out"] = np.asarray(batch["answer_out"])
        return host

    def _free_slots(self, n: int) -> list:
        from ._lib import VD_E_STATE, VdError
        free = [s for s, r in enumerate(self.eng.dialog_slots()) if r < 0]
        if len(free) < n:
            raise VdError(VD_E_STATE, "the pool has fewer free slots than dialogs to join")
        return free[:n]

    def _join_rounds(self, inds, transcripts, slots, bases):
        """conversations on dialogs `inds`' images and captions, each resumed from its transcript in its slot"""
        host = self._batch(inds)
        rounds, host["ques_fwd"], ans = transcript_arrays(transcripts, self.R, self.width)
        self.eng.dialog_join_rounds(Batch(host), rounds, ans if self.histWidth else None, slots, bases)
        for i, s in enumerate(slots):
            q, a = transcripts[i]
            self.convs[int(s)] = {"ind": int(inds[i]), "base": int(bases[i]), "ques": list(q), "ans": list(a)}

    def join(self, inds, rounds=None) -> list:
        """Joins dialogs `inds` (0-based, of the split) as new conversations; returns their slots.  At round 0 by default;
        with `rounds` (one per dialog, each below maxQuesCount) dialog i continues from round rounds[i] on its own
        questions and ground-truth answers of the earlier rounds, in one device pass.  Raises VdError (VD_E_STATE) and
        joins none when fewer slots are free."""
        inds = [int(i) for i in inds]
        base = np.asarray([(self.offset + i) * self.R for i in inds], np.int64)
        if rounds is None:
            slots = self.eng.dialog_join(Batch(self._batch(inds)), base).tolist()
            for i, s, b in zip(inds, slots, base):
                self.convs[s] = {"ind": i, "base": int(b), "ques": [], "ans": []}
            return slots
        if len(rounds) != len(inds):
            raise ValueError("one round per joined dialog")
        gt = self._batch(inds, gt=True)
        transcripts = [([gt["ques_fwd"][d, j] for j in range(int(r))],
                        [history_answer(gt["answer_out"][d, j], self.end) for j in range(int(r))])
                       for d, r in enumerate(rounds)]
        slots = self._free_slots(len(inds))
        self._join_rounds(inds, transcripts, slots, base)
        return slots

    def resume(self, ind: int, transcript) -> int:
        """A conversation about dialog `ind`'s image and caption that already had the rounds of `transcript`, a list of
        (question, answer) pairs, each text (utils.question_ids / answer_ids) or token ids, fewer than maxQuesCount: it
        joins at round len(transcript) with them as its history.  Returns its slot."""
        from .utils import answer_ids, question_ids
        q = [question_ids(x, self.dl.word2ind, self.width) for x, _ in transcript]
        a = [[int(t) for t in answer_ids(y, self.dl.word2ind, self.maxAnsLen) if t] for _, y in transcript]
        slot = self._free_slots(1)
        self._join_rounds([int(ind)], [(q, a)], slot, [(self.offset + int(ind)) * self.R])
        return slot[0]

    def reopen(self):
        """After Model.load / set_parameters / a math-mode change, which leave the engine's pool stale: reopens it at the
        same capacity and rejoins every live conversation in its own slot, at its round, with its draw base, in one
        device pass (a disc model's answer pool is encoded again).  A conversation that has had maxQuesCount rounds has
        nothing left to ask and is not rejoined."""
        if self.disc:
            self.eng.answer_pool_encode(self.pool)
        self.eng.dialog_open(int(self.capacity), self.width, self.histWidth, self.maxAnsLen)
        live = sorted(s for s, c in self.convs.items() if len(c["ques"]) < self.R)
        self.convs = {s: c for s, c in self.convs.items() if s in live}
        if live:
            c = [self.convs[s] for s in live]
            self._join_rounds([x["ind"] for x in c], [(x["ques"], x["ans"]) for x in c], live, [x["base"] for x in c])

    def ask(self, questions: dict) -> dict:
        """Asks each slot of `questions` ({slot: question}, text or token ids) its next round, all in one device call.
        Returns {slot: entry} with DialogSession.ask's entries."""
        from .utils import question_ids
        slots = [int(s) for s in questions]
        q = np.stack([question_ids(questions[s], self.dl.word2ind, self.width) for s in slots])
        return dict(zip(slots, self._ask(slots, q)))

    def _ask(self, slots, q) -> list:
        from .utils import idToWords
        text = (lambda ids: idToWords(ids, self.words)) if self.words else None
        out = []
        if self.disc:
            index, score = self.eng.dialog_ask_pool_slots(slots, q, self.topK)
            given = [history_answer(self.pool[index[b, 0]], self.end) for b in range(len(q))]
            for b in range(len(q)):
                a = [int(t) for t in self.pool[index[b, 0]] if t != 0]
                out.append({"question": [int(t) for t in q[b] if t], "answer": a, "index": int(index[b, 0]),
                            "score": float(score[b, 0]),
                            "topK": [{"index": int(i), "score": float(v),
                                      "answer": [int(t) for t in self.pool[i] if t != 0]} for i, v in zip(index[b], score[b])]})
        elif self.sampleWords:
            if self.truncated:
                with rules_set(self.eng, self.rules):
                    ans, _ = self.eng.dialog_ask_truncated_slots(slots, q, self.beamLen, self.start, self.end,
                                                                 self.temperature, self.seed, self.rowOffset, self.topK,
                                                                 self.topP)
            else:
                with rules_set(self.eng, self.rules):
                    ans, _ = self.eng.dialog_ask_sample_slots(slots, q, self.beamLen, self.start, self.end, self.temperature,
                                                              self.seed, self.rowOffset)
            given = [history_answer(ans[b, 1:], self.end) for b in range(len(q))]
            out = [{"question": [int(t) for t in q[b] if t], "answer": ans[b].tolist()} for b in range(len(q))]
        elif self.lengthPenalty != 0.0 or self.nBest != 1:
            with rules_set(self.eng, self.rules):
                ans, length, score, norm = self.eng.dialog_ask_nbest_slots(slots, q, self.beamSize, self.groups,
                                                                           self.diversity, self.lengthPenalty, self.nBest,
                                                                           self.beamLen, self.start, self.end)
            given = []
            for b in range(len(q)):
                e = listed_entry(ans[b], length[b], score[b], norm[b],
                                 lambda a, **sc: dict(answer=a.tolist(), **sc))
                given.append(history_answer(e["answer"], self.end, e["length"]) if e else [])
                out.append(dict(e, question=[int(t) for t in q[b] if t]) if e else None)
        elif self.groups > 1:
            with rules_set(self.eng, self.rules):
                ans, length, score = self.eng.dialog_ask_diverse_slots(slots, q, self.beamSize, self.groups, self.diversity,
                                                                       self.beamLen, self.start, self.end)
            given = []
            for b in range(len(q)):
                gs = [{"answer": ans[b, g].tolist(), "score": float(score[b, g]), "length": int(length[b, g])}
                      if length[b, g] > 0 else None for g in range(self.groups)]
                best = pick_group(length[b], score[b])
                given.append(history_answer(ans[b, best], self.end, length[b, best]) if best >= 0 else [])
                out.append(dict(gs[best], question=[int(t) for t in q[b] if t], groups=gs) if best >= 0 else None)
        else:
            with rules_set(self.eng, self.rules):
                ans, length, score = self.eng.dialog_ask_beam_slots(slots, q, self.beamSize, self.beamLen, self.start,
                                                                    self.end)
            given = [history_answer(ans[b], self.end, length[b]) for b in range(len(q))]
            out = [{"question": [int(t) for t in q[b] if t], "answer": ans[b].tolist(), "score": float(score[b]),
                    "length": int(length[b])} if length[b] > 0 else None for b in range(len(q))]
        for s, row, a in zip(slots, q, given):            # the transcript a later resume or reopen replays
            if s in self.convs:
                self.convs[s]["ques"].append(np.array(row, np.int32))
                self.convs[s]["ans"].append(a)
        if text:
            for e in out:
                if e is not None:
                    e["question_text"], e["answer_text"] = text(e["question"]), text(e["answer"])
                    for x in list(e.get("groups", ())) + list(e.get("nbest", ())):
                        if x is not None:
                            x["answer_text"] = text(x["answer"])
        return out

    def leave(self, slots):
        self.eng.dialog_leave([int(s) for s in slots])
        for s in slots:
            self.convs.pop(int(s), None)

    def round(self, slot: int) -> int:
        """The slot's next round to be asked (R once it has had maxQuesCount), -1 when free."""
        return int(self.eng.dialog_slots()[int(slot)])

    def history(self, slots) -> np.ndarray:
        """The history rows the encoder reads, (len(slots), maxQuesCount, width)."""
        return self.eng.dialog_slot_history([int(s) for s in slots], self.histWidth)

    def close(self):
        self.eng.dialog_end()


class DialogSession(DialogPool):
    """Dialogs that are asked one question per round, each round answered before the next is asked (vd_dialog_begin,
    DESIGN §19): the pool whose slots 0..B-1 are dialogs `inds`, all asked at every round.  Fed the dataset's questions, a
    session answers as generateAnswers / retrieveAnswers with `history = "generated"` do."""

    def __init__(self, model, dataloader, dtype, inds, params):
        super().__init__(model, dataloader, dtype, params)
        self.inds = np.asarray(list(inds), dtype=np.int64)
        self.rowOffset = (self.offset + int(self.inds[0])) * self.R      # draws as generateAnswers' for consecutive inds
        img = getattr(dataloader, "unique_img_" + dtype, None)
        self.image_ids = [_image_id(img[self.offset + int(i)]) if img is not None else self.offset + int(i) for i in self.inds]
        host = self._batch(self.inds)
        self.eng.dialog_begin(Batch(host), self.histWidth, self.maxAnsLen)
        self.capacity = len(self.inds)
        self.convs = {b: {"ind": int(i), "base": b * self.R, "ques": [], "ans": []} for b, i in enumerate(self.inds)}
        self.caption = host["hist"][:, 0] if "hist" in host else None      # round 0's history row

    @property
    def round(self) -> int:
        return self.eng.dialog_round()[0]

    def ask(self, questions) -> list:
        """Asks the next round: one question per dialog, text (utils.question_words, unknown words as UNK) or token ids.
        Returns one entry per dialog as generateAnswers' (question, answer token lists, score / length for the beam, and
        their text), or retrieveAnswers' for disc models; None where no beam reached <END>."""
        from .utils import question_ids
        if len(questions) != len(self.inds):
            raise ValueError("one question per dialog: %d dialogs, %d questions" % (len(self.inds), len(questions)))
        q = np.stack([question_ids(x, self.dl.word2ind, self.width) for x in questions])
        return self._ask(list(range(len(q))), q)

    def history(self) -> np.ndarray:
        """The history rows the encoder reads, (dialogs, maxQuesCount, width)."""
        return self.eng.dialog_history(self.histWidth)
