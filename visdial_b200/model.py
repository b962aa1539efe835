"""Mirror of the reference's `Model` class (/root/reference/model.lua:8-430) over the C engine.
Same method names, argument meaning and call order as the Lua original, so that the parity tests
read like the reference's own driver code.  `generateAnswers` (beam search / sampling, model.lua:432-613) runs the beam
search and the sampling entirely on the device (vd_gen_beam_search, vd_gen_sample); the reference-structured beam loop steps
the decoder through vd_gen_decoder_step and keeps the hypothesis bookkeeping on the host like the Lua."""
from __future__ import annotations

import numpy as np

from . import decoders, encoders
from .engine import Batch, DEFAULT_PARAMS, derive_flags
from .modules import Criterion, Sequential
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
        through vd_gen_beam_search / vd_gen_sample, for `params.dialogsPerCall` dialogs (default 1) per encoder forward:
        every round of those dialogs is searched or sampled at once.  `hostBeam = 1` (the reference's loop structure) goes
        one dialog at a time, the decoder stepped through vd_gen_decoder_step and the hypothesis bookkeeping on the host as
        the Lua does it.  Returns the reference's answerTable with token-id lists (and text when the dataloader carries
        ind2word).  `strict=False` yields None for a round where no beam reached <END> (the reference indexes nil there,
        model.lua:575)."""
        if self.params["decoder"] == "disc":                                            # :434-437
            raise ValueError("Sampling/beam search only for generative model")
        params = params or {}
        sampleWords = bool(params.get("sampleWords", 0) == 1)                           # :443
        temperature = float(params.get("temperature", 1.0))
        beamSize, beamLen = int(params.get("beamSize", 5)), int(params.get("beamLen", 20))
        startToken, endToken = dataloader.word2ind["<START>"], dataloader.word2ind["<END>"]   # :453-454
        numThreads = int(params.get("maxThreads") or dataloader.numThreads[dtype])      # :455
        ind2word = getattr(dataloader, "ind2word", None)
        eng, H = self.engine, self.params["rnnHiddenSize"]
        words = (lambda ids: " ".join(ind2word.get(int(t), "<UNK>") for t in ids if int(t) > 0)) if ind2word else None
        img = getattr(dataloader, "unique_img_" + dtype, None)
        # getIndexData hands out this rank's slice of the split: the image list is indexed by the global dialog id
        first = dataloader.part[dtype][0] if hasattr(dataloader, "part") and dtype in getattr(dataloader, "part", {}) else 0

        def image_id(convId):
            gid = convId + first
            return _image_id(img[gid]) if img is not None else gid

        def entry(q, answer, score, length):
            e = {"question": q.tolist(), "answer": answer.tolist(), "score": score, "length": length}
            if words:
                e["question_text"], e["answer_text"] = words(q), words(answer)
            return e

        dialogsPerCall = max(1, int(params.get("dialogsPerCall", 1)))
        if sampleWords:
            return self._generate_sample(dataloader, dtype, numThreads, dialogsPerCall, beamLen, startToken, temperature,
                                         int(params.get("seed", 1234)), first, image_id, words)
        if not params.get("hostBeam"):
            return self._generate_beam(dataloader, dtype, numThreads, dialogsPerCall, beamSize, beamLen, startToken, endToken,
                                       strict, image_id, entry)
        state_buf = [eng.device_alloc(max(beamSize, self.params["maxQuesCount"]) * H * 4) for _ in range(4)]
        answerTable = []
        try:
            for convId in range(numThreads):
                self.wrapper.evaluate()                                                 # :460
                batch = dataloader.getIndexData(np.array([convId]), self.params, dtype)  # :462-463
                encOut = self.forwardBackward(batch, True, True).numpy()                # :467 (N,H), N = 10
                ques = batch["ques_fwd"].reshape(-1, batch.c.Tq)
                N = encOut.shape[0]
                layers = [eng.encoder_rnn_state(l, N) for l in range(2)]
                has_layers = layers[0][0] is not None
                encH = [(layers[l][0].numpy(), layers[l][1].numpy()) for l in range(2)] if has_layers else None
                threadAnswers = []

                def step(tokens, Hs, Cs):
                    n = len(tokens)
                    for i, a in enumerate(Hs + Cs):
                        eng.upload(state_buf[i], a[:n])
                    return eng.gen_decoder_step(tokens, state_buf[0:2], state_buf[2:4])

                # the reference's own loop structure (one round at a time, log-probabilities and state through the host):
                # kept as the cross-check of the device search (params.hostBeam = 1)
                for it in range(N):                                                 # :472
                    beams = np.zeros((beamLen, beamSize), dtype=np.int64)           # :479
                    if has_layers:                                                  # :482-491
                        Hs = [encH[0][0][it], encOut[it]]
                        Cs = [encH[0][1][it], encH[1][1][it]]
                    else:                                                           # :493-501
                        Hs = [np.zeros(H, np.float32), encOut[it]]
                        Cs = [np.zeros(H, np.float32), np.zeros(H, np.float32)]
                    Hs = [np.repeat(h[None], beamSize, 0).astype(np.float32) for h in Hs]
                    Cs = [np.repeat(c[None], beamSize, 0).astype(np.float32) for c in Cs]
                    beams[0] = startToken                                           # :506
                    scores = np.zeros(beamSize, dtype=np.float64)                   # :507
                    finishBeams = []
                    for stp in range(1, beamLen):                                   # :510
                        cands = []
                        exploreSize = 1 if stp == 1 else beamSize                   # :516
                        decOut, nH, nC = step(beams[stp - 1], Hs, Cs)               # :519-526
                        for wordId in range(exploreSize):                           # :529
                            order = np.argsort(-decOut[wordId], kind="stable")[:beamSize]   # :538-542 topk, sorted
                            for candId in range(beamSize):                          # :544
                                candBeam = beams[:, wordId].copy()
                                tok = int(order[candId]) + 1
                                candBeam[stp] = tok
                                sc = float(scores[wordId]) + float(decOut[wordId, order[candId]])
                                if tok == endToken:                                 # :548
                                    finishBeams.append({"beam": candBeam, "length": stp + 1, "score": sc})
                                else:
                                    cands.append((sc, candBeam, [h[wordId].copy() for h in nH], [c[wordId].copy() for c in nC]))
                        cands.sort(key=lambda t: -t[0])                             # :558
                        for candId in range(min(len(cands), beamSize)):             # :560-569
                            beams[:, candId] = cands[candId][1]
                            for lv in range(2):
                                Hs[lv][candId] = cands[candId][2][lv]
                                Cs[lv][candId] = cands[candId][3][lv]
                            scores[candId] = cands[candId][0]
                    finishBeams.sort(key=lambda d: -d["score"])                     # :572
                    if not finishBeams:
                        if strict:
                            raise IndexError("no beam reached <END> within beamLen (model.lua:575 indexes nil here)")
                        threadAnswers.append(None)
                        continue
                    best = finishBeams[0]
                    threadAnswers.append(entry(ques[it], best["beam"], best["score"], best["length"]))
                self.wrapper.training()                                                 # :605
                answerTable.append({"image_id": image_id(convId), "dialog": threadAnswers})   # :606
        finally:
            for p in state_buf:
                eng.device_free(p)
        return answerTable

    def _generate_beam(self, dataloader, dtype, numThreads, dialogsPerCall, beamSize, beamLen, startToken, endToken, strict,
                       image_id, entry):
        """generateAnswers' beam search, `dialogsPerCall` dialogs per encoder forward and per vd_gen_beam_search call.  One
        dialog per call gives exactly the per-dialog trimming and kernel shapes of the reference's loop; more dialogs per call
        run wider kernels (in the tensor-core math modes their rounding can differ from per-dialog runs)."""
        answerTable = []
        ques_len = None
        for first in range(0, numThreads, dialogsPerCall):
            inds = np.arange(first, min(numThreads, first + dialogsPerCall))
            self.wrapper.evaluate()                                                     # :460
            batch = dataloader.getIndexData(inds, self.params, dtype)                   # :462-463
            self.forwardBackward(batch, True, True)                                     # :467
            ques = batch["ques_fwd"]                                                    # (D, maxQuesCount, Tq)
            Tq = ques.shape[2]
            answer, length, score = self.engine.gen_beam_search(beamSize, beamLen, startToken, endToken)   # :472-579
            answer = answer.reshape(len(inds), -1, beamLen)
            length, score = length.reshape(len(inds), -1), score.reshape(len(inds), -1)
            self.wrapper.training()                                                     # :605
            for d, convId in enumerate(inds):
                w, ques_len = _question_width(dataloader, dtype, inds, convId, Tq, ques_len)
                threadAnswers = []
                for it in range(ques.shape[1]):
                    if length[d, it] == 0:
                        if strict:
                            raise IndexError("no beam reached <END> within beamLen (model.lua:575 indexes nil here)")
                        threadAnswers.append(None)
                        continue
                    threadAnswers.append(entry(ques[d, it, Tq - w:], answer[d, it], float(score[d, it]), int(length[d, it])))
                answerTable.append({"image_id": image_id(int(convId)), "dialog": threadAnswers})   # :606
        return answerTable

    def _generate_sample(self, dataloader, dtype, numThreads, dialogsPerCall, beamLen, startToken, temperature, seed,
                         split_offset, image_id, words):
        """generateAnswers' sampling (model.lua:581-602), `dialogsPerCall` dialogs per encoder forward and per vd_gen_sample
        call.  The draws of a round depend only on (seed, its global round index, the step): the call passes the index of
        its first round in the split (this rank's offset included), so the answers do not depend on dialogsPerCall or on
        how the split is sharded over ranks, only on the logits."""
        R = self.params["maxQuesCount"]
        answerTable = []
        ques_len = None
        for first in range(0, numThreads, dialogsPerCall):
            inds = np.arange(first, min(numThreads, first + dialogsPerCall))
            self.wrapper.evaluate()                                                     # :460
            batch = dataloader.getIndexData(inds, self.params, dtype)                   # :462-463
            self.forwardBackward(batch, True, True)                                     # :467
            ques = batch["ques_fwd"]                                                    # (D, maxQuesCount, Tq)
            Tq = ques.shape[2]
            answer, _ = self.engine.gen_sample(beamLen, startToken, temperature, seed, (split_offset + first) * R)   # :582-594
            answer = answer.reshape(len(inds), -1, beamLen + 1)
            self.wrapper.training()                                                     # :605
            for d, convId in enumerate(inds):
                w, ques_len = _question_width(dataloader, dtype, inds, convId, Tq, ques_len)
                threadAnswers = []
                for it in range(ques.shape[1]):
                    q, a = ques[d, it, Tq - w:], answer[d, it]
                    e = {"question": q.tolist(), "answer": a.tolist()}
                    if words:
                        e["question_text"], e["answer_text"] = words(q), words(a)
                    threadAnswers.append(e)
                answerTable.append({"image_id": image_id(int(convId)), "dialog": threadAnswers})   # :606
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
