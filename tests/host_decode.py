"""TEST INFRASTRUCTURE ONLY.  Host reference of Model:generateAnswers' decoder loop (model.lua:472-602): forwardConnect's
start state, one decoder step through vd_gen_decoder_step with the state passed through the host, and the beam search with
the candidate merge of model.lua:529-569 on the host.  The search runs the device search's decoder kernels at its row count
(N rounds x k hypotheses) and takes the top k from the same log-probability bits, and the host copies of the state are
exact, so its answers, lengths and fp64 scores are those of vd_gen_beam_search bit for bit."""
import numpy as np


def start_state(eng, encOut, k=1):
    """forwardConnect's (h, c) for every round of the last encoder forward (model.lua:478-503, gen.lua:30-42) as host
    arrays: h = [layer-1 h at Tq, encOut], c = [layer-1 c, layer-2 c], each round's row repeated k times.  Encoders without
    .rnnLayers feed explicit zero rows, as the device search and sampler do."""
    N, H = encOut.shape
    (h1, c1), (_, c2) = [eng.encoder_rnn_state(l, N) for l in range(2)]
    if h1 is None:                                                              # :493-501
        h1 = c1 = c2 = np.zeros((N, H), np.float32)
    else:                                                                       # :482-491
        h1, c1, c2 = h1.numpy(), c1.numpy(), c2.numpy()
    h = [np.repeat(a, k, 0) for a in (h1, np.asarray(encOut, np.float32))]
    c = [np.repeat(a, k, 0) for a in (c1, c2)]
    return h, c


class HostStep:
    """One decoder step (vd_gen_decoder_step) on `rows` rows with the state passed through the host: uploads h = [h1, h2]
    and c = [c1, c2] (each (rows, H)) into four device buffers it owns and returns (logp (rows, V), [h1, h2], [c1, c2]) as
    numpy.  A context manager: the buffers are freed on exit."""

    def __init__(self, eng, rows):
        self.eng, self.shape = eng, (rows, eng.params["rnnHiddenSize"])
        self.bufs = [eng.device_alloc(rows * self.shape[1] * 4) for _ in range(4)]

    def __call__(self, tokens, h, c):
        assert len(tokens) == self.shape[0], (len(tokens), self.shape)
        for b, a in zip(self.bufs, h + c):
            assert a.shape == self.shape, (a.shape, self.shape)
            self.eng.upload(b, a)
        return self.eng.gen_decoder_step(tokens, self.bufs[0:2], self.bufs[2:4])

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        for b in self.bufs:
            self.eng.device_free(b)


def host_beam_search(eng, encOut, k, L, start, end, stats=None):
    """The beam branch of Model.generateAnswers for all rounds of the last encoder forward at once, the candidate merge of
    model.lua:529-569 — with its quirks — on the host.  Returns (answer (N, L), length (N), score (N)) in
    vd_gen_beam_search's format.  `stats` counts the cases worth covering: beam columns left without a candidate, pad
    tokens fed to the decoder, and the steps at which some hypothesis reached `end`."""
    N = encOut.shape[0]
    h, c = start_state(eng, encOut, k)
    beams = np.zeros((N, L, k), dtype=np.int64)                                 # :479
    beams[:, 0, :] = start                                                      # :506
    scores = np.zeros((N, k), dtype=np.float64)                                 # :507
    finish = [[] for _ in range(N)]                                             # :508
    with HostStep(eng, N * k) as step:
        for stp in range(1, L):                                                 # :510
            fed = beams[:, stp - 1, :].reshape(-1)
            logp, out_h, out_c = step(fed, h, c)                                # :519-526
            top = np.argsort(-logp, axis=1, kind="stable")[:, :k]               # :538-542 topk, sorted; ties: lower class
            h, c = [a.copy() for a in h], [a.copy() for a in c]                 # a column without a candidate keeps its state
            exploreSize = 1 if stp == 1 else k                                  # :516
            if stats is not None:
                stats["pad_rows"] += int((fed == 0).sum())
            for it in range(N):
                cands = []
                for wordId in range(exploreSize):                               # :529
                    r = it * k + wordId
                    for cls in top[r]:                                          # :544
                        tok = int(cls) + 1
                        sc = float(scores[it, wordId]) + float(logp[r, cls])
                        if tok == end:                                          # :548
                            cb = beams[it, :, wordId].copy()
                            cb[stp] = tok
                            finish[it].append({"beam": cb, "length": stp + 1, "score": sc})
                            if stats is not None:
                                stats["end_steps"].add(stp)
                        else:
                            cands.append((sc, wordId, tok))
                cands.sort(key=lambda t: -t[0])                                 # :558 (stable)
                if stats is not None and len(cands) < k:
                    stats["stale"] += k - len(cands)
                old = beams[it].copy()
                for candId in range(min(len(cands), k)):                        # :560-569
                    sc, wordId, tok = cands[candId]
                    beams[it, :, candId] = old[:, wordId]
                    beams[it, stp, candId] = tok
                    scores[it, candId] = sc
                    for a, o in zip(h + c, out_h + out_c):
                        a[it * k + candId] = o[it * k + wordId]
    answer = np.zeros((N, L), np.int32)
    length = np.zeros(N, np.int32)
    score = np.zeros(N, np.float64)
    for it in range(N):
        finish[it].sort(key=lambda d: -d["score"])                              # :572
        if finish[it]:
            best = finish[it][0]
            answer[it], length[it], score[it] = best["beam"], best["length"], best["score"]
    return answer, length, score
