"""How the Python layer answers questions, without a device: Model.generateAnswers / retrieveAnswers and DialogSession /
DialogPool asks over the real Engine wrappers, whose C library is a stand-in.  The stand-in records every answering call
in its general form (the narrow entry points expanded by the C ABI's equivalences, DESIGN §22-§24: a plain search is the
n-best search at G = 1, n = 1, alpha = 0 and lambda = 0; an untruncated draw is the truncated one at top_k = 0, top_p = 1),
with whether the call asked for norms, refuses what the library refuses, and answers with pseudo-random outputs seeded
from that general form, so that a narrow call and its general equivalent return the same data, as the library does.
The calls and the entries returned (the SHA-256 of their JSON, key order included: it is in the bytes of results.json)
are pinned by tests/golden/answer_spec_host.json; `PYTHONPATH=. python tests/test_answer_spec_host.py` rewrites it."""
import ctypes as C
import hashlib
import json
import math
import os
import types
import zlib

import numpy as np
import pytest

from visdial_b200._lib import VD_E_BADARG, VdError
from visdial_b200.engine import DEFAULT_PARAMS, Batch, Engine, derive_flags
from visdial_b200.model import Model

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "answer_spec_host.json")

VOCAB = ["UNK", "is", "it", "red", "?", "yes", "no", "a", "dog", "the", "cat", "blue", "two", "on", "<START>", "<END>"]
V, R = len(VOCAB), 3
START, END = V - 1, V
THREADS, OFFSET, POOL_ROWS = 4, 2, 10


def _arr(ptr, ctype, n):
    return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(ctype)), (n,))


def _refuse(ok, what):
    if not ok:
        raise VdError(VD_E_BADARG, what)


class FakeLib:
    """The answering and dialog entry points of libvisdial_b200 the wrappers reach, on the host."""

    def __init__(self, log):
        self.log, self.rows, self.pool_m, self.slots = log, None, 0, []

    # ---- outputs
    def _rng(self, canon):
        return np.random.default_rng(zlib.crc32(repr(canon).encode()))

    def _beam(self, canon, rows, G, nb, L, alpha, ptrs, norms):
        self.log.append(list(canon) + [norms])
        k, lam = canon[-8], canon[-6]
        _refuse(1 <= nb <= 32 and math.isfinite(alpha) and alpha >= 0, "nbest / length_penalty")
        _refuse(1 <= k <= min(32, V) and L >= 2, "beam_size / beam_len")
        _refuse(G >= 1 and k % G == 0, "groups")
        _refuse(math.isfinite(lam) and lam >= 0, "diversity")
        rng, n = self._rng(canon), rows * G * nb
        length = rng.integers(2, L + 1, n).astype(np.int32) * (rng.random(n) > 0.2)
        ans = rng.integers(1, V + 1, (n, L)).astype(np.int32)
        score = -rng.random(n) * 10
        norm = score if alpha == 0 and nb == 1 else -rng.random(n) * 10
        for p, ct, a in zip(ptrs, (C.c_int32, C.c_int32, C.c_double, C.c_double), (ans, length, score, norm)):
            if p is not None:
                _arr(p, ct, a.size)[:] = a.ravel()

    def _sample(self, canon, rows, L, temperature, start, row_offset, top_k, top_p, ans_p, logp_p):
        self.log.append(list(canon))
        _refuse(L >= 1 and math.isfinite(temperature) and temperature > 0 and row_offset >= 0 and 1 <= start <= V, "sample")
        _refuse(top_k >= 0 and math.isfinite(top_p) and 0 < top_p <= 1, "top_k / top_p")
        rng = self._rng(canon)
        ans = rng.integers(1, V + 1, (rows, L + 1)).astype(np.int32)
        ans[:, 0] = start
        _arr(ans_p, C.c_int32, ans.size)[:] = ans.ravel()
        if logp_p is not None:
            _arr(logp_p, C.c_float, rows * L)[:] = -rng.random(rows * L)

    def _pool(self, canon, rows, k, index_p, score_p):
        self.log.append(list(canon))
        _refuse(1 <= k <= min(32, self.pool_m), "k")
        rng = self._rng(canon)
        _arr(index_p, C.c_int32, rows * k)[:] = rng.integers(0, self.pool_m, rows * k)
        _arr(score_p, C.c_float, rows * k)[:] = rng.random(rows * k)

    @staticmethod
    def _batch(b):
        b = b._obj
        return [int(b.B), int(b.Tq), int(b.Th)]

    def _asked(self, slots_p, n, ques_p, Tq):
        s = _arr(slots_p, C.c_int32, n).tolist()
        q = _arr(ques_p, C.c_int32, n * Tq).reshape(n, Tq).tolist()
        for x in s:
            self.slots[x] += 1
        return s, q

    # ---- the split: the rounds of the last encoder forward
    def vd_gen_nbest_beam_search(self, h, k, G, lam, alpha, nb, L, start, end, a, ln, sc, nm):
        self._beam(("split", "beam", k, G, lam, alpha, nb, L, start, end), self.rows, G, nb, L, alpha, (a, ln, sc, nm),
                   nm is not None)

    def vd_gen_diverse_beam_search(self, h, k, G, lam, L, start, end, a, ln, sc):
        self.vd_gen_nbest_beam_search(h, k, G, lam, 0.0, 1, L, start, end, a, ln, sc, None)

    def vd_gen_beam_search(self, h, k, L, start, end, a, ln, sc):
        self.vd_gen_diverse_beam_search(h, k, 1, 0.0, L, start, end, a, ln, sc)

    def vd_gen_truncated_sample(self, h, L, start, T, seed, off, top_k, top_p, a, lp):
        self._sample(("split", "sample", L, start, T, seed, off, top_k, top_p), self.rows, L, T, start, off, top_k, top_p,
                     a, lp)

    def vd_gen_sample(self, h, L, start, T, seed, off, a, lp):
        self.vd_gen_truncated_sample(h, L, start, T, seed, off, 0, 1.0, a, lp)

    def vd_answer_pool_retrieve(self, h, b, k, index, score):
        self.rows = b._obj.B * R
        self._pool(("split", "pool", self._batch(b), k), self.rows, k, index, score)

    # ---- the dialog loop: every round of a batch's dialogs on their own answers
    def vd_gen_dialog_nbest_beam_search(self, h, b, k, G, lam, alpha, nb, L, start, end, hw, mal, a, ln, sc, nm, hist):
        self.rows = b._obj.B * R
        self._beam(("dialog", "beam", self._batch(b), hw, mal, k, G, lam, alpha, nb, L, start, end), self.rows, G, nb, L,
                   alpha, (a, ln, sc, nm), nm is not None)

    def vd_gen_dialog_diverse_beam_search(self, h, b, k, G, lam, L, start, end, hw, mal, a, ln, sc, hist):
        self.vd_gen_dialog_nbest_beam_search(h, b, k, G, lam, 0.0, 1, L, start, end, hw, mal, a, ln, sc, None, hist)

    def vd_gen_dialog_beam_search(self, h, b, k, L, start, end, hw, mal, a, ln, sc, hist):
        self.vd_gen_dialog_diverse_beam_search(h, b, k, 1, 0.0, L, start, end, hw, mal, a, ln, sc, hist)

    def vd_gen_dialog_truncated_sample(self, h, b, L, start, end, T, seed, off, top_k, top_p, hw, mal, a, lp, hist):
        self.rows = b._obj.B * R
        self._sample(("dialog", "sample", self._batch(b), hw, mal, L, start, end, T, seed, off, top_k, top_p), self.rows, L,
                     T, start, off, top_k, top_p, a, lp)

    def vd_gen_dialog_sample(self, h, b, L, start, end, T, seed, off, hw, mal, a, lp, hist):
        self.vd_gen_dialog_truncated_sample(h, b, L, start, end, T, seed, off, 0, 1.0, hw, mal, a, lp, hist)

    def vd_answer_pool_dialog(self, h, b, k, hw, mal, index, score, hist):
        self.rows = b._obj.B * R
        self._pool(("dialog", "pool", self._batch(b), hw, mal, k), self.rows, k, index, score)

    # ---- slot asks of a session or a pool
    def vd_dialog_ask_nbest_slots(self, h, slots, n, ques, Tq, k, G, lam, alpha, nb, L, start, end, a, ln, sc, nm):
        s, q = self._asked(slots, n, ques, Tq)
        self._beam(("slots", "beam", s, q, k, G, lam, alpha, nb, L, start, end), n, G, nb, L, alpha, (a, ln, sc, nm),
                   nm is not None)

    def vd_dialog_ask_diverse_slots(self, h, slots, n, ques, Tq, k, G, lam, L, start, end, a, ln, sc):
        self.vd_dialog_ask_nbest_slots(h, slots, n, ques, Tq, k, G, lam, 0.0, 1, L, start, end, a, ln, sc, None)

    def vd_dialog_ask_beam_slots(self, h, slots, n, ques, Tq, k, L, start, end, a, ln, sc):
        self.vd_dialog_ask_diverse_slots(h, slots, n, ques, Tq, k, 1, 0.0, L, start, end, a, ln, sc)

    def vd_dialog_ask_truncated_slots(self, h, slots, n, ques, Tq, L, start, end, T, seed, off, top_k, top_p, a, lp):
        s, q = self._asked(slots, n, ques, Tq)
        self._sample(("slots", "sample", s, q, L, start, end, T, seed, off, top_k, top_p), n, L, T, start, off, top_k, top_p,
                     a, lp)

    def vd_dialog_ask_sample_slots(self, h, slots, n, ques, Tq, L, start, end, T, seed, off, a, lp):
        self.vd_dialog_ask_truncated_slots(h, slots, n, ques, Tq, L, start, end, T, seed, off, 0, 1.0, a, lp)

    def vd_dialog_ask_pool_slots(self, h, slots, n, ques, Tq, k, index, score):
        s, q = self._asked(slots, n, ques, Tq)
        self._pool(("slots", "pool", s, q, k), n, k, index, score)

    # ---- state the wrappers keep around the answering calls
    def vd_set_answer_rules(self, h, r):
        r = r._obj if r is not None else None
        self.log.append(["rules"] + ([r.min_words, r.no_repeat_ngram, [r.banned[i] for i in range(r.n_banned)]]
                                     if r is not None else []))

    def vd_answer_pool_encode(self, h, tokens, m, width):
        self.pool_m = m
        self.log.append(["pool_encode", m, width])

    def vd_dialog_begin(self, h, b, hw, mal):
        self.slots = [0] * b._obj.B
        self.log.append(["begin", self._batch(b), hw, mal])

    def vd_dialog_open(self, h, cap, Tq, hw, mal):
        self.slots = [-1] * cap
        self.log.append(["open", cap, Tq, hw, mal])

    def vd_dialog_join(self, h, b, base, slots):
        B = b._obj.B
        free = [s for s, r in enumerate(self.slots) if r < 0][:B]
        for s in free:
            self.slots[s] = 0
        _arr(slots, C.c_int32, B)[:] = free
        self.log.append(["join", self._batch(b), _arr(base, C.c_int64, B).tolist(), free])

    def vd_dialog_join_rounds(self, h, b, rounds, answers, Ta, base, slots):
        B = b._obj.B
        r, s = _arr(rounds, C.c_int32, B).tolist(), _arr(slots, C.c_int32, B).tolist()
        for x, y in zip(s, r):
            self.slots[x] = y
        q = np.ctypeslib.as_array(C.cast(b._obj.ques_fwd, C.POINTER(C.c_int32)), (B * R * b._obj.Tq,)).tolist()
        a = _arr(answers, C.c_int32, B * R * Ta).tolist() if answers is not None else None
        self.log.append(["join_rounds", self._batch(b), r, s, _arr(base, C.c_int64, B).tolist(), q, a])

    def vd_dialog_slots(self, h, rounds, cap):
        cap._obj.value = len(self.slots)
        if rounds is not None:
            _arr(rounds, C.c_int32, len(self.slots))[:] = self.slots

    def vd_dialog_round(self, h, r, b):
        r._obj.value, b._obj.value = self.slots[0], len(self.slots)

    def vd_dialog_leave(self, h, slots, n):
        for s in _arr(slots, C.c_int32, n).tolist():
            self.slots[s] = -1

    def vd_dialog_end(self, h):
        self.log.append(["end"])


def _returns_ok(fn):
    def call(*args):
        fn(*args)
        return 0
    return call


for _name in [n for n in vars(FakeLib) if n.startswith("vd_")]:
    setattr(FakeLib, _name, _returns_ok(getattr(FakeLib, _name)))


class _Batch(Batch):
    def __contains__(self, k):
        return k in self.arrays


class StubLoader:
    """The dataloader fields the answering paths read, for THREADS dialogs of split "val" from dialog OFFSET on."""
    maxQuesLen, maxAnsLen, maxHistoryLen, concatHistory = 6, 5, 12, False

    def __init__(self):
        rng = np.random.default_rng(7)
        n = OFFSET + THREADS + 1
        self.word2ind = {w: i + 1 for i, w in enumerate(VOCAB)}
        self.ind2word = {i: w for w, i in self.word2ind.items()}
        self.numThreads = {"val": THREADS}
        self.part = {"val": (OFFSET, OFFSET + THREADS)}
        self.unique_img_val = ["COCO_val2014_%012d.jpg" % (100 + i) for i in range(n)]
        qlen = rng.integers(1, self.maxQuesLen + 1, (n, R))
        self.corpus = {"val": types.SimpleNamespace(raw={"ques_length": qlen})}
        self.ques = np.zeros((n, R, self.maxQuesLen), np.int32)
        self.ans = np.zeros((n, R, self.maxAnsLen + 1), np.int32)
        for d in range(n):
            for r in range(R):
                self.ques[d, r, self.maxQuesLen - qlen[d, r]:] = rng.integers(1, START, qlen[d, r])
                la = int(rng.integers(1, self.maxAnsLen + 1))
                self.ans[d, r, :la] = rng.integers(1, START, la)
                self.ans[d, r, la] = END
        self.hist = rng.integers(0, START, (n, R, self.maxHistoryLen)).astype(np.int32)
        self.pool = rng.integers(1, V + 1, (POOL_ROWS, self.maxAnsLen)).astype(np.int32)
        self.pool[:, 3:] *= rng.random((POOL_ROWS, self.maxAnsLen - 3)) > 0.5

    def getIndexData(self, inds, params, dtype):
        g = self.part[dtype][0] + np.asarray(inds, dtype=np.int64).reshape(-1)
        Tq = int(self.corpus[dtype].raw["ques_length"][g].max())
        return _Batch({"ques_fwd": self.ques[g][:, :, self.maxQuesLen - Tq:], "hist": self.hist[g], "answer_out": self.ans[g]})

    def answerPool(self, dtype):
        return self.pool


def _model(decoder, log, encoder="hre-ques-hist"):
    """A Model over an Engine whose library is FakeLib: the encoder forward of generateAnswers' split path sets the rows"""
    m = Model.__new__(Model)
    m.params = derive_flags(dict(DEFAULT_PARAMS, encoder=encoder, decoder=decoder, vocabSize=V, maxQuesCount=R))
    eng = Engine.__new__(Engine)
    eng.lib, eng.h, eng.params, eng._enc_rows = FakeLib(log), None, m.params, None
    m.engine = eng
    m.wrapper = types.SimpleNamespace(evaluate=lambda: None, training=lambda: None)

    def forwardBackward(batch, onlyForward=False, encOutOnly=False):
        assert onlyForward and encOutOnly
        eng._enc_rows = eng.lib.rows = len(batch["ques_fwd"]) * R
        log.append(["encode", len(batch["ques_fwd"])])
    m.forwardBackward = forwardBackward
    return m


GEN = {
    "plain": {},
    "groups2": {"beamGroups": 2, "beamSize": 4, "diversity": 0.3},
    "nbest3": {"nBest": 3, "lengthPenalty": 0.7},
    "groups2_nbest2": {"beamGroups": 2, "nBest": 2, "beamSize": 4},
    "alpha_only": {"lengthPenalty": 0.5, "beamGroups": 2, "beamSize": 4},
    "sample": {"sampleWords": 1, "temperature": 0.8, "seed": 99, "beamLen": 4},
    "topk5": {"sampleWords": 1, "topK": 5},
    "topp": {"sampleWords": 1, "topP": 0.9},
    "topk_v": {"sampleWords": 1, "topK": V},
    "rules_beam": {"minWords": 2, "noRepeatNgram": 2, "bannedWords": ["red", "dog"]},
    "rules_sample": {"sampleWords": 1, "minWords": 1, "bannedWords": ["no"], "topK": 3},
    "groups0": {"beamGroups": 0},
    "groups0_nbest2": {"beamGroups": 0, "nBest": 2},
    "diversity_neg": {"diversity": -1.0},
    "diversity_neg_nbest2": {"diversity": -1.0, "nBest": 2},
    "topk_neg": {"sampleWords": 1, "topK": -1},
    "topp_big": {"sampleWords": 1, "topP": 1.5},
    "nbest0": {"nBest": 0},
    "unknown_banned": {"bannedWords": ["zebra"]},
}
DISC = {"top1": {}, "top3": {"topK": 3}, "top0": {"topK": 0}, "rules_ignored": {"topK": 2, "minWords": 3}}


def _run(fn):
    try:
        return {"out": hashlib.sha256(json.dumps(fn()).encode()).hexdigest()}
    except (VdError, ValueError, IndexError) as e:
        return {"raise": type(e).__name__}


def _dialogs(m, dl, params, log):
    """a session on dialogs 0 and 2, then a pool: joins, asks, a join with rounds, a resume, a reopen"""
    out = {}
    s = m.openDialogs(dl, "val", [0, 2], params)
    out["session"] = [s.ask([[3, 2, 4], "is the cat blue"]), s.ask(["two dogs?", []])]
    s.close()
    p = m.openDialogPool(dl, "val", 4, params)
    a = p.join([1, 3])
    asks = [p.ask({a[0]: "is it red", a[1]: [5, 9, 10]})]
    b = p.join([0], rounds=[2])
    c = p.resume(2, [("is it a dog", "yes"), ([2, 3], [6, 7, 0])])
    asks.append(p.ask({a[1]: "on the cat", b[0]: "is it", c: [12, 13]}))
    p.reopen()
    asks.append(p.ask({c: "blue?", a[0]: "no"}))
    p.leave([a[1]])
    out["pool"] = asks
    out["convs"] = {str(k): {"ind": v["ind"], "base": v["base"], "ques": [np.asarray(x).tolist() for x in v["ques"]],
                             "ans": [list(map(int, x)) for x in v["ans"]]} for k, v in sorted(p.convs.items())}
    p.close()
    return out


def cases():
    """(case id, decoder, params, what to run): every answering path over the params grid"""
    for name, params in GEN.items():
        for history in ("gt", "generated"):
            for dpc in (1, 3):
                yield ("gen/%s/%s/dpc%d" % (name, history, dpc), "gen", params,
                       lambda m, dl, p, log, h=history, d=dpc: m.generateAnswers(dl, "val", dict(p, history=h, dialogsPerCall=d),
                                                                                strict=False))
        yield ("gen/%s/strict" % name, "gen", params, lambda m, dl, p, log: m.generateAnswers(dl, "val", p))
        yield ("gen/%s/dialogs" % name, "gen", params, _dialogs)
    for name, params in DISC.items():
        for history in ("gt", "generated"):
            for dpc in (1, 3):
                yield ("disc/%s/%s/dpc%d" % (name, history, dpc), "disc", params,
                       lambda m, dl, p, log, h=history, d=dpc: m.retrieveAnswers(dl, "val", dict(p, history=h, dialogsPerCall=d)))
        yield ("disc/%s/dialogs" % name, "disc", params, _dialogs)


def record(case):
    cid, decoder, params, fn = case
    log = []
    m = _model(decoder, log)
    got = _run(lambda: fn(m, StubLoader(), dict(params), log))
    got["calls"] = json.loads(json.dumps(log))
    return got


_CASES = list(cases())


@pytest.fixture(scope="module")
def golden():
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.mark.parametrize("case", _CASES, ids=[c[0] for c in _CASES])
def test_answering_calls_and_entries(case, golden):
    want, got = golden[case[0]], record(case)
    assert got["calls"] == want["calls"]
    assert got.get("raise") == want.get("raise")
    assert got.get("out") == want.get("out")       # the JSON text's hash: key order included


def test_every_case_is_pinned(golden):
    assert sorted(golden) == sorted(c[0] for c in _CASES)


if __name__ == "__main__":
    with open(GOLDEN, "w") as f:
        json.dump({c[0]: record(c) for c in _CASES}, f, indent=0, sort_keys=True)
        f.write("\n")
