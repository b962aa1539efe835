"""Thin Python handle over the C engine (include/visdial_b200.h).  Only numpy + ctypes: torch is
not needed for the single-GPU path."""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Tuple

import numpy as np

from . import _lib
from ._lib import vd_batch, vd_params, check

# opts.lua:6-40 defaults (+ train.lua:55-59 fields the dataloader adds)
DEFAULT_PARAMS = dict(
    encoder="lf-ques-hist", decoder="gen", vocabSize=0, embedSize=300, rnnHiddenSize=512, numLayers=2,
    imgFeatureSize=4096, imgSpatialSize=14, imgEmbedSize=300, commonEmbeddingSize=512,
    numAttentionLayers=1, maxQuesCount=10, numOptions=100, dropout=0.5, gpuid=0,
    batchSize=40, learningRate=1e-3, lrDecayRate=0.9997592083, minLRate=5e-5, useGt=True,
    imgNorm=1,                                  # opts.lua:15; forced to 0 for 'att' encoders (opts.lua:66)
)


def derive_flags(params: dict) -> dict:
    """opts.lua:55-67: feature switches derived from the encoder name."""
    enc = params["encoder"]
    params["useHistory"] = "hist" in enc
    params["useIm"] = "im" in enc
    params["concatHistory"] = "lf" in enc
    if "att" in enc:
        params["imgNorm"] = 0
    return params


def to_c_params(params: dict) -> vd_params:
    p = vd_params()
    p.encoder = params["encoder"].encode()
    p.decoder = params["decoder"].encode()
    for k in ("vocabSize", "embedSize", "rnnHiddenSize", "numLayers", "imgFeatureSize", "imgSpatialSize",
              "imgEmbedSize", "commonEmbeddingSize", "numAttentionLayers", "maxQuesCount", "numOptions", "gpuid"):
        setattr(p, k, int(params.get(k, DEFAULT_PARAMS[k])))
    p.dropout = float(params.get("dropout", 0.5))
    p.imgRegions = int(params.get("imgRegions", 0))     # 0: the grid; P > 0: region rows (DESIGN §26)
    return p


class Segment:
    __slots__ = ("name", "offset", "rows", "cols", "init", "fan_in")

    def __init__(self, name, offset, rows, cols, init, fan_in):
        self.name, self.offset, self.rows, self.cols, self.init, self.fan_in = name, offset, rows, cols, init, fan_in

    @property
    def size(self):
        return self.rows * self.cols


def layout(params: dict) -> Tuple[List[Segment], int]:
    """Parameter layout of the flat vector (host-only; works without a GPU)."""
    lib = _lib.load()
    cp = to_c_params(params)
    nseg, ntot = C.c_int32(), C.c_int64()
    check(lib.vd_layout_count(C.byref(cp), C.byref(nseg), C.byref(ntot)))
    segs = []
    name = C.create_string_buffer(128)
    for i in range(nseg.value):
        off, rows, cols, fan = C.c_int64(), C.c_int64(), C.c_int64(), C.c_int64()
        kind = C.c_int32()
        check(lib.vd_layout_segment(C.byref(cp), i, name, 128, C.byref(off), C.byref(rows), C.byref(cols),
                                    C.byref(kind), C.byref(fan)))
        segs.append(Segment(name.value.decode(), off.value, rows.value, cols.value, kind.value, fan.value))
    return segs, ntot.value


def init_parameters(params: dict, seed: int = 1234) -> np.ndarray:
    """Upstream default initialisers, applied on the host like torch's nn constructors do
    (model_utils/weight-init.lua is a no-op on these graphs, SURVEY.md §2 #8):
    LookupTable N(0,1); Linear U(+-1/sqrt(in)); SeqLSTM W ~ N(0, 1/sqrt(D+H)), b = 0 except the
    forget block = 1 [upstream]."""
    segs, n = layout(params)
    rng = np.random.default_rng(seed)
    w = np.zeros(n, dtype=np.float32)
    H = int(params.get("rnnHiddenSize", 512))
    for s in segs:
        v = w[s.offset:s.offset + s.size]
        if s.init == _lib.INIT_EMBED:
            v[:] = rng.standard_normal(s.size, dtype=np.float32)
            v[:s.cols] = 0.0                              # pad row
        elif s.init in (_lib.INIT_LINEAR_W, _lib.INIT_LINEAR_B):
            b = 1.0 / np.sqrt(float(s.fan_in))
            v[:] = rng.uniform(-b, b, s.size).astype(np.float32)
        elif s.init == _lib.INIT_LSTM_W:
            v[:] = (rng.standard_normal(s.size) / np.sqrt(float(s.fan_in))).astype(np.float32)
        elif s.init == _lib.INIT_LSTM_B:
            v[:] = 0.0
            v[H:2 * H] = 1.0
    return w


def split_parameters(params: dict, flat: np.ndarray) -> Dict[str, np.ndarray]:
    """name -> array view of the flat vector (LSTM / Linear weights 2-D, biases 1-D)."""
    segs, _ = layout(params)
    out = {}
    for s in segs:
        v = flat[s.offset:s.offset + s.size]
        is_bias = s.init in (_lib.INIT_LINEAR_B, _lib.INIT_LSTM_B)
        out[s.name] = v.reshape(s.cols) if is_bias else v.reshape(s.rows, s.cols)
    return out


class DeviceTensor:
    """A device pointer + shape owned by the engine (the analogue of a module's .output tensor)."""

    def __init__(self, eng: "Engine", ptr: int, shape, dtype=np.float32):
        self.eng, self.ptr, self.shape, self.dtype = eng, ptr, tuple(int(x) for x in shape), np.dtype(dtype)

    def numpy(self) -> np.ndarray:
        out = np.empty(self.shape, dtype=self.dtype)
        check(self.eng.lib.vd_memcpy_d2h(self.eng.h, out.ctypes.data, self.ptr, out.nbytes))
        return out


def _ptr(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data


class Batch:
    """Keeps the numpy arrays alive and exposes the vd_batch struct.  Arrays are the dataloader's batch
    table (SURVEY.md Appendix A): int32 ids, float32 features, C-contiguous.  Region engines (imgRegions > 0) also take
    `img_count` (B,), each image's region count (DESIGN §26); without it every region is present."""

    KEYS_I32 = ("ques_fwd", "hist", "options", "answer_ind", "answer_in", "answer_out", "option_in", "option_out",
                "img_count")

    def __init__(self, arrays: Dict[str, np.ndarray]):
        self.arrays = {}
        for k, v in arrays.items():
            if v is None:
                continue
            if k in self.KEYS_I32:
                v = np.ascontiguousarray(v, dtype=np.int32)
            elif k == "img_feat":
                v = np.ascontiguousarray(v, dtype=np.float32)
            self.arrays[k] = v
        a = self.arrays
        b = vd_batch()
        q = a["ques_fwd"]
        b.B, b.Tq = q.shape[0], q.shape[2]
        b.Th = a["hist"].shape[2] if "hist" in a else 0
        b.Ta = a["answer_in"].shape[2] if "answer_in" in a else 0
        if "options" in a and "option_in" in a:
            raise ValueError("a batch carries either raw `options` (disc) or `option_in/option_out` (gen eval), not both")
        if "options" in a:
            b.To = a["options"].shape[2]
        elif "option_in" in a:
            b.To = a["option_in"].shape[3]
        else:
            b.To = 0
        for k in self.KEYS_I32 + ("img_feat",):
            setattr(b, k, _ptr(a.get(k)))
        b.on_device = 0
        self.c = b
        self.h2d_bytes = sum(int(v.nbytes) for k, v in a.items() if k in self.KEYS_I32 + ("img_feat",))

    def __getitem__(self, k):
        return self.arrays[k]

    def to_device(self, eng: "Engine") -> "Batch":
        """A copy of this batch resident in HBM (vd_batch.on_device = 1)."""
        out = Batch.__new__(Batch)
        out.arrays = self.arrays
        out.h2d_bytes = 0
        b = vd_batch()
        C.memmove(C.byref(b), C.byref(self.c), C.sizeof(vd_batch))
        out._dev = []
        for k in self.KEYS_I32 + ("img_feat",):
            a = self.arrays.get(k)
            if a is None:
                continue
            p = C.c_void_p()
            check(eng.lib.vd_device_alloc(eng.h, C.byref(p), a.nbytes))
            check(eng.lib.vd_memcpy_h2d(eng.h, p, a.ctypes.data, a.nbytes))
            setattr(b, k, p.value)
            out._dev.append(p)
        b.on_device = 1
        out.c = b
        return out


class Engine:
    """vd_engine handle.  Raises VdError on any failure; never falls back to the CPU."""

    def __init__(self, params: dict):
        self.lib = _lib.load()
        self.params = dict(DEFAULT_PARAMS)
        self.params.update(params)
        derive_flags(self.params)
        self.cparams = to_c_params(self.params)
        h = C.c_void_p()
        check(self.lib.vd_create(C.byref(self.cparams), C.byref(h)))
        self.h = h
        self._enc_rows = None          # N of the last encoder forward: the row count of vd_gen_beam_search's outputs
        n = C.c_int64()
        check(self.lib.vd_num_params(self.h, C.byref(n)))
        self.num_params = n.value

    def close(self):
        if getattr(self, "h", None):
            self.lib.vd_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- parameters -------------------------------------------------------------------------
    def set_parameters(self, flat: np.ndarray):
        flat = np.ascontiguousarray(flat, dtype=np.float32)
        check(self.lib.vd_set_parameters(self.h, flat.ctypes.data, flat.size))

    def get_parameters(self) -> np.ndarray:
        out = np.empty(self.num_params, dtype=np.float32)
        check(self.lib.vd_get_parameters(self.h, out.ctypes.data, out.size))
        return out

    def get_gradients(self) -> np.ndarray:
        out = np.empty(self.num_params, dtype=np.float32)
        check(self.lib.vd_get_gradients(self.h, out.ctypes.data, out.size))
        return out

    def param_buffers(self) -> Tuple[int, int]:
        w, dw = C.c_void_p(), C.c_void_p()
        check(self.lib.vd_param_buffers(self.h, C.byref(w), C.byref(dw)))
        return w.value, dw.value

    def optim_state(self) -> Tuple[np.ndarray, np.ndarray, int]:
        m, v, t = C.c_void_p(), C.c_void_p(), C.c_int64()
        check(self.lib.vd_optim_buffers(self.h, C.byref(m), C.byref(v), C.byref(t)))
        return (DeviceTensor(self, m.value, (self.num_params,)).numpy(),
                DeviceTensor(self, v.value, (self.num_params,)).numpy(), t.value)

    def set_optim_state(self, m: np.ndarray, v: np.ndarray, t: int):
        m = np.ascontiguousarray(m, dtype=np.float32)
        v = np.ascontiguousarray(v, dtype=np.float32)
        if m.size != self.num_params or v.size != self.num_params:
            raise ValueError("Adam state must have vd_num_params elements")
        check(self.lib.vd_set_optim_state(self.h, m.ctypes.data, v.ctypes.data, int(t)))

    def zero_grad(self):
        check(self.lib.vd_zero_grad(self.h))

    # ---- modes -------------------------------------------------------------------------------
    def set_training(self, mode: int):
        check(self.lib.vd_set_training(self.h, int(mode)))

    def set_dropout_seed(self, seed: int, iteration: int):
        check(self.lib.vd_set_dropout_seed(self.h, seed, iteration))

    def set_math_mode(self, mode: int):
        check(self.lib.vd_set_math_mode(self.h, mode))

    def set_answer_rules(self, min_words: int = 0, no_repeat_ngram: int = 0, banned=()):
        """The answer rules of every later beam search and sampling call (vd_set_answer_rules, DESIGN §25): <END> barred
        while an answer has fewer than `min_words` words, no repeated `no_repeat_ngram`-gram (0 = off), and the `banned`
        token ids never chosen.  All three at their defaults turn the rules off."""
        ids = np.ascontiguousarray(np.asarray(list(banned), dtype=np.int64).astype(np.int32).ravel())
        if min_words == 0 and no_repeat_ngram == 0 and ids.size == 0:
            check(self.lib.vd_set_answer_rules(self.h, None))
            return
        r = _lib.vd_answer_rules(int(min_words), int(no_repeat_ngram), int(ids.size),
                                 ids.ctypes.data_as(C.POINTER(C.c_int32)) if ids.size else None)
        check(self.lib.vd_set_answer_rules(self.h, C.byref(r)))

    def set_lazy_decout(self, on: bool):
        check(self.lib.vd_set_lazy_decout(self.h, 1 if on else 0))

    def set_option_overlap(self, on: bool, reserve_sms: int = -1):
        check(self.lib.vd_set_option_overlap(self.h, int(on), int(reserve_sms)))

    def set_deterministic(self, on: bool):
        """Deterministic training (vd_set_deterministic, DESIGN §27): every training step's loss, gradients and Adam update
        repeat bit for bit for the same parameters, math mode, weights, optimiser state, batch and dropout seed, whatever
        the GPU's SM count or the option stream's overlap.  Off by default; one GPU only."""
        check(self.lib.vd_set_deterministic(self.h, 1 if on else 0))

    # ---- module protocol -----------------------------------------------------------------------
    def _N(self, batch: Batch) -> int:
        return batch.c.B * self.params["maxQuesCount"]

    def encoder_forward(self, batch: Batch) -> DeviceTensor:
        p = C.c_void_p()
        self._enc_rows = None
        check(self.lib.vd_encoder_forward(self.h, C.byref(batch.c), C.byref(p)))
        self._enc_rows = self._N(batch)
        return DeviceTensor(self, p.value, (self._N(batch), self.params["rnnHiddenSize"]))

    def forward_connect(self):
        check(self.lib.vd_forward_connect(self.h))

    def decoder_forward(self, batch: Batch) -> DeviceTensor:
        p = C.c_void_p()
        check(self.lib.vd_decoder_forward(self.h, C.byref(batch.c), C.byref(p)))
        if self.params["decoder"] == "disc":
            shape = (self._N(batch), self.params["numOptions"])
        else:
            shape = (batch.c.Ta, self._N(batch), self.params["vocabSize"])
        return DeviceTensor(self, p.value, shape)

    def criterion_forward(self, batch: Batch) -> float:
        loss = C.c_float()
        check(self.lib.vd_criterion_forward(self.h, C.byref(batch.c), C.byref(loss)))
        return loss.value

    def criterion_backward(self, batch: Batch):
        check(self.lib.vd_criterion_backward(self.h, C.byref(batch.c)))

    def decoder_backward(self, batch: Batch):
        check(self.lib.vd_decoder_backward(self.h, C.byref(batch.c)))

    def backward_connect(self, batch: Batch) -> DeviceTensor:
        p = C.c_void_p()
        check(self.lib.vd_backward_connect(self.h, C.byref(p)))
        return DeviceTensor(self, p.value, (self._N(batch), self.params["rnnHiddenSize"]))

    def encoder_backward(self, batch: Batch, grad: DeviceTensor):
        check(self.lib.vd_encoder_backward(self.h, C.byref(batch.c), grad.ptr))

    # ---- fused ------------------------------------------------------------------------------------
    def forward_backward(self, batch: Batch, only_forward: bool = False) -> float:
        loss = C.c_float()
        self._enc_rows = None
        check(self.lib.vd_forward_backward(self.h, C.byref(batch.c), int(only_forward), C.byref(loss)))
        self._enc_rows = self._N(batch)
        return loss.value

    def forward_backward_dense(self, batch: Batch, rounds, relevance) -> float:
        """vd_forward_backward_dense: one step of the soft-target cross-entropy against dense relevances.  rounds (B,)
        0-based annotated round of each dialog, relevance (B, numOptions) >= 0 with positive row sums."""
        B, K = batch.c.B, self.params["numOptions"]
        rounds = np.ascontiguousarray(rounds, dtype=np.int32).reshape(-1)
        relevance = np.ascontiguousarray(relevance, dtype=np.float32)
        if rounds.shape != (B,) or relevance.shape != (B, K):
            raise ValueError("rounds must be (%d,) and relevance (%d, %d)" % (B, B, K))
        loss = C.c_float()
        self._enc_rows = None
        check(self.lib.vd_forward_backward_dense(self.h, C.byref(batch.c), rounds.ctypes.data, relevance.ctypes.data,
                                                 C.byref(loss)))
        self._enc_rows = self._N(batch)
        return loss.value

    def forward_backward_dense_gen(self, batch: Batch, rounds, relevance) -> float:
        """vd_forward_backward_dense_gen: the same step for the gen decoder, whose scores are the annotated rounds' option
        log-likelihoods.  batch carries option_in / option_out (a mode-2 batch); rounds and relevance as
        forward_backward_dense."""
        B, K = batch.c.B, self.params["numOptions"]
        rounds = np.ascontiguousarray(rounds, dtype=np.int32).reshape(-1)
        relevance = np.ascontiguousarray(relevance, dtype=np.float32)
        if rounds.shape != (B,) or relevance.shape != (B, K):
            raise ValueError("rounds must be (%d,) and relevance (%d, %d)" % (B, B, K))
        loss = C.c_float()
        self._enc_rows = None
        check(self.lib.vd_forward_backward_dense_gen(self.h, C.byref(batch.c), rounds.ctypes.data, relevance.ctypes.data,
                                                     C.byref(loss)))
        self._enc_rows = self._N(batch)
        return loss.value

    def retrieve(self, batch: Batch, use_gt: bool = True) -> np.ndarray:
        N = self._N(batch)
        out = np.empty((N,) if use_gt else (N, self.params["numOptions"]), dtype=np.int32)
        self._enc_rows = None
        check(self.lib.vd_retrieve(self.h, C.byref(batch.c), int(use_gt), out.ctypes.data))
        self._enc_rows = N
        return out

    # ---- Model:generateAnswers building blocks (model.lua:432-613) ---------------------------------------------
    def encoder_rnn_state(self, level: int, rows: int):
        """enc.rnnLayers[level+1].output[Tq] / .cell[Tq] as (rows,H) device tensors, or (None, None)."""
        hp, cp = C.c_void_p(), C.c_void_p()
        check(self.lib.vd_encoder_rnn_state(self.h, int(level), C.byref(hp), C.byref(cp)))
        H = self.params["rnnHiddenSize"]
        if not hp.value:
            return None, None
        return DeviceTensor(self, hp.value, (rows, H)), DeviceTensor(self, cp.value, (rows, H))

    def gen_decoder_step(self, tokens: np.ndarray, h_prev, c_prev):
        """One decoder step on len(tokens) rows.  h_prev / c_prev: two device pointers (int) or None each.
        Returns (log-probs (rows,V) numpy, [h1, h2] numpy, [c1, c2] numpy)."""
        tokens = np.ascontiguousarray(tokens, dtype=np.int32)
        rows = tokens.shape[0]
        arr = C.c_void_p * 2
        hp = arr(*[C.c_void_p(p) if p else C.c_void_p(None) for p in (h_prev or (None, None))])
        cp = arr(*[C.c_void_p(p) if p else C.c_void_p(None) for p in (c_prev or (None, None))])
        logp, ho, co = C.c_void_p(), arr(), arr()
        check(self.lib.vd_gen_decoder_step(self.h, rows, tokens.ctypes.data, hp, cp, C.byref(logp), ho, co))
        H, V = self.params["rnnHiddenSize"], self.params["vocabSize"]
        return (DeviceTensor(self, logp.value, (rows, V)).numpy(),
                [DeviceTensor(self, ho[i], (rows, H)).numpy() for i in range(2)],
                [DeviceTensor(self, co[i], (rows, H)).numpy() for i in range(2)])

    def gen_beam_search(self, k: int, L: int, start: int, end: int):
        """The whole beam search for every round of the last encoder forward on the device (vd_gen_beam_search).  Returns
        (answer (N, L) int32, length (N) int32 — 0 where no beam reached `end` — and score (N) float64)."""
        N = self._enc_rows
        if N is None:
            raise _lib.VdError(_lib.VD_E_STATE, "gen_beam_search before encoder_forward")
        ans = np.zeros((N, int(L)), dtype=np.int32)
        length = np.zeros(N, dtype=np.int32)
        score = np.zeros(N, dtype=np.float64)
        check(self.lib.vd_gen_beam_search(self.h, int(k), int(L), int(start), int(end), ans.ctypes.data, length.ctypes.data,
                                          score.ctypes.data))
        return ans, length, score

    def gen_diverse_beam_search(self, k: int, G: int, diversity: float, L: int, start: int, end: int):
        """Diverse beam search for every round of the last encoder forward (vd_gen_diverse_beam_search, DESIGN §22): k
        columns in G groups of k / G, Hamming diversity `diversity`.  Returns each group's best finished hypothesis as
        (answer (N, G, L) int32, length (N, G) int32 — 0 where the group finished none — and score (N, G) float64)."""
        N = self._enc_rows
        if N is None:
            raise _lib.VdError(_lib.VD_E_STATE, "gen_diverse_beam_search before encoder_forward")
        G = int(G)                         # buffers for G >= 1; the library refuses a G it cannot take
        ans = np.zeros((N, max(G, 1), int(L)), dtype=np.int32)
        length = np.zeros((N, max(G, 1)), dtype=np.int32)
        score = np.zeros((N, max(G, 1)), dtype=np.float64)
        check(self.lib.vd_gen_diverse_beam_search(self.h, int(k), G, float(diversity), int(L), int(start), int(end),
                                                  ans.ctypes.data, length.ctypes.data, score.ctypes.data))
        return ans, length, score

    def gen_nbest_beam_search(self, k: int, G: int, diversity: float, length_penalty: float, nbest: int, L: int, start: int,
                              end: int):
        """n-best lists of a (diverse) beam search for every round of the last encoder forward (vd_gen_nbest_beam_search,
        DESIGN §24): each group's `nbest` best finished hypotheses by norm = score / ((5 + l) / 6)^length_penalty, l = length
        - 1.  Returns (answer (N, G, nbest, L) int32, length (N, G, nbest) int32 — 0 for an entry never filled — score and
        norm (N, G, nbest) float64), each list best first."""
        N = self._enc_rows
        if N is None:
            raise _lib.VdError(_lib.VD_E_STATE, "gen_nbest_beam_search before encoder_forward")
        G, nb = int(G), int(nbest)         # buffers for G, nbest >= 1; the library refuses what it cannot take
        shape = (N, max(G, 1), max(nb, 1))
        ans = np.zeros(shape + (int(L),), dtype=np.int32)
        length = np.zeros(shape, dtype=np.int32)
        score = np.zeros(shape, dtype=np.float64)
        norm = np.zeros(shape, dtype=np.float64)
        check(self.lib.vd_gen_nbest_beam_search(self.h, int(k), G, float(diversity), float(length_penalty), nb, int(L),
                                                int(start), int(end), ans.ctypes.data, length.ctypes.data, score.ctypes.data,
                                                norm.ctypes.data))
        return ans, length, score, norm

    def gen_sample(self, L: int, start: int, temperature: float, seed: int, row_offset: int = 0):
        """Ancestral sampling for every round of the last encoder forward on the device (vd_gen_sample).  Returns (answer
        (N, L+1) int32 — column 0 = `start` — and logp (N, L) float32, each sample's un-tempered log-probability).  Row r's
        draws depend only on (seed, row_offset + r, step): pass the global index of the call's first round."""
        N = self._enc_rows
        if N is None:
            raise _lib.VdError(_lib.VD_E_STATE, "gen_sample before encoder_forward")
        ans = np.zeros((N, int(L) + 1), dtype=np.int32)
        logp = np.zeros((N, int(L)), dtype=np.float32)
        check(self.lib.vd_gen_sample(self.h, int(L), int(start), float(temperature), int(seed) & 0xFFFFFFFFFFFFFFFF,
                                     int(row_offset), ans.ctypes.data, logp.ctypes.data))
        return ans, logp

    def gen_truncated_sample(self, L: int, start: int, temperature: float, seed: int, row_offset: int = 0, top_k: int = 0,
                             top_p: float = 1.0):
        """gen_sample with top-k / top-p truncation (vd_gen_truncated_sample, DESIGN §23): each step draws from the first
        `top_k` classes by (logit desc, class asc) (0: all), then the shortest prefix of those holding `top_p` of their mass
        (1: all), with gen_sample's Philox draws.  Returns (answer (N, L+1), logp (N, L)) as gen_sample's."""
        N = self._enc_rows
        if N is None:
            raise _lib.VdError(_lib.VD_E_STATE, "gen_truncated_sample before encoder_forward")
        ans = np.zeros((N, int(L) + 1), dtype=np.int32)
        logp = np.zeros((N, int(L)), dtype=np.float32)
        check(self.lib.vd_gen_truncated_sample(self.h, int(L), int(start), float(temperature), int(seed) & 0xFFFFFFFFFFFFFFFF,
                                               int(row_offset), int(top_k), float(top_p), ans.ctypes.data, logp.ctypes.data))
        return ans, logp

    def gen_dialog_beam_search(self, batch: Batch, k: int, L: int, start: int, end: int, hist_width: int, max_ans_len: int):
        """Dialogs on the model's own answers with the beam search (vd_gen_dialog_beam_search): every round of `batch`,
        round r's encoder reading the answers generated for rounds < r.  Returns (answer (N, L), length (N), score (N),
        the history rows the encoder read (B, maxQuesCount, hist_width)), the first three as gen_beam_search's."""
        B, R = batch.c.B, self.params["maxQuesCount"]
        ans = np.zeros((B * R, int(L)), dtype=np.int32)
        length = np.zeros(B * R, dtype=np.int32)
        score = np.zeros(B * R, dtype=np.float64)
        hist = np.zeros((B, R, int(hist_width)), dtype=np.int32)
        self._enc_rows = None
        check(self.lib.vd_gen_dialog_beam_search(self.h, C.byref(batch.c), int(k), int(L), int(start), int(end),
                                                 int(hist_width), int(max_ans_len), ans.ctypes.data, length.ctypes.data,
                                                 score.ctypes.data, hist.ctypes.data))
        self._enc_rows = B * R
        return ans, length, score, hist

    def gen_dialog_diverse_beam_search(self, batch: Batch, k: int, G: int, diversity: float, L: int, start: int, end: int,
                                       hist_width: int, max_ans_len: int):
        """Dialogs on the model's own answers with diverse beam search (vd_gen_dialog_diverse_beam_search): round r's
        history takes each round's pick.  Returns (answer (N, G, L), length (N, G), score (N, G), history rows (B,
        maxQuesCount, hist_width))."""
        B, R, G = batch.c.B, self.params["maxQuesCount"], int(G)
        ans = np.zeros((B * R, max(G, 1), int(L)), dtype=np.int32)
        length = np.zeros((B * R, max(G, 1)), dtype=np.int32)
        score = np.zeros((B * R, max(G, 1)), dtype=np.float64)
        hist = np.zeros((B, R, int(hist_width)), dtype=np.int32)
        self._enc_rows = None
        check(self.lib.vd_gen_dialog_diverse_beam_search(self.h, C.byref(batch.c), int(k), G, float(diversity), int(L),
                                                         int(start), int(end), int(hist_width), int(max_ans_len),
                                                         ans.ctypes.data, length.ctypes.data, score.ctypes.data,
                                                         hist.ctypes.data))
        self._enc_rows = B * R
        return ans, length, score, hist

    def gen_dialog_nbest_beam_search(self, batch: Batch, k: int, G: int, diversity: float, length_penalty: float, nbest: int,
                                     L: int, start: int, end: int, hist_width: int, max_ans_len: int):
        """Dialogs on the model's own answers with n-best lists (vd_gen_dialog_nbest_beam_search): round r's history takes
        each round's pick.  Returns (answer (N, G, nbest, L), length, score, norm (N, G, nbest), history rows (B,
        maxQuesCount, hist_width))."""
        B, R, G, nb = batch.c.B, self.params["maxQuesCount"], int(G), int(nbest)
        shape = (B * R, max(G, 1), max(nb, 1))
        ans = np.zeros(shape + (int(L),), dtype=np.int32)
        length = np.zeros(shape, dtype=np.int32)
        score = np.zeros(shape, dtype=np.float64)
        norm = np.zeros(shape, dtype=np.float64)
        hist = np.zeros((B, R, int(hist_width)), dtype=np.int32)
        self._enc_rows = None
        check(self.lib.vd_gen_dialog_nbest_beam_search(self.h, C.byref(batch.c), int(k), G, float(diversity),
                                                       float(length_penalty), nb, int(L), int(start), int(end),
                                                       int(hist_width), int(max_ans_len), ans.ctypes.data, length.ctypes.data,
                                                       score.ctypes.data, norm.ctypes.data, hist.ctypes.data))
        self._enc_rows = B * R
        return ans, length, score, norm, hist

    def gen_dialog_sample(self, batch: Batch, L: int, start: int, end: int, temperature: float, seed: int, row_offset: int,
                          hist_width: int, max_ans_len: int):
        """Dialogs on the model's own answers with sampling (vd_gen_dialog_sample).  Returns (answer (N, L+1), logp (N, L),
        history rows (B, maxQuesCount, hist_width)); round r of dialog b draws as global round row_offset + b R + r."""
        B, R = batch.c.B, self.params["maxQuesCount"]
        ans = np.zeros((B * R, int(L) + 1), dtype=np.int32)
        logp = np.zeros((B * R, int(L)), dtype=np.float32)
        hist = np.zeros((B, R, int(hist_width)), dtype=np.int32)
        self._enc_rows = None
        check(self.lib.vd_gen_dialog_sample(self.h, C.byref(batch.c), int(L), int(start), int(end), float(temperature),
                                            int(seed) & 0xFFFFFFFFFFFFFFFF, int(row_offset), int(hist_width), int(max_ans_len),
                                            ans.ctypes.data, logp.ctypes.data, hist.ctypes.data))
        self._enc_rows = B * R
        return ans, logp, hist

    def gen_dialog_truncated_sample(self, batch: Batch, L: int, start: int, end: int, temperature: float, seed: int,
                                    row_offset: int, hist_width: int, max_ans_len: int, top_k: int = 0, top_p: float = 1.0):
        """gen_dialog_sample with gen_truncated_sample's draw (vd_gen_dialog_truncated_sample): (answer (N, L+1), logp (N, L),
        history rows (B, maxQuesCount, hist_width))."""
        B, R = batch.c.B, self.params["maxQuesCount"]
        ans = np.zeros((B * R, int(L) + 1), dtype=np.int32)
        logp = np.zeros((B * R, int(L)), dtype=np.float32)
        hist = np.zeros((B, R, int(hist_width)), dtype=np.int32)
        self._enc_rows = None
        check(self.lib.vd_gen_dialog_truncated_sample(self.h, C.byref(batch.c), int(L), int(start), int(end), float(temperature),
                                                      int(seed) & 0xFFFFFFFFFFFFFFFF, int(row_offset), int(top_k), float(top_p),
                                                      int(hist_width), int(max_ans_len), ans.ctypes.data, logp.ctypes.data,
                                                      hist.ctypes.data))
        self._enc_rows = B * R
        return ans, logp, hist

    def answer_pool_encode(self, tokens: np.ndarray):
        """Encode the split's answer pool (vd_answer_pool_encode): tokens (m, width) as opt_list stores them; replaces any
        earlier pool."""
        t = np.ascontiguousarray(tokens, dtype=np.int32)
        if t.ndim != 2:
            raise ValueError("answer pool tokens must be (m, width)")
        check(self.lib.vd_answer_pool_encode(self.h, t.ctypes.data, int(t.shape[0]), int(t.shape[1])))

    def answer_pool(self) -> DeviceTensor:
        """The pool embeddings (m, rnnHiddenSize) of the last encode (vd_answer_pool)."""
        p, m = C.c_void_p(), C.c_int64()
        check(self.lib.vd_answer_pool(self.h, C.byref(p), C.byref(m)))
        return DeviceTensor(self, p.value, (m.value, self.params["rnnHiddenSize"]))

    def answer_pool_retrieve(self, batch: Batch, k: int = 1):
        """The k best pool rows of every round of `batch` (vd_answer_pool_retrieve): (index (N, k) 0-based, score (N, k))."""
        N = batch.c.B * self.params["maxQuesCount"]
        index = np.zeros((N, int(k)), dtype=np.int32)
        score = np.zeros((N, int(k)), dtype=np.float32)
        self._enc_rows = None
        check(self.lib.vd_answer_pool_retrieve(self.h, C.byref(batch.c), int(k), index.ctypes.data, score.ctypes.data))
        self._enc_rows = N
        return index, score

    def answer_pool_dialog(self, batch: Batch, k: int, hist_width: int, max_ans_len: int):
        """Dialogs on the model's own retrieved answers (vd_answer_pool_dialog): (index (N, k), score (N, k), the history
        rows the encoder read (B, maxQuesCount, hist_width))."""
        B, R = batch.c.B, self.params["maxQuesCount"]
        index = np.zeros((B * R, int(k)), dtype=np.int32)
        score = np.zeros((B * R, int(k)), dtype=np.float32)
        hist = np.zeros((B, R, int(hist_width)), dtype=np.int32)
        self._enc_rows = None
        check(self.lib.vd_answer_pool_dialog(self.h, C.byref(batch.c), int(k), int(hist_width), int(max_ans_len),
                                             index.ctypes.data, score.ctypes.data, hist.ctypes.data))
        self._enc_rows = B * R
        return index, score, hist

    # ---- dialog sessions (DESIGN §19): one session per engine; begin and each ask end the last encoder forward
    def dialog_begin(self, batch: Batch, hist_width: int, max_ans_len: int):
        """Open a session on the B dialogs of `batch` (vd_dialog_begin): their image rows and round-0 history rows."""
        self._enc_rows = None
        check(self.lib.vd_dialog_begin(self.h, C.byref(batch.c), int(hist_width), int(max_ans_len)))

    def _questions(self, ques) -> np.ndarray:
        """the ask's (B, Tq) rows: the C side reads and writes as many rows as the open session has dialogs"""
        q = np.ascontiguousarray(ques, dtype=np.int32)
        if q.ndim != 2:
            raise ValueError("question rows must be (B, Tq)")
        B = self.dialog_round()[1]
        if q.shape[0] != B:
            raise ValueError("one question row per dialog: the session has %d dialogs, %d rows given" % (B, q.shape[0]))
        return q

    def dialog_ask_beam(self, ques, k: int, L: int, start: int, end: int):
        """Ask the next round (vd_dialog_ask_beam): ques (B, Tq) right-aligned rows.  Returns (answer (B, L), length (B),
        score (B)) as gen_beam_search's."""
        q = self._questions(ques)
        B = q.shape[0]
        ans = np.zeros((B, int(L)), dtype=np.int32)
        length = np.zeros(B, dtype=np.int32)
        score = np.zeros(B, dtype=np.float64)
        self._enc_rows = None
        check(self.lib.vd_dialog_ask_beam(self.h, q.ctypes.data, int(q.shape[1]), int(k), int(L), int(start), int(end),
                                          ans.ctypes.data, length.ctypes.data, score.ctypes.data))
        self._dialog_rows = B
        return ans, length, score

    def dialog_ask_sample(self, ques, L: int, start: int, end: int, temperature: float, seed: int, row_offset: int):
        """Ask the next round r with sampling (vd_dialog_ask_sample): (answer (B, L+1), logp (B, L)); row b draws as global
        round row_offset + b maxQuesCount + r."""
        q = self._questions(ques)
        B = q.shape[0]
        ans = np.zeros((B, int(L) + 1), dtype=np.int32)
        logp = np.zeros((B, int(L)), dtype=np.float32)
        self._enc_rows = None
        check(self.lib.vd_dialog_ask_sample(self.h, q.ctypes.data, int(q.shape[1]), int(L), int(start), int(end),
                                            float(temperature), int(seed) & 0xFFFFFFFFFFFFFFFF, int(row_offset),
                                            ans.ctypes.data, logp.ctypes.data))
        self._dialog_rows = B
        return ans, logp

    def dialog_ask_pool(self, ques, k: int = 1):
        """Ask the next round of a disc model (vd_dialog_ask_pool): (index (B, k) 0-based pool rows, score (B, k))."""
        q = self._questions(ques)
        B = q.shape[0]
        index = np.zeros((B, int(k)), dtype=np.int32)
        score = np.zeros((B, int(k)), dtype=np.float32)
        self._enc_rows = None
        check(self.lib.vd_dialog_ask_pool(self.h, q.ctypes.data, int(q.shape[1]), int(k), index.ctypes.data,
                                          score.ctypes.data))
        self._dialog_rows = B
        return index, score

    def dialog_round(self):
        """(next round to be asked, B) of the open session (vd_dialog_round)."""
        r, b = C.c_int32(), C.c_int32()
        check(self.lib.vd_dialog_round(self.h, C.byref(r), C.byref(b)))
        return r.value, b.value

    def dialog_history(self, hist_width: int) -> np.ndarray:
        """The session's history rows (B, maxQuesCount, hist_width) (vd_dialog_history)."""
        _, B = self.dialog_round()
        hist = np.zeros((B, self.params["maxQuesCount"], int(hist_width)), dtype=np.int32)
        check(self.lib.vd_dialog_history(self.h, hist.ctypes.data))
        return hist

    def dialog_encoding(self) -> DeviceTensor:
        """The last ask's encoder output (rows, rnnHiddenSize) on the device, in the ask's row order (vd_dialog_encoding)."""
        B = getattr(self, "_dialog_rows", 0)
        p = C.c_void_p()
        check(self.lib.vd_dialog_encoding(self.h, C.byref(p)))
        return DeviceTensor(self, p.value, (B, self.params["rnnHiddenSize"]))

    def dialog_rnn_state(self, level: int):
        """encoder_rnn_state for the last ask (vd_dialog_rnn_state): question-LSTM layer `level`'s (h, c) as (B, H) device
        tensors, or (None, None) for encoders without .rnnLayers."""
        B = getattr(self, "_dialog_rows", 0)
        hp, cp = C.c_void_p(), C.c_void_p()
        check(self.lib.vd_dialog_rnn_state(self.h, int(level), C.byref(hp), C.byref(cp)))
        if not hp.value:
            return None, None
        H = self.params["rnnHiddenSize"]
        return DeviceTensor(self, hp.value, (B, H)), DeviceTensor(self, cp.value, (B, H))

    def dialog_end(self):
        """Close the session (vd_dialog_end)."""
        check(self.lib.vd_dialog_end(self.h))

    # ---- dialog pools (DESIGN §20): conversations that join, are asked and leave on their own, each at its own round
    def dialog_open(self, capacity: int, Tq: int, hist_width: int, max_ans_len: int):
        """Open a pool of `capacity` free slots (vd_dialog_open); replaces any session."""
        self._dialog_rows = 0
        check(self.lib.vd_dialog_open(self.h, int(capacity), int(Tq), int(hist_width), int(max_ans_len)))

    def dialog_join(self, batch: Batch, draw_base=None) -> np.ndarray:
        """Join the batch's B dialogs (their image rows and round-0 history rows) into free slots (vd_dialog_join);
        draw_base (B) is each one's global round of round 0 for sampling (None: 0).  Returns the slot ids (B)."""
        B = int(batch.c.B)
        slots = np.zeros(B, dtype=np.int32)
        base = None
        if draw_base is not None:
            base = np.ascontiguousarray(draw_base, dtype=np.int64)
            if base.shape != (B,):
                raise ValueError("one draw base per joined dialog")
        self._enc_rows = None
        check(self.lib.vd_dialog_join(self.h, C.byref(batch.c), base.ctypes.data if base is not None else None,
                                      slots.ctypes.data))
        return slots

    def dialog_join_rounds(self, batch: Batch, rounds, answers, slots, draw_base=None):
        """Resume the batch's B dialogs in the free slots `slots` (B) at `rounds` (B) (vd_dialog_join_rounds, DESIGN §21):
        their questions 0..r-1 are the batch's ques_fwd rows, their answers `answers` (B, maxQuesCount, Ta) left-aligned
        word ids (None for the encoders without history); draw_base as dialog_join's."""
        B, R = int(batch.c.B), self.params["maxQuesCount"]
        r = np.ascontiguousarray(rounds, dtype=np.int32).ravel()
        s = np.ascontiguousarray(slots, dtype=np.int32).ravel()
        if r.shape != (B,) or s.shape != (B,):
            raise ValueError("one round and one slot per joined dialog")
        a, Ta = None, 1
        if answers is not None:
            a = np.ascontiguousarray(answers, dtype=np.int32)
            if a.ndim != 3 or a.shape[:2] != (B, R):
                raise ValueError("answers must be (B, maxQuesCount, Ta)")
            Ta = a.shape[2]
        base = None
        if draw_base is not None:
            base = np.ascontiguousarray(draw_base, dtype=np.int64)
            if base.shape != (B,):
                raise ValueError("one draw base per joined dialog")
        self._enc_rows = None
        check(self.lib.vd_dialog_join_rounds(self.h, C.byref(batch.c), r.ctypes.data, a.ctypes.data if a is not None else None,
                                             int(Ta), base.ctypes.data if base is not None else None, s.ctypes.data))

    def dialog_leave(self, slots):
        """Free the slots (vd_dialog_leave)."""
        s = np.ascontiguousarray(slots, dtype=np.int32).ravel()
        check(self.lib.vd_dialog_leave(self.h, s.ctypes.data, int(s.size)))

    @staticmethod
    def _slot_rows(slots, ques):
        s = np.ascontiguousarray(slots, dtype=np.int32).ravel()
        q = np.ascontiguousarray(ques, dtype=np.int32)
        if q.ndim != 2 or q.shape[0] != s.size:
            raise ValueError("one question row per asked slot: %d slots, question rows of shape %s" % (s.size, q.shape))
        return s, q

    def dialog_ask_beam_slots(self, slots, ques, k: int, L: int, start: int, end: int):
        """Ask slots (n) one question each (vd_dialog_ask_beam_slots), each at its own round: (answer (n, L), length (n),
        score (n)) in row order."""
        s, q = self._slot_rows(slots, ques)
        n = s.size
        ans = np.zeros((n, int(L)), dtype=np.int32)
        length = np.zeros(n, dtype=np.int32)
        score = np.zeros(n, dtype=np.float64)
        self._enc_rows = None
        check(self.lib.vd_dialog_ask_beam_slots(self.h, s.ctypes.data, n, q.ctypes.data, int(q.shape[1]), int(k), int(L),
                                                int(start), int(end), ans.ctypes.data, length.ctypes.data, score.ctypes.data))
        self._dialog_rows = n
        return ans, length, score

    def dialog_ask_diverse_slots(self, slots, ques, k: int, G: int, diversity: float, L: int, start: int, end: int):
        """Ask slots (n) one question each with diverse beam search (vd_dialog_ask_diverse_slots): (answer (n, G, L),
        length (n, G), score (n, G)) in row order; each slot's history takes its row's pick."""
        s, q = self._slot_rows(slots, ques)
        n, G = s.size, int(G)
        ans = np.zeros((n, max(G, 1), int(L)), dtype=np.int32)
        length = np.zeros((n, max(G, 1)), dtype=np.int32)
        score = np.zeros((n, max(G, 1)), dtype=np.float64)
        self._enc_rows = None
        check(self.lib.vd_dialog_ask_diverse_slots(self.h, s.ctypes.data, n, q.ctypes.data, int(q.shape[1]), int(k), G,
                                                   float(diversity), int(L), int(start), int(end), ans.ctypes.data,
                                                   length.ctypes.data, score.ctypes.data))
        self._dialog_rows = n
        return ans, length, score

    def dialog_ask_nbest_slots(self, slots, ques, k: int, G: int, diversity: float, length_penalty: float, nbest: int, L: int,
                               start: int, end: int):
        """Ask slots (n) one question each with n-best lists (vd_dialog_ask_nbest_slots): (answer (n, G, nbest, L), length,
        score, norm (n, G, nbest)) in row order; each slot's history takes its row's pick."""
        s, q = self._slot_rows(slots, ques)
        n, G, nb = s.size, int(G), int(nbest)
        shape = (n, max(G, 1), max(nb, 1))
        ans = np.zeros(shape + (int(L),), dtype=np.int32)
        length = np.zeros(shape, dtype=np.int32)
        score = np.zeros(shape, dtype=np.float64)
        norm = np.zeros(shape, dtype=np.float64)
        self._enc_rows = None
        check(self.lib.vd_dialog_ask_nbest_slots(self.h, s.ctypes.data, n, q.ctypes.data, int(q.shape[1]), int(k), G,
                                                 float(diversity), float(length_penalty), nb, int(L), int(start), int(end),
                                                 ans.ctypes.data, length.ctypes.data, score.ctypes.data, norm.ctypes.data))
        self._dialog_rows = n
        return ans, length, score, norm

    def dialog_ask_sample_slots(self, slots, ques, L: int, start: int, end: int, temperature: float, seed: int,
                                row_offset: int = 0):
        """vd_dialog_ask_sample_slots: (answer (n, L+1), logp (n, L)); row i draws as global round row_offset +
        draw_base[slot] + the slot's round."""
        s, q = self._slot_rows(slots, ques)
        n = s.size
        ans = np.zeros((n, int(L) + 1), dtype=np.int32)
        logp = np.zeros((n, int(L)), dtype=np.float32)
        self._enc_rows = None
        check(self.lib.vd_dialog_ask_sample_slots(self.h, s.ctypes.data, n, q.ctypes.data, int(q.shape[1]), int(L), int(start),
                                                  int(end), float(temperature), int(seed) & 0xFFFFFFFFFFFFFFFF, int(row_offset),
                                                  ans.ctypes.data, logp.ctypes.data))
        self._dialog_rows = n
        return ans, logp

    def dialog_ask_truncated_slots(self, slots, ques, L: int, start: int, end: int, temperature: float, seed: int,
                                   row_offset: int = 0, top_k: int = 0, top_p: float = 1.0):
        """dialog_ask_sample_slots with gen_truncated_sample's draw (vd_dialog_ask_truncated_slots): (answer (n, L+1),
        logp (n, L)) in row order."""
        s, q = self._slot_rows(slots, ques)
        n = s.size
        ans = np.zeros((n, int(L) + 1), dtype=np.int32)
        logp = np.zeros((n, int(L)), dtype=np.float32)
        self._enc_rows = None
        check(self.lib.vd_dialog_ask_truncated_slots(self.h, s.ctypes.data, n, q.ctypes.data, int(q.shape[1]), int(L),
                                                     int(start), int(end), float(temperature), int(seed) & 0xFFFFFFFFFFFFFFFF,
                                                     int(row_offset), int(top_k), float(top_p), ans.ctypes.data,
                                                     logp.ctypes.data))
        self._dialog_rows = n
        return ans, logp

    def dialog_ask_pool_slots(self, slots, ques, k: int = 1):
        """vd_dialog_ask_pool_slots: (index (n, k) 0-based pool rows, score (n, k))."""
        s, q = self._slot_rows(slots, ques)
        n = s.size
        index = np.zeros((n, int(k)), dtype=np.int32)
        score = np.zeros((n, int(k)), dtype=np.float32)
        self._enc_rows = None
        check(self.lib.vd_dialog_ask_pool_slots(self.h, s.ctypes.data, n, q.ctypes.data, int(q.shape[1]), int(k),
                                                index.ctypes.data, score.ctypes.data))
        self._dialog_rows = n
        return index, score

    def dialog_slots(self) -> np.ndarray:
        """Each slot's next round, -1 when free (vd_dialog_slots); its length is the capacity."""
        cap = C.c_int32()
        check(self.lib.vd_dialog_slots(self.h, None, C.byref(cap)))
        rounds = np.zeros(cap.value, dtype=np.int32)
        check(self.lib.vd_dialog_slots(self.h, rounds.ctypes.data, C.byref(cap)))
        return rounds

    def dialog_slot_history(self, slots, hist_width: int) -> np.ndarray:
        """The history rows (n, maxQuesCount, hist_width) of the slots (vd_dialog_slot_history)."""
        s = np.ascontiguousarray(slots, dtype=np.int32).ravel()
        hist = np.zeros((s.size, self.params["maxQuesCount"], int(hist_width)), dtype=np.int32)
        check(self.lib.vd_dialog_slot_history(self.h, s.ctypes.data, int(s.size), hist.ctypes.data))
        return hist

    def upload(self, dev_ptr: int, a: np.ndarray):
        a = np.ascontiguousarray(a, dtype=np.float32)
        check(self.lib.vd_memcpy_h2d(self.h, C.c_void_p(dev_ptr), a.ctypes.data, a.nbytes))

    def device_alloc(self, nbytes: int) -> int:
        p = C.c_void_p()
        check(self.lib.vd_device_alloc(self.h, C.byref(p), int(nbytes)))
        return p.value

    def device_free(self, dev_ptr: int):
        check(self.lib.vd_device_free(self.h, C.c_void_p(dev_ptr)))

    def clamp_adam_step(self, lr: float):
        check(self.lib.vd_clamp_adam_step(self.h, float(lr)))

    # ---- comm --------------------------------------------------------------------------------------
    def comm_unique_id(self) -> bytes:
        buf = C.create_string_buffer(_lib.VD_COMM_ID_BYTES)
        check(self.lib.vd_comm_unique_id(buf))
        return buf.raw

    def comm_init(self, uid: bytes, rank: int, world: int):
        buf = C.create_string_buffer(uid, _lib.VD_COMM_ID_BYTES)
        check(self.lib.vd_comm_init(self.h, buf, rank, world))

    # ---- plumbing ------------------------------------------------------------------------------------
    def synchronize(self):
        check(self.lib.vd_synchronize(self.h))

    def timer_start(self):
        check(self.lib.vd_timer_start(self.h))

    def timer_stop(self) -> float:
        ms = C.c_float()
        check(self.lib.vd_timer_stop(self.h, C.byref(ms)))
        return ms.value

    def profile(self, on: bool):
        check(self.lib.vd_profile_enable(self.h, int(on)))

    def profile_reset(self):
        check(self.lib.vd_profile_reset(self.h))

    def launch_count(self) -> int:
        n = C.c_int64()
        check(self.lib.vd_launch_count(self.h, C.byref(n)))
        return n.value

    def kernel_stats(self, name: str) -> dict:
        n, ms, fl, by = C.c_int64(), C.c_double(), C.c_double(), C.c_double()
        check(self.lib.vd_kernel_stats(self.h, name.encode(), C.byref(n), C.byref(ms), C.byref(fl), C.byref(by)))
        return {"launches": n.value, "ms": ms.value, "flops": fl.value, "bytes": by.value}

    def profiler_range(self, start: bool):
        check(self.lib.vd_profiler_range(self.h, int(start)))

    def flush_l2(self):
        check(self.lib.vd_flush_l2(self.h))


def pinned_empty(shape, dtype) -> np.ndarray:
    """numpy array over cudaHostAlloc'ed memory (async H2D needs pinned buffers)."""
    lib = _lib.load()
    dt = np.dtype(dtype)
    n = int(np.prod(shape)) * dt.itemsize
    p = C.c_void_p()
    check(lib.vd_host_alloc(C.byref(p), n))
    buf = (C.c_char * max(n, 1)).from_address(p.value)
    arr = np.frombuffer(buf, dtype=dt, count=int(np.prod(shape))).reshape(shape)
    return arr
