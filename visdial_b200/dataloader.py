"""Mirror of the reference `dataloader` (/root/reference/dataloader.lua) over an HBM-resident corpus.

Same method names and argument meaning as the Lua module; the tensors live on the device:
  initialize(opt, subsets)    :10-137   raw datasets -> HBM, prepareDataset on the device (vd_corpus_create)
  getTrainBatch(params, B)    :324-341  random dialog indices (host RNG, like torch.LongTensor:random), gather on device
  getTestBatch(startId, ...)  :344-375  consecutive dialogs; returns (batch, nextStartId)
  getIndexData/getIndexOption :378-478  folded into ONE C call (vd_corpus_get_batch): two kernel launches per batch
The HDF5 / JSON reads of initialize (:13-129) stay with the caller: `data[dtype]` holds the numpy arrays of one split
under the h5 dataset names without the `_<dtype>` suffix (visdial_b200.synthetic.make_corpus builds such a dict).

There is no CPU path: without libvisdial_b200.so and a GPU every call raises.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional

import numpy as np

from ._lib import check, vd_batch, vd_corpus_desc
from .engine import Batch, Engine

_I32_KEYS = ("ques", "ques_length", "ans", "ans_length", "cap", "cap_length", "opt", "opt_list", "opt_length",
             "ans_index", "img_pos", "num_rounds")


class DeviceBatch(Batch):
    """A batch table whose tensors are device buffers owned by the corpus (vd_batch.on_device = 1).  `batch[key]` reads
    the tensor back to the host (tests, display); the engine consumes the device pointers directly.

    LIFETIME: the corpus assembles batches into a two-slot ring of device buffers (csrc/corpus.cu), so a DeviceBatch is valid until the
    SECOND later `getTrainBatch` / `getTestBatch` call on the same dataloader — enough to prepare batch i+1 while the engine consumes batch i.
    Keep a host copy (`batch[key]`) of anything needed longer."""

    _SHAPES = {
        "ques_fwd": lambda b, R, K: (b.B, R, b.Tq), "hist": lambda b, R, K: (b.B, R, b.Th),
        "answer_in": lambda b, R, K: (b.B, R, b.Ta), "answer_out": lambda b, R, K: (b.B, R, b.Ta),
        "answer_ind": lambda b, R, K: (b.B, R), "options": lambda b, R, K: (b.B * R, K, b.To),
        "option_in": lambda b, R, K: (b.B, R, K, b.To), "option_out": lambda b, R, K: (b.B, R, K, b.To),
    }

    def __init__(self, eng: Engine, c: vd_batch, R: int, K: int, img_shape, num_answer_tokens: int,
                 num_rounds: Optional[np.ndarray], h2d_bytes: int):
        self.eng, self.c, self.R, self.K, self.img_shape = eng, c, R, K, img_shape
        self.arrays = {}
        self.num_answer_tokens = num_answer_tokens          # == (answer_out > 0).sum(), from the host length table
        self.num_rounds = num_rounds
        self.h2d_bytes = h2d_bytes

    def keys(self):
        ks = [k for k in self._SHAPES if getattr(self.c, k)]
        return ks + (["img_feat"] if self.c.img_feat else [])

    def __contains__(self, k):
        return k in self.keys() or (k == "num_rounds" and self.num_rounds is not None)

    def __getitem__(self, k):
        if k == "num_rounds":
            return self.num_rounds
        ptr = getattr(self.c, k)
        if not ptr:
            raise KeyError(k)
        if k == "img_feat":
            out = np.empty((self.c.B,) + tuple(self.img_shape), dtype=np.float32)
        else:
            out = np.empty(self._SHAPES[k](self.c, self.R, self.K), dtype=np.int32)
            if k == "answer_ind" and self.c.options:      # disc batches carry the flattened view (dataloader.lua:334-336)
                out = out.reshape(-1)
        check(self.eng.lib.vd_memcpy_d2h(self.eng.h, out.ctypes.data, ptr, out.nbytes))
        return out

    def numpy(self) -> Dict[str, np.ndarray]:
        return {k: self[k] for k in self.keys()}

    def to_device(self, eng):
        return self


class Corpus:
    """One split resident in HBM (vd_corpus handle)."""

    def __init__(self, eng: Engine, raw: Dict[str, np.ndarray], opt: dict, start: int, end: int):
        self.eng = eng
        self.raw = {}
        for k in _I32_KEYS:
            if raw.get(k) is not None:
                self.raw[k] = np.ascontiguousarray(raw[k], dtype=np.int32)
        if raw.get("images") is not None:
            self.raw["images"] = np.ascontiguousarray(raw["images"], dtype=np.float32)
        r = self.raw
        d = vd_corpus_desc()
        d.numThreads, d.numRounds, d.maxQuesLen = r["ques"].shape
        d.maxAnsLen = r["ans"].shape[2]
        d.maxCapLen = r["cap"].shape[1] if "cap" in r else 0
        d.numOptions = r["opt"].shape[2]
        d.numOptList = r["opt_list"].shape[0]
        d.useHistory = int(bool(opt.get("useHistory")))
        d.concatHistory = int(bool(opt.get("concatHistory")))
        d.useIm = int(bool(opt.get("useIm")))
        d.maxHistoryLen = int(opt.get("maxHistoryLen") or 60)                       # dataloader.lua:142
        d.imgNorm = int(opt.get("imgNorm", 1))          # opts.lua:15 default 1; opts.lua:66 (derive_flags) sets 0 for 'att' encoders
        att = "att" in opt.get("encoder", "")                                       # :70
        d.imgAtt = int(att)
        if d.useIm:
            im = r["images"]
            d.numImages, d.imgChannels = im.shape[0], im.shape[1]
            d.imgSpatial = im.shape[2] if att else 0
        d.startToken, d.endToken = start, end
        for field, key in (("ques", "ques"), ("ques_len", "ques_length"), ("ans", "ans"), ("ans_len", "ans_length"),
                           ("cap", "cap"), ("cap_len", "cap_length"), ("opt", "opt"), ("opt_list", "opt_list"),
                           ("opt_len", "opt_length"), ("ans_index", "ans_index"), ("img_pos", "img_pos"),
                           ("num_rounds", "num_rounds"), ("images", "images")):
            a = r.get(key)
            if a is not None and (d.useHistory or key not in ("cap", "cap_length")) \
                    and (d.useIm or key not in ("img_pos", "images")):
                setattr(d, field, a.ctypes.data)
        self.desc = d
        h = C.c_void_p()
        check(eng.lib.vd_corpus_create(eng.h, C.byref(d), C.byref(h)))
        self.h = h
        self.numThreads = int(d.numThreads)
        self.R, self.K = int(d.numRounds), int(d.numOptions)
        self.ans_len1 = r["ans_length"].astype(np.int64) + 1                        # :196
        self.num_rounds = r.get("num_rounds")
        if d.useIm:
            im = r["images"]
            self.img_shape = (im.shape[2], im.shape[3], im.shape[1]) if att else (im.shape[1],)
        else:
            self.img_shape = None
        # the host copies of the big arrays are not needed after the upload
        for k in ("ques", "ans", "cap", "opt", "opt_list", "images"):
            self.raw.pop(k, None)

    def get_batch(self, inds0: np.ndarray, decoder_gen: int, with_num_rounds: bool = False) -> DeviceBatch:
        inds0 = np.ascontiguousarray(inds0, dtype=np.int64)
        b = vd_batch()
        check(self.eng.lib.vd_corpus_get_batch(self.h, inds0.ctypes.data, len(inds0), decoder_gen, C.byref(b)))
        nr = self.num_rounds[inds0].astype(np.int64) if (with_num_rounds and self.num_rounds is not None) else None
        return DeviceBatch(self.eng, b, self.R, self.K, self.img_shape, int(self.ans_len1[inds0].sum()), nr,
                           h2d_bytes=4 * len(inds0))

    def read(self, name: str) -> np.ndarray:
        n = C.c_int64()
        check(self.eng.lib.vd_corpus_read(self.h, name.encode(), None, C.byref(n)))
        out = np.empty(n.value, dtype=np.float32 if name == "img_fv" else np.int32)
        check(self.eng.lib.vd_corpus_read(self.h, name.encode(), out.ctypes.data, C.byref(n)))
        return out

    def batch_bytes(self):
        by, ln = C.c_int64(), C.c_int32()
        check(self.eng.lib.vd_corpus_batch_bytes(self.h, C.byref(by), C.byref(ln)))
        return by.value, ln.value

    def close(self):
        if getattr(self, "h", None):
            self.eng.lib.vd_corpus_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def eval_partition(n: int, rank: int, world: int):
    """Contiguous share [lo, hi) of an n-dialog evaluation split for `rank` (never splits a dialog)."""
    from .dist import shard_range
    return shard_range(n, rank, world)


def test_batch_indices(startId: int, batchSize: int, lo: int, hi: int):
    """getTestBatch's index range (dataloader.lua:347-357) inside a rank's partition [lo, hi): `startId` counts from the
    partition's first dialog (0-based); returns (global 0-based dialog indices, nextStartId)."""
    nxt = min(hi - lo, startId + batchSize)
    return lo + np.arange(startId, nxt), nxt


test_batch_indices.__test__ = False          # not a pytest test


class Dataloader:
    """`dataloader` table of the reference (dataloader.lua:5-8) bound to one engine."""

    def __init__(self, eng: Engine, seed: int = 1234, rank: int = 0, world: int = 1):
        """`rank` / `world`: data-parallel use (one process per GPU, SURVEY §8e).  Every rank holds the whole corpus;
        training batches are drawn independently per rank (seed + rank: the global batch is world x batchSize dialogs
        sampled with replacement, as the reference samples one batch, :326); evaluation splits are partitioned into
        `world` contiguous dialog ranges, so that a rank-ordered gather of the per-rank results
        (visdial_b200.dist.gather_ranks) is the unsharded order.  No collective touches the data path."""
        self.eng = eng
        self.rank, self.world = int(rank), int(world)
        self.rng = np.random.default_rng(seed + 7919 * self.rank)
        self.numThreads: Dict[str, int] = {}
        self.part: Dict[str, tuple] = {}             # dtype -> (first dialog, one past the last) of this rank
        self.corpus: Dict[str, Corpus] = {}

    def initialize(self, opt: dict, subsets, data: Dict[str, Dict[str, np.ndarray]], vocab_size_no_specials: int = None):
        """dataloader:initialize(opt, subsets), dataloader.lua:10-137.  `opt` carries encoder / useHistory /
        concatHistory / useIm / maxHistoryLen / imgNorm as opts.lua:55-59 derives them; `vocabSize` already counts
        <START>, <END> (:17-22) unless `vocab_size_no_specials` gives len(word2ind) of the json."""
        if vocab_size_no_specials is not None:
            self.vocabSize = vocab_size_no_specials + 2                             # :17-22
        else:
            self.vocabSize = int(opt["vocabSize"])
        w2i = dict(getattr(self, "word2ind", None) or {})                           # the json's words, when read from files
        w2i["<START>"], w2i["<END>"] = self.vocabSize - 1, self.vocabSize           # :17-22
        self.word2ind = w2i
        self.ind2word = {v: k for k, v in w2i.items()}                              # :24-29
        self.useHistory, self.concatHistory, self.useIm = bool(opt.get("useHistory")), bool(opt.get("concatHistory")), bool(opt.get("useIm"))
        self.maxHistoryLen = int(opt.get("maxHistoryLen") or 60)                    # :142
        for dtype in subsets:
            c = Corpus(self.eng, data[dtype], opt, self.word2ind["<START>"], self.word2ind["<END>"])
            self.corpus[dtype] = c
            self.part[dtype] = eval_partition(c.numThreads, self.rank, self.world) if dtype != "train" else (0, c.numThreads)
            self.numThreads[dtype] = self.part[dtype][1] - self.part[dtype][0]      # :94-105 (this rank's share)
            if c.num_rounds is not None:                                            # :110, read by Model.retrieve / predict
                setattr(self, dtype + "_num_rounds", c.num_rounds)
            self.maxQuesCount = c.R                                                 # :122
            self.numOptions = c.K                                                   # :112
            self.maxQuesLen = int(c.desc.maxQuesLen)                                # :124
            self.maxAnsLen = int(c.desc.maxAnsLen)                                  # :126
        if "train" in self.corpus:
            self.numTrainThreads = self.numThreads["train"]
        if "val" in self.corpus:
            self.numValThreads = self.numThreads["val"]
        if "test" in self.corpus:
            self.numTestThreads = self.numThreads["test"]
        if self.concatHistory:
            self.maxHistoryLen = min(self.maxQuesCount * (self.maxQuesLen + self.maxAnsLen), 300)   # :217
        return self

    def initialize_from_files(self, opt: dict, subsets):
        """The file-reading half of dataloader:initialize (dataloader.lua:13-129): `opt.inputJson` (word2ind ...),
        `opt.inputQues` (visdial_data.h5) and, when the encoder uses the image, `opt.inputImg` (data_img.h5), read with
        visdial_b200.h5lite (no h5py / libhdf5 in this image; DESIGN.md §13 for what that reader covers)."""
        import json
        from . import h5lite
        info = json.load(open(opt["inputJson"]))                                    # :13-15
        for k, v in info.items():
            setattr(self, k, v)
        n_words = len(info["word2ind"])                                             # :17-22
        ques = h5lite.read(opt["inputQues"])                                        # :33-34 (memory-mapped)
        data = {}
        for dtype in subsets:
            d = h5lite.split(ques, dtype)                                           # :45-57,108-129
            if not d:
                raise ValueError("no '%s' datasets in %s" % (dtype, opt["inputQues"]))
            if opt.get("useIm"):                                                    # :36-37,61: only the asked splits
                try:
                    d["images"] = h5lite.read(opt["inputImg"], ["images_" + dtype])["images_" + dtype]
                except h5lite.H5Error as e:
                    raise ValueError("no 'images_%s' in %s (%s)" % (dtype, opt["inputImg"], e))
            data[dtype] = d
        return self.initialize(dict(opt, vocabSize=n_words + 2), subsets, data, vocab_size_no_specials=n_words)

    def restrict(self, dtype: str, n: int):
        """Keep the first `n` dialogs of evaluation split `dtype` and re-partition that prefix over the ranks (generate.lua's
        maxThreads on several GPUs).  Dialog indices stay global, so rank r's share of the prefix is the dialogs a 1-GPU run
        generates at those positions, with the same sampling row offsets."""
        lo, hi = eval_partition(min(int(n), self.corpus[dtype].numThreads), self.rank, self.world)
        self.part[dtype] = (lo, hi)
        self.numThreads[dtype] = hi - lo
        if dtype in ("val", "test"):
            setattr(self, "num%sThreads" % dtype.capitalize(), hi - lo)
        return self

    def getTrainBatch(self, params: dict, batchSize: int = None) -> DeviceBatch:
        size = int(batchSize or params["batchSize"])                                # :325
        inds = self.rng.integers(0, self.numThreads["train"], size=size)            # :326 (uniform with replacement)
        return self.corpus["train"].get_batch(inds, 0 if params["decoder"] == "disc" else 1)   # :329-337

    def getIndexData(self, inds0, params: dict, dtype: str) -> DeviceBatch:
        """dataloader.getIndexData (dataloader.lua:378-433) for explicit dialog indices (0-based, within this rank's
        share of the split): the call Model:generateAnswers makes per dialog (model.lua:464)."""
        inds = self.part[dtype][0] + np.asarray(inds0, dtype=np.int64).reshape(-1)
        return self.corpus[dtype].get_batch(inds, 1)

    def getTestBatch(self, startId: int, params: dict, dtype: str = "val"):
        """`startId` is 0-based here (Lua's startId - 1); returns (batch, nextStartId) like :344-375."""
        inds, nxt = test_batch_indices(startId, int(params["batchSize"]), *self.part[dtype])   # :347-357
        mode = 0 if params["decoder"] == "disc" else 2                              # :362-371
        return self.corpus[dtype].get_batch(inds, mode, with_num_rounds=True), nxt

    def close(self):
        for c in self.corpus.values():
            c.close()
        self.corpus = {}
