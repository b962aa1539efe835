"""Shared test helpers: small configs, batches, oracle <-> engine parameter plumbing, device buffers with guard bands."""
import ctypes as C

import numpy as np
import torch

from visdial_b200 import engine as E
from visdial_b200._lib import check
from visdial_b200.synthetic import make_batch

CONFIGS = [("lf-ques", "gen"), ("lf-ques-im-hist", "disc"), ("hrea-ques-im-hist", "gen"),
           ("mn-att-ques-im-hist", "disc"), ("lf-ques", "disc"), ("mn-att-ques-im-hist", "gen"),
           ("hrea-ques-im-hist", "disc"), ("lf-ques-im-hist", "gen"),
           # the seven sub-graph encoders of encoders/*.lua (each once with either decoder; the ones that export
           # rnnLayers to decoderConnect also with gen)
           ("lf-ques-im", "disc"), ("lf-ques-im", "gen"), ("lf-ques-hist", "gen"), ("hre-ques-hist", "disc"),
           ("hre-ques-hist", "gen"), ("hre-ques-im-hist", "gen"), ("mn-ques-hist", "gen"), ("mn-ques-im-hist", "disc"),
           ("lf-att-ques-im-hist", "disc"), ("lf-att-ques-im-hist", "gen")]
ALL_ENCODERS = ("lf-ques", "lf-ques-im", "lf-ques-hist", "lf-ques-im-hist", "lf-att-ques-im-hist", "hre-ques-hist",
                "hre-ques-im-hist", "hrea-ques-im-hist", "mn-ques-hist", "mn-ques-im-hist", "mn-att-ques-im-hist")


def small_params(encoder, decoder, **kw):
    p = dict(E.DEFAULT_PARAMS)
    p.update(encoder=encoder, decoder=decoder, vocabSize=40, embedSize=12, rnnHiddenSize=32, numLayers=2,
             imgFeatureSize=8 if "att" in encoder else 24, imgSpatialSize=3, imgEmbedSize=8,
             commonEmbeddingSize=16, numAttentionLayers=1, maxQuesCount=10, numOptions=7, dropout=0.5, gpuid=0)
    p.update(kw)
    return E.derive_flags(p)


def full_params(encoder, decoder, **kw):
    p = dict(E.DEFAULT_PARAMS)
    p.update(encoder=encoder, decoder=decoder, vocabSize=10000,
             imgFeatureSize=512 if "att" in encoder else 4096)
    p.update(kw)
    return E.derive_flags(p)


def small_batch(params, B=3, seed=7, gen_eval=False):
    return make_batch(params, B, seed=seed, max_ques_len=6, max_ans_len=5, max_cap_len=8, max_hist_len=9,
                      max_hist_concat=30, gen_eval=gen_eval, empty_round_every=2)


def torch_batch(batch):
    out = {}
    for k, v in batch.items():
        t = torch.from_numpy(np.ascontiguousarray(v))
        out[k] = t.long() if v.dtype.kind in "iu" else t
    return out


def torch_params(params, flat, dtype=torch.float32):
    return {k: torch.from_numpy(np.array(v)).to(dtype) for k, v in E.split_parameters(params, flat).items()}


def flat_from_named(params, named):
    segs, n = E.layout(params)
    flat = np.zeros(n, dtype=np.float32)
    for s in segs:
        flat[s.offset:s.offset + s.size] = np.asarray(named[s.name].detach().cpu().numpy(), dtype=np.float32).reshape(-1)
    return flat


def seg_slices(params):
    segs, _ = E.layout(params)
    return {s.name: slice(s.offset, s.offset + s.size) for s in segs}


class Buf:
    """One device allocation holding a host image (any numpy dtype); ptr(off) = address of element `off`."""

    def __init__(self, eng, img):
        self.eng, self.img = eng, np.ascontiguousarray(img)
        p = C.c_void_p()
        check(eng.lib.vd_device_alloc(eng.h, C.byref(p), self.img.nbytes))
        self.p = p
        check(eng.lib.vd_memcpy_h2d(eng.h, p, self.img.ctypes.data, self.img.nbytes))

    def ptr(self, off=0):
        return C.c_void_p(self.p.value + self.img.itemsize * off)

    def get(self):
        out = np.empty_like(self.img)
        check(self.eng.lib.vd_memcpy_d2h(self.eng.h, out.ctypes.data, self.p, out.nbytes))
        return out

    def free(self):
        check(self.eng.lib.vd_device_free(self.eng.h, self.p))


def call(eng, name, ptrs, ints=(), reals=()):
    """vd_test_kernel by name; ptrs are device buffers (anything with .ptr()), ctypes pointers or None.  Returns the code."""
    P = (C.c_void_p * max(1, len(ptrs)))(*[None if p is None else (p.ptr().value if hasattr(p, "ptr") else p.value)
                                           for p in ptrs])
    I = (C.c_int64 * max(1, len(ints)))(*[int(i) for i in ints])
    X = (C.c_double * max(1, len(reals)))(*[float(x) for x in reals])
    return eng.lib.vd_test_kernel(eng.h, name.encode(), P, len(ptrs), I, len(ints), X, len(reals))


def run(eng, name, ptrs, ints=(), reals=()):
    check(call(eng, name, ptrs, ints, reals))


def within(got, ref, bound, what):
    """|got - ref| <= bound elementwise (bound broadcasts), got finite; names the worst element otherwise"""
    got = np.asarray(got)
    ref = np.broadcast_to(np.asarray(ref, np.float64), got.shape)
    assert np.isfinite(got).all(), (what, "non-finite output: a NaN-poisoned element was read, or an overflow")
    err = np.abs(got.astype(np.float64) - ref)
    bad = err > bound
    if bad.any():
        i = np.unravel_index(np.argmax(err - bound), err.shape)
        raise AssertionError("%s: %d elements out of bound, worst at %s: got %r ref %r bound %r"
                             % (what, int(bad.sum()), i, got[i], ref[i], np.broadcast_to(bound, err.shape)[i]))


G = 64                       # guard elements on each side of every buffer (256 bytes keeps float4 alignment)
ISENT = -123456789           # int32 guard sentinel of outputs


class Dev:
    """A device copy of array x between guard bands.  Float buffers use NaN guards, int32 inputs 0 (a stray id read stays
    in bounds), int32 outputs the sentinel; fp16 buffers are passed as uint16 bit patterns with 0x7e00 (NaN) guards."""

    def __init__(self, eng, x, guard_fill=None):
        x = np.ascontiguousarray(x)
        self.shape, self.n, self.dtype = x.shape, x.size, x.dtype
        if guard_fill is None:
            guard_fill = {np.dtype(np.float32): np.nan, np.dtype(np.int32): 0, np.dtype(np.uint16): 0x7e00,
                          np.dtype(np.uint32): 0}[x.dtype]
        self.fill = guard_fill
        img = np.full(self.n + 2 * G, guard_fill, x.dtype)
        img[G:G + self.n] = x.reshape(-1)
        self.buf = Buf(eng, img)

    def ptr(self, off=0):
        return self.buf.ptr(G + off)

    def get(self):
        img = self.buf.get()
        guard = np.concatenate([img[:G], img[G + self.n:]])
        if self.dtype == np.float32 and np.isnan(self.fill):
            assert np.isnan(guard).all(), "a kernel wrote outside its output"
        else:
            assert (guard == self.fill).all(), "a kernel wrote outside its output"
        return img[G:G + self.n].reshape(self.shape)

    def free(self):
        self.buf.free()


class Pool:
    def __init__(self, eng):
        self.eng, self.bufs = eng, []

    def __call__(self, x, guard_fill=None):
        d = Dev(self.eng, x, guard_fill)
        self.bufs.append(d)
        return d

    def out(self, shape, dtype=np.float32):
        """an "out =" buffer: NaN (or sentinel) inside and outside"""
        fill = {np.float32: np.nan, np.int32: ISENT, np.uint16: 0x7e00}[dtype]
        return self(np.full(shape, fill, dtype), fill)

    def free(self):
        for d in self.bufs:
            d.free()
        self.bufs = []


def _image(X, off, ld, rows_extra=0, fill=np.nan):
    """X (r, c) placed at element offset `off` with row pitch ld; everything else (offset, padding columns, extra rows) = fill"""
    r, c = X.shape
    img = np.full(off + (r + rows_extra) * ld, fill, np.float32)
    img[off:off + r * ld].reshape(r, ld)[:, :c] = X
    return img


def _view(img, off, rows, cols, ld):
    return img[off:off + rows * ld].reshape(rows, ld)[:, :cols]


def lstm_step_fwd_ref(z_x, h_prev, Wh, c_prev, mask):
    """One nn.SeqLSTM forward step in fp64 numpy.  z_x (R,4H): x-projection + bias; h_prev (R,H) or None;
    Wh (H,4H): the h rows of the (D+H,4H) weight; c_prev (R,H) or None; mask (R,) bool = rows reset to zero.
    Returns the activated gates [i f o g] (R,4H), c_t and h_t."""
    z = np.asarray(z_x, np.float64).copy()
    H = z.shape[1] // 4
    if h_prev is not None:
        z += np.asarray(h_prev, np.float64) @ np.asarray(Wh, np.float64)
    a = np.empty_like(z)
    a[:, :3 * H] = 1.0 / (1.0 + np.exp(-z[:, :3 * H]))
    a[:, 3 * H:] = np.tanh(z[:, 3 * H:])
    i, f, o, g = a[:, :H], a[:, H:2 * H], a[:, 2 * H:3 * H], a[:, 3 * H:]
    cp = np.zeros_like(i) if c_prev is None else np.asarray(c_prev, np.float64)
    c = f * cp + i * g
    h = o * np.tanh(c)
    if mask is not None:
        a[mask] = 0
        c[mask] = 0
        h[mask] = 0
    return a, c, h


def lstm_step_bwd_ref(gates, c_prev, c_cur, dh, dc, mask):
    """The matching backward step: gates = activated [i f o g] of step t, dh = gradient wrt h_t (recurrent + external),
    dc = cell-gradient carry from step t+1.  Returns da_t (R,4H) and the carry for step t-1."""
    a = np.asarray(gates, np.float64)
    H = a.shape[1] // 4
    i, f, o, g = a[:, :H], a[:, H:2 * H], a[:, 2 * H:3 * H], a[:, 3 * H:]
    cp = np.zeros_like(i) if c_prev is None else np.asarray(c_prev, np.float64)
    tc = np.tanh(np.asarray(c_cur, np.float64))
    dh = np.asarray(dh, np.float64)
    d = np.asarray(dc, np.float64) + dh * o * (1 - tc * tc)
    da = np.concatenate([d * g * i * (1 - i), d * cp * f * (1 - f), dh * tc * o * (1 - o), d * i * (1 - g * g)], axis=1)
    dc_prev = d * f
    if mask is not None:
        da[mask] = 0
        dc_prev[mask] = 0
    return da, dc_prev
