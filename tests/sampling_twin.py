"""TEST INFRASTRUCTURE ONLY.  numpy twin of the engine's sampling rule (visdial_b200/csrc/common.cuh, Engine::gen_sample):
the token drawn at step t (1-based) for row r is 1 + argmax_j (x_j / T + g_j), ties to the lower class, with
g_j = -log(-log(u_j)), u_j = ((w >> 8) + 0.5) 2^-24 and w = Philox4x32-10 word idx % 4 at counter
(idx // 4 lo, idx // 4 hi, SITE_SAMPLE, t), key = seed, idx = (row_offset + r) V + j.  Everything here is float64, so a
device draw may differ from the twin only where the two best keys are closer than the device's float32 rounding.
`generate_answers_sample` is oracle.generate_answers' sampling branch with this rule in place of torch.multinomial."""
import numpy as np
import torch

from oracle import visdial_oracle as O
from oracle.philox import MASK, philox4x32_10

SITE_SAMPLE = 64


def gumbel_of_words(w) -> np.ndarray:
    """g of Philox words (uint32 array), float64"""
    m = np.asarray(w, dtype=np.uint64) >> np.uint64(8)
    u = (m.astype(np.float64) + 0.5) * 2.0 ** -24
    return -np.log(-np.log(u))


def sample_words(seed: int, step: int, row_offset: int, rows: int, V: int) -> np.ndarray:
    """the (rows, V) Philox words of step `step` for the rows row_offset .. row_offset + rows - 1"""
    idx = (np.uint64(row_offset) + np.arange(rows, dtype=np.uint64)[:, None]) * np.uint64(V) + np.arange(V, dtype=np.uint64)
    q = idx >> np.uint64(2)
    out = philox4x32_10(q & MASK, q >> np.uint64(32), np.full(q.shape, SITE_SAMPLE, np.uint64),
                        np.full(q.shape, step & 0xFFFFFFFF, np.uint64), seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    words = np.stack(out, -1)                                               # (rows, V, 4)
    return np.take_along_axis(words, (idx & np.uint64(3)).astype(np.int64)[..., None], -1)[..., 0]


def gumbel_keys(x, temperature: float, seed: int, step: int, row_offset: int) -> np.ndarray:
    """x / T + g for logits (or log-probabilities: a per-row shift does not move the argmax) x (rows, V)"""
    x = np.asarray(x, dtype=np.float64)
    return x / temperature + gumbel_of_words(sample_words(seed, step, row_offset, x.shape[0], x.shape[1]))


def draw(x, temperature: float, seed: int, step: int, row_offset: int = 0):
    """(1-based tokens (rows,), gap between each row's two best keys (rows,))"""
    k = gumbel_keys(x, temperature, seed, step, row_offset)
    cls = np.argmax(k, 1)                                                   # first maximum: the lower class on ties
    if k.shape[1] == 1:
        return cls + 1, np.full(k.shape[0], np.inf)
    top2 = -np.partition(-k, 1, axis=1)[:, :2]
    return cls + 1, top2[:, 0] - top2[:, 1]


def generate_answers_sample(cfg, P, batch, start_token: int, beam_len: int, temperature: float, philox_seed: int,
                            row_offset: int = 0):
    """Model:generateAnswers' sampling (model.lua:581-602) for one batch, on the oracle's step decoder, drawing with the
    rule above.  Returns (answers (R, beam_len + 1) int64 with column 0 = start_token, log-probabilities of the drawn
    tokens (R, beam_len) float64, key gaps (R, beam_len))."""
    with torch.no_grad():
        inputs = O.prepare_inputs(cfg, batch)
        encOut, state = O.ENCODERS[cfg["encoder"]](O.Ctx(train=False), cfg, P, inputs)
        R = encOut.shape[0]
        H0, C0 = O.gen_forward_connect(state, encOut)
        H = [h if h is not None else encOut.new_zeros(R, encOut.shape[1]) for h in H0]
        Cc = [c if c is not None else encOut.new_zeros(R, encOut.shape[1]) for c in C0]
        tok = torch.full((R,), start_token, dtype=torch.long)
        ans, lps, gaps = [tok.numpy().copy()], [], []
        for t in range(1, beam_len + 1):                                    # :584
            logp, H, Cc = O.decoder_gen_step(cfg, P, tok, H, Cc)            # :586-588 (+ decoderConnect)
            lp = logp.double().numpy()
            cls, gap = draw(lp, temperature, philox_seed, t, row_offset)
            lps.append(lp[np.arange(R), cls - 1])
            gaps.append(gap)
            ans.append(cls)
            tok = torch.from_numpy(cls.astype(np.int64))
    return np.stack(ans, 1), np.stack(lps, 1), np.stack(gaps, 1)
