"""tests/seq_lstm_ref.py against oracle.visdial_oracle.seq_lstm (torch fp64 autograd through its hand-written BPTT), on the CPU.

The oracle derives its mask from the input (an all-zero x row), the reference takes mask ids.  The inputs here make the two agree:
dense x whose masked rows are zero, and embedding-gathered x whose masked rows are the pad token's (a zero row of the table).
The unmasked gathered case keeps pad tokens in the sequence: their rows are zero inputs that still step the LSTM, so the pad
row of the embedding gets a gradient, which the oracle keeps and table_grads must reproduce."""
import numpy as np
import pytest
import torch

import seq_lstm_ref as S
from oracle import visdial_oracle as O


def _case(T, R, D, H, V, seed):
    rng = np.random.default_rng(seed)
    W = rng.standard_normal((D + H, 4 * H)) / np.sqrt(D + H)
    b = rng.standard_normal(4 * H) * 0.5
    emb = rng.standard_normal((V + 1, D))
    emb[0] = 0
    tok = rng.integers(0, V + 1, (T, R))
    tok[:, 0] = 0                                   # an all-pad row
    tok[T - 1, 1] = V                               # the last table row
    g = lambda *s: rng.standard_normal(s)
    return W, b, emb, tok, g(R, H), g(R, H), g(T, R, H), g(R, H), g(R, H)


def _oracle(W, b, x, h0, c0, maskzero, dh_all, dh_last, dc_last, emb=None, tok=None):
    t = lambda a: torch.tensor(a, dtype=torch.float64, requires_grad=True)
    Wt, bt, h0t, c0t = t(W), t(b), t(h0), t(c0)
    if emb is not None:
        et = t(emb)
        xt = O.lookup_table_mask_zero(et, torch.tensor(tok))
    else:
        xt = t(x)
    h, c = O.seq_lstm(xt, Wt, bt, h0t, c0t, maskzero=maskzero)
    loss = (h * torch.tensor(dh_all)).sum() + (h[-1] * torch.tensor(dh_last)).sum() + (c[-1] * torch.tensor(dc_last)).sum()
    loss.backward()
    out = {"h": h.detach().numpy(), "c": c.detach().numpy(), "dW": Wt.grad.numpy(), "db": bt.grad.numpy(),
           "dh0": h0t.grad.numpy(), "dc0": c0t.grad.numpy()}
    out["dx"] = et.grad.numpy() if emb is not None else xt.grad.numpy()
    return out


def _close(got, ref, what):
    assert np.abs(np.asarray(got) - ref).max() <= 1e-11 * (1 + np.abs(ref).max()), what


@pytest.mark.parametrize("T", [1, 2, 5])
def test_dense_masked(T):
    R, D, H = 7, 6, 8
    W, b, _, tok, h0, c0, dh_all, dh_last, dc_last = _case(T, R, D, H, 5, T)
    mask = tok == 0
    x = np.random.default_rng(T).standard_normal((T, R, D))
    x[mask] = 0
    ref = _oracle(W, b, x, h0, c0, True, dh_all, dh_last, dc_last)
    gates, c, h, _ = S.forward(W, b, x, mask, h0, c0)
    _close(h, ref["h"], "h")
    _close(c, ref["c"], "c")
    da, _, _, dc0 = S.backward(W, gates, c, c0, mask, dh_all, dh_last, dc_last)
    g = S.weight_grads(W, x, h, da, h0)
    _close(np.concatenate([g["dWx"][0], g["dWh"][0]]), ref["dW"], "dW")
    _close(g["db"][0], ref["db"], "db")
    _close(g["dx"][0], ref["dx"], "dx")
    _close(g["dh0"][0], ref["dh0"], "dh0")
    _close(dc0, ref["dc0"], "dc0")


@pytest.mark.parametrize("masked", [True, False], ids=["masked", "pads-unmasked"])
def test_gathered_table_grads(masked):
    """the table route's dP / dWx / db / dEmb against the oracle's embedding gradient, pad row included"""
    T, R, D, H, V = 4, 9, 6, 8, 5
    W, b, emb, tok, h0, c0, dh_all, dh_last, dc_last = _case(T, R, D, H, V, 11 + masked)
    mask = tok == 0 if masked else None
    x = emb[tok]
    ref = _oracle(W, b, None, h0, c0, masked, dh_all, dh_last, dc_last, emb=emb, tok=tok)
    gates, c, h, _ = S.forward(W, b, x, mask, h0, c0)
    _close(h, ref["h"], "h")
    da, _, _, _ = S.backward(W, gates, c, c0, mask, dh_all, dh_last, dc_last)
    g = S.weight_grads(W, x, h, da, h0)
    tg = S.table_grads(W, emb, tok, da)
    _close(np.concatenate([tg["dWx"][0], g["dWh"][0]]), ref["dW"], "dW")
    _close(tg["db"][0], ref["db"], "db")
    _close(tg["dEmb"][0], ref["dx"], "dEmb")
    if masked:
        assert (tg["dEmb"][0][0] == 0).all()        # every pad row is masked: no gradient reaches the pad row
    else:
        assert np.abs(ref["dx"][0]).max() > 1e-3    # the oracle keeps the pad row's gradient


def test_teacher_forced_is_free_running_on_exact_state():
    """fed the reference's own state, the teacher-forced forward and BPTT reproduce the free-running ones exactly"""
    T, R, D, H = 5, 7, 6, 8
    W, b, _, tok, h0, c0, dh_all, dh_last, dc_last = _case(T, R, D, H, 5, 3)
    mask = tok == 0
    x = np.random.default_rng(3).standard_normal((T, R, D))
    gates, c, h, _ = S.forward(W, b, x, mask, h0, c0)
    g2, c2, h2, _ = S.forward(W, b, x, mask, h0, c0, tf=(h, c))
    assert (g2 == gates).all() and (c2 == c).all() and (h2 == h).all()
    da, _, _, dc0 = S.backward(W, gates, c, c0, mask, dh_all, dh_last, dc_last)
    da2, _, _, dc02 = S.backward(W, gates, c, c0, mask, dh_all, dh_last, dc_last, tf_da=da)
    assert (da2 == da).all() and (dc02 == dc0).all()
