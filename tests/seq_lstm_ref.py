"""nn.SeqLSTM forward and BPTT in fp64 numpy, step by step on tests/helpers.py's lstm_step_fwd_ref / lstm_step_bwd_ref, with
explicit mask ids as the engine takes them (test_seq_lstm_ref.py pins it to oracle.visdial_oracle.seq_lstm).

Time-major arrays: x (T, R, D), h / c (T, R, H), gates / da (T, R, 4H); mask (T, R) bool, True = the row is reset at that step
(token id 0).  W is the (D + H, 4H) weight, x rows first, gate blocks [i f o g]; b the (4H,) bias.

Two modes.  Free-running: the whole sequence from the inputs.  Teacher-forced (tf given): step t starts from the state the device
saved at t-1, and in the BPTT the recurrent gradient of step t is da_{t+1} of the device, while the cell-gradient carry runs free.
Each step then carries one step's error only.  The gradients (weight_grads, table_grads) are contractions of whatever operands they
are given: the reference's own, or the device's saved h / da.  Every function also returns the contraction of the absolute values,
sum_k |a_k b_k|, the scale of an accumulated contraction's rounding error."""
import numpy as np

from helpers import lstm_step_bwd_ref, lstm_step_fwd_ref


def _f64(a):
    return None if a is None else np.asarray(a, np.float64)


def forward(W, b, x, mask=None, h0=None, c0=None, tf=None):
    """gates, c, h (T, R, .) and S (T, R, 4H) = |x||Wx| + |b| + |h_prev||Wh|, the pre-activation's absolute terms.
    tf = (h, c) of the device: step t reads them at t-1 instead of the reference's own."""
    W, x = _f64(W), _f64(x)
    T, R, D = x.shape
    Wx, Wh = W[:D], W[D:]
    H = Wh.shape[0]
    zx = (x.reshape(T * R, D) @ Wx + _f64(b)).reshape(T, R, 4 * H)
    S = (np.abs(x.reshape(T * R, D)) @ np.abs(Wx) + np.abs(_f64(b))).reshape(T, R, 4 * H)
    gates, c, h = np.zeros((T, R, 4 * H)), np.zeros((T, R, H)), np.zeros((T, R, H))
    for t in range(T):
        if t == 0:
            hp, cp = _f64(h0), _f64(c0)
        elif tf is None:
            hp, cp = h[t - 1], c[t - 1]
        else:
            hp, cp = _f64(tf[0][t - 1]), _f64(tf[1][t - 1])
        if hp is not None:
            S[t] += np.abs(hp) @ np.abs(Wh)
        gates[t], c[t], h[t] = lstm_step_fwd_ref(zx[t], hp, Wh, cp, None if mask is None else mask[t])
    return gates, c, h, S


def backward(W, gates, c, c0=None, mask=None, dh_all=None, dh_last=None, dc_last=None, tf_da=None):
    """da (T, R, 4H), dh (T, R, H) = the full gradient wrt h_t each step took, Sdh its absolute terms, and dc0 (R, H) = the carry
    past step 0.  dh_all (T, R, H) enters every step, dh_last / dc_last the last one.  tf_da: the device's da; step t's recurrent
    gradient is tf_da[t+1] Wh^T instead of the reference's own."""
    gates, c = _f64(gates), _f64(c)
    T, R, G = gates.shape
    H = G // 4
    Wh = _f64(W)[-H:]
    da, dh, Sdh = np.zeros((T, R, G)), np.zeros((T, R, H)), np.zeros((T, R, H))
    dc = np.zeros((R, H)) if dc_last is None else _f64(dc_last)
    for t in reversed(range(T)):
        if dh_all is not None:
            dh[t] += dh_all[t]
            Sdh[t] += np.abs(dh_all[t])
        if t == T - 1:
            if dh_last is not None:
                dh[t] += dh_last
                Sdh[t] += np.abs(dh_last)
        else:
            nxt = da[t + 1] if tf_da is None else _f64(tf_da[t + 1])
            dh[t] += nxt @ Wh.T
            Sdh[t] += np.abs(nxt) @ np.abs(Wh.T)
        cp = c[t - 1] if t else _f64(c0)
        da[t], dc = lstm_step_bwd_ref(gates[t], cp, c[t], dh[t], dc, None if mask is None else mask[t])
    return da, dh, Sdh, dc


def weight_grads(W, x, h, da, h0=None):
    """{name: (value, sum |a b|)} for dWx = sum_t x_t^T da_t, dWh = sum_t h_{t-1}^T da_t (h_{-1} = h0, or no term), db = sum da,
    dx = da Wx^T and dh0 = da_0 Wh^T"""
    W, x, h, da = _f64(W), _f64(x), _f64(h), _f64(da)
    T, R, D = x.shape
    H = h.shape[2]
    Wx, Wh = W[:D], W[D:]
    A = da.reshape(T * R, -1)
    X = x.reshape(T * R, D)
    hp = np.concatenate([np.zeros((1, R, H)) if h0 is None else _f64(h0)[None], h[:-1]]).reshape(T * R, H)
    out = {"dWx": (X.T @ A, np.abs(X).T @ np.abs(A)), "dWh": (hp.T @ A, np.abs(hp).T @ np.abs(A)),
           "db": (A.sum(0), np.abs(A).sum(0)),
           "dx": ((A @ Wx.T).reshape(T, R, D), (np.abs(A) @ np.abs(Wx.T)).reshape(T, R, D)),
           "dh0": (da[0] @ Wh.T, np.abs(da[0]) @ np.abs(Wh.T))}
    if h0 is None:
        out["dh0"] = (np.zeros_like(out["dh0"][0]), out["dh0"][1])
    return out


def table_grads(W, emb, tok, da):
    """the x-side gradients of an embedding-gathered input in projected space: dP[v] = sum of da over the rows whose token is
    v, then dWx = Emb^T dP, db = colsum dP, dEmb = dP Wx^T.  The pad row is an ordinary row here: its dP (rows of token 0 that
    were not masked) reaches dEmb[0] as the oracle's LookupTableMaskZero gradient does; Emb[0] is zero, so it adds nothing to
    dWx.  {name: (value, sum |a b| over the whole chain)}"""
    W, emb, da = _f64(W), _f64(emb), _f64(da)
    V1, E = emb.shape
    G = da.shape[-1]
    Wx = W[:E]
    A = da.reshape(-1, G)
    tok = np.asarray(tok).reshape(-1)
    dP, aP = np.zeros((V1, G)), np.zeros((V1, G))
    np.add.at(dP, tok, A)
    np.add.at(aP, tok, np.abs(A))
    return {"dWx": (emb.T @ dP, np.abs(emb).T @ aP), "db": (dP.sum(0), aP.sum(0)), "dEmb": (dP @ Wx.T, aP @ np.abs(Wx.T))}
