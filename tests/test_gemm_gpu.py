"""The engine's dense contractions per element against fp64, on every route: Engine::gemm_tn (k_tc_gemm MODE_GENERIC or
k_gemm_tn) and Engine::gemm_atb (k_tc_atb or k_gemm_atb), through vd_test_kernel's `gemm_tn` / `gemm_atb` entries, so the
route is the engine's decision in its math mode.

Every case asserts from the launch counters which of the four kernels ran, against tests/gemm_ref.py's mirror of the
acceptance predicates (and nothing on the tensor cores in FP32 mode), and holds every element of C to gemm_ref's bound:
(n + 3) U (sum_k |a_k b_k| + |bias| + |beta C0|), n = K for gemm_tn and the longest split plus the split count for gemm_atb,
plus 2^-9 sum_k |a_k b_k| where fp32 operands meet the tensor cores, through tanh' and the tanh's own error for act = 1.
Tensor-core cases run on TF32-exact operands, so only the accumulation order separates them from fp64; fp32-operand cases
carry a witness element (a row and a column of 1 + 2^-11) whose error must exceed the fp32-only bound, which shows that the
tensor cores really ran.  Random-sign operands keep a first-order bound meaningful up to K ~ 2 000; past that a block of
output columns has non-negative operands, where sum |a b| = |sum a b| and a lost or doubled k-block or split is far outside.

Buffers follow test_tc_edges_gpu.py: NaN guard bands and padding around C (nothing outside C[0:M, 0:N] may change), NaN in
C when beta = 0, NaN between K and the operands' pitch, NaN in the table rows no gather id names.  The largest err / bound
per case is printed (RATIO lines, pytest -s)."""
import ctypes as C

import numpy as np
import pytest
import torch

import gemm_ref as G
from helpers import call, small_params
from visdial_b200 import VD_MATH_F16, VD_MATH_FP32, VD_MATH_TF32, Engine
from visdial_b200._lib import check

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")
NAN = float("nan")
KERNELS = ("k_tc_gemm", "gemm_tn_simt", "k_tc_atb", "gemm_atb_simt")
MODES = {"fp32": VD_MATH_FP32, "tf32": VD_MATH_TF32, "f16": VD_MATH_F16}
RANDOM_SIGN_MAX_K = 2048
NONNEG_COLS = 16               # past RANDOM_SIGN_MAX_K: output columns [0, 16) of gemm_atb have non-negative operands,
NONNEG_ROWS = 16               # and the rows [0, 16) of gemm_tn's A (gathered: its table) and B


@pytest.fixture(scope="module")
def eng():
    e = Engine(small_params("lf-ques", "disc"))
    e.profile(True)
    yield e
    e.close()


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _launches(eng):
    return {n: eng.kernel_stats(n)["launches"] for n in KERNELS}


def _ptr(t, off=0):
    return None if t is None else C.c_void_p(t.data_ptr() + t.element_size() * off)


def _image(X, off, ld, rows_extra=1):
    """X (r, c) at element offset `off` with row pitch ld, NaN everywhere else (offset, padding, extra rows)"""
    r, c = X.shape
    img = torch.full((off + (r + rows_extra) * ld,), NAN, dtype=torch.float32, device=DEV)
    img[off:off + r * ld].view(r, ld)[:, :c] = X
    return img


def _view(img, off, r, c, ld):
    return img[off:off + r * ld].view(r, ld)[:, :c]


def _tf32(x):
    return (x.view(torch.int32) & -8192).view(torch.float32)


def _operand(gen, shape, kind, scale=1.0):
    x = torch.randn(shape, generator=gen, device=DEV) * scale
    return _tf32(x) if kind == "exact" else x


def _check_c(img, off, M, N, ldc, what):
    """the C image: finite inside C[0:M, 0:N], untouched NaN outside"""
    got = _view(img, off, M, N, ldc).double()
    assert torch.isfinite(got).all(), (what, "non-finite C: a NaN guard, padding or (beta = 0) C element was read")
    rest = img.clone()
    _view(rest, off, M, N, ldc).fill_(NAN)
    assert torch.isnan(rest).all(), (what, "written outside C[0:M, 0:N]")
    return got


def _route(eng, before, want, what):
    d = {n: v - before[n] for n, v in _launches(eng).items()}
    assert d == {n: int(n == want) for n in KERNELS}, (what, "expected one launch of " + want, d)


def _report(what, err, bnd):
    """the largest err / bound; an element whose bound is 0 (a zero table row, no bias, beta = 0) must be exact"""
    assert bool((err[bnd == 0] == 0).all()), (what, "an element with a zero bound is not exact")
    ratio = float((err / torch.where(bnd > 0, bnd, 1.0)).max())
    print("RATIO %-52s %.3g" % (what, ratio))
    assert ratio <= 1, (what, ratio)
    return ratio


# ---------------------------------------------------------------------------------------------- C = act(beta C + bias + A B^T)
def run_tn(eng, mode, M, N, K, lda=None, ldb=None, ldc=None, offA=0, offB=0, offC=0, beta=0.0, bias=False, act=0,
           gather=None, table_rows=0, kind=None, tanh_edges=False, seed=0, label="", repeat=False):
    """one gemm_tn call in `mode`; returns C (M, N) as an fp64 tensor.  gather: "pad" (mostly pad id 0, whose table row is zero, as the
    engine's embedding), "repeat" (ids drawn with repeats, id 0 included) or None.  kind: "exact" (TF32-exact operands) or
    "fp32"; by default exact on the tensor cores and fp32 otherwise."""
    what = "tn %s %s M=%d N=%d K=%d" % (label, mode, M, N, K)
    tcmode = mode != "fp32"
    lda, ldb, ldc = lda or K, ldb or K, ldc or N
    tc = G.tn_takes_tc(tcmode, M, N, K, gather, G.aligned(offA, lda), G.aligned(offB, ldb), G.aligned(offC, ldc))
    kind = kind or ("exact" if tc else "fp32")
    gen = torch.Generator(device=DEV).manual_seed(seed)
    sa = 1.0
    if act and not tanh_edges:
        sa = 2.0 ** -round(np.log2(np.sqrt(K)))        # pre-activations O(1): tanh neither linear nor saturated
    if tanh_edges:
        sa = 2.0 ** -7
    B = _operand(gen, (N, K), kind)
    A = _operand(gen, (table_rows if gather else M, K), kind, sa)
    if K > RANDOM_SIGN_MAX_K:
        A[:NONNEG_ROWS] = A[:NONNEG_ROWS].abs()
        B[:NONNEG_ROWS] = B[:NONNEG_ROWS].abs()
    ids = None
    if gather:
        V = table_rows
        if gather == "pad":
            ids = torch.randint(1, V, (M,), generator=gen, device=DEV, dtype=torch.int32)
            ids[torch.rand(M, generator=gen, device=DEV) < 0.6] = 0
            A[0] = 0
        else:
            ids = torch.randint(0, max(2, M // 4), (M,), generator=gen, device=DEV, dtype=torch.int32)
            ids[::7] = 0
        named = torch.zeros(V, dtype=torch.bool, device=DEV)
        named[ids.long()] = True
        A[~named] = NAN                                   # rows no id names must never be read
        Ag = A[ids.long()]
    else:
        if kind == "fp32" and not act:
            A[0], B[0] = float(G.WITNESS), float(G.WITNESS)
        Ag = A
    C0 = torch.randn((M, N), generator=gen, device=DEV)
    bv = torch.randn(N, generator=gen, device=DEV) if bias else None
    if tanh_edges:                                        # columns at pre-activation ~ 9, ~ -9 and ~ 0
        bv = torch.tensor([9.0, -9.0, 0.0], device=DEV).repeat(N // 3 + 1)[:N]
        C0 = C0 * 1e-3
    imgA, imgB = _image(A, offA, lda), _image(B, offB, ldb)
    imgC = _image(C0 if beta != 0 else torch.full((M, N), NAN, device=DEV), offC, ldc, rows_extra=2)
    outs = []
    for _ in range(2 if repeat else 1):
        c = imgC.clone()
        torch.cuda.synchronize()
        eng.set_math_mode(MODES[mode])
        before = _launches(eng)
        check(call(eng, "gemm_tn", [_ptr(imgA, offA), _ptr(ids), _ptr(imgB, offB), _ptr(c, offC), _ptr(bv)],
                   [M, N, K, lda, ldb, ldc, act], [beta]))
        _route(eng, before, "k_tc_gemm" if tc else "gemm_tn_simt", what)
        outs.append(_check_c(c, offC, M, N, ldc, what))
    A64, B64 = Ag.double(), B.double()
    pre = A64 @ B64.T
    sabs = A64.abs() @ B64.abs().T
    extra = torch.zeros((), dtype=torch.float64, device=DEV)
    if bias or tanh_edges:
        pre += bv.double()
        extra = extra + bv.double().abs()
    if beta != 0:
        pre += beta * C0.double()
        extra = extra + abs(beta) * C0.double().abs()
    ref = torch.tanh(pre) if act else pre
    err = (outs[0] - ref).abs()
    bnd = G.bound(K, sabs, extra, tc, kind == "exact", act, ref)
    _report(what, err, bnd)
    if tc and kind == "fp32" and not act and not gather and K < 2 ** 14:
        b32 = G.bound(K, sabs, extra, False, True)
        assert float((err / b32).max()) > 1, (what, "the witness element shows no TF32 error: not reduced precision")
    if repeat:
        assert torch.equal(outs[0], outs[1]), (what, "two launches differ")
    return outs[0]


# ---------------------------------------------------------------------------------------------- C += A^T B
def run_atb(eng, mode, M, N, K, lda=None, ldb=None, ldc=None, offA=0, offB=0, offC=0, gather=None, table_rows=0,
            kind=None, budget=0, sms=132, seed=0, label="", repeat=False):
    what = "atb %s %s M=%d N=%d K=%d budget=%d" % (label, mode, M, N, K, budget)
    tcmode = mode != "fp32"
    lda, ldb, ldc = lda or M, ldb or N, ldc or N
    tc = G.atb_takes_tc(tcmode, M, N, K, gather, G.aligned(offA, lda), G.aligned(offB, ldb))
    kind = kind or ("exact" if tc else "fp32")
    gen = torch.Generator(device=DEV).manual_seed(seed)
    B = _operand(gen, (K, N), kind)
    rows = table_rows if gather else K
    A = _operand(gen, (rows, M), kind)
    if K > RANDOM_SIGN_MAX_K:
        A[:, :NONNEG_COLS] = A[:, :NONNEG_COLS].abs()
        B[:, :NONNEG_COLS] = B[:, :NONNEG_COLS].abs()
    ids = None
    if gather:
        ids = torch.randint(1, rows, (K,), generator=gen, device=DEV, dtype=torch.int32)
        ids[torch.rand(K, generator=gen, device=DEV) < (0.6 if gather == "pad" else 0.1)] = 0
        if gather == "pad":
            A[0] = 0
        named = torch.zeros(rows, dtype=torch.bool, device=DEV)
        named[ids.long()] = True
        A[~named] = NAN
        Ag = A[ids.long()]
    else:
        if kind == "fp32":
            A[:, 0], B[:, 0] = float(G.WITNESS), float(G.WITNESS)
        Ag = A
    C0 = torch.randn((M, N), generator=gen, device=DEV)
    imgA, imgB, imgC = _image(A, offA, lda), _image(B, offB, ldb), _image(C0, offC, ldc, rows_extra=2)
    outs = []
    for _ in range(2 if repeat else 1):
        c = imgC.clone()
        torch.cuda.synchronize()
        eng.set_math_mode(MODES[mode])
        before = _launches(eng)
        check(call(eng, "gemm_atb", [_ptr(imgA, offA), _ptr(ids), _ptr(imgB, offB), _ptr(c, offC)],
                   [M, N, K, lda, ldb, ldc, budget]))
        _route(eng, before, "k_tc_atb" if tc else "gemm_atb_simt", what)
        outs.append(_check_c(c, offC, M, N, ldc, what))
    ref = C0.double().clone()
    sabs = torch.zeros_like(ref)
    step = max(1, (1 << 27) // (M + N))                 # fp64 chunks of ~1 GB over K
    for k0 in range(0, K, step):
        a, b = Ag[k0:k0 + step].double(), B[k0:k0 + step].double()
        ref += a.T @ b
        sabs += a.abs().T @ b.abs()
    n = G.chain("atb", K, tc, M, N, sms, budget)
    bnd = G.bound(n, sabs, C0.double().abs(), tc, kind == "exact")
    _report(what, (outs[0] - ref).abs(), bnd)
    if tc and kind == "fp32" and not gather and K < 2 ** 14:
        b32 = G.bound(n, sabs, C0.double().abs(), False, True)
        assert float(((outs[0] - ref).abs() / b32).max()) > 1, (what, "the witness element shows no TF32 error")
    if repeat:
        splits = (G.atb_tc_splits(M, N, K, sms, budget) if tc else G.atb_simt_splits(M, N, K, sms))[0]
        if splits == 1:
            assert torch.equal(outs[0], outs[1]), (what, "one split, yet two launches differ")
    return outs[0]


# ---------------------------------------------------------------------------------------------- a) the engine's call sites
# C4 (mn-att-ques-im-hist + disc) and C3 (hrea-ques-im-hist + gen) at B = 32: E = 300, H = 512, G = 4H, V + 1 = 10 001,
# R = 320 encoder rows (32 dialogs x 10 rounds), TR = 20 R rows of a 20-token run.  Operand pitches and offsets are the
# engine's (engine.cu).
E, H, V1, R = 300, 512, 10001, 320
G4, TR = 4 * 512, 20 * 320

TN_SITES = {
    # lstm_forward_begin, Opt16: (V+1, 4H) projection table E Wx^T, Wx^T = the x columns of the [4H, D+H] shadow, no bias
    "ptable": dict(M=V1, N=G4, K=E, lda=E, ldb=E + H, ldc=G4),
    # lstm_forward_begin, Tc with a gathered input: the same table with the bias folded in
    "ptable_bias": dict(M=V1, N=G4, K=E, lda=E, ldb=E + H, ldc=G4, bias=True),
    # lstm_backward_end, table route: dEmb = dP Wx into the caller's buffer (demb_out), and dEmb += dP Wx into dW's rows
    "emb_fold_out": dict(M=V1, N=E, K=G4, ldc=E),
    "emb_fold_acc": dict(M=V1, N=E, K=G4, ldc=E, beta=1.0),
    # lstm_backward_end: dh0 = da_0 Wh (Wh = rows D.. of the (D+H, 4H) weight)
    "dh0": dict(M=R, N=H, K=G4, ldc=H),
    # lstm_backward_end: dx = da Wx of a dense-input run (layer 2, D = H; layer 1 of a pair, D = E)
    "dx_layer2": dict(M=TR, N=H, K=G4, ldc=H),
    "dx_layer1": dict(M=TR, N=E, K=G4, ldc=E),
    # lstm_xproj: gathered x-projection (Simt route: no bias), ids mostly the pad 0
    "xproj_gather": dict(M=TR, N=G4, K=E, lda=E, ldb=E + H, ldc=G4, gather="pad", table_rows=V1),
    # lstm_xproj: layer 2's dense x-projection with the bias (Tc route)
    "xproj_dense": dict(M=TR, N=G4, K=H, lda=H, ldb=2 * H, ldc=G4, bias=True),
    # lstm_simt_fwd_step: gates += h Wh^T, Wh^T = the h columns of [4H, D+H] (offset D, pitch D+H)
    "step_fwd": dict(M=R, N=G4, K=H, ldb=E + H, offB=E, beta=1.0),
    # lstm_simt_bwd_step and lstm_pair_backward's per-step d(h1) = da2_t Wx2: (R, H) = (R, 4H) (4H, H)
    "step_bwd": dict(M=R, N=H, K=G4),
}
ATB_SITES = {
    # lstm_backward_end, table route: dWx += E^T dP
    "table_grad": dict(M=E, N=G4, K=V1),
    # lstm_backward_end: dWh += h_{0..T-2}^T da_{1..T-1} into rows D.. of dW (da offset R rows, dW offset D rows)
    "dwh": dict(M=H, N=G4, K=TR - R, offB=R * G4, offC=E * G4),
    "dwh_h0": dict(M=H, N=G4, K=R, offC=E * G4),
    # lstm_backward_end: gathered dWx += Emb[ids]^T da (ids mostly the pad 0)
    "dwx_gather": dict(M=E, N=G4, K=TR, gather="pad", table_rows=V1),
    # lstm_backward_end: dense dWx of layer 2
    "dwx_dense": dict(M=H, N=G4, K=TR),
}
# linear_fwd / linear_bwd (engine.cu): (out, in, rows, act, beta_dx or None without dx)
LINEARS = {
    "c4.mn.fact": (512, 512, R, 1, 0.0),
    "c4.mn.query": (512, 512, R, 1, 0.0),
    "c4.san.img": (512, 512, 32 * 196, 1, None),
    "c4.san.hop1.img_common": (512, 512, R * 196, 0, 1.0),
    "c4.san.hop1.ques_common": (512, 512, R, 0, 1.0),
    "c4.san.out": (512, 512, R, 1, 0.0),
    "c3.img.embed": (300, 4096, R, 0, None),
    "c3.dec.out": (10000, 512, TR, 0, 0.0),
}
# the call sites VD_MATH_F16 routes to these kernels too (its option LSTM takes the table route without bias; its encoder
# pairs' dx and every linear layer)
F16_SITES = ("ptable", "emb_fold_acc", "dx_layer1", "table_grad")


@pytest.mark.parametrize("mode", ["tf32", "fp32", "f16"])
@pytest.mark.parametrize("site", sorted(TN_SITES))
def test_tn_call_sites(eng, site, mode):
    if mode == "f16" and site not in F16_SITES:
        pytest.skip("VD_MATH_F16 does not reach this call site")
    run_tn(eng, mode, label=site, seed=sum(map(ord, site)), **TN_SITES[site])


@pytest.mark.parametrize("mode", ["tf32", "fp32", "f16"])
@pytest.mark.parametrize("site", sorted(ATB_SITES))
def test_atb_call_sites(eng, sms, site, mode):
    if mode == "f16" and site not in F16_SITES:
        pytest.skip("VD_MATH_F16 does not reach this call site")
    run_atb(eng, mode, sms=sms, label=site, seed=sum(map(ord, site)), **ATB_SITES[site])


@pytest.mark.parametrize("mode", ["tf32", "fp32", "f16"])
@pytest.mark.parametrize("seg", sorted(LINEARS))
def test_linear_layers(eng, sms, seg, mode):
    out, inp, rows, act, beta_dx = LINEARS[seg]
    run_tn(eng, mode, rows, out, inp, bias=True, act=act, label=seg + ".fwd", seed=1)           # y = act(x W^T + b)
    run_atb(eng, mode, out, inp, rows, sms=sms, label=seg + ".dW", seed=2)                     # dW += dy^T x
    if beta_dx is not None:
        run_tn(eng, mode, rows, inp, out, beta=beta_dx, label=seg + ".dx", seed=3)             # dx (+)= dy W


@pytest.mark.parametrize("mode", ["tf32", "f16"])
def test_tensor_cores_on_fp32_operands(eng, sms, mode):
    """fp32 operands that TF32 cannot hold: the bound takes the truncation term, and the witness element's error exceeds
    the fp32-only bound (the tensor cores ran, in reduced precision)"""
    run_tn(eng, mode, **dict(TN_SITES["ptable_bias"], label="ptable_bias, fp32 operands", kind="fp32", seed=21))
    run_tn(eng, mode, **dict(TN_SITES["emb_fold_acc"], label="emb_fold_acc, fp32 operands", kind="fp32", seed=22))
    run_tn(eng, mode, 129, 68, 33, beta=0.5, bias=True, ldc=72, label="fp32 operands", kind="fp32", seed=23)
    run_atb(eng, mode, **dict(ATB_SITES["table_grad"], label="table_grad, fp32 operands", kind="fp32", sms=sms, seed=24))
    run_atb(eng, mode, 129, 257, 1000, label="fp32 operands", kind="fp32", sms=sms, seed=25)


# ---------------------------------------------------------------------------------------------- large K
@pytest.mark.parametrize("mode", ["tf32", "fp32"])
@pytest.mark.parametrize("M,N,K", [(300, 2048, 10001), (129, 257, 100000)])
def test_atb_split_k(eng, sms, mode, M, N, K):
    run_atb(eng, mode, M, N, K, sms=sms, label="split-K", seed=K)


@pytest.mark.parametrize("mode", ["tf32", "fp32"])
def test_atb_c4_option_dwh(eng, sms, mode):
    """the TF32 option LSTM's dWh, gemm_atb(H, 4H, T R - R): K = 608 000 at C4 (32 000 rows, 20 steps).  Non-negative
    operands everywhere (A 1.2 GB, B 5 GB), so every element's bound is a share of its own value"""
    M, N, K = H, G4, 608000
    tc = mode != "fp32"
    gen = torch.Generator(device=DEV).manual_seed(608)
    A = torch.rand((K, M), generator=gen, device=DEV)
    B = torch.rand((K, N), generator=gen, device=DEV)
    if tc:
        A, B = _tf32(A), _tf32(B)
    C0 = torch.rand((M, N), generator=gen, device=DEV)
    c = C0.clone()
    torch.cuda.synchronize()
    eng.set_math_mode(MODES[mode])
    before = _launches(eng)
    check(call(eng, "gemm_atb", [_ptr(A), None, _ptr(B), _ptr(c)], [M, N, K, M, N, N, 0]))
    what = "atb c4 option dWh %s K=%d" % (mode, K)
    _route(eng, before, "k_tc_atb" if tc else "gemm_atb_simt", what)
    ref = C0.double()
    for k0 in range(0, K, 65536):
        ref = ref + A[k0:k0 + 65536].double().T @ B[k0:k0 + 65536].double()
    n = G.chain("atb", K, tc, M, N, sms)
    _report(what, (c.double() - ref).abs(), G.bound(n, ref - C0.double(), C0.double(), tc, True))
    del A, B
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------- b) edges
@pytest.mark.parametrize("mode", ["tf32", "fp32"])
@pytest.mark.parametrize("N", [20, 24, 28, 300])
def test_tn_beta_ragged_column_group(eng, mode, N):
    """beta != 0 with N % 16 in {4, 8, 12}: the last 16-column group of each tile takes the epilogue's element-wise C load;
    products small beside bias and beta C, so an epilogue that rounds either to TF32 or drops C fails"""
    for beta in (1.0, -0.5):
        run_tn(eng, mode, 129, N, 64, beta=beta, bias=True, ldc=N + 4, offC=4, label="beta ragged", seed=N)
        run_tn_small(eng, mode, 130, N, 40, beta, label="beta ragged, small products", seed=N + 1)


def run_tn_small(eng, mode, M, N, K, beta, label, seed):
    """run_tn with A scaled by 2^-6: the epilogue's terms dominate every element's bound"""
    tcmode = mode != "fp32"
    tc = G.tn_takes_tc(tcmode, M, N, K, None, True, True, True)
    kind = "exact" if tc else "fp32"
    gen = torch.Generator(device=DEV).manual_seed(seed)
    A = _operand(gen, (M, K), kind, 2.0 ** -6)
    B = _operand(gen, (N, K), kind)
    C0 = torch.randn((M, N), generator=gen, device=DEV)
    bv = torch.randn(N, generator=gen, device=DEV)
    c = _image(C0, 0, N, rows_extra=2)
    torch.cuda.synchronize()
    eng.set_math_mode(MODES[mode])
    before = _launches(eng)
    what = "tn %s %s M=%d N=%d K=%d beta=%g" % (label, mode, M, N, K, beta)
    check(call(eng, "gemm_tn", [_ptr(A), None, _ptr(B), _ptr(c), _ptr(bv)], [M, N, K, K, K, N, 0], [beta]))
    _route(eng, before, "k_tc_gemm" if tc else "gemm_tn_simt", what)
    got = _check_c(c, 0, M, N, N, what)
    ref = A.double() @ B.double().T + bv.double() + beta * C0.double()
    sabs = A.double().abs() @ B.double().abs().T
    bnd = G.bound(K, sabs, bv.double().abs() + abs(beta) * C0.double().abs(), tc, True)
    _report(what, (got - ref).abs(), bnd)


@pytest.mark.parametrize("mode", ["tf32", "fp32"])
@pytest.mark.parametrize("M,N,K", [(129, 36, 64), (300, 132, 300)])
def test_tn_tanh_edges(eng, mode, M, N, K):
    """act = 1 at pre-activations near 0 (ftanh's relative error is largest) and near +-9 (tanh saturates)"""
    run_tn(eng, mode, M, N, K, beta=0.5, act=1, tanh_edges=True, label="tanh edges", seed=M)


@pytest.mark.parametrize("mode", ["tf32", "fp32"])
def test_gathers_repeated_ids(eng, sms, mode):
    """gathered rows with repeated ids and id 0: both CUDA-core kernels in every mode (the tensor-core ones refuse a gather)"""
    run_tn(eng, mode, 257, 132, 300, bias=True, gather="repeat", table_rows=97, label="gather repeat", seed=5)
    run_tn(eng, mode, 64, 68, 33, beta=1.0, gather="repeat", table_rows=40, lda=36, label="gather repeat", seed=6)
    run_atb(eng, mode, 300, 260, 1000, gather="repeat", table_rows=50, sms=sms, label="gather repeat", seed=7)
    run_atb(eng, mode, 36, 2048, 5000, gather="repeat", table_rows=3000, lda=40, sms=sms, label="gather repeat", seed=8)


@pytest.mark.parametrize("budget", [0, 48, 96, 40])
def test_atb_sm_budget(eng, sms, budget):
    """the split count under an SM budget (the option stream's); 40 is below the 64 tiles of (512, 2048): one split"""
    for M, N, K in ((512, 2048, 6080), (128, 128, 100000), (300, 2048, 10001)):
        run_atb(eng, "tf32", M, N, K, budget=budget, sms=sms, label="budget", seed=budget + K)


@pytest.mark.parametrize("M,N", [(2304, 1280), (4096, 1280), (4096, 2560)])
def test_tn_persistent_waves(eng, sms, M, N):
    """more tiles than SMs: each persistent CTA walks 2 or more tiles (persistent_grid's balanced rounds)"""
    assert -(-M // 128) * -(-N // 128) > sms
    run_tn(eng, "tf32", M, N, 128, beta=1.0, bias=True, label="waves", seed=M + N)


# ---------------------------------------------------------------------------------------------- c) determinism
@pytest.mark.parametrize("mode", ["tf32", "fp32"])
def test_tn_bitwise_reproducible(eng, mode):
    run_tn(eng, mode, 4096, 1280, 300, beta=1.0, bias=True, label="repeat", seed=11, repeat=True)
    run_tn(eng, mode, 257, 65, 300, act=1, label="repeat", seed=12, repeat=True)


@pytest.mark.parametrize("mode", ["tf32", "fp32"])
def test_atb_bitwise_reproducible_with_one_split(eng, sms, mode):
    # one split on both routes: tc splits = min(2 #SM / 64 tiles, ...) > 1, so the budget 40 forces one; the CUDA-core
    # kernel keeps K <= 512 in one split
    run_atb(eng, mode, 512, 2048, 500, budget=40, sms=sms, label="repeat", seed=13, repeat=True)
    assert (G.atb_tc_splits(512, 2048, 500, sms, 40)[0], G.atb_simt_splits(512, 2048, 500, sms)[0]) == (1, 1)
