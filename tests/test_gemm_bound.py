"""The per-element GEMM bound of tests/gemm_ref.py (used by test_gemm_gpu.py) has teeth, without a GPU.

gemm_ref's numpy emulation of each kernel's arithmetic (exact TF32 products accumulated in fp32 per k-block, split partials
added in fp32, the epilogue's bias, then beta C, then tanh) must pass the bound in every case class of test_gemm_gpu.py:
TF32-exact and fp32 operands on the tensor cores, fp32 operands on the CUDA cores, the tanh epilogue near 0 and near +-9,
split-K with random-sign and with non-negative operands up to the option LSTM's K = 608 000.  Each mutant, a plausible kernel
bug, must fail it in the case class that exposes it; the factor it fails by is printed (RATIO lines, pytest -s)."""
import numpy as np
import pytest

import gemm_ref as G

SMS = 132


def _ratio(got, ref, bnd):
    assert np.isfinite(got).all()
    return float((np.abs(got.astype(np.float64) - ref) / bnd).max())


def _operands(rng, shape, kind):
    x = rng.random(shape) if kind == "nonneg" else rng.standard_normal(shape)
    x = x.astype(np.float32)
    return G.tf32(x) if kind in ("exact", "nonneg") else x


def tn_case(name, mutant=None):
    """(ratio, the fp32-only ratio) of one gemm_tn class"""
    rng = np.random.default_rng(sum(map(ord, name)))
    M, N, K, act, beta, tc, kind, scale = {
        "tc_exact": (16, 20, 300, 0, 1.0, True, "exact", 1.0),
        "tc_fp32": (16, 20, 300, 0, 0.0, True, "fp32", 1.0),
        "tc_tanh": (16, 20, 300, 1, 0.5, True, "exact", None),
        "simt": (16, 20, 300, 0, 1.0, False, "fp32", 1.0),
        "simt_tanh": (16, 20, 300, 1, 1.0, False, "fp32", None),
        "tc_epilogue": (16, 20, 64, 0, 1.0, True, "exact", 2.0 ** -6),     # products small beside bias and beta C
    }[name]
    A, B = _operands(rng, (M, K), kind), _operands(rng, (N, K), kind)
    if kind == "fp32":
        A[0], B[0] = G.WITNESS, G.WITNESS
    C0 = rng.standard_normal((M, N)).astype(np.float32)
    bias = rng.standard_normal(N).astype(np.float32)
    if scale is None:      # tanh: pre-activations spread over 0 +- 1e-3 and +-9
        A = G.tf32(A * np.float32(2.0 ** -7))
        bias = np.where(np.arange(N) % 3 == 0, 9.0, np.where(np.arange(N) % 3 == 1, -9.0, 0.0)).astype(np.float32)
        C0 = (C0 * np.float32(1e-3)).astype(np.float32)
    else:
        A = (A * np.float32(scale)).astype(np.float32)
    A64, B64 = A.astype(np.float64), B.astype(np.float64)
    pre = A64 @ B64.T + bias + beta * C0.astype(np.float64)
    ref = np.tanh(pre) if act else pre
    sabs = np.abs(A64) @ np.abs(B64).T
    extra = np.abs(bias) + np.abs(beta * C0.astype(np.float64))
    got = G.emulate_tn(A, B, C0, beta, bias, act, tc, mutant)
    b = G.bound(K, sabs, extra, tc, kind != "fp32", act, ref)
    b32 = G.bound(K, sabs, extra, False, True, act, ref)
    return _ratio(got, ref, b), _ratio(got, ref, b32)


def atb_case(name, mutant=None):
    rng = np.random.default_rng(sum(map(ord, name)))
    M, N, K, tc, kind, budget = {
        "tc_split": (300, 2048, 10001, True, "exact", 0),            # the table gradient's shape: 5 splits of 2 016
        "tc_budget": (512, 2048, 6080, True, "exact", 48),           # under the option stream's budget: 1 split
        "tc_nonneg": (129, 257, 100000, True, "nonneg", 0),          # 44 splits of 2 304
        "tc_c4_dwh": (512, 2048, 608000, True, "nonneg", 0),         # the TF32 option dWh: 4 splits of 152 000
        "simt_split": (300, 2048, 10001, False, "fp32", 0),
        "simt_nonneg": (129, 257, 100000, False, "nonneg", 0),
    }[name]
    m, n = 3, 2                                       # the columns emulated; the split count follows (M, N)
    A, B = _operands(rng, (K, m), kind), _operands(rng, (K, n), kind)
    if kind == "fp32":
        A[:, 0], B[:, 0] = G.WITNESS, G.WITNESS
    C0 = rng.standard_normal((m, n)).astype(np.float32)
    A64, B64 = A.astype(np.float64), B.astype(np.float64)
    ref = C0 + A64.T @ B64
    sabs = np.abs(A64).T @ np.abs(B64)
    got = G.emulate_atb(A, B, C0, tc, SMS, budget, mutant, MN=(M, N))
    nch = G.chain("atb", K, tc, M, N, SMS, budget)
    return _ratio(got, ref, G.bound(nch, sabs, np.abs(C0), tc, kind != "fp32")), None


TN = ("tc_exact", "tc_fp32", "tc_tanh", "simt", "simt_tanh", "tc_epilogue")
ATB = ("tc_split", "tc_budget", "tc_nonneg", "tc_c4_dwh", "simt_split", "simt_nonneg")


def _run(case, mutant=None):
    return tn_case(case, mutant) if case in TN else atb_case(case, mutant)


@pytest.mark.parametrize("case", TN + ATB)
def test_emulation_passes(case):
    r, r32 = _run(case)
    print("RATIO emulation %-12s %.3g" % (case, r))
    assert r <= 1, (case, r)
    if case == "tc_fp32":        # the witness element: TF32 shows beyond the fp32-only bound
        assert r32 > 1, r32


def test_split_mirrors():
    assert G.atb_tc_splits(300, 2048, 10001, SMS) == (5, 2016)
    assert G.atb_tc_splits(512, 2048, 608000, SMS) == (4, 152000)
    assert G.atb_tc_splits(512, 2048, 608000, SMS, budget=48) == (1, 608000)     # budget below the 64 tiles
    assert G.atb_tc_splits(128, 128, 100000, SMS, budget=96) == (95, 1056)
    assert G.atb_simt_splits(512, 2048, 6080, SMS) == (9, 688)


# mutant: the case that exposes it
MUTANTS = {
    "drop_last_kblock": ("tc_exact", "simt"),       # the last partial k-block of K = 300 dropped
    "split_lost": ("tc_split", "tc_nonneg", "tc_c4_dwh", "simt_split", "simt_nonneg"),
    "split_twice": ("tc_split", "tc_nonneg", "tc_c4_dwh", "simt_split", "simt_nonneg"),
    "betac_tf32": ("tc_epilogue",),                 # beta C0 rounded to TF32 in the epilogue
    "bias_tf32": ("tc_epilogue",),                  # the bias rounded to TF32
    "bf16_blocks": ("tc_exact", "tc_split"),        # the accumulator rounded to bf16 after every k-block
    "tf32_on_fp32_route": ("simt", "simt_split"),   # an FP32-route tile contracted on TF32 operands
}


@pytest.mark.parametrize("mutant,case", [(m, c) for m, cs in MUTANTS.items() for c in cs])
def test_mutant_fails(mutant, case):
    r, _ = _run(case, mutant)
    print("RATIO %-18s %-12s %.3g" % (mutant, case, r))
    assert r > 1, (mutant, case, r)
