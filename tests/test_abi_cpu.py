"""CPU-only checks of the drop-in boundary: the C-ABI library loads and exports every symbol
include/rten_b200.h declares, and fails loudly (no fallback) when no H100 is present."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib_path():
    from rten_b200 import _build
    return _build.build()


def header_symbols():
    src = open(os.path.join(ROOT, "include", "rten_b200.h")).read()
    return sorted(set(re.findall(r"\b(rten_b200_[a-z0-9_]+)\s*\(", src)))


def test_header_declares_the_hot_path():
    syms = header_symbols()
    for need in ["rten_b200_gemm", "rten_b200_matmul", "rten_b200_matmul_integer", "rten_b200_conv2d", "rten_b200_conv_integer",
                 "rten_b200_softmax", "rten_b200_layer_norm", "rten_b200_erf", "rten_b200_gelu", "rten_b200_dynamic_quantize_linear",
                 "rten_b200_prepack_b", "rten_b200_ctx_create", "rten_b200_last_error"]:
        assert need in syms


def test_library_exports_every_declared_symbol(lib_path):
    lib = ctypes.CDLL(lib_path)
    for s in header_symbols():
        assert hasattr(lib, s), f"{s} declared in include/rten_b200.h but not exported"


def test_python_binding_covers_the_header(lib_path):
    from rten_b200 import _lib
    assert set(_lib.declared_symbols()) == set(header_symbols())
    _lib.load()


def test_version_and_no_cpu_fallback(lib_path):
    import torch
    from rten_b200 import _lib
    lib = _lib.load()
    assert b"sm_90a" in lib.rten_b200_version()
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    import rten_b200 as rt
    with pytest.raises(rt.OpError) as e:
        rt.Context(0)
    assert e.value.kind == "Cuda"


def test_struct_layout_matches_header(lib_path):
    from rten_b200._lib import RtenConvParams, RtenTensor
    assert ctypes.sizeof(RtenTensor) == 8 + 4 + 4 + 64 + 64 + 4 + 4
    assert ctypes.sizeof(RtenConvParams) == 16 + 4 + 4 + 8 + 8 + 4 + 4


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "rten_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cc")):
                txt = open(os.path.join(dirpath, f), errors="ignore").read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", txt, re.M), f"{f} imports the oracle"
                assert "librten_oracle" not in txt and "rten_oracle.c" not in txt, f"{f} links the oracle"


def test_fastdiv_magic_numbers():
    """The tile decode of umma_gemm.cu divides by launch-time constants with multiply-high + shift (FastDiv::set).
    Same arithmetic restated here: exact for every 0 <= n < 2^31 -- checked on boundary values and random samples."""
    import random

    def magic(d):
        if d == 1:
            return 0, 0
        lg = (d - 1).bit_length()  # ceil(log2(d))
        p = 31 + lg
        return ((1 << p) + d - 1) // d, p - 32

    def fdiv(n, d, mul, shr):
        return n if d == 1 else ((n * mul) >> 32) >> shr

    rnd = random.Random(1234)
    divisors = list(range(1, 300)) + [392, 784, 1568, 3136, 4095, 4096, 4097, 65535, 65536, 100352, 401408, (1 << 31) - 1]
    for d in divisors:
        mul, shr = magic(d)
        assert mul < (1 << 32)
        samples = [0, 1, d - 1, d, d + 1, 2 * d - 1, 2 * d, (1 << 31) - 1, (1 << 31) - d] + [rnd.randrange(1 << 31) for _ in range(200)]
        for n in samples:
            if 0 <= n < (1 << 31):
                assert fdiv(n, d, mul, shr) == n // d, (n, d)


def test_ctypes_signatures_have_the_header_arity():
    """Every prototype of include/rten_b200.h and its ctypes signature in rten_b200/_lib.py take the same number of
    parameters (a silently mismatched arity corrupts the call instead of failing)."""
    from rten_b200 import _lib
    src = open(os.path.join(ROOT, "include", "rten_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", " ", src, flags=re.S)
    protos = dict(re.findall(r"\b(rten_b200_[a-z0-9_]+)\s*\(([^;{]*?)\)\s*;", src, flags=re.S))
    assert set(protos) == set(_lib.declared_symbols())
    for name, params in protos.items():
        params = params.strip()
        n = 0 if params in ("", "void") else len([p for p in params.split(",") if p.strip()])
        assert n == len(_lib._SIGNATURES[name][1]), f"{name}: header has {n} parameters, _lib.py {len(_lib._SIGNATURES[name][1])}"
