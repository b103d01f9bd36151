"""CPU-only: every `__global__` kernel defined in rten_b200/csrc (*.cu and *.cuh) is in exactly one by-name table -- the
row kernels, glue, elementwise math and operand staging of rowops.cu, TopK / arg-reduce, the mask kernels, the
depthwise / GroupNorm / Resize / Concat / ReduceSum / rotary table, the single-query attention / MatMulNBits table,
the prefill attention table, the GRU / LSTM table and the wgmma GEMM / wide-tile / halo table.  Each of those tables is kept equal to the compiled instances and
checked kernel by kernel, bit for bit, by its GPU test.  A kernel added without a by-name test fails here before any GPU
time is spent.

Two kernels are named only by their own operator's tests (`AD_HOC`: the encoder attention kernel and the multi-GPU range
exchange).  For those this file checks only that the test module's source names
the kernel -- a weaker guarantee than a table: nothing here proves the module asserts that the kernel ran, or covers
every instance."""
import glob
import os
import re

import test_gpu_conv_norm_resize_kernels as ck
import test_gpu_decode_step_kernels as dk
import test_gpu_elementwise_math as em
import test_gpu_glue_kernels as gk
import test_gpu_mask_ops as mo
import test_gpu_prefill_attention_kernels as pk
import test_gpu_rnn_kernels as nk
import test_gpu_row_kernels as rk
import test_gpu_select as sel
import test_gpu_staging_kernels as sk
import test_gpu_wgmma_kernels as wk

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "rten_b200", "csrc")

# kernel -> the test module that names it (and checks, in its own way, that it runs)
AD_HOC = {
    "attn_fused_kernel": "test_gpu_attention_encoder",
    "peer_minmax_kernel": "test_gpu_sharded",
}


def tables():
    return {"row kernels": set(rk.VARIANTS) | set(rk.GENERIC), "glue": set(gk.VARIANTS), "elementwise math": set(em.KERNELS),
            "staging": set(sk.VARIANTS), "select": set(sel.KERNELS), "masks": set(mo.VARIANTS),
            "conv / norm / resize": set(ck.VARIANTS), "decode step": set(dk.VARIANTS),
            "prefill attention": set(pk.VARIANTS), "GRU / LSTM": set(nk.VARIANTS),
            "wgmma GEMM / halo": set(wk.VARIANTS)}


_GLOBAL = re.compile(r"\b__global__\b")
_IDENT = re.compile(r"\s*(\w+)")


def _strip_comments(src):
    return re.sub(r"//[^\n]*|/\*.*?\*/", " ", src, flags=re.S)


def _skip_parens(src, i):
    """the index just past the parenthesised group that starts at src[i] == '('"""
    depth = 0
    for j in range(i, len(src)):
        depth += {"(": 1, ")": -1}.get(src[j], 0)
        if depth == 0:
            return j + 1
    raise ValueError("unbalanced parentheses")


def global_kernels(src):
    """the names of the `__global__` functions defined in CUDA source text: after `__global__`, any of `void`,
    `__launch_bounds__(...)` (parentheses nested to any depth) and `__cluster_dims__(...)`, across lines; the name is
    the identifier before the parameter list"""
    src = _strip_comments(src)
    names = set()
    for m in _GLOBAL.finditer(src):
        i, last = m.end(), None
        while True:
            t = _IDENT.match(src, i)
            if not t:
                break
            i = t.end()
            while src[i].isspace():
                i += 1
            if t.group(1) in ("__launch_bounds__", "__cluster_dims__") and src[i] == "(":
                i = _skip_parens(src, i)
                continue
            last = t.group(1)
            if src[i] == "(":
                break
        if last is not None and src[i] == "(":
            names.add(last)
    return names


def library_kernels(paths=None):
    """{kernel: the sources that define it} over rten_b200/csrc/*.cu and *.cuh (or `paths`)"""
    paths = paths or sorted(glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cuh")))
    out = {}
    for p in paths:
        with open(p) as f:
            for n in global_kernels(f.read()):
                out.setdefault(n, []).append(os.path.basename(p))
    return out


def unlisted(paths=None):
    """(kernels in no by-name table and not named ad hoc, kernels in more than one table, ad-hoc kernels whose test
    module does not name them)"""
    ts = tables()
    names = library_kernels(paths)
    homes = {n: [t for t, ks in ts.items() if n in ks] for n in names}
    missing = sorted(n for n, h in homes.items() if not h and n not in AD_HOC)
    twice = sorted(n for n, h in homes.items() if len(h) + (n in AD_HOC) > 1)
    unnamed = []
    for n in sorted(set(names) & set(AD_HOC)):
        with open(os.path.join(HERE, AD_HOC[n] + ".py")) as f:
            if not re.search(rf"\b{n}\b", f.read()):
                unnamed.append((n, AD_HOC[n]))
    return missing, twice, unnamed


def test_every_kernel_is_tested_by_name():
    names = library_kernels()
    assert len(names) >= 80, f"the parser found only {sorted(names)}"
    missing, twice, unnamed = unlisted()
    assert not missing, f"kernels no by-name test covers: {[(n, names[n]) for n in missing]}"
    assert not twice, f"kernels in more than one by-name table: {twice}"
    assert not unnamed, f"kernels their test module does not name: {unnamed}"
    stale = sorted(set(AD_HOC) - set(names))
    assert not stale, f"AD_HOC names kernels the library no longer defines: {stale}"


def test_the_parser_reads_every_declaration_form():
    src = """
    template <int DH, int NW>
    __global__ void __launch_bounds__(NW * 32, DH == 64 ? (NW == 8 ? 3 : 4) : 1) nested_kernel(const P p) {}
    __global__ void __launch_bounds__(256)
    split_kernel(const float* x,
                 float* y) {}
    __global__ void plain_kernel(int* mm) {}
    // __global__ void commented_kernel(int* mm) {}
    __global__ void __launch_bounds__(AP_THREADS, 1)
    attn_like_kernel(const __grid_constant__ CUtensorMap tma_q) {}
    """
    assert global_kernels(src) == {"nested_kernel", "split_kernel", "plain_kernel", "attn_like_kernel"}


def test_the_completeness_check_reports_a_new_kernel(tmp_path):
    for name in ("rowops.cu", "depthwise.cu", "skinny.cu", "umma_kernel.cuh"):
        with open(os.path.join(CSRC, name)) as f:
            src = f.read()
        extra = tmp_path / name
        extra.write_text(src + "\nnamespace rtb {\ntemplate <int N>\n__global__ void __launch_bounds__(N * 32, N == 4 ? (N > 2 ? 2 : 1) : 1)\n"
                               "staged_new_kernel(const float* x) {}\n}\n")
        assert unlisted([str(extra)])[0] == ["staged_new_kernel"], name


def test_the_completeness_check_reports_a_dropped_table_row(monkeypatch):
    monkeypatch.delitem(ck.VARIANTS, "gn_stats_kernel")
    assert unlisted([os.path.join(CSRC, "groupnorm.cu")])[0] == ["gn_stats_kernel"]
