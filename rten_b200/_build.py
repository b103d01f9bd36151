"""Build librten_b200.so (sm_90a only) in-tree with nvcc.  No torch involved: the library is a plain
CUDA runtime shared object behind the C ABI of include/rten_b200.h."""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "librten_b200.so")
SOURCES = ["umma_gemm.cu", "umma_halo.cu", "rowops.cu", "groupnorm.cu", "reduce.cu", "topk.cu", "depthwise.cu", "resize.cu", "skinny.cu", "attn_fused.cu", "attn_prefill.cu", "nbits.cu", "rotary.cu", "rnn.cu", "masks.cu", "api_core.cu", "api_ops.cu", "api_conv.cu", "api_rows.cu", "api_fused.cu", "api_attention.cu", "api_rnn.cu", "api_masks.cu", "onnx_reader.cu", "model.cu", "comm.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "--cudart", "static",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc")):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def _stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "rten_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not _stale():
        return LIB
    nvcc = _nvcc()
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    procs = []
    objs = []
    env = dict(os.environ)
    # the image's CC/CXX may point at a wrapper gcc; let nvcc use the system host compiler
    for src in SOURCES:
        obj = os.path.join(objdir, src.replace(".cu", ".o"))
        objs.append(obj)
        cmd = [nvcc, *NVCC_FLAGS, "-ccbin", "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++",
               "-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, env=env)))
    for src, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode != 0:
            sys.stderr.write(out.decode())
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}")
    cmd = [nvcc, "-shared", "--cudart", "static", "-ccbin", "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++",
           "-o", LIB, *objs, "-Xlinker", "--exclude-libs,ALL", "-lpthread", "-ldl", "-lrt"]
    subprocess.check_call(cmd, env=env)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
