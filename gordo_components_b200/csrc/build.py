"""
Builds libgordo_b200.so (the C-ABI library, include/gordo_b200.h) in-tree with nvcc for the H100 (sm_90a).
Cross-compiles without a GPU; the .so and the object files are build products, ignored by git.

    python gordo_components_b200/csrc/build.py [--force] [--verbose]
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "libgordo_b200.so")
OBJ = os.path.join(HERE, "build")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
SOURCES = ["gb_api.cu", "ffae_infer_fma.cu", "ffae_infer_small.cu", "ffae_infer_tc.cu", "anomaly_reduce.cu", "threshold_pair.cu", "smooth.cu", "gather.cu", "ffae_fit.cu", "ffae_fit_drop.cu", "ffae_fit_group.cu", "lstm_infer.cu", "lstm_infer_tc.cu", "lstm_fit.cu", "lstm_fit_tc.cu"]
HEADERS = ["gb_common.cuh", "ffae_fit_body.cuh", "ffae_fit_kernels.cuh", "gb_sm90.cuh", "lstm_fit_common.cuh", "postprocess.cuh", os.path.join("..", "..", "include", "gordo_b200.h")]
NVCC_FLAGS = [
    *ARCH, "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: the CUDA extension cannot be built (there is no CPU fallback)")


def _digest() -> str:
    h = hashlib.sha256()
    for f in SOURCES + HEADERS:
        p = os.path.join(HERE, f)
        if os.path.exists(p):
            h.update(open(p, "rb").read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    stamp = os.path.join(OBJ, "stamp")
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read() == dig:
        return LIB
    os.makedirs(OBJ, exist_ok=True)
    nvcc = _nvcc()
    srcs = [s for s in SOURCES if os.path.exists(os.path.join(HERE, s))]

    def compile_one(src):
        obj = os.path.join(OBJ, src.replace(".cu", ".o"))
        cmd = [nvcc, *NVCC_FLAGS, "-c", os.path.join(HERE, src), "-o", obj]
        if verbose:
            cmd[1:1] = ["-Xptxas", "-v"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            sys.stderr.write(r.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(compile_one, srcs))
    cmd = [nvcc, "-shared", *ARCH, "-o", LIB, *objs, "-Xcompiler", "-fPIC"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    with open(stamp, "w") as f:
        f.write(dig)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
