"""Build recipe for the sm_90a C-ABI library (in-tree: genrec_b200/libgenrec_b200.so).

nvcc cross-compiles without a GPU.  The .so is a build product (git-ignored); build() makes it in the package directory.
"""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libgenrec_b200.so")
# --use_fast_math: flush-to-zero + approximate div/sqrt.  Without .ftz every ex2.approx / rcp.approx in the SiLU, softmax and
# cross-entropy inner loops carries a 3-instruction denormal fix-up (FSETP + 2 predicated FMUL); the operands are bf16-rounded
# activations, so denormal inputs carry no information here.
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "--use_fast_math",
              "-Xcompiler", "-fPIC", "-shared"]


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(os.path.dirname(HERE), "include", "genrec_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not _stale():
        return LIB
    nvcc = os.environ.get("NVCC", "nvcc")
    cmd = [nvcc, *NVCC_FLAGS, "-o", LIB, *sources()]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
        print(" ".join(cmd), file=sys.stderr)
    subprocess.check_call(cmd, cwd=CSRC)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
