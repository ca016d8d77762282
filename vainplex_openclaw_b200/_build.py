"""In-tree build of libopenclaw_gov.so (nvcc, sm_90a only).  No JIT cache, no pip install."""
from __future__ import annotations

import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libopenclaw_gov.so")
SOURCES = ["capi.cu", "scan_kernels.cu", "span_resolve.cu", "sha256_kernels.cu", "policy_eval.cu", "policy_eval_one.cu", "rulec.cpp", "ruleset_image.cpp"]
HEADERS = ["dev_buffer.h", "kernels.h", "policy_eval.h", "rulec.h", "pike_vm.h", "gram_filter.h", "ruleset_image.h", os.path.join("..", "..", "include", "openclaw_gov.h")]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC,-fvisibility=hidden", "-shared"]


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(os.path.join(CSRC, f)) > t for f in SOURCES + HEADERS)


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile every CUDA/C++ source of the hot path into vainplex_openclaw_b200/libopenclaw_gov.so."""
    if not force and not needs_build():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", LIB] + [os.path.join(CSRC, s) for s in SOURCES]
    subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build(force=True, verbose=True))
