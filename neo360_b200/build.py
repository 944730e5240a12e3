"""Builds libneo360_b200.so in-tree with nvcc for sm_90a (no torch headers: the library is a plain C ABI)."""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libneo360_b200.so")
SOURCES = ["scene.cu", "sampling.cu", "field_fp32.cu", "field_tc.cu", "render.cu", "vanilla.cu", "mip.cu", "gemm_tc.cu", "encoder.cu", "metrics.cu", "det.cu", "lpips.cu", "field_train.cu", "dense_train.cu", "pixelnerf.cu", "mesh.cu"]
FLAGS = ["-shared", "-Xcompiler", "-fPIC", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3",
         "-std=c++17", "--threads", "4"]


def _stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "neo360_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not _stale():
        return LIB
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found; libneo360_b200.so must be prebuilt")
    tmp = f"{LIB}.{os.getpid()}.tmp"      # per process: ranks that decide to build at the same time do not write into each other's file
    cmd = [nvcc] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", tmp] + [os.path.join(CSRC, s) for s in SOURCES]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        if os.path.exists(tmp):
            os.remove(tmp)
        raise RuntimeError("nvcc failed:\n" + res.stdout + res.stderr)
    os.replace(tmp, LIB)   # atomic: a concurrent reader never sees a half-written library
    if verbose:
        print(res.stderr)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
