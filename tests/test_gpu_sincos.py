"""GPU: sincosf gives the same bits as sinf and cosf for every fp32 input.

The tensor-core field kernel (csrc/field_tc.cu, stage_items) computes each positional-encoding pair with one sincosf call where it
used to call sinf and cosf separately; its fp16 operands stay the same only if the two forms agree bit for bit.  One kernel evaluates
all 2^32 bit patterns, compiled with the library's own nvcc flags (neo360_b200/build.py), and counts the inputs where either result
differs (NaN results compared by their bits as well).
"""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import pytest

from neo360_b200 import build as B

pytestmark = pytest.mark.gpu

SRC = r"""
#include <cstdint>
#include <cuda_runtime.h>

__global__ void sincos_vs_sin_cos(unsigned long long* mismatches, unsigned int* first) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    unsigned long long bad = 0;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < (1ull << 32); i += stride) {
        const float a = __uint_as_float((unsigned int)i);
        float s, c;
        sincosf(a, &s, &c);
        if (__float_as_uint(s) != __float_as_uint(sinf(a)) || __float_as_uint(c) != __float_as_uint(cosf(a))) {
            ++bad;
            atomicMin(first, (unsigned int)i);
        }
    }
    if (bad) atomicAdd(mismatches, bad);
}

// returns 0 and the number of mismatching inputs (and the smallest such bit pattern, 0xffffffff if none), or a CUDA error code
extern "C" int run_sincos_check(unsigned long long* mismatches, unsigned int* first) {
    unsigned long long* d_bad = nullptr;
    unsigned int* d_first = nullptr;
    cudaError_t e = cudaMalloc(&d_bad, sizeof(*d_bad));
    if (e == cudaSuccess) e = cudaMalloc(&d_first, sizeof(*d_first));
    if (e == cudaSuccess) e = cudaMemset(d_bad, 0, sizeof(*d_bad));
    if (e == cudaSuccess) e = cudaMemset(d_first, 0xff, sizeof(*d_first));
    if (e == cudaSuccess) {
        sincos_vs_sin_cos<<<132 * 16, 256>>>(d_bad, d_first);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e == cudaSuccess) e = cudaMemcpy(mismatches, d_bad, sizeof(*d_bad), cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) e = cudaMemcpy(first, d_first, sizeof(*d_first), cudaMemcpyDeviceToHost);
    cudaFree(d_bad);
    cudaFree(d_first);
    return (int)e;
}
"""


def test_sincosf_matches_sinf_cosf_for_every_float():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    with tempfile.TemporaryDirectory(prefix="neo360_sincos_") as d:
        src, lib = os.path.join(d, "sincos_check.cu"), os.path.join(d, "sincos_check.so")
        with open(src, "w") as f:
            f.write(SRC)
        flags = [x for x in B.FLAGS if x not in ("--threads", "4")]
        res = subprocess.run([nvcc] + flags + ["-o", lib, src], capture_output=True, text=True)
        assert res.returncode == 0, res.stdout + res.stderr
        so = C.CDLL(lib)
        bad, first = C.c_ulonglong(0), C.c_uint(0)
        rc = so.run_sincos_check(C.byref(bad), C.byref(first))
        assert rc == 0, f"CUDA error {rc}"
        print(f"sincosf vs sinf / cosf over 2^32 inputs: {bad.value} mismatches")
        assert bad.value == 0, f"{bad.value} inputs differ, the first is 0x{first.value:08x}"
