"""The blend forward's fp32 mapped depth (surfel_common.cuh: mapped_depth_fast / mapped_depth_fp32) against the
double-precision mapped_depth it stands in for, over every float the blend can pass it: each bit pattern from 0.2f to
+inf, and every NaN (a NaN depth passes the blend's !(depth < 0.2f) test).  Zero mismatches is the pass condition; the
checkers also count how often the fast path hands over to the DP sequence.

* CPU: the host build of mapped_depth_fp32 (same header, IEEE single with explicit fmaf) against the same DP sequence
  on the host, with every reciprocal the GPU's rcp.approx.ftz can return (the correctly rounded 1/d, its two float
  neighbours, and 0 where 1/d is subnormal).  About a minute of CPU time, spread over the cores with OpenMP.
* GPU: a checker kernel built from the header calls mapped_depth_fast and mapped_depth on the device.
"""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "lara_b200", "csrc")
N_FINITE = 0x7F800000 - 0x3E4CCCCD  # bit patterns of [0.2f, FLT_MAX]
N_NAN = 2 * (0x7FFFFF)               # +NaN and -NaN patterns

_CPU_SRC = r"""
#include "surfel_common.cuh"
#include <math.h>
#include <stdio.h>
#include <string.h>

static float md_ref(float depth) {  // mapped_depth() on the host: fma, multiply and divide in IEEE double
    const double d = (double)depth;
    return (float)(fma(d, 100.0, -(100.0 * 0.2)) / ((100.0 - 0.2) * d));
}
static unsigned bits(float x) { unsigned u; memcpy(&u, &x, 4); return u; }
static float fl(unsigned u) { float x; memcpy(&x, &u, 4); return x; }

int main() {
    unsigned long long bad = 0, fallback = 0, n = 0;
#pragma omp parallel for reduction(+ : bad, fallback, n) schedule(static, 1 << 16)
    for (long long u = 0x3e4ccccdLL; u <= 0x7f800000LL; ++u) {
        const float d = fl((unsigned)u);
        const float ref = md_ref(d);
        const float r0 = 1.0f / d;
        const float rd[4] = {nextafterf(r0, 0.0f), r0, nextafterf(r0, INFINITY), 0.0f};
        for (int k = 0; k < (r0 < 0x1p-126f ? 4 : 3); ++k) {
            float m;
            if (mapped_depth_fp32(d, rd[k], m)) bad += bits(m) != bits(ref);
            else if (k == 1) ++fallback;
        }
        ++n;
    }
    for (unsigned s = 0; s < 2; ++s)  // NaN depths must not take the fast path
        for (unsigned u = 0x7f800001u; u <= 0x7fffffffu; ++u) {
            float m;
            const float d = fl(u | (s << 31));
            if (mapped_depth_fp32(d, 1.0f / d, m)) ++bad;
            ++n;
        }
    printf("checked %llu mismatches %llu fallback %llu\n", n, bad, fallback);
    return 0;
}
"""

_GPU_SRC = r"""
#include "surfel_common.cuh"
#include <stdio.h>

__global__ void check(unsigned long long* out) {
    unsigned long long bad = 0, fallback = 0;
    const unsigned long long n_fin = 0x7f800000ull - 0x3e4ccccdull + 1, n = n_fin + 2ull * 0x7fffffull;
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < n;
         i += (unsigned long long)gridDim.x * blockDim.x) {
        unsigned u;
        if (i < n_fin) u = 0x3e4ccccdu + (unsigned)i;                   // [0.2f, +inf]
        else u = (0x7f800001u + (unsigned)((i - n_fin) >> 1)) | ((unsigned)(i - n_fin) << 31);  // +-NaN
        const float d = __uint_as_float(u);
        float m;
        fallback += !mapped_depth_fp32(d, rcp_approx(d), m);
        bad += __float_as_uint(mapped_depth_fast(d)) != __float_as_uint(mapped_depth(d));
    }
    atomicAdd(out, bad); atomicAdd(out + 1, fallback);
}

int main() {
    unsigned long long* d_out; unsigned long long h[2] = {0, 0};
    if (cudaMalloc(&d_out, sizeof(h)) != cudaSuccess) { printf("no device\n"); return 2; }
    cudaMemset(d_out, 0, sizeof(h));
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    cudaEventRecord(e0);
    check<<<132 * 16, 256>>>(d_out);
    cudaEventRecord(e1);
    cudaError_t err = cudaMemcpy(h, d_out, sizeof(h), cudaMemcpyDeviceToHost);
    float ms = 0; cudaEventElapsedTime(&ms, e0, e1);
    if (err != cudaSuccess) { printf("error %s\n", cudaGetErrorString(err)); return 2; }
    printf("checked %llu mismatches %llu fallback %llu ms %.1f\n",
           0x7f800000ull - 0x3e4ccccdull + 1 + 2ull * 0x7fffffull, h[0], h[1], ms);
    return 0;
}
"""


def _nvcc():
    from lara_b200 import build
    return build._nvcc()


def _build_and_run(tmp_path, src, name, flags, timeout):
    path = tmp_path / (name + ".cu")
    path.write_text(src)
    exe = str(tmp_path / name)
    subprocess.run([_nvcc(), "-O2", "-std=c++17", "-I", CSRC, "-gencode", "arch=compute_90a,code=sm_90a"] + flags +
                   [str(path), "-o", exe], check=True, timeout=600)
    out = subprocess.run([exe], check=True, capture_output=True, text=True, timeout=timeout).stdout
    m = re.search(r"checked (\d+) mismatches (\d+) fallback (\d+)", out)
    assert m, out
    print(out.strip())
    return int(m.group(1)), int(m.group(2)), int(m.group(3))


def _check_counts(n, bad, fallback):
    assert n == N_FINITE + 1 + N_NAN
    assert bad == 0
    # the DP fallback: NaN and inf always, finite depths within the tolerance of a rounding midpoint (~4e3)
    assert fallback - (N_NAN + 1) < 10_000


def test_mapped_depth_fast_path_cpu_exhaustive(tmp_path):
    n, bad, fallback = _build_and_run(tmp_path, _CPU_SRC, "md_cpu", ["-Xcompiler", "-fopenmp,-ffp-contract=off", "-lgomp"],
                                      timeout=1800)
    assert n == N_FINITE + 1 + N_NAN and bad == 0
    assert fallback < 10_000  # finite depths (and inf) only: NaNs are counted as mismatches if they pass


@pytest.mark.gpu
def test_mapped_depth_fast_path_gpu_exhaustive(tmp_path, cuda_device):
    n, bad, fallback = _build_and_run(tmp_path, _GPU_SRC, "md_gpu", [], timeout=600)
    _check_counts(n, bad, fallback)
