// fixed_sums.cuh -- the fixed summation orders that keep the fused ops' sums bit-reproducible (DESIGN §3.13), and the
// fp32 warp sum.  Everything here has internal linkage: each translation unit compiles its own copy.
//
// Order A, part_sums: element e of the n elements is sum over p < nparts of (double)parts[p * stride + e], added in
//   p order in fp64 and rounded once to the output type.  The elements go to the (dst, count) segments in turn.
// Order B, warp_strided_sum: one warp sums n doubles read at a stride, lane l the terms l, l + 32, ... in that order,
//   then an xor butterfly.  Every lane holds the total.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

namespace srf {
namespace {

constexpr int kMaxSumSegs = 6;

template <typename T>
struct SumSeg { T* dst; int n; };

template <typename T>
SumSeg<T> seg(T* dst, int n) { return SumSeg<T>{dst, n}; }

template <typename T>
struct SumSegs { SumSeg<T> s[kMaxSumSegs]; };   // unused entries have n = 0

template <typename TI, typename TO>
__global__ void part_sums_kernel(const TI* parts, int nparts, size_t stride, int n, const SumSegs<TO> segs) {
    int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    double s = 0.0;
    int p = 0;
    for (; p + 16 <= nparts; p += 16) {     // 16 loads in flight before their adds, which stay in p order
        TI v[16];
#pragma unroll
        for (int k = 0; k < 16; ++k) v[k] = parts[(size_t)(p + k) * stride + e];
#pragma unroll
        for (int k = 0; k < 16; ++k) s += (double)v[k];
    }
    for (; p < nparts; ++p) s += (double)parts[(size_t)p * stride + e];
#pragma unroll
    for (int k = 0; k < kMaxSumSegs; ++k) {
        if (e < segs.s[k].n) { segs.s[k].dst[e] = (TO)s; return; }
        e -= segs.s[k].n;
    }
}

// order A over the elements of the segments, which lie back to back in each row of parts
template <typename TI, typename TO, typename... Rest>
void part_sums(cudaStream_t stream, const TI* parts, int nparts, size_t stride, SumSeg<TO> first, Rest... rest) {
    static_assert(1 + sizeof...(Rest) <= kMaxSumSegs, "part_sums: too many segments");
    const SumSegs<TO> segs = {{first, rest...}};
    const int n = (first.n + ... + rest.n);
    part_sums_kernel<TI, TO><<<(n + 255) / 256, 256, 0, stream>>>(parts, nparts, stride, n, segs);
}

// order B; call with the whole warp
__device__ __forceinline__ double warp_strided_sum(const double* src, int n, int stride) {
    double s = 0.0;
    for (int i = threadIdx.x & 31; i < n; i += 32) s += src[(size_t)i * stride];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    return s;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

}  // namespace
}  // namespace srf
