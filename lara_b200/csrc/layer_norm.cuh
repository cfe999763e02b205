// layer_norm.cuh -- the residual add + LayerNorm kernels shared by the VolTransformer (vol_transformer.cu, C <= 512)
// and the image encoder (image_encoder.cu, C in {384, 768}), a warp per row of C channels, C / 32 values per lane:
//   ln_fwd_kernel<J>  y = a + b, the mean, the centred variance (two passes over the registers), n = LN(y).
//   ln_bwd_kernel<J>  a CTA per block of 64 rows: recomputes the statistics from y, writes dL/da = dL/dy + the vjp,
//                     and the block's dgamma / dbeta partials, its warps added in warp order.
//   ln_backward<J>    the backward launch and the partials summed over the blocks in block order in fp64
//                     (part_sums, fixed_sums.cuh).
// J is the largest C / 32 the instantiation takes.  Everything here has internal linkage.
#pragma once
#include <string.h>

#include "fixed_sums.cuh"

namespace srf {
namespace {

constexpr int kLnWarps = 8;
constexpr int kLnRows = 64;              // rows per CTA of the LayerNorm backward (one partial each)

struct LnArgs {
    int rows, C;
    float eps;
    const float *a, *b, *gamma, *beta, *ys, *gn, *gy;    // ys: the backward's y
    float *y, *n, *ga, *parts;
};

// mean and 1 / sqrt(var + eps) of the lane's nj values of a row of C
template <int J>
__device__ __forceinline__ void ln_stats(const float* y, int nj, int C, float eps, float& mean, float& rstd) {
    float s = 0.0f;
#pragma unroll
    for (int j = 0; j < J; ++j)
        if (j < nj) s += y[j];
    mean = warp_sum(s) / (float)C;
    float v = 0.0f;
#pragma unroll
    for (int j = 0; j < J; ++j)
        if (j < nj) { const float d = y[j] - mean; v = fmaf(d, d, v); }
    rstd = 1.0f / sqrtf(warp_sum(v) / (float)C + eps);
}

template <int J>
__global__ void __launch_bounds__(kLnWarps * 32) ln_fwd_kernel(LnArgs a) {
    const int lane = threadIdx.x & 31, row = blockIdx.x * kLnWarps + (threadIdx.x >> 5);
    if (row >= a.rows) return;
    const int C = a.C, nj = C / 32;
    const size_t base = (size_t)row * C + lane;
    float y[J];
#pragma unroll
    for (int j = 0; j < J; ++j)
        if (j < nj) y[j] = a.b ? __ldg(a.a + base + 32 * j) + __ldg(a.b + base + 32 * j) : __ldg(a.a + base + 32 * j);
    float mean, rstd;
    ln_stats<J>(y, nj, C, a.eps, mean, rstd);
#pragma unroll
    for (int j = 0; j < J; ++j) {
        if (j >= nj) continue;
        const int c = lane + 32 * j;
        if (a.y) a.y[base + 32 * j] = y[j];
        a.n[base + 32 * j] = fmaf((y[j] - mean) * rstd, __ldg(a.gamma + c), __ldg(a.beta + c));
    }
}

template <int J>
__global__ void __launch_bounds__(kLnWarps * 32) ln_bwd_kernel(LnArgs a) {
    __shared__ float acc_s[2][J * 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, C = a.C, nj = C / 32;
    const int r0 = blockIdx.x * kLnRows, r1 = min(r0 + kLnRows, a.rows);
    float gam[J], dg[J], db[J];
#pragma unroll
    for (int j = 0; j < J; ++j) {
        gam[j] = j < nj ? __ldg(a.gamma + lane + 32 * j) : 0.0f;
        dg[j] = 0.0f;
        db[j] = 0.0f;
    }
    for (int row = r0 + warp; row < r1; row += kLnWarps) {
        const size_t base = (size_t)row * C + lane;
        float y[J], g[J];
#pragma unroll
        for (int j = 0; j < J; ++j)
            if (j < nj) { y[j] = __ldg(a.ys + base + 32 * j); g[j] = __ldg(a.gn + base + 32 * j); }
        float mean, rstd;
        ln_stats<J>(y, nj, C, a.eps, mean, rstd);
        float s1 = 0.0f, s2 = 0.0f;
#pragma unroll
        for (int j = 0; j < J; ++j) {
            if (j >= nj) continue;
            y[j] = (y[j] - mean) * rstd;                  // the normalised value from here on
            dg[j] = fmaf(g[j], y[j], dg[j]);
            db[j] += g[j];
            g[j] *= gam[j];
            s1 += g[j];
            s2 = fmaf(g[j], y[j], s2);
        }
        const float m1 = warp_sum(s1) / (float)C, m2 = warp_sum(s2) / (float)C;
#pragma unroll
        for (int j = 0; j < J; ++j) {
            if (j >= nj) continue;
            const float d = rstd * (g[j] - m1 - y[j] * m2);
            a.ga[base + 32 * j] = a.gy ? __ldg(a.gy + base + 32 * j) + d : d;
        }
    }
    // the warps' sums, added in warp order
    for (int w = 0; w < kLnWarps; ++w) {
        if (warp == w) {
#pragma unroll
            for (int j = 0; j < J; ++j) {
                if (j >= nj) continue;
                const int c = lane + 32 * j;
                acc_s[0][c] = w ? acc_s[0][c] + dg[j] : dg[j];
                acc_s[1][c] = w ? acc_s[1][c] + db[j] : db[j];
            }
        }
        __syncthreads();
    }
    float* part = a.parts + (size_t)blockIdx.x * 2 * C;
    for (int e = threadIdx.x; e < 2 * C; e += kLnWarps * 32) part[e] = acc_s[e / C][e % C];
}

// bytes of the dgamma / dbeta partials of a backward over `rows` rows
size_t ln_parts_bytes(int rows, int C) {
    const size_t nparts = ((size_t)rows + kLnRows - 1) / kLnRows;
    return sizeof(float) * 2 * (size_t)C * (nparts ? nparts : 1);
}

template <int J>
void ln_forward(cudaStream_t stream, int rows, int C, float eps, const float* a, const float* b, const float* gamma,
                const float* beta, float* y, float* n) {
    if (rows == 0) return;
    LnArgs la;
    memset(&la, 0, sizeof(la));
    la.rows = rows; la.C = C; la.eps = eps; la.a = a; la.b = b; la.gamma = gamma; la.beta = beta; la.y = y; la.n = n;
    const unsigned grid = (unsigned)((rows + kLnWarps - 1) / kLnWarps);
    ln_fwd_kernel<J><<<grid, kLnWarps * 32, 0, stream>>>(la);
}

// the backward over `rows` rows with its partials in `parts` (ln_parts_bytes), then d_gamma, d_beta
template <int J>
void ln_backward(cudaStream_t stream, int rows, int C, float eps, const float* y, const float* gamma, const float* gn,
                 const float* gy, float* parts, float* ga, float* d_gamma, float* d_beta) {
    const int nparts = (rows + kLnRows - 1) / kLnRows;
    if (nparts > 0) {
        LnArgs la;
        memset(&la, 0, sizeof(la));
        la.rows = rows; la.C = C; la.eps = eps; la.ys = y; la.gamma = gamma; la.gn = gn; la.gy = gy;
        la.ga = ga; la.parts = parts;
        ln_bwd_kernel<J><<<(unsigned)nparts, kLnWarps * 32, 0, stream>>>(la);
    }
    part_sums(stream, static_cast<const float*>(parts), nparts, 2 * (size_t)C, seg(d_gamma, C), seg(d_beta, C));
}

}  // namespace
}  // namespace srf
