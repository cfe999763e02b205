// vol_transformer.cu -- the fused parts of LaRa's VolTransformer blocks (GroupAttBlock.forward,
// lightning/network.py:81-102, and the tail of VolTransformer.forward, :152-164) on a channels-last volume, DESIGN
// §3.19.  The C entries of include/surfel_vol_transformer.h are defined here.  The projections, the MLP and the
// (de)convolutions stay with cuBLAS / cuDNN.
//
// Group cross-attention, a CTA per (group, slice of Hs heads), one thread per (query, head) of the slice:
//   ga_fwd_kernel   the thread reads its query's D columns (float4), finds the maximum score over the S keys, then
//                   sums exp(s - max) and exp(s - max) v in key order and writes o = sum / sum of weights.
//   ga_bwd_kernel   recomputes the maximum, the sum and Di = sum_j P_j (dO . v_j) per thread, then per key j forms
//                   dS_j = P_j (dO . v_j - Di), adds dS_j k_j into its dq, and stages P_j dO and dS_j q in shared
//                   memory; after a barrier the CTA sums the staged rows over the bs^3 queries in query order into
//                   dv[G, j] and dk[G, j] of its heads.  No atomics: every output element has one writer.
// Residual add + LayerNorm, a warp per row of C <= 512 channels (C / 32 values per lane):
//   ln_fwd_kernel   y = a + b, the mean, the centred variance (two passes over the registers), n = LN(y).
//   ln_bwd_kernel   a CTA per block of 64 rows: recomputes the statistics from y, writes dL/da = dL/dy + the vjp,
//                   and the block's dgamma / dbeta partials, its warps added in warp order.
//   part_sums_kernel  the partials summed over the blocks in block order in fp64 (fixed_sums.cuh).
#include <math.h>
#include <string.h>

#include "../../include/surfel_vol_transformer.h"
#include "fixed_sums.cuh"
#include "surfel_kernels.h"

namespace srf {
namespace {

constexpr int kGaMaxThreadCols = 4096;   // threads x D of an attention CTA: 2 x 16 KB of backward staging
constexpr int kGaMaxS = 4096;
constexpr int kLnWarps = 8;
constexpr int kLnRows = 64;              // rows per CTA of the LayerNorm backward (one partial each)
constexpr int kLnMaxJ = 16;              // C <= 512

struct GaArgs {
    int R, g, bs, nq, S, C, H, Hs;
    float scale;
    const float *q, *k, *v, *go;
    float *o, *gq, *gk, *gv;
};

// channels-last row of query l (in unfold order) of group G
__device__ __forceinline__ size_t ga_voxel(const GaArgs& a, int G, int l) {
    const int g = a.g, bs = a.bs, R = a.R, g3 = g * g * g;
    const int b = G / g3, gi = G % g3;
    const int z = (gi / (g * g)) * bs + l / (bs * bs), y = ((gi / g) % g) * bs + (l / bs) % bs, x = (gi % g) * bs + l % bs;
    return (((size_t)b * R + z) * R + y) * R + x;
}

template <int D>
__device__ __forceinline__ void load_row(const float* p, float* r) {
#pragma unroll
    for (int i = 0; i < D; i += 4) {
        const float4 t = __ldg(reinterpret_cast<const float4*>(p + i));
        r[i] = t.x; r[i + 1] = t.y; r[i + 2] = t.z; r[i + 3] = t.w;
    }
}

template <int D>
__device__ __forceinline__ void store_row(float* p, const float* r, float s) {
#pragma unroll
    for (int i = 0; i < D; i += 4)
        *reinterpret_cast<float4*>(p + i) = make_float4(r[i] * s, r[i + 1] * s, r[i + 2] * s, r[i + 3] * s);
}

template <int D>
__device__ __forceinline__ float dot_row(const float* x, const float* p) {
    float s = 0.0f;
#pragma unroll
    for (int i = 0; i < D; i += 4) {
        const float4 t = __ldg(reinterpret_cast<const float4*>(p + i));
        s = fmaf(x[i], t.x, s); s = fmaf(x[i + 1], t.y, s); s = fmaf(x[i + 2], t.z, s); s = fmaf(x[i + 3], t.w, s);
    }
    return s;
}

// the thread's (group, head, query row): G, its head h, the query's row n
struct GaThread { int G, h0, hl, l; size_t n; };

__device__ __forceinline__ GaThread ga_thread(const GaArgs& a) {
    const int ns = a.H / a.Hs;
    GaThread t;
    t.G = blockIdx.x / ns;
    t.h0 = (blockIdx.x % ns) * a.Hs;
    t.hl = threadIdx.x % a.Hs;
    t.l = threadIdx.x / a.Hs;
    t.n = ga_voxel(a, t.G, t.l);
    return t;
}

template <int D>
__global__ void __launch_bounds__(256) ga_fwd_kernel(GaArgs a) {
    const GaThread t = ga_thread(a);
    const int C = a.C, col = (t.h0 + t.hl) * D;
    float q[D], acc[D];
    load_row<D>(a.q + t.n * C + col, q);
    const float* kb = a.k + (size_t)t.G * a.S * C + col;
    const float* vb = a.v + (size_t)t.G * a.S * C + col;
    float m = -INFINITY;
    for (int j = 0; j < a.S; ++j) m = fmaxf(m, dot_row<D>(q, kb + (size_t)j * C) * a.scale);
    float sum = 0.0f;
#pragma unroll
    for (int i = 0; i < D; ++i) acc[i] = 0.0f;
    for (int j = 0; j < a.S; ++j) {
        const float e = expf(dot_row<D>(q, kb + (size_t)j * C) * a.scale - m);
        sum += e;
        const float* vr = vb + (size_t)j * C;
#pragma unroll
        for (int i = 0; i < D; i += 4) {
            const float4 w = __ldg(reinterpret_cast<const float4*>(vr + i));
            acc[i] = fmaf(e, w.x, acc[i]); acc[i + 1] = fmaf(e, w.y, acc[i + 1]);
            acc[i + 2] = fmaf(e, w.z, acc[i + 2]); acc[i + 3] = fmaf(e, w.w, acc[i + 3]);
        }
    }
    store_row<D>(a.o + t.n * C + col, acc, 1.0f / sum);
}

template <int D>
__global__ void __launch_bounds__(256) ga_bwd_kernel(GaArgs a) {
    extern __shared__ __align__(16) float stage[];         // [2][threads][D]: P dO, then dS q
    const GaThread t = ga_thread(a);
    const int C = a.C, col = (t.h0 + t.hl) * D, nt = blockDim.x, tid = threadIdx.x;
    float q[D], go[D], gq[D];
    load_row<D>(a.q + t.n * C + col, q);
    load_row<D>(a.go + t.n * C + col, go);
    const float* kb = a.k + (size_t)t.G * a.S * C + col;
    const float* vb = a.v + (size_t)t.G * a.S * C + col;
    float m = -INFINITY;
    for (int j = 0; j < a.S; ++j) m = fmaxf(m, dot_row<D>(q, kb + (size_t)j * C) * a.scale);
    float sum = 0.0f, pd = 0.0f;
    for (int j = 0; j < a.S; ++j) {
        const float e = expf(dot_row<D>(q, kb + (size_t)j * C) * a.scale - m);
        sum += e;
        pd = fmaf(e, dot_row<D>(go, vb + (size_t)j * C), pd);
    }
    const float inv = 1.0f / sum, di = pd * inv;
#pragma unroll
    for (int i = 0; i < D; ++i) gq[i] = 0.0f;
    const int cols = a.Hs * D;
    float* gk_row = a.gk + (size_t)t.G * a.S * C + t.h0 * D;
    float* gv_row = a.gv + (size_t)t.G * a.S * C + t.h0 * D;
    for (int j = 0; j < a.S; ++j) {
        const float* kr = kb + (size_t)j * C;
        const float p = expf(dot_row<D>(q, kr) * a.scale - m) * inv;
        const float ds = p * (dot_row<D>(go, vb + (size_t)j * C) - di);
#pragma unroll
        for (int i = 0; i < D; i += 4) {
            const float4 w = __ldg(reinterpret_cast<const float4*>(kr + i));
            gq[i] = fmaf(ds, w.x, gq[i]); gq[i + 1] = fmaf(ds, w.y, gq[i + 1]);
            gq[i + 2] = fmaf(ds, w.z, gq[i + 2]); gq[i + 3] = fmaf(ds, w.w, gq[i + 3]);
        }
        store_row<D>(stage + (size_t)tid * D, go, p);
        store_row<D>(stage + (size_t)(nt + tid) * D, q, ds);
        __syncthreads();
        // thread (l, hl) staged at row l Hs + hl: the column sums over l, in query order
        for (int e = tid; e < 2 * cols; e += nt) {
            const int arr = e / cols, c = e % cols, hl = c / D, d = c % D;
            const float* src = stage + (size_t)arr * nt * D + hl * D + d;
            float s = 0.0f;
            for (int l = 0; l < a.nq; ++l) s += src[(size_t)l * a.Hs * D];
            if (arr) gk_row[(size_t)j * C + c] = s * a.scale;
            else gv_row[(size_t)j * C + c] = s;
        }
        __syncthreads();
    }
    store_row<D>(a.gq + t.n * C + col, gq, a.scale);
}

struct LnArgs {
    int rows, C;
    float eps;
    const float *a, *b, *gamma, *beta, *ys, *gn, *gy;    // ys: the backward's y
    float *y, *n, *ga, *parts;
};

// mean and 1 / sqrt(var + eps) of the lane's nj values of a row of C
__device__ __forceinline__ void ln_stats(const float* y, int nj, int C, float eps, float& mean, float& rstd) {
    float s = 0.0f;
#pragma unroll
    for (int j = 0; j < kLnMaxJ; ++j)
        if (j < nj) s += y[j];
    mean = warp_sum(s) / (float)C;
    float v = 0.0f;
#pragma unroll
    for (int j = 0; j < kLnMaxJ; ++j)
        if (j < nj) { const float d = y[j] - mean; v = fmaf(d, d, v); }
    rstd = 1.0f / sqrtf(warp_sum(v) / (float)C + eps);
}

__global__ void __launch_bounds__(kLnWarps * 32) ln_fwd_kernel(LnArgs a) {
    const int lane = threadIdx.x & 31, row = blockIdx.x * kLnWarps + (threadIdx.x >> 5);
    if (row >= a.rows) return;
    const int C = a.C, nj = C / 32;
    const size_t base = (size_t)row * C + lane;
    float y[kLnMaxJ];
#pragma unroll
    for (int j = 0; j < kLnMaxJ; ++j)
        if (j < nj) y[j] = a.b ? __ldg(a.a + base + 32 * j) + __ldg(a.b + base + 32 * j) : __ldg(a.a + base + 32 * j);
    float mean, rstd;
    ln_stats(y, nj, C, a.eps, mean, rstd);
#pragma unroll
    for (int j = 0; j < kLnMaxJ; ++j) {
        if (j >= nj) continue;
        const int c = lane + 32 * j;
        if (a.y) a.y[base + 32 * j] = y[j];
        a.n[base + 32 * j] = fmaf((y[j] - mean) * rstd, __ldg(a.gamma + c), __ldg(a.beta + c));
    }
}

__global__ void __launch_bounds__(kLnWarps * 32) ln_bwd_kernel(LnArgs a) {
    __shared__ float acc_s[2][kLnMaxJ * 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, C = a.C, nj = C / 32;
    const int r0 = blockIdx.x * kLnRows, r1 = min(r0 + kLnRows, a.rows);
    float gam[kLnMaxJ], dg[kLnMaxJ], db[kLnMaxJ];
#pragma unroll
    for (int j = 0; j < kLnMaxJ; ++j) {
        gam[j] = j < nj ? __ldg(a.gamma + lane + 32 * j) : 0.0f;
        dg[j] = 0.0f;
        db[j] = 0.0f;
    }
    for (int row = r0 + warp; row < r1; row += kLnWarps) {
        const size_t base = (size_t)row * C + lane;
        float y[kLnMaxJ], g[kLnMaxJ];
#pragma unroll
        for (int j = 0; j < kLnMaxJ; ++j)
            if (j < nj) { y[j] = __ldg(a.ys + base + 32 * j); g[j] = __ldg(a.gn + base + 32 * j); }
        float mean, rstd;
        ln_stats(y, nj, C, a.eps, mean, rstd);
        float s1 = 0.0f, s2 = 0.0f;
#pragma unroll
        for (int j = 0; j < kLnMaxJ; ++j) {
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
        for (int j = 0; j < kLnMaxJ; ++j) {
            if (j >= nj) continue;
            const float d = rstd * (g[j] - m1 - y[j] * m2);
            a.ga[base + 32 * j] = a.gy ? __ldg(a.gy + base + 32 * j) + d : d;
        }
    }
    // the warps' sums, added in warp order
    for (int w = 0; w < kLnWarps; ++w) {
        if (warp == w) {
#pragma unroll
            for (int j = 0; j < kLnMaxJ; ++j) {
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

bool misaligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) != 0; }

// the heads per CTA: the largest divisor Hs of H with bs^3 Hs D <= kGaMaxThreadCols
int ga_check(const char* fn, int B, int R, int g, int S, int C, int H, int* Hs) {
    if (B < 1 || g < 1 || R < 1 || R > 1024 || R % g != 0)
        return set_error("%s: bad sizes (B=%d, R=%d, g=%d): need B, g >= 1 and R <= 1024 a multiple of g", fn, B, R,
                         g);
    if (S < 1 || S > kGaMaxS) return set_error("%s: bad sizes (S=%d): need 1 <= S <= %d", fn, S, kGaMaxS);
    if (H < 1 || C < 1 || C % H != 0 || (C / H != 16 && C / H != 32))
        return set_error("%s: bad sizes (C=%d, H=%d): need a head dim C/H of 16 or 32", fn, C, H);
    const long long bs = R / g, nq = bs * bs * bs, D = C / H;
    if (nq * D > kGaMaxThreadCols)
        return set_error("%s: bad sizes (R=%d, g=%d, C/H=%lld): need (R/g)^3 * C/H <= %d", fn, R, g, D,
                         kGaMaxThreadCols);
    if ((long long)B * g * g * g * H > INT32_MAX)
        return set_error("%s: bad sizes (B=%d, g=%d, H=%d): need B g^3 H < 2^31", fn, B, g, H);
    int hs = 1;
    for (int d = 1; d <= H; ++d)
        if (H % d == 0 && nq * d * D <= kGaMaxThreadCols) hs = d;
    *Hs = hs;
    return 0;
}

GaArgs ga_args(int R, int g, int S, int C, int H, int Hs) {
    GaArgs a;
    memset(&a, 0, sizeof(a));
    a.R = R; a.g = g; a.bs = R / g; a.nq = a.bs * a.bs * a.bs; a.S = S; a.C = C; a.H = H; a.Hs = Hs;
    a.scale = 1.0f / sqrtf((float)(C / H));
    return a;
}

int ln_check(const char* fn, int rows, int C, float eps) {
    if (rows < 0) return set_error("%s: bad sizes (rows=%d): need rows >= 0", fn, rows);
    if (C < 32 || C > 32 * kLnMaxJ || C % 32 != 0)
        return set_error("%s: bad sizes (C=%d): need a multiple of 32 up to %d", fn, C, 32 * kLnMaxJ);
    if (!(eps > 0.0f) || !isfinite(eps)) return set_error("%s: bad eps (%g): need a positive finite value", fn, eps);
    return 0;
}

}  // namespace
}  // namespace srf

using srf::cuda_error;
using srf::set_error;

extern "C" int srf_group_attn_forward(void* stream_, int B, int R, int g, int S, int C, int H, const float* q,
                                      const float* k, const float* v, float* o) {
    const char* fn = "srf_group_attn_forward";
    int Hs;
    if (srf::ga_check(fn, B, R, g, S, C, H, &Hs)) return 1;
    if (!q || !k || !v || !o) return set_error("%s: null pointer", fn);
    if (srf::misaligned16(q) || srf::misaligned16(k) || srf::misaligned16(v) || srf::misaligned16(o))
        return set_error("%s: pointers must be 16-byte aligned", fn);
    srf::GaArgs a = srf::ga_args(R, g, S, C, H, Hs);
    a.q = q; a.k = k; a.v = v; a.o = o;
    const unsigned grid = (unsigned)((long long)B * g * g * g * (H / Hs));
    const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (C / H == 16) srf::ga_fwd_kernel<16><<<grid, a.nq * Hs, 0, stream>>>(a);
    else srf::ga_fwd_kernel<32><<<grid, a.nq * Hs, 0, stream>>>(a);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_error("group_attn forward launch", e);
}

extern "C" int srf_group_attn_backward(void* stream_, int B, int R, int g, int S, int C, int H, const float* q,
                                       const float* k, const float* v, const float* dL_do, float* dL_dq,
                                       float* dL_dk, float* dL_dv) {
    const char* fn = "srf_group_attn_backward";
    int Hs;
    if (srf::ga_check(fn, B, R, g, S, C, H, &Hs)) return 1;
    if (!q || !k || !v || !dL_do || !dL_dq || !dL_dk || !dL_dv) return set_error("%s: null pointer", fn);
    if (srf::misaligned16(q) || srf::misaligned16(k) || srf::misaligned16(v) || srf::misaligned16(dL_do) ||
        srf::misaligned16(dL_dq) || srf::misaligned16(dL_dk) || srf::misaligned16(dL_dv))
        return set_error("%s: pointers must be 16-byte aligned", fn);
    srf::GaArgs a = srf::ga_args(R, g, S, C, H, Hs);
    a.q = q; a.k = k; a.v = v; a.go = dL_do; a.gq = dL_dq; a.gk = dL_dk; a.gv = dL_dv;
    const unsigned grid = (unsigned)((long long)B * g * g * g * (H / Hs));
    const int threads = a.nq * Hs;
    const size_t smem = sizeof(float) * 2 * (size_t)threads * (C / H);
    const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (C / H == 16) srf::ga_bwd_kernel<16><<<grid, threads, smem, stream>>>(a);
    else srf::ga_bwd_kernel<32><<<grid, threads, smem, stream>>>(a);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_error("group_attn backward launch", e);
}

extern "C" int srf_add_layernorm_forward(void* stream_, int rows, int C, float eps, const float* a, const float* b,
                                         const float* gamma, const float* beta, float* y, float* n) {
    const char* fn = "srf_add_layernorm_forward";
    if (srf::ln_check(fn, rows, C, eps)) return 1;
    if (!a || !gamma || !beta || !n) return set_error("%s: null pointer", fn);
    if (b && !y) return set_error("%s: null y with a residual b", fn);
    if (rows == 0) return 0;
    srf::LnArgs la;
    memset(&la, 0, sizeof(la));
    la.rows = rows; la.C = C; la.eps = eps; la.a = a; la.b = b; la.gamma = gamma; la.beta = beta; la.y = y; la.n = n;
    const unsigned grid = (unsigned)((rows + srf::kLnWarps - 1) / srf::kLnWarps);
    srf::ln_fwd_kernel<<<grid, srf::kLnWarps * 32, 0, static_cast<cudaStream_t>(stream_)>>>(la);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_error("add_layernorm forward launch", e);
}

extern "C" int srf_add_layernorm_workspace_bytes(int rows, int C, size_t* bytes) {
    const char* fn = "srf_add_layernorm_workspace_bytes";
    if (srf::ln_check(fn, rows, C, 1.0f)) return 1;
    if (!bytes) return set_error("%s: null output", fn);
    const size_t nparts = ((size_t)rows + srf::kLnRows - 1) / srf::kLnRows;
    *bytes = srf::align_up(sizeof(float) * 2 * (size_t)C * (nparts ? nparts : 1));
    return 0;
}

extern "C" int srf_add_layernorm_backward(void* stream_, int rows, int C, float eps, const float* y,
                                          const float* gamma, const float* dL_dn, const float* dL_dy,
                                          void* workspace, float* dL_da, float* d_gamma, float* d_beta) {
    const char* fn = "srf_add_layernorm_backward";
    if (srf::ln_check(fn, rows, C, eps)) return 1;
    if (!y || !gamma || !dL_dn) return set_error("%s: null input pointer", fn);
    if (!dL_da || !d_gamma || !d_beta) return set_error("%s: null gradient pointer", fn);
    if (!workspace || srf::misaligned(workspace)) return set_error("%s: workspace must be 256-byte aligned", fn);
    const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const int nparts = (rows + srf::kLnRows - 1) / srf::kLnRows;
    if (nparts > 0) {
        srf::LnArgs la;
        memset(&la, 0, sizeof(la));
        la.rows = rows; la.C = C; la.eps = eps; la.ys = y; la.gamma = gamma; la.gn = dL_dn; la.gy = dL_dy;
        la.ga = dL_da; la.parts = static_cast<float*>(workspace);
        srf::ln_bwd_kernel<<<(unsigned)nparts, srf::kLnWarps * 32, 0, stream>>>(la);
    }
    srf::part_sums(stream, static_cast<const float*>(workspace), nparts, 2 * (size_t)C, srf::seg(d_gamma, C),
                   srf::seg(d_beta, C));
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_error("add_layernorm backward launch", e);
}
