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
// Residual add + LayerNorm: ln_fwd_kernel<16> / ln_bwd_kernel<16> of layer_norm.cuh (C <= 512).
#include <math.h>
#include <string.h>

#include "../../include/surfel_vol_transformer.h"
#include "fixed_sums.cuh"
#include "layer_norm.cuh"
#include "surfel_kernels.h"

namespace srf {
namespace {

constexpr int kGaMaxThreadCols = 4096;   // threads x D of an attention CTA: 2 x 16 KB of backward staging
constexpr int kGaMaxS = 4096;
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
    // an empty tensor may have no storage: the row arrays may be NULL when rows == 0
    if ((rows > 0 && (!a || !n)) || !gamma || !beta) return set_error("%s: null pointer", fn);
    if (rows > 0 && b && !y) return set_error("%s: null y with a residual b", fn);
    srf::ln_forward<srf::kLnMaxJ>(static_cast<cudaStream_t>(stream_), rows, C, eps, a, b, gamma, beta, y, n);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_error("add_layernorm forward launch", e);
}

extern "C" int srf_add_layernorm_workspace_bytes(int rows, int C, size_t* bytes) {
    const char* fn = "srf_add_layernorm_workspace_bytes";
    if (srf::ln_check(fn, rows, C, 1.0f)) return 1;
    if (!bytes) return set_error("%s: null output", fn);
    *bytes = srf::align_up(srf::ln_parts_bytes(rows, C));
    return 0;
}

extern "C" int srf_add_layernorm_backward(void* stream_, int rows, int C, float eps, const float* y,
                                          const float* gamma, const float* dL_dn, const float* dL_dy,
                                          void* workspace, float* dL_da, float* d_gamma, float* d_beta) {
    const char* fn = "srf_add_layernorm_backward";
    if (srf::ln_check(fn, rows, C, eps)) return 1;
    if ((rows > 0 && (!y || !dL_dn)) || !gamma) return set_error("%s: null input pointer", fn);
    if ((rows > 0 && !dL_da) || !d_gamma || !d_beta) return set_error("%s: null gradient pointer", fn);
    if (!workspace || srf::misaligned(workspace)) return set_error("%s: workspace must be 256-byte aligned", fn);
    srf::ln_backward<srf::kLnMaxJ>(static_cast<cudaStream_t>(stream_), rows, C, eps, y, gamma, dL_dn, dL_dy,
                                   static_cast<float*>(workspace), dL_da, d_gamma, d_beta);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_error("add_layernorm backward launch", e);
}
