// image_encoder.cu -- the fused parts of LaRa's image encoder (DinoWrapper, lightning/network.py:14-55, 442-445): timm's
// DINO ViT at C in {384, 768}, DESIGN §3.25.  The C entries of include/surfel_image_encoder.h are defined here.  The
// patch GEMM, qkv, the attention core, proj and the MLP stay with cuBLAS and torch.
//
//   patchify_kernel     a thread per element of the patch matrix: one image read at any strides, Normalize as two
//                       fp32 operations.  No backward: the images are constants.
//   tok_ln_fwd_kernel   a warp per token row: x = cls + pos0 or (patch_out + bias) + pos_r, then LN(x) (norm1 of
//                       block 0).  Its backward is ln_bwd_kernel<24> followed by fixed-order sums over the images.
//   ln_fwd_kernel<24> / ln_bwd_kernel<24>  the residual add + LayerNorms of the blocks (layer_norm.cuh).
//   final_ln_fwd_kernel a warp per token row: y = a + b, LN(y); the CTA's 8 rows are staged in shared memory and stored
//                       transposed to [N, C, L], 8 consecutive tokens per channel, the cls row dropped.
//   final_gather_kernel the backward's dL/dmaps [N, C, L] gathered back to token rows (zero on the cls rows), the same
//                       staging in reverse; then ln_bwd_kernel<24>.
#include <math.h>
#include <string.h>

#include "../../include/surfel_image_encoder.h"
#include "fixed_sums.cuh"
#include "layer_norm.cuh"
#include "surfel_kernels.h"

namespace srf {
namespace {

constexpr int kVitJ = 24;                // C <= 768
constexpr int kVitMaxC = 32 * kVitJ;
constexpr int kPatch = 16;
constexpr int kPatchK = 3 * kPatch * kPatch;

struct PatchArgs {
    int h, w;
    long long sn, sc, sy, sx;
    size_t total;
    const float* img;
    float* out;
};

__global__ void __launch_bounds__(256) patchify_kernel(PatchArgs a) {
    const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= a.total) return;
    const int k = (int)(e % kPatchK), kx = k % kPatch, ky = (k / kPatch) % kPatch, c = k / (kPatch * kPatch);
    const size_t row = e / kPatchK;
    const int px = (int)(row % a.w), py = (int)((row / a.w) % a.h);
    const long long n = (long long)(row / ((size_t)a.w * a.h));
    const float v = __ldg(a.img + n * a.sn + c * a.sc + (long long)(py * kPatch + ky) * a.sy +
                          (long long)(px * kPatch + kx) * a.sx);
    const float mean = c == 0 ? 0.485f : (c == 1 ? 0.456f : 0.406f);
    const float sd = c == 0 ? 0.229f : (c == 1 ? 0.224f : 0.225f);
    a.out[e] = __fdiv_rn(__fsub_rn(v, mean), sd);
}

struct TokArgs {
    int N, L, C;
    float eps;
    const float *patch, *bias, *cls, *pos0, *pos_r, *gamma, *beta;
    float *x, *n;
};

__global__ void __launch_bounds__(kLnWarps * 32) tok_ln_fwd_kernel(TokArgs a) {
    const int lane = threadIdx.x & 31, row = blockIdx.x * kLnWarps + (threadIdx.x >> 5);
    if (row >= a.N * (a.L + 1)) return;
    const int C = a.C, nj = C / 32, r = row % (a.L + 1), l = r ? r - 1 : 0;
    const size_t base = (size_t)row * C + lane;
    const float* prow = a.patch + ((size_t)(row / (a.L + 1)) * a.L + l) * C + lane;
    const float* qrow = a.pos_r + (size_t)l * C + lane;
    float y[kVitJ];
#pragma unroll
    for (int j = 0; j < kVitJ; ++j) {
        if (j >= nj) continue;
        const int c = lane + 32 * j;
        y[j] = r == 0 ? __ldg(a.cls + c) + __ldg(a.pos0 + c)
                      : (__ldg(prow + 32 * j) + __ldg(a.bias + c)) + __ldg(qrow + 32 * j);
    }
    float mean, rstd;
    ln_stats<kVitJ>(y, nj, C, a.eps, mean, rstd);
#pragma unroll
    for (int j = 0; j < kVitJ; ++j) {
        if (j >= nj) continue;
        const int c = lane + 32 * j;
        a.x[base + 32 * j] = y[j];
        a.n[base + 32 * j] = fmaf((y[j] - mean) * rstd, __ldg(a.gamma + c), __ldg(a.beta + c));
    }
}

struct FinalArgs {
    int N, L, C;
    float eps;
    const float *a, *b, *gamma, *beta, *gmaps;
    float *y, *maps, *gn;
};

__global__ void __launch_bounds__(kLnWarps * 32) final_ln_fwd_kernel(FinalArgs a) {
    __shared__ float st[kLnWarps][kVitMaxC];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, C = a.C, nj = C / 32, T = a.L + 1;
    const int rows = a.N * T, row0 = blockIdx.x * kLnWarps, row = row0 + warp;
    if (row < rows) {
        const size_t base = (size_t)row * C + lane;
        float y[kVitJ];
#pragma unroll
        for (int j = 0; j < kVitJ; ++j)
            if (j < nj) y[j] = __ldg(a.a + base + 32 * j) + __ldg(a.b + base + 32 * j);
        float mean, rstd;
        ln_stats<kVitJ>(y, nj, C, a.eps, mean, rstd);
#pragma unroll
        for (int j = 0; j < kVitJ; ++j) {
            if (j >= nj) continue;
            const int c = lane + 32 * j;
            if (a.y) a.y[base + 32 * j] = y[j];
            st[warp][c] = fmaf((y[j] - mean) * rstd, __ldg(a.gamma + c), __ldg(a.beta + c));
        }
    }
    __syncthreads();
    for (int e = threadIdx.x; e < kLnWarps * C; e += kLnWarps * 32) {
        const int c = e / kLnWarps, w = e % kLnWarps, rw = row0 + w, r = rw % T;
        if (rw < rows && r != 0) a.maps[((size_t)(rw / T) * C + c) * a.L + (r - 1)] = st[w][c];
    }
}

__global__ void __launch_bounds__(kLnWarps * 32) final_gather_kernel(FinalArgs a) {
    __shared__ float st[kLnWarps][kVitMaxC];
    const int C = a.C, T = a.L + 1, rows = a.N * T, row0 = blockIdx.x * kLnWarps;
    for (int e = threadIdx.x; e < kLnWarps * C; e += kLnWarps * 32) {
        const int c = e / kLnWarps, w = e % kLnWarps, rw = row0 + w, r = rw % T;
        if (rw < rows) st[w][c] = r ? __ldg(a.gmaps + ((size_t)(rw / T) * C + c) * a.L + (r - 1)) : 0.0f;
    }
    __syncthreads();
    for (int e = threadIdx.x; e < kLnWarps * C; e += kLnWarps * 32) {
        const int w = e / C, c = e % C, rw = row0 + w;
        if (rw < rows) a.gn[(size_t)rw * C + c] = st[w][c];
    }
}

int vit_c_check(const char* fn, int C, float eps) {
    if (C != 384 && C != 768) return set_error("%s: bad sizes (C=%d): need 384 or 768", fn, C);
    if (!(eps > 0.0f) || !isfinite(eps)) return set_error("%s: bad eps (%g): need a positive finite value", fn, eps);
    return 0;
}

int vit_check(const char* fn, int N, int L, int C, float eps) {
    if (N < 1 || L < 1 || (long long)N * (L + 1) > INT32_MAX || (long long)L * C > INT32_MAX)
        return set_error("%s: bad sizes (N=%d, L=%d): need N, L >= 1, N (1 + L) < 2^31 and L C < 2^31", fn, N, L);
    return vit_c_check(fn, C, eps);
}

int vit_rows_check(const char* fn, int rows, int C, float eps) {
    if (rows < 0) return set_error("%s: bad sizes (rows=%d): need rows >= 0", fn, rows);
    return vit_c_check(fn, C, eps);
}

size_t tokens_pos_offset(int N, int L, int C) { return align_up(ln_parts_bytes(N * (L + 1), C)); }
size_t final_parts_offset(int N, int L, int C) { return align_up(sizeof(float) * (size_t)N * (L + 1) * C); }

int launched(const char* what) {
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_error(what, e);
}

}  // namespace
}  // namespace srf

using srf::set_error;

extern "C" int srf_vit_patchify(void* stream_, int N, int H, int W, long long sn, long long sc, long long sy,
                                long long sx, const float* image, float* patches) {
    const char* fn = "srf_vit_patchify";
    if (N < 1 || H < srf::kPatch || W < srf::kPatch || H % srf::kPatch != 0 || W % srf::kPatch != 0)
        return set_error("%s: bad sizes (N=%d, H=%d, W=%d): need N >= 1 and H, W positive multiples of 16", fn, N, H,
                         W);
    const long long rows = (long long)N * (H / srf::kPatch) * (W / srf::kPatch);
    if (rows > INT32_MAX) return set_error("%s: bad sizes (N=%d, H=%d, W=%d): need N h w < 2^31", fn, N, H, W);
    if (!image || !patches) return set_error("%s: null pointer", fn);
    srf::PatchArgs a;
    memset(&a, 0, sizeof(a));
    a.h = H / srf::kPatch; a.w = W / srf::kPatch; a.sn = sn; a.sc = sc; a.sy = sy; a.sx = sx;
    a.total = (size_t)rows * srf::kPatchK; a.img = image; a.out = patches;
    srf::patchify_kernel<<<(unsigned)((a.total + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream_)>>>(a);
    return srf::launched("vit_patchify launch");
}

extern "C" int srf_vit_tokens_forward(void* stream_, int N, int L, int C, float eps, const float* patch_out,
                                      const float* bias, const float* cls, const float* pos0, const float* pos_r,
                                      const float* gamma, const float* beta, float* x, float* n1) {
    const char* fn = "srf_vit_tokens_forward";
    if (srf::vit_check(fn, N, L, C, eps)) return 1;
    if (!patch_out || !bias || !cls || !pos0 || !pos_r || !gamma || !beta || !x || !n1)
        return set_error("%s: null pointer", fn);
    srf::TokArgs a;
    memset(&a, 0, sizeof(a));
    a.N = N; a.L = L; a.C = C; a.eps = eps; a.patch = patch_out; a.bias = bias; a.cls = cls; a.pos0 = pos0;
    a.pos_r = pos_r; a.gamma = gamma; a.beta = beta; a.x = x; a.n = n1;
    const unsigned grid = (unsigned)(((long long)N * (L + 1) + srf::kLnWarps - 1) / srf::kLnWarps);
    srf::tok_ln_fwd_kernel<<<grid, srf::kLnWarps * 32, 0, static_cast<cudaStream_t>(stream_)>>>(a);
    return srf::launched("vit_tokens forward launch");
}

extern "C" int srf_vit_tokens_workspace_bytes(int N, int L, int C, size_t* bytes) {
    const char* fn = "srf_vit_tokens_workspace_bytes";
    if (srf::vit_check(fn, N, L, C, 1.0f)) return 1;
    if (!bytes) return set_error("%s: null output", fn);
    *bytes = srf::tokens_pos_offset(N, L, C) + srf::align_up(sizeof(double) * (size_t)L * C);
    return 0;
}

extern "C" int srf_vit_tokens_backward(void* stream_, int N, int L, int C, float eps, const float* x,
                                       const float* gamma, const float* dL_dn1, const float* dL_dx, void* workspace,
                                       float* dL_dtokens, float* d_bias, float* d_cls, float* d_pos_r,
                                       float* d_gamma, float* d_beta) {
    const char* fn = "srf_vit_tokens_backward";
    if (srf::vit_check(fn, N, L, C, eps)) return 1;
    if (!x || !gamma || !dL_dn1) return set_error("%s: null input pointer", fn);
    if (!dL_dtokens || !d_bias || !d_cls || !d_pos_r || !d_gamma || !d_beta)
        return set_error("%s: null gradient pointer", fn);
    if (!workspace || srf::misaligned(workspace)) return set_error("%s: workspace must be 256-byte aligned", fn);
    const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    char* ws = static_cast<char*>(workspace);
    double* pos_d = reinterpret_cast<double*>(ws + srf::tokens_pos_offset(N, L, C));
    const size_t T = (size_t)(L + 1) * C;
    srf::ln_backward<srf::kVitJ>(stream, N * (L + 1), C, eps, x, gamma, dL_dn1, dL_dx, reinterpret_cast<float*>(ws),
                                 dL_dtokens, d_gamma, d_beta);
    srf::part_sums(stream, static_cast<const float*>(dL_dtokens + C), N, T, srf::seg(pos_d, L * C));
    srf::part_sums(stream, static_cast<const double*>(pos_d), L, (size_t)C, srf::seg(d_bias, C));
    srf::part_sums(stream, static_cast<const double*>(pos_d), 1, (size_t)L * C, srf::seg(d_pos_r, L * C));
    srf::part_sums(stream, static_cast<const float*>(dL_dtokens), N, T, srf::seg(d_cls, C));
    return srf::launched("vit_tokens backward launch");
}

extern "C" int srf_vit_layernorm_forward(void* stream_, int rows, int C, float eps, const float* a, const float* b,
                                         const float* gamma, const float* beta, float* y, float* n) {
    const char* fn = "srf_vit_layernorm_forward";
    if (srf::vit_rows_check(fn, rows, C, eps)) return 1;
    // an empty tensor may have no storage: the row arrays may be NULL when rows == 0
    if ((rows > 0 && (!a || !n)) || !gamma || !beta) return set_error("%s: null pointer", fn);
    if (rows > 0 && b && !y) return set_error("%s: null y with a residual b", fn);
    srf::ln_forward<srf::kVitJ>(static_cast<cudaStream_t>(stream_), rows, C, eps, a, b, gamma, beta, y, n);
    return srf::launched("vit_layernorm forward launch");
}

extern "C" int srf_vit_layernorm_workspace_bytes(int rows, int C, size_t* bytes) {
    const char* fn = "srf_vit_layernorm_workspace_bytes";
    if (srf::vit_rows_check(fn, rows, C, 1.0f)) return 1;
    if (!bytes) return set_error("%s: null output", fn);
    *bytes = srf::align_up(srf::ln_parts_bytes(rows, C));
    return 0;
}

extern "C" int srf_vit_layernorm_backward(void* stream_, int rows, int C, float eps, const float* y,
                                          const float* gamma, const float* dL_dn, const float* dL_dy,
                                          void* workspace, float* dL_da, float* d_gamma, float* d_beta) {
    const char* fn = "srf_vit_layernorm_backward";
    if (srf::vit_rows_check(fn, rows, C, eps)) return 1;
    if ((rows > 0 && (!y || !dL_dn)) || !gamma) return set_error("%s: null input pointer", fn);
    if ((rows > 0 && !dL_da) || !d_gamma || !d_beta) return set_error("%s: null gradient pointer", fn);
    if (!workspace || srf::misaligned(workspace)) return set_error("%s: workspace must be 256-byte aligned", fn);
    srf::ln_backward<srf::kVitJ>(static_cast<cudaStream_t>(stream_), rows, C, eps, y, gamma, dL_dn, dL_dy,
                                 static_cast<float*>(workspace), dL_da, d_gamma, d_beta);
    return srf::launched("vit_layernorm backward launch");
}

extern "C" int srf_vit_final_norm_forward(void* stream_, int N, int L, int C, float eps, const float* a,
                                          const float* b, const float* gamma, const float* beta, float* y,
                                          float* maps) {
    const char* fn = "srf_vit_final_norm_forward";
    if (srf::vit_check(fn, N, L, C, eps)) return 1;
    if (!a || !b || !gamma || !beta || !maps) return set_error("%s: null pointer", fn);
    srf::FinalArgs fa;
    memset(&fa, 0, sizeof(fa));
    fa.N = N; fa.L = L; fa.C = C; fa.eps = eps; fa.a = a; fa.b = b; fa.gamma = gamma; fa.beta = beta; fa.y = y;
    fa.maps = maps;
    const unsigned grid = (unsigned)(((long long)N * (L + 1) + srf::kLnWarps - 1) / srf::kLnWarps);
    srf::final_ln_fwd_kernel<<<grid, srf::kLnWarps * 32, 0, static_cast<cudaStream_t>(stream_)>>>(fa);
    return srf::launched("vit_final_norm forward launch");
}

extern "C" int srf_vit_final_norm_workspace_bytes(int N, int L, int C, size_t* bytes) {
    const char* fn = "srf_vit_final_norm_workspace_bytes";
    if (srf::vit_check(fn, N, L, C, 1.0f)) return 1;
    if (!bytes) return set_error("%s: null output", fn);
    *bytes = srf::final_parts_offset(N, L, C) + srf::align_up(srf::ln_parts_bytes(N * (L + 1), C));
    return 0;
}

extern "C" int srf_vit_final_norm_backward(void* stream_, int N, int L, int C, float eps, const float* y,
                                           const float* gamma, const float* dL_dmaps, void* workspace, float* dL_da,
                                           float* d_gamma, float* d_beta) {
    const char* fn = "srf_vit_final_norm_backward";
    if (srf::vit_check(fn, N, L, C, eps)) return 1;
    if (!y || !gamma || !dL_dmaps) return set_error("%s: null input pointer", fn);
    if (!dL_da || !d_gamma || !d_beta) return set_error("%s: null gradient pointer", fn);
    if (!workspace || srf::misaligned(workspace)) return set_error("%s: workspace must be 256-byte aligned", fn);
    const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    char* ws = static_cast<char*>(workspace);
    float* gn = reinterpret_cast<float*>(ws);
    srf::FinalArgs fa;
    memset(&fa, 0, sizeof(fa));
    fa.N = N; fa.L = L; fa.C = C; fa.gmaps = dL_dmaps; fa.gn = gn;
    const int rows = N * (L + 1);
    srf::final_gather_kernel<<<(unsigned)((rows + srf::kLnWarps - 1) / srf::kLnWarps), srf::kLnWarps * 32, 0,
                                stream>>>(fa);
    srf::ln_backward<srf::kVitJ>(stream, rows, C, eps, y, gamma, gn, nullptr,
                                 reinterpret_cast<float*>(ws + srf::final_parts_offset(N, L, C)), dL_da, d_gamma,
                                 d_beta);
    return srf::launched("vit_final_norm backward launch");
}
