// loss.cu -- fused loss -> dL/d(render_img outputs) producer (SURVEY 8f rank 3).
//
// Restates the rasterizer-facing terms of LaRa's training loss (lightning/loss.py:33-60):
//     loss  = mean((image - tar_rgb)^2)                                   (:33-34)
//           + 1000 * mean(rend_dist)                                      (:48-51, iter > 1000)
//           + 0.2 * mean((1 - sum_c rend_normal_c * depth_normal_c) * acc_map.detach())   (:53-59)
// (the MS-SSIM term :42-46 is ms_ssim.cu, a separate autograd node; its gradient simply adds to g_image).
// In torch these are ~15 elementwise / reduction kernels forward and ~20 backward, each a full-image HBM round
// trip over the [H, V*W, C] concatenation of the views.  Here:
//   loss_sums_kernel : one pass over the stacked planar outputs of the fused epilogue ([V,C,H,W]) -> three sums
//                      (four with the fine pass: its squared error against the same target, read once)
//   loss_grads_kernel: one pass writing g_image (and the fine pass's) / g_rend_normal / g_depth_normal / g_rend_dist,
//                      already planar and stacked, i.e. exactly what srf_views_epilogue_backward consumes -- scaled by
//                      the upstream scalar read from device memory (no host sync).
// `target` is read in the batch's own channel-last layout [V,H,W,3] (lightning/loss.py:24 permutes a view of it).
// V may be the B*V views of a whole batch.  Without a fine image the kernels do exactly what they did before the
// fine pass existed: srf_loss_forward / _backward are that case of srf_loss_passes_*.
// The C entries srf_loss_* (include/surfel_rasterizer.h) are defined here.
#include <string.h>

#include "../../include/surfel_rasterizer.h"
#include "fixed_sums.cuh"
#include "surfel_common.cuh"
#include "surfel_kernels.h"

namespace srf {

struct LossArgs {
    int W, H, nviews;
    int with_reg;                // iter > 1000: distortion and normal-consistency terms are on
    float w_mse, w_dist, w_normal;   // weights already divided by the reference's mean() denominators
    const float* image;          // [V,3,H,W]
    const float* image_fine;     // [V,3,H,W] or null: the fine pass, read against the same target (no regularisers)
    const float* target;         // [V,H,W,3] channel-last, the batch's own layout
    const float* rend_normal;    // [V,3,H,W]
    const float* depth_normal;   // [V,3,H,W]
    const float* acc;            // [V,H,W]
    const float* dist;           // [V,H,W]
    double* sums;                // [nterms]: sum (image-target)^2, sum dist, sum (1 - <rn,dn>) acc, sum (image_fine-target)^2
    int nterms;                  // 3, or 4 with image_fine
    double* partials;            // [loss_det_blocks][nterms] or null: deterministic sums (written, then reduced in a fixed order)
    const float* gout;           // device scalar: upstream gradient of the loss (null = 1)
    float* g_image;              // [V,3,H,W] out (may be null: forward statistics only)
    float* g_image_fine;         // [V,3,H,W] out with image_fine
    float* g_rend_normal; float* g_depth_normal; float* g_dist;
};

template <bool kDet>
__global__ void __launch_bounds__(256) loss_sums_kernel(LossArgs a) {
    const size_t npix = (size_t)a.W * a.H, total = npix * (size_t)a.nviews;
    float s_mse = 0.f, s_dist = 0.f, s_norm = 0.f, s_fine = 0.f;
    for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (size_t)gridDim.x * 256) {
        const size_t v = i / npix, pix = i - v * npix;
        const float* img = a.image + v * 3 * npix + pix;
        const float* tar = a.target + i * 3;
        float t[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            t[c] = __ldg(tar + c);
            const float d = img[c * npix] - t[c];
            s_mse = fmaf(d, d, s_mse);
        }
        if (a.image_fine) {
            const float* imf = a.image_fine + v * 3 * npix + pix;
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float d = imf[c * npix] - t[c];
                s_fine = fmaf(d, d, s_fine);
            }
        }
        if (a.with_reg) {
            s_dist += a.dist[i];
            const float* rn = a.rend_normal + v * 3 * npix + pix;
            const float* dn = a.depth_normal + v * 3 * npix + pix;
            const float dot = rn[0] * dn[0] + rn[npix] * dn[npix] + rn[2 * npix] * dn[2 * npix];
            s_norm = fmaf(1.0f - dot, a.acc[i], s_norm);
        }
    }
    // warp -> block -> one double atomic per block and term
    __shared__ float s_part[4][8];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        s_mse += __shfl_xor_sync(0xffffffffu, s_mse, o);
        s_dist += __shfl_xor_sync(0xffffffffu, s_dist, o);
        s_norm += __shfl_xor_sync(0xffffffffu, s_norm, o);
        s_fine += __shfl_xor_sync(0xffffffffu, s_fine, o);
    }
    if (lane == 0) { s_part[0][wid] = s_mse; s_part[1][wid] = s_dist; s_part[2][wid] = s_norm; s_part[3][wid] = s_fine; }
    __syncthreads();
    if (threadIdx.x < a.nterms) {
        double t = 0.0;
#pragma unroll
        for (int w = 0; w < 8; ++w) t += (double)s_part[threadIdx.x][w];
        if (kDet) a.partials[a.nterms * blockIdx.x + threadIdx.x] = t;
        else atomicAdd(a.sums + threadIdx.x, t);
    }
}

// blocks (= partial-sum triples) of the deterministic sums: a grid that does not depend on the device, so the same
// partials, and the same bits, on every GPU
static size_t loss_det_blocks(size_t total) { return min((size_t)1024, (total + 255) / 256); }

// deterministic path: the per-block partials of loss_sums_kernel<true> summed in a fixed order, warp w for term w
// (one warp per term: nterms warps)
__global__ void __launch_bounds__(128) loss_sums_finalize_kernel(const double* partials, int nblocks, int nterms,
                                                                 double* sums) {
    const int term = threadIdx.x >> 5;
    const double t = warp_strided_sum(partials + term, nblocks, nterms);
    if ((threadIdx.x & 31) == 0) sums[term] = t;
}

__global__ void __launch_bounds__(256) loss_grads_kernel(LossArgs a) {
    const size_t npix = (size_t)a.W * a.H, total = npix * (size_t)a.nviews;
    const size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= total) return;
    const float up = a.gout ? __ldg(a.gout) : 1.0f;
    const size_t v = i / npix, pix = i - v * npix;
    const float* img = a.image + v * 3 * npix + pix;
    const float* tar = a.target + i * 3;
    float* gi = a.g_image + v * 3 * npix + pix;
    const float k_mse = 2.0f * a.w_mse * up;
    float t[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        t[c] = __ldg(tar + c);
        gi[c * npix] = k_mse * (img[c * npix] - t[c]);
    }
    if (a.image_fine) {
        const float* imf = a.image_fine + v * 3 * npix + pix;
        float* gf = a.g_image_fine + v * 3 * npix + pix;
#pragma unroll
        for (int c = 0; c < 3; ++c) gf[c * npix] = k_mse * (imf[c * npix] - t[c]);
    }
    if (a.g_dist) a.g_dist[i] = a.with_reg ? a.w_dist * up : 0.0f;
    if (a.g_rend_normal && a.g_depth_normal) {
        float* grn = a.g_rend_normal + v * 3 * npix + pix;
        float* gdn = a.g_depth_normal + v * 3 * npix + pix;
        if (a.with_reg) {
            const float k = -a.w_normal * up * a.acc[i];
            const float* rn = a.rend_normal + v * 3 * npix + pix;
            const float* dn = a.depth_normal + v * 3 * npix + pix;
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                grn[c * npix] = k * dn[c * npix];
                gdn[c * npix] = k * rn[c * npix];
            }
        } else {
#pragma unroll
            for (int c = 0; c < 3; ++c) { grn[c * npix] = 0.0f; gdn[c * npix] = 0.0f; }
        }
    }
}

}  // namespace srf

using srf::cuda_error;
using srf::set_error;

// V*H*W pixels: every index is a size_t, so the limit is the backward's grid (one thread per pixel, 2^31 - 1 CTAs)
static int loss_sizes(const char* fn, int V, int H, int W) {
    if (V <= 0 || H <= 0 || W <= 0) return set_error("%s: bad sizes", fn);
    if ((double)V * H * W > (double)0x7fffffff * 256.0)
        return set_error("%s: V*H*W = %.0f pixels exceeds the launch grid", fn, (double)V * H * W);
    return 0;
}

static int loss_aligned(const char* fn, const float* const* p, int n) {
    for (int k = 0; k < n; ++k)
        if (reinterpret_cast<uintptr_t>(p[k]) & 3) return set_error("%s: buffers must be 4-byte aligned", fn);
    return 0;
}

static int loss_forward(const char* fn, srf_stream_t stream_, int V, int image_height, int image_width, int with_reg,
                        const float* image, const float* image_fine, const float* target_hwc, const float* rend_normal,
                        const float* depth_normal, const float* acc_map, const float* rend_dist, double* sums,
                        void* workspace) {
    if (loss_sizes(fn, V, image_height, image_width)) return 1;
    if (!image || !target_hwc || !sums) return set_error("%s: null pointer", fn);
    if (with_reg && (!rend_normal || !depth_normal || !acc_map || !rend_dist)) return set_error("%s: null regulariser input", fn);
    if (reinterpret_cast<uintptr_t>(workspace) & 7) return set_error("%s: workspace must be 8-byte aligned", fn);
    const float* in[7] = {image, image_fine, target_hwc, rend_normal, depth_normal, acc_map, rend_dist};
    if (loss_aligned(fn, in, 7)) return 1;
    if (reinterpret_cast<uintptr_t>(sums) & 7) return set_error("%s: sums must be 8-byte aligned", fn);
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    cudaError_t e;
    const int nterms = image_fine ? 4 : 3;
    // the deterministic path writes every sum from its partials; the atomics need zeroed sums
    if (!workspace && (e = cudaMemsetAsync(sums, 0, nterms * sizeof(double), stream)) != cudaSuccess)
        return cuda_error("memset loss sums", e);
    srf::LossArgs a;
    memset(&a, 0, sizeof(a));
    a.W = image_width; a.H = image_height; a.nviews = V; a.with_reg = with_reg ? 1 : 0;
    a.image = image; a.image_fine = image_fine; a.target = target_hwc; a.rend_normal = rend_normal;
    a.depth_normal = depth_normal; a.acc = acc_map; a.dist = rend_dist;
    a.sums = sums; a.nterms = nterms; a.partials = static_cast<double*>(workspace);
    const size_t total = (size_t)image_width * image_height * (size_t)V;
    if (workspace) {
        const int grid = (int)srf::loss_det_blocks(total);
        srf::loss_sums_kernel<true><<<grid, 256, 0, stream>>>(a);
        srf::loss_sums_finalize_kernel<<<1, 32 * nterms, 0, stream>>>(a.partials, grid, nterms, a.sums);
    } else {
        const int grid = (int)min((size_t)srf::sm_count() * 8, (total + 255) / 256);
        srf::loss_sums_kernel<false><<<grid, 256, 0, stream>>>(a);
    }
    e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_error("loss_sums launch", e);
}

static int loss_backward(const char* fn, srf_stream_t stream, int V, int image_height, int image_width, int with_reg,
                         float w_mse, float w_dist, float w_normal, const float* image, const float* image_fine,
                         const float* target_hwc, const float* rend_normal, const float* depth_normal,
                         const float* acc_map, const float* upstream, float* g_image, float* g_image_fine,
                         float* g_rend_normal, float* g_depth_normal, float* g_rend_dist) {
    if (loss_sizes(fn, V, image_height, image_width)) return 1;
    if (!image || !target_hwc || !g_image) return set_error("%s: null pointer", fn);
    if (!image_fine != !g_image_fine) return set_error("%s: image_fine and g_image_fine go together", fn);
    if (with_reg && (!rend_normal || !depth_normal || !acc_map || !g_rend_normal || !g_depth_normal || !g_rend_dist))
        return set_error("%s: null regulariser pointer", fn);
    const float* buf[12] = {image, image_fine, target_hwc, rend_normal, depth_normal, acc_map, upstream,
                            g_image, g_image_fine, g_rend_normal, g_depth_normal, g_rend_dist};
    if (loss_aligned(fn, buf, 12)) return 1;
    srf::LossArgs a;
    memset(&a, 0, sizeof(a));
    a.W = image_width; a.H = image_height; a.nviews = V; a.with_reg = with_reg ? 1 : 0;
    a.w_mse = w_mse; a.w_dist = w_dist; a.w_normal = w_normal;
    a.image = image; a.image_fine = image_fine; a.target = target_hwc; a.rend_normal = rend_normal;
    a.depth_normal = depth_normal; a.acc = acc_map;
    a.gout = upstream;
    a.g_image = g_image; a.g_image_fine = g_image_fine;
    a.g_rend_normal = g_rend_normal; a.g_depth_normal = g_depth_normal; a.g_dist = g_rend_dist;
    const size_t total = (size_t)image_width * image_height * (size_t)V;
    srf::loss_grads_kernel<<<(unsigned)((total + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(a);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_error("loss_grads launch", e);
}

static int loss_workspace_bytes(const char* fn, int V, int image_height, int image_width, int nterms, size_t* bytes) {
    if (loss_sizes(fn, V, image_height, image_width)) return 1;
    if (!bytes) return set_error("%s: null pointer", fn);
    *bytes = srf::loss_det_blocks((size_t)V * image_height * image_width) * nterms * sizeof(double);
    return 0;
}

extern "C" int srf_loss_forward(srf_stream_t stream, int V, int image_height, int image_width, int with_reg,
                                const float* image, const float* target_hwc, const float* rend_normal,
                                const float* depth_normal, const float* acc_map, const float* rend_dist, double* sums,
                                void* workspace) {
    return loss_forward("srf_loss_forward", stream, V, image_height, image_width, with_reg, image, nullptr, target_hwc,
                        rend_normal, depth_normal, acc_map, rend_dist, sums, workspace);
}

extern "C" int srf_loss_deterministic_workspace_bytes(int V, int image_height, int image_width, size_t* bytes) {
    return loss_workspace_bytes("srf_loss_deterministic_workspace_bytes", V, image_height, image_width, 3, bytes);
}

extern "C" int srf_loss_backward(srf_stream_t stream, int V, int image_height, int image_width, int with_reg,
                                 float w_mse, float w_dist, float w_normal, const float* image, const float* target_hwc,
                                 const float* rend_normal, const float* depth_normal, const float* acc_map,
                                 const float* upstream, float* g_image, float* g_rend_normal, float* g_depth_normal,
                                 float* g_rend_dist) {
    return loss_backward("srf_loss_backward", stream, V, image_height, image_width, with_reg, w_mse, w_dist, w_normal,
                         image, nullptr, target_hwc, rend_normal, depth_normal, acc_map, upstream, g_image, nullptr,
                         g_rend_normal, g_depth_normal, g_rend_dist);
}

extern "C" int srf_loss_passes_forward(srf_stream_t stream, int V, int image_height, int image_width, int with_reg,
                                       const float* image, const float* image_fine, const float* target_hwc,
                                       const float* rend_normal, const float* depth_normal, const float* acc_map,
                                       const float* rend_dist, double* sums, void* workspace) {
    return loss_forward("srf_loss_passes_forward", stream, V, image_height, image_width, with_reg, image, image_fine,
                        target_hwc, rend_normal, depth_normal, acc_map, rend_dist, sums, workspace);
}

extern "C" int srf_loss_passes_deterministic_workspace_bytes(int V, int image_height, int image_width, int with_fine,
                                                             size_t* bytes) {
    return loss_workspace_bytes("srf_loss_passes_deterministic_workspace_bytes", V, image_height, image_width,
                                with_fine ? 4 : 3, bytes);
}

extern "C" int srf_loss_passes_backward(srf_stream_t stream, int V, int image_height, int image_width, int with_reg,
                                        float w_mse, float w_dist, float w_normal, const float* image,
                                        const float* image_fine, const float* target_hwc, const float* rend_normal,
                                        const float* depth_normal, const float* acc_map, const float* upstream,
                                        float* g_image, float* g_image_fine, float* g_rend_normal,
                                        float* g_depth_normal, float* g_rend_dist) {
    return loss_backward("srf_loss_passes_backward", stream, V, image_height, image_width, with_reg, w_mse, w_dist,
                         w_normal, image, image_fine, target_hwc, rend_normal, depth_normal, acc_map, upstream,
                         g_image, g_image_fine, g_rend_normal, g_depth_normal, g_rend_dist);
}
