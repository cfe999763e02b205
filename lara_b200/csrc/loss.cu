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
//   loss_grads_kernel: one pass writing g_image / g_rend_normal / g_depth_normal / g_rend_dist, already planar
//                      and stacked, i.e. exactly what srf_views_epilogue_backward consumes -- scaled by the upstream
//                      scalar read from device memory (no host sync).
// `target` is read in the batch's own channel-last layout [V,H,W,3] (lightning/loss.py:24 permutes a view of it).
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
    const float* target;         // [V,H,W,3] channel-last, the batch's own layout
    const float* rend_normal;    // [V,3,H,W]
    const float* depth_normal;   // [V,3,H,W]
    const float* acc;            // [V,H,W]
    const float* dist;           // [V,H,W]
    double* sums;                // [3]: sum (image-target)^2, sum dist, sum (1 - <rn,dn>) acc   (zeroed by the caller); null = skip
    double* partials;            // [loss_det_blocks][3] or null: deterministic sums (written, then reduced in a fixed order)
    const float* gout;           // device scalar: upstream gradient of the loss (null = 1)
    float* g_image;              // [V,3,H,W] out (may be null: forward statistics only)
    float* g_rend_normal; float* g_depth_normal; float* g_dist;
};

template <bool kDet>
__global__ void __launch_bounds__(256) loss_sums_kernel(LossArgs a) {
    const size_t npix = (size_t)a.W * a.H, total = npix * (size_t)a.nviews;
    float s_mse = 0.f, s_dist = 0.f, s_norm = 0.f;
    for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (size_t)gridDim.x * 256) {
        const size_t v = i / npix, pix = i - v * npix;
        const float* img = a.image + v * 3 * npix + pix;
        const float* tar = a.target + i * 3;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float d = img[c * npix] - __ldg(tar + c);
            s_mse = fmaf(d, d, s_mse);
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
    __shared__ float s_part[3][8];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        s_mse += __shfl_xor_sync(0xffffffffu, s_mse, o);
        s_dist += __shfl_xor_sync(0xffffffffu, s_dist, o);
        s_norm += __shfl_xor_sync(0xffffffffu, s_norm, o);
    }
    if (lane == 0) { s_part[0][wid] = s_mse; s_part[1][wid] = s_dist; s_part[2][wid] = s_norm; }
    __syncthreads();
    if (threadIdx.x < 3) {
        double t = 0.0;
#pragma unroll
        for (int w = 0; w < 8; ++w) t += (double)s_part[threadIdx.x][w];
        if (kDet) a.partials[3 * blockIdx.x + threadIdx.x] = t;
        else atomicAdd(a.sums + threadIdx.x, t);
    }
}

// blocks (= partial-sum triples) of the deterministic sums: a grid that does not depend on the device, so the same
// partials, and the same bits, on every GPU
static size_t loss_det_blocks(size_t total) { return min((size_t)1024, (total + 255) / 256); }

// deterministic path: the per-block partials of loss_sums_kernel<true> summed in a fixed order, warp w for term w
__global__ void __launch_bounds__(96) loss_sums_finalize_kernel(const double* partials, int nblocks, double* sums) {
    const int term = threadIdx.x >> 5;
    const double t = warp_strided_sum(partials + term, nblocks, 3);
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
#pragma unroll
    for (int c = 0; c < 3; ++c) gi[c * npix] = k_mse * (img[c * npix] - __ldg(tar + c));
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

extern "C" int srf_loss_forward(srf_stream_t stream_, int V, int image_height, int image_width, int with_reg,
                                const float* image, const float* target_hwc, const float* rend_normal,
                                const float* depth_normal, const float* acc_map, const float* rend_dist, double* sums,
                                void* workspace) {
    if (V <= 0 || image_height <= 0 || image_width <= 0) return set_error("srf_loss_forward: bad sizes");
    if (!image || !target_hwc || !sums) return set_error("srf_loss_forward: null pointer");
    if (with_reg && (!rend_normal || !depth_normal || !acc_map || !rend_dist)) return set_error("srf_loss_forward: null regulariser input");
    if (reinterpret_cast<uintptr_t>(workspace) & 7) return set_error("srf_loss_forward: workspace must be 8-byte aligned");
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    cudaError_t e;
    // the deterministic path writes every sum from its partials; the atomics need zeroed sums
    if (!workspace && (e = cudaMemsetAsync(sums, 0, 3 * sizeof(double), stream)) != cudaSuccess)
        return cuda_error("memset loss sums", e);
    srf::LossArgs a;
    memset(&a, 0, sizeof(a));
    a.W = image_width; a.H = image_height; a.nviews = V; a.with_reg = with_reg ? 1 : 0;
    a.image = image; a.target = target_hwc; a.rend_normal = rend_normal; a.depth_normal = depth_normal;
    a.acc = acc_map; a.dist = rend_dist; a.sums = sums; a.partials = static_cast<double*>(workspace);
    const size_t total = (size_t)image_width * image_height * (size_t)V;
    if (workspace) {
        const int grid = (int)srf::loss_det_blocks(total);
        srf::loss_sums_kernel<true><<<grid, 256, 0, stream>>>(a);
        srf::loss_sums_finalize_kernel<<<1, 96, 0, stream>>>(a.partials, grid, a.sums);
    } else {
        const int grid = (int)min((size_t)srf::sm_count() * 8, (total + 255) / 256);
        srf::loss_sums_kernel<false><<<grid, 256, 0, stream>>>(a);
    }
    e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_error("loss_sums launch", e);
}

extern "C" int srf_loss_deterministic_workspace_bytes(int V, int image_height, int image_width, size_t* bytes) {
    if (V <= 0 || image_height <= 0 || image_width <= 0 || !bytes)
        return set_error("srf_loss_deterministic_workspace_bytes: bad arguments");
    *bytes = srf::loss_det_blocks((size_t)V * image_height * image_width) * 3 * sizeof(double);
    return 0;
}

extern "C" int srf_loss_backward(srf_stream_t stream, int V, int image_height, int image_width, int with_reg,
                                 float w_mse, float w_dist, float w_normal, const float* image, const float* target_hwc,
                                 const float* rend_normal, const float* depth_normal, const float* acc_map,
                                 const float* upstream, float* g_image, float* g_rend_normal, float* g_depth_normal,
                                 float* g_rend_dist) {
    if (V <= 0 || image_height <= 0 || image_width <= 0) return set_error("srf_loss_backward: bad sizes");
    if (!image || !target_hwc || !g_image) return set_error("srf_loss_backward: null pointer");
    if (with_reg && (!rend_normal || !depth_normal || !acc_map || !g_rend_normal || !g_depth_normal || !g_rend_dist))
        return set_error("srf_loss_backward: null regulariser pointer");
    srf::LossArgs a;
    memset(&a, 0, sizeof(a));
    a.W = image_width; a.H = image_height; a.nviews = V; a.with_reg = with_reg ? 1 : 0;
    a.w_mse = w_mse; a.w_dist = w_dist; a.w_normal = w_normal;
    a.image = image; a.target = target_hwc; a.rend_normal = rend_normal; a.depth_normal = depth_normal; a.acc = acc_map;
    a.gout = upstream;
    a.g_image = g_image; a.g_rend_normal = g_rend_normal; a.g_depth_normal = g_depth_normal; a.g_dist = g_rend_dist;
    const size_t total = (size_t)image_width * image_height * (size_t)V;
    srf::loss_grads_kernel<<<(unsigned)((total + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(a);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_error("loss_grads launch", e);
}
