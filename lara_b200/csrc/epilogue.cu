// epilogue.cu -- fused post-processing of the rasterizer's outputs (SURVEY 8f rank 2).
//
// Restates, as two kernels (forward / backward), the dozen small torch ops of
// LaRa's Renderer.render_img after the rasterizer call (lightning/renderer_2dgs.py:220-268,
// depth_to_normal :74-89): clamp of the colour image, alpha split, normal rotation into
// world space, expected depth = D/alpha with nan_to_num, median depth, surface depth mix,
// pseudo surface normals by central differences of the back-projected depth, alpha-weighted.
// Each of those ops is a full-image HBM round trip in the reference (and again in autograd);
// here one pass reads the 11 input planes + rays and writes the six outputs.
//
// Layouts: color [3,H,W], allmap [8,H,W], rays [H,W,6] (origin xyz, direction xyz),
// viewmatrix [16] (row-major memory of world_view_transform = w2c^T).  Outputs are planar
// [C,H,W]; the Python layer returns the .permute(1,2,0) views the reference returns.  The C entries
// srf_views_epilogue_forward / _backward (include/surfel_rasterizer.h) are defined here.
#include <string.h>

#include "../../include/surfel_rasterizer.h"
#include "surfel_common.cuh"
#include "surfel_kernels.h"

namespace srf {

// all images planar [V,C,H,W] fp32
struct EpilogueArgs {
    int W, H;
    int nviews;
    float depth_ratio;
    const float* color;          // [V,3,H,W] rasterizer colour
    const float* allmap;         // [V,8,H,W] rasterizer aux maps
    const float* rays;           // [V,H,W,6] or null (then no pseudo normals)
    const float* viewmatrix;     // [16] per view, cam_stride floats apart
    size_t cam_stride;
    // forward outputs
    float* image;                // [V,3,H,W]
    float* depth;                // [V,1,H,W]
    float* acc;                  // [V,H,W]
    float* rend_normal;          // [V,3,H,W]
    float* depth_normal;         // [V,3,H,W]
    float* dist;                 // [V,H,W]
    // backward inputs (any may be null = zero) and outputs
    const float* g_image; const float* g_depth; const float* g_acc;
    const float* g_rend_normal; const float* g_depth_normal; const float* g_dist;
    float* scratch;              // [V,3,H,W]
    float* dL_dcolor;            // [V,3,H,W]
    float* dL_dallmap;           // [V,8,H,W]
};

__device__ __forceinline__ float nan_to_num0(float v) {
    // torch.nan_to_num(v, nan=0, posinf=0): NaN and +inf -> 0, -inf -> lowest finite
    if (v != v) return 0.0f;
    if (v == INFINITY) return 0.0f;
    if (v == -INFINITY) return -3.4028234663852886e38f;
    return v;
}

__device__ __forceinline__ float surf_depth_at(const EpilogueArgs& a, size_t pix, size_t npix) {
    const float alpha = a.allmap[pix + npix];
    const float dexp = nan_to_num0(a.allmap[pix] / alpha);
    const float dmed = nan_to_num0(a.allmap[pix + 5 * npix]);
    return dexp * (1.0f - a.depth_ratio) + a.depth_ratio * dmed;
}

__device__ __forceinline__ void point_at(const EpilogueArgs& a, int x, int y, size_t npix, float p[3]) {
    const size_t pix = (size_t)y * a.W + x;
    const float d = surf_depth_at(a, pix, npix);
    const float* r = a.rays + pix * 6;
    p[0] = r[0] + d * r[3]; p[1] = r[1] + d * r[4]; p[2] = r[2] + d * r[5];
}

// blockIdx.z = view: all images are stacked [V,C,H,W] (rays [V,H,W,6]); null pointers stay null
__device__ __forceinline__ void select_view(EpilogueArgs& a) {
    const size_t v = blockIdx.z;
    if (v == 0) return;
    const size_t npix = (size_t)a.W * a.H;
    auto adv = [&](const float*& p, size_t n) { if (p) p += v * n; };
    auto advm = [&](float*& p, size_t n) { if (p) p += v * n; };
    adv(a.color, 3 * npix); adv(a.allmap, 8 * npix); adv(a.rays, 6 * npix);
    a.viewmatrix += v * a.cam_stride;
    advm(a.image, 3 * npix); advm(a.depth, npix); advm(a.acc, npix);
    advm(a.rend_normal, 3 * npix); advm(a.depth_normal, 3 * npix); advm(a.dist, npix);
    adv(a.g_image, 3 * npix); adv(a.g_depth, npix); adv(a.g_acc, npix);
    adv(a.g_rend_normal, 3 * npix); adv(a.g_depth_normal, 3 * npix); adv(a.g_dist, npix);
    advm(a.scratch, 3 * npix); advm(a.dL_dcolor, 3 * npix); advm(a.dL_dallmap, 8 * npix);
}

__global__ void __launch_bounds__(256) epilogue_fwd_kernel(EpilogueArgs a) {
    select_view(a);
    const int x = blockIdx.x * 32 + (threadIdx.x & 31);
    const int y = blockIdx.y * 8 + (threadIdx.x >> 5);
    if (x >= a.W || y >= a.H) return;
    const size_t npix = (size_t)a.W * a.H, pix = (size_t)y * a.W + x;
    const float* vm = a.viewmatrix;
#pragma unroll
    for (int c = 0; c < 3; ++c) a.image[pix + c * npix] = fminf(fmaxf(a.color[pix + c * npix], 0.0f), 1.0f);
    const float alpha = a.allmap[pix + npix];
    a.acc[pix] = alpha;
    const float n0 = a.allmap[pix + 2 * npix], n1 = a.allmap[pix + 3 * npix], n2 = a.allmap[pix + 4 * npix];
    // (n^T @ vm[:3,:3].T)_j = sum_i vm[j][i] n_i
#pragma unroll
    for (int j = 0; j < 3; ++j)
        a.rend_normal[pix + j * npix] = n0 * __ldg(vm + 4 * j) + n1 * __ldg(vm + 4 * j + 1) + n2 * __ldg(vm + 4 * j + 2);
    a.depth[pix] = surf_depth_at(a, pix, npix);
    a.dist[pix] = a.allmap[pix + 6 * npix];
    float nx = 0.f, ny = 0.f, nz = 0.f;
    if (a.rays != nullptr && x >= 1 && x <= a.W - 2 && y >= 1 && y <= a.H - 2) {
        float pu[3], pd[3], pl[3], pr[3];
        point_at(a, x, y + 1, npix, pd); point_at(a, x, y - 1, npix, pu);
        point_at(a, x + 1, y, npix, pr); point_at(a, x - 1, y, npix, pl);
        const float dx0 = pd[0] - pu[0], dx1 = pd[1] - pu[1], dx2 = pd[2] - pu[2];   // along rows ("dx" in the reference)
        const float dy0 = pr[0] - pl[0], dy1 = pr[1] - pl[1], dy2 = pr[2] - pl[2];   // along columns
        const float c0 = dx1 * dy2 - dx2 * dy1, c1 = dx2 * dy0 - dx0 * dy2, c2 = dx0 * dy1 - dx1 * dy0;
        const float len = fmaxf(sqrtf(c0 * c0 + c1 * c1 + c2 * c2), 1e-12f);
        nx = c0 / len * alpha; ny = c1 / len * alpha; nz = c2 / len * alpha;
    }
    a.depth_normal[pix] = nx; a.depth_normal[pix + npix] = ny; a.depth_normal[pix + 2 * npix] = nz;
}

// Backward pass 1: gradient wrt the (unnormalised) cross product of every interior pixel.
__global__ void __launch_bounds__(256) epilogue_bwd_cross_kernel(EpilogueArgs a) {
    select_view(a);
    const int x = blockIdx.x * 32 + (threadIdx.x & 31);
    const int y = blockIdx.y * 8 + (threadIdx.x >> 5);
    if (x >= a.W || y >= a.H) return;
    const size_t npix = (size_t)a.W * a.H, pix = (size_t)y * a.W + x;
    float g0 = 0.f, g1 = 0.f, g2 = 0.f;
    if (a.g_depth_normal != nullptr && x >= 1 && x <= a.W - 2 && y >= 1 && y <= a.H - 2) {
        float pu[3], pd[3], pl[3], pr[3];
        point_at(a, x, y + 1, npix, pd); point_at(a, x, y - 1, npix, pu);
        point_at(a, x + 1, y, npix, pr); point_at(a, x - 1, y, npix, pl);
        const float dx0 = pd[0] - pu[0], dx1 = pd[1] - pu[1], dx2 = pd[2] - pu[2];
        const float dy0 = pr[0] - pl[0], dy1 = pr[1] - pl[1], dy2 = pr[2] - pl[2];
        const float c0 = dx1 * dy2 - dx2 * dy1, c1 = dx2 * dy0 - dx0 * dy2, c2 = dx0 * dy1 - dx1 * dy0;
        const float norm = sqrtf(c0 * c0 + c1 * c1 + c2 * c2);
        const float alpha = a.allmap[pix + npix];   // detached in the reference
        const float G0 = a.g_depth_normal[pix] * alpha, G1 = a.g_depth_normal[pix + npix] * alpha,
                    G2 = a.g_depth_normal[pix + 2 * npix] * alpha;
        if (norm > 1e-12f) {
            const float inv = 1.0f / norm;
            const float n0 = c0 * inv, n1 = c1 * inv, n2 = c2 * inv;
            const float nd = n0 * G0 + n1 * G1 + n2 * G2;
            g0 = (G0 - n0 * nd) * inv; g1 = (G1 - n1 * nd) * inv; g2 = (G2 - n2 * nd) * inv;
        } else {
            g0 = G0 * 1e12f; g1 = G1 * 1e12f; g2 = G2 * 1e12f;   // clamp_min(eps) branch: n = c / eps
        }
        // also keep dx, dy implicitly: pass 2 recomputes them
    }
    a.scratch[pix] = g0; a.scratch[pix + npix] = g1; a.scratch[pix + 2 * npix] = g2;
}

__device__ __forceinline__ void cross3(const float u[3], const float v[3], float o[3]) {
    o[0] = u[1] * v[2] - u[2] * v[1]; o[1] = u[2] * v[0] - u[0] * v[2]; o[2] = u[0] * v[1] - u[1] * v[0];
}

// d(loss)/d(p_q) contribution of centre (cx,cy): sign * (dy x gc) for the row neighbours,
// sign * (gc x dx) for the column neighbours.
__device__ __forceinline__ void add_center(const EpilogueArgs& a, int cx, int cy, size_t npix, bool row_term, float sign,
                                           float acc[3]) {
    if (cx < 1 || cx > a.W - 2 || cy < 1 || cy > a.H - 2) return;
    const size_t cp = (size_t)cy * a.W + cx;
    const float gc[3] = {a.scratch[cp], a.scratch[cp + npix], a.scratch[cp + 2 * npix]};
    if (gc[0] == 0.f && gc[1] == 0.f && gc[2] == 0.f) return;
    float t[3];
    if (row_term) {          // c = dx x dy, dL/d(dx) = dy x gc
        float pl[3], pr[3];
        point_at(a, cx + 1, cy, npix, pr); point_at(a, cx - 1, cy, npix, pl);
        const float dy[3] = {pr[0] - pl[0], pr[1] - pl[1], pr[2] - pl[2]};
        cross3(dy, gc, t);
    } else {                 // dL/d(dy) = gc x dx
        float pu[3], pd[3];
        point_at(a, cx, cy + 1, npix, pd); point_at(a, cx, cy - 1, npix, pu);
        const float dx[3] = {pd[0] - pu[0], pd[1] - pu[1], pd[2] - pu[2]};
        cross3(gc, dx, t);
    }
    acc[0] += sign * t[0]; acc[1] += sign * t[1]; acc[2] += sign * t[2];
}

__global__ void __launch_bounds__(256) epilogue_bwd_kernel(EpilogueArgs a) {
    select_view(a);
    const int x = blockIdx.x * 32 + (threadIdx.x & 31);
    const int y = blockIdx.y * 8 + (threadIdx.x >> 5);
    if (x >= a.W || y >= a.H) return;
    const size_t npix = (size_t)a.W * a.H, pix = (size_t)y * a.W + x;
    const float* vm = a.viewmatrix;
    // colour: clamp passes the gradient where 0 <= c <= 1
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float v = a.color[pix + c * npix];
        const float g = a.g_image ? a.g_image[pix + c * npix] : 0.f;
        a.dL_dcolor[pix + c * npix] = (v >= 0.0f && v <= 1.0f) ? g : 0.0f;
    }
    // surface-depth gradient: direct + the four neighbouring pseudo-normals
    float g_sd = a.g_depth ? a.g_depth[pix] : 0.f;
    if (a.g_depth_normal != nullptr && a.rays != nullptr) {
        float gp[3] = {0.f, 0.f, 0.f};
        add_center(a, x, y - 1, npix, true, 1.0f, gp);    // this pixel is p[y+1] of the centre above
        add_center(a, x, y + 1, npix, true, -1.0f, gp);   // ... and p[y-1] of the centre below
        add_center(a, x - 1, y, npix, false, 1.0f, gp);   // p[x+1] of the centre to the left
        add_center(a, x + 1, y, npix, false, -1.0f, gp);  // p[x-1] of the centre to the right
        const float* r = a.rays + pix * 6;
        g_sd += gp[0] * r[3] + gp[1] * r[4] + gp[2] * r[5];
    }
    const float D = a.allmap[pix], alpha = a.allmap[pix + npix], dmed_raw = a.allmap[pix + 5 * npix];
    const float q = D / alpha;
    const bool q_ok = (q == q) && (q != INFINITY) && (q != -INFINITY);
    const bool m_ok = (dmed_raw == dmed_raw) && (dmed_raw != INFINITY) && (dmed_raw != -INFINITY);
    const float g_exp = q_ok ? g_sd * (1.0f - a.depth_ratio) : 0.0f;
    float d_alpha = a.g_acc ? a.g_acc[pix] : 0.f;
    float d_D = 0.f;
    if (q_ok) {
        d_D = g_exp / alpha;
        // torch's div backward, -g * ((D / alpha) / alpha): alpha * alpha would underflow to 0 below alpha ~ 1e-19
        d_alpha += -g_exp * (q / alpha);
    }
    a.dL_dallmap[pix] = d_D;
    a.dL_dallmap[pix + npix] = d_alpha;
    float gn[3] = {0.f, 0.f, 0.f};
    if (a.g_rend_normal) { gn[0] = a.g_rend_normal[pix]; gn[1] = a.g_rend_normal[pix + npix]; gn[2] = a.g_rend_normal[pix + 2 * npix]; }
#pragma unroll
    for (int i = 0; i < 3; ++i)
        a.dL_dallmap[pix + (2 + i) * npix] = gn[0] * __ldg(vm + i) + gn[1] * __ldg(vm + 4 + i) + gn[2] * __ldg(vm + 8 + i);
    a.dL_dallmap[pix + 5 * npix] = m_ok ? g_sd * a.depth_ratio : 0.0f;
    a.dL_dallmap[pix + 6 * npix] = a.g_dist ? a.g_dist[pix] : 0.f;
    a.dL_dallmap[pix + 7 * npix] = 0.0f;
}

}  // namespace srf

using srf::cuda_error;
using srf::set_error;

extern "C" int srf_views_epilogue_forward(srf_stream_t stream, int V, int image_height, int image_width,
                                          float depth_ratio, const float* color, const float* allmap, const float* rays,
                                          const float* cams, float* image, float* depth, float* acc_map,
                                          float* rend_normal, float* depth_normal, float* rend_dist) {
    const char* fn = "srf_views_epilogue_forward";
    if (V <= 0 || image_height <= 0 || image_width <= 0) return set_error("%s: bad sizes", fn);
    if (!color || !allmap || !cams || !image || !depth || !acc_map || !rend_normal || !depth_normal || !rend_dist)
        return set_error("%s: null pointer", fn);
    srf::EpilogueArgs a;
    memset(&a, 0, sizeof(a));
    a.W = image_width; a.H = image_height; a.nviews = V; a.depth_ratio = depth_ratio;
    a.color = color; a.allmap = allmap; a.rays = rays; a.viewmatrix = cams + SRF_CAM_VIEW; a.cam_stride = SRF_CAM_FLOATS;
    a.image = image; a.depth = depth; a.acc = acc_map; a.rend_normal = rend_normal; a.depth_normal = depth_normal;
    a.dist = rend_dist;
    const dim3 grid((a.W + 31) / 32, (a.H + 7) / 8, V);
    srf::epilogue_fwd_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(a);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_error("epilogue_fwd launch", e);
}

extern "C" int srf_views_epilogue_backward(srf_stream_t stream_, int V, int image_height, int image_width,
                                           float depth_ratio, const float* color, const float* allmap,
                                           const float* rays, const float* cams, const float* g_image,
                                           const float* g_depth, const float* g_acc_map, const float* g_rend_normal,
                                           const float* g_depth_normal, const float* g_rend_dist, float* scratch,
                                           float* dL_dcolor, float* dL_dallmap) {
    const char* fn = "srf_views_epilogue_backward";
    if (V <= 0 || image_height <= 0 || image_width <= 0) return set_error("%s: bad sizes", fn);
    if (!color || !allmap || !cams || !dL_dcolor || !dL_dallmap) return set_error("%s: null pointer", fn);
    if (g_depth_normal && rays && !scratch) return set_error("%s: scratch [V,3,H,W] required", fn);
    srf::EpilogueArgs a;
    memset(&a, 0, sizeof(a));
    a.W = image_width; a.H = image_height; a.nviews = V; a.depth_ratio = depth_ratio;
    a.color = color; a.allmap = allmap; a.rays = rays; a.viewmatrix = cams + SRF_CAM_VIEW; a.cam_stride = SRF_CAM_FLOATS;
    a.g_image = g_image; a.g_depth = g_depth; a.g_acc = g_acc_map; a.g_rend_normal = g_rend_normal;
    a.g_depth_normal = g_depth_normal; a.g_dist = g_rend_dist;
    a.scratch = scratch; a.dL_dcolor = dL_dcolor; a.dL_dallmap = dL_dallmap;
    const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const dim3 grid((a.W + 31) / 32, (a.H + 7) / 8, V);
    // pass 1 (the pseudo normals' cross-product gradients) only when they have a gradient
    if (g_depth_normal && rays) srf::epilogue_bwd_cross_kernel<<<grid, 256, 0, stream>>>(a);
    srf::epilogue_bwd_kernel<<<grid, 256, 0, stream>>>(a);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_error("epilogue_bwd launch", e);
}
