// point_feats.cu -- the fine pass's point-feature sampler (LaRa Network.get_point_feats, lightning/network.py:390-411,
// with projection() at :182-187), forward and backward, one thread per point.
//
// For each of the n (masked) Gaussian centres and each of the V source views:
//   p = K (R x + t)  with w2c [V,4,4] and K [V,3,3] row-major;  xy = p.xy / p.z,  z = p.z
//   g = (xy + 0.5) / [W,H] * 2 - 1                    (network.py:401)
//   ix = ((g.x + 1) W - 1) / 2,  iy = ((g.y + 1) H - 1) / 2   (grid_sample's unnormalisation, align_corners=False)
//   feats[v, c, i] = bilinear sample, zero padding, of the 8-channel stack
//                    img_ref(3) | image(3) | acc_map(1) | depth(1),   channel 7 replaced by |s_depth - z|
// The chain of roundings is kept as written: folding it to ix = x moves points across pixel-centre lines at the
// ulp level, and those lines are where the point gradient jumps.  The projection sums in the order of a k-ordered
// FMA loop, the tap weights are grid_sampler_2d's.
//
// A tap is used only if its sample coordinate is finite and its integer index lies in the image: the bounds are
// tested on the floored float before any conversion, so no input can make the kernels read outside the images.
// A point in a source camera's plane (z = 0) thus samples 0 and gets no gradient through the grid.
//
// Backward: the upstream gradient g[V,8,n] is read coalesced; dL/dpoints[n,3] is summed over the views in registers
// and written once; the gradients of the 5 differentiable channels go into planar g_image[V,3,H,W], g_acc[V,H,W]
// and g_depth[V,H,W] with red.global.add.f32 (cleared by the caller).  No gradient is formed for img_ref.
#include "surfel_kernels.h"

namespace srf {
namespace {

constexpr int kPfThreads = 256;

struct PfTaps {
    float tx0, tx1, ty0, ty1;    // ix - floor(ix), floor(ix) + 1 - ix, same for y
    float w[4];                  // nw, ne, sw, se
    int off[4];                  // y * W + x of each tap, -1 = not used
    bool any;
};

// p = K (R x + t) for view v; returns xy / z in xy, z in z
__device__ __forceinline__ void pf_project(const PointFeatsArgs& a, int v, float x0, float x1, float x2,
                                           float& px, float& py, float& pz, float m[21]) {
    const float* E = a.w2cs + 16 * (size_t)v;
    const float* K = a.ixts + 9 * (size_t)v;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
#pragma unroll
        for (int k = 0; k < 4; ++k) m[4 * r + k] = __ldg(E + 4 * r + k);
    }
#pragma unroll
    for (int k = 0; k < 9; ++k) m[12 + k] = __ldg(K + k);
    float q[3];
#pragma unroll
    for (int r = 0; r < 3; ++r)      // points @ R^T, then + t (two torch ops)
        q[r] = __fadd_rn(__fmaf_rn(x2, m[4 * r + 2], __fmaf_rn(x1, m[4 * r + 1], __fmul_rn(x0, m[4 * r]))), m[4 * r + 3]);
    float p[3];
#pragma unroll
    for (int r = 0; r < 3; ++r)      // @ K^T
        p[r] = __fmaf_rn(q[2], m[12 + 3 * r + 2], __fmaf_rn(q[1], m[12 + 3 * r + 1], __fmul_rn(q[0], m[12 + 3 * r])));
    px = p[0]; py = p[1]; pz = p[2];
}

// network.py:401 followed by grid_sample's unnormalisation, one rounding per torch operation
__device__ __forceinline__ float pf_source_coord(float xy, float size) {
    const float g = __fadd_rn(__fmul_rn(__fdiv_rn(__fadd_rn(xy, 0.5f), size), 2.0f), -1.0f);
    return __fdiv_rn(__fadd_rn(__fmul_rn(__fadd_rn(g, 1.0f), size), -1.0f), 2.0f);
}

__device__ __forceinline__ PfTaps pf_taps(float ix, float iy, int W, int H) {
    PfTaps t;
    const float fx = floorf(ix), fy = floorf(iy);
    t.tx1 = __fsub_rn(__fadd_rn(fx, 1.0f), ix); t.tx0 = __fsub_rn(ix, fx);
    t.ty1 = __fsub_rn(__fadd_rn(fy, 1.0f), iy); t.ty0 = __fsub_rn(iy, fy);
    t.w[0] = __fmul_rn(t.tx1, t.ty1);    // nw = (ix_se - ix) * (iy_se - iy)
    t.w[1] = __fmul_rn(t.tx0, t.ty1);    // ne = (ix - ix_sw) * (iy_sw - iy)
    t.w[2] = __fmul_rn(t.tx1, t.ty0);    // sw = (ix_ne - ix) * (iy - iy_ne)
    t.w[3] = __fmul_rn(t.tx0, t.ty0);    // se = (ix - ix_nw) * (iy - iy_nw)
    // comparisons with NaN are false and +-inf fails one side: non-finite coordinates use no tap
    const bool x0 = fx >= 0.0f && fx <= (float)(W - 1), x1 = fx >= -1.0f && fx <= (float)(W - 2);
    const bool y0 = fy >= 0.0f && fy <= (float)(H - 1), y1 = fy >= -1.0f && fy <= (float)(H - 2);
    const int xi = (x0 || x1) ? (int)fx : 0, yi = (y0 || y1) ? (int)fy : 0;
    t.off[0] = (x0 && y0) ? yi * W + xi : -1;
    t.off[1] = (x1 && y0) ? yi * W + xi + 1 : -1;
    t.off[2] = (x0 && y1) ? (yi + 1) * W + xi : -1;
    t.off[3] = (x1 && y1) ? (yi + 1) * W + xi + 1 : -1;
    t.any = (x0 || x1) && (y0 || y1);
    return t;
}

// plane of channel c (0..7) of view v in the stack img_ref | image | acc | depth
__device__ __forceinline__ const float* pf_plane(const PointFeatsArgs& a, int v, int c, size_t HW) {
    if (c < 3) return a.img_ref + ((size_t)v * 3 + c) * HW;
    if (c < 6) return a.image + ((size_t)v * 3 + (c - 3)) * HW;
    return (c == 6 ? a.acc : a.depth) + (size_t)v * HW;
}

__device__ __forceinline__ float pf_sample(const float* plane, const PfTaps& t, float vals[4]) {
    float s = 0.0f;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        vals[k] = t.off[k] >= 0 ? __ldg(plane + t.off[k]) : 0.0f;
        if (t.off[k] >= 0) s = __fmaf_rn(vals[k], t.w[k], s);
    }
    return s;
}

__device__ __forceinline__ void pf_red(float* p, float v) {
    asm volatile("red.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}

__global__ void __launch_bounds__(kPfThreads) point_feats_fwd_kernel(PointFeatsArgs a) {
    const int i = blockIdx.x * kPfThreads + threadIdx.x;
    if (i >= a.n) return;
    const float x0 = a.points[3 * (size_t)i], x1 = a.points[3 * (size_t)i + 1], x2 = a.points[3 * (size_t)i + 2];
    const size_t HW = (size_t)a.H * a.W, n = (size_t)a.n;
    for (int v = 0; v < a.V; ++v) {
        float px, py, pz, m[21];
        pf_project(a, v, x0, x1, x2, px, py, pz, m);
        const float ix = pf_source_coord(__fdiv_rn(px, pz), (float)a.W);
        const float iy = pf_source_coord(__fdiv_rn(py, pz), (float)a.H);
        const PfTaps t = pf_taps(ix, iy, a.W, a.H);
        float* out = a.feats + (size_t)v * 8 * n + i;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            float vals[4];
            float s = pf_sample(pf_plane(a, v, c, HW), t, vals);
            if (c == 7) s = fabsf(__fsub_rn(s, pz));      // z_diff = |s_depth - z|
            out[c * n] = s;
        }
    }
}

__global__ void __launch_bounds__(kPfThreads) point_feats_bwd_kernel(PointFeatsArgs a) {
    const int i = blockIdx.x * kPfThreads + threadIdx.x;
    if (i >= a.n) return;
    const float x0 = a.points[3 * (size_t)i], x1 = a.points[3 * (size_t)i + 1], x2 = a.points[3 * (size_t)i + 2];
    const size_t HW = (size_t)a.H * a.W, n = (size_t)a.n;
    float gx0 = 0.0f, gx1 = 0.0f, gx2 = 0.0f;           // dL/dpoint, summed over the views
    for (int v = 0; v < a.V; ++v) {
        float px, py, pz, m[21];
        pf_project(a, v, x0, x1, x2, px, py, pz, m);
        const float xs = __fdiv_rn(px, pz), ys = __fdiv_rn(py, pz);
        const PfTaps t = pf_taps(pf_source_coord(xs, (float)a.W), pf_source_coord(ys, (float)a.H), a.W, a.H);
        const float* g = a.g_feats + (size_t)v * 8 * n + i;
        // z_diff = |s_depth - z|: vjp with sign(0) = 0
        float dvals[4];
        const float sd = pf_sample(pf_plane(a, v, 7, HW), t, dvals);
        const float d = __fsub_rn(sd, pz);
        const float sgn = d > 0.0f ? 1.0f : (d < 0.0f ? -1.0f : 0.0f);
        const float g7 = g[7 * n];
        const float g_sd = g7 * sgn;
        float gix = 0.0f, giy = 0.0f;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const float go = c == 7 ? g_sd : g[c * n];
            float vals[4];
            if (c == 7) {
#pragma unroll
                for (int k = 0; k < 4; ++k) vals[k] = dvals[k];
            } else if (a.g_points) {
                pf_sample(pf_plane(a, v, c, HW), t, vals);
            }
            if (a.g_points) {   // grid_sampler_2d_backward's gix / giy, untouched taps read as 0
                gix = __fmaf_rn(go, __fadd_rn(__fmul_rn(__fsub_rn(vals[1], vals[0]), t.ty1), __fmul_rn(__fsub_rn(vals[3], vals[2]), t.ty0)), gix);
                giy = __fmaf_rn(go, __fadd_rn(__fmul_rn(__fsub_rn(vals[2], vals[0]), t.tx1), __fmul_rn(__fsub_rn(vals[3], vals[1]), t.tx0)), giy);
            }
            float* dst = nullptr;
            if (c >= 3 && c < 6) dst = a.g_image ? a.g_image + ((size_t)v * 3 + (c - 3)) * HW : nullptr;
            else if (c == 6) dst = a.g_acc ? a.g_acc + (size_t)v * HW : nullptr;
            else if (c == 7) dst = a.g_depth ? a.g_depth + (size_t)v * HW : nullptr;
            if (dst && go != 0.0f) {
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    if (t.off[k] >= 0) pf_red(dst + t.off[k], __fmul_rn(t.w[k], go));
            }
        }
        if (!a.g_points) continue;
        // back through ix = ((g+1) W - 1)/2, g = (x + 0.5)/W*2 - 1: dL/dx = gix * (W/2) * 2 / W
        float dpx = 0.0f, dpy = 0.0f, dpz = -g_sd;        // z enters z_diff directly
        if (t.any) {                                      // then xs, ys and 1/pz are finite
            const float gxs = __fdiv_rn(__fmul_rn(__fmul_rn(gix, 0.5f * (float)a.W), 2.0f), (float)a.W);
            const float gys = __fdiv_rn(__fmul_rn(__fmul_rn(giy, 0.5f * (float)a.H), 2.0f), (float)a.H);
            dpx = __fdiv_rn(gxs, pz);
            dpy = __fdiv_rn(gys, pz);
            dpz = __fsub_rn(dpz, __fadd_rn(__fmul_rn(gxs, __fdiv_rn(xs, pz)), __fmul_rn(gys, __fdiv_rn(ys, pz))));
        }
        // p = K q, q = R x + t
        float dq[3], dx[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) dq[k] = dpx * m[12 + k] + dpy * m[15 + k] + dpz * m[18 + k];
#pragma unroll
        for (int k = 0; k < 3; ++k) dx[k] = dq[0] * m[k] + dq[1] * m[4 + k] + dq[2] * m[8 + k];
        gx0 += dx[0]; gx1 += dx[1]; gx2 += dx[2];
    }
    if (a.g_points) {
        a.g_points[3 * (size_t)i] = gx0;
        a.g_points[3 * (size_t)i + 1] = gx1;
        a.g_points[3 * (size_t)i + 2] = gx2;
    }
}

}  // namespace

cudaError_t launch_point_feats(const PointFeatsArgs& a, bool backward, cudaStream_t stream) {
    if (a.n <= 0) return cudaSuccess;
    const unsigned grid = (unsigned)((a.n + kPfThreads - 1) / kPfThreads);
    if (backward) point_feats_bwd_kernel<<<grid, kPfThreads, 0, stream>>>(a);
    else point_feats_fwd_kernel<<<grid, kPfThreads, 0, stream>>>(a);
    return cudaGetLastError();
}

}  // namespace srf
