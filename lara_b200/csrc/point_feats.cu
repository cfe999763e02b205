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
// FMA loop, the tap weights are grid_sampler_2d's.  Projection, coordinate chain and taps are in sample_taps.cuh,
// shared with feat_volume.cu.
//
// A tap is used only if its sample coordinate is finite and its integer index lies in the image: the bounds are
// tested on the floored float before any conversion, so no input can make the kernels read outside the images.
// A point in a source camera's plane (z = 0) thus samples 0 and gets no gradient through the grid.
//
// Backward: the upstream gradient g[V,8,n] is read coalesced; dL/dpoints[n,3] is summed over the views in registers
// and written once; the gradients of the 5 differentiable channels go into planar g_image[V,3,H,W], g_acc[V,H,W]
// and g_depth[V,H,W] with red.global.add.f32 (cleared by the entry).  No gradient is formed for img_ref.
// The C entries srf_point_feats_* (include/surfel_rasterizer.h) are defined here.
#include <string.h>

#include "../../include/surfel_rasterizer.h"
#include "det_sum.cuh"
#include "sample_taps.cuh"
#include "surfel_kernels.h"

namespace srf {

// n points sampled in V source views from the 8-channel stack img_ref | image | acc | depth; all images planar fp32
struct PointFeatsArgs {
    int V, n, H, W;
    const float* points;         // [n,3]
    const float* w2cs;           // [V,4,4] row-major
    const float* ixts;           // [V,3,3] row-major
    const float* img_ref;        // [V,3,H,W]
    const float* image;          // [V,3,H,W]
    const float* acc;            // [V,H,W]
    const float* depth;          // [V,H,W]
    float* feats;                // [V,8,n] forward output
    const float* g_feats;        // [V,8,n] backward input
    float* g_points;             // [n,3] written (may be null)
    float* g_image; float* g_acc; float* g_depth;   // accumulated into, cleared by the entry (each may be null)
    // deterministic backward (null = default): int64 planes [5V,H,W] in the layout g_image | g_acc | g_depth and a
    // header det[0] = max |g_feats| (fp32 bits), det[1] = overflow; both zeroed by the entry.  The float outputs are
    // then written, not accumulated into.
    long long* g_fixed;
    uint32_t* det;
};

namespace {

constexpr int kPfThreads = 256;

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
        pf_project(a.w2cs + 16 * (size_t)v, a.ixts + 9 * (size_t)v, x0, x1, x2, px, py, pz, m);
        const float ix = pf_source_coord(__fdiv_rn(px, pz), (float)a.W, (float)a.W);
        const float iy = pf_source_coord(__fdiv_rn(py, pz), (float)a.H, (float)a.H);
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

__device__ __forceinline__ void pf_red_u64(long long* p, long long v) {
    asm volatile("red.global.add.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// Deterministic backward (DESIGN §3.13): every term a tap adds into a rendering gradient is w go with w <= 1 and
// |go| <= max |g_feats|, and a pixel of a plane receives at most 4 V n of them.  The bound kernel takes that max
// (det[0], fp32 bits); the backward adds the terms in 64-bit fixed point into planes laid out as g_image | g_acc |
// g_depth; the convert kernel writes the fp32 results.  det[1] is set if a term was over its budget or not finite.
__global__ void __launch_bounds__(kPfThreads) pf_bound_kernel(const float* g, size_t count, uint32_t* det) {
    uint32_t m = 0;
    for (size_t i = (size_t)blockIdx.x * kPfThreads + threadIdx.x; i < count; i += (size_t)gridDim.x * kPfThreads)
        m = max(m, det::abs_bits(__ldg(g + i)));
    m = __reduce_max_sync(0xffffffffu, m);
    if ((threadIdx.x & 31) == 0 && m != 0u) atomicMax(det, m);
}

__global__ void __launch_bounds__(kPfThreads) pf_convert_kernel(PointFeatsArgs a) {
    const size_t HW = (size_t)a.H * a.W, n_img = 3 * (size_t)a.V * HW, n_one = (size_t)a.V * HW;
    const size_t j = (size_t)blockIdx.x * kPfThreads + threadIdx.x;
    if (j >= n_img + 2 * n_one) return;
    const int L = det::ceil_log2(4ull * (uint64_t)a.V * (uint64_t)a.n);
    const int k = det::scale_exp(__ldg(a.det), L);
    float* dst = j < n_img ? (a.g_image ? a.g_image + j : nullptr)
               : j < n_img + n_one ? (a.g_acc ? a.g_acc + (j - n_img) : nullptr)
                                   : (a.g_depth ? a.g_depth + (j - n_img - n_one) : nullptr);
    if (dst) *dst = det::to_float(a.g_fixed[j], k);
}

template <bool kDet>
__global__ void __launch_bounds__(kPfThreads) point_feats_bwd_kernel(PointFeatsArgs a) {
    const int i = blockIdx.x * kPfThreads + threadIdx.x;
    if (i >= a.n) return;
    int L = 0, kq = 0;
    bool ok = true;
    if (kDet) {
        L = det::ceil_log2(4ull * (uint64_t)a.V * (uint64_t)a.n);
        kq = det::scale_exp(__ldg(a.det), L);
    }
    const float x0 = a.points[3 * (size_t)i], x1 = a.points[3 * (size_t)i + 1], x2 = a.points[3 * (size_t)i + 2];
    const size_t HW = (size_t)a.H * a.W, n = (size_t)a.n;
    float gx0 = 0.0f, gx1 = 0.0f, gx2 = 0.0f;           // dL/dpoint, summed over the views
    for (int v = 0; v < a.V; ++v) {
        float px, py, pz, m[21];
        pf_project(a.w2cs + 16 * (size_t)v, a.ixts + 9 * (size_t)v, x0, x1, x2, px, py, pz, m);
        const float xs = __fdiv_rn(px, pz), ys = __fdiv_rn(py, pz);
        const PfTaps t = pf_taps(pf_source_coord(xs, (float)a.W, (float)a.W),
                                 pf_source_coord(ys, (float)a.H, (float)a.H), a.W, a.H);
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
                if (kDet) {
                    const size_t plane = c < 6 ? (size_t)v * 3 + (c - 3) : (size_t)(c == 6 ? 3 : 4) * a.V + v;
                    long long* qd = a.g_fixed + plane * HW;
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        if (t.off[k] < 0) continue;
                        long long q;
                        ok &= det::quantize(__fmul_rn(t.w[k], go), kq, L, q);
                        if (q != 0) pf_red_u64(qd + t.off[k], q);
                    }
                } else {
#pragma unroll
                    for (int k = 0; k < 4; ++k)
                        if (t.off[k] >= 0) pf_red(dst + t.off[k], __fmul_rn(t.w[k], go));
                }
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
    if (kDet && !ok) atomicOr(a.det + 1, 1u);
    if (a.g_points) {
        a.g_points[3 * (size_t)i] = gx0;
        a.g_points[3 * (size_t)i + 1] = gx1;
        a.g_points[3 * (size_t)i + 2] = gx2;
    }
}

}  // namespace

}  // namespace srf

using srf::cuda_error;
using srf::set_error;

static int point_feats_check(const char* fn, int V, int n, int H, int W, const float* points, const float* w2cs,
                             const float* ixts, const float* img_ref, const float* image, const float* acc,
                             const float* depth) {
    if (V <= 0 || n < 0 || H <= 0 || W <= 0) return set_error("%s: bad sizes (V=%d, n=%d, H=%d, W=%d)", fn, V, n, H, W);
    if (H > (1 << 24) || W > (1 << 24)) return set_error("%s: image too large", fn);    // pixel indices exact in fp32
    // an empty point set has no storage: points (and feats / g_feats) are only needed when n > 0
    if ((n > 0 && !points) || !w2cs || !ixts || !img_ref || !image || !acc || !depth) return set_error("%s: null input pointer", fn);
    return 0;
}

extern "C" int srf_point_feats_forward(srf_stream_t stream, int V, int n, int H, int W, const float* points,
                                       const float* w2cs, const float* ixts, const float* img_ref, const float* image,
                                       const float* acc, const float* depth, float* feats) {
    const char* fn = "srf_point_feats_forward";
    if (point_feats_check(fn, V, n, H, W, points, w2cs, ixts, img_ref, image, acc, depth)) return 1;
    if (n > 0 && !feats) return set_error("%s: null output pointer", fn);
    if (n == 0) return 0;
    srf::PointFeatsArgs a;
    memset(&a, 0, sizeof(a));
    a.V = V; a.n = n; a.H = H; a.W = W;
    a.points = points; a.w2cs = w2cs; a.ixts = ixts; a.img_ref = img_ref; a.image = image; a.acc = acc; a.depth = depth;
    a.feats = feats;
    const unsigned grid = (unsigned)((n + srf::kPfThreads - 1) / srf::kPfThreads);
    srf::point_feats_fwd_kernel<<<grid, srf::kPfThreads, 0, static_cast<cudaStream_t>(stream)>>>(a);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_error("point_feats_fwd launch", e);
}

// deterministic workspace: header (max |g_feats|, overflow flag), then the int64 planes g_image | g_acc | g_depth
static size_t pf_det_planes_offset() { return 256; }
static size_t pf_det_workspace_bytes(int V, int H, int W) {
    return pf_det_planes_offset() + 5 * (size_t)V * H * W * sizeof(long long);
}

extern "C" int srf_point_feats_backward(srf_stream_t stream_, int V, int n, int H, int W, const float* points,
                                        const float* w2cs, const float* ixts, const float* img_ref, const float* image,
                                        const float* acc, const float* depth, const float* g_feats, float* g_points,
                                        float* g_image, float* g_acc, float* g_depth, void* workspace) {
    const char* fn = "srf_point_feats_backward";
    if (point_feats_check(fn, V, n, H, W, points, w2cs, ixts, img_ref, image, acc, depth)) return 1;
    if (n > 0 && !g_feats) return set_error("%s: null upstream gradient", fn);
    if (workspace && srf::misaligned(workspace)) return set_error("%s: workspace must be 256-byte aligned", fn);
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const bool nothing = n == 0 || (!g_points && !g_image && !g_acc && !g_depth);
    // the default path adds into cleared outputs; the deterministic one writes them from its fixed-point planes
    if (!workspace || nothing) {
        const size_t plane = (size_t)V * H * W * sizeof(float);
        cudaError_t e = cudaSuccess;
        if (g_image && (e = cudaMemsetAsync(g_image, 0, 3 * plane, stream)) != cudaSuccess) return cuda_error("memset g_image", e);
        if (g_acc && (e = cudaMemsetAsync(g_acc, 0, plane, stream)) != cudaSuccess) return cuda_error("memset g_acc", e);
        if (g_depth && (e = cudaMemsetAsync(g_depth, 0, plane, stream)) != cudaSuccess) return cuda_error("memset g_depth", e);
    }
    if (nothing) return 0;
    srf::PointFeatsArgs a;
    memset(&a, 0, sizeof(a));
    a.V = V; a.n = n; a.H = H; a.W = W;
    a.points = points; a.w2cs = w2cs; a.ixts = ixts; a.img_ref = img_ref; a.image = image; a.acc = acc; a.depth = depth;
    a.g_feats = g_feats; a.g_points = g_points; a.g_image = g_image; a.g_acc = g_acc; a.g_depth = g_depth;
    const unsigned grid = (unsigned)((n + srf::kPfThreads - 1) / srf::kPfThreads);
    cudaError_t e;
    if (!workspace) {
        srf::point_feats_bwd_kernel<false><<<grid, srf::kPfThreads, 0, stream>>>(a);
    } else {
        e = cudaMemsetAsync(workspace, 0, pf_det_workspace_bytes(V, H, W), stream);
        if (e != cudaSuccess) return cuda_error("memset point_feats workspace", e);
        a.det = static_cast<uint32_t*>(workspace);
        a.g_fixed = reinterpret_cast<long long*>(static_cast<char*>(workspace) + pf_det_planes_offset());
        const size_t count = (size_t)V * 8 * n, planes = 5 * (size_t)V * H * W;
        srf::pf_bound_kernel<<<(unsigned)min((count + srf::kPfThreads - 1) / srf::kPfThreads, (size_t)srf::sm_count() * 8),
                               srf::kPfThreads, 0, stream>>>(a.g_feats, count, a.det);
        srf::point_feats_bwd_kernel<true><<<grid, srf::kPfThreads, 0, stream>>>(a);
        srf::pf_convert_kernel<<<(unsigned)((planes + srf::kPfThreads - 1) / srf::kPfThreads), srf::kPfThreads, 0, stream>>>(a);
    }
    if ((e = cudaGetLastError()) != cudaSuccess) return cuda_error("point_feats_bwd launch", e);
    return workspace ? srf::check_overflow_flag(fn, a.det + 1, stream) : 0;
}

extern "C" int srf_point_feats_deterministic_workspace_bytes(int V, int H, int W, size_t* bytes) {
    if (V <= 0 || H <= 0 || W <= 0 || !bytes) return set_error("srf_point_feats_deterministic_workspace_bytes: bad arguments");
    *bytes = pf_det_workspace_bytes(V, H, W);
    return 0;
}
