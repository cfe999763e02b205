// point_feats.cu -- the fine pass's point-feature sampler (LaRa Network.get_point_feats, lightning/network.py:390-411,
// with projection() at :182-187), forward and backward, one thread per point, over the S scenes of a batch.
//
// For each of the n (masked) Gaussian centres and each of the Vs source views of its scene:
//   p = K (R x + t)  with w2c [Vs,4,4] and K [Vs,3,3] row-major;  xy = p.xy / p.z,  z = p.z
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
// Scenes (DESIGN §3.26): point i belongs to the scene s with off[s] <= i < off[s+1] (host offsets, passed by value);
// it reads its centre from row rows[i] of centers [S*P,3] (rows null: row i), its cameras from s*Vs + v, img_ref
// through a stride record, and the renderings from the planar [S*Vr,C,H,W] buffers at view s*Vr + v.  The one-scene
// entries are S = 1, no rows, Vr = Vs and a contiguous img_ref.  Per point the float operations are those of one scene.
//
// Backward: the upstream gradient g[Vs,8,n] is read coalesced; dL/dcenter is summed over the views in registers and
// written once to the point's row; the gradients of the 5 differentiable channels go into planar g_image [S*Vr,3,H,W],
// g_acc and g_depth [S*Vr,H,W] with red.global.add.f32 (cleared by the entry; views v >= Vs of a scene stay 0).  No
// gradient is formed for img_ref.  The C entries srf_point_feats_* (include/surfel_rasterizer.h) are defined here.
#include <string.h>

#include "../../include/surfel_rasterizer.h"
#include "det_sum.cuh"
#include "sample_taps.cuh"
#include "surfel_kernels.h"

namespace srf {

// element strides of img_ref [S,Vs,3,H,W] (srf_pf_image_addr)
struct PfRefAddr {
    long long ss, sv, sc, sy, sx;
};

// n points of S scenes sampled in Vs source views each from the 8-channel stack img_ref | image | acc | depth
struct PointFeatsArgs {
    int Vs, Vr, n, H, W;         // Vr: rendering views per scene (>= Vs)
    long long rows_total;        // S * P rows of centers
    const float* centers;        // [S*P,3]
    const int* rows;             // [n] row of each point, or null (point i is row i)
    const float* w2cs;           // [S*Vs,4,4] row-major
    const float* ixts;           // [S*Vs,3,3] row-major
    const float* img_ref;        // [S,Vs,3,H,W] at the strides of `ref`
    PfRefAddr ref;
    const float* image;          // [S*Vr,3,H,W]
    const float* acc;            // [S*Vr,H,W]
    const float* depth;          // [S*Vr,H,W]
    float* feats;                // [Vs,8,n] forward output
    const float* g_feats;        // [Vs,8,n] backward input
    float* g_centers;            // [S*P,3] written at the points' rows (may be null)
    float* g_image; float* g_acc; float* g_depth;   // accumulated into, cleared by the entry (each may be null)
    // deterministic backward (null = default): int64 planes [5 S Vs,H,W] in the layout g_image | g_acc | g_depth and a
    // header det[0] = overflow, det[1 + s] = scene s's max |g_feats| (fp32 bits); both zeroed by the entry.  The float
    // outputs are then written, not accumulated into.
    long long* g_fixed;
    uint32_t* det;
};

// the scene bounds of the points, by value (a __grid_constant__ kernel parameter): scene s is points [off[s], off[s+1])
struct PfScenes {
    int S;
    int off[SRF_MAX_SCENES + 1];
};

namespace {

constexpr int kPfThreads = 256;

// the scene of point i: the last s with off[s] <= i (empty scenes are skipped over)
__device__ __forceinline__ int pf_scene(const PfScenes& sc, int i) {
    int lo = 0, hi = sc.S - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (sc.off[mid] <= i) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// the centre row of point i, or -1 if its index is outside [0, S*P)
__device__ __forceinline__ long long pf_row(const PointFeatsArgs& a, int i) {
    const long long r = a.rows ? (long long)__ldg(a.rows + i) : (long long)i;
    return (r >= 0 && r < a.rows_total) ? r : -1;
}

// plane of rendering channel c (3..7) of rendering view vr
__device__ __forceinline__ const float* pf_plane(const PointFeatsArgs& a, int vr, int c, size_t HW) {
    if (c < 6) return a.image + ((size_t)vr * 3 + (c - 3)) * HW;
    return (c == 6 ? a.acc : a.depth) + (size_t)vr * HW;
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

// the nw tap of view v of scene s in img_ref, at its strides
__device__ __forceinline__ const float* pf_ref_base(const PointFeatsArgs& a, int s, int v, const PfTaps& t) {
    return a.img_ref + s * a.ref.ss + v * a.ref.sv + t.yi * a.ref.sy + t.xi * a.ref.sx;
}

// channel c (0..7) at the taps: img_ref's channels through `ref` (pf_ref_base), the renderings' planes of view vr;
// the same taps, weights and sum for both
__device__ __forceinline__ float pf_sample_c(const PointFeatsArgs& a, const float* ref, int vr, int c, size_t HW,
                                             const PfTaps& t, float vals[4]) {
    if (c >= 3) return pf_sample(pf_plane(a, vr, c, HW), t, vals);
    const float* base = ref + c * a.ref.sc;
    float sum = 0.0f;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        vals[k] = t.off[k] >= 0 ? __ldg(base + ((k >> 1) ? a.ref.sy : 0) + ((k & 1) ? a.ref.sx : 0)) : 0.0f;
        if (t.off[k] >= 0) sum = __fmaf_rn(vals[k], t.w[k], sum);
    }
    return sum;
}

__device__ __forceinline__ void pf_red(float* p, float v) {
    asm volatile("red.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}

__global__ void __launch_bounds__(kPfThreads) point_feats_fwd_kernel(PointFeatsArgs a,
                                                                       const __grid_constant__ PfScenes sc) {
    const int i = blockIdx.x * kPfThreads + threadIdx.x;
    if (i >= a.n) return;
    const size_t HW = (size_t)a.H * a.W, n = (size_t)a.n;
    const long long row = pf_row(a, i);
    if (row < 0) {                                       // a row outside the centers: features 0
        for (int v = 0; v < a.Vs; ++v)
            for (int c = 0; c < 8; ++c) a.feats[((size_t)v * 8 + c) * n + i] = 0.0f;
        return;
    }
    const int s = pf_scene(sc, i);
    const float x0 = a.centers[3 * row], x1 = a.centers[3 * row + 1], x2 = a.centers[3 * row + 2];
    for (int v = 0; v < a.Vs; ++v) {
        const int vc = s * a.Vs + v, vr = s * a.Vr + v;
        float px, py, pz, m[21];
        pf_project(a.w2cs + 16 * (size_t)vc, a.ixts + 9 * (size_t)vc, x0, x1, x2, px, py, pz, m);
        const float ix = pf_source_coord(__fdiv_rn(px, pz), (float)a.W, (float)a.W);
        const float iy = pf_source_coord(__fdiv_rn(py, pz), (float)a.H, (float)a.H);
        const PfTaps t = pf_taps(ix, iy, a.W, a.H);
        float* out = a.feats + (size_t)v * 8 * n + i;
        const float* ref = pf_ref_base(a, s, v, t);
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            float vals[4];
            float sv = pf_sample_c(a, ref, vr, c, HW, t, vals);
            if (c == 7) sv = fabsf(__fsub_rn(sv, pz));    // z_diff = |s_depth - z|
            out[c * n] = sv;
        }
    }
}

__device__ __forceinline__ void pf_red_u64(long long* p, long long v) {
    asm volatile("red.global.add.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// fixed-point sum exponent budget of scene s: its Vs views, n_s points, 4 taps each
__device__ __forceinline__ int pf_det_L(const PfScenes& sc, int Vs, int s) {
    return det::ceil_log2(4ull * (uint64_t)Vs * (uint64_t)(sc.off[s + 1] - sc.off[s]));
}

// Deterministic backward (DESIGN §3.13, §3.26): every term a tap adds into a rendering gradient of scene s is w go with
// w <= 1 and |go| <= scene s's max |g_feats|, and a pixel of one of its planes receives at most 4 Vs n_s of them.  The
// bound kernel takes each scene's max (det[1 + s], fp32 bits); the backward adds the terms in 64-bit fixed point into
// planes laid out as g_image | g_acc | g_depth; the convert kernel writes the fp32 results.  det[0] is set if a term
// was over its budget or not finite.  Each scene's sums are those of the same call on that scene alone.
__global__ void __launch_bounds__(kPfThreads) pf_bound_kernel(const float* g, int Vs, int n, uint32_t* det,
                                                                const __grid_constant__ PfScenes sc) {
    for (int i0 = blockIdx.x * kPfThreads; i0 < n; i0 += gridDim.x * kPfThreads) {
        const int i = i0 + threadIdx.x;
        uint32_t m = 0;
        int s = -1;
        if (i < n) {
            s = pf_scene(sc, i);
            for (int e = 0; e < 8 * Vs; ++e) m = max(m, det::abs_bits(__ldg(g + (size_t)e * n + i)));
        }
        const unsigned same = __match_any_sync(0xffffffffu, s);     // the lanes of one scene
        m = __reduce_max_sync(same, m);
        if (s >= 0 && (threadIdx.x & 31) == __ffs(same) - 1 && m != 0u) atomicMax(det + 1 + s, m);
    }
}

__global__ void __launch_bounds__(kPfThreads) pf_convert_kernel(PointFeatsArgs a, const __grid_constant__ PfScenes sc) {
    const size_t HW = (size_t)a.H * a.W, SVr = (size_t)sc.S * a.Vr, SVs = (size_t)sc.S * a.Vs;
    const size_t n_img = 3 * SVr * HW, n_one = SVr * HW;
    const size_t j = (size_t)blockIdx.x * kPfThreads + threadIdx.x;
    if (j >= n_img + 2 * n_one) return;
    // output plane (view vr, channel plane of that view) and the fixed-point plane of the same (scene, view, channel)
    float* dst;
    size_t vr, fixed_plane;
    if (j < n_img) {
        dst = a.g_image ? a.g_image + j : nullptr;
        vr = j / (3 * HW);
        fixed_plane = 3 * ((vr / a.Vr) * a.Vs + vr % a.Vr) + (j / HW) % 3;
    } else {
        const size_t jj = j < n_img + n_one ? j - n_img : j - n_img - n_one;
        dst = j < n_img + n_one ? (a.g_acc ? a.g_acc + jj : nullptr) : (a.g_depth ? a.g_depth + jj : nullptr);
        vr = jj / HW;
        fixed_plane = (j < n_img + n_one ? 3 : 4) * SVs + (vr / a.Vr) * a.Vs + vr % a.Vr;
    }
    if (!dst) return;
    const int s = (int)(vr / a.Vr), v = (int)(vr % a.Vr);
    if (v >= a.Vs) { *dst = 0.0f; return; }
    const int k = det::scale_exp(__ldg(a.det + 1 + s), pf_det_L(sc, a.Vs, s));
    *dst = det::to_float(a.g_fixed[fixed_plane * HW + j % HW], k);
}

template <bool kDet>
__global__ void __launch_bounds__(kPfThreads) point_feats_bwd_kernel(PointFeatsArgs a,
                                                                       const __grid_constant__ PfScenes sc) {
    const int i = blockIdx.x * kPfThreads + threadIdx.x;
    if (i >= a.n) return;
    const long long row = pf_row(a, i);
    if (row < 0) return;                                 // a row outside the centers: no gradient
    const int s = pf_scene(sc, i);
    int L = 0, kq = 0;
    bool ok = true;
    if (kDet) {
        L = pf_det_L(sc, a.Vs, s);
        kq = det::scale_exp(__ldg(a.det + 1 + s), L);
    }
    const float x0 = a.centers[3 * row], x1 = a.centers[3 * row + 1], x2 = a.centers[3 * row + 2];
    const size_t HW = (size_t)a.H * a.W, n = (size_t)a.n, SVs = (size_t)sc.S * a.Vs;
    float gx0 = 0.0f, gx1 = 0.0f, gx2 = 0.0f;           // dL/dpoint, summed over the views
    for (int v = 0; v < a.Vs; ++v) {
        const int vc = s * a.Vs + v, vr = s * a.Vr + v;
        float px, py, pz, m[21];
        pf_project(a.w2cs + 16 * (size_t)vc, a.ixts + 9 * (size_t)vc, x0, x1, x2, px, py, pz, m);
        const float xs = __fdiv_rn(px, pz), ys = __fdiv_rn(py, pz);
        const PfTaps t = pf_taps(pf_source_coord(xs, (float)a.W, (float)a.W),
                                 pf_source_coord(ys, (float)a.H, (float)a.H), a.W, a.H);
        const float* g = a.g_feats + (size_t)v * 8 * n + i;
        const float* ref = pf_ref_base(a, s, v, t);
        // z_diff = |s_depth - z|: vjp with sign(0) = 0
        float dvals[4];
        const float sd = pf_sample(pf_plane(a, vr, 7, HW), t, dvals);
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
            } else if (a.g_centers) {
                pf_sample_c(a, ref, vr, c, HW, t, vals);
            }
            if (a.g_centers) {  // grid_sampler_2d_backward's gix / giy, untouched taps read as 0
                gix = __fmaf_rn(go, __fadd_rn(__fmul_rn(__fsub_rn(vals[1], vals[0]), t.ty1), __fmul_rn(__fsub_rn(vals[3], vals[2]), t.ty0)), gix);
                giy = __fmaf_rn(go, __fadd_rn(__fmul_rn(__fsub_rn(vals[2], vals[0]), t.tx1), __fmul_rn(__fsub_rn(vals[3], vals[1]), t.tx0)), giy);
            }
            float* dst = nullptr;
            if (c >= 3 && c < 6) dst = a.g_image ? a.g_image + ((size_t)vr * 3 + (c - 3)) * HW : nullptr;
            else if (c == 6) dst = a.g_acc ? a.g_acc + (size_t)vr * HW : nullptr;
            else if (c == 7) dst = a.g_depth ? a.g_depth + (size_t)vr * HW : nullptr;
            if (dst && go != 0.0f) {
                if (kDet) {
                    const size_t plane = c < 6 ? (size_t)vc * 3 + (c - 3) : (size_t)(c == 6 ? 3 : 4) * SVs + vc;
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
        if (!a.g_centers) continue;
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
    if (kDet && !ok) atomicOr(a.det, 1u);
    if (a.g_centers) {
        a.g_centers[3 * row] = gx0;
        a.g_centers[3 * row + 1] = gx1;
        a.g_centers[3 * row + 2] = gx2;
    }
}

}  // namespace

}  // namespace srf

using srf::cuda_error;
using srf::set_error;

namespace {

// One checked call of the scene kernels: sizes, pointers and the host offsets, everything before any launch.
struct PfCall {
    srf::PointFeatsArgs a;
    srf::PfScenes sc;
};

int pf_prepare(const char* fn, int S, int Vs, int Vr, int P, int n, int H, int W, const int64_t* offsets,
               const int32_t* rows, const float* centers, const float* w2cs, const float* ixts, const float* img_ref,
               const srf_pf_image_addr* ref, const float* image, const float* acc, const float* depth, PfCall& c) {
    if (S <= 0 || S > SRF_MAX_SCENES) return set_error("%s: S = %d scenes, need 0 < S <= %d", fn, S, SRF_MAX_SCENES);
    if (Vs <= 0 || Vr < Vs || P < 0 || n < 0 || H <= 0 || W <= 0)
        return set_error("%s: bad sizes (S=%d, Vs=%d, Vr=%d, P=%d, n=%d, H=%d, W=%d): need Vs > 0, Vr >= Vs, P >= 0, "
                         "n >= 0 and H, W > 0", fn, S, Vs, Vr, P, n, H, W);
    if ((long long)S * P >= (1ll << 31)) return set_error("%s: S*P = %lld rows are over the int32 index range", fn, (long long)S * P);
    if ((long long)S * Vr > 65535) return set_error("%s: S*Vr = %lld views, at most 65535", fn, (long long)S * Vr);
    if (H > (1 << 24) || W > (1 << 24)) return set_error("%s: image too large", fn);    // pixel indices exact in fp32
    // an empty point set has no storage: centers (and feats / g_feats) are only needed when n > 0
    if ((n > 0 && !centers) || !w2cs || !ixts || !img_ref || !image || !acc || !depth) return set_error("%s: null input pointer", fn);
    if (!offsets || !ref) return set_error("%s: null host offsets or img_ref strides", fn);
    if (offsets[0] != 0 || offsets[S] != n)
        return set_error("%s: offsets must run from 0 to n = %d, got %lld .. %lld", fn, n, (long long)offsets[0],
                         (long long)offsets[S]);
    for (int s = 0; s < S; ++s)
        if (offsets[s + 1] < offsets[s] || offsets[s + 1] - offsets[s] > P)
            return set_error("%s: offsets must not decrease and give each scene at most P = %d points (scene %d: %lld .. "
                             "%lld)", fn, P, s, (long long)offsets[s], (long long)offsets[s + 1]);
    memset(&c, 0, sizeof(c));
    srf::PointFeatsArgs& a = c.a;
    a.Vs = Vs; a.Vr = Vr; a.n = n; a.H = H; a.W = W;
    a.rows_total = (long long)S * P;
    a.centers = centers; a.rows = rows; a.w2cs = w2cs; a.ixts = ixts; a.img_ref = img_ref;
    a.ref = srf::PfRefAddr{ref->ss, ref->sv, ref->sc, ref->sy, ref->sx};
    a.image = image; a.acc = acc; a.depth = depth;
    c.sc.S = S;
    for (int s = 0; s <= S; ++s) c.sc.off[s] = (int)offsets[s];
    return 0;
}

unsigned pf_grid(int n) { return (unsigned)((n + srf::kPfThreads - 1) / srf::kPfThreads); }

int pf_forward(const char* fn, cudaStream_t stream, const PfCall& c, float* feats) {
    if (c.a.n > 0 && !feats) return set_error("%s: null output pointer", fn);
    if (c.a.n == 0) return 0;
    srf::PointFeatsArgs a = c.a;
    a.feats = feats;
    srf::point_feats_fwd_kernel<<<pf_grid(a.n), srf::kPfThreads, 0, stream>>>(a, c.sc);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_error("point_feats_fwd launch", e);
}

// deterministic workspace: header (overflow flag, one max |g_feats| per scene), then the int64 planes
// g_image | g_acc | g_depth of the S*Vs sampled views
size_t pf_det_planes_offset(int S) { return ((size_t)4 * (S + 1) + 255) / 256 * 256; }
size_t pf_det_workspace_bytes(int S, int Vs, int H, int W) {
    return pf_det_planes_offset(S) + 5 * (size_t)S * Vs * H * W * sizeof(long long);
}

int pf_backward(const char* fn, cudaStream_t stream, const PfCall& c, const float* g_feats, float* g_centers,
                float* g_image, float* g_acc, float* g_depth, void* workspace) {
    const int n = c.a.n, S = c.sc.S;
    if (n > 0 && !g_feats) return set_error("%s: null upstream gradient", fn);
    if (workspace && srf::misaligned(workspace)) return set_error("%s: workspace must be 256-byte aligned", fn);
    const bool nothing = n == 0 || (!g_centers && !g_image && !g_acc && !g_depth);
    cudaError_t e = cudaSuccess;
    // rows that no point writes are 0
    if (g_centers && (c.a.rows || n < c.a.rows_total) &&
        (e = cudaMemsetAsync(g_centers, 0, 3 * (size_t)c.a.rows_total * sizeof(float), stream)) != cudaSuccess)
        return cuda_error("memset g_centers", e);
    // the default path adds into cleared outputs; the deterministic one writes them from its fixed-point planes
    if (!workspace || nothing) {
        const size_t plane = (size_t)S * c.a.Vr * c.a.H * c.a.W * sizeof(float);
        if (g_image && (e = cudaMemsetAsync(g_image, 0, 3 * plane, stream)) != cudaSuccess) return cuda_error("memset g_image", e);
        if (g_acc && (e = cudaMemsetAsync(g_acc, 0, plane, stream)) != cudaSuccess) return cuda_error("memset g_acc", e);
        if (g_depth && (e = cudaMemsetAsync(g_depth, 0, plane, stream)) != cudaSuccess) return cuda_error("memset g_depth", e);
    }
    if (nothing) return 0;
    srf::PointFeatsArgs a = c.a;
    a.g_feats = g_feats; a.g_centers = g_centers; a.g_image = g_image; a.g_acc = g_acc; a.g_depth = g_depth;
    if (!workspace) {
        srf::point_feats_bwd_kernel<false><<<pf_grid(n), srf::kPfThreads, 0, stream>>>(a, c.sc);
    } else {
        e = cudaMemsetAsync(workspace, 0, pf_det_workspace_bytes(S, a.Vs, a.H, a.W), stream);
        if (e != cudaSuccess) return cuda_error("memset point_feats workspace", e);
        a.det = static_cast<uint32_t*>(workspace);
        a.g_fixed = reinterpret_cast<long long*>(static_cast<char*>(workspace) + pf_det_planes_offset(S));
        const size_t planes = 5 * (size_t)S * a.Vr * a.H * a.W;
        srf::pf_bound_kernel<<<min(pf_grid(n), (unsigned)srf::sm_count() * 8), srf::kPfThreads, 0, stream>>>(
            a.g_feats, a.Vs, n, a.det, c.sc);
        srf::point_feats_bwd_kernel<true><<<pf_grid(n), srf::kPfThreads, 0, stream>>>(a, c.sc);
        srf::pf_convert_kernel<<<(unsigned)((planes + srf::kPfThreads - 1) / srf::kPfThreads), srf::kPfThreads, 0, stream>>>(a, c.sc);
    }
    if ((e = cudaGetLastError()) != cudaSuccess) return cuda_error("point_feats_bwd launch", e);
    return workspace ? srf::check_overflow_flag(fn, a.det, stream) : 0;
}

// the one-scene call as S = 1: no rows, Vr = V, contiguous img_ref [V,3,H,W]
int pf_one_scene(const char* fn, int V, int n, int H, int W, const float* points, const float* w2cs, const float* ixts,
                 const float* img_ref, const float* image, const float* acc, const float* depth, PfCall& c) {
    if (V <= 0 || n < 0 || H <= 0 || W <= 0) return set_error("%s: bad sizes (V=%d, n=%d, H=%d, W=%d)", fn, V, n, H, W);
    if (H > (1 << 24) || W > (1 << 24)) return set_error("%s: image too large", fn);
    if ((n > 0 && !points) || !w2cs || !ixts || !img_ref || !image || !acc || !depth) return set_error("%s: null input pointer", fn);
    const long long HW = (long long)H * W;
    const srf_pf_image_addr ref = {0, 3 * HW, HW, W, 1};
    const int64_t off[2] = {0, n};
    return pf_prepare(fn, 1, V, V, n, n, H, W, off, nullptr, points, w2cs, ixts, img_ref, &ref, image, acc, depth, c);
}

}  // namespace

extern "C" int srf_point_feats_forward(srf_stream_t stream, int V, int n, int H, int W, const float* points,
                                       const float* w2cs, const float* ixts, const float* img_ref, const float* image,
                                       const float* acc, const float* depth, float* feats) {
    const char* fn = "srf_point_feats_forward";
    PfCall c;
    if (pf_one_scene(fn, V, n, H, W, points, w2cs, ixts, img_ref, image, acc, depth, c)) return 1;
    return pf_forward(fn, static_cast<cudaStream_t>(stream), c, feats);
}

extern "C" int srf_point_feats_backward(srf_stream_t stream, int V, int n, int H, int W, const float* points,
                                        const float* w2cs, const float* ixts, const float* img_ref, const float* image,
                                        const float* acc, const float* depth, const float* g_feats, float* g_points,
                                        float* g_image, float* g_acc, float* g_depth, void* workspace) {
    const char* fn = "srf_point_feats_backward";
    PfCall c;
    if (pf_one_scene(fn, V, n, H, W, points, w2cs, ixts, img_ref, image, acc, depth, c)) return 1;
    return pf_backward(fn, static_cast<cudaStream_t>(stream), c, g_feats, g_points, g_image, g_acc, g_depth, workspace);
}

extern "C" int srf_point_feats_deterministic_workspace_bytes(int V, int H, int W, size_t* bytes) {
    if (V <= 0 || H <= 0 || W <= 0 || !bytes) return set_error("srf_point_feats_deterministic_workspace_bytes: bad arguments");
    *bytes = pf_det_workspace_bytes(1, V, H, W);
    return 0;
}

extern "C" int srf_point_feats_scenes_forward(srf_stream_t stream, int S, int Vs, int Vr, int P, int n, int H, int W,
                                              const int64_t* offsets, const int32_t* rows, const float* centers,
                                              const float* w2cs, const float* ixts, const float* img_ref,
                                              const srf_pf_image_addr* img_ref_addr, const float* image,
                                              const float* acc, const float* depth, float* feats) {
    const char* fn = "srf_point_feats_scenes_forward";
    PfCall c;
    if (pf_prepare(fn, S, Vs, Vr, P, n, H, W, offsets, rows, centers, w2cs, ixts, img_ref, img_ref_addr, image, acc,
                   depth, c))
        return 1;
    return pf_forward(fn, static_cast<cudaStream_t>(stream), c, feats);
}

extern "C" int srf_point_feats_scenes_backward(srf_stream_t stream, int S, int Vs, int Vr, int P, int n, int H, int W,
                                               const int64_t* offsets, const int32_t* rows, const float* centers,
                                               const float* w2cs, const float* ixts, const float* img_ref,
                                               const srf_pf_image_addr* img_ref_addr, const float* image,
                                               const float* acc, const float* depth, const float* g_feats,
                                               float* g_centers, float* g_image, float* g_acc, float* g_depth,
                                               void* workspace) {
    const char* fn = "srf_point_feats_scenes_backward";
    PfCall c;
    if (pf_prepare(fn, S, Vs, Vr, P, n, H, W, offsets, rows, centers, w2cs, ixts, img_ref, img_ref_addr, image, acc,
                   depth, c))
        return 1;
    return pf_backward(fn, static_cast<cudaStream_t>(stream), c, g_feats, g_centers, g_image, g_acc, g_depth, workspace);
}

extern "C" int srf_point_feats_scenes_deterministic_workspace_bytes(int S, int Vs, int H, int W, size_t* bytes) {
    if (S <= 0 || S > SRF_MAX_SCENES || Vs <= 0 || H <= 0 || W <= 0 || !bytes)
        return set_error("srf_point_feats_scenes_deterministic_workspace_bytes: bad arguments");
    *bytes = pf_det_workspace_bytes(S, Vs, H, W);
    return 0;
}
