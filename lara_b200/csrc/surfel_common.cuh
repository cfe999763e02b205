// surfel_common.cuh -- shared device definitions of the surfel rasterizer (sm_90a).
//
// Data layout in HBM (all produced by the forward, consumed by render fwd/bwd and the
// backward preprocess; see DESIGN.md "Data layout"):
//
//   GeomRecord  : 6 x float4 = 96 B per Gaussian, record-major, 32 B aligned so one
//                 gather touches exactly three DRAM sectors.
//       q0 = Tu.x Tv.x Tu.y Tv.y          (rows of the splat->screen homography T, reference
//       q1 = Tu.z Tv.z Tw.x Tw.y           forward.cu:75-128; Tu/Tv interleaved = f32x2 operands)
//       q2 = Tw.z cx   cy   opacity       (cx,cy = screen-space AABB centre)
//       q3 = n.x  n.y  n.z  depth         (view-space normal, view-space z)
//       q4 = r    g    b    clamp-bits    (SH->RGB colour, 3 clamp flags as int bits)
//       q5 = 8 x fp16: lo/hi offsets from (cx,cy) along x, y, x+y, x-y of a conservative octagon
//            around {alpha >= 1/255}, for warp culling
//
// Every float op on the integer-critical chain (depth bits -> sort key, T -> AABB ->
// radius -> tile rect, and the per-pixel alpha/transmittance chain that decides
// n_contrib) is written with explicit round-to-nearest intrinsics in exactly the
// order nvcc 12.9 emitted for the reference (sm_100 SASS of forward.cu), so that
// fused-multiply-add contraction cannot differ between the two builds.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#define SRF_TILE 16
#define SRF_TILE_PIX 256
#define SRF_REC_QUADS 6
#define SRF_GRAD_FLOATS 20  // per-Gaussian gradient accumulation record (5 x float4)

// gradient accumulation record layout (floats)
// slots 0..15 are what every contributing pair produces (one power-of-two reduce-scatter); the two
// low-pass-branch values follow
#define SRF_G_DT 0        // 9: (dk.x, -dl.x, dk.y, -dl.y, dk.z, -dl.z) = (-dL/dTu, dL/dTv) interleaved, then dL/dTw
#define SRF_G_DOPAC 9     // 1
#define SRF_G_DNORMAL 10  // 3
#define SRF_G_DCOLOR 13   // 3
#define SRF_G_DMEAN2D 16  // 2: dL/dmean2D (low-pass branch only)
// 18,19: padding

#define SRF_NEAR_F 0.2f

// Blend CTAs: a 16x16 tile is eight 8x4 warp blocks; one CTA owns SRF_CTA_WARPS of them (a 16x8 half
// tile) and walks the tile's list in rounds of SRF_BATCH staged splats (one per thread).  Smaller CTAs
// wait less at the per-round barriers (the warps of a tile are unevenly loaded).
#define SRF_CTA_WARPS 8
#define SRF_CTA_THREADS (SRF_CTA_WARPS * 32)
#define SRF_BATCH SRF_CTA_THREADS
#define SRF_BATCH_CHUNKS (SRF_BATCH / 32)
#define SRF_CTAS_PER_TILE (8 / SRF_CTA_WARPS)

// Per-tile counters live in their own 256-byte block (word 0: instance count, word 1:
// bucket cursor).  Dense u32 counters put every atomic of a view into a handful of cache
// lines -- i.e. a handful of L2 slices -- and serialise there; one block per tile spreads
// them over the whole L2.
#define SRF_TILE_CTR_STRIDE 64

__device__ __forceinline__ float fmul_(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fadd_(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fma_(float a, float b, float c) { return __fmaf_rn(a, b, c); }

// Paired fp32 arithmetic: the blend kernels carry colour / normal / gradient channels two at a time.
// sm_90 has no packed fp32 instruction, so each pair is two scalar round-to-nearest operations (no
// contraction across them): the same IEEE results lane by lane as a packed fp32x2 form would give.
typedef float2 f32x2;
__device__ __forceinline__ f32x2 pk2(float lo, float hi) { return make_float2(lo, hi); }
__device__ __forceinline__ f32x2 bc2(float s) { return make_float2(s, s); }
__device__ __forceinline__ float2 up2(f32x2 v) { return v; }
__device__ __forceinline__ f32x2 fma2(f32x2 a, f32x2 b, f32x2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }
// acc = a * b + acc in place
__device__ __forceinline__ void fma2_acc(f32x2& acc, f32x2 a, f32x2 b) { acc = fma2(a, b, acc); }
// acc += a in place
__device__ __forceinline__ void add2_acc(f32x2& acc, f32x2 a) { acc = make_float2(__fadd_rn(acc.x, a.x), __fadd_rn(acc.y, a.y)); }
__device__ __forceinline__ f32x2 mul2(f32x2 a, f32x2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ f32x2 add2(f32x2 a, f32x2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ f32x2 sub2(f32x2 a, f32x2 b) { return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y)); }
__device__ __forceinline__ f32x2 zero2() { return make_float2(0.0f, 0.0f); }

// Result of intersecting one pixel ray with one splat (reference forward.cu:353-398,
// backward.cu:258-318).  `valid` is false when the reference would `continue`.
struct PairEval {
    float kx, ky, kz, lx, ly, lz;  // the two homogeneous planes
    float px, py, pz;              // their cross product (homogeneous splat point)
    float sx, sy;                  // splat-space uv
    float dx, dy;                  // centre - pixel
    float rho3d, rho2d;
    float depth;
    float G;      // exp(-rho/2)
    float alpha;  // min(0.99, opacity*G)
    bool valid;
};

// The exact instruction sequence of the reference's per-(pixel,splat) evaluation.
//   q0,q1,q2 : first three quads of the GeomRecord.
__device__ __forceinline__ void eval_pair(const float4 q0, const float4 q1, const float4 q2,
                                          const float pixx, const float pixy, PairEval& e) {
    const float Twx = q1.z, Twy = q1.w, Twz = q2.x;
    const float opac = q2.w;
    // Straight-line code: the reference `continue`s at five places, but within a warp those
    // early-outs almost never agree, so the rejection tests are folded into one predicate at the
    // end (division by p.z == 0 just yields inf/NaN, which the predicate discards).
    // k = pix.x * Tw - Tu ; l = pix.y * Tw - Tv
    // -- as three fma2: (k.c, l.c) = (pix.x, pix.y) * Tw.c - (Tu.c, Tv.c); each lane is the same
    // single-rounding fma as the scalar form, so the results are bit-identical
    const f32x2 pix2 = pk2(pixx, pixy);
    const float2 klx = up2(fma2(pix2, bc2(Twx), pk2(-q0.x, -q0.y)));
    const float2 kly = up2(fma2(pix2, bc2(Twy), pk2(-q0.z, -q0.w)));
    const float2 klz = up2(fma2(pix2, bc2(Twz), pk2(-q1.x, -q1.y)));
    e.kx = klx.x; e.lx = klx.y; e.ky = kly.x; e.ly = kly.y; e.kz = klz.x; e.lz = klz.y;
    // p = k x l, each component fma(a,b,-(c*d))
    e.pz = fma_(e.kx, e.ly, -fmul_(e.ky, e.lx));
    e.px = fma_(e.ky, e.lz, -fmul_(e.kz, e.ly));
    e.py = fma_(e.kz, e.lx, -fmul_(e.kx, e.lz));
    e.sx = __fdiv_rn(e.px, e.pz);
    e.sy = __fdiv_rn(e.py, e.pz);
    e.rho3d = fma_(e.sx, e.sx, fmul_(e.sy, e.sy));
    const float2 dxy = up2(sub2(pk2(q2.y, q2.z), pix2));      // centre - pixel
    e.dx = dxy.x; e.dy = dxy.y;
    // FilterInvSquare * |d|^2 is evaluated in double by the reference; the double
    // constant 1/(0.70710678118654762)^2 rounds the product to exactly 2*|d|^2 in fp32.
    e.rho2d = fmul_(2.0f, fma_(e.dx, e.dx, fmul_(e.dy, e.dy)));
    const float rho = fminf(e.rho3d, e.rho2d);
    const float depth3d = fadd_(Twz, fma_(Twx, e.sx, fmul_(Twy, e.sy)));
    const float depth = (e.rho3d <= e.rho2d) ? depth3d : Twz;
    e.depth = depth;
    const float power = fmul_(rho, -0.5f);
    e.G = expf(power);
    e.alpha = fminf(0.99f, fmul_(opac, e.G));
    // reference: skip if p.z == 0, if (double)depth < 0.2 (== depth < 0.2f), if power > 0,
    // if alpha < 1/255
    e.valid = (e.pz != 0.0f) && !(depth < SRF_NEAR_F) && !(power > 0.0f) && !(e.alpha < 0.00392156862745098f);
}

// mapped depth for the distortion loss, evaluated in double exactly as the reference
// (forward.cu:412: (FAR*d - FAR*NEAR) / ((FAR-NEAR)*d), FAR=100.0, NEAR=0.2).
__device__ __forceinline__ float mapped_depth(float depth) {
    const double d = (double)depth;
    const double num = __fma_rn(d, 100.0, -(100.0 * 0.2));   // DFMA in the reference SASS
    const double den = __dmul_rn(100.0 - 0.2, d);
    return (float)__ddiv_rn(num, den);
}

// pixel owned by thread `tid` of a 256-thread tile CTA: each warp covers an 8x4 block.
__device__ __forceinline__ void tile_pixel(int tid, int& lx, int& ly) {
    const int w = tid >> 5, l = tid & 31;
    lx = ((w & 1) << 3) + (l & 7);
    ly = ((w >> 1) << 2) + (l >> 3);
}

__device__ __forceinline__ float4 ldg4(const float4* p) { return __ldg(p); }

// LaRa's activations (lightning/renderer_2dgs.py:106-114, 183-188), in the operation order of
// torch's CUDA kernels: sigmoid = 1/(1+exp(-x)); exp; F.normalize = x / max(||x||_2, 1e-12).  The
// 4-element sum of squares is torch 2.11's reduction tree for a contiguous [P,4] tensor,
// (x0^2+x2^2)+(x1^2+x3^2) (found by bitwise probing on a GPU, tools/probe/act_probe.py): with it the
// fused path is bit-identical to activations-in-torch; another torch build could differ by 1 ulp.
__device__ __forceinline__ float act_sigmoid(float x) { return __fdiv_rn(1.0f, fadd_(1.0f, expf(-x))); }
__device__ __forceinline__ float act_quat_norm(float4 q) {
    const float n = __fsqrt_rn(fadd_(fadd_(fmul_(q.x, q.x), fmul_(q.z, q.z)), fadd_(fmul_(q.y, q.y), fmul_(q.w, q.w))));
    return fmaxf(n, 1e-12f);
}

// Pixel-centre bounds of a warp's 8x4 block along x, y, x+y, x-y.
struct WarpRect {
    float xmin, xmax, ymin, ymax, umin, umax, vmin, vmax;
};
__device__ __forceinline__ WarpRect make_warp_rect(int tile_x, int tile_y, int wid) {
    WarpRect w;
    w.xmin = (float)(tile_x * SRF_TILE + ((wid & 1) << 3)) + 0.5f; w.xmax = w.xmin + 7.0f;
    w.ymin = (float)(tile_y * SRF_TILE + ((wid >> 1) << 2)) + 0.5f; w.ymax = w.ymin + 3.0f;
    w.umin = w.xmin + w.ymin; w.umax = w.xmax + w.ymax;
    w.vmin = w.xmin - w.ymax; w.vmax = w.xmax - w.ymin;
    return w;
}
// the same rectangle from the block's first pixel centre
__device__ __forceinline__ WarpRect warp_rect_at(float xmin, float ymin) {
    WarpRect w;
    w.xmin = xmin; w.xmax = xmin + 7.0f;
    w.ymin = ymin; w.ymax = ymin + 3.0f;
    w.umin = w.xmin + w.ymin; w.umax = w.xmax + w.ymax;
    w.vmin = w.xmin - w.ymax; w.vmax = w.xmax - w.ymin;
    return w;
}
// true if the splat's conservative octagon (q5, centred at q2.yz) may touch the warp's block
__device__ __forceinline__ bool octagon_hits(const float4 q2, const float4 q5, const WarpRect& w) {
    const float cx = q2.y, cy = q2.z;
    const unsigned ux = __float_as_uint(q5.x), uy = __float_as_uint(q5.y), uu = __float_as_uint(q5.z), uv = __float_as_uint(q5.w);
    const float2 ex = __half22float2(*reinterpret_cast<const __half2*>(&ux));
    const float2 ey = __half22float2(*reinterpret_cast<const __half2*>(&uy));
    const float2 eu = __half22float2(*reinterpret_cast<const __half2*>(&uu));
    const float2 ev = __half22float2(*reinterpret_cast<const __half2*>(&uv));
    const float cu = cx + cy, cv = cx - cy;
    const bool out = (cx + ex.x > w.xmax) || (cx + ex.y < w.xmin) || (cy + ey.x > w.ymax) || (cy + ey.y < w.ymin) ||
                     (cu + eu.x > w.umax) || (cu + eu.y < w.umin) || (cv + ev.x > w.vmax) || (cv + ev.y < w.vmin);
    return !out;
}

// Which pixels of the warp's 8x4 block (bit = lane owning the pixel, tile_pixel()) can the splat's
// conservative octagon touch?  Same eight half-planes as octagon_hits(), evaluated per pixel row:
// columns [lo, hi] of row r are inside.  SRF_MASK_EPS widens every bound: the octagon is already
// rounded outwards, this only guards the few float roundings of the row arithmetic.
#define SRF_MASK_EPS 0.0009765625f
__device__ __forceinline__ uint32_t octagon_pixel_mask(const float4 q2, const float4 q5, const WarpRect& w) {
    const float cx = q2.y, cy = q2.z;
    const unsigned ux = __float_as_uint(q5.x), uy = __float_as_uint(q5.y), uu = __float_as_uint(q5.z), uv = __float_as_uint(q5.w);
    const float2 ex = __half22float2(*reinterpret_cast<const __half2*>(&ux));
    const float2 ey = __half22float2(*reinterpret_cast<const __half2*>(&uy));
    const float2 eu = __half22float2(*reinterpret_cast<const __half2*>(&uu));
    const float2 ev = __half22float2(*reinterpret_cast<const __half2*>(&uv));
    const float cu = cx + cy, cv = cx - cy;
    // bounds relative to the block's first pixel centre (w.xmin, w.ymin), widened by eps
    const float xlo = (cx + ex.x) - w.xmin - SRF_MASK_EPS, xhi = (cx + ex.y) - w.xmin + SRF_MASK_EPS;
    const float ylo = (cy + ey.x) - w.ymin - SRF_MASK_EPS, yhi = (cy + ey.y) - w.ymin + SRF_MASK_EPS;
    // x + y in [ulo, uhi], x - y in [vlo, vhi]  (x, y now block-relative: u0 = xmin + ymin, v0 = xmin - ymin)
    const float ulo = (cu + eu.x) - w.umin - SRF_MASK_EPS, uhi = (cu + eu.y) - w.umin + SRF_MASK_EPS;
    const float v0 = w.xmin - w.ymin;
    const float vlo = (cv + ev.x) - v0 - SRF_MASK_EPS, vhi = (cv + ev.y) - v0 + SRF_MASK_EPS;
    uint32_t mask = 0;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        const float y = (float)r;
        const float lo = fmaxf(xlo, fmaxf(ulo - y, vlo + y));
        const float hi = fminf(xhi, fminf(uhi - y, vhi + y));
        int ilo = __float2int_ru(lo), ihi = __float2int_rd(hi);
        ilo = max(ilo, 0); ihi = min(ihi, 7);
        const bool ok = (ilo <= ihi) && (y >= ylo) && (y <= yhi);
        const uint32_t row = ok ? ((2u << ihi) - (1u << ilo)) : 0u;
        mask |= row << (8 * r);
    }
    return mask;
}

// 32x32 bit-matrix transpose across a warp: lane i passes row i, receives column i.
__device__ __forceinline__ uint32_t transpose32(uint32_t x, int lane) {
    const unsigned full = 0xffffffffu;
    uint32_t y;
    y = __shfl_xor_sync(full, x, 16); x = (lane & 16) ? ((x & 0xffff0000u) | (y >> 16)) : ((x & 0x0000ffffu) | (y << 16));
    y = __shfl_xor_sync(full, x, 8);  x = (lane & 8) ? ((x & 0xff00ff00u) | ((y & 0xff00ff00u) >> 8)) : ((x & 0x00ff00ffu) | ((y & 0x00ff00ffu) << 8));
    y = __shfl_xor_sync(full, x, 4);  x = (lane & 4) ? ((x & 0xf0f0f0f0u) | ((y & 0xf0f0f0f0u) >> 4)) : ((x & 0x0f0f0f0fu) | ((y & 0x0f0f0f0fu) << 4));
    y = __shfl_xor_sync(full, x, 2);  x = (lane & 2) ? ((x & 0xccccccccu) | ((y & 0xccccccccu) >> 2)) : ((x & 0x33333333u) | ((y & 0x33333333u) << 2));
    y = __shfl_xor_sync(full, x, 1);  x = (lane & 1) ? ((x & 0xaaaaaaaau) | ((y & 0xaaaaaaaau) >> 1)) : ((x & 0x55555555u) | ((y & 0x55555555u) << 1));
    return x;
}
