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
#include <string.h>

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

// Blend-forward CTAs: a 16x16 tile is eight 8x4 warp blocks; one CTA of SRF_CTA_WARPS = 8 warps owns all
// of them (the full tile) and walks the tile's list in rounds of SRF_BATCH staged splats (one per thread).
// The blend backward sizes its CTAs itself (render_bwd.cu).
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

// The same float from fp32 arithmetic: mapped_depth_fp32(d, rd, m) sets m = mapped_depth(d) and returns true,
// or returns false when the estimate cannot settle the rounding (then the caller takes mapped_depth).  d >= 0.2f
// or NaN, as the blend calls it; rd is a reciprocal of d within 1 ulp, or 0 where 1/d is subnormal (MUFU.RCP with
// flush to zero on the GPU).  Host and device builds run the same operations (tests/test_fwd_fastpath.py checks every
// float on both).
//
// With B = RN_d(99.8), the DP sequence returns RN_f(q_d), q_d = RN_d(RN_d(100d - 20) / RN_d(B d)), and
// |q_d - r| < 3.01 * 2^-53 for r = (100d - 20) / (B d) = K - J / d, K = 100 / B, J = 20 / B, r in (0, K).
// The estimate y = h + e + w of r (absolute errors, d >= 0.2f so 1/d < 5; 1 ulp of rd is < 2^-23 rd):
//   g = RN(JH rd)          g = (JH / d)(1 + n), |n| < 1.51 * 2^-23, g < 1.0021;
//   rem = RN(JH - g d)     exact value -JH n, |.| < 2^-24.7, rounding < 2^-48.7, / d: < 2^-46.4;
//   s = RN(rem + JL)       |s| < 2^-24.5, rounding < 2^-48.5, / d: < 2^-46.2;  J = JH + JL to 2^-55, / d: < 2^-52.6;
//   w = RN(KL -+ tol - s rd)  rd's error on s / d: < 2^-45.2, rounding |w| < 2^-22.1: < 2^-46.1; K = KH + KL to 2^-51.3;
//   h = RN(KH - g), e      Fast2Sum (g < 2, so exponent(KH) >= exponent(g)): KH - g = h + e exactly, |e| <= 2^-24;
//   RN(e + w)              |e + w| < 2^-21.9, rounding < 2^-45.9.
// Summed with the DP's own error, |y -+ tol - q_d| stays within 5.8 * 2^-46 < 2^-43.4 of the exact y -+ tol.  So
// hi = RN(h + RN(e + w+)) and lo = RN(h + RN(e + w-)), w+- = RN(KL +- 2^-41 - s rd), bracket q_d, and RN_f is monotonic:
// hi == lo means RN_f(q_d) == hi.  Where rd is 0 (d >= 2^126), y = K + KL +- tol differs from r by J / d < 2^-127.
// They differ (fallback) where y lies within ~2^-41 of a midpoint between floats: about 2^-16 of the depths with r
// >= 0.5, more for depths closer to 0.2 (r small, its ulp fine).  NaN and inf give NaN (0 * inf in rem) and fall back.
#define SRF_MD_KH 0x1.008356p+0f     // RN(K), K = 100 / RN_d(99.8)
#define SRF_MD_KLP -0x1.4c6edep-26f  // RN(K - KH) + 2^-41 (exact)
#define SRF_MD_KLM -0x1.4c72dep-26f  // RN(K - KH) - 2^-41 (exact)
#define SRF_MD_JH 0x1.9a6bbcp-3f     // RN(J), J = 20 / RN_d(99.8)
#define SRF_MD_JL 0x1.1f4b6ap-29f    // RN(J - JH)
#ifdef __CUDA_ARCH__
#define SRF_HD_ADD(a, b) __fadd_rn(a, b)
#define SRF_HD_MUL(a, b) __fmul_rn(a, b)
#define SRF_HD_FMA(a, b, c) __fmaf_rn(a, b, c)
#else  // host: IEEE single, built with -ffp-contract=off
#define SRF_HD_ADD(a, b) ((a) + (b))
#define SRF_HD_MUL(a, b) ((a) * (b))
#define SRF_HD_FMA(a, b, c) fmaf(a, b, c)
#endif
__host__ __device__ __forceinline__ bool mapped_depth_fp32(float d, float rd, float& m) {
    const float g = SRF_HD_MUL(SRF_MD_JH, rd);
    const float s = SRF_HD_ADD(SRF_HD_FMA(-g, d, SRF_MD_JH), SRF_MD_JL);
    const float wp = SRF_HD_FMA(-s, rd, SRF_MD_KLP);
    const float wm = SRF_HD_FMA(-s, rd, SRF_MD_KLM);
    const float h = SRF_HD_ADD(SRF_MD_KH, -g);
    const float e = SRF_HD_ADD(-g, -SRF_HD_ADD(h, -SRF_MD_KH));
    const float hi = SRF_HD_ADD(h, SRF_HD_ADD(e, wp));
    const float lo = SRF_HD_ADD(h, SRF_HD_ADD(e, wm));
    m = hi;
    return hi == lo;
}
__device__ __forceinline__ float rcp_approx(float x) {
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
// mapped_depth() for every float depth, the DP sequence only where mapped_depth_fp32 cannot decide
__device__ __forceinline__ float mapped_depth_fast(float depth) {
    float m;
    if (mapped_depth_fp32(depth, rcp_approx(depth), m)) return m;
    return mapped_depth(depth);
}

// explicit 32-bit shared-memory addressing for the blend loops: with pointer-typed accesses the compiler
// rebuilds the shared window base (S2R SR_CgaCtaId + LEA) inside the loop, in front of the first dependent load
__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ float4 lds_f4(uint32_t a) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ uint32_t lds_u8(uint32_t a) {
    uint32_t v;
    asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ uint32_t lds_u32(uint32_t a) {
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ float2 lds_f2(uint32_t a) {
    float2 v;
    asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ void sts_u32(uint32_t a, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }

// (1 << n) - 1 for n in [0, 32], in one BMSK and without a constant in a register.  The blend loops walk bit-reversed
// words: the next entry is the highest set bit p = 31 - clz, and w & bits_below(p) drops it.
__device__ __forceinline__ uint32_t bits_below(int n) {
    uint32_t m;
    asm("bmsk.clamp.b32 %0, 0, %1;" : "=r"(m) : "r"(n));
    return m;
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
__host__ __device__ __forceinline__ WarpRect make_warp_rect(int tile_x, int tile_y, int wid) {
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
// The two fp16 offsets packed in one float of q5, as floats (host and device)
__host__ __device__ __forceinline__ float2 unpack_half2(float f) {
    __half2 h;
    memcpy(&h, &f, sizeof(h));
    return __half22float2(h);
}
// true if the splat's conservative octagon (q5, centred at q2.yz) may touch the warp's block (the blend forward culls
// with octagon_block_bits, which is this test for all eight blocks of a tile; this form is kept as its definition)
__host__ __device__ __forceinline__ bool octagon_hits(const float4 q2, const float4 q5, const WarpRect& w) {
    const float cx = q2.y, cy = q2.z;
    const float2 ex = unpack_half2(q5.x), ey = unpack_half2(q5.y), eu = unpack_half2(q5.z), ev = unpack_half2(q5.w);
    const float cu = cx + cy, cv = cx - cy;
    const bool out = (cx + ex.x > w.xmax) || (cx + ex.y < w.xmin) || (cy + ey.x > w.ymax) || (cy + ey.y < w.ymin) ||
                     (cu + eu.x > w.umax) || (cu + eu.y < w.umin) || (cv + ev.x > w.vmax) || (cv + ev.y < w.vmin);
    return !out;
}

// octagon_hits() against all eight 8x4 blocks of tile (tile_x, tile_y) at once: bit b is
// octagon_hits(q2, q5, make_warp_rect(tile_x, tile_y, b)), with the same float operations and comparisons, so the bits
// are exactly that test's.  The x bounds depend only on the block's column (b & 1), the y bounds only on its row (b >> 1),
// and the offsets of the splat's octagon are decoded once for all eight blocks.  The blend forward runs it once per
// staged splat, in the thread that staged it.
__host__ __device__ __forceinline__ uint32_t octagon_block_bits(const float4 q2, const float4 q5, int tile_x, int tile_y) {
    const float cx = q2.y, cy = q2.z;
    const float2 ex = unpack_half2(q5.x), ey = unpack_half2(q5.y), eu = unpack_half2(q5.z), ev = unpack_half2(q5.w);
    const float cu = cx + cy, cv = cx - cy;
    const float xlo = cx + ex.x, xhi = cx + ex.y, ylo = cy + ey.x, yhi = cy + ey.y;
    const float ulo = cu + eu.x, uhi = cu + eu.y, vlo = cv + ev.x, vhi = cv + ev.y;
    float xmin[2], xmax[2];
    bool xin[2];
#pragma unroll
    for (int col = 0; col < 2; ++col) {
        xmin[col] = (float)(tile_x * SRF_TILE + (col << 3)) + 0.5f; xmax[col] = xmin[col] + 7.0f;
        xin[col] = !(xlo > xmax[col]) && !(xhi < xmin[col]);
    }
    uint32_t bits = 0;
#pragma unroll
    for (int row = 0; row < 4; ++row) {
        const float ymin = (float)(tile_y * SRF_TILE + (row << 2)) + 0.5f, ymax = ymin + 3.0f;
        const bool yin = !(ylo > ymax) && !(yhi < ymin);
#pragma unroll
        for (int col = 0; col < 2; ++col) {
            const float umin = xmin[col] + ymin, umax = xmax[col] + ymax;
            const float vmin = xmin[col] - ymax, vmax = xmax[col] - ymin;
            const bool in = xin[col] && yin && !(ulo > umax) && !(uhi < umin) && !(vlo > vmax) && !(vhi < vmin);
            bits |= (uint32_t)in << (2 * row + col);
        }
    }
    return bits;
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
