// render_bwd.cu -- reverse-order per-pixel backward of the blend (K7), two-phase form.
// Replaces reference backward.cu:143-449 (renderCUDA backward).
//
// The backward of a (pixel, splat) pair has two very different halves:
//   * a per-PIXEL sequential part -- transmittance T <- T/(1-alpha), the accum_rec recursions, the
//     distortion / median terms (backward.cu:321-396) -- whose result is just three scalars per pair:
//         w = alpha*T,   GdA = G * dL/dalpha,   dL/dz ;
//   * a per-SPLAT reduction: every one of the 18 gradient values of the splat is a sum over pixels of
//     terms LINEAR in (w, GdA, dL/dz) with coefficients that depend only on the pixel position and the
//     splat's own record (backward.cu:398-446).
// The reference does both per pixel and emits 10-16 global atomics per pair; round 1 of this repository
// did both per pixel and reduced the 16 partials across the warp with a 16-shuffle reduce-scatter per
// (warp, splat) visit -- ~100 of its ~300 warp instructions per visit, at 13/32 useful lanes.
//
// Here the two halves run in the layout that suits each (per warp, on its 8x4 pixel block, for groups of
// 16 splats of the tile list that the forward blended into some pixel of the block):
//   phase 1  lane = pixel.  Every lane walks ITS OWN contributing pairs (the forward's contribution record,
//            RenderFwdArgs::masks, transposed to per-pixel words) back to front, does the sequential part and
//            parks (w, GdA, dL/dz) in shared memory
//            (3 floats per pair, XOR-swizzled so that both phases are bank-conflict free or nearly so).
//   phase 2  lanes in proportion to work.  The 32 lanes are allotted to the group's splats by their number of contributing
//            pixels (n_i = ceil(c_i / C) lanes for splat i, C the smallest chunk size for which 32 lanes suffice); every lane
//            takes a chunk of its splat's pixels, rebuilds the pixel-dependent coefficients from the splat's record held in
//            registers and accumulates the 18 gradient values in registers -- no cross-lane reduction at all; the partial
//            sums go out as 4 (5) red.global.add.v4.f32 per lane.
// Phase 1 evaluates pairs with MUFU.RCP / MUFU.EX2 and re-evaluates with the forward's exact sequence only within a
// narrow band around rho3d = rho2d (eval_pair_bwd below); which pairs were blended it takes from the record.
// Each warp walks its own block's entries of the tile list back to front from its own deepest contributor, gathers their
// records into its own ring and meets the CTA's other warps at no barrier.  What is kept from round 1: tiles in LPT
// order (one 4-warp CTA per 16x8 half tile, five per SM), paired fp32 arithmetic, MUFU.RCP.
#include "det_sum.cuh"
#include "surfel_common.cuh"
#include "surfel_kernels.h"

namespace srf {

namespace {

constexpr int kBwdGroup = 16;                 // splats per phase-1 / phase-2 group (X tile = 16 splats x 32 pixels)
constexpr int kBwdWarps = 4;                  // warps per CTA: one CTA per 16x8 half tile, two CTAs walk a tile's list
constexpr int kBwdThreads = kBwdWarps * 32;
constexpr int kBwdWindow = 128;               // list positions a warp reads masks of per step of its walk, 4 per lane
constexpr int kBwdChunk = 32;                 // compacted entries per chunk: two groups, one record gather
constexpr int kBwdQueue = kBwdChunk - 1 + kBwdWindow;   // a step's new entries behind those carried from the last
constexpr int kBwdCtasPerSM = 5;             // resident CTAs per SM that __launch_bounds__ sizes the registers for
// The staged record of a splat, five float4 planes: the first three as in the geometry record (q0 q1 q2), then
//   plane 3 = n.x n.y n.z r        plane 4 = g b splat-id (unused)
// so that phase 1 reads the normal and colour it needs with one 16-byte and one 8-byte load instead of two 16-byte
// ones.  The record's depth and clamp bits (q3.w, q4.w) and its cull octagon (q5) are not used here.
constexpr int kBwdRecQuads = 5;

__device__ __forceinline__ float rcp_fast(float x) {
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

__device__ __forceinline__ void red_add_v4(float* addr, float a, float b, float c, float d) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

__device__ __forceinline__ void sts_f(uint32_t a, float v) { asm volatile("st.shared.f32 [%0], %1;" ::"r"(a), "f"(v) : "memory"); }
__device__ __forceinline__ float lds_f(uint32_t a) {
    float v;
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(a) : "memory");
    return v;
}

__device__ __forceinline__ float ex2_fast(float x) {
    float r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

// Pair evaluation of phase 1, for pairs the forward blended (its contribution record says which): the accept / reject
// decisions are not taken again.  What must still agree with the forward BIT FOR BIT is which of the two footprints is
// the smaller one (rho3d vs rho2d picks the depth and the gradient path: a splat whose projected sigma is ~0.707 px has
// rho3d ~ rho2d at every pixel); the values only need ~1e-6.  So the two IEEE divisions and expf() of eval_pair() become
// MUFU.RCP / MUFU.EX2 (<= 2 ulp), and a pair within a 1e-5 relative band of rho3d = rho2d is re-evaluated with the
// forward's exact sequence.
struct PairBwd {
    float depth, G, alpha;
    bool lowpass;
};
__device__ __forceinline__ void eval_pair_bwd(const float4 q0, const float4 q1, const float4 q2, const float pixx,
                                              const float pixy, PairBwd& r) {
    const float Twx = q1.z, Twy = q1.w, Twz = q2.x;
    const f32x2 pix2 = pk2(pixx, pixy);
    const float2 klx = up2(fma2(pix2, bc2(Twx), pk2(-q0.x, -q0.y)));
    const float2 kly = up2(fma2(pix2, bc2(Twy), pk2(-q0.z, -q0.w)));
    const float2 klz = up2(fma2(pix2, bc2(Twz), pk2(-q1.x, -q1.y)));
    const float pz = fma_(klx.x, kly.y, -fmul_(kly.x, klx.y));
    const float px = fma_(kly.x, klz.y, -fmul_(klz.x, kly.y));
    const float py = fma_(klz.x, klx.y, -fmul_(klx.x, klz.y));
    const float rpz = rcp_fast(pz);
    const float sx = px * rpz, sy = py * rpz;
    const float rho3d = fmaf(sx, sx, sy * sy);
    const float2 d = up2(sub2(pk2(q2.y, q2.z), pix2));
    const float rho2d = 2.0f * fmaf(d.x, d.x, d.y * d.y);
    r.lowpass = !(rho3d <= rho2d);
    const float rho = fminf(rho3d, rho2d);
    r.depth = r.lowpass ? Twz : Twz + fmaf(Twx, sx, Twy * sy);
    r.G = ex2_fast(rho * -0.72134752044448170f);          // exp(-rho/2)
    const float araw = q2.w * r.G;
    r.alpha = fminf(0.99f, araw);
    if (fabsf(rho3d - rho2d) <= 1.0e-5f * rho2d) {
        PairEval e;
        eval_pair(q0, q1, q2, pixx, pixy, e);
        r.depth = e.depth; r.G = e.G; r.alpha = e.alpha; r.lowpass = !(e.rho3d <= e.rho2d);
    }
}

// Every region is per warp: after the prologue the warps share nothing and meet at no barrier.
struct BwdSmem {
    static constexpr size_t rec = 0;                                                         // float4 [warps][kBwdRecQuads][kBwdChunk]
    static constexpr size_t x = rec + sizeof(float4) * kBwdWarps * kBwdRecQuads * kBwdChunk; // float [warps][3][16][32]
    static constexpr size_t pixA = x + sizeof(float) * kBwdWarps * 3 * kBwdGroup * 32;       // float4 [threads] dn0 dn1 dn2 dpix0
    static constexpr size_t pixB = pixA + sizeof(float4) * kBwdThreads;                      // float4 [threads] dpix1 dpix2 pixel centre x y
    static constexpr size_t qmask = pixB + sizeof(float4) * kBwdThreads;                     // u32 [warps][kBwdQueue + 1]
    static constexpr size_t qpos = qmask + sizeof(uint32_t) * kBwdWarps * (kBwdQueue + 1);   // int [warps][kBwdQueue + 1]
    static constexpr size_t total = qpos + sizeof(int) * kBwdWarps * (kBwdQueue + 1);
};

// What phase 2 does with a lane's 18 partial sums (its epilogue).  kEpiFloat is the default path: red.add into the fp32
// gradient record, in whatever order the lanes arrive.  The deterministic path (DESIGN §3.13) runs the same kernel body
// twice over DetRecords (a.ggrad): kEpiBound takes each channel's largest |partial| and counts the partials, kEpiFixed
// adds them in 64-bit fixed point scaled by that bound; det_convert_kernel turns the sums into the fp32 record.
enum BwdEpilogue { kEpiFloat = 0, kEpiBound = 1, kEpiFixed = 2 };

// one (Gaussian, view) of the deterministic path: the 18 channels of the gradient record
struct DetRecord {
    long long sum[18];           // kEpiFixed: sum of round(partial 2^k)
    uint32_t bound[18];          // kEpiBound: largest |partial| (fp32 bits)
    uint32_t count;              // kEpiBound: number of lanes that sent partials
    uint32_t overflow;           // kEpiFixed: a partial was over its budget or not finite
};
static_assert(sizeof(DetRecord) == 224 && sizeof(DetRecord) % 16 == 0, "DetRecord is read with vector loads");

__device__ __forceinline__ void red_add_u64(long long* addr, long long v) {
    asm volatile("red.global.add.u64 [%0], %1;" ::"l"(addr), "l"(v) : "memory");
}

template <int kEpi>
__device__ __forceinline__ void det_epilogue(DetRecord* r, const float (&v)[18]) {
    if (kEpi == kEpiBound) {
        atomicAdd(&r->count, 1u);
#pragma unroll
        for (int c = 0; c < 18; ++c) {
            const uint32_t b = det::abs_bits(v[c]);
            if (b != 0u) atomicMax(&r->bound[c], b);
        }
    } else {
        const int L = det::ceil_log2(__ldg(&r->count));
        const uint4* bq = reinterpret_cast<const uint4*>(r->bound);
        uint32_t bd[18];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const uint4 t = __ldg(bq + k);
            bd[4 * k] = t.x; bd[4 * k + 1] = t.y; bd[4 * k + 2] = t.z; bd[4 * k + 3] = t.w;
        }
        const uint2 t2 = __ldg(reinterpret_cast<const uint2*>(r->bound + 16));
        bd[16] = t2.x; bd[17] = t2.y;
        bool ok = true;
#pragma unroll
        for (int c = 0; c < 18; ++c) {
            if (v[c] == 0.0f) continue;
            long long q;
            ok &= det::quantize(v[c], det::scale_exp(bd[c], L), L, q);
            if (q != 0) red_add_u64(&r->sum[c], q);
        }
        if (!ok) atomicOr(&r->overflow, 1u);
    }
}

template <int kEpi>
__global__ void __launch_bounds__(kBwdThreads, kBwdCtasPerSM) render_bwd_kernel(RenderBwdArgs a) {
    static_assert(kBwdWindow == 4 * 32, "a walk step reads four mask words per lane");
    extern __shared__ __align__(16) unsigned char smem[];
    typedef BwdSmem L;
    float4* s_pixA = reinterpret_cast<float4*>(smem + L::pixA);
    float4* s_pixB = reinterpret_cast<float4*>(smem + L::pixB);

    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    // this warp's queue of compacted list entries: pixel mask and list position
    uint32_t* s_qmask = reinterpret_cast<uint32_t*>(smem + L::qmask) + wid * (kBwdQueue + 1);
    int* s_qpos = reinterpret_cast<int*>(smem + L::qpos) + wid * (kBwdQueue + 1);
    float4* s_recw = reinterpret_cast<float4*>(smem + L::rec) + wid * (kBwdRecQuads * kBwdChunk);
    uint32_t sa_base = smem_addr(smem);
    asm volatile("" : "+r"(sa_base));                     // opaque: kept in a register, not rebuilt at every use
    const uint32_t sa_rec = sa_base + (uint32_t)(L::rec + wid * (kBwdRecQuads * kBwdChunk * sizeof(float4))),
                   sa_x = sa_base + (uint32_t)(L::x + wid * (3 * kBwdGroup * 32 * sizeof(float))),
                   sa_qpos = sa_base + (uint32_t)(L::qpos + wid * (kBwdQueue + 1) * sizeof(int));

    const int view = blockIdx.y;
    const size_t npix = (size_t)a.W * a.H;
    a.ranges = view_ptr(a.ranges, view, a.tile_stride);
    a.tile_order = view_ptr(a.tile_order, view, a.tile_stride);
    a.point_list = view_ptr(a.point_list, view, a.plist_stride);
    a.masks = view_ptr(a.masks, view, a.plist_stride);
    a.rec = view_ptr(a.rec, view, a.geom_stride);
    a.bg += (size_t)view * a.cam_stride;
    a.accum = view_ptr(a.accum, view, a.image_stride);
    a.n_contrib = view_ptr(a.n_contrib, view, a.image_stride);
    a.dL_dpix += (size_t)view * 3 * npix;
    a.dL_dothers += (size_t)view * 8 * npix;
    a.ggrad = view_ptr(a.ggrad, view, a.ggrad_stride);

    // two CTAs per tile, one per 16x8 half
    const int tile = (int)a.tile_order[blockIdx.x / 2];
    const int gw = (int)(blockIdx.x % 2) * kBwdWarps + wid;       // which of the tile's eight 8x4 blocks
    const int tyi = tile / a.gx, txi = tile - tyi * a.gx;
    int lx, ly;
    tile_pixel(gw * 32 + lane, lx, ly);
    const int pxi = txi * SRF_TILE + lx, pyi = tyi * SRF_TILE + ly;
    const bool inside = pxi < a.W && pyi < a.H;
    const size_t pix = (size_t)pyi * a.W + pxi;
    // first pixel centre of this warp's 8x4 block; the block's bounds are rebuilt from it where needed
    // (two live registers instead of eight)
    const float bx0 = (float)(txi * SRF_TILE + ((gw & 1) << 3)) + 0.5f, by0 = (float)(tyi * SRF_TILE + ((gw >> 1) << 2)) + 0.5f;

    uint2 range = a.ranges[tile];
    if (range.y > a.capacity) range.y = range.x;

    const float T_final = inside ? a.accum[pix] : 0.0f;
    float T = T_final;
    const int last_contributor = inside ? (int)a.n_contrib[pix] : 0;
    const int median_contributor = inside ? (int)a.n_contrib[pix + npix] : 0;
    float dpix0 = 0.f, dpix1 = 0.f, dpix2 = 0.f;
    float dL_ddepth = 0.f, dL_daccum = 0.f, dL_dreg = 0.f, dn0 = 0.f, dn1 = 0.f, dn2 = 0.f;
    float dL_dmedian_depth = 0.f, dL_dmax_dweight = 0.f;
    float final_D = 0.f, final_D2 = 0.f;
    if (inside) {
        dpix0 = a.dL_dpix[pix]; dpix1 = a.dL_dpix[pix + npix]; dpix2 = a.dL_dpix[pix + 2 * npix];
        dL_ddepth = a.dL_dothers[pix];
        dL_daccum = a.dL_dothers[pix + npix];
        dn0 = a.dL_dothers[pix + 2 * npix];
        dn1 = a.dL_dothers[pix + 3 * npix];
        dn2 = a.dL_dothers[pix + 4 * npix];
        dL_dmedian_depth = a.dL_dothers[pix + 5 * npix];
        dL_dreg = a.dL_dothers[pix + 6 * npix];
        dL_dmax_dweight = a.dL_dothers[pix + 7 * npix];
        final_D = a.accum[pix + npix];
        final_D2 = a.accum[pix + 2 * npix];
    }
    const float final_A = 1.0f - T_final;
    const float bg_dot_dpixel = __ldg(a.bg + 0) * dpix0 + __ldg(a.bg + 1) * dpix1 + __ldg(a.bg + 2) * dpix2;
    // this lane's pixel centre, held in two registers instead of being rebuilt from the lane id per pair
    float pixx = bx0 + (float)(lane & 7), pixy = by0 + (float)(lane >> 3);
    // what phase 2 reads per pixel, indexed by the pixel's thread id (= wid*32 + lane): the upstream values it
    // multiplies w with, and the pixel centre (the same floats phase 1 uses)
    s_pixA[tid] = make_float4(dn0, dn1, dn2, dpix0);
    s_pixB[tid] = make_float4(dpix1, dpix2, pixx, pixy);
    asm volatile("" : "+f"(pixx), "+f"(pixy));

    // deepest list entry any pixel of the warp blended: the warp walks from there, whatever the other warps do
    int wmax = last_contributor;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) wmax = max(wmax, __shfl_xor_sync(0xffffffffu, wmax, o));
    const int steps = (wmax + kBwdWindow - 1) / kBwdWindow;
    // the list position of the pixel's median contributor (-1: none)
    int pos_median = median_contributor - 1;
    asm volatile("" : "+r"(pos_median));             // kept in a register, not rebuilt at every phase-1 trip

    // accum_rec / last_* recursions of backward.cu:331-385.  Of the eight accum_rec channels (colour, depth, normal,
    // alpha) dL_dalpha only ever needs sum_k (c_k - accum_rec_k) g_k, g_k the channel's upstream gradient, so the
    // recursion is carried as the one scalar acc_g = sum_k accum_rec_k g_k:
    //     sum_k (c_k - accum_rec_k) g_k = sum_k c_k g_k - acc_g,
    //     accum_rec_k <- accum_rec_k + alpha (c_k - accum_rec_k)   gives   acc_g <- acc_g + alpha * (that sum)
    // (the reference keeps the previous splat in last_* and folds it in at the top of the next iteration;
    //  folding it in at the bottom of its own iteration is the same arithmetic and needs no such state)
    float acc_g = 0.f;
    float last_dL_dT = 0.f;
    const float nTfinal_bg = -T_final * bg_dot_dpixel;
    // the distortion terms of a pair with mapped depth m (backward.cu:350-368), per pixel constants folded in:
    //   dL_dweight = (D2 + m^2 A - 2 m D) dL_dreg,   dL_dmd = 2 w (m A - D) dL_dreg,   dm/dd = c2 / d^2,
    // with m = c1 - c2 r, r = 1/d (c1 = 100 / 99.8, c2 = 20 / 99.8).  As polynomials in r, with the per-pixel
    // coefficients taken once here (in double, rounded once):
    //   dL_dweight = (W2 r - Z0) r + W0,   dL_dmd * dm/dd = w (Z1 r + Z0) r^2
    float W2, W0, Z1, Z0;
    {
        const double c1 = 100.0 / 99.8, c2 = 20.0 / 99.8;
        const double Ar = (double)final_A * dL_dreg, nDr = -2.0 * (double)final_D * dL_dreg, D2r = (double)final_D2 * dL_dreg;
        W2 = (float)(Ar * c2 * c2);
        W0 = (float)((c1 * Ar + nDr) * c1 + D2r);
        Z1 = (float)(-2.0 * c2 * c2 * Ar);
        Z0 = (float)(c2 * (2.0 * c1 * Ar + nDr));
    }

    // phase-2 identity of this lane: its candidate chunk size C = (lane & 15) + 1 and the multiplier that turns
    // n / C into a multiply ((n * M) >> 16 == n / C exactly while n * C < 65536; n <= 47, C <= 16 here)
    const uint32_t candM = 65536u / (uint32_t)((lane & (kBwdGroup - 1)) + 1) + 1u;
    const uint32_t hshift = (uint32_t)lane & 16u;          // 16 * (which half of a 32-entry chunk this lane stands for)
    const uint32_t sa_hm = sa_base + (uint32_t)(L::qmask + wid * (kBwdQueue + 1) * sizeof(uint32_t));
    const uint32_t sa_pixA = sa_base + (uint32_t)(L::pixA + wid * 32 * sizeof(float4));
    const uint32_t sa_pixB = sa_base + (uint32_t)(L::pixB + wid * 32 * sizeof(float4));

    // this warp's row of the forward's contribution record, by list position
    const uint32_t* wmasks = a.masks + (size_t)gw * a.capacity + range.x;
    const uint32_t* plist = a.point_list + range.x;

    // The warp walks its own block's list positions back to front from its own deepest contributor, kBwdWindow per
    // step, and appends the entries the forward blended into some pixel of the block to its queue.  Every full 32-entry
    // chunk of the queue is processed at once; the rest waits for the next step, so that every group but the warp's
    // last is full.  Nothing here depends on the other warps of the CTA.
    int nq = 0;                                           // entries in the queue, carried from the last step
    for (int b = 0; b < steps; ++b) {
        // ---- the block's contribution masks of positions wmax-1-(b kBwdWindow + 32 k + lane), k = 0..3, all requested
        // before the first is used
        uint32_t mk[kBwdWindow / 32];
#pragma unroll
        for (int k = 0; k < kBwdWindow / 32; ++k) {
            const int pos = wmax - 1 - (b * kBwdWindow + k * 32 + lane);
            mk[k] = pos >= 0 ? __ldg(wmasks + pos) : 0u;
        }
        // ---- appended to the queue, in walk order, with their list positions
#pragma unroll
        for (int k = 0; k < kBwdWindow / 32; ++k) {
            const bool hit = mk[k] != 0u;
            const unsigned hits = __ballot_sync(0xffffffffu, hit);
            if (hit) {
                const int h = nq + __popc(hits & ((1u << lane) - 1u));
                s_qpos[h] = wmax - 1 - (b * kBwdWindow + k * 32 + lane);
                s_qmask[h] = mk[k];
            }
            nq += __popc(hits);
        }
        // the full chunks of the queue; at the warp's last step, all of it
        const int nh = b == steps - 1 ? nq : (nq & ~(kBwdChunk - 1));
        __syncwarp();

        for (int g0 = 0; g0 < nh; g0 += kBwdChunk) {
            // ---- gather the chunk's records into the warp's ring (slot i = chunk entry i), five planes:
            //   q0 q1 q2, (n.x n.y n.z r), (g b splat-id)
            // The previous chunk's last group ended with a __syncwarp, so its records are no longer read.
            if (g0 + lane < nh) {
                const uint32_t id = __ldg(plist + s_qpos[g0 + lane]);
                const float4* r = a.rec + (size_t)id * SRF_REC_QUADS;
                const float4 q0 = ldg4(r), q1 = ldg4(r + 1), q2 = ldg4(r + 2), q3 = ldg4(r + 3), q4 = ldg4(r + 4);
                s_recw[lane] = q0;
                s_recw[kBwdChunk + lane] = q1;
                s_recw[2 * kBwdChunk + lane] = q2;
                s_recw[3 * kBwdChunk + lane] = make_float4(q3.x, q3.y, q3.z, q4.x);
                s_recw[4 * kBwdChunk + lane] = make_float4(q4.y, q4.z, __uint_as_float(id), 0.0f);
            }
            __syncwarp();
            // pixel mask of chunk entry g0 + lane (0 past the end of the list); the 32x32 bit transpose of the chunk's
            // masks hands lane p the word "which of these 32 splats were blended into MY pixel"
            const uint32_t ew = g0 + lane < nh ? lds_u32(sa_hm + 4u * (uint32_t)(g0 + lane)) : 0u;
            const uint32_t colword = transpose32(ew, lane);

            // ---- phase-2 schedule of both 16-entry groups of the chunk, in one pass (lane l stands for entry g0 + l of
            // group l >> 4).  C of a group is the smallest chunk size with sum_i ceil(c_i / C) <= 32 over its entries; the
            // sum is monotone in C, so a 4-step binary search finds it (C = 16 always suffices, c_i <= 32).  One
            // __reduce_add_sync per step sums both groups: each lane adds ceil(c / C) of its own group's candidate into
            // that group's 16-bit field (a sum is at most 16 * 32).
            const int cnt = __popc(ew);
            int cm1 = 0;                                  // C - 1 of this lane's group: how many smaller C do not suffice
#pragma unroll
            for (int st = 8; st > 0; st >>= 1) {
                // candidate C = cm1 + st (the first step tries C = 8 in both groups)
                const uint32_t M = st == 8 ? 65536u / 8u + 1u : __shfl_sync(0xffffffffu, candM, cm1 + st - 1);
                const uint32_t n = ((uint32_t)(cnt + cm1 + st - 1) * M) >> 16;
                const uint32_t tot = __reduce_add_sync(0xffffffffu, n << hshift);
                if (((tot >> hshift) & 0xffffu) > 32u) cm1 += st;
            }
            // lanes per entry n = ceil(c / C) and their inclusive scan within the group: the lanes of entry i are
            // [end_i - n_i, end_i).  Kept for both groups in one word: end | n << 8 | (C - 1) << 16.
            const uint32_t n_mine = ((uint32_t)(cnt + cm1) * __shfl_sync(0xffffffffu, candM, cm1)) >> 16;
            uint32_t end = n_mine;
#pragma unroll
            for (int o = 1; o < kBwdGroup; o <<= 1) {
                const uint32_t v = __shfl_up_sync(0xffffffffu, end, o);
                if ((lane & (kBwdGroup - 1)) >= o) end += v;
            }
            const uint32_t sched = end | (n_mine << 8) | ((uint32_t)cm1 << 16);

#pragma unroll 1
            for (int sub = 0; sub < 2; ++sub) {
                const int gbase = g0 + sub * kBwdGroup;
                if (gbase >= nh) break;

                // ================= phase 1: lane = pixel =================
                // The lane's contributing entries of the group, bit-reversed: entry i is bit 31 - i, so the next one
                // back to front is the highest set bit (one FLO) and dropping it keeps the bits below (BMSK, LOP3).
                // Each lane loops over its own pairs and leaves when it has none left; the warp reconverges once,
                // after the loop, not at every trip.
                uint32_t rbits = __brev(colword >> (sub * kBwdGroup)) & 0xffff0000u;
                // entry i of the group is queue entry gbase + i and ring slot sub * 16 + i
                const uint32_t sa_pos_g = sa_qpos + 4u * (uint32_t)(gbase + 31);
                const uint32_t sa_rec_g = sa_rec + 16u * (uint32_t)(sub * kBwdGroup + 31);
                while (rbits != 0u) {
                    const int p = 31 - __clz(rbits);             // entry i = 31 - p of the group
                    rbits &= bits_below(p);
                    const int pos = (int)lds_u32(sa_pos_g - 4u * (uint32_t)p);
                    PairBwd e;
                    const uint32_t sa_j = sa_rec_g - 16u * (uint32_t)p;
                    // all five loads go out before the pair evaluation, so that their latency overlaps it
                    const float4 q0 = lds_f4(sa_j), q1 = lds_f4(sa_j + 16u * kBwdChunk), q2 = lds_f4(sa_j + 32u * kBwdChunk);
                    const float4 q3 = lds_f4(sa_j + 48u * kBwdChunk);   // n.x n.y n.z r
                    const float2 q4 = lds_f2(sa_j + 64u * kBwdChunk);   // g b
                    eval_pair_bwd(q0, q1, q2, pixx, pixy, e);
                    const bool lowpass = e.lowpass;
                    const float alpha = e.alpha, c_d = e.depth;

                    // one reciprocal serves T / (1-alpha) and the background term's T_final / (1-alpha)
                    const float r1ma = rcp_fast(1.0f - alpha);   // 1 - alpha >= 0.01
                    T = T * r1ma;
                    const float w = alpha * T;
                    // dL_dalpha += (channel - accum_rec) * dL_dchannel over colour, depth, normal, alpha (alpha's
                    // channel value is 1), then accum_rec <- accum_rec + alpha * (channel - accum_rec), as acc_g
                    float cg = fmaf(q3.w, dpix0, dL_daccum);
                    cg = fmaf(q4.x, dpix1, cg);
                    cg = fmaf(q4.y, dpix2, cg);
                    cg = fmaf(q3.x, dn0, cg);
                    cg = fmaf(q3.y, dn1, cg);
                    cg = fmaf(q3.z, dn2, cg);
                    cg = fmaf(c_d, dL_ddepth, cg);
                    const float dsum = cg - acc_g;
                    acc_g = fmaf(alpha, dsum, acc_g);

                    float dL_dz = w * dL_ddepth;
                    // distortion / median terms (backward.cu:350-368).  m_d = (FAR d - FAR NEAR)/((FAR-NEAR) d)
                    // = c1 - c2/d and d m_d/dd = c2/d^2; the reference evaluates both in double.  fp32 is
                    // enough here: the weight term is stationary in m_d (its derivative is
                    // 2 (m_d A - D) ~ 0), and the gradients carry 1e-6 atomic-order noise anyway.
                    const float rcd = rcp_fast(c_d);             // depth >= 0.2
                    float dL_dweight = fmaf(fmaf(W2, rcd, -Z0), rcd, W0);
                    if (pos == pos_median) {
                        dL_dz += dL_dmedian_depth;
                        dL_dweight += dL_dmax_dweight;
                    }
                    const float ddw = dL_dweight - last_dL_dT;
                    float dL_dalpha = dsum + ddw;
                    last_dL_dT = fmaf(alpha, ddw, last_dL_dT);   // dL_dweight * alpha + (1 - alpha) * last_dL_dT
                    dL_dz = fmaf(w * fmaf(Z1, rcd, Z0), rcd * rcd, dL_dz);       // += dL_dmd * dm_d/dd
                    dL_dalpha *= T;
                    // background term (backward.cu:391-396)
                    dL_dalpha = fmaf(nTfinal_bg, r1ma, dL_dalpha);

                    // park the three scalars phase 2 needs; the sign of w carries the branch (w > 0 always)
                    // at row i, column lane ^ i; with i = 31 - p that is word 31*32 + ((lane ^ 31) ^ p) - 32 p
                    const uint32_t xa = sa_x + 4u * (31 * 32) + 4u * (uint32_t)(((lane ^ 31) ^ p) - 32 * p);
                    sts_f(xa, lowpass ? -w : w);
                    sts_f(xa + 4u * kBwdGroup * 32, e.G * dL_dalpha);
                    sts_f(xa + 8u * kBwdGroup * 32, dL_dz);
                }

                __syncwarp();     // phase-1 stores to the X tile are visible to the whole warp

                // ================= phase 2: lane = (splat, chunk of its pixels) =================
                // Lanes in proportion to work.  Splat i has c_i contributing pixels; with chunk size C it gets
                // n_i = ceil(c_i / C) lanes, lane r of them takes its pixels of rank [r C, (r + 1) C), and the loop
                // below makes C trips.  C is the smallest value for which the lanes suffice (sum n_i <= 32;
                // C = 16 always does): ~8.5 trips per group on the bench scene against ~15 with two lanes per
                // splat (tools/phase2_balance.py).  C, n_i and the scan of the n_i were set up for the chunk (sched).
                const int hb = sub * kBwdGroup;               // the lanes of sched that stand for this group
                const uint32_t end = sched & 0xffu;
                const int lanes_used = (int)__shfl_sync(0xffffffffu, end, hb + kBwdGroup - 1);
                // owner of this lane, the splat of the group it accumulates for: the first splat whose lanes end
                // beyond it (lower bound over end[0..15])
                int own = 0;
#pragma unroll
                for (int st = kBwdGroup / 2; st > 0; st >>= 1) {
                    const int e = (int)__shfl_sync(0xffffffffu, end, hb + own + st - 1);
                    if (e <= lane) own += st;
                }
                const uint32_t own_s = __shfl_sync(0xffffffffu, sched, hb + own);
                const int own_end = (int)(own_s & 0xffu), own_n = (int)((own_s >> 8) & 0xffu), C = (int)(own_s >> 16) + 1;
                // Every compacted entry has a non-zero mask, so every group has work.  The pixel mask of entry gbase + i
                // is the word "which pixels contributed to splat i": the very word the queue holds, which the chunk's
                // transpose was made from and which transposing phase 1's words back would rebuild.
                const uint32_t word = lds_u32(sa_hm + 4u * (uint32_t)(gbase + own));
                const bool have = lane < lanes_used;
                // drop the lowest r C contributing pixels of the word (r = rank of this lane among the splat's
                // lanes; r C < c_own): the largest pos with popc(word below pos) <= r C
                const int skip = (lane - (own_end - own_n)) * C;
                int pos = 0;
#pragma unroll
                for (int st = 16; st > 0; st >>= 1) {
                    const int below = __popc(word & ((1u << (pos + st)) - 1u));
                    if (below <= skip) pos += st;
                }
                uint32_t mybits = have ? (word & (0xffffffffu << pos)) : 0u;
                // only a lane in use (it has at least one pair) loads the record, accumulates and sends partial sums
                if (mybits != 0) {
                    const uint32_t sa_j2 = sa_rec + 16u * (uint32_t)(sub * kBwdGroup + own);
                    const float4 q0 = lds_f4(sa_j2), q1 = lds_f4(sa_j2 + 16u * kBwdChunk), q2 = lds_f4(sa_j2 + 32u * kBwdChunk);
                    const uint32_t splat_id = lds_u32(sa_j2 + 64u * kBwdChunk + 8u);
                    const f32x2 nTu_x = pk2(-q0.x, -q0.y), nTu_y = pk2(-q0.z, -q0.w), nTu_z = pk2(-q1.x, -q1.y);
                    const float Twx = q1.z, Twy = q1.w, Twz = q2.x;
                    const f32x2 Twxy = pk2(Twx, Twy), cen = pk2(q2.y, q2.z);
                    const float nopac = -q2.w, n2opac = 2.0f * nopac;
                    // accumulators, laid out as the gradient record: (DT0,DT1) (DT2,DT3) (DT4,DT5) (DT6,DT7) (DT8,DOPAC)
                    // (DN0,DN1) (DN2,DC0) (DC1,DC2) (DM0,DM1)
                    f32x2 A0 = zero2(), A1 = zero2(), A2 = zero2(), A3 = zero2(), A4 = zero2(), A5 = zero2(), A6 = zero2(), A7 = zero2(), A8 = zero2();
                    const uint32_t sa_xrow = sa_x + 128u * (uint32_t)own;   // the splat's row of the X tile
                    // every lane walks its own contributing pixels, C of them (fewer in a splat's last lane); the warp makes
                    // max-over-lanes trips
                    // (bit-reversed as in phase 1: pixel t is bit 31 - t, the next one is the highest set bit)
                    int n_take = min(C, __popc(mybits));
                    uint32_t rbits = __brev(mybits);
                    do {
                        const int p = 31 - __clz(rbits);             // pixel t = 31 - p
                        rbits &= bits_below(p);
                        const uint32_t xa = sa_xrow + 4u * (uint32_t)((own ^ 31) ^ p);   // column t ^ own
                        const float ws = lds_f(xa), GdA = lds_f(xa + 4u * kBwdGroup * 32), dL_dz = lds_f(xa + 8u * kBwdGroup * 32);
                        const float4 pa = lds_f4(sa_pixA + 16u * 31 - 16u * (uint32_t)p);
                        const float4 pb = lds_f4(sa_pixB + 16u * 31 - 16u * (uint32_t)p);
                        const float ppx = pb.z, ppy = pb.w;
                        const float w = fabsf(ws);
                        const f32x2 w2 = bc2(w);
                        fma2_acc(A5, w2, pk2(pa.x, pa.y));      // dL/dnormal
                        fma2_acc(A6, w2, pk2(pa.z, pa.w));      // dL/dnormal.z, dL/dcolor.r
                        fma2_acc(A7, w2, pk2(pb.x, pb.y));      // dL/dcolor.gb
                        const f32x2 pix2 = pk2(ppx, ppy);
                        A4.y = __fadd_rn(A4.y, GdA);            // dL/dopacity, both branches
                        float tw8;                              // dL/dTw.z of the pair: A4.x's term in both branches
                        if (ws > 0.0f) {
                            // ray-splat branch: vjp through s = p.xy / p.z, p = k x l (backward.cu:405-435)
                            const float2 klx = up2(fma2(pix2, bc2(Twx), nTu_x));
                            const float2 kly = up2(fma2(pix2, bc2(Twy), nTu_y));
                            const float2 klz = up2(fma2(pix2, bc2(Twz), nTu_z));
                            const float pz = fmaf(klx.x, kly.y, -(kly.x * klx.y));
                            const float px = fmaf(kly.x, klz.y, -(klz.x * kly.y));
                            const float py = fmaf(klz.x, klx.y, -(klx.x * klz.y));
                            const float rpz = rcp_fast(pz);
                            const f32x2 S = mul2(pk2(px, py), bc2(rpz));
                            // dL_dG * -G = -opacity * (G dL_dalpha)
                            const f32x2 dS = fma2(S, bc2(nopac * GdA), mul2(Twxy, bc2(dL_dz)));   // (dL_dsx, dL_dsy)
                            const f32x2 dPxy = mul2(dS, bc2(rpz));                              // (dL_dpx, dL_dpy)
                            const float2 dp = up2(dPxy), dps = up2(mul2(dPxy, S));
                            const float dpz = -(dps.x + dps.y);
                            // dL_dk = l x dL_dp, dL_dl = dL_dp x k, as the pairs (dk.c, -dl.c) = the record's layout
                            const f32x2 Sx = pk2(klx.y, klx.x), Sy = pk2(kly.y, kly.x), Sz = pk2(klz.y, klz.x);
                            const f32x2 Dx = fma2(Sy, bc2(dpz), mul2(Sz, bc2(-dp.y)));
                            const f32x2 Dy = fma2(Sz, bc2(dp.x), mul2(Sx, bc2(-dpz)));
                            const f32x2 Dz = fma2(Sx, bc2(dp.y), mul2(Sy, bc2(-dp.x)));
                            add2_acc(A0, Dx); add2_acc(A1, Dy); add2_acc(A2, Dz);
                            // dL_dTw = pix.x dk + pix.y dl + dL_dz (s, 1)  (record holds -dl, hence -pix.y)
                            const float2 Dx_ = up2(Dx), Dy_ = up2(Dy), Dz_ = up2(Dz);
                            f32x2 tw67 = mul2(S, bc2(dL_dz));
                            tw67 = fma2(bc2(ppx), pk2(Dx_.x, Dy_.x), tw67);
                            tw67 = fma2(bc2(-ppy), pk2(Dx_.y, Dy_.y), tw67);
                            add2_acc(A3, tw67);
                            tw8 = fmaf(ppx, Dz_.x, fmaf(-ppy, Dz_.y, dL_dz));
                        } else {
                            // low-pass branch (backward.cu:436-443); FilterInvSquare == 2 after fp32 rounding
                            const f32x2 d = sub2(cen, pix2);
                            fma2_acc(A8, d, bc2(n2opac * GdA));
                            tw8 = dL_dz;
                        }
                        A4.x = __fadd_rn(A4.x, tw8);
                    } while (--n_take != 0);
                    // the lane's partial sums
                    const float2 a0 = up2(A0), a1 = up2(A1), a2 = up2(A2), a3 = up2(A3), a8 = up2(A8);
                    const float2 a4 = up2(A4), a5 = up2(A5), a6 = up2(A6), a7 = up2(A7);
                    if (kEpi == kEpiFloat) {
                        float* dst = a.ggrad + (size_t)splat_id * SRF_GRAD_FLOATS;
                        red_add_v4(dst + 0, a0.x, a0.y, a1.x, a1.y);
                        red_add_v4(dst + 4, a2.x, a2.y, a3.x, a3.y);
                        red_add_v4(dst + 8, a4.x, a4.y, a5.x, a5.y);
                        red_add_v4(dst + 12, a6.x, a6.y, a7.x, a7.y);
                        if (a8.x != 0.0f || a8.y != 0.0f) red_add_v4(dst + 16, a8.x, a8.y, 0.0f, 0.0f);
                    } else {
                        const float v[18] = {a0.x, a0.y, a1.x, a1.y, a2.x, a2.y, a3.x, a3.y, a4.x, a4.y,
                                             a5.x, a5.y, a6.x, a6.y, a7.x, a7.y, a8.x, a8.y};
                        det_epilogue<kEpi>(reinterpret_cast<DetRecord*>(a.ggrad) + splat_id, v);
                    }
                }
                __syncwarp();     // phase 1 of the next group overwrites the X tile
            }
        }
        // ---- the entries of a partial chunk move to the front of the queue and wait for the next step
        const int rest = nq - nh;
        if (nh > 0 && rest > 0) {
            uint32_t m = 0u;
            int p = 0;
            if (lane < rest) { m = s_qmask[nh + lane]; p = s_qpos[nh + lane]; }
            __syncwarp();
            if (lane < rest) { s_qmask[lane] = m; s_qpos[lane] = p; }
            __syncwarp();
        }
        nq = rest;
    }
}

// one thread per (Gaussian, view): the fixed-point sums of a DetRecord -> the fp32 gradient record preprocess_bwd reads
__global__ void __launch_bounds__(256) det_convert_kernel(const DetRecord* det, size_t det_stride, float* ggrad,
                                                          size_t ggrad_stride, int P, int nviews, uint32_t* overflow) {
    const size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= (size_t)P * nviews) return;
    const int view = (int)(i / (size_t)P), g = (int)(i - (size_t)view * P);
    const DetRecord* r = view_ptr(det, view, det_stride) + g;
    float4* out = reinterpret_cast<float4*>(view_ptr(ggrad, view, ggrad_stride) + (size_t)g * SRF_GRAD_FLOATS);
    const int L = det::ceil_log2(r->count);
    float f[20];
#pragma unroll
    for (int c = 0; c < 18; ++c) f[c] = det::to_float(r->sum[c], det::scale_exp(r->bound[c], L));
    f[18] = f[19] = 0.0f;
#pragma unroll
    for (int k = 0; k < 5; ++k) out[k] = make_float4(f[4 * k], f[4 * k + 1], f[4 * k + 2], f[4 * k + 3]);
    if (r->overflow) atomicOr(overflow, 1u);
}

template <int kEpi>
cudaError_t launch_render_bwd_t(const RenderBwdArgs& a, cudaStream_t stream) {
    const int ntiles = a.gx * a.gy;
    prof_start(K_RENDER_BWD, stream);
    // the opt-in is per device (and cheap): made on every call for the current device
    cudaError_t e = cudaFuncSetAttribute(render_bwd_kernel<kEpi>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BwdSmem::total);
    if (e == cudaSuccess)
        render_bwd_kernel<kEpi><<<dim3(ntiles * 2, a.nviews), kBwdThreads, BwdSmem::total, stream>>>(a);   // two CTAs per tile
    prof_stop(K_RENDER_BWD, stream);
    return e != cudaSuccess ? e : cudaGetLastError();
}

}  // namespace

size_t det_record_bytes() { return sizeof(DetRecord); }

cudaError_t launch_render_bwd(const RenderBwdArgs& a, cudaStream_t stream) {
    const int ntiles = a.gx * a.gy;
    if (ntiles <= 0 || a.nviews <= 0) return cudaSuccess;
    return launch_render_bwd_t<kEpiFloat>(a, stream);
}

cudaError_t launch_render_bwd_det(const RenderBwdArgs& a, int P, float* ggrad, size_t ggrad_stride, uint32_t* overflow,
                                  cudaStream_t stream) {
    const int ntiles = a.gx * a.gy;
    if (ntiles <= 0 || a.nviews <= 0 || P <= 0) return cudaSuccess;
    cudaError_t e = launch_render_bwd_t<kEpiBound>(a, stream);
    if (e == cudaSuccess) e = launch_render_bwd_t<kEpiFixed>(a, stream);
    if (e != cudaSuccess) return e;
    const size_t n = (size_t)P * a.nviews;
    det_convert_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(reinterpret_cast<const DetRecord*>(a.ggrad),
                                                                        a.ggrad_stride, ggrad, ggrad_stride, P, a.nviews, overflow);
    return cudaGetLastError();
}

}  // namespace srf
