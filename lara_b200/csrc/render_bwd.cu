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
// What is kept from round 1: tiles in LPT order (one 4-warp CTA per 16x8 half tile, five per SM), the list walked back
// to front from the tile's deepest used entry in staged rounds, paired fp32 arithmetic, MUFU.RCP.
#include "surfel_common.cuh"
#include "surfel_kernels.h"

namespace srf {

namespace {

constexpr int kBwdGroup = 16;                 // splats per phase-1 / phase-2 group (X tile = 16 splats x 32 pixels)
constexpr int kBwdWarps = 4;                  // warps per CTA: one CTA per 16x8 half tile, two CTAs walk a tile's list
constexpr int kBwdThreads = kBwdWarps * 32;
constexpr int kBwdBatch = 128;                // splats staged per round, one per thread
constexpr int kBwdCtasPerSM = 5;             // resident CTAs per SM that __launch_bounds__ sizes the registers for

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

struct BwdSmem {
    static constexpr size_t rec = 0;                                                         // float4 [6][kBwdBatch]
    static constexpr size_t x = rec + sizeof(float4) * SRF_REC_QUADS * kBwdBatch;            // float [warps][3][16][32]
    static constexpr size_t pixA = x + sizeof(float) * kBwdWarps * 3 * kBwdGroup * 32;       // float4 [threads] dn0 dn1 dn2 dpix0
    static constexpr size_t pixB = pixA + sizeof(float4) * kBwdThreads;                      // float4 [threads] dpix1 dpix2 pixel centre x y
    static constexpr size_t hm = pixB + sizeof(float4) * kBwdThreads;                        // u32 [warps][kBwdBatch]
    static constexpr size_t list = hm + sizeof(uint32_t) * kBwdWarps * kBwdBatch;            // uint8 [warps][kBwdBatch]
    static constexpr size_t wmax = list + (size_t)kBwdWarps * kBwdBatch;                     // int [warps]
    static constexpr size_t total = wmax + sizeof(int) * kBwdWarps;
};

__global__ void __launch_bounds__(kBwdThreads, kBwdCtasPerSM) render_bwd_kernel(RenderBwdArgs a) {
    static_assert(kBwdBatch <= 256, "hit lists are uint8");
    static_assert(kBwdBatch == kBwdThreads, "every thread stages one list entry per round");
    extern __shared__ __align__(16) unsigned char smem[];
    typedef BwdSmem L;
    float4 (*s_rec)[kBwdBatch] = reinterpret_cast<float4 (*)[kBwdBatch]>(smem + L::rec);
    float4* s_pixA = reinterpret_cast<float4*>(smem + L::pixA);
    float4* s_pixB = reinterpret_cast<float4*>(smem + L::pixB);
    int* s_wmax = reinterpret_cast<int*>(smem + L::wmax);

    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    uint8_t* s_listw = reinterpret_cast<uint8_t*>(smem + L::list) + wid * kBwdBatch;
    uint32_t* s_hmw = reinterpret_cast<uint32_t*>(smem + L::hm) + wid * kBwdBatch;
    uint32_t sa_base = smem_addr(smem);
    asm volatile("" : "+r"(sa_base));                     // opaque: kept in a register, not rebuilt at every use
    const uint32_t sa_rec = sa_base + (uint32_t)L::rec, sa_x = sa_base + (uint32_t)(L::x + wid * (3 * kBwdGroup * 32 * sizeof(float))),
                   sa_list = sa_base + (uint32_t)(L::list + wid * kBwdBatch);

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

    // deepest list entry any pixel of the warp / of the tile blended
    int wmax = last_contributor;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) wmax = max(wmax, __shfl_xor_sync(0xffffffffu, wmax, o));
    if (lane == 0) s_wmax[wid] = wmax;
    __syncthreads();
    int n_eff = 0;
#pragma unroll
    for (int w = 0; w < kBwdWarps; ++w) n_eff = max(n_eff, s_wmax[w]);
    const int rounds = (n_eff + kBwdBatch - 1) / kBwdBatch;

    // accum_rec / last_* recursions of backward.cu:331-385, two channels per f32x2 pair:
    // (c0,c1) (c2,depth) (n0,n1) (n2,alpha); the matching upstream gradients are paired the same way
    // (the reference keeps the previous splat in last_* and folds it in at the top of the next iteration;
    //  folding it in at the bottom of its own iteration is the same arithmetic and needs no such state)
    f32x2 acc_c01 = zero2(), acc_c2d = zero2(), acc_n01 = zero2(), acc_n2a = zero2();
    const f32x2 r_dpix01 = pk2(dpix0, dpix1), r_dpix2d = pk2(dpix2, dL_ddepth);
    const f32x2 r_dn01 = pk2(dn0, dn1), r_dn2a = pk2(dn2, dL_daccum);
    float last_dL_dT = 0.f;
    const float nTfinal_bg = -T_final * bg_dot_dpixel;
    // the distortion terms of a pair with mapped depth m (backward.cu:350-368), per pixel constants folded in:
    //   dL_dweight = (D2 + m^2 A - 2 m D) dL_dreg = m (m A_r + nD_r) + D2_r,
    //   dL_dmd     = 2 w (m A - D) dL_dreg         = w (m A2_r + nD_r)
    // (A_r = A dL_dreg, A2_r = 2 A_r, nD_r = -2 D dL_dreg, D2_r = D2 dL_dreg); dL_dmd * dm/dd = dL_dmd c2 / d^2 with the
    // factor c2 = 20 / 99.8 taken into kA2_r, knD_r
    const float A_r = final_A * dL_dreg, nD_r = -2.0f * final_D * dL_dreg, D2_r = final_D2 * dL_dreg;
    const float kA2_r = (float)(2.0 * 20.0 / 99.8) * A_r, knD_r = (float)(20.0 / 99.8) * nD_r;

    // phase-2 identity of this lane: its candidate chunk size C = (lane & 15) + 1 and the multiplier that turns
    // n / C into a multiply ((n * M) >> 16 == n / C exactly while n * C < 65536; n <= 47, C <= 16 here)
    const uint32_t candM = 65536u / (uint32_t)((lane & (kBwdGroup - 1)) + 1) + 1u;
    const uint32_t hshift = (uint32_t)lane & 16u;          // 16 * (which half of a 32-entry chunk this lane stands for)
    const uint32_t sa_hm = sa_base + (uint32_t)(L::hm + wid * kBwdBatch * sizeof(uint32_t));
    const uint32_t sa_pixA = sa_base + (uint32_t)(L::pixA + wid * 32 * sizeof(float4));
    const uint32_t sa_pixB = sa_base + (uint32_t)(L::pixB + wid * 32 * sizeof(float4));

    // every thread fetches the list entry it will stage in the NEXT round while the current round is being
    // processed, so that a round's staging waits for one global load, not two dependent ones
    uint32_t next_id = 0;
    if (n_eff - 1 - tid >= 0) next_id = __ldg(a.point_list + range.x + (n_eff - 1 - tid));

    // this warp's row of the forward's contribution record, by list position
    const uint32_t* wmasks = a.masks + (size_t)gw * a.capacity + range.x;

    for (int b = 0; b < rounds; ++b) {
        // ---- the warp's contribution masks of batch b, requested first so that they arrive with the records (lane
        // takes slots lane + 32 k); positions at or behind the warp's deepest contributor were not recorded: 0
        uint32_t mk[kBwdBatch / 32];
#pragma unroll
        for (int k = 0; k < kBwdBatch / 32; ++k) {
            const int pos = n_eff - 1 - (b * kBwdBatch + k * 32 + lane);
            mk[k] = (pos >= 0 && pos < wmax) ? __ldg(wmasks + pos) : 0u;
        }
        // ---- stage batch b (back to front: slot j holds list position n_eff-1-(b*kBwdBatch+j))
        __syncthreads();                                  // every warp is done with the previous batch's records
        for (int jt = tid; jt < kBwdBatch; jt += kBwdThreads) {
            const int pos = n_eff - 1 - (b * kBwdBatch + jt);
            if (pos >= 0) {
                const uint32_t id = next_id;
                const float4* r = a.rec + (size_t)id * SRF_REC_QUADS;
#pragma unroll
                for (int k = 0; k < SRF_REC_QUADS; ++k) s_rec[k][jt] = ldg4(r + k);
                // the splat id rides in the (otherwise unused by the blend) clamp-bits word of q4
                s_rec[4][jt].w = __uint_as_float(id);
            }
        }
        const int npos = n_eff - 1 - ((b + 1) * kBwdBatch + tid);
        if (npos >= 0) next_id = __ldg(a.point_list + range.x + npos);
        __syncthreads();

        // ---- compacted list of the staged splats the forward blended into some pixel of this warp's block, with
        // their pixel masks
        int nh = 0;
#pragma unroll
        for (int k = 0; k < kBwdBatch / 32; ++k) {
            const bool hit = mk[k] != 0u;
            const unsigned hits = __ballot_sync(0xffffffffu, hit);
            if (hit) {
                const int h = nh + __popc(hits & ((1u << lane) - 1u));
                s_listw[h] = (uint8_t)(k * 32 + lane);
                s_hmw[h] = mk[k];
            }
            nh += __popc(hits);
        }
        __syncwarp();
        // the batch slot of the pixel's median contributor: slot j holds list position n_eff - 1 - (b kBwdBatch + j)
        const int j_median = n_eff - median_contributor - b * kBwdBatch;

        for (int g0 = 0; g0 < nh; g0 += 32) {
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
                uint32_t bits = (colword >> (sub * kBwdGroup)) & 0xffffu;
                const int iters1 = (int)__reduce_max_sync(0xffffffffu, (unsigned)__popc(bits));
                for (int it = 0; it < iters1; ++it) {
                    if (bits == 0) continue;
                    const int i = __ffs(bits) - 1;
                    bits &= bits - 1;
                    const int j = (int)lds_u8(sa_list + gbase + i);
                    PairBwd e;
                    const uint32_t sa_j = sa_rec + 16u * j;
                    eval_pair_bwd(lds_f4(sa_j), lds_f4(sa_j + 16u * kBwdBatch), lds_f4(sa_j + 32u * kBwdBatch), pixx, pixy, e);
                    const bool lowpass = e.lowpass;
                    const float4 q3 = lds_f4(sa_j + 48u * kBwdBatch);
                    const float4 q4 = lds_f4(sa_j + 64u * kBwdBatch);
                    const float alpha = e.alpha, c_d = e.depth;

                    // one reciprocal serves T / (1-alpha) and the background term's T_final / (1-alpha)
                    const float r1ma = rcp_fast(1.0f - alpha);   // 1 - alpha >= 0.01
                    T = T * r1ma;
                    const float w = alpha * T;
                    const f32x2 cur_c01 = pk2(q4.x, q4.y), cur_c2d = pk2(q4.z, c_d);
                    const f32x2 cur_n01 = pk2(q3.x, q3.y), cur_n2a = pk2(q3.z, 1.0f);
                    // dL_dalpha += (channel - accum_rec) * dL_dchannel over colour, depth, normal, alpha
                    const f32x2 d_c01 = sub2(cur_c01, acc_c01), d_c2d = sub2(cur_c2d, acc_c2d);
                    const f32x2 d_n01 = sub2(cur_n01, acc_n01), d_n2a = sub2(cur_n2a, acc_n2a);
                    f32x2 dsum = mul2(d_c01, r_dpix01);
                    dsum = fma2(d_c2d, r_dpix2d, dsum);
                    dsum = fma2(d_n01, r_dn01, dsum);
                    dsum = fma2(d_n2a, r_dn2a, dsum);
                    const float2 dsum_ = up2(dsum);
                    // accum_rec <- alpha * channel + (1 - alpha) * accum_rec = accum_rec + alpha * (channel - accum_rec)
                    // (all eight channels), for the next splat: one fma on the differences dL_dalpha already took
                    const f32x2 la2 = bc2(alpha);
                    acc_c01 = fma2(d_c01, la2, acc_c01);
                    acc_c2d = fma2(d_c2d, la2, acc_c2d);
                    acc_n01 = fma2(d_n01, la2, acc_n01);
                    acc_n2a = fma2(d_n2a, la2, acc_n2a);

                    float dL_dz = w * up2(r_dpix2d).y;
                    // distortion / median terms (backward.cu:350-368).  m_d = (FAR d - FAR NEAR)/((FAR-NEAR) d)
                    // = c1 - c2/d and d m_d/dd = c2/d^2; the reference evaluates both in double.  fp32 is
                    // enough here: the weight term is stationary in m_d (its derivative is
                    // 2 (m_d A - D) ~ 0), and the gradients carry 1e-6 atomic-order noise anyway.
                    const float rcd = rcp_fast(c_d);             // depth >= 0.2
                    const float m_d = fmaf(-(float)(20.0 / 99.8), rcd, (float)(100.0 / 99.8));
                    float dL_dweight = fmaf(m_d, fmaf(m_d, A_r, nD_r), D2_r);
                    if (j == j_median) {
                        dL_dz += dL_dmedian_depth;
                        dL_dweight += dL_dmax_dweight;
                    }
                    const float ddw = dL_dweight - last_dL_dT;
                    float dL_dalpha = (dsum_.x + dsum_.y) + ddw;
                    last_dL_dT = fmaf(alpha, ddw, last_dL_dT);   // dL_dweight * alpha + (1 - alpha) * last_dL_dT
                    dL_dz = fmaf(w * fmaf(m_d, kA2_r, knD_r), rcd * rcd, dL_dz);   // += dL_dmd * dm_d/dd
                    dL_dalpha *= T;
                    // background term (backward.cu:391-396)
                    dL_dalpha = fmaf(nTfinal_bg, r1ma, dL_dalpha);

                    // park the three scalars phase 2 needs; the sign of w carries the branch (w > 0 always)
                    const uint32_t xa = sa_x + 4u * (uint32_t)(i * 32 + (lane ^ i));
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
                // is the word "which pixels contributed to splat i": the very word s_hmw holds, which the chunk's
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
                    const uint32_t sa_j2 = sa_rec + 16u * lds_u8(sa_list + gbase + own);
                    const float4 q0 = lds_f4(sa_j2), q1 = lds_f4(sa_j2 + 16u * kBwdBatch), q2 = lds_f4(sa_j2 + 32u * kBwdBatch);
                    const uint32_t splat_id = lds_u32(sa_j2 + 64u * kBwdBatch + 12u);
                    const f32x2 nTu_x = pk2(-q0.x, -q0.y), nTu_y = pk2(-q0.z, -q0.w), nTu_z = pk2(-q1.x, -q1.y);
                    const float Twx = q1.z, Twy = q1.w, Twz = q2.x;
                    const f32x2 Twxy = pk2(Twx, Twy), cen = pk2(q2.y, q2.z);
                    const float nopac = -q2.w;
                    // accumulators, laid out as the gradient record: (DT0,DT1) (DT2,DT3) (DT4,DT5) (DT6,DT7) (DT8,DOPAC)
                    // (DN0,DN1) (DN2,DC0) (DC1,DC2) (DM0,DM1)
                    f32x2 A0 = zero2(), A1 = zero2(), A2 = zero2(), A3 = zero2(), A4 = zero2(), A5 = zero2(), A6 = zero2(), A7 = zero2(), A8 = zero2();
                    const uint32_t sa_xrow = sa_x + 128u * (uint32_t)own;   // the splat's row of the X tile
                    // every lane walks its own contributing pixels, C of them (fewer in a splat's last lane); the warp makes
                    // max-over-lanes trips
                    int n_take = min(C, __popc(mybits));
                    do {
                        const int t = __ffs(mybits) - 1;
                        mybits &= mybits - 1;
                        const uint32_t xa = sa_xrow + 4u * (uint32_t)(t ^ own);
                        const float ws = lds_f(xa), GdA = lds_f(xa + 4u * kBwdGroup * 32), dL_dz = lds_f(xa + 8u * kBwdGroup * 32);
                        const float4 pa = lds_f4(sa_pixA + 16u * t);
                        const float4 pb = lds_f4(sa_pixB + 16u * t);
                        const float ppx = pb.z, ppy = pb.w;
                        const float w = fabsf(ws);
                        const f32x2 w2 = bc2(w);
                        fma2_acc(A5, w2, pk2(pa.x, pa.y));      // dL/dnormal
                        fma2_acc(A6, w2, pk2(pa.z, pa.w));      // dL/dnormal.z, dL/dcolor.r
                        fma2_acc(A7, w2, pk2(pb.x, pb.y));      // dL/dcolor.gb
                        const f32x2 pix2 = pk2(ppx, ppy);
                        A4.y = __fadd_rn(A4.y, GdA);            // dL/dopacity, both branches
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
                            const float tw8 = fmaf(ppx, Dz_.x, fmaf(-ppy, Dz_.y, dL_dz));
                            A4.x = __fadd_rn(A4.x, tw8);
                        } else {
                            // low-pass branch (backward.cu:436-443); FilterInvSquare == 2 after fp32 rounding
                            const f32x2 d = sub2(cen, pix2);
                            fma2_acc(A8, d, bc2(2.0f * nopac * GdA));
                            A4.x = __fadd_rn(A4.x, dL_dz);
                        }
                    } while (--n_take != 0);
                    // the lane's partial sums
                    float* dst = a.ggrad + (size_t)splat_id * SRF_GRAD_FLOATS;
                    const float2 a0 = up2(A0), a1 = up2(A1), a2 = up2(A2), a3 = up2(A3), a8 = up2(A8);
                    const float2 a4 = up2(A4), a5 = up2(A5), a6 = up2(A6), a7 = up2(A7);
                    red_add_v4(dst + 0, a0.x, a0.y, a1.x, a1.y);
                    red_add_v4(dst + 4, a2.x, a2.y, a3.x, a3.y);
                    red_add_v4(dst + 8, a4.x, a4.y, a5.x, a5.y);
                    red_add_v4(dst + 12, a6.x, a6.y, a7.x, a7.y);
                    if (a8.x != 0.0f || a8.y != 0.0f) red_add_v4(dst + 16, a8.x, a8.y, 0.0f, 0.0f);
                }
                __syncwarp();     // phase 1 of the next group overwrites the X tile
            }
        }
    }
}

}  // namespace

cudaError_t launch_render_bwd(const RenderBwdArgs& a, cudaStream_t stream) {
    const int ntiles = a.gx * a.gy;
    if (ntiles <= 0 || a.nviews <= 0) return cudaSuccess;
    prof_start(K_RENDER_BWD, stream);
    // the opt-in is per device (and cheap): made on every call for the current device
    cudaError_t e = cudaFuncSetAttribute(render_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BwdSmem::total);
    if (e == cudaSuccess)
        render_bwd_kernel<<<dim3(ntiles * 2, a.nviews), kBwdThreads, BwdSmem::total, stream>>>(a);   // two CTAs per tile
    prof_stop(K_RENDER_BWD, stream);
    return e != cudaSuccess ? e : cudaGetLastError();
}

}  // namespace srf
