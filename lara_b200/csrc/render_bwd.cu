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
// 16 splats of the tile list that can touch the block):
//   phase 1  lane = pixel.  Every lane walks ITS OWN hits (per-pixel octagon masks, as the forward does)
//            back to front, does the sequential part and parks (w, GdA, dL/dz) in shared memory
//            (3 floats per pair, XOR-swizzled so that both phases are bank-conflict free or nearly so).
//   phase 2  lanes in proportion to work.  The 32 lanes are allotted to the group's splats by their number of contributing
//            pixels (n_i = ceil(c_i / C) lanes for splat i, C the smallest chunk size for which 32 lanes suffice); every lane
//            takes a chunk of its splat's pixels, rebuilds the pixel-dependent coefficients from the splat's record held in
//            registers and accumulates the 18 gradient values in registers -- no cross-lane reduction at all; the partial
//            sums go out as 4 (5) red.global.add.v4.f32 per lane.  (P2WALK 0..2 are the earlier fixed layouts, two lanes
//            per splat, kept for A/B.)
// Phase 1 evaluates pairs with MUFU.RCP / MUFU.EX2 and re-evaluates with the forward's exact sequence only within a
// narrow band around the forward's decision thresholds (eval_pair_bwd below).
// What is kept from round 1: tiles in LPT order (the default variant runs one 4-warp CTA per 16x8 half tile, five per
// SM), the list walked back to front from the tile's deepest used entry in staged rounds, warp-level octagon cull,
// paired fp32 arithmetic, MUFU.RCP.
#include "surfel_common.cuh"
#include "surfel_kernels.h"

namespace srf {

namespace {

constexpr int kBwdGroup = 16;                 // splats per phase-1 / phase-2 group (X tile = 16 splats x 32 pixels)

__device__ __forceinline__ float rcp_fast(float x) {
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

__device__ __forceinline__ void red_add_v4(float* addr, float a, float b, float c, float d) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

__device__ __forceinline__ f32x2 shfl_xor2(f32x2 v, int m) {
    return make_float2(__shfl_xor_sync(0xffffffffu, v.x, m), __shfl_xor_sync(0xffffffffu, v.y, m));
}

// explicit 32-bit shared-memory addressing for the phase-1 loop (SADDR): with pointer-typed accesses the compiler
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
__device__ __forceinline__ void sts_f(uint32_t a, float v) { asm volatile("st.shared.f32 [%0], %1;" ::"r"(a), "f"(v) : "memory"); }

__device__ __forceinline__ float ex2_fast(float x) {
    float r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

// Pair evaluation of phase 1.  What must agree with the forward BIT FOR BIT are the accept / reject decisions
// (a pair taken by one pass and not by the other shifts the whole transmittance chain of its pixel); the values
// only need ~1e-6.  So the two IEEE divisions and expf() of eval_pair() become MUFU.RCP / MUFU.EX2 (<= 2 ulp), and a
// pair that lands within a 1e-4 / 1e-5 relative band of a decision threshold (alpha = 1/255, depth = 0.2, rho3d = rho2d)
// -- one in ~1e4 -- is re-evaluated with the forward's exact sequence.  k, l and p = k x l are the forward's own operations, so the
// p.z != 0 test is exact as is.
struct PairBwd {
    float depth, G, alpha;
    bool lowpass, valid;
};
template <bool EXACT>
__device__ __forceinline__ void eval_pair_bwd(const float4 q0, const float4 q1, const float4 q2, const float pixx,
                                              const float pixy, PairBwd& r) {
    if (EXACT) {
        PairEval e;
        eval_pair(q0, q1, q2, pixx, pixy, e);
        r.depth = e.depth; r.G = e.G; r.alpha = e.alpha; r.lowpass = !(e.rho3d <= e.rho2d); r.valid = e.valid;
        return;
    }
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
    r.valid = (pz != 0.0f) && !(r.depth < SRF_NEAR_F) && !(araw < 0.00392156862745098f);
    // decisions of the forward that the approximate values could take differently: alpha vs 1/255, depth vs the
    // near plane, and WHICH of the two footprints is the smaller one (rho3d vs rho2d picks the gradient path: a splat
    // whose projected sigma is ~0.707 px has rho3d ~ rho2d at every pixel)
    const bool near_thr = fabsf(araw - 0.00392156862745098f) < 4.0e-7f || fabsf(r.depth - SRF_NEAR_F) < 2.0e-5f ||
                          fabsf(rho3d - rho2d) <= 1.0e-5f * rho2d;
    if (near_thr && pz != 0.0f) {
        PairEval e;
        eval_pair(q0, q1, q2, pixx, pixy, e);
        r.depth = e.depth; r.G = e.G; r.alpha = e.alpha; r.lowpass = !(e.rho3d <= e.rho2d); r.valid = e.valid;
    }
}

template <int BATCH, int NW>
struct BwdSmem {
    static constexpr size_t rec = 0;                                                         // float4 [6][BATCH]
    static constexpr size_t x = rec + sizeof(float4) * SRF_REC_QUADS * BATCH;                // float [warps][3][16][32]
    static constexpr size_t pixA = x + sizeof(float) * NW * 3 * kBwdGroup * 32;              // float4 [threads] dn0 dn1 dn2 dpix0
    static constexpr size_t pixB = pixA + sizeof(float4) * NW * 32;                          // float4 [threads] dpix1 dpix2 dL_ddepth dL_dalpha
    static constexpr size_t list = pixB + sizeof(float4) * NW * 32;                          // uint8 [warps][BATCH]
    static constexpr size_t wmax = list + (size_t)NW * BATCH;                                // int [warps]
    static constexpr size_t total = wmax + sizeof(int) * 8;
};

// EXACT : phase 1 evaluates pairs with the forward's exact sequence (else approximate + exact re-check at thresholds)
// P2WALK: 0 = all phase-2 lanes step through the 16 pixels of their half block together; 1 = every lane walks the
//         contributing pixels of its own half block; 2 = the two lanes of a splat share ALL its contributing pixels
//         alternately (a splat that only touches one half block no longer leaves its other lane idle); 3 = the 32
//         lanes are allotted to the group's splats in proportion to their contributing pixels (see phase 2 below)
// SMEMC : phase 1 reads the pixel's upstream gradients from shared memory (eight registers less)
// NW    : warps per CTA -- 8 = one CTA per 16x16 tile, 4 = one CTA per 16x8 half tile (two CTAs walk the tile's list)
// PREF  : (BATCH == threads) every thread fetches the list entry it will stage in the NEXT round while the current
//         round is being processed, so that a round's staging waits for one global load, not two dependent ones
template <int BATCH, int NW, int MINB, bool EXACT, int P2WALK, bool SMEMC, bool PREF = false, bool SADDR = false, bool PIXREG = false>
__global__ void __launch_bounds__(NW * 32, MINB) render_bwd_kernel(RenderBwdArgs a) {
    static_assert(BATCH <= 256, "hit lists are uint8");
    extern __shared__ __align__(16) unsigned char smem[];
    typedef BwdSmem<BATCH, NW> L;
    constexpr int NT = NW * 32;
    float4 (*s_rec)[BATCH] = reinterpret_cast<float4 (*)[BATCH]>(smem + L::rec);
    float4* s_pixA = reinterpret_cast<float4*>(smem + L::pixA);
    float4* s_pixB = reinterpret_cast<float4*>(smem + L::pixB);
    int* s_wmax = reinterpret_cast<int*>(smem + L::wmax);

    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    float* s_xw = reinterpret_cast<float*>(smem + L::x) + wid * (3 * kBwdGroup * 32);
    uint8_t* s_listw = reinterpret_cast<uint8_t*>(smem + L::list) + wid * BATCH;
    uint32_t sa_base = SADDR ? smem_addr(smem) : 0u;
    if (SADDR) asm volatile("" : "+r"(sa_base));          // opaque: kept in a register, not rebuilt at every use
    const uint32_t sa_rec = sa_base + (uint32_t)L::rec, sa_x = sa_base + (uint32_t)(L::x + wid * (3 * kBwdGroup * 32 * sizeof(float))),
                   sa_list = sa_base + (uint32_t)(L::list + wid * BATCH);

    const int view = blockIdx.y;
    const size_t npix = (size_t)a.W * a.H;
    a.ranges = view_ptr(a.ranges, view, a.tile_stride);
    a.tile_order = view_ptr(a.tile_order, view, a.tile_stride);
    a.point_list = view_ptr(a.point_list, view, a.plist_stride);
    a.rec = view_ptr(a.rec, view, a.geom_stride);
    a.bg += (size_t)view * a.cam_stride;
    a.accum = view_ptr(a.accum, view, a.image_stride);
    a.n_contrib = view_ptr(a.n_contrib, view, a.image_stride);
    a.dL_dpix += (size_t)view * 3 * npix;
    a.dL_dothers += (size_t)view * 8 * npix;
    a.ggrad = view_ptr(a.ggrad, view, a.ggrad_stride);

    const int tile = (int)a.tile_order[blockIdx.x / (8 / NW)];
    const int gw = (int)(blockIdx.x % (8 / NW)) * NW + wid;       // which of the tile's eight 8x4 blocks
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
    // the upstream values phase 2 multiplies w with, indexed by the pixel's thread id (= wid*32 + lane)
    s_pixA[tid] = make_float4(dn0, dn1, dn2, dpix0);
    s_pixB[tid] = make_float4(dpix1, dpix2, dL_ddepth, dL_daccum);

    // deepest list entry any pixel of the warp / of the tile blended
    int wmax = last_contributor;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) wmax = max(wmax, __shfl_xor_sync(0xffffffffu, wmax, o));
    if (lane == 0) s_wmax[wid] = wmax;
    __syncthreads();
    int n_eff = 0;
#pragma unroll
    for (int w = 0; w < NW; ++w) n_eff = max(n_eff, s_wmax[w]);
    const int rounds = (n_eff + BATCH - 1) / BATCH;

    // accum_rec / last_* recursions of backward.cu:331-385, two channels per f32x2 pair:
    // (c0,c1) (c2,depth) (n0,n1) (n2,alpha); the matching upstream gradients are paired the same way
    // (the reference keeps the previous splat in last_* and folds it in at the top of the next iteration;
    //  folding it in at the bottom of its own iteration is the same arithmetic and needs no such state)
    f32x2 acc_c01 = zero2(), acc_c2d = zero2(), acc_n01 = zero2(), acc_n2a = zero2();
    const f32x2 r_dpix01 = pk2(dpix0, dpix1), r_dpix2d = pk2(dpix2, dL_ddepth);
    const f32x2 r_dn01 = pk2(dn0, dn1), r_dn2a = pk2(dn2, dL_daccum);
    float last_dL_dT = 0.f;
    const float nTfinal_bg = -T_final * bg_dot_dpixel;

    // this lane's pixel centre (PIXREG: held in two registers instead of being rebuilt from the lane id per pair)
    float pixx = bx0 + (float)(lane & 7), pixy = by0 + (float)(lane >> 3);
    if (PIXREG) asm volatile("" : "+f"(pixx), "+f"(pixy));

    // phase-2 identity of this lane
    const int p2_i = lane & (kBwdGroup - 1), p2_h = lane >> 4;
    // P2WALK 3: this lane's candidate chunk size C = p2_i + 1 and the multiplier that turns n / C into a multiply
    // ((n * M) >> 16 == n / C exactly while n * C < 65536; n <= 47, C <= 16 here)
    const uint32_t candM = 65536u / (uint32_t)(p2_i + 1) + 1u;

    static_assert(!PREF || BATCH == NW * 32, "PREF stages one entry per thread and round");
    uint32_t next_id = 0;
    if (PREF && n_eff - 1 - tid >= 0) next_id = __ldg(a.point_list + range.x + (n_eff - 1 - tid));

    for (int b = 0; b < rounds; ++b) {
        // ---- stage batch b (back to front: slot j holds list position n_eff-1-(b*BATCH+j))
        __syncthreads();                                  // every warp is done with the previous batch's records
        for (int jt = tid; jt < BATCH; jt += NT) {
            const int pos = n_eff - 1 - (b * BATCH + jt);
            if (pos >= 0) {
                const uint32_t id = PREF ? next_id : __ldg(a.point_list + range.x + pos);
                const float4* r = a.rec + (size_t)id * SRF_REC_QUADS;
#pragma unroll
                for (int k = 0; k < SRF_REC_QUADS; ++k) s_rec[k][jt] = ldg4(r + k);
                // the splat id rides in the (otherwise unused by the blend) clamp-bits word of q4
                s_rec[4][jt].w = __uint_as_float(id);
            }
        }
        if (PREF) {
            const int npos = n_eff - 1 - ((b + 1) * BATCH + tid);
            if (npos >= 0) next_id = __ldg(a.point_list + range.x + npos);
        }
        __syncthreads();
        const int cnt = min(BATCH, n_eff - b * BATCH);

        // ---- warp-level cull: compacted list of the staged splats whose alpha >= 1/255 octagon can touch
        // this warp's 8x4 block and that are not behind the warp's deepest contributor
        int nh = 0;
        for (int c = 0; c < cnt; c += 32) {
            const int jt = c + lane;
            bool hit = false;
            if (jt < cnt && n_eff - 1 - (b * BATCH + jt) < wmax) hit = octagon_hits(s_rec[2][jt], s_rec[5][jt], warp_rect_at(bx0, by0));
            const unsigned hits = __ballot_sync(0xffffffffu, hit);
            if (hit) s_listw[nh + __popc(hits & ((1u << lane) - 1u))] = (uint8_t)jt;
            nh += __popc(hits);
        }
        __syncwarp();

        for (int g0 = 0; g0 < nh; g0 += 32) {
            // per-pixel hit words of 32 list entries: lane l rasterises splat g0+l over the block, the 32x32
            // bit transpose hands lane p the word "which of these 32 splats can touch MY pixel"
            uint32_t colword;
            {
                uint32_t m = 0;
                if (g0 + lane < nh) {
                    const int j = s_listw[g0 + lane];
                    m = octagon_pixel_mask(s_rec[2][j], s_rec[5][j], warp_rect_at(bx0, by0));
                }
                colword = transpose32(m, lane);
            }
#pragma unroll 1
            for (int sub = 0; sub < 2; ++sub) {
                const int gbase = g0 + sub * kBwdGroup;
                if (gbase >= nh) break;
                const uint8_t* lst = s_listw + gbase;

                // ================= phase 1: lane = pixel =================
                uint32_t bits = (colword >> (sub * kBwdGroup)) & 0xffffu;
                if (last_contributor == 0) bits = 0;
                uint32_t vbits = 0;
                const int iters1 = (int)__reduce_max_sync(0xffffffffu, (unsigned)__popc(bits));
                for (int it = 0; it < iters1; ++it) {
                    if (bits == 0) continue;
                    const int i = __ffs(bits) - 1;
                    bits &= bits - 1;
                    const int j = SADDR ? (int)lds_u8(sa_list + gbase + i) : (int)lst[i];
                    const int pos = n_eff - 1 - (b * BATCH + j);   // 0-based position in the tile list
                    if (pos >= last_contributor) continue;
                    PairBwd e;
                    const uint32_t sa_j = sa_rec + 16u * j;
                    if (SADDR)
                        eval_pair_bwd<EXACT>(lds_f4(sa_j), lds_f4(sa_j + 16u * BATCH), lds_f4(sa_j + 32u * BATCH), pixx, pixy, e);
                    else
                        eval_pair_bwd<EXACT>(s_rec[0][j], s_rec[1][j], s_rec[2][j], pixx, pixy, e);
                    if (!e.valid) continue;
                    const bool lowpass = e.lowpass;
                    const float4 q3 = SADDR ? lds_f4(sa_j + 48u * BATCH) : s_rec[3][j];
                    const float4 q4 = SADDR ? lds_f4(sa_j + 64u * BATCH) : s_rec[4][j];
                    const float alpha = e.alpha, c_d = e.depth;

                    // one reciprocal serves T / (1-alpha) and the background term's T_final / (1-alpha)
                    const float r1ma = rcp_fast(1.0f - alpha);   // 1 - alpha >= 0.01
                    T = T * r1ma;
                    const float w = alpha * T;
                    const f32x2 cur_c01 = pk2(q4.x, q4.y), cur_c2d = pk2(q4.z, c_d);
                    const f32x2 cur_n01 = pk2(q3.x, q3.y), cur_n2a = pk2(q3.z, 1.0f);
                    // dL_dalpha += (channel - accum_rec) * dL_dchannel over colour, depth, normal, alpha
                    f32x2 dpix01 = r_dpix01, dpix2d = r_dpix2d, dn01 = r_dn01, dn2a = r_dn2a;
                    if (SMEMC) {
                        const float4 ua = s_pixA[tid], ub = s_pixB[tid];
                        dpix01 = pk2(ua.w, ub.x); dpix2d = pk2(ub.y, ub.z); dn01 = pk2(ua.x, ua.y); dn2a = pk2(ua.z, ub.w);
                    }
                    f32x2 dsum = mul2(sub2(cur_c01, acc_c01), dpix01);
                    dsum = fma2(sub2(cur_c2d, acc_c2d), dpix2d, dsum);
                    dsum = fma2(sub2(cur_n01, acc_n01), dn01, dsum);
                    dsum = fma2(sub2(cur_n2a, acc_n2a), dn2a, dsum);
                    const float2 dsum_ = up2(dsum);
                    // accum_rec <- alpha * channel + (1 - alpha) * accum_rec  (all eight channels), for the next splat
                    const f32x2 la2 = bc2(alpha), oma2 = bc2(1.0f - alpha);
                    acc_c01 = fma2(cur_c01, la2, mul2(acc_c01, oma2));
                    acc_c2d = fma2(cur_c2d, la2, mul2(acc_c2d, oma2));
                    acc_n01 = fma2(cur_n01, la2, mul2(acc_n01, oma2));
                    acc_n2a = fma2(cur_n2a, la2, mul2(acc_n2a, oma2));

                    float dL_dz = w * up2(dpix2d).y, dL_dweight = 0.0f;
                    // distortion / median terms (backward.cu:350-368).  m_d = (FAR d - FAR NEAR)/((FAR-NEAR) d)
                    // = c1 - c2/d and d m_d/dd = c2/d^2; the reference evaluates both in double.  fp32 is
                    // enough here: the weight term below is stationary in m_d (its derivative is
                    // 2 (m_d A - D) ~ 0), and the gradients carry 1e-6 atomic-order noise anyway.
                    const float rcd = rcp_fast(c_d);             // depth >= 0.2
                    const float m_d = fmaf(-(float)(20.0 / 99.8), rcd, (float)(100.0 / 99.8));
                    const float dmd_dd = (float)(20.0 / 99.8) * rcd * rcd;
                    if (pos == median_contributor - 1) {
                        dL_dz += dL_dmedian_depth;
                        dL_dweight += dL_dmax_dweight;
                    }
                    dL_dweight += (final_D2 + m_d * m_d * final_A - 2.0f * m_d * final_D) * dL_dreg;
                    float dL_dalpha = (dsum_.x + dsum_.y) + (dL_dweight - last_dL_dT);
                    last_dL_dT = dL_dweight * alpha + (1.0f - alpha) * last_dL_dT;
                    const float dL_dmd = 2.0f * w * (m_d * final_A - final_D) * dL_dreg;
                    dL_dz += dL_dmd * dmd_dd;
                    dL_dalpha *= T;
                    // background term (backward.cu:391-396)
                    dL_dalpha = fmaf(nTfinal_bg, r1ma, dL_dalpha);

                    // park the three scalars phase 2 needs; the sign of w carries the branch (w > 0 always)
                    if (SADDR) {
                        const uint32_t xa = sa_x + 4u * (uint32_t)(i * 32 + (lane ^ i));
                        sts_f(xa, lowpass ? -w : w);
                        sts_f(xa + 4u * kBwdGroup * 32, e.G * dL_dalpha);
                        sts_f(xa + 8u * kBwdGroup * 32, dL_dz);
                    } else {
                        float* xp = s_xw + (i * 32 + (lane ^ i));
                        xp[0] = lowpass ? -w : w;
                        xp[kBwdGroup * 32] = e.G * dL_dalpha;
                        xp[2 * kBwdGroup * 32] = dL_dz;
                    }
                    vbits |= 1u << i;
                }

                __syncwarp();     // phase-1 stores to the X tile are visible to the whole warp

                // ================= phase 2: lane = (splat, chunk of its pixels) =================
                // valid-pair words: lane i (< 16) receives "which pixels contributed to splat i"
                const uint32_t tw = transpose32(vbits, lane);
                int own = p2_i;               // the splat of the group this lane accumulates for
                uint32_t word, mybits, tmask = 0u;
                bool have;
                int iters2;
                if (P2WALK == 3) {
                    // Lanes in proportion to work.  Splat i has c_i contributing pixels; with chunk size C it gets
                    // n_i = ceil(c_i / C) lanes, lane r of them takes its pixels of rank [r C, (r + 1) C), and the loop
                    // below makes C trips.  C is the smallest value for which the lanes suffice (sum n_i <= 32;
                    // C = 16 always does): ~8.5 trips per group on the bench scene against ~15 with two lanes per
                    // splat (tools/phase2_balance.py).
                    const int npx = __popc(tw);                    // lanes >= 16 hold no word: 0
                    if (__ballot_sync(0xffffffffu, npx != 0) == 0u) continue;
                    // lane (C - 1) + 16 h adds up ceil(c_i / C) over the splats 8 h .. 8 h + 7
                    int part = 0;
#pragma unroll
                    for (int k = 0; k < 8; ++k) {
                        const int c = __shfl_sync(0xffffffffu, npx, p2_h * 8 + k);
                        part += (int)(((uint32_t)(c + p2_i) * candM) >> 16);
                    }
                    const int lanes_needed = part + __shfl_xor_sync(0xffffffffu, part, 16);
                    const int C = __ffs(__ballot_sync(0xffffffffu, lanes_needed <= 32) & 0xffffu);      // 1..16
                    const uint32_t M = __shfl_sync(0xffffffffu, candM, C - 1);
                    const int n_mine = (int)(((uint32_t)(npx + C - 1) * M) >> 16);                       // lanes >= 16: 0
                    int end = n_mine;                              // inclusive scan over the lanes 0..15
#pragma unroll
                    for (int o = 1; o < kBwdGroup; o <<= 1) {
                        const int v = __shfl_up_sync(0xffffffffu, end, o);
                        if (lane >= o) end += v;
                    }
                    const int lanes_used = __shfl_sync(0xffffffffu, end, kBwdGroup - 1);
                    // owner of this lane: the first splat whose lanes end beyond it (lower bound over end[0..15])
                    own = 0;
#pragma unroll
                    for (int st = kBwdGroup / 2; st > 0; st >>= 1) {
                        const int e = __shfl_sync(0xffffffffu, end, own + st - 1);
                        if (e <= lane) own += st;
                    }
                    const int own_end = __shfl_sync(0xffffffffu, end, own);
                    const int own_n = __shfl_sync(0xffffffffu, n_mine, own);
                    word = __shfl_sync(0xffffffffu, tw, own);
                    have = lane < lanes_used;
                    // drop the lowest r C contributing pixels of the word (r = rank of this lane among the splat's
                    // lanes; r C < c_own): the largest pos with popc(word below pos) <= r C
                    const int skip = (lane - (own_end - own_n)) * C;
                    int pos = 0;
#pragma unroll
                    for (int st = 16; st > 0; st >>= 1) {
                        const int below = __popc(word & ((1u << (pos + st)) - 1u));
                        if (below <= skip) pos += st;
                    }
                    mybits = have ? (word & (0xffffffffu << pos)) : 0u;
                    if (!have) { own = 0; word = 0u; }
                    iters2 = C;
                } else {
                    word = __shfl_sync(0xffffffffu, tw, p2_i);
                    have = gbase + p2_i < nh;
                    mybits = have ? ((word >> (16 * p2_h)) & 0xffffu) : 0u;
                    if (P2WALK == 2) {
                        mybits = have ? word : 0u;
                        if (p2_h) mybits &= mybits - 1;        // the second lane of a splat starts at its second pixel
                    }
                    tmask = __reduce_or_sync(0xffffffffu, mybits);
                    iters2 = P2WALK == 2 ? (int)__reduce_max_sync(0xffffffffu, (unsigned)(__popc(mybits) + 1) >> 1)
                           : P2WALK == 1 ? (int)__reduce_max_sync(0xffffffffu, (unsigned)__popc(mybits)) : __popc(tmask);
                }
                if (iters2 == 0) continue;
                const int j2 = have ? (int)lst[own] : 0;
                const float4 q0 = s_rec[0][j2], q1 = s_rec[1][j2], q2 = s_rec[2][j2];
                const uint32_t splat_id = __float_as_uint(s_rec[4][j2].w);
                const f32x2 nTu_x = pk2(-q0.x, -q0.y), nTu_y = pk2(-q0.z, -q0.w), nTu_z = pk2(-q1.x, -q1.y);
                const float Twx = q1.z, Twy = q1.w, Twz = q2.x;
                const f32x2 Twxy = pk2(Twx, Twy), cen = pk2(q2.y, q2.z);
                const float nopac = -q2.w;
                // accumulators, laid out as the gradient record: (DT0,DT1) (DT2,DT3) (DT4,DT5) (DT6,DT7) (DT8,DOPAC)
                // (DN0,DN1) (DN2,DC0) (DC1,DC2) (DM0,DM1)
                f32x2 A0 = zero2(), A1 = zero2(), A2 = zero2(), A3 = zero2(), A4 = zero2(), A5 = zero2(), A6 = zero2(), A7 = zero2(), A8 = zero2();
                const float* xrow = s_xw + own * 32;
                const float ybase = by0 + (P2WALK >= 2 ? 0.0f : (float)(2 * p2_h));
                const int pbase = wid * 32 + (P2WALK >= 2 ? 0 : 16 * p2_h);
#pragma unroll 1
                for (int it = 0; it < iters2; ++it) {
                    int t;
                    if (P2WALK == 2) {
                        if (mybits == 0) continue;
                        t = __ffs(mybits) - 1;             // mine ...
                        mybits &= mybits - 1;
                        mybits &= mybits - 1;              // ... and the next one is the partner lane's
                    } else if (P2WALK == 1 || P2WALK == 3) {
                        if (mybits == 0) continue;
                        t = __ffs(mybits) - 1;             // every lane walks its own contributing pixels
                        mybits &= mybits - 1;
                    } else {
                        t = __ffs(tmask) - 1;              // all lanes step through the half block's pixels together
                        tmask &= tmask - 1;
                        if (!((mybits >> t) & 1u)) continue;
                    }
                    const int p = P2WALK >= 2 ? t : t + 16 * p2_h;
                    const float ppx = bx0 + (float)(t & 7), ppy = ybase + (float)(t >> 3);
                    const float* xp = xrow + (p ^ own);
                    const float ws = xp[0], GdA = xp[kBwdGroup * 32], dL_dz = xp[2 * kBwdGroup * 32];
                    const float4 pa = s_pixA[pbase + t];
                    const float4 pb = s_pixB[pbase + t];
                    const float w = fabsf(ws);
                    const f32x2 w2 = bc2(w);
                    fma2_acc(A5, w2, pk2(pa.x, pa.y));      // dL/dnormal
                    fma2_acc(A6, w2, pk2(pa.z, pa.w));      // dL/dnormal.z, dL/dcolor.r
                    fma2_acc(A7, w2, pk2(pb.x, pb.y));      // dL/dcolor.gb
                    const f32x2 pix2 = pk2(ppx, ppy);
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
                        add2_acc(A4, pk2(tw8, GdA));
                    } else {
                        // low-pass branch (backward.cu:436-443); FilterInvSquare == 2 after fp32 rounding
                        const f32x2 d = sub2(cen, pix2);
                        fma2_acc(A8, d, bc2(2.0f * nopac * GdA));
                        add2_acc(A4, pk2(dL_dz, GdA));
                    }
                }
                if (P2WALK == 3) {
                    // every lane sends its own partial sums (a lane that is in use took at least one pair)
                    if (have) {
                        float* dst = a.ggrad + (size_t)splat_id * SRF_GRAD_FLOATS;
                        const float2 a0 = up2(A0), a1 = up2(A1), a2 = up2(A2), a3 = up2(A3), a8 = up2(A8);
                        const float2 a4 = up2(A4), a5 = up2(A5), a6 = up2(A6), a7 = up2(A7);
                        red_add_v4(dst + 0, a0.x, a0.y, a1.x, a1.y);
                        red_add_v4(dst + 4, a2.x, a2.y, a3.x, a3.y);
                        red_add_v4(dst + 8, a4.x, a4.y, a5.x, a5.y);
                        red_add_v4(dst + 12, a6.x, a6.y, a7.x, a7.y);
                        if (a8.x != 0.0f || a8.y != 0.0f) red_add_v4(dst + 16, a8.x, a8.y, 0.0f, 0.0f);
                    }
                    __syncwarp();
                    continue;
                }
                // combine the two half blocks and send the totals out: lanes of half 0 own record quads 0,1
                // (and 4 if a low-pass pair touched the splat), lanes of half 1 own quads 2,3
                A0 = add2(A0, shfl_xor2(A0, 16)); A1 = add2(A1, shfl_xor2(A1, 16));
                A2 = add2(A2, shfl_xor2(A2, 16)); A3 = add2(A3, shfl_xor2(A3, 16));
                A4 = add2(A4, shfl_xor2(A4, 16)); A5 = add2(A5, shfl_xor2(A5, 16));
                A6 = add2(A6, shfl_xor2(A6, 16)); A7 = add2(A7, shfl_xor2(A7, 16));
                A8 = add2(A8, shfl_xor2(A8, 16));
                if (have && word != 0u) {
                    float* dst = a.ggrad + (size_t)splat_id * SRF_GRAD_FLOATS;
                    if (p2_h == 0) {
                        const float2 a0 = up2(A0), a1 = up2(A1), a2 = up2(A2), a3 = up2(A3), a8 = up2(A8);
                        red_add_v4(dst + 0, a0.x, a0.y, a1.x, a1.y);
                        red_add_v4(dst + 4, a2.x, a2.y, a3.x, a3.y);
                        if (a8.x != 0.0f || a8.y != 0.0f) red_add_v4(dst + 16, a8.x, a8.y, 0.0f, 0.0f);
                    } else {
                        const float2 a4 = up2(A4), a5 = up2(A5), a6 = up2(A6), a7 = up2(A7);
                        red_add_v4(dst + 8, a4.x, a4.y, a5.x, a5.y);
                        red_add_v4(dst + 12, a6.x, a6.y, a7.x, a7.y);
                    }
                }
                __syncwarp();     // phase 1 of the next group overwrites the X tile
            }
        }
    }
}

}  // namespace

cudaError_t launch_render_bwd_v1(const RenderBwdArgs& a, cudaStream_t stream);

template <int B, int NW, int MINB, bool EXACT, int P2WALK, bool SMEMC, bool PREF = false, bool SADDR = false, bool PIXREG = false>
static cudaError_t launch_variant(const RenderBwdArgs& a, cudaStream_t stream) {
    auto k = render_bwd_kernel<B, NW, MINB, EXACT, P2WALK, SMEMC, PREF, SADDR, PIXREG>;
    // the opt-in is per device (and cheap): made on every call for the current device
    cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BwdSmem<B, NW>::total);
    if (e != cudaSuccess) return e;
    k<<<dim3(a.gx * a.gy * (8 / NW), a.nviews), NW * 32, BwdSmem<B, NW>::total, stream>>>(a);
    return cudaSuccess;
}

cudaError_t launch_render_bwd(const RenderBwdArgs& a, cudaStream_t stream) {
    const int ntiles = a.gx * a.gy;
    if (ntiles <= 0 || a.nviews <= 0) return cudaSuccess;
    const int variant = bwd_variant();
    if (variant == 1) return launch_render_bwd_v1(a, stream);
    prof_start(K_RENDER_BWD, stream);
    cudaError_t e = cudaSuccess;
    // <splats per round, warps per CTA, CTAs per SM, exact pair evaluation, phase-2 walk, upstream gradients from smem,
    //  list-entry prefetch, explicit shared addressing in phase 1, pixel centre pinned in registers>
    // 2..8 are the fixed phase-2 layouts of the first two-phase kernel, 9..17 the steps from there to the default; compare
    // them with SRF_BWD_VARIANT=<n> python bench.py (kernels_us.render_bwd).
    switch (variant) {
        case 2: e = launch_variant<256, 8, 2, false, 1, false>(a, stream); break;      // one CTA per tile, own-half phase-2 lanes
        case 3: e = launch_variant<160, 8, 3, false, 1, true>(a, stream); break;       // three CTAs per SM
        case 4: e = launch_variant<256, 8, 2, false, 0, false>(a, stream); break;      // lock-step phase 2
        case 5: e = launch_variant<256, 8, 2, true, 1, false>(a, stream); break;       // exact pair evaluation everywhere
        case 6: e = launch_variant<256, 4, 4, false, 1, false>(a, stream); break;      // half-tile CTAs
        case 7: e = launch_variant<256, 4, 4, false, 2, false>(a, stream); break;      // half-tile CTAs, shared phase-2 lanes
        case 8: e = launch_variant<256, 8, 2, false, 2, false>(a, stream); break;      // one CTA per tile, shared phase-2 lanes
        case 9: e = launch_variant<256, 4, 4, false, 3, false>(a, stream); break;      // 7 + phase-2 lanes in proportion to work
        case 10: e = launch_variant<256, 8, 2, false, 3, false>(a, stream); break;     // the same, one CTA per tile
        case 11: e = launch_variant<128, 4, 5, false, 3, true>(a, stream); break;      // five half-tile CTAs per SM, upstream grads from smem
        case 12: e = launch_variant<128, 4, 5, false, 3, false>(a, stream); break;     // five half-tile CTAs per SM
        case 13: e = launch_variant<64, 4, 6, false, 3, true>(a, stream); break;       // six CTAs per SM, 64-splat rounds
        case 14: e = launch_variant<128, 8, 3, false, 3, true>(a, stream); break;      // six CTAs' worth of warps as three 8-warp CTAs
        case 15: e = launch_variant<128, 4, 5, false, 2, false>(a, stream); break;     // five CTAs per SM WITHOUT the allotment
        case 16: e = launch_variant<128, 4, 5, false, 3, false, true>(a, stream); break;        // 12 + prefetch
        case 17: e = launch_variant<128, 4, 5, false, 3, false, true, true>(a, stream); break;  // 16 + explicit shared addressing
        default: e = launch_variant<128, 4, 5, false, 3, false, true, true, true>(a, stream); break;   // 18: 17 + pinned pixel centre
    }
    prof_stop(K_RENDER_BWD, stream);
    return e != cudaSuccess ? e : cudaGetLastError();
}

}  // namespace srf
