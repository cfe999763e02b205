// render_bwd_v1.cu -- round-1 form of the blend backward (K7), kept for A/B timing (SRF_BWD_VARIANT=1).
// Replaces reference backward.cu:143-449 (renderCUDA backward).
//
// Same tiling as the forward: one CTA per 16x16 tile, one thread per pixel, the tile's
// list walked back-to-front in shared-memory rounds of SRF_BATCH = 256 splats.  The reference emits
// 10-16 global float atomics per (pixel, splat) pair, 256 threads hammering the same
// <=18 addresses.  Here each warp first transposes-and-reduces the 16 partial
// derivatives every contributing pair produces across its 32 lanes with a 16-shuffle
// reduce-scatter (8+4+2+1+1; the two extra low-pass-branch values take a small butterfly
// on the ~6 % of visits that have them), adds the warp totals into a per-batch shared-memory accumulator
// (bank-conflict-free, 18 consecutive words per splat) and the CTA finally issues at
// most five 128-bit vector reductions (red.global.add.v4.f32) per splat per tile.
// Further savings the reference does not have:
//   * the walk starts at the tile's last *used* list entry (max n_contrib over the
//     tile) instead of the end of the list,
//   * warp-uniform skips: entries beyond the warp's deepest contributor, and splats
//     that no lane of the warp touches, cost no reduction traffic at all.
#include "surfel_common.cuh"
#include "surfel_kernels.h"

namespace srf {

// MUFU.RCP, <= 1 ulp: the gradients need no bit-exactness (the forward-deciding chain in eval_pair()
// keeps its IEEE divisions), and an IEEE reciprocal costs ~9 instructions plus a slow-path call.
__device__ __forceinline__ float rcp_fast(float x) {
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

__device__ __forceinline__ void red_add_v4(float* addr, float4 v) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(v.x), "f"(v.y), "f"(v.z),
                 "f"(v.w)
                 : "memory");
}

// Reduce-scatter of 16 per-lane values over the warp (16 -> 8 -> 4 -> 2 -> 1 values per lane, then the
// two lanes of a pair are combined): every lane returns the warp total of value (lane >> 1) & 15.
// 16 shuffles; a power of two, so there is no padding logic.
__device__ __forceinline__ float warp_reduce_scatter16(const float (&v)[16], int lane) {
    const unsigned full = 0xffffffffu;
    const bool u4 = (lane & 16) != 0, u3 = (lane & 8) != 0, u2 = (lane & 4) != 0, u1 = (lane & 2) != 0;
    float a[8], b[4], c[2];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const float keep = u4 ? v[8 + i] : v[i];
        const float send = u4 ? v[i] : v[8 + i];
        a[i] = keep + __shfl_xor_sync(full, send, 16);
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float keep = u3 ? a[4 + i] : a[i];
        const float send = u3 ? a[i] : a[4 + i];
        b[i] = keep + __shfl_xor_sync(full, send, 8);
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const float keep = u2 ? b[2 + i] : b[i];
        const float send = u2 ? b[i] : b[2 + i];
        c[i] = keep + __shfl_xor_sync(full, send, 4);
    }
    float d = (u1 ? c[1] : c[0]) + __shfl_xor_sync(full, u1 ? c[0] : c[1], 2);
    d += __shfl_xor_sync(full, d, 1);
    return d;
}

__global__ void __launch_bounds__(SRF_CTA_THREADS, 768 / SRF_CTA_THREADS) render_bwd_v1_kernel(RenderBwdArgs a) {
    __shared__ float4 s_rec[SRF_REC_QUADS][SRF_BATCH];
    __shared__ __align__(16) float s_grad[SRF_BATCH * SRF_GRAD_FLOATS];
    __shared__ uint32_t s_id[SRF_BATCH];
    __shared__ int s_touched[SRF_BATCH];
    __shared__ int s_wmax[SRF_CTA_WARPS];

    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int tile = (int)a.tile_order[blockIdx.x / SRF_CTAS_PER_TILE];
    const int gw = (int)(blockIdx.x % SRF_CTAS_PER_TILE) * SRF_CTA_WARPS + wid;   // which of the tile's eight 8x4 blocks
    const int tyi = tile / a.gx, txi = tile - tyi * a.gx;
    int lx, ly;
    tile_pixel(gw * 32 + lane, lx, ly);
    const int pxi = txi * SRF_TILE + lx, pyi = tyi * SRF_TILE + ly;
    const bool inside = pxi < a.W && pyi < a.H;
    const float pixx = (float)pxi + 0.5f, pixy = (float)pyi + 0.5f;
    const size_t npix = (size_t)a.W * a.H;
    const size_t pix = (size_t)pyi * a.W + pxi;
    const WarpRect wrect = make_warp_rect(txi, tyi, gw);

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

    // deepest list entry any pixel of the warp / of the tile blended
    int wmax = last_contributor;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) wmax = max(wmax, __shfl_xor_sync(0xffffffffu, wmax, o));
    if (lane == 0) s_wmax[wid] = wmax;
    __syncthreads();
    int n_eff = 0;
#pragma unroll
    for (int w = 0; w < SRF_CTA_WARPS; ++w) n_eff = max(n_eff, s_wmax[w]);
    const int rounds = (n_eff + SRF_BATCH - 1) / SRF_BATCH;

    // accum_rec / last_* recursions of backward.cu:331-385, two channels per f32x2 pair:
    // (c0,c1) (c2,depth) (n0,n1) (n2,alpha); the matching upstream gradients are paired the same way
    f32x2 acc_c01 = zero2(), acc_c2d = zero2(), acc_n01 = zero2(), acc_n2a = zero2();
    f32x2 last_c01 = zero2(), last_c2d = zero2(), last_n01 = zero2(), last_n2a = zero2();
    float last_alpha = 0.f;
    const f32x2 dpix01 = pk2(dpix0, dpix1), dpix2d = pk2(dpix2, dL_ddepth);
    const f32x2 dn01 = pk2(dn0, dn1), dn2a = pk2(dn2, dL_daccum);
    const float npixy = -pixy;
    float last_dL_dT = 0.f;

    for (int b = 0; b < rounds; ++b) {
        // stage batch b (back to front) and clear the accumulator rows this thread owns
        const int pos_mine = n_eff - 1 - (b * SRF_BATCH + tid);
        if (pos_mine >= 0) {
            const uint32_t id = __ldg(a.point_list + range.x + pos_mine);
            s_id[tid] = id;
            const float4* r = a.rec + (size_t)id * SRF_REC_QUADS;
#pragma unroll
            for (int k = 0; k < SRF_REC_QUADS; ++k) s_rec[k][tid] = ldg4(r + k);
        }
        {
            float4* g4 = reinterpret_cast<float4*>(s_grad + tid * SRF_GRAD_FLOATS);
#pragma unroll
            for (int k = 0; k < SRF_GRAD_FLOATS / 4; ++k) g4[k] = make_float4(0.f, 0.f, 0.f, 0.f);
            s_touched[tid] = 0;
        }
        __syncthreads();

        const int cnt = min(SRF_BATCH, n_eff - b * SRF_BATCH);
        const int nchunks = (cnt + 31) >> 5;
        for (int c = 0; c < nchunks; ++c) {
          // warp-level cull, 32 splats per ballot: skip splats behind the warp's deepest
          // contributor and splats whose alpha >= 1/255 box misses the warp's 8x4 pixel block
          unsigned hits;
          {
            const int jt = (c << 5) + lane;
            bool hit = false;
            if (jt < cnt && n_eff - 1 - (b * SRF_BATCH + jt) < wmax) {
                hit = octagon_hits(s_rec[2][jt], s_rec[5][jt], wrect);
            }
            hits = __ballot_sync(0xffffffffu, hit);
          }
          while (hits) {
            const int j = (c << 5) + __ffs(hits) - 1;
            hits &= hits - 1;
            const int pos = n_eff - 1 - (b * SRF_BATCH + j);   // 0-based position in the tile list
            bool contrib = inside && pos < last_contributor;
            PairEval e;
            const float4 q0 = s_rec[0][j], q1 = s_rec[1][j], q2 = s_rec[2][j];
            if (contrib) {
                eval_pair(q0, q1, q2, pixx, pixy, e);
                contrib = e.valid;
            }
            if (!__any_sync(0xffffffffu, contrib)) continue;

            float g[18];
#pragma unroll
            for (int i = 0; i < 18; ++i) g[i] = 0.0f;
            bool lowpass = false;

            if (contrib) {
                const float4 q3 = s_rec[3][j];
                const float4 q4 = s_rec[4][j];
                const float alpha = e.alpha, G = e.G, c_d = e.depth;
                const float Twx = q1.z, Twy = q1.w;
                const float opac = q2.w;

                // one reciprocal serves T / (1-alpha) and the background term's T_final / (1-alpha)
                const float r1ma = rcp_fast(1.0f - alpha);   // 1 - alpha >= 0.01
                T = T * r1ma;
                const float w = alpha * T;  // dchannel_dcolor
                // accum_rec <- last_alpha * last + (1 - last_alpha) * accum_rec  (all eight channels)
                const f32x2 la2 = bc2(last_alpha), oma2 = bc2(1.0f - last_alpha);
                acc_c01 = fma2(last_c01, la2, mul2(acc_c01, oma2));
                acc_c2d = fma2(last_c2d, la2, mul2(acc_c2d, oma2));
                acc_n01 = fma2(last_n01, la2, mul2(acc_n01, oma2));
                acc_n2a = fma2(last_n2a, la2, mul2(acc_n2a, oma2));
                last_c01 = pk2(q4.x, q4.y); last_c2d = pk2(q4.z, c_d);
                last_n01 = pk2(q3.x, q3.y); last_n2a = pk2(q3.z, 1.0f);
                // dL_dalpha += (channel - accum_rec) * dL_dchannel over colour, depth, normal, alpha
                f32x2 dsum = mul2(sub2(last_c01, acc_c01), dpix01);
                dsum = fma2(sub2(last_c2d, acc_c2d), dpix2d, dsum);
                dsum = fma2(sub2(last_n01, acc_n01), dn01, dsum);
                dsum = fma2(sub2(last_n2a, acc_n2a), dn2a, dsum);
                const float2 dsum_ = up2(dsum);
                // w * upstream: colour and normal gradients of the splat, and w * dL_ddepth for dL_dz
                const f32x2 w2 = bc2(w);
                const float2 gc01 = up2(mul2(dpix01, w2)), gc2d = up2(mul2(dpix2d, w2)), gn01 = up2(mul2(dn01, w2));
                g[SRF_G_DCOLOR + 0] = gc01.x; g[SRF_G_DCOLOR + 1] = gc01.y; g[SRF_G_DCOLOR + 2] = gc2d.x;
                g[SRF_G_DNORMAL + 0] = gn01.x; g[SRF_G_DNORMAL + 1] = gn01.y; g[SRF_G_DNORMAL + 2] = w * dn2;

                float dL_dz = gc2d.y, dL_dweight = 0.0f;
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
                last_alpha = alpha;
                // background term (backward.cu:391-396)
                dL_dalpha += (-T_final * r1ma) * bg_dot_dpixel;

                const float dL_dG = opac * dL_dalpha;

                if (e.rho3d <= e.rho2d) {
                    // ray-splat branch: vjp through s = p.xy / p.z, p = k x l (backward.cu:405-435)
                    const f32x2 S = pk2(e.sx, e.sy);
                    const f32x2 dS = fma2(S, bc2(dL_dG * -G), mul2(pk2(Twx, Twy), bc2(dL_dz)));   // (dL_dsx, dL_dsy)
                    const f32x2 dPxy = mul2(dS, bc2(rcp_fast(e.pz)));                           // (dL_dpx, dL_dpy)
                    const float2 dp = up2(dPxy), dps = up2(mul2(dPxy, S));
                    const float dpz = -(dps.x + dps.y);
                    // dL_dk = l x dL_dp, dL_dl = dL_dp x k, as the pairs (dk.c, -dl.c) = the gradient record's layout:
                    //   (dk.x,-dl.x) = (l.y,k.y) dpz - (l.z,k.z) dpy   and cyclic
                    const f32x2 Sx = pk2(e.lx, e.kx), Sy = pk2(e.ly, e.ky), Sz = pk2(e.lz, e.kz);
                    const float2 Dx = up2(fma2(Sy, bc2(dpz), mul2(Sz, bc2(-dp.y))));
                    const float2 Dy = up2(fma2(Sz, bc2(dp.x), mul2(Sx, bc2(-dpz))));
                    const float2 Dz = up2(fma2(Sx, bc2(dp.y), mul2(Sy, bc2(-dp.x))));
                    g[SRF_G_DT + 0] = Dx.x; g[SRF_G_DT + 1] = Dx.y;
                    g[SRF_G_DT + 2] = Dy.x; g[SRF_G_DT + 3] = Dy.y;
                    g[SRF_G_DT + 4] = Dz.x; g[SRF_G_DT + 5] = Dz.y;
                    // dL_dTw = pix.x dk + pix.y dl + dL_dz (s, 1)
                    const float2 zs = up2(mul2(S, bc2(dL_dz)));
                    g[SRF_G_DT + 6] = fmaf(pixx, Dx.x, fmaf(npixy, Dx.y, zs.x));
                    g[SRF_G_DT + 7] = fmaf(pixx, Dy.x, fmaf(npixy, Dy.y, zs.y));
                    g[SRF_G_DT + 8] = fmaf(pixx, Dz.x, fmaf(npixy, Dz.y, dL_dz));
                } else {
                    // low-pass branch (backward.cu:436-443); FilterInvSquare == 2 after fp32 rounding
                    lowpass = true;
                    const float2 gm = up2(mul2(pk2(e.dx, e.dy), bc2(dL_dG * (-2.0f * G))));
                    g[SRF_G_DMEAN2D + 0] = gm.x;
                    g[SRF_G_DMEAN2D + 1] = gm.y;
                    g[SRF_G_DT + 8] = dL_dz;
                }
                g[SRF_G_DOPAC] = G * dL_dalpha;
            }

            // slots 0..15 in one power-of-two reduce-scatter; even lanes own value lane >> 1
            {
                float v16[16];
#pragma unroll
                for (int i = 0; i < 16; ++i) v16[i] = g[i];
                const float total = warp_reduce_scatter16(v16, lane);
                if ((lane & 1) == 0) atomicAdd(&s_grad[j * SRF_GRAD_FLOATS + (lane >> 1)], total);
            }
            // the two dL/dmean2D values exist only on low-pass lanes (~6 % of the visits)
            if (__any_sync(0xffffffffu, lowpass)) {
                float m0 = g[SRF_G_DMEAN2D + 0], m1 = g[SRF_G_DMEAN2D + 1];
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
                    m0 += __shfl_xor_sync(0xffffffffu, m0, o);
                    m1 += __shfl_xor_sync(0xffffffffu, m1, o);
                }
                if (lane < 2) atomicAdd(&s_grad[j * SRF_GRAD_FLOATS + SRF_G_DMEAN2D + lane], lane ? m1 : m0);
            }
            if (lane == 0) s_touched[j] = 1;
          }
        }
        __syncthreads();

        // flush: one thread per staged splat, five 128-bit vector reductions
        if (pos_mine >= 0 && s_touched[tid]) {
            const float4* g4 = reinterpret_cast<const float4*>(s_grad + tid * SRF_GRAD_FLOATS);
            float* dst = a.ggrad + (size_t)s_id[tid] * SRF_GRAD_FLOATS;
#pragma unroll
            for (int k = 0; k < 4; ++k) red_add_v4(dst + 4 * k, g4[k]);
            const float4 gm = g4[4];                     // dL/dmean2D: only if a low-pass pair touched the splat
            if (gm.x != 0.0f || gm.y != 0.0f) red_add_v4(dst + 16, gm);
        }
        // (the same thread re-zeroes its row and restages its slot at the top of the loop;
        //  s_rec rows are protected by the barrier above)
    }
}

cudaError_t launch_render_bwd_v1(const RenderBwdArgs& a0, cudaStream_t stream) {
    const int ntiles = a0.gx * a0.gy;
    if (ntiles <= 0) return cudaSuccess;
    const size_t npix = (size_t)a0.W * a0.H;
    for (int v = 0; v < a0.nviews; ++v) {
        RenderBwdArgs a = a0;
        a.ranges = view_ptr(a0.ranges, v, a0.tile_stride);
        a.tile_order = view_ptr(a0.tile_order, v, a0.tile_stride);
        a.point_list = view_ptr(a0.point_list, v, a0.plist_stride);
        a.rec = view_ptr(a0.rec, v, a0.geom_stride);
        a.bg = a0.bg + (size_t)v * a0.cam_stride;
        a.accum = view_ptr(a0.accum, v, a0.image_stride);
        a.n_contrib = view_ptr(a0.n_contrib, v, a0.image_stride);
        a.dL_dpix = a0.dL_dpix + (size_t)v * 3 * npix;
        a.dL_dothers = a0.dL_dothers + (size_t)v * 8 * npix;
        a.ggrad = view_ptr(a0.ggrad, v, a0.ggrad_stride);
        prof_start(K_RENDER_BWD, stream);
        render_bwd_v1_kernel<<<ntiles * SRF_CTAS_PER_TILE, SRF_CTA_THREADS, 0, stream>>>(a);
        prof_stop(K_RENDER_BWD, stream);
    }
    return cudaGetLastError();
}

}  // namespace srf
