// preprocess.cu -- per-Gaussian forward preprocess (K1) and frustum visibility (K10).
//
// Replaces reference forward.cu:166-260 (preprocessCUDA) + auxiliary.h:160-185
// (in_frustum), forward.cu:75-128 (computeTransMat), :133-163 (computeAABB),
// :20-71 (computeColorFromSH), auxiliary.h:64-74 (getRect) and
// rasterizer_impl.cu:54-66 (checkFrustum).
//
// One thread per Gaussian, 256 per CTA.  Positions are staged through shared memory
// with 128-bit coalesced loads (a [P,3] fp32 array is not 16 B-strided per row);
// quaternions / scales / SH rows are loaded with native 128/64-bit vector loads.
// Instead of emitting tiles_touched for a prefix sum + duplicate pass, the kernel
// directly counts instances per tile (tile_count[]), the first half of the
// tile-bucketed binning that replaces the reference's global 64-bit radix sort.
#include <cuda_fp16.h>
#include <stdio.h>

#include "surfel_common.cuh"
#include "surfel_kernels.h"
#include "sh_eval.cuh"

namespace srf {

// Cooperative, 128-bit staging of `rows` consecutive rows of `row_floats` floats each
// starting at `src` into shared memory (falls back to scalar loads when unaligned).
__device__ __forceinline__ void stage_rows(float* __restrict__ dst, const float* __restrict__ src, int nfloats,
                                           int tid, int nthreads) {
    if ((reinterpret_cast<uintptr_t>(src) & 15) == 0) {
        const int nvec = nfloats >> 2;
        const float4* s4 = reinterpret_cast<const float4*>(src);
        float4* d4 = reinterpret_cast<float4*>(dst);
        for (int i = tid; i < nvec; i += nthreads) d4[i] = __ldg(s4 + i);
        for (int i = (nvec << 2) + tid; i < nfloats; i += nthreads) dst[i] = __ldg(src + i);
    } else {
        for (int i = tid; i < nfloats; i += nthreads) dst[i] = __ldg(src + i);
    }
}

// Adds one instance to every tile of rect [x0,x1) x [y0,y1).
__device__ __forceinline__ void count_tiles_serial(uint32_t* tile_count, int gx, int x0, int y0, int x1, int y1) {
    for (int y = y0; y < y1; ++y)
        for (int x = x0; x < x1; ++x) atomicAdd(&tile_count[(size_t)(y * gx + x) * SRF_TILE_CTR_STRIDE], 1u);
}

// The view's scene (blockIdx.y / Vs) gives the Gaussian rows and the field of view; one scene is S = 1.
__global__ void __launch_bounds__(256) preprocess_fwd_kernel(PreprocessArgs a, const __grid_constant__ SceneArgs s) {
    __shared__ __align__(16) float s_means[256 * 3];
    __shared__ float s_view[16];
    __shared__ float s_cam[3];
    extern __shared__ __align__(16) float s_sh[];  // 256 * 3M floats when SH staging is enabled

    const int tid = threadIdx.x;
    const int base = blockIdx.x * 256;
    const int idx = base + tid;
    const int nrows = min(256, a.P - base);
    const bool in_range = idx < a.P;
    // view of this CTA (blockIdx.y): own camera, own geom / tile workspace, own radii row; its scene's Gaussian rows
    const int view = blockIdx.y, scene = view / s.views_per_scene;
    a.viewmatrix += (size_t)view * a.cam_stride;
    a.campos += (size_t)view * a.cam_stride;
    a.radii += (size_t)view * a.P;
    a.rec = view_ptr(a.rec, view, a.geom_stride);
    a.depths = view_ptr(a.depths, view, a.geom_stride);
    a.rects = view_ptr(a.rects, view, a.geom_stride);
    a.tile_count = view_ptr(a.tile_count, view, a.tile_stride);
    const size_t row = (size_t)scene * a.P;
    a.means3D = rows_at(a.means3D, row, 3);
    a.scales = rows_at(a.scales, row, 2);
    a.rotations = rows_at(a.rotations, row, 4);
    a.opacities = rows_at(a.opacities, row, 1);
    a.shs = rows_at(a.shs, row, 3 * a.M);
    a.transMat_precomp = rows_at(a.transMat_precomp, row, 9);
    a.colors_precomp = rows_at(a.colors_precomp, row, 3);
    const float focal_x = s.fov[scene].x, focal_y = s.fov[scene].y;

    stage_rows(s_means, a.means3D + (size_t)base * 3, nrows * 3, tid, 256);
    if (tid < 16) s_view[tid] = __ldg(a.viewmatrix + tid);
    if (tid < 3) s_cam[tid] = __ldg(a.campos + tid);
    const int sh_row = 3 * a.M;
    const bool use_sh = (a.colors_precomp == nullptr);
    if (use_sh && a.stage_sh) stage_rows(s_sh, a.shs + (size_t)base * sh_row, nrows * sh_row, tid, 256);
    __syncthreads();

    int radius = 0;
    int x0 = 0, y0 = 0, x1 = 0, y1 = 0;
    int ntiles = 0;

    if (in_range) {
        const float px = s_means[3 * tid + 0], py = s_means[3 * tid + 1], pz = s_means[3 * tid + 2];
        const float v0 = s_view[0], v1 = s_view[1], v2 = s_view[2];
        const float v4 = s_view[4], v5 = s_view[5], v6 = s_view[6];
        const float v8 = s_view[8], v9 = s_view[9], v10 = s_view[10];
        const float v12 = s_view[12], v13 = s_view[13], v14 = s_view[14];

        // view-space z: the depth whose raw bits order the per-tile lists.
        const float pvz = fadd_(fma_(pz, v10, fma_(px, v2, fmul_(py, v6))), v14);
        bool ok = !(pvz <= 0.2f);
        if (!ok && a.prefiltered) {
            printf("Point is filtered although prefiltered is set. This shouldn't happen!");
            __trap();
        }

        float Tux = 0, Tuy = 0, Tuz = 0, Tvx = 0, Tvy = 0, Tvz = 0, Twx = 0, Twy = 0, Twz = 0;
        float nx = 0.f, ny = 0.f, nz = 0.f;
        if (ok) {
            if (a.transMat_precomp != nullptr) {
                const float* t = a.transMat_precomp + (size_t)idx * 9;
                Tux = __ldg(t + 0); Tuy = __ldg(t + 1); Tuz = __ldg(t + 2);
                Tvx = __ldg(t + 3); Tvy = __ldg(t + 4); Tvz = __ldg(t + 5);
                Twx = __ldg(t + 6); Twy = __ldg(t + 7); Twz = __ldg(t + 8);
            } else {
                float4 q = __ldg(reinterpret_cast<const float4*>(a.rotations) + idx);
                float2 sc = __ldg(reinterpret_cast<const float2*>(a.scales) + idx);
                if (a.raw_act) {       // fused activations: exp on the log-scales, F.normalize on the quaternion
                    sc.x = expf(sc.x); sc.y = expf(sc.y);
                    const float n = act_quat_norm(q);
                    q = make_float4(__fdiv_rn(q.x, n), __fdiv_rn(q.y, n), __fdiv_rn(q.z, n), __fdiv_rn(q.w, n));
                }
                // quat_to_rotmat (auxiliary.h:188-210); glm stores (w,x,y,z) in (.x,.y,.z,.w)
                const float n2 = fma_(q.z, q.z, fma_(q.y, q.y, fma_(q.w, q.w, fmul_(q.x, q.x))));
                const float s = rsqrtf(n2);
                const float w = fmul_(q.x, s), x = fmul_(q.y, s), y = fmul_(q.z, s), z = fmul_(q.w, s);
                const float wz = fmul_(w, z), wy = fmul_(w, y), wx = fmul_(w, x);
                const float yy = fmul_(y, y), zz = fmul_(z, z);
                const float xy_p = fma_(x, y, wz), xy_m = fma_(x, y, -wz);
                const float yz_p = fma_(y, z, wx), yz_m = fma_(y, z, -wx);
                const float xz_m = fma_(x, z, -wy), xz_p = fma_(x, z, wy);
                const float yyzz = fadd_(yy, zz), xxzz = fma_(x, x, zz), xxyy = fma_(x, x, yy);
                const float R00 = fadd_(1.0f, -fadd_(yyzz, yyzz));
                const float R01 = fadd_(xy_p, xy_p);
                const float R02 = fadd_(xz_m, xz_m);
                const float R10 = fadd_(xy_m, xy_m);
                const float R11 = fadd_(1.0f, -fadd_(xxzz, xxzz));
                const float R12 = fadd_(yz_p, yz_p);
                const float R20 = fadd_(xz_p, xz_p);
                const float R21 = fadd_(yz_m, yz_m);
                const float R22 = fadd_(1.0f, -fadd_(xxyy, xxyy));
                // R * diag(sx, sy, 1)
                const float a0x = fmul_(R00, sc.x), a0y = fmul_(R01, sc.x), a0z = fmul_(R02, sc.x);
                const float a1x = fmul_(R10, sc.y), a1y = fmul_(R11, sc.y), a1z = fmul_(R12, sc.y);
                // p_view = W p + t
                const float pvx = fadd_(v12, fma_(pz, v8, fma_(px, v0, fmul_(py, v4))));
                const float pvy = fadd_(v13, fma_(pz, v9, fma_(px, v1, fmul_(py, v5))));
                // tn = W R[2]
                const float tnx = fma_(v8, R22, fma_(v0, R20, fmul_(v4, R21)));
                const float tny = fma_(v9, R22, fma_(v1, R20, fmul_(v5, R21)));
                const float tnz = fma_(v10, R22, fma_(v2, R20, fmul_(v6, R21)));
                const float cosv = fma_(-pvz, tnz, fma_(pvy, -tny, -fmul_(pvx, tnx)));
                if (cosv == 0.0f) ok = false;
                // M0 = W (R[0] sx), M1 = W (R[1] sy)
                const float M0x = fma_(v8, a0z, fma_(v0, a0x, fmul_(v4, a0y)));
                const float M0y = fma_(v9, a0z, fma_(v1, a0x, fmul_(v5, a0y)));
                const float M0z = fma_(v10, a0z, fma_(v2, a0x, fmul_(v6, a0y)));
                const float M1x = fma_(v8, a1z, fma_(v0, a1x, fmul_(v4, a1y)));
                const float M1y = fma_(v9, a1z, fma_(v1, a1x, fmul_(v5, a1y)));
                const float M1z = fma_(v10, a1z, fma_(v2, a1x, fmul_(v6, a1y)));
                const float cxh = fmul_((float)a.W, 0.5f), cyh = fmul_((float)a.H, 0.5f);
                Tux = fma_(M0z, cxh, fmul_(M0x, focal_x));
                Tuy = fma_(M1z, cxh, fmul_(M1x, focal_x));
                Tuz = fma_(pvz, cxh, fmul_(pvx, focal_x));
                Tvx = fma_(M0z, cyh, fmul_(M0y, focal_y));
                Tvy = fma_(M1z, cyh, fmul_(M1y, focal_y));
                Tvz = fma_(pvz, cyh, fmul_(pvy, focal_y));
                Twx = M0z; Twy = M1z; Twz = pvz;
                const float mult = cosv > 0.0f ? 1.0f : -1.0f;
                nx = fmul_(tnx, mult); ny = fmul_(tny, mult); nz = fmul_(tnz, mult);
            }
        }

        float cxs = 0.f, cys = 0.f;
        if (ok) {
            // screen-space AABB (forward.cu:133-163)
            const float d = fma_(-Twz, Twz, fma_(Twx, Twx, fmul_(Twy, Twy)));
            if (d == 0.0f) {
                ok = false;
            } else {
                const float inv = __frcp_rn(d);
                float t = fmul_(fmul_(Tux, Twx), inv);
                t = fma_(fmul_(Tuy, Twy), inv, t);
                cxs = fma_(fmul_(Tuz, Twz), -inv, t);
                float b = fmul_(fmul_(Tux, Tux), inv);
                b = fma_(fmul_(Tuy, Tuy), inv, b);
                const float h0x = fma_(cxs, cxs, fma_(fmul_(Tuz, Tuz), inv, -b));
                t = fmul_(fmul_(Tvx, Twx), inv);
                t = fma_(fmul_(Tvy, Twy), inv, t);
                cys = fma_(fmul_(Tvz, Twz), -inv, t);
                b = fmul_(fmul_(Tvx, Tvx), inv);
                b = fma_(fmul_(Tvy, Tvy), inv, b);
                const float h0y = fma_(cys, cys, fma_(fmul_(Tvz, Tvz), inv, -b));
                const float ex = __fsqrt_rn(fmaxf(0.0f, h0x));
                const float ey = __fsqrt_rn(fmaxf(0.0f, h0y));
                const float e = fmaxf(ex, ey);
                // radius = ceil(3 * max(extent, FilterSize)) evaluated in double (forward.cu:239)
                const double rd = ceil(3.0 * fmax((double)e, 0.7071067811865476));
                radius = (int)(float)rd;
                const float rf = (float)radius;
                // tile rectangle (auxiliary.h:64-74)
                int mx0 = (int)fmul_(fadd_(cxs, -rf), 0.0625f);
                int my0 = (int)fmul_(fadd_(cys, -rf), 0.0625f);
                int mx1 = (int)fmul_(fadd_(fadd_(fadd_(cxs, rf), 16.0f), -1.0f), 0.0625f);
                int my1 = (int)fmul_(fadd_(fadd_(fadd_(cys, rf), 16.0f), -1.0f), 0.0625f);
                x0 = min(a.gx, max(0, mx0)); y0 = min(a.gy, max(0, my0));
                x1 = min(a.gx, max(0, mx1)); y1 = min(a.gy, max(0, my1));
                ntiles = (x1 - x0) * (y1 - y0);
                if (ntiles == 0) ok = false;
            }
        }

        if (ok) {
            float rgb[3];
            int clampbits = 0;
            if (use_sh) {
                float dx = fadd_(px, -s_cam[0]), dy = fadd_(py, -s_cam[1]), dz = fadd_(pz, -s_cam[2]);
                const float len = __fsqrt_rn(fma_(dz, dz, fma_(dx, dx, fmul_(dy, dy))));
                dx = __fdiv_rn(dx, len); dy = __fdiv_rn(dy, len); dz = __fdiv_rn(dz, len);
                if (a.stage_sh) {
                    sh_to_rgb(a.D, s_sh + tid * sh_row, dx, dy, dz, rgb);
                } else {
                    sh_to_rgb(a.D, a.shs + (size_t)idx * sh_row, dx, dy, dz, rgb);
                }
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    if (rgb[c] < 0.0f) { clampbits |= (1 << c); }
                    rgb[c] = fmaxf(rgb[c], 0.0f);
                }
            } else {
                rgb[0] = __ldg(a.colors_precomp + (size_t)idx * 3 + 0);
                rgb[1] = __ldg(a.colors_precomp + (size_t)idx * 3 + 1);
                rgb[2] = __ldg(a.colors_precomp + (size_t)idx * 3 + 2);
            }
            const float opac = a.raw_act ? act_sigmoid(__ldg(a.opacities + idx)) : __ldg(a.opacities + idx);
            // Conservative screen-space *octagon* of the pixels where this splat's alpha can reach
            // 1/255 (the blend's skip threshold): alpha >= 1/255  =>  min(rho3d, rho2d) <= tau with
            // tau = 2 ln(255 opacity).  rho2d <= tau is a disc around the AABB centre; rho3d <= tau
            // is the projected ellipse u^2+v^2 <= tau, whose exact extent along any screen direction
            // follows from the reference's own AABB quadratic form with diag(1,1,-1) replaced by
            // diag(tau,tau,-1) -- evaluated here along x, y, x+y and x-y.  Stored as eight fp16
            // offsets from the centre, rounded outwards; used only to skip work per warp, and
            // widened by a margin so that it can never change a result.
            float lo[4], hi[4];   // x, y, x+y, x-y
            if (opac < 0.00392156862745098f) {
                for (int k = 0; k < 4; ++k) { lo[k] = 3.0e38f; hi[k] = -3.0e38f; }   // opacity*G < 1/255 for every G <= 1
            } else {
                const float tau = 2.0f * logf(opac * 255.0f) * 1.0001f + 1.0e-3f;
                const float r2 = sqrtf(0.5f * tau);
                const float qw = tau * (Twx * Twx + Twy * Twy) - Twz * Twz;
                if (qw < 0.0f) {
                    const float iq = 1.0f / qw;
                    // rows whose projective extent we need: Tu, Tv, Tu+Tv, Tu-Tv, TRANSLATED so that the splat's screen
                    // centre is the origin (row - centre * Tw).  Evaluated in absolute pixel coordinates the extent
                    // h^2 = c^2 - (...) cancels catastrophically: c^2 ~ 1e6 at 1024^2 has an fp32 spacing of 0.125,
                    // as large as h^2 itself for small low-opacity splats (measured: 2 wrongly culled pairs per
                    // 262144-splat 1024^2 view).  Around the centre every term is O(h^2).
                    const float dc[4] = {cxs, cys, cxs + cys, cxs - cys};
                    const float ax[4] = {Tux, Tvx, Tux + Tvx, Tux - Tvx};
                    const float ay[4] = {Tuy, Tvy, Tuy + Tvy, Tuy - Tvy};
                    const float az[4] = {Tuz, Tvz, Tuz + Tvz, Tuz - Tvz};
                    const float dr[4] = {r2, r2, 1.41421357f * r2, 1.41421357f * r2};
                    const float mg[4] = {0.0625f, 0.0625f, 0.0884f, 0.0884f};   // 1/16 px (x sqrt2 along the diagonals): the masks are per pixel now
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        const float rx = fmaf(-dc[k], Twx, ax[k]), ry = fmaf(-dc[k], Twy, ay[k]), rz = fmaf(-dc[k], Twz, az[k]);
                        const float c = (tau * (rx * Twx + ry * Twy) - rz * Twz) * iq;          // offset of the ellipse centre from (cxs, cys)
                        const float h = sqrtf(fmaxf(0.0f, c * c - (tau * (rx * rx + ry * ry) - rz * rz) * iq));
                        const float l0 = fminf(-dr[k], c - h), h0 = fmaxf(dr[k], c + h);
                        // margin: 1/16 px + 0.1 % of the width + the rounding of the translated rows (|row| * 2^-22 / |Tw.z|)
                        const float m = mg[k] + 1.0e-3f * (h0 - l0) + 4.0e-7f * (fabsf(az[k]) + fabsf(dc[k] * Twz)) * fabsf(Twz * iq);
                        lo[k] = l0 - m;      // offsets from the centre (x, y, x+y, x-y of it)
                        hi[k] = h0 + m;
                    }
                } else {
                    for (int k = 0; k < 4; ++k) { lo[k] = -3.0e38f; hi[k] = 3.0e38f; }   // tau-ellipse crosses the camera plane: unbounded
                }
            }
            // fp16, rounded outwards (NaNs stay NaN: every comparison against them fails = "not culled")
            __half2 hb[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) hb[k] = __halves2half2(__float2half_rd(lo[k]), __float2half_ru(hi[k]));
            float4 cullq;
            cullq.x = __uint_as_float(*reinterpret_cast<unsigned*>(&hb[0]));
            cullq.y = __uint_as_float(*reinterpret_cast<unsigned*>(&hb[1]));
            cullq.z = __uint_as_float(*reinterpret_cast<unsigned*>(&hb[2]));
            cullq.w = __uint_as_float(*reinterpret_cast<unsigned*>(&hb[3]));
            float4* r = a.rec + (size_t)idx * SRF_REC_QUADS;
            r[0] = make_float4(Tux, Tvx, Tuy, Tvy);     // (Tu.c, Tv.c) interleaved: f32x2 operands of eval_pair()
            r[1] = make_float4(Tuz, Tvz, Twx, Twy);
            r[2] = make_float4(Twz, cxs, cys, opac);
            r[3] = make_float4(nx, ny, nz, pvz);
            r[4] = make_float4(rgb[0], rgb[1], rgb[2], __int_as_float(clampbits));
            r[5] = cullq;
            a.depths[idx] = pvz;
        } else {
            radius = 0; x0 = y0 = x1 = y1 = 0; ntiles = 0;
        }
        a.radii[idx] = radius;
        a.rects[idx] = make_uint2((uint32_t)x0 | ((uint32_t)y0 << 16), (uint32_t)x1 | ((uint32_t)y1 << 16));
    }

    // per-tile instance counting; rectangles larger than a few tiles are spread over the warp
    const int kSerialMax = 8;
    if (ntiles > 0 && ntiles <= kSerialMax) count_tiles_serial(a.tile_count, a.gx, x0, y0, x1, y1);
    unsigned big = __ballot_sync(0xffffffffu, ntiles > kSerialMax);
    const int lane = tid & 31;
    while (big) {
        const int src = __ffs(big) - 1;
        big &= big - 1;
        const int bx0 = __shfl_sync(0xffffffffu, x0, src), by0 = __shfl_sync(0xffffffffu, y0, src);
        const int bx1 = __shfl_sync(0xffffffffu, x1, src), by1 = __shfl_sync(0xffffffffu, y1, src);
        const int w = bx1 - bx0, n = w * (by1 - by0);
        for (int t = lane; t < n; t += 32) {
            const int ty = t / w, tx = t - ty * w;
            atomicAdd(&a.tile_count[(size_t)((by0 + ty) * a.gx + bx0 + tx) * SRF_TILE_CTR_STRIDE], 1u);
        }
    }
}

// reference rasterizer_impl.cu:54-66 + auxiliary.h:160-185: present = (view z > 0.2)
__global__ void __launch_bounds__(256) mark_visible_kernel(int P, const float* __restrict__ means3D,
                                                            const float* __restrict__ viewmatrix,
                                                            uint8_t* __restrict__ present) {
    __shared__ __align__(16) float s_means[256 * 3];
    const int tid = threadIdx.x, base = blockIdx.x * 256, idx = base + tid;
    const int nrows = min(256, P - base);
    stage_rows(s_means, means3D + (size_t)base * 3, nrows * 3, tid, 256);
    __syncthreads();
    if (idx >= P) return;
    const float px = s_means[3 * tid], py = s_means[3 * tid + 1], pz = s_means[3 * tid + 2];
    const float pvz = fadd_(fma_(pz, __ldg(viewmatrix + 10), fma_(px, __ldg(viewmatrix + 2), fmul_(py, __ldg(viewmatrix + 6)))),
                            __ldg(viewmatrix + 14));
    present[idx] = (pvz <= 0.2f) ? 0 : 1;
}

cudaError_t launch_preprocess_fwd(const PreprocessArgs& a, const SceneArgs& s, cudaStream_t stream) {
    if (a.P <= 0 || a.nviews <= 0) return cudaSuccess;
    PreprocessArgs args = a;
    const size_t sh_bytes = (size_t)256 * 3 * a.M * sizeof(float);
    // stage SH rows through shared memory when they fit next to the static buffers
    // (M <= 10 -> 30 KB; larger rows are read directly) and are 16 B aligned
    args.stage_sh = (a.colors_precomp == nullptr && a.M > 0 && sh_bytes <= 32 * 1024 &&
                     (reinterpret_cast<uintptr_t>(a.shs) & 15) == 0 && ((256 * 3 * a.M) % 4) == 0)
                        ? 1 : 0;
    const size_t dyn = args.stage_sh ? sh_bytes : 0;
    const int grid = (a.P + 255) / 256;
    prof_start(K_PREPROCESS_FWD, stream);
    preprocess_fwd_kernel<<<dim3(grid, a.nviews), 256, dyn, stream>>>(args, s);
    prof_stop(K_PREPROCESS_FWD, stream);
    return cudaGetLastError();
}

cudaError_t launch_mark_visible(int P, const float* means3D, const float* viewmatrix, uint8_t* present,
                                cudaStream_t stream) {
    if (P <= 0) return cudaSuccess;
    mark_visible_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, means3D, viewmatrix, present);
    return cudaGetLastError();
}

}  // namespace srf
