// preprocess_bwd.cu -- per-Gaussian backward (K8 + K9 fused).
// Replaces reference backward.cu:599-649 (computeAABB backward), :533-597
// (preprocessCUDA backward), :451-529 (computeTransMat vjp), :20-139 (SH vjp) and
// auxiliary.h:213-257 (quat_to_rotmat_vjp), :125-135 (dnormvdv).
//
// One thread per (Gaussian, scene), summing the scene's views.  Reads the 80 B gradient record accumulated by the blend
// backward plus the forward's GeomRecord, and writes *every* output gradient row --
// zeros for culled Gaussians -- so the host never pre-fills nine zero tensors as the
// reference does (rasterize_points.cu:194-202).  With accumulate=1 the kernel adds into
// the outputs instead (view-sharded accumulation before the NCCL all-reduce).
#include "surfel_common.cuh"
#include "surfel_kernels.h"

namespace srf {

__device__ const float kC0 = 0.28209479177387814f;
__device__ const float kC1 = 0.4886025119029199f;
__device__ const float kC2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f,
                                 -1.0925484305920792f, 0.5462742152960396f};
__device__ const float kC3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f,
                                 0.3731763325901154f,  -0.4570457994644658f, 1.445305721320277f,
                                 -0.5900435899266435f};

struct V3 { float x, y, z; };
__device__ __forceinline__ V3 v3(float x, float y, float z) { V3 r = {x, y, z}; return r; }
__device__ __forceinline__ V3 operator*(float s, V3 a) { return v3(s * a.x, s * a.y, s * a.z); }
__device__ __forceinline__ V3 operator+(V3 a, V3 b) { return v3(a.x + b.x, a.y + b.y, a.z + b.z); }
__device__ __forceinline__ float dot3(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }

template <bool ACC>
__device__ __forceinline__ void put(float* p, float v) {
    if (ACC) *p += v; else *p = v;
}
template <bool ACC>
__device__ __forceinline__ void put4(float* p, float4 v) {   // p must be 16-byte aligned
    float4* q = reinterpret_cast<float4*>(p);
    if (ACC) { const float4 o = *q; v.x += o.x; v.y += o.y; v.z += o.z; v.w += o.w; }
    *q = v;
}
template <bool ACC>
__device__ __forceinline__ void put2(float* p, float2 v) {   // p must be 8-byte aligned
    float2* q = reinterpret_cast<float2*>(p);
    if (ACC) { const float2 o = *q; v.x += o.x; v.y += o.y; }
    *q = v;
}

// One thread per (Gaussian, scene = blockIdx.y); it sums that scene's Vs views.  The scene gives the rows of the inputs
// and outputs, the first view and the field of view.  One scene is S = 1.  Both instantiations fit 2 CTAs per SM
// (128 registers) without spills or a local frame.
template <bool ACC>
__global__ void __launch_bounds__(256, 2) preprocess_bwd_kernel(PreprocessBwdArgs a, const __grid_constant__ SceneArgs s) {
    const int idx = blockIdx.x * 256 + threadIdx.x;
    const int scene = blockIdx.y;
    size_t row = (size_t)scene * a.P;
    int n = a.P;
    if (s.offsets) {
        row = (size_t)s.offsets[scene];
        n = (int)(s.offsets[scene + 1] - s.offsets[scene]);
    }
    const int nviews = s.views_per_scene, v0 = scene * nviews;
    a.radii += (size_t)v0 * a.P;
    a.rec = view_ptr(a.rec, v0, a.geom_stride);
    a.ggrad = view_ptr(a.ggrad, v0, a.ggrad_stride);
    a.viewmatrix += (size_t)v0 * a.cam_stride;
    a.campos += (size_t)v0 * a.cam_stride;
    const float focal_x = s.fov[scene].x, focal_y = s.fov[scene].y;
    const float tan_fovx = s.fov[scene].z, tan_fovy = s.fov[scene].w;
    a.means3D = rows_at(a.means3D, row, 3);
    a.scales = rows_at(a.scales, row, 2);
    a.rotations = rows_at(a.rotations, row, 4);
    a.shs = rows_at(a.shs, row, 3 * a.M);
    a.dL_dmeans3D = rows_at(a.dL_dmeans3D, row, 3);
    a.dL_dmeans2D = rows_at(a.dL_dmeans2D, row, 3);
    a.dL_dsh = rows_at(a.dL_dsh, row, 3 * a.M);
    a.dL_dcolors = rows_at(a.dL_dcolors, row, 3);
    a.dL_dopacity = rows_at(a.dL_dopacity, row, 1);
    a.dL_dscales = rows_at(a.dL_dscales, row, 2);
    a.dL_drotations = rows_at(a.dL_drotations, row, 4);
    a.dL_dtransMat = rows_at(a.dL_dtransMat, row, 9);
    if (idx >= n) return;
    const int M3 = 3 * a.M;

    // sums over the scene's views
    float dmean3D[3] = {0.f, 0.f, 0.f};
    float dmean2D[2] = {0.f, 0.f};
    float dscale[2] = {0.f, 0.f};
    float drot[4] = {0.f, 0.f, 0.f, 0.f};
    float dopac = 0.f;
    float dT[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    float dcol[3] = {0.f, 0.f, 0.f};
    float dsh4[12] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};   // M == 4 rows (LaRa's degree 1)
    const bool sh_fast = (a.M == 4 && a.vec_ok);
    bool sh_rows_written = false;          // general-M path: rows are accumulated in place
    bool any_visible = false;
    float act_opacity = 0.f;

    const bool want_sh = (a.shs != nullptr) && !a.has_precomp_color;
    // per-Gaussian inputs, shared by all views
    const float px = __ldg(a.means3D + 3 * (size_t)idx), py = __ldg(a.means3D + 3 * (size_t)idx + 1),
                pz = __ldg(a.means3D + 3 * (size_t)idx + 2);
    float4 q_in = make_float4(1.f, 0.f, 0.f, 0.f), q = q_in;
    float2 sc = make_float2(1.f, 1.f);
    float qn = 1.0f;
    V3 R0 = v3(1.f, 0.f, 0.f), R1 = v3(0.f, 1.f, 0.f), R2 = v3(0.f, 0.f, 1.f);
    float qw = 1.f, qx = 0.f, qy = 0.f, qz = 0.f;
    if (!a.has_precomp_T) {
        q_in = __ldg(reinterpret_cast<const float4*>(a.rotations) + idx);
        q = q_in;
        sc = __ldg(reinterpret_cast<const float2*>(a.scales) + idx);
        if (a.raw_act) {
            sc.x = expf(sc.x); sc.y = expf(sc.y);
            qn = act_quat_norm(q);
            q = make_float4(__fdiv_rn(q.x, qn), __fdiv_rn(q.y, qn), __fdiv_rn(q.z, qn), __fdiv_rn(q.w, qn));
        }
        const float s = rsqrtf(q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z);
        qw = q.x * s; qx = q.y * s; qy = q.z * s; qz = q.w * s;
        const float w = qw, x = qx, y = qy, z = qz;
        R0 = v3(1.f - 2.f * (y * y + z * z), 2.f * (x * y + w * z), 2.f * (x * z - w * y));
        R1 = v3(2.f * (x * y - w * z), 1.f - 2.f * (x * x + z * z), 2.f * (y * z + w * x));
        R2 = v3(2.f * (x * z + w * y), 2.f * (y * z - w * x), 1.f - 2.f * (x * x + y * y));
    }
    const float* sh = want_sh ? a.shs + (size_t)idx * M3 : nullptr;

    for (int view = 0; view < nviews; ++view) {
        if (!(a.radii[(size_t)view * a.P + idx] > 0)) continue;
        any_visible = true;
        const float4* r = view_ptr(a.rec, view, a.geom_stride) + (size_t)idx * SRF_REC_QUADS;
        const float4 q0 = ldg4(r), q1 = ldg4(r + 1), q2 = ldg4(r + 2), q4 = ldg4(r + 4);
        act_opacity = q2.w;
        const float4* gq = reinterpret_cast<const float4*>(view_ptr(a.ggrad, view, a.ggrad_stride) + (size_t)idx * SRF_GRAD_FLOATS);
        const float4 g0 = ldg4(gq), g1 = ldg4(gq + 1), g2 = ldg4(gq + 2), g3 = ldg4(gq + 3), g4 = ldg4(gq + 4);
        // record slots 0..5 hold (dk.x, -dl.x, dk.y, -dl.y, dk.z, -dl.z); dL_dTu = -dk, dL_dTv = -dl
        float vT[9];
        vT[0] = -g0.x; vT[3] = g0.y; vT[1] = -g0.z; vT[4] = g0.w;
        vT[2] = -g1.x; vT[5] = g1.y; vT[6] = g1.z; vT[7] = g1.w;
        vT[8] = g2.x;
        dopac += g2.y;
        const float dnx = g2.z, dny = g2.w, dnz = g3.x;
        const float vcol[3] = {g3.y, g3.z, g3.w};
        dcol[0] += vcol[0]; dcol[1] += vcol[1]; dcol[2] += vcol[2];
        const float dmx = g4.x, dmy = g4.y;

        const V3 Tu = v3(q0.x, q0.z, q1.x), Tv = v3(q0.y, q0.w, q1.y), Tw = v3(q1.z, q1.w, q2.x);

        // ---- K8: AABB-centre vjp (backward.cu:599-649)
        {
            const float d = Tw.x * Tw.x + Tw.y * Tw.y - Tw.z * Tw.z;
            const float inv = 1.0f / d;
            const V3 f = v3(inv, inv, -inv);
            const V3 fTw = v3(f.x * Tw.x, f.y * Tw.y, f.z * Tw.z);
            const V3 dT0 = dmx * fTw;
            const V3 dT1 = dmy * fTw;
            V3 dT3 = dmx * v3(f.x * Tu.x, f.y * Tu.y, f.z * Tu.z) + dmy * v3(f.x * Tv.x, f.y * Tv.y, f.z * Tv.z);
            const V3 dL_df = dmx * v3(Tu.x * Tw.x, Tu.y * Tw.y, Tu.z * Tw.z) +
                             dmy * v3(Tv.x * Tw.x, Tv.y * Tw.y, Tv.z * Tw.z);
            const float dL_dd = dot3(dL_df, f) * (-1.0f / d);
            const V3 dd_dT3 = v3(2.0f * Tw.x, 2.0f * Tw.y, -2.0f * Tw.z);
            dT3 = dT3 + dL_dd * dd_dT3;
            vT[0] += dT0.x; vT[1] += dT0.y; vT[2] += dT0.z;
            vT[3] += dT1.x; vT[4] += dT1.y; vT[5] += dT1.z;
            vT[6] += dT3.x; vT[7] += dT3.y; vT[8] += dT3.z;
            // the value Python receives as grad_means2D (densification statistic, :645-648)
            const float Wc = focal_x * tan_fovx, Hc = focal_y * tan_fovy;
            dmean2D[0] += vT[2] * Tw.z * Wc;
            dmean2D[1] += vT[5] * Tw.z * Hc;
        }
#pragma unroll
        for (int k = 0; k < 9; ++k) dT[k] += vT[k];

        if (!a.has_precomp_T) {
            // ---- K9: homography vjp (backward.cu:451-529)
            const float* vm = a.viewmatrix + (size_t)view * a.cam_stride;
            const float v0 = __ldg(vm + 0), v1 = __ldg(vm + 1), v2 = __ldg(vm + 2);
            const float v4 = __ldg(vm + 4), v5 = __ldg(vm + 5), v6 = __ldg(vm + 6);
            const float v8 = __ldg(vm + 8), v9 = __ldg(vm + 9), v10 = __ldg(vm + 10);
            const float v12 = __ldg(vm + 12), v13 = __ldg(vm + 13), v14 = __ldg(vm + 14);
            const float fx = focal_x, fy = focal_y;
            const float cx = focal_x * tan_fovx, cy = focal_y * tan_fovy;
            const float w = qw, x = qx, y = qy, z = qz;

            const V3 pview = v3(v0 * px + v4 * py + v8 * pz + v12, v1 * px + v5 * py + v9 * pz + v13,
                                v2 * px + v6 * py + v10 * pz + v14);

            // dL_dM columns: P^T applied to the rows of dL_dT
            V3 dM[3];
#pragma unroll
            for (int j = 0; j < 3; ++j)
                dM[j] = v3(fx * vT[j], fy * vT[3 + j], cx * vT[j] + cy * vT[3 + j] + vT[6 + j]);
            // dL_dRS = W^T dL_dM
            V3 dRS[3];
#pragma unroll
            for (int j = 0; j < 3; ++j)
                dRS[j] = v3(v0 * dM[j].x + v1 * dM[j].y + v2 * dM[j].z, v4 * dM[j].x + v5 * dM[j].y + v6 * dM[j].z,
                            v8 * dM[j].x + v9 * dM[j].y + v10 * dM[j].z);
            dmean3D[0] += dRS[2].x; dmean3D[1] += dRS[2].y; dmean3D[2] += dRS[2].z;

            V3 dtn = v3(v0 * dnx + v1 * dny + v2 * dnz, v4 * dnx + v5 * dny + v6 * dnz, v8 * dnx + v9 * dny + v10 * dnz);
            const V3 tn = v3(v0 * R2.x + v4 * R2.y + v8 * R2.z, v1 * R2.x + v5 * R2.y + v9 * R2.z,
                             v2 * R2.x + v6 * R2.y + v10 * R2.z);
            const float cosv = -(tn.x * pview.x + tn.y * pview.y + tn.z * pview.z);
            const float mult = cosv > 0.f ? 1.f : -1.f;
            dtn = mult * dtn;

            // dL_dR columns
            const V3 dR0 = sc.x * dRS[0], dR1 = sc.y * dRS[1], dR2 = dtn;
            // vR[c][r]: column c, row r
            const float vR00 = dR0.x, vR01 = dR0.y, vR02 = dR0.z;
            const float vR10 = dR1.x, vR11 = dR1.y, vR12 = dR1.z;
            const float vR20 = dR2.x, vR21 = dR2.y, vR22 = dR2.z;
            drot[0] += 2.f * (x * (vR12 - vR21) + y * (vR20 - vR02) + z * (vR01 - vR10));
            drot[1] += 2.f * (-2.f * x * (vR11 + vR22) + y * (vR01 + vR10) + z * (vR02 + vR20) + w * (vR12 - vR21));
            drot[2] += 2.f * (x * (vR01 + vR10) - 2.f * y * (vR00 + vR22) + z * (vR12 + vR21) + w * (vR20 - vR02));
            drot[3] += 2.f * (x * (vR02 + vR20) + y * (vR12 + vR21) - 2.f * z * (vR00 + vR11) + w * (vR01 - vR10));
            dscale[0] += dot3(dRS[0], R0);
            dscale[1] += dot3(dRS[1], R1);
        }

        // ---- SH vjp (backward.cu:20-139).  Runs for every visible Gaussian with SHs, also on the
        // transMat_precomp path (reference backward.cu:596 calls computeColorFromSH whenever shs is set).
        if (want_sh) {
            const int clampbits = __float_as_int(q4.w);
            const float dRGB[3] = {(clampbits & 1) ? 0.f : vcol[0], (clampbits & 2) ? 0.f : vcol[1],
                                   (clampbits & 4) ? 0.f : vcol[2]};
            const float* cp = a.campos + (size_t)view * a.cam_stride;
            const V3 dir_orig = v3(px - __ldg(cp), py - __ldg(cp + 1), pz - __ldg(cp + 2));
            const float len = sqrtf(dir_orig.x * dir_orig.x + dir_orig.y * dir_orig.y + dir_orig.z * dir_orig.z);
            const V3 dir = v3(dir_orig.x / len, dir_orig.y / len, dir_orig.z / len);
            // the basis values (coefficient rows): rows 0..3 for the M = 4 path, every row written as it is
            // computed on the general-M path, where rows accumulate in place (same thread re-reads its own stores)
            float coef[4] = {0.f, 0.f, 0.f, 0.f};
            float* const rows = (a.dL_dsh != nullptr && !sh_fast) ? a.dL_dsh + (size_t)idx * M3 : nullptr;
            const bool add = ACC || sh_rows_written;
            auto row = [&](int k, float ck) {
                if (rows == nullptr || k >= a.M) return;
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    float* o = rows + 3 * k + c;
                    const float val = ck * dRGB[c];
                    *o = add ? (*o + val) : val;
                }
            };
            int nrows = 1;                       // rows set from the basis; the rest up to M get zero coefficients
            const float x = dir.x, y = dir.y, z = dir.z;
            V3 dRGBdx = v3(0.f, 0.f, 0.f), dRGBdy = v3(0.f, 0.f, 0.f), dRGBdz = v3(0.f, 0.f, 0.f);
            auto SH = [&](int k) { return v3(__ldg(sh + 3 * k), __ldg(sh + 3 * k + 1), __ldg(sh + 3 * k + 2)); };
            coef[0] = kC0;
            if (a.D > 0) {
                coef[1] = -kC1 * y; coef[2] = kC1 * z; coef[3] = -kC1 * x;
                nrows = 4;
                dRGBdx = (-kC1) * SH(3);
                dRGBdy = (-kC1) * SH(1);
                dRGBdz = kC1 * SH(2);
                if (a.D > 1) {
                    const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
                    row(4, kC2[0] * xy); row(5, kC2[1] * yz); row(6, kC2[2] * (2.f * zz - xx - yy));
                    row(7, kC2[3] * xz); row(8, kC2[4] * (xx - yy));
                    nrows = 9;
                    dRGBdx = dRGBdx + (kC2[0] * y) * SH(4) + (kC2[2] * 2.f * -x) * SH(6) + (kC2[3] * z) * SH(7) +
                             (kC2[4] * 2.f * x) * SH(8);
                    dRGBdy = dRGBdy + (kC2[0] * x) * SH(4) + (kC2[1] * z) * SH(5) + (kC2[2] * 2.f * -y) * SH(6) +
                             (kC2[4] * 2.f * -y) * SH(8);
                    dRGBdz = dRGBdz + (kC2[1] * y) * SH(5) + (kC2[2] * 2.f * 2.f * z) * SH(6) + (kC2[3] * x) * SH(7);
                    if (a.D > 2) {
                        row(9, kC3[0] * y * (3.f * xx - yy));
                        row(10, kC3[1] * xy * z);
                        row(11, kC3[2] * y * (4.f * zz - xx - yy));
                        row(12, kC3[3] * z * (2.f * zz - 3.f * xx - 3.f * yy));
                        row(13, kC3[4] * x * (4.f * zz - xx - yy));
                        row(14, kC3[5] * z * (xx - yy));
                        row(15, kC3[6] * x * (xx - 3.f * yy));
                        nrows = 16;
                        dRGBdx = dRGBdx + (kC3[0] * 3.f * 2.f * xy) * SH(9) + (kC3[1] * yz) * SH(10) +
                                 (kC3[2] * -2.f * xy) * SH(11) + (kC3[3] * -3.f * 2.f * xz) * SH(12) +
                                 (kC3[4] * (-3.f * xx + 4.f * zz - yy)) * SH(13) + (kC3[5] * 2.f * xz) * SH(14) +
                                 (kC3[6] * 3.f * (xx - yy)) * SH(15);
                        dRGBdy = dRGBdy + (kC3[0] * 3.f * (xx - yy)) * SH(9) + (kC3[1] * xz) * SH(10) +
                                 (kC3[2] * (-3.f * yy + 4.f * zz - xx)) * SH(11) + (kC3[3] * -3.f * 2.f * yz) * SH(12) +
                                 (kC3[4] * -2.f * xy) * SH(13) + (kC3[5] * -2.f * yz) * SH(14) +
                                 (kC3[6] * -3.f * 2.f * xy) * SH(15);
                        dRGBdz = dRGBdz + (kC3[1] * xy) * SH(10) + (kC3[2] * 4.f * 2.f * yz) * SH(11) +
                                 (kC3[3] * 3.f * (2.f * zz - xx - yy)) * SH(12) + (kC3[4] * 4.f * 2.f * xz) * SH(13) +
                                 (kC3[5] * (xx - yy)) * SH(14);
                    }
                }
            }
            const V3 g = v3(dRGB[0], dRGB[1], dRGB[2]);
            const V3 dL_ddir = v3(dot3(dRGBdx, g), dot3(dRGBdy, g), dot3(dRGBdz, g));
            // dnormvdv (auxiliary.h:125-135)
            const V3 v = dir_orig;
            const float sum2 = v.x * v.x + v.y * v.y + v.z * v.z;
            const float invsum32 = 1.0f / sqrtf(sum2 * sum2 * sum2);
            dmean3D[0] += ((sum2 - v.x * v.x) * dL_ddir.x - v.y * v.x * dL_ddir.y - v.z * v.x * dL_ddir.z) * invsum32;
            dmean3D[1] += (-v.x * v.y * dL_ddir.x + (sum2 - v.y * v.y) * dL_ddir.y - v.z * v.y * dL_ddir.z) * invsum32;
            dmean3D[2] += (-v.x * v.z * dL_ddir.x - v.y * v.z * dL_ddir.y + (sum2 - v.z * v.z) * dL_ddir.z) * invsum32;

            if (a.dL_dsh != nullptr) {
                if (sh_fast) {
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        dsh4[3 * k + 0] += coef[k] * dRGB[0];
                        dsh4[3 * k + 1] += coef[k] * dRGB[1];
                        dsh4[3 * k + 2] += coef[k] * dRGB[2];
                    }
                } else {
#pragma unroll
                    for (int k = 0; k < 4; ++k) row(k, coef[k]);
                    for (int k = nrows; k < a.M; ++k) row(k, 0.f);
                    sh_rows_written = true;
                }
            }
        }
    }

    if (a.raw_act && !a.has_precomp_T) {
        // vjps of the fused activations (linear in the summed gradients): d exp = g * y;
        // d normalize = g/n - x (g.x)/n^3 (n > eps); d sigmoid = g (1 - y) y
        dscale[0] *= sc.x; dscale[1] *= sc.y;
        const float gx = drot[0] * q_in.x + drot[1] * q_in.y + drot[2] * q_in.z + drot[3] * q_in.w;
        const float inv = 1.0f / qn;
        if (qn > 1e-12f) {
            const float k = gx * inv * inv * inv;
            drot[0] = drot[0] * inv - q_in.x * k; drot[1] = drot[1] * inv - q_in.y * k;
            drot[2] = drot[2] * inv - q_in.z * k; drot[3] = drot[3] * inv - q_in.w * k;
        } else {
            drot[0] *= inv; drot[1] *= inv; drot[2] *= inv; drot[3] *= inv;
        }
        if (any_visible) dopac = dopac * (1.0f - act_opacity) * act_opacity;
    }

    // ---- dL_dsh rows (zeros when culled / unused coefficients)
    if (a.dL_dsh != nullptr) {
        float* out = a.dL_dsh + (size_t)idx * M3;
        if (sh_fast) {
            // LaRa's case (degree 1): one 48-byte row = three 128-bit stores
            put4<ACC>(out + 0, make_float4(dsh4[0], dsh4[1], dsh4[2], dsh4[3]));
            put4<ACC>(out + 4, make_float4(dsh4[4], dsh4[5], dsh4[6], dsh4[7]));
            put4<ACC>(out + 8, make_float4(dsh4[8], dsh4[9], dsh4[10], dsh4[11]));
        } else if (!sh_rows_written && !ACC) {
            for (int k = 0; k < M3; ++k) out[k] = 0.f;
        }
    }

    put<ACC>(a.dL_dmeans3D + 3 * (size_t)idx + 0, dmean3D[0]);
    put<ACC>(a.dL_dmeans3D + 3 * (size_t)idx + 1, dmean3D[1]);
    put<ACC>(a.dL_dmeans3D + 3 * (size_t)idx + 2, dmean3D[2]);
    if (a.dL_dmeans2D != nullptr) {
        put<ACC>(a.dL_dmeans2D + 3 * (size_t)idx + 0, dmean2D[0]);
        put<ACC>(a.dL_dmeans2D + 3 * (size_t)idx + 1, dmean2D[1]);
        put<ACC>(a.dL_dmeans2D + 3 * (size_t)idx + 2, 0.f);
    }
    put<ACC>(a.dL_dopacity + idx, dopac);
    if (a.vec_ok) {
        put2<ACC>(a.dL_dscales + 2 * (size_t)idx, make_float2(dscale[0], dscale[1]));
        put4<ACC>(a.dL_drotations + 4 * (size_t)idx, make_float4(drot[0], drot[1], drot[2], drot[3]));
    } else {
        put<ACC>(a.dL_dscales + 2 * (size_t)idx + 0, dscale[0]);
        put<ACC>(a.dL_dscales + 2 * (size_t)idx + 1, dscale[1]);
#pragma unroll
        for (int k = 0; k < 4; ++k) put<ACC>(a.dL_drotations + 4 * (size_t)idx + k, drot[k]);
    }
    if (a.dL_dcolors != nullptr) {
#pragma unroll
        for (int k = 0; k < 3; ++k) put<ACC>(a.dL_dcolors + 3 * (size_t)idx + k, dcol[k]);
    }
    if (a.dL_dtransMat != nullptr) {
#pragma unroll
        for (int k = 0; k < 9; ++k) put<ACC>(a.dL_dtransMat + 9 * (size_t)idx + k, dT[k]);
    }
}

cudaError_t launch_preprocess_bwd(const PreprocessBwdArgs& a, const SceneArgs& s, int S, cudaStream_t stream) {
    if (a.P <= 0) return cudaSuccess;
    const dim3 grid((a.P + 255) / 256, S);
    PreprocessBwdArgs args = a;
    // every row is a whole number of 16-byte rotation / 8-byte scale / (M = 4) 48-byte SH rows from the base
    auto al = [](const void* p, uintptr_t n) { return (reinterpret_cast<uintptr_t>(p) & (n - 1)) == 0; };
    args.vec_ok = (al(a.dL_drotations, 16) && al(a.dL_dscales, 8) && (a.dL_dsh == nullptr || al(a.dL_dsh, 16))) ? 1 : 0;
    prof_start(K_PREPROCESS_BWD, stream);
    if (a.accumulate)
        preprocess_bwd_kernel<true><<<grid, 256, 0, stream>>>(args, s);
    else
        preprocess_bwd_kernel<false><<<grid, 256, 0, stream>>>(args, s);
    prof_stop(K_PREPROCESS_BWD, stream);
    return cudaGetLastError();
}

}  // namespace srf
