// sh_eval.cuh -- SH -> RGB of the forward preprocess, shared by the kernels that write a record's colour word q4
// (preprocess.cu, and subset.cu, which recomputes q4 for new SH coefficients on the coarse pass's geometry).
#pragma once
#include "surfel_common.cuh"

namespace srf {

__device__ const float kSH_C0 = 0.28209479177387814f;
__device__ const float kSH_C1 = 0.4886025119029199f;
__device__ const float kSH_C2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f,
                                    -1.0925484305920792f, 0.5462742152960396f};
__device__ const float kSH_C3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f,
                                    0.3731763325901154f,  -0.4570457994644658f, 1.445305721320277f,
                                    -0.5900435899266435f};

// SH -> RGB (reference forward.cu:20-71), written in the exact fp32 operation order of the
// reference build (sm_100 SASS of computeColorFromSH: every term is fma(coef, sh[k], acc) with
// coef = (C * basis) evaluated as below), so the colour is bit-identical too.
// `sh` points at this Gaussian's M x 3 block, (x,y,z) is the normalised view direction.
__device__ __forceinline__ void sh_to_rgb(int deg, const float* __restrict__ sh, float x, float y, float z,
                                          float rgb[3]) {
    float r0 = fmul_(sh[0], kSH_C0), r1 = fmul_(sh[1], kSH_C0), r2 = fmul_(sh[2], kSH_C0);
#define SRF_SH_ACC(coef, k)                       \
    r0 = fma_((coef), sh[3 * (k) + 0], r0);       \
    r1 = fma_((coef), sh[3 * (k) + 1], r1);       \
    r2 = fma_((coef), sh[3 * (k) + 2], r2);
    if (deg > 0) {
        const float c1 = -fmul_(y, kSH_C1), c2 = fmul_(z, kSH_C1), c3 = -fmul_(x, kSH_C1);
        SRF_SH_ACC(c1, 1) SRF_SH_ACC(c2, 2) SRF_SH_ACC(c3, 3)
        if (deg > 1) {
            const float xy = fmul_(y, x), yz = fmul_(z, y), xz = fmul_(z, x);
            const float xx = fmul_(x, x), yy = fmul_(y, y), zz = fmul_(z, z);
            const float zz2 = fadd_(zz, zz);
            const float c4 = fmul_(xy, kSH_C2[0]);
            const float c5 = fmul_(yz, kSH_C2[1]);
            const float c6 = fmul_(fadd_(fadd_(zz2, -xx), -yy), kSH_C2[2]);
            const float c7 = fmul_(xz, kSH_C2[3]);
            const float xx_yy = fadd_(xx, -yy);
            const float c8 = fmul_(xx_yy, kSH_C2[4]);
            SRF_SH_ACC(c4, 4) SRF_SH_ACC(c5, 5) SRF_SH_ACC(c6, 6) SRF_SH_ACC(c7, 7) SRF_SH_ACC(c8, 8)
            if (deg > 2) {
                const float c9 = fmul_(fmul_(y, kSH_C3[0]), fma_(xx, 3.0f, -yy));
                const float c10 = fmul_(fmul_(xy, kSH_C3[1]), z);
                const float q = fadd_(fma_(zz, 4.0f, -xx), -yy);            // 4zz - xx - yy
                const float c11 = fmul_(fmul_(y, kSH_C3[2]), q);
                const float c12 = fmul_(fmul_(z, kSH_C3[3]), fma_(yy, -3.0f, fma_(xx, -3.0f, zz2)));
                const float c13 = fmul_(q, fmul_(x, kSH_C3[4]));
                const float c14 = fmul_(xx_yy, fmul_(z, kSH_C3[5]));
                const float c15 = fmul_(fmul_(x, kSH_C3[6]), fma_(yy, -3.0f, xx));
                SRF_SH_ACC(c9, 9) SRF_SH_ACC(c10, 10) SRF_SH_ACC(c11, 11) SRF_SH_ACC(c12, 12)
                SRF_SH_ACC(c13, 13) SRF_SH_ACC(c14, 14) SRF_SH_ACC(c15, 15)
            }
        }
    }
#undef SRF_SH_ACC
    rgb[0] = fadd_(r0, 0.5f); rgb[1] = fadd_(r1, 0.5f); rgb[2] = fadd_(r2, 0.5f);
}

}  // namespace srf
