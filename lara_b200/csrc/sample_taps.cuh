// sample_taps.cuh -- the projection, sample-coordinate chain and bilinear taps shared by the point-feature sampler
// (point_feats.cu) and the feature-volume lifting (feat_volume.cu).  Both restate LaRa's projection()
// (lightning/network.py:182-187), its normalisation by the source image size and grid_sample's bilinear taps
// (zeros padding, align_corners=False), with one rounding per torch operation.
#pragma once

namespace srf {

struct PfTaps {
    float tx0, tx1, ty0, ty1;    // ix - floor(ix), floor(ix) + 1 - ix, same for y
    float w[4];                  // nw, ne, sw, se
    int off[4];                  // y * W + x of each tap, -1 = not used
    int xi, yi;                  // the nw tap's pixel (0 on an axis where neither tap column / row is in the image)
    bool any;
};

// p = K (R x + t) with the row-major w2c E [4,4] and intrinsics K [3,3]; returns xy / z in xy, z in z
__device__ __forceinline__ void pf_project(const float* E, const float* K, float x0, float x1, float x2,
                                           float& px, float& py, float& pz, float m[21]) {
#pragma unroll
    for (int r = 0; r < 3; ++r) {
#pragma unroll
        for (int k = 0; k < 4; ++k) m[4 * r + k] = __ldg(E + 4 * r + k);
    }
#pragma unroll
    for (int k = 0; k < 9; ++k) m[12 + k] = __ldg(K + k);
    float q[3];
#pragma unroll
    for (int r = 0; r < 3; ++r)      // points @ R^T, then + t (two torch ops)
        q[r] = __fadd_rn(__fmaf_rn(x2, m[4 * r + 2], __fmaf_rn(x1, m[4 * r + 1], __fmul_rn(x0, m[4 * r]))), m[4 * r + 3]);
    float p[3];
#pragma unroll
    for (int r = 0; r < 3; ++r)      // @ K^T
        p[r] = __fmaf_rn(q[2], m[12 + 3 * r + 2], __fmaf_rn(q[1], m[12 + 3 * r + 1], __fmul_rn(q[0], m[12 + 3 * r])));
    px = p[0]; py = p[1]; pz = p[2];
}

// (xy + 0.5) / image_size * 2 - 1 (network.py:361 and :401), then grid_sample's unnormalisation onto a map of
// map_size pixels; one rounding per torch operation.  The point sampler passes the same size twice.
__device__ __forceinline__ float pf_source_coord(float xy, float image_size, float map_size) {
    const float g = __fadd_rn(__fmul_rn(__fdiv_rn(__fadd_rn(xy, 0.5f), image_size), 2.0f), -1.0f);
    return __fdiv_rn(__fadd_rn(__fmul_rn(__fadd_rn(g, 1.0f), map_size), -1.0f), 2.0f);
}

__device__ __forceinline__ PfTaps pf_taps(float ix, float iy, int W, int H) {
    PfTaps t;
    const float fx = floorf(ix), fy = floorf(iy);
    t.tx1 = __fsub_rn(__fadd_rn(fx, 1.0f), ix); t.tx0 = __fsub_rn(ix, fx);
    t.ty1 = __fsub_rn(__fadd_rn(fy, 1.0f), iy); t.ty0 = __fsub_rn(iy, fy);
    t.w[0] = __fmul_rn(t.tx1, t.ty1);    // nw = (ix_se - ix) * (iy_se - iy)
    t.w[1] = __fmul_rn(t.tx0, t.ty1);    // ne = (ix - ix_sw) * (iy_sw - iy)
    t.w[2] = __fmul_rn(t.tx1, t.ty0);    // sw = (ix_ne - ix) * (iy - iy_ne)
    t.w[3] = __fmul_rn(t.tx0, t.ty0);    // se = (ix - ix_nw) * (iy - iy_nw)
    // comparisons with NaN are false and +-inf fails one side: non-finite coordinates use no tap
    const bool x0 = fx >= 0.0f && fx <= (float)(W - 1), x1 = fx >= -1.0f && fx <= (float)(W - 2);
    const bool y0 = fy >= 0.0f && fy <= (float)(H - 1), y1 = fy >= -1.0f && fy <= (float)(H - 2);
    const int xi = (x0 || x1) ? (int)fx : 0, yi = (y0 || y1) ? (int)fy : 0;
    t.xi = xi; t.yi = yi;
    t.off[0] = (x0 && y0) ? yi * W + xi : -1;
    t.off[1] = (x1 && y0) ? yi * W + xi + 1 : -1;
    t.off[2] = (x0 && y1) ? (yi + 1) * W + xi : -1;
    t.off[3] = (x1 && y1) ? (yi + 1) * W + xi + 1 : -1;
    t.any = (x0 || x1) && (y0 || y1);
    return t;
}

}  // namespace srf
