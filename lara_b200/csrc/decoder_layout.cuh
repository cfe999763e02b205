// decoder_layout.cuh -- the decoder epilogue of one Gaussian, shared by decoder.cu (the layout alone) and
// coarse_head.cu (the layout fused behind mlp_coarse).
//
// A row of C = 10 + sh_dim floats is split into
//   offset[3] | sh[sh_dim] | opacity[1] | scaling[2] | rotation[4]
// opacity += opacity_shift, scaling += scaling_shift, offset = sigmoid(offset)*2 - 1 and, with CENTERS,
// centers = group_centers[n] + offset * half_cell (Decoder.forward_coarse and Network.get_offseted_pt,
// lightning/network.py:261-278 and :425-429).  Outputs are written in the 16/8-byte aligned row layout
// preprocess_fwd_kernel loads with vector instructions.
#pragma once

#include <stddef.h>

namespace srf {

struct DecoderArgs {
    size_t total;                // B * N * K Gaussians
    int N, K, C, sh_dim;         // voxels per scene, Gaussians per voxel, floats per row (10 + sh_dim), SH floats
    float opacity_shift, scaling_shift, half_cell;
    const float* params;         // [B,N,K*C] MLP output (fp32)
    const float* group_centers;  // [N,3]
    float* centers; float* shs; float* opacity; float* scaling; float* rotation;     // forward outputs
    const float* g_centers; const float* g_shs; const float* g_opacity; const float* g_scaling; const float* g_rotation;
    float* g_params;             // [B,N,K*C] backward output
};

__device__ __forceinline__ float dec_sigmoid(float x) { return __fdiv_rn(1.0f, 1.0f + expf(-x)); }   // torch's CUDA sigmoid

// Gaussian g (rows ordered [b][n][k]) from its row: the five outputs of a.  Without CENTERS the first output is the
// offset itself (Decoder.forward_coarse), written to a.centers.
template <bool CENTERS>
__device__ __forceinline__ void layout_store(const DecoderArgs& a, const float* row, size_t g) {
    // torch evaluates sigmoid(x)*2 - 1.0 as two roundings (mul, then sub); keep that order
    if (CENTERS) {
        const size_t n = (g / a.K) % a.N;
        const float cx = __ldg(a.group_centers + 3 * n), cy = __ldg(a.group_centers + 3 * n + 1), cz = __ldg(a.group_centers + 3 * n + 2);
        const float ox2 = __fadd_rn(__fmul_rn(dec_sigmoid(row[0]), 2.0f), -1.0f);
        const float oy2 = __fadd_rn(__fmul_rn(dec_sigmoid(row[1]), 2.0f), -1.0f);
        const float oz2 = __fadd_rn(__fmul_rn(dec_sigmoid(row[2]), 2.0f), -1.0f);
        a.centers[3 * g + 0] = __fadd_rn(cx, __fmul_rn(ox2, a.half_cell));
        a.centers[3 * g + 1] = __fadd_rn(cy, __fmul_rn(oy2, a.half_cell));
        a.centers[3 * g + 2] = __fadd_rn(cz, __fmul_rn(oz2, a.half_cell));
    } else {
#pragma unroll
        for (int c = 0; c < 3; ++c) a.centers[3 * g + c] = __fadd_rn(__fmul_rn(dec_sigmoid(row[c]), 2.0f), -1.0f);
    }
    const int S = a.sh_dim;
    float* sh = a.shs + g * S;
    if ((S & 3) == 0) {
        for (int k = 0; k < S; k += 4) *reinterpret_cast<float4*>(sh + k) = make_float4(row[3 + k], row[4 + k], row[5 + k], row[6 + k]);
    } else {
        for (int k = 0; k < S; ++k) sh[k] = row[3 + k];
    }
    a.opacity[g] = __fadd_rn(row[3 + S], a.opacity_shift);
    *reinterpret_cast<float2*>(a.scaling + 2 * g) = make_float2(__fadd_rn(row[4 + S], a.scaling_shift), __fadd_rn(row[5 + S], a.scaling_shift));
    *reinterpret_cast<float4*>(a.rotation + 4 * g) = make_float4(row[6 + S], row[7 + S], row[8 + S], row[9 + S]);
}

// The gradient row of Gaussian g from the five upstream gradients (a null one counts as 0) and the raw offsets
// raw(0..2) (the sigmoid's vjp), each read before row[c] is written, so row may hold them.  The offset form passes
// half_cell = 1.
template <class RawOffset>
__device__ __forceinline__ void layout_grad_row(const DecoderArgs& a, RawOffset raw, float* row, size_t g) {
    const int S = a.sh_dim;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float s = dec_sigmoid(raw(c));
        const float gc = a.g_centers ? a.g_centers[3 * g + c] : 0.0f;
        row[c] = gc * a.half_cell * 2.0f * s * (1.0f - s);
    }
    const float* gsh = a.g_shs ? a.g_shs + g * S : nullptr;
    for (int k = 0; k < S; ++k) row[3 + k] = gsh ? gsh[k] : 0.0f;
    row[3 + S] = a.g_opacity ? a.g_opacity[g] : 0.0f;
    row[4 + S] = a.g_scaling ? a.g_scaling[2 * g] : 0.0f;
    row[5 + S] = a.g_scaling ? a.g_scaling[2 * g + 1] : 0.0f;
#pragma unroll
    for (int c = 0; c < 4; ++c) row[6 + S + c] = a.g_rotation ? a.g_rotation[4 * g + c] : 0.0f;
}

}  // namespace srf
