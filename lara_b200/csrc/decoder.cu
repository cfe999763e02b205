// decoder.cu -- decoder epilogue: MLP output -> the five contiguous Gaussian-parameter tensors K1 consumes
// (SURVEY 8f rank 4).
//
// Restates Decoder.forward_coarse after the MLP (lightning/network.py:261-278) and Network.get_offseted_pt
// (:425-429): the [B, N, K*C] MLP output is viewed as [B, N, K, C] and split into
//   offset[3] | sh[sh_dim] | opacity[1] | scaling[2] | rotation[4]            (C = 10 + sh_dim)
// opacity += opacity_shift, scaling += scaling_shift, offset = sigmoid(offset)*2 - 1,
// centers = group_centers[n] + offset * half_cell_size.
// In torch the split yields strided views into the MLP output: sh and rotation stay non-contiguous and are
// copied by `.contiguous()` inside EVERY rasterizer call (8-16 times per scene), the shifts and the sigmoid
// are five more elementwise kernels, and autograd replays all of it.  One pass here reads the 4*C bytes of a
// Gaussian once (rows staged through shared memory with 128-bit loads) and writes the five tensors in the
// 16/8-byte aligned row layout preprocess_fwd_kernel loads with vector instructions; the backward is the
// mirror image (five gradient tensors in, one [B,N,K*C] gradient out, sigmoid vjp applied in registers).
// The C entries srf_decoder_layout_forward / _backward (include/surfel_rasterizer.h) are defined here.
#include <string.h>

#include "../../include/surfel_rasterizer.h"
#include "surfel_common.cuh"
#include "surfel_kernels.h"

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

template <bool BWD>
__global__ void __launch_bounds__(256) decoder_layout_kernel(DecoderArgs a) {
    extern __shared__ __align__(16) float s_rows[];          // 256 rows x C floats
    const int C = a.C, tid = threadIdx.x;
    const size_t base = (size_t)blockIdx.x * 256;
    const int nrows = (int)min((size_t)256, a.total - base);
    const int nfl = nrows * C;
    const size_t g = base + tid;
    const bool in_range = tid < nrows;
    if (!BWD) {
        // stage the rows of this CTA: contiguous, 16-byte aligned when the tensor is (256*C*4 bytes per CTA)
        const float* src = a.params + base * C;
        if ((reinterpret_cast<uintptr_t>(src) & 15) == 0) {
            const float4* s4 = reinterpret_cast<const float4*>(src);
            float4* d4 = reinterpret_cast<float4*>(s_rows);
            for (int i = tid; i < (nfl >> 2); i += 256) d4[i] = __ldg(s4 + i);
            for (int i = ((nfl >> 2) << 2) + tid; i < nfl; i += 256) s_rows[i] = __ldg(src + i);
        } else {
            for (int i = tid; i < nfl; i += 256) s_rows[i] = __ldg(src + i);
        }
        __syncthreads();
        if (!in_range) return;
        const float* row = s_rows + tid * C;
        // voxel of this Gaussian: rows are ordered [b][n][k]
        const size_t n = (g / a.K) % a.N;
        const float cx = __ldg(a.group_centers + 3 * n), cy = __ldg(a.group_centers + 3 * n + 1), cz = __ldg(a.group_centers + 3 * n + 2);
        // torch evaluates sigmoid(x)*2 - 1.0 as two roundings (mul, then sub); keep that order
        const float ox2 = __fadd_rn(__fmul_rn(dec_sigmoid(row[0]), 2.0f), -1.0f);
        const float oy2 = __fadd_rn(__fmul_rn(dec_sigmoid(row[1]), 2.0f), -1.0f);
        const float oz2 = __fadd_rn(__fmul_rn(dec_sigmoid(row[2]), 2.0f), -1.0f);
        a.centers[3 * g + 0] = __fadd_rn(cx, __fmul_rn(ox2, a.half_cell));
        a.centers[3 * g + 1] = __fadd_rn(cy, __fmul_rn(oy2, a.half_cell));
        a.centers[3 * g + 2] = __fadd_rn(cz, __fmul_rn(oz2, a.half_cell));
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
    } else {
        // gradient rows are assembled in shared memory and written out with coalesced 128-bit stores
        if (in_range) {
            float* row = s_rows + tid * C;
            const float* prow = a.params + g * C;             // raw offsets for the sigmoid vjp
            const int S = a.sh_dim;
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float s = dec_sigmoid(__ldg(prow + c));
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
        __syncthreads();
        float* dst = a.g_params + base * C;
        if ((reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
            float4* d4 = reinterpret_cast<float4*>(dst);
            const float4* s4 = reinterpret_cast<const float4*>(s_rows);
            for (int i = tid; i < (nfl >> 2); i += 256) d4[i] = s4[i];
            for (int i = ((nfl >> 2) << 2) + tid; i < nfl; i += 256) dst[i] = s_rows[i];
        } else {
            for (int i = tid; i < nfl; i += 256) dst[i] = s_rows[i];
        }
    }
}

}  // namespace srf

using srf::cuda_error;
using srf::set_error;

extern "C" int srf_decoder_layout_forward(srf_stream_t stream, size_t B, int N, int K, int sh_dim,
                                          float opacity_shift, float scaling_shift, float half_cell_size,
                                          const float* params, const float* group_centers, float* centers, float* shs,
                                          float* opacity, float* scaling, float* rotation) {
    if (N <= 0 || K <= 0 || sh_dim < 3 || sh_dim % 3 != 0) return set_error("srf_decoder_layout_forward: bad sizes");
    if (!params || !group_centers || !centers || !shs || !opacity || !scaling || !rotation)
        return set_error("srf_decoder_layout_forward: null pointer");
    if ((reinterpret_cast<uintptr_t>(rotation) & 15) || (reinterpret_cast<uintptr_t>(scaling) & 7) ||
        ((sh_dim & 3) == 0 && (reinterpret_cast<uintptr_t>(shs) & 15)))
        return set_error("srf_decoder_layout_forward: outputs must be 16-byte aligned");
    srf::DecoderArgs a;
    memset(&a, 0, sizeof(a));
    a.total = B * (size_t)N * (size_t)K; a.N = N; a.K = K; a.C = 10 + sh_dim; a.sh_dim = sh_dim;
    a.opacity_shift = opacity_shift; a.scaling_shift = scaling_shift; a.half_cell = half_cell_size;
    a.params = params; a.group_centers = group_centers;
    a.centers = centers; a.shs = shs; a.opacity = opacity; a.scaling = scaling; a.rotation = rotation;
    if (a.total == 0) return 0;
    const size_t smem = (size_t)256 * a.C * sizeof(float);
    cudaError_t e = cudaFuncSetAttribute(srf::decoder_layout_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem);
    if (e == cudaSuccess) {
        srf::decoder_layout_kernel<false><<<(unsigned)((a.total + 255) / 256), 256, smem, (cudaStream_t)stream>>>(a);
        e = cudaGetLastError();
    }
    return e == cudaSuccess ? 0 : cuda_error("decoder_layout launch", e);
}

extern "C" int srf_decoder_layout_backward(srf_stream_t stream, size_t B, int N, int K, int sh_dim,
                                           float half_cell_size, const float* params, const float* g_centers,
                                           const float* g_shs, const float* g_opacity, const float* g_scaling,
                                           const float* g_rotation, float* g_params) {
    if (N <= 0 || K <= 0 || sh_dim < 3 || sh_dim % 3 != 0) return set_error("srf_decoder_layout_backward: bad sizes");
    if (!params || !g_params) return set_error("srf_decoder_layout_backward: null pointer");
    srf::DecoderArgs a;
    memset(&a, 0, sizeof(a));
    a.total = B * (size_t)N * (size_t)K; a.N = N; a.K = K; a.C = 10 + sh_dim; a.sh_dim = sh_dim;
    a.half_cell = half_cell_size;
    a.params = params;
    a.g_centers = g_centers; a.g_shs = g_shs; a.g_opacity = g_opacity; a.g_scaling = g_scaling; a.g_rotation = g_rotation;
    a.g_params = g_params;
    if (a.total == 0) return 0;
    const size_t smem = (size_t)256 * a.C * sizeof(float);
    cudaError_t e = cudaFuncSetAttribute(srf::decoder_layout_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem);
    if (e == cudaSuccess) {
        srf::decoder_layout_kernel<true><<<(unsigned)((a.total + 255) / 256), 256, smem, (cudaStream_t)stream>>>(a);
        e = cudaGetLastError();
    }
    return e == cudaSuccess ? 0 : cuda_error("decoder_layout backward launch", e);
}
