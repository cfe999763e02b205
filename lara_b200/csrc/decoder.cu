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
// The per-Gaussian split is decoder_layout.cuh's.  The C entries srf_decoder_layout_forward / _backward
// (include/surfel_rasterizer.h) are defined here.
#include <string.h>

#include "../../include/surfel_rasterizer.h"
#include "decoder_layout.cuh"
#include "surfel_common.cuh"
#include "surfel_kernels.h"

namespace srf {

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
        layout_store<true>(a, s_rows + tid * C, g);
    } else {
        // gradient rows are assembled in shared memory and written out with coalesced 128-bit stores
        if (in_range) {
            const float* prow = a.params + g * C;             // raw offsets for the sigmoid vjp
            layout_grad_row(a, [&](int c) { return __ldg(prow + c); }, s_rows + tid * C, g);
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
