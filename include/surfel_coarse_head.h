/* surfel_coarse_head.h -- C ABI of the fused coarse-pass decoder head (LaRa's Decoder.forward_coarse,
 * lightning/network.py:259-278, optionally followed by Network.get_offseted_pt, :425-429).  Part of the same library
 * and ABI version as surfel_rasterizer.h; the same conventions hold (device pointers, int status, 0 = ok,
 * srf_last_error() on failure, only enqueues work on `stream`).  All tensors are contiguous fp32.
 *
 * Per row r of feats [rows, D] (rows = B*N, voxel n = r % N):
 *   h1 = relu(W0 x + b0), h2 = relu(W1 h1 + b1), y = W2 h2 + b2         W0, W1 [D,D], W2 [K*C, D], C = 10 + sh_dim
 * and y, viewed as K rows of C, goes through the decoder layout of srf_decoder_layout_forward: the outputs are the
 * five tensors it writes, Gaussian g = r*K + k:
 *   centers_or_offset [rows*K,3], shs [rows*K,sh_dim], opacity [rows*K], scaling [rows*K,2], rotation [rows*K,4].
 * group_centers [N,3] NULL: the first output is offset = sigmoid(y[0:3])*2 - 1 (Decoder.forward_coarse);
 * otherwise it is group_centers[n] + offset * half_cell (get_offseted_pt).
 * D is a multiple of 16 in [16, 128], 1 <= K <= 4, sh_dim is 3, 12, 27 or 48, rows is a multiple of N and
 * rows*K < 2^31.  Weights are in torch's [out, in] layout.  Products run as 3xTF32 tensor-core MMAs (each fp32 operand
 * split into a high and a low TF32 part) with fp32 accumulation.
 */
#ifndef SURFEL_COARSE_HEAD_H_
#define SURFEL_COARSE_HEAD_H_

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

int srf_coarse_head_forward(void* stream, int rows, int N, int D, int K, int sh_dim,
                            float opacity_shift, float scaling_shift, float half_cell,
                            const float* feats, const float* group_centers,
                            const float* w0, const float* b0, const float* w1, const float* b1,
                            const float* w2, const float* b2,
                            float* centers_or_offset, float* shs, float* opacity, float* scaling, float* rotation);

/* Bytes of the backward's workspace (256-byte aligned, allocated by the caller) on the current device. */
int srf_coarse_head_workspace_bytes(int rows, int D, int K, int sh_dim, size_t* bytes);

/* Recomputes the forward per tile of rows and writes (no accumulation, no atomics; two identical calls give identical
 * bits) dL_dfeats [rows, D] and the six parameter gradients, summed over the rows in a fixed order.  A null upstream
 * gradient counts as zero. */
int srf_coarse_head_backward(void* stream, int rows, int N, int D, int K, int sh_dim, float half_cell,
                             const float* feats, const float* group_centers,
                             const float* w0, const float* b0, const float* w1, const float* b1,
                             const float* w2, const float* b2,
                             const float* dL_dcenters_or_offset, const float* dL_dshs, const float* dL_dopacity,
                             const float* dL_dscaling, const float* dL_drotation, void* workspace,
                             float* dL_dfeats, float* d_w0, float* d_b0, float* d_w1, float* d_b1, float* d_w2,
                             float* d_b2);

#ifdef __cplusplus
}
#endif
#endif /* SURFEL_COARSE_HEAD_H_ */
