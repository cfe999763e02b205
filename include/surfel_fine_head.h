/* surfel_fine_head.h -- C ABI of the fused fine-pass decoder head (next-row: LaRa's Decoder.forward_fine,
 * lightning/network.py:280-284, with the mask gathers and residual of :508-512).  Part of the same library and ABI
 * version as surfel_rasterizer.h; the same conventions hold (device pointers, int status, 0 = ok, srf_last_error() on
 * failure, only enqueues work on `stream`).  All tensors are contiguous fp32 unless noted.
 *
 * Per point p: x = LayerNorm(volume_feat[row(p)]) (eps 1e-5, affine); 8-head cross-attention of the query x over the V
 * keys / values point_feats[:, :, p] (q/k/v projections Wq [D,D], Wk [D,8], Wv [D,8], out_proj Wo [D,D], no biases);
 * sh = W2 relu(W1 y + b1) + b2 (W1 [64,D], W2 [sh_dim,64]).  D is a multiple of 8 up to 128, 1 <= V <= 8, sh_dim is
 * 3, 12, 27 or 48.  Weights are in torch's [out, in] layout.
 *
 * Plain mode (idx = NULL): row(p) = p, volume_feat is [n,D], no residual (Decoder.forward_fine).
 * Gather mode: idx [n] int32, strictly increasing in [0, N*K) (the masked Gaussians); row(p) = idx[p] / K, volume_feat
 * is [N,D], and shs_coarse [N*K, sh_dim] (optional) adds the residual shs_coarse[idx[p]].
 * point_feats is [V,8,n], n fastest (what srf_point_feats_forward writes); sh_out is [n, sh_dim].
 */
#ifndef SURFEL_FINE_HEAD_H_
#define SURFEL_FINE_HEAD_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

int srf_fine_head_forward(void* stream, int n, int V, int D, int sh_dim, int K, int N,
                          const float* volume_feat, const int32_t* idx, const float* point_feats,
                          const float* shs_coarse, const float* norm_w, const float* norm_b,
                          const float* wq, const float* wk, const float* wv, const float* wo,
                          const float* w1, const float* b1, const float* w2, const float* b2,
                          float* sh_out);

/* Bytes of the backward's workspace (256-byte aligned, allocated by the caller) for n points on the current device;
 * gather != 0 for gather mode. */
int srf_fine_head_workspace_bytes(int n, int V, int D, int sh_dim, int gather, size_t* bytes);

/* Recomputes the forward per tile of points and writes (no accumulation, no atomics; two identical calls give
 * identical bits): dL_dvolume_feat ([n,D] plain, [N,D] gather: the sum over the voxel's points, 0 for a voxel without
 * one), dL_dpoint_feats [V,8,n], dL_dshs_coarse (gather mode, optional: dL_dsh on the rows idx, 0 elsewhere) and the
 * ten parameter gradients, summed over the points in a fixed order. */
int srf_fine_head_backward(void* stream, int n, int V, int D, int sh_dim, int K, int N,
                           const float* volume_feat, const int32_t* idx, const float* point_feats,
                           const float* norm_w, const float* norm_b,
                           const float* wq, const float* wk, const float* wv, const float* wo,
                           const float* w1, const float* b1, const float* w2, const float* b2,
                           const float* dL_dsh, void* workspace,
                           float* dL_dvolume_feat, float* dL_dpoint_feats, float* dL_dshs_coarse,
                           float* d_norm_w, float* d_norm_b, float* d_wq, float* d_wk, float* d_wv,
                           float* d_wo, float* d_w1, float* d_b1, float* d_w2, float* d_b2);

#ifdef __cplusplus
}
#endif
#endif /* SURFEL_FINE_HEAD_H_ */
