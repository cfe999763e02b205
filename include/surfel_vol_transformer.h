/* surfel_vol_transformer.h -- C ABI of the fused parts of LaRa's VolTransformer blocks (GroupAttBlock.forward,
 * lightning/network.py:81-102, and the tail of VolTransformer.forward, :152-164): the group-local cross-attention core
 * and the residual add + LayerNorm, both on a channels-last volume [B,R,R,R,C].  Part of the same library and ABI
 * version as surfel_rasterizer.h; the same conventions hold (device pointers, int status, 0 = ok, srf_last_error() on
 * failure, only enqueues work on `stream`).  All tensors are contiguous fp32 and 16-byte aligned.
 *
 * Group cross-attention.  The volume has R^3 voxels per scene, cut into g^3 groups of bs^3 voxels (bs = R / g); voxel
 * (z, y, x) of scene b belongs to group G = b g^3 + ((z/bs) g + y/bs) g + x/bs, the row order of the conditions.  With
 * D = C / H and, for head h, the columns [h D, (h+1) D):
 *   q   [B R^3, C]  queries in channels-last voxel order, row ((b R + z) R + y) R + x
 *   k,v [B g^3, S, C] projected keys and values of each group
 *   o[n, h] = sum_j softmax_j(q[n, h] . k[G, j, h] / sqrt(D)) v[G, j, h]
 * computed in fp32, the softmax subtracting the per-(query, head) maximum.  Sizes: B, g >= 1, R a multiple of g,
 * 1 <= S <= 4096, C a multiple of H, D in {16, 32}, bs^3 D <= 4096, B g^3 < 2^31 / H.
 *
 * Residual add + LayerNorm on `rows` rows of C channels (C a multiple of 32 up to 512):
 *   y = a + b (b may be NULL: then y = a and y may be NULL),  n = (y - mean(y)) / sqrt(var(y) + eps) gamma + beta.
 * rows may be 0: then the row arrays may be NULL, nothing is written but d_gamma = d_beta = 0.
 */
#ifndef SURFEL_VOL_TRANSFORMER_H_
#define SURFEL_VOL_TRANSFORMER_H_

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

int srf_group_attn_forward(void* stream, int B, int R, int g, int S, int C, int H, const float* q, const float* k,
                           const float* v, float* o);

/* From dL_do [B R^3, C] writes dL_dq [B R^3, C], dL_dk and dL_dv [B g^3, S, C].  It recomputes the softmax and uses no
 * atomics: each (group, head) gradient of k and v is summed over the group's bs^3 queries in query order by the CTA
 * that owns it, so two identical calls give identical bits. */
int srf_group_attn_backward(void* stream, int B, int R, int g, int S, int C, int H, const float* q, const float* k,
                            const float* v, const float* dL_do, float* dL_dq, float* dL_dk, float* dL_dv);

int srf_add_layernorm_forward(void* stream, int rows, int C, float eps, const float* a, const float* b,
                              const float* gamma, const float* beta, float* y, float* n);

/* Bytes of the workspace (256-byte aligned, allocated by the caller) of srf_add_layernorm_backward. */
int srf_add_layernorm_workspace_bytes(int rows, int C, size_t* bytes);

/* From y (the forward's y, or a when it had no b), dL_dn and the optional extra gradient dL_dy (NULL = 0), writes
 * dL_da = dL_db = dL_dy + the LayerNorm's vjp, d_gamma and d_beta.  d_gamma and d_beta are per-CTA partials over fixed
 * blocks of 64 rows, summed in CTA order in fp64: two identical calls give identical bits. */
int srf_add_layernorm_backward(void* stream, int rows, int C, float eps, const float* y, const float* gamma,
                               const float* dL_dn, const float* dL_dy, void* workspace, float* dL_da, float* d_gamma,
                               float* d_beta);

#ifdef __cplusplus
}
#endif
#endif /* SURFEL_VOL_TRANSFORMER_H_ */
