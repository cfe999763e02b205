/* surfel_feat_volume.h -- C ABI of the fused feature-volume lifting of LaRa's coarse pass (Network.build_feat_vol,
 * lightning/network.py:352-379, the view-embedding concatenation of :451-452 and the block layout VolTransformer.forward
 * builds at :145-150).  Part of the same library and ABI version as surfel_rasterizer.h; the same conventions hold
 * (device pointers, int status, 0 = ok, srf_last_error() on failure, only enqueues work on `stream`).  All tensors are
 * contiguous fp32.
 *
 * For scene b, view v and token (y, x) of the h x w token map (C channels):
 *   d^ = d / max(|d|, 1e-12), m = o x d^ with (o, d) = rays[b,v,y,x,0:3], [3:6]
 *   f  = [rsh_cart_3(d^), rsh_cart_3(m)]                                   32 values
 *   shift, scale = mlp_w silu(f) + mlp_b                                   mlp_w [2C,32] (torch's [out,in]), mlp_b [2C]
 *   y  = LayerNorm(img_feats[b V + v, :, y, x]; eps 1e-6, norm_w, norm_b) (1 + scale) + shift
 * and for voxel g of grid [R^3,3] (flattened i R^2 + j R + k) and view v:
 *   p  = K (R_w2c g + t)  with w2c [B,V,4,4], ixt [B,V,3,3] row-major
 *   u  = (p.xy / p.z + 0.5) / [W_img, H_img] * 2 - 1
 *   sample = grid_sample(y, u; bilinear, zeros, align_corners=False) on the h x w map.
 * A voxel whose sample coordinate is not finite samples 0 and passes no gradient.
 *
 * n_group selects the output layout:
 *   0       drop-in: out [B,V,C,R,R,R] (build_feat_vol's value); E must be 0.
 *   g > 0   condition layout, g | R, bs = R / g: out [B g^3, V bs^3, C+E], row (b g^3 + G) holding voxel (i, j, k) of
 *           block G = (i/bs g + j/bs) g + k/bs at sequence index v bs^3 + (i%bs bs + j%bs) bs + k%bs; its last E
 *           columns are view_embed[v, :] (view_embed [Vmax,E], NULL when E = 0).
 * Sizes: B >= 1, 1 <= V <= 8, C a multiple of 32 up to 1024, h, w >= 1, 1 <= R <= 64, 0 <= E <= 128, V <= Vmax when
 * E > 0, H_img, W_img >= 1.
 */
#ifndef SURFEL_FEAT_VOLUME_H_
#define SURFEL_FEAT_VOLUME_H_

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Bytes of the workspace (256-byte aligned, allocated by the caller) that both the forward and the backward take. */
int srf_feat_volume_workspace_bytes(int B, int V, int C, int h, int w, int R, int E, size_t* bytes);

int srf_feat_volume_forward(void* stream, int B, int V, int C, int h, int w, int R, int E, int Vmax, int H_img,
                            int W_img, int n_group, const float* img_feats, const float* rays, const float* w2c,
                            const float* ixt, const float* grid, const float* norm_w, const float* norm_b,
                            const float* mlp_w, const float* mlp_b, const float* view_embed, void* workspace,
                            float* out);

/* From dL_dout in the layout n_group selects, writes dL_dimg_feats [B V,C,h,w], d_norm_w [C], d_norm_b [C],
 * d_mlp_w [2C,32], d_mlp_b [2C] and, when E > 0, d_view_embed [Vmax,E] (rows >= V are 0).  It recomputes the forward
 * and uses no atomics on floats: the taps are bucketed per token in voxel order and gathered, and the parameter
 * gradients are summed in a fixed order, so two identical calls give identical bits. */
int srf_feat_volume_backward(void* stream, int B, int V, int C, int h, int w, int R, int E, int Vmax, int H_img,
                             int W_img, int n_group, const float* img_feats, const float* rays, const float* w2c,
                             const float* ixt, const float* grid, const float* norm_w, const float* norm_b,
                             const float* mlp_w, const float* mlp_b, const float* dL_dout, void* workspace,
                             float* dL_dimg_feats, float* d_norm_w, float* d_norm_b, float* d_mlp_w, float* d_mlp_b,
                             float* d_view_embed);

#ifdef __cplusplus
}
#endif
#endif /* SURFEL_FEAT_VOLUME_H_ */
