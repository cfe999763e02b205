/* surfel_image_encoder.h -- C ABI of the fused parts of LaRa's image encoder (DinoWrapper, lightning/network.py:14-55,
 * 442-445): timm's DINO ViT-B/16 or ViT-S/16 with the patch and position embedding and the residual LayerNorms in
 * CUDA.  The GEMMs and the attention core stay with cuBLAS and torch.  Part of the same library and ABI version as
 * surfel_rasterizer.h; the same conventions hold (device pointers, int status, 0 = ok, srf_last_error() on failure,
 * only enqueues work on `stream`).  Every tensor but the images is contiguous fp32.
 *
 * Sizes: N images of H x W (multiples of 16) give h = H / 16, w = W / 16 and L = h w patch tokens, and 1 + L tokens per
 * image, the cls token first.  C is 384 or 768.  N (1 + L) < 2^31 and L C < 2^31.
 *
 * Patchify: the images [N,3,H,W], element (n, c, y, x) at image[n sn + c sc + y sy + x sx] (strides in elements),
 * normalised as (v - mean[c]) / std[c] with mean = (0.485, 0.456, 0.406), std = (0.229, 0.224, 0.225), are written as
 * the patch matrix [N L, 3 16 16]: row (n, py, px), column (c, ky, kx), the order of the patch conv's weight.
 *
 * Tokens and norm1 of block 0, with the patch GEMM's output patch_out [N L, C] (no bias), pos0 = row 0 of pos_embed and
 * pos_r [L, C] its patch rows resampled to (h, w):
 *   x[n, 0] = cls + pos0,  x[n, 1 + l] = (patch_out[n L + l] + bias) + pos_r[l],  n1 = LN(x)    x, n1 [N, 1 + L, C]
 *
 * Residual add + LayerNorm: as srf_add_layernorm_* (include/surfel_vol_transformer.h) at C in {384, 768}.
 *
 * Final norm: y = a + b, maps[n, c, l] = LN(y)[n, 1 + l, c]: the cls row dropped and the result stored as [N, C, h, w].
 *
 * Every backward uses no float atomics: its sums run in a fixed order, so two identical calls give identical bits.
 */
#ifndef SURFEL_IMAGE_ENCODER_H_
#define SURFEL_IMAGE_ENCODER_H_

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

/* The images are constants: there is no backward. */
int srf_vit_patchify(void* stream, int N, int H, int W, long long sn, long long sc, long long sy, long long sx,
                     const float* image, float* patches);

int srf_vit_tokens_forward(void* stream, int N, int L, int C, float eps, const float* patch_out, const float* bias,
                           const float* cls, const float* pos0, const float* pos_r, const float* gamma,
                           const float* beta, float* x, float* n1);

/* Bytes of the workspace (256-byte aligned, allocated by the caller) of srf_vit_tokens_backward. */
int srf_vit_tokens_workspace_bytes(int N, int L, int C, size_t* bytes);

/* From x, dL_dn1 and the optional dL_dx (NULL = 0), writes dL_dtokens [N, 1 + L, C] (the gradient of x's rows, so
 * dL_dpatch_out is its rows 1 ..), d_bias, d_cls (= the gradient of pos0), d_pos_r [L, C], d_gamma and d_beta.  d_pos_r
 * sums over the images in image order in fp64, d_bias sums those fp64 sums in token order, d_cls sums over the images in
 * image order; d_gamma and d_beta as srf_add_layernorm_backward. */
int srf_vit_tokens_backward(void* stream, int N, int L, int C, float eps, const float* x, const float* gamma,
                            const float* dL_dn1, const float* dL_dx, void* workspace, float* dL_dtokens,
                            float* d_bias, float* d_cls, float* d_pos_r, float* d_gamma, float* d_beta);

/* rows may be 0: then the row arrays may be NULL, nothing is written but d_gamma = d_beta = 0. */
int srf_vit_layernorm_forward(void* stream, int rows, int C, float eps, const float* a, const float* b,
                              const float* gamma, const float* beta, float* y, float* n);

int srf_vit_layernorm_workspace_bytes(int rows, int C, size_t* bytes);

int srf_vit_layernorm_backward(void* stream, int rows, int C, float eps, const float* y, const float* gamma,
                               const float* dL_dn, const float* dL_dy, void* workspace, float* dL_da, float* d_gamma,
                               float* d_beta);

/* a, b [N, 1 + L, C]; y (NULL when no backward follows) [N, 1 + L, C]; maps [N, C, L]. */
int srf_vit_final_norm_forward(void* stream, int N, int L, int C, float eps, const float* a, const float* b,
                               const float* gamma, const float* beta, float* y, float* maps);

int srf_vit_final_norm_workspace_bytes(int N, int L, int C, size_t* bytes);

/* From the forward's y and dL_dmaps [N, C, L], writes dL_da = dL_db [N, 1 + L, C] (zero on the cls rows), d_gamma and
 * d_beta, as srf_add_layernorm_backward. */
int srf_vit_final_norm_backward(void* stream, int N, int L, int C, float eps, const float* y, const float* gamma,
                                const float* dL_dmaps, void* workspace, float* dL_da, float* d_gamma, float* d_beta);

#ifdef __cplusplus
}
#endif
#endif /* SURFEL_IMAGE_ENCODER_H_ */
