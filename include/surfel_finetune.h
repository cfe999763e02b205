/* surfel_finetune.h -- C ABI of the per-scene refinement of LaRa's predicted Gaussians (configs/infer.yaml's
 * `finetuning` block, lightning/renderer_2dgs.py:142-152 `Renderer.get_params`): one Adam step over the five tensors of
 * the Gaussian record in one launch.  Part of the same library and ABI version as surfel_rasterizer.h; the same
 * conventions hold (device pointers unless "host", int status, 0 = ok, srf_last_error() on failure, only enqueues work
 * on `stream`).
 */
#ifndef SURFEL_FINETUNE_H_
#define SURFEL_FINETUNE_H_

#include <stddef.h>
#include <stdint.h>

#include "surfel_rasterizer.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Parameter groups of get_params, the order of `lr`. */
#define SRF_ADAM_XYZ 0       /* centers [n,3] */
#define SRF_ADAM_F_DC 1      /* shs[:, 0, :] */
#define SRF_ADAM_F_REST 2    /* shs[:, 1:, :] */
#define SRF_ADAM_OPACITY 3   /* opacity [n,1] */
#define SRF_ADAM_SCALING 4   /* scaling [n,2] */
#define SRF_ADAM_ROTATION 5  /* rotation [n,4] */
#define SRF_ADAM_GROUPS 6

/* One step of torch.optim.Adam (single-tensor path, amsgrad off, no weight decay) over
 *   params[0] centers [n,3], params[1] shs [n,M,3], params[2] opacity [n,1], params[3] scaling [n,2],
 *   params[4] rotation [n,4]
 * (host array of 5 device pointers, contiguous fp32, updated in place) with the gradients grads[0..4] (same shapes).
 * `moments` is fp32 [2, n (10 + 3 M)]: exp_avg, then exp_avg_sq, each laid out as the five tensors back to back in the
 * order above; the caller zeroes it before the first step.  lr is a host double [6] in SRF_ADAM_* order.  The bias
 * corrections are the caller's, in fp64 from the step count t: bias_correction1 = 1 - beta1^t,
 * bias_correction2_sqrt = (1 - beta2^t)^0.5.  Per element, rounded as torch's CUDA kernels round:
 *   m = lerp(m, g, fp32(1 - beta1))                         fma(w, g - m, m), or g - (g - m)(1 - w) for w >= 0.5
 *   v = v fp32(beta2);  v = fma(fp32(1 - beta2), g g, v)    mul_ then addcmul_
 *   d = sqrt(v) fp32(1 / bias_correction2_sqrt) + fp32(eps)  torch divides by a host scalar as a product with its
 *                                                           reciprocal, taken in fp64 and rounded once
 *   p = fma(fp32(-(lr / bias_correction1)), m / d, p)       addcdiv_
 * zero_grads = 1 stores 0 to every gradient element after reading it.  M must be 1, 4, 9 or 16 and n >= 0; n = 0
 * then returns 0 without reading a pointer (empty tensors may have null data).  Otherwise a null pointer, beta1 or beta2 outside [0, 1), eps < 0 or bias corrections <= 0 are rejected without a
 * launch. */
int srf_gaussian_adam_step(srf_stream_t stream, int n, int M, float* const params[5], float* const grads[5],
                           float* moments, const double lr[6], double beta1, double beta2, double eps,
                           double bias_correction1, double bias_correction2_sqrt, int zero_grads);

#ifdef __cplusplus
}
#endif
#endif /* SURFEL_FINETUNE_H_ */
