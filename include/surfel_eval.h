/* surfel_eval.h -- C ABI of LaRa's evaluation on the GPU (evaluation.py:83-141): the novel-view metrics of one scene
 * in one pass, and the turntable video's uint8 frames.  Part of the same library and ABI version as
 * surfel_rasterizer.h; the same conventions hold (device pointers unless "host", int status, 0 = ok, srf_last_error()
 * on failure, only enqueues work on `stream`).  Every image is read through an srf_ms_ssim_addr (surfel_rasterizer.h),
 * so LaRa's concatenated [H, V W, C] tensors, per-view [V,H,W,C] stacks and planar [V,C,H,W] views are read in place.
 */
#ifndef SURFEL_EVAL_H_
#define SURFEL_EVAL_H_

#include <stddef.h>
#include <stdint.h>

#include "surfel_rasterizer.h"

#ifdef __cplusplus
extern "C" {
#endif

#define SRF_EVAL_MAX_THRESHOLDS 8

/* Bytes of srf_eval_metrics' workspace (256-byte aligned, allocated by the caller); independent of the sizes. */
int srf_eval_workspace_bytes(size_t* bytes);

/* The sums behind LaRa's per-scene metrics, over V views of H x W read as one H x (V W) image, in one pass with a
 * fixed-order fp64 reduction (no atomics: two identical calls give identical bits).
 *   image, target : logical [1,3,H,V W] (b = 0); only the columns of views [v0, v1) are read (0 <= v0 <= v1 <= V).
 *   depth, depth_gt, mask : logical [1,1,H,V W] over all V views; mask is one byte per pixel, nonzero = inside.
 *                   depth == NULL skips the depth sums (depth_gt and mask are then not read).
 *   thresholds    : host, n_thresholds <= SRF_EVAL_MAX_THRESHOLDS values; each is rounded to fp32 and compared with
 *                   the fp32 error, as NumPy compares a float32 array with a Python float.
 * out (device, 3 + n_thresholds doubles):
 *   out[0] = sum over the view range and channels of fp32((x - y)^2), each term rounded as torch rounds it;
 *   out[1] = sum over the mask of |fp32(d - d_gt)|;  out[2] = the mask's pixel count;
 *   out[3 + t] = the count of masked pixels with |fp32(d - d_gt)| < fp32(thresholds[t]).                        */
int srf_eval_metrics(srf_stream_t stream, int V, int H, int W, int v0, int v1,
                     const float* image, const srf_ms_ssim_addr* image_addr,
                     const float* target, const srf_ms_ssim_addr* target_addr,
                     const float* depth, const srf_ms_ssim_addr* depth_addr,
                     const float* depth_gt, const srf_ms_ssim_addr* depth_gt_addr,
                     const uint8_t* mask, const srf_ms_ssim_addr* mask_addr,
                     int n_thresholds, const double* thresholds, void* workspace, double* out);

/* uint8 video frames [N,H,W,3] of N rendered frames, each value rounded as LaRa's separate torch / NumPy operations
 * round it (evaluation.py:132-136):
 *   rgb[n,y,x,c] = uint8(rint(fp32(image * 255)))
 *   nrm[n,y,x,c] = uint8(rint(fp32(fp32(fp32(fp32(fp32(normal * alpha) + 1) - alpha) + 1) / 2) * 255)))
 * with rint rounding half to even (np.round).  image and normal are logical [N,3,H,W] (b = frame), alpha is logical
 * [N,1,H,W].  A value outside [0, 255] after rounding saturates to 0 or 255 and NaN gives 0 (LaRa's astype('uint8')
 * is undefined there).  image == NULL skips rgb; normal == NULL skips nrm (alpha is then not read).             */
int srf_video_frames(srf_stream_t stream, int N, int H, int W,
                     const float* image, const srf_ms_ssim_addr* image_addr,
                     const float* normal, const srf_ms_ssim_addr* normal_addr,
                     const float* alpha, const srf_ms_ssim_addr* alpha_addr,
                     uint8_t* rgb, uint8_t* nrm);

#ifdef __cplusplus
}
#endif
#endif /* SURFEL_EVAL_H_ */
