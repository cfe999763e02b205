/* surfel_batch.h -- C ABI of LaRa's training batch on the GPU (dataLoader/gobjverse.py:40-141, dataLoader/utils.py:21-34):
 * uint8 views in, the composited images, masks, rotated normals and rays out, in LaRa's collated layouts.  Part of the
 * same library and ABI version as surfel_rasterizer.h; the same conventions hold (device pointers, int status, 0 = ok,
 * srf_last_error() on failure, only enqueues work on `stream`).
 */
#ifndef SURFEL_BATCH_H_
#define SURFEL_BATCH_H_

#include <stddef.h>
#include <stdint.h>

#include "surfel_rasterizer.h"

#ifdef __cplusplus
extern "C" {
#endif

/* One pass over B scenes of N views of H x W (H, W >= 16, so that LaRa's 1/16 rays are not empty).
 * Inputs (contiguous):
 *   rgba     uint8 [B,N,H,W,4], 4-byte aligned;  normal uint8 [B,N,H,W,3] or NULL (no normals: nrm_rot and tar_nrm are
 *            then not read or written);  bg f32 [B,N,3];
 *   i2w, i2w_down f32 [B,N,3,3]: LaRa's inv(K)^T c2w[:3,:3]^T at full resolution and with K[:2] scaled by 1/16;
 *   origin   f32 [B,N,3] (c2w[:3,3]);  nrm_rot f32 [B,3,3] (transform_mats[0,:3,:3]).
 * Outputs (contiguous, 4-byte aligned):
 *   tar_rgb  f32 [B,N,H,W,3]  = fp32(fp32(c a) + fp32(bg fp32(1 - a))), c = fp32(c_u8 / 255), a = fp32(a_u8 / 255);
 *   tar_msk  u8  [B,N,H,W]    = a_u8 > 0;
 *   tar_nrm  f32 [B,H,N W,3]  = n R^T with n = fp32(fp32(fp32(n_u8 / 255) 2) - 1): the three products are exact in
 *                               fp64, summed j = 0, 1, 2 in fp64 and rounded once to fp32;
 *   tar_rays f32 [B,N,H,W,6]  = (origin, sum_j XYZ_j i2w[j][i]), XYZ = (x + 0.5, y + 0.5, 1), the sum in fp64 in the
 *                               order j = 0, 1, 2 and rounded once to fp32;
 *   tar_rays_down f32 [B,N,H/16,W/16,6] (integer division) the same with i2w_down.                                 */
int srf_batch_assemble(srf_stream_t stream, int B, int N, int H, int W,
                       const uint8_t* rgba, const uint8_t* normal, const float* bg,
                       const float* i2w, const float* i2w_down, const float* origin, const float* nrm_rot,
                       float* tar_rgb, uint8_t* tar_msk, float* tar_nrm, float* tar_rays, float* tar_rays_down);

#ifdef __cplusplus
}
#endif
#endif /* SURFEL_BATCH_H_ */
