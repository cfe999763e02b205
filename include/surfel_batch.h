/* surfel_batch.h -- C ABI of LaRa's training batch on the GPU (dataLoader/gobjverse.py:40-141, dataLoader/utils.py:21-34):
 * uint8 views in, the composited images, masks, rotated normals and rays out, in LaRa's collated layouts, and the
 * camera records of the batch's target views (lightning/network.py:486-492).  Part of the
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

/* The camera records (SRF_CAM_*) of a batch's n = B*N target views, built on the device from LaRa's `tar_c2w` and
 * `bg_color` as rasterizer.pack_cameras builds them from LaRa's MiniCam (lightning/utils.py:22-48), one thread per view:
 *   c2w  f32 [n,4,4], bg f32 [n,3] (contiguous, 4-byte aligned);  cams f32 [n, SRF_CAM_FLOATS] out:
 *   [SRF_CAM_VIEW, +16)  inverse(c2w)^T in row-major memory, the inverse computed in fp64 (cofactors over the fp64
 *                        determinant) and rounded once to fp32;
 *   [SRF_CAM_CAMPOS, +3) -c2w[:3,3] (MiniCam's sign, kept);  [SRF_CAM_BG, +3) bg;  the rest 0.
 * A pose with a non-finite entry or |det| < 1e-12 gets a record whose view matrix maps every finite point to view depth
 * -1, behind the near plane, with campos 0: the view renders its background only.  (MiniCam's torch.inverse raises on
 * a singular pose instead.)  0 < n <= 65535; the pointers are checked before any launch.                          */
int srf_batch_cameras(srf_stream_t stream, int n, const float* c2w, const float* bg, float* cams);

#ifdef __cplusplus
}
#endif
#endif /* SURFEL_BATCH_H_ */
