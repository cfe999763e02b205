/* surfel_rasterizer.h -- C ABI of the H100-native (sm_90a) 2D-Gaussian-surfel rasterizer.
 *
 * Drop-in boundary for LaRa's third_party/diff-surfel-rasterization ("DSR").  The
 * reference crosses Python -> native at three pybind entry points
 * (DSR/ext.cpp:15-19, DSR/rasterize_points.h:18-68):
 *
 *     rasterize_gaussians            -> srf_forward_preprocess + srf_forward_render
 *     rasterize_gaussians_backward   -> srf_backward
 *     mark_visible                   -> srf_mark_visible
 *
 * which in turn call CudaRasterizer::Rasterizer::{forward,backward,markVisible}
 * (DSR/cuda_rasterizer/rasterizer.h:24-86) with raw pointers.  This header is the
 * raw-pointer level: plain C, device pointers + sizes + a cudaStream_t, int status
 * return (0 = ok; otherwise srf_last_error() describes the failure).  No torch
 * types, no allocation inside the library: the caller owns every buffer (the
 * reference's three growable byte blobs become caller-allocated workspaces whose
 * sizes the srf_*_bytes functions report).  All entry points only enqueue work on
 * `stream`; none of them synchronises.
 *
 * Pointer conventions: every pointer is a CUDA device pointer unless it says "host".
 * Workspaces must be 256-byte aligned.  Matrices follow the reference:
 * `viewmatrix` / `projmatrix` are 16 floats, column-major (i.e. the row-major
 * memory of LaRa's world_view_transform = w2c^T, lightning/utils.py:33-48).
 */
#ifndef SURFEL_RASTERIZER_H_
#define SURFEL_RASTERIZER_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SRF_ABI_VERSION 6

/* cudaStream_t without pulling in cuda_runtime.h */
typedef void* srf_stream_t;

/* Library / ABI identification. */
int srf_abi_version(void);
/* Thread-local description of the last failure (never NULL). */
const char* srf_last_error(void);

/* ---- workspace sizing (host-only, no CUDA calls) --------------------------------
 * Replaces the reference's required<GeometryState/ImageState/BinningState>(n)
 * (DSR/cuda_rasterizer/rasterizer_impl.h:64-70, rasterizer_impl.cu:155-194).
 *   geom  : per-Gaussian state  (GeomRecord[P], depths[P], rects[P])
 *   tile  : per-tile state      (counts, counters, ranges, cursors, big-tile list)
 *   image : per-pixel state     (final_T/dist1/dist2 planes, n_contrib/median planes)
 *   entries / point_list : per-instance scratch and the sorted per-tile index list,
 *                          sized by an instance *capacity* chosen by the caller.
 *                          The point_list workspace also holds, after the list (at
 *                          byte offset 4*capacity rounded up to 256), the forward's
 *                          contribution masks, u32 [8][capacity] (36 B per instance
 *                          of capacity in all); keep it from forward to backward.
 */
int srf_geom_state_bytes(int P, size_t* bytes);
int srf_tile_state_bytes(int H, int W, size_t* bytes);
int srf_image_state_bytes(int H, int W, size_t* bytes);
int srf_binning_bytes(size_t capacity, size_t* entries_bytes, size_t* point_list_bytes);
/* scratch needed by srf_backward: one 80-byte gradient accumulation record per Gaussian */
int srf_backward_scratch_bytes(int P, size_t* bytes);

/* Byte offsets of the sub-arrays inside the workspaces (for tests / tooling that
 * inspect state the way the reference's blobs can be parsed).
 *   geom_off[3]  : rec, depths, rects
 *   tile_off[5]  : tile blocks (one 256 B block per tile: u32 count, u32 cursor, padding),
 *                  counters(4 x u32: num_rendered, n_big, -, -), ranges(uint2), first cursor, big_list
 *   image_off[2] : accum(3 float planes), n_contrib(2 u32 planes)                    */
int srf_state_layout(int P, int H, int W, size_t geom_off[3], size_t tile_off[5], size_t image_off[2]);

/* ---- forward, stage 1: per-Gaussian preprocess + per-tile counting + tile scan ----
 * Replaces FORWARD::preprocess, cub::DeviceScan::InclusiveSum and the blocking
 * cudaMemcpy of num_rendered (rasterizer_impl.cu:241-282).  Writes radii[P] and the
 * geom/tile workspaces; copies num_rendered (uint32) asynchronously to
 * `num_rendered_host` (pinned host memory, may be NULL) -- wait on the stream or an
 * event to read it.  `shs` XOR `colors_precomp`, (`scales`,`rotations`) XOR
 * `transMat_precomp` as in the reference (NULL = not given).  scale_modifier and
 * projmatrix are accepted for signature parity and ignored, exactly like the
 * reference (forward.cu:95; auxiliary.h:173-184 only uses the view matrix).
 * raw_activations != 0 (next-row extension, no reference counterpart): `opacities`, `scales`,
 * `rotations` are LaRa's raw network outputs and the kernel applies the activations of
 * lightning/renderer_2dgs.py:183-188 itself (sigmoid, exp, F.normalize); pass the same flag and
 * the same raw tensors to srf_backward, whose gradients are then wrt the raw parameters. */
int srf_forward_preprocess(srf_stream_t stream, int P, int D, int M,
                           const float* means3D, const float* shs, const float* colors_precomp,
                           const float* opacities, const float* scales, float scale_modifier,
                           const float* rotations, const float* transMat_precomp,
                           const float* viewmatrix, const float* projmatrix, const float* campos,
                           float tan_fovx, float tan_fovy, int image_height, int image_width,
                           int prefiltered,
                           int* radii, void* geom_state, void* tile_state,
                           uint32_t* num_rendered_host, int raw_activations);

/* ---- forward, stage 2: tile-bucket scatter, per-tile depth sort, blend ------------
 * Replaces duplicateWithKeys, cub::DeviceRadixSort::SortPairs, identifyTileRanges and
 * FORWARD::render (rasterizer_impl.cu:290-341).  `capacity` is the number of
 * instances `entries` / `point_list` can hold.  If num_rendered > capacity nothing is
 * written out of bounds, the outputs are unspecified, and the caller must call this
 * function again with larger buffers (stage 1 need not be repeated).
 * Outputs: out_color[3,H,W], out_others[8,H,W] (depth, alpha, normal xyz, median
 * depth, distortion, median weight -- auxiliary.h:25-30). */
int srf_forward_render(srf_stream_t stream, int P, int image_height, int image_width,
                       size_t capacity, const void* geom_state, void* tile_state,
                       void* entries, uint32_t* point_list, void* image_state,
                       const float* background, float* out_color, float* out_others);

/* ---- forward, both stages in one call (= srf_forward_preprocess followed by srf_forward_render): what
 * rasterize_gaussians maps to when the caller sizes the binning buffers optimistically.  If the count copied to
 * num_rendered_host exceeds `capacity`, call srf_forward_render again with larger buffers.  `count_event` (a
 * cudaEvent_t, may be NULL) is recorded between the two stages: waiting on it waits for the count, not for the blend. */
int srf_forward(srf_stream_t stream, int P, int D, int M,
                const float* means3D, const float* shs, const float* colors_precomp,
                const float* opacities, const float* scales, float scale_modifier,
                const float* rotations, const float* transMat_precomp,
                const float* viewmatrix, const float* projmatrix, const float* campos,
                float tan_fovx, float tan_fovy, int image_height, int image_width, int prefiltered,
                const float* background, size_t capacity,
                int* radii, void* geom_state, void* tile_state, void* entries, uint32_t* point_list, void* image_state,
                float* out_color, float* out_others, uint32_t* num_rendered_host, void* count_event, int raw_activations);

/* ---- backward ------------------------------------------------------------------
 * Replaces Rasterizer::backward (rasterizer_impl.cu:346-448): BACKWARD::render,
 * computeAABB backward, BACKWARD::preprocess.  Consumes the state the forward left in
 * geom/tile/image workspaces and point_list.  Output pointers may be NULL when that
 * gradient is not wanted (dL_dmeans3D, dL_dopacity, dL_dscales, dL_drotations are
 * required).  Every non-NULL output row is written (zeros for culled Gaussians), so
 * the outputs need no initialisation -- unless accumulate != 0, in which case the
 * kernel adds into them (used to sum several views before one all-reduce).
 *   dL_dmeans2D[P,3] receives the reference's densification statistic
 *   (backward.cu:645-648), dL_dcolors[P,3] the gradient wrt the (pre-clamp) RGB,
 *   dL_dtransMat[P,9] the gradient wrt the homography (cov3D_precomp slot).
 * raw_activations: the flag given to srf_forward_preprocess; `scales` / `rotations` are then
 * the raw tensors and dL_dopacity / dL_dscales / dL_drotations are wrt the raw parameters
 * (the activated opacity is read back from geom_state).                               */
int srf_backward(srf_stream_t stream, int P, int D, int M, int image_height, int image_width,
                 size_t capacity, const float* background,
                 const float* means3D, const float* shs, int colors_were_precomputed,
                 const float* scales, const float* rotations, int transmat_was_precomputed,
                 const float* viewmatrix, const float* projmatrix, const float* campos,
                 float tan_fovx, float tan_fovy, const int* radii,
                 const void* geom_state, const void* tile_state, const uint32_t* point_list,
                 const void* image_state,
                 const float* dL_dout_color, const float* dL_dout_others,
                 void* scratch, int accumulate,
                 float* dL_dmeans3D, float* dL_dmeans2D, float* dL_dsh, float* dL_dcolors,
                 float* dL_dopacity, float* dL_dscales, float* dL_drotations, float* dL_dtransMat,
                 int raw_activations);

/* ---- fused render_img epilogue (next-row: lightning/renderer_2dgs.py:220-268, :74-89) ---------
 * One pass over the rasterizer's outputs instead of ~12 torch ops (and ~20 autograd ops):
 * image = clamp(color,0,1); acc_map = alpha; rend_normal = viewmatrix[:3,:3] . normal;
 * depth = nan_to_num(D/alpha)*(1-depth_ratio) + depth_ratio*nan_to_num(median depth);
 * depth_normal = alpha * normalize(cross(d/drow, d/dcol of (ray_o + depth*ray_d))) on interior pixels;
 * rend_dist = distortion.  All images planar [C,H,W] fp32; rays [H,W,6] may be NULL (no pseudo
 * normals).  The backward takes the gradients of the six outputs (NULL = zero) and writes
 * dL_dcolor [3,H,W] and dL_dallmap [8,H,W], ready for srf_backward; where the reference's
 * autograd produces NaN (0/0 at alpha == 0) this writes 0.  scratch: [3,H,W] floats.          */
int srf_epilogue_forward(srf_stream_t stream, int image_height, int image_width, float depth_ratio,
                         const float* color, const float* allmap, const float* rays, const float* viewmatrix,
                         float* image, float* depth, float* acc_map, float* rend_normal, float* depth_normal,
                         float* rend_dist);
int srf_epilogue_backward(srf_stream_t stream, int image_height, int image_width, float depth_ratio,
                          const float* color, const float* allmap, const float* rays, const float* viewmatrix,
                          const float* g_image, const float* g_depth, const float* g_acc_map,
                          const float* g_rend_normal, const float* g_depth_normal, const float* g_rend_dist,
                          float* scratch, float* dL_dcolor, float* dL_dallmap);

/* ---- all target views of one scene in one launch set (next-row: the caller loop -----------------
 * lightning/network.py:484-497 renders the 8-16 target views of ONE Gaussian set one call at a
 * time; no reference native counterpart).  Same three stages as above, but every kernel carries a
 * view dimension, so a scene costs one launch set instead of V.
 *
 *   cams          : device array of V camera records, SRF_CAM_FLOATS floats each:
 *                   [0..15] viewmatrix (as `viewmatrix` above), [16..18] campos, [19..21] background
 *                   colour, [22..23] padding.  All views share tan_fovx/tan_fovy and the image size.
 *   workspaces    : V per-view workspaces of identical layout back to back; total sizes from
 *                   srf_views_workspace_bytes: bytes[0..5] = geom, tile, image, entries, point_list,
 *                   backward scratch.  `capacity` is the per-view instance capacity.
 *   radii         : [V,P];  out_color [V,3,H,W];  out_others [V,8,H,W];  upstream gradients alike.
 *   num_rendered_host : pinned host array of V uint32 (may be NULL).
 *   srf_views_backward: the per-Gaussian backward sums the gradients of all V views in registers
 *                   and writes (or, accumulate != 0, adds) every output row once.  dL_dmeans2D (may be
 *                   NULL) receives the sum over views of the densification statistic.             */
#define SRF_CAM_FLOATS 24
#define SRF_CAM_VIEW 0
#define SRF_CAM_CAMPOS 16
#define SRF_CAM_BG 19
int srf_views_workspace_bytes(int V, int P, int H, int W, size_t capacity, size_t bytes[6]);
int srf_views_forward_preprocess(srf_stream_t stream, int V, int P, int D, int M,
                                 const float* means3D, const float* shs, const float* colors_precomp,
                                 const float* opacities, const float* scales, const float* rotations,
                                 const float* transMat_precomp, const float* cams,
                                 float tan_fovx, float tan_fovy, int image_height, int image_width,
                                 int prefiltered, int* radii, void* geom_state, void* tile_state,
                                 uint32_t* num_rendered_host, int raw_activations);
int srf_views_forward_render(srf_stream_t stream, int V, int P, int image_height, int image_width,
                             size_t capacity, const void* geom_state, void* tile_state,
                             void* entries, uint32_t* point_list, void* image_state,
                             const float* cams, float* out_color, float* out_others);
int srf_views_backward(srf_stream_t stream, int V, int P, int D, int M, int image_height, int image_width,
                       size_t capacity, const float* cams,
                       const float* means3D, const float* shs, int colors_were_precomputed,
                       const float* scales, const float* rotations, int transmat_was_precomputed,
                       float tan_fovx, float tan_fovy, const int* radii,
                       const void* geom_state, const void* tile_state, const uint32_t* point_list,
                       const void* image_state,
                       const float* dL_dout_color, const float* dL_dout_others,
                       void* scratch, int accumulate,
                       float* dL_dmeans3D, float* dL_dmeans2D, float* dL_dsh, float* dL_dcolors,
                       float* dL_dopacity, float* dL_dscales, float* dL_drotations, float* dL_dtransMat,
                       int raw_activations);
/* the fused render_img epilogue over V stacked views ([V,C,H,W] images, rays [V,H,W,6], `cams` as above) */
int srf_views_epilogue_forward(srf_stream_t stream, int V, int image_height, int image_width, float depth_ratio,
                               const float* color, const float* allmap, const float* rays, const float* cams,
                               float* image, float* depth, float* acc_map, float* rend_normal, float* depth_normal,
                               float* rend_dist);
int srf_views_epilogue_backward(srf_stream_t stream, int V, int image_height, int image_width, float depth_ratio,
                                const float* color, const float* allmap, const float* rays, const float* cams,
                                const float* g_image, const float* g_depth, const float* g_acc_map,
                                const float* g_rend_normal, const float* g_depth_normal, const float* g_rend_dist,
                                float* scratch, float* dL_dcolor, float* dL_dallmap);

/* ---- fused loss -> dL/d(render_img outputs) producer (next-row: lightning/loss.py:33-60) ------------
 * The rasterizer-facing terms of LaRa's loss over the V stacked views of a scene:
 *   sums[0] = sum (image - target)^2,  sums[1] = sum rend_dist,  sums[2] = sum (1 - <rend_normal, depth_normal>) acc_map
 * (with_reg == 0: only sums[0]; the caller divides by the element counts of the reference's mean()s and applies the
 * weights 1, 1000, 0.2; MS-SSIM stays a library call).  Images planar stacked [V,C,H,W] as the fused epilogue writes
 * them; `target_hwc` is the batch's own channel-last [V,H,W,3].  srf_loss_backward writes the four gradient maps
 * srf_views_epilogue_backward consumes, scaled by the device scalar `upstream` (NULL = 1):
 *   g_image = 2 w_mse (image - target), g_rend_dist = w_dist, g_rend_normal = -w_normal acc depth_normal,
 *   g_depth_normal = -w_normal acc rend_normal   (w_* = weight / element count).                          */
int srf_loss_forward(srf_stream_t stream, int V, int image_height, int image_width, int with_reg,
                     const float* image, const float* target_hwc, const float* rend_normal, const float* depth_normal,
                     const float* acc_map, const float* rend_dist, double* sums);
int srf_loss_backward(srf_stream_t stream, int V, int image_height, int image_width, int with_reg,
                      float w_mse, float w_dist, float w_normal,
                      const float* image, const float* target_hwc, const float* rend_normal, const float* depth_normal,
                      const float* acc_map, const float* upstream,
                      float* g_image, float* g_rend_normal, float* g_depth_normal, float* g_rend_dist);

/* ---- decoder epilogue: MLP output -> Gaussian-parameter tensors (next-row: lightning/network.py:261-278,425-429) ----
 * `params` is the decoder MLP's fp32 output [B, N, K*C], C = 10 + sh_dim, each row = offset[3] | sh[sh_dim] |
 * opacity[1] | scaling[2] | rotation[4].  Writes the five CONTIGUOUS tensors the rasterizer consumes, for all B*N*K
 * Gaussians in [b][n][k] order:  centers = group_centers[n] + (sigmoid(offset)*2 - 1) * half_cell_size,
 * shs (row copy), opacity + opacity_shift, scaling + scaling_shift, rotation (row copy).  The backward takes the
 * five gradients (NULL = zero) and writes g_params [B,N,K*C] (sigmoid vjp applied).                          */
int srf_decoder_layout_forward(srf_stream_t stream, size_t B, int N, int K, int sh_dim,
                               float opacity_shift, float scaling_shift, float half_cell_size,
                               const float* params, const float* group_centers,
                               float* centers, float* shs, float* opacity, float* scaling, float* rotation);
int srf_decoder_layout_backward(srf_stream_t stream, size_t B, int N, int K, int sh_dim, float half_cell_size,
                                const float* params, const float* g_centers, const float* g_shs, const float* g_opacity,
                                const float* g_scaling, const float* g_rotation, float* g_params);

/* ---- fine-pass point features (next-row: Network.get_point_feats, lightning/network.py:390-411, :182-187) ---------
 * Each of the n points is projected into the V source views, p = K (R x + t) with `w2cs` [V,4,4] and `ixts` [V,3,3]
 * row-major, and the 8-channel stack img_ref [V,3,H,W] | image [V,3,H,W] | acc [V,H,W] | depth [V,H,W] (all planar,
 * contiguous) is sampled bilinearly with zero padding at grid_sample's (align_corners=False) coordinates of
 * (p.xy/p.z + 0.5)/[W,H]*2 - 1.  feats [V,8,n]; channel 7 is |sampled depth - p.z|.  A tap whose coordinate is not
 * finite or whose index is outside the image is not used (a point with p.z = 0 samples 0).
 * The backward writes g_points [n,3] (summed over views) and adds the gradients of image, acc and depth into
 * g_image / g_acc / g_depth, which it clears first; img_ref gets no gradient.  Each gradient output may be
 * NULL (not wanted).  n == 0 launches no kernel (the backward still clears the rendering gradients) and
 * points, feats and g_feats may then be NULL.                                                                      */
int srf_point_feats_forward(srf_stream_t stream, int V, int n, int H, int W,
                            const float* points, const float* w2cs, const float* ixts,
                            const float* img_ref, const float* image, const float* acc, const float* depth,
                            float* feats);
int srf_point_feats_backward(srf_stream_t stream, int V, int n, int H, int W,
                             const float* points, const float* w2cs, const float* ixts,
                             const float* img_ref, const float* image, const float* acc, const float* depth,
                             const float* g_feats, float* g_points, float* g_image, float* g_acc, float* g_depth);

/* ---- optional per-kernel timing (no reference counterpart; used by bench.py's roofline) --
 * Between srf_profile_begin() and srf_profile_end() every kernel launch made by this
 * library is bracketed by CUDA events on its launching stream.  srf_profile_end waits for
 * them and returns, per kernel id, the summed device time in ms and the launch count.
 * Kernel ids: 0 preprocess_fwd, 1 tile_scan, 2 scatter, 3 sort_small, 4 sort_big,
 * 5 render_fwd, 6 render_bwd, 7 preprocess_bwd (SRF_NUM_KERNELS entries).  Not thread-safe. */
#define SRF_NUM_KERNELS 8
int srf_profile_begin(void);
int srf_profile_end(float* ms_out, int* launches_out, int n);

/* ---- markVisible (DSR/rasterize_points.cu:242-261, rasterizer_impl.cu:141-153) ----
 * present[i] = 1 iff the view-space z of means3D[i] is > 0.2 (one byte per Gaussian). */
int srf_mark_visible(srf_stream_t stream, int P, const float* means3D,
                     const float* viewmatrix, const float* projmatrix, uint8_t* present);

#ifdef __cplusplus
}
#endif
#endif /* SURFEL_RASTERIZER_H_ */
