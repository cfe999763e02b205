/* surfel_rasterizer.h -- C ABI of the H100-native (sm_90a) 2D-Gaussian-surfel rasterizer.
 *
 * Drop-in boundary for LaRa's third_party/diff-surfel-rasterization ("DSR").  The
 * reference crosses Python -> native at three pybind entry points
 * (DSR/ext.cpp:15-19, DSR/rasterize_points.h:18-68):
 *
 *     rasterize_gaussians            -> srf_scenes_forward   (S = 1, Vs = 1)
 *     rasterize_gaussians_backward   -> srf_scenes_backward  (S = 1, Vs = 1)
 *     mark_visible                   -> srf_mark_visible
 *
 * which in turn call CudaRasterizer::Rasterizer::{forward,backward,markVisible}
 * (DSR/cuda_rasterizer/rasterizer.h:24-86) with raw pointers.  This header is the
 * raw-pointer level: plain C, device pointers + sizes + a cudaStream_t, int status
 * return (0 = ok; otherwise srf_last_error() describes the failure).  No torch
 * types, no allocation inside the library: the caller owns every buffer (the
 * reference's three growable byte blobs become caller-allocated workspaces whose
 * sizes srf_views_workspace_bytes reports).  All entry points only enqueue work on
 * `stream`; none of them synchronises.  A render no gradient flows through
 * (no_grad / inference_mode) passes for_backward = 0 to the forward: the same
 * outputs, bit for bit, without the state the backward needs.
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

#define SRF_ABI_VERSION 13

/* cudaStream_t without pulling in cuda_runtime.h */
typedef void* srf_stream_t;

/* Library / ABI identification. */
int srf_abi_version(void);
/* Thread-local description of the last failure (never NULL). */
const char* srf_last_error(void);

/* ---- camera records ----------------------------------------------------------------
 * Every rasterizer and epilogue entry takes its V cameras as one device array `cams` of V records,
 * SRF_CAM_FLOATS floats each:
 *   [SRF_CAM_VIEW, +16)   viewmatrix (as above), [SRF_CAM_CAMPOS, +3) campos,
 *   [SRF_CAM_BG, +3)      background colour, the rest padding.
 * The views of one call share the image size and the SH degree, and the views of one scene its field of view
 * (below).  One view of the reference's interface is V = 1: one record. */
#define SRF_CAM_FLOATS 24
#define SRF_CAM_VIEW 0
#define SRF_CAM_CAMPOS 16
#define SRF_CAM_BG 19

/* ---- workspace sizing (host-only, no CUDA calls) --------------------------------
 * Replaces the reference's required<GeometryState/ImageState/BinningState>(n)
 * (DSR/cuda_rasterizer/rasterizer_impl.h:64-70, rasterizer_impl.cu:155-194).  The caller allocates V
 * per-view workspaces of identical layout back to back; bytes[0..5] are the totals for V views
 * (each V times the one-view size):
 *   [0] geom       : per-Gaussian state  (GeomRecord[P], depths[P], rects[P])
 *   [1] tile       : per-tile state      (counts, counters, ranges, cursors, big-tile list)
 *   [2] image      : per-pixel state     (final_T/dist1/dist2 planes, n_contrib/median planes)
 *   [3] entries    : per-instance scratch of the binning, sized by the per-view instance
 *   [4] point_list : the sorted per-tile index list,     `capacity` the caller chooses.
 *                    The point_list workspace also holds, after the list (at byte offset
 *                    4*capacity rounded up to 256), the forward's contribution masks,
 *                    u32 [8][capacity] (36 B per instance of capacity in all); keep it from
 *                    forward to backward.
 *   [5] scratch    : srf_scenes_backward's scratch, one 80-byte gradient record per Gaussian and view.
 * for_backward = 0 sizes the workspaces of a forward-only srf_scenes_forward (below): image and scratch are 0
 * (not needed) and point_list is the list alone, 4 B per instance of capacity rounded up to 256 B per view. */
int srf_views_workspace_bytes(int V, int P, int H, int W, size_t capacity, int for_backward, size_t bytes[6]);

/* Byte offsets of the sub-arrays inside one view's workspaces (for tests / tooling that
 * inspect state the way the reference's blobs can be parsed).
 *   geom_off[3]  : rec, depths, rects
 *   tile_off[5]  : tile blocks (one 256 B block per tile: u32 count, u32 cursor, padding),
 *                  counters(4 x u32: num_rendered, n_big, -, -), ranges(uint2), first cursor, big_list
 *   image_off[2] : accum(3 float planes), n_contrib(2 u32 planes)                    */
int srf_state_layout(int P, int H, int W, size_t geom_off[3], size_t tile_off[5], size_t image_off[2]);

/* ---- scenes -------------------------------------------------------------------------------------------------------
 * The forward, subset forward and backward take S scenes of Vs views each, every scene its own Gaussians, laid out as
 * one call of V = S*Vs views: view v (camera record v of `cams` [S*Vs, SRF_CAM_FLOATS], workspace slot v, output image
 * v) belongs to scene v / Vs.  The views of one scene share its field of view, tan_fov[2s] (x) and tan_fov[2s+1] (y), a
 * host array [S,2] of finite positive values; all views share the image size and the SH degree.  One scene of V views
 * (the reference's interface: V = 1) is S = 1, Vs = V.  Each view's outputs and state are bit-identical to those of
 * the same call on its scene alone, and each scene's gradient rows too (with deterministic != 0; otherwise up to the
 * order of float atomics).  0 < S <= SRF_MAX_SCENES, Vs > 0, S*Vs <= 65535.  The per-view entries below
 * (srf_views_forward_render, the workspace and scratch queries) take V = S*Vs.                                        */
#define SRF_MAX_SCENES 128

/* ---- forward ------------------------------------------------------------------------
 * Stage 1 replaces FORWARD::preprocess, cub::DeviceScan::InclusiveSum and the blocking cudaMemcpy of
 * num_rendered (rasterizer_impl.cu:241-282); stage 2 replaces duplicateWithKeys,
 * cub::DeviceRadixSort::SortPairs, identifyTileRanges and FORWARD::render (rasterizer_impl.cu:290-341).
 * srf_scenes_forward runs both stages.  Gaussian inputs are [S,P,...] (means3D [S,P,3], shs [S,P,M,3], ...).
 * Stage 1 writes radii [V,P] and the geom/tile workspaces (sized by srf_views_workspace_bytes(V, P, ...)) and
 * stores each view's instance count (uint32) in `num_rendered_host` (pinned host array of V, may be
 * NULL) asynchronously -- wait on the stream or on `count_event` (a cudaEvent_t, may be NULL), which is
 * recorded between the two stages: waiting on it waits for the counts, not for the blend.
 * `capacity` is the per-view number of instances `entries` / `point_list` can hold.  If a count exceeds
 * it nothing is written out of bounds, the outputs are unspecified, and the caller runs stage 2 again
 * with srf_views_forward_render and larger buffers (stage 1 need not be repeated; stage 2 reads no Gaussian input).
 * Outputs: out_color [V,3,H,W], out_others [V,8,H,W] (depth, alpha, normal xyz, median depth,
 * distortion, median weight -- auxiliary.h:25-30).
 * `shs` XOR `colors_precomp`, (`scales`,`rotations`) XOR `transMat_precomp` as in the reference
 * (NULL = not given).  The reference's scale_modifier and projmatrix are not taken: it ignores them
 * too (forward.cu:95; auxiliary.h:173-184 only uses the view matrix).
 * raw_activations != 0 (next-row extension, no reference counterpart): `opacities`, `scales`,
 * `rotations` are LaRa's raw network outputs and the kernel applies the activations of
 * lightning/renderer_2dgs.py:183-188 itself (sigmoid, exp, F.normalize); pass the same flag and the same
 * raw tensors to the backward, whose gradients are then wrt the raw parameters.
 * for_backward = 0 (forward-only): the forward of a render that no backward will follow.  Same stages, same deferred
 * counts and bit-identical out_color / out_others / radii, but the blend keeps no contribution record and writes no
 * per-pixel image state, so `point_list` holds only the sorted list and `image_state` is not used (may be NULL); size
 * the workspaces with srf_views_workspace_bytes(..., for_backward = 0, ...).  The state it leaves cannot feed
 * srf_scenes_backward.
 * Every argument check of both stages, including null or misaligned workspaces, is made before anything is enqueued. */
int srf_scenes_forward(srf_stream_t stream, int S, int Vs, int P, int D, int M,
                       const float* means3D, const float* shs, const float* colors_precomp,
                       const float* opacities, const float* scales, const float* rotations,
                       const float* transMat_precomp, const float* cams, const float* tan_fov,
                       int image_height, int image_width, int prefiltered,
                       size_t capacity, int* radii, void* geom_state, void* tile_state, void* entries,
                       uint32_t* point_list, void* image_state, float* out_color, float* out_others,
                       uint32_t* num_rendered_host, void* count_event, int raw_activations, int for_backward);
/* stage 2 alone, on the state stage 1 left: the re-run with larger binning buffers; for_backward as given to the
 * forward */
int srf_views_forward_render(srf_stream_t stream, int V, int P, int image_height, int image_width,
                             size_t capacity, const void* geom_state, void* tile_state,
                             void* entries, uint32_t* point_list, void* image_state,
                             const float* cams, float* out_color, float* out_others, int for_backward);

/* ---- subset forward (LaRa's fine pass, lightning/network.py:486-525; DESIGN §3.18) ----------------------------
 * Renders a subset of each scene's Gaussians of a coarse srf_scenes_forward with the same cameras and image size and
 * new SH coefficients, from the coarse forward's state instead of a preprocess and a binning: the records, depths,
 * rects and radii of the subset are the coarse ones of its Gaussians, with the colour word recomputed from the new
 * SH; each tile's list is the coarse list with the other Gaussians removed.  The outputs are bit-identical to
 * srf_scenes_forward on the gathered subsets (means3D[idx], opacities[idx], ...) with the same raw_activations flag,
 * and the state it leaves feeds srf_scenes_backward with P = n_max and the same `offsets` (for_backward != 0) exactly
 * as that forward's would.
 * `idx` [n] is the concatenation of the S strictly ascending index lists, each into its scene's P coarse Gaussians;
 * `offsets` (device int64 [S+1], from 0, non-decreasing, ending at n) splits it: scene s's subset is
 * idx[offsets[s] .. offsets[s+1]).  shs [n,M,3] is concatenated the same way; means3D [S,P,3] are the coarse centers.
 * The entry reads `offsets` back to check it, so it waits for the stream.  offsets == NULL is one scene (S = 1), whose
 * subset is idx[0..n) with n_max == n: nothing is read back and nothing waits for the stream.
 * The subset state is laid out as V views of n_max Gaussians each (n_max >= every scene's count, <= P): radii
 * [V,n_max], workspaces srf_views_workspace_bytes(V, n_max, H, W, capacity, for_backward) (entries are not used);
 * view v holds scene v / Vs's subset in its first slots.  The kept entries stay at the coarse tile's list offsets, so
 * the subset's `point_list` workspace is sized, like the coarse one, by `capacity`, which must equal the coarse
 * forward's capacity (`coarse_capacity`, whose counts must have fit it: re-run the coarse stage 2 first if they did
 * not).  Inputs: the coarse state (radii [V,P], geom / tile workspaces, point_list, and whether the coarse forward was
 * for_backward) and cams as given to the coarse forward.  out_color / out_others as srf_scenes_forward.
 * `workspace`: 256-byte aligned, srf_views_subset_workspace_bytes(S*P).  colors_precomp is not supported (must be
 * NULL).  A scene with an empty subset (n == 0 included) renders the background.  Every argument check is made before
 * anything is enqueued. */
int srf_scenes_subset_forward(srf_stream_t stream, int S, int Vs, int P, int n, int n_max, int D, int M,
                              const int64_t* idx, const int64_t* offsets, const float* means3D, const float* shs,
                              const float* colors_precomp, const float* cams, int image_height, int image_width,
                              size_t capacity, const int* coarse_radii, const void* coarse_geom_state,
                              const void* coarse_tile_state, const uint32_t* coarse_point_list, size_t coarse_capacity,
                              int coarse_for_backward, int* radii, void* geom_state, void* tile_state,
                              uint32_t* point_list, void* image_state, float* out_color, float* out_others,
                              void* workspace, int for_backward);
int srf_views_subset_workspace_bytes(int P, size_t* bytes);

/* ---- backward ------------------------------------------------------------------
 * Replaces Rasterizer::backward (rasterizer_impl.cu:346-448): BACKWARD::render,
 * computeAABB backward, BACKWARD::preprocess.  Consumes the state the forward left in the
 * geom/tile/image workspaces and point_list; upstream gradients dL_dout_color [V,3,H,W],
 * dL_dout_others [V,8,H,W].  `P` is the number of Gaussians per view slot and `offsets` says where each scene's
 * inputs and gradient rows are:
 *   NULL for srf_scenes_forward's state: scene s's rows are [s*P, (s+1)*P) of [S,P,...] arrays;
 *   the subset forward's offsets, with P = n_max: scene s's rows are [offsets[s], offsets[s+1]) of the concatenated
 *   [n,...] arrays (the gathered subset inputs).  The entry reads them back to check them (waits for the stream).
 * The per-Gaussian backward sums the gradients of a scene's Vs views in registers, in view order, and writes every
 * output row once (zeros for culled Gaussians), so the outputs need
 * no initialisation -- unless accumulate != 0, in which case the kernel adds into them (used to
 * sum several calls before one all-reduce).  Output pointers may be NULL when that gradient is
 * not wanted (dL_dmeans3D, dL_dopacity, dL_dscales, dL_drotations are required).
 *   dL_dmeans2D[P,3] receives the sum over views of the reference's densification statistic
 *   (backward.cu:645-648), dL_dcolors[P,3] the gradient wrt the (pre-clamp) RGB,
 *   dL_dtransMat[P,9] the gradient wrt the homography (cov3D_precomp slot).
 * raw_activations: the flag given to the forward; `scales` / `rotations` are then the raw
 * tensors and dL_dopacity / dL_dscales / dL_drotations are wrt the raw parameters (the
 * activated opacity is read back from geom_state).
 * deterministic != 0 (also for V = 1): same results, but the blend backward's per-lane partial sums are added in
 * 64-bit fixed point (two passes of the blend backward: per-channel bounds, then the sums), so two calls on the same
 * inputs give bit-identical gradients.  `scratch` (256-byte aligned) is then
 * srf_views_backward_deterministic_scratch_bytes(V, P) bytes, and the call waits for the stream before it returns: if a
 * partial sum is not finite or beyond the fixed-point range it returns an error instead of a gradient (the output
 * arrays then hold no meaningful values, and with accumulate != 0 they have been added to).                          */
int srf_scenes_backward(srf_stream_t stream, int S, int Vs, int P, const int64_t* offsets, int D, int M,
                        int image_height, int image_width, size_t capacity, const float* cams,
                        const float* means3D, const float* shs, int colors_were_precomputed,
                        const float* scales, const float* rotations, int transmat_was_precomputed,
                        const float* tan_fov, const int* radii,
                        const void* geom_state, const void* tile_state, const uint32_t* point_list,
                        const void* image_state,
                        const float* dL_dout_color, const float* dL_dout_others,
                        void* scratch, int accumulate,
                        float* dL_dmeans3D, float* dL_dmeans2D, float* dL_dsh, float* dL_dcolors,
                        float* dL_dopacity, float* dL_dscales, float* dL_drotations, float* dL_dtransMat,
                        int raw_activations, int deterministic);
int srf_views_backward_deterministic_scratch_bytes(int V, int P, size_t* bytes);

/* ---- fused render_img epilogue (next-row: lightning/renderer_2dgs.py:220-268, :74-89) ---------
 * One pass over the rasterizer's outputs of V stacked views instead of ~12 torch ops (and ~20 autograd
 * ops) per view: image = clamp(color,0,1); acc_map = alpha; rend_normal = viewmatrix[:3,:3] . normal;
 * depth = nan_to_num(D/alpha)*(1-depth_ratio) + depth_ratio*nan_to_num(median depth);
 * depth_normal = alpha * normalize(cross(d/drow, d/dcol of (ray_o + depth*ray_d))) on interior pixels;
 * rend_dist = distortion.  All images planar stacked [V,C,H,W] fp32; rays [V,H,W,6] may be NULL (no
 * pseudo normals).  Of each camera record the epilogue reads only the view matrix, floats
 * [SRF_CAM_VIEW, SRF_CAM_VIEW + 16): for V = 1 a bare 16-float view matrix is a valid `cams`.
 * The backward takes the gradients of the six outputs (NULL = zero) and writes dL_dcolor [V,3,H,W] and
 * dL_dallmap [V,8,H,W], ready for srf_scenes_backward; where the reference's autograd produces NaN
 * (0/0 at alpha == 0) this writes 0.  scratch: [V,3,H,W] floats.                                      */
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
 * weights 1, 1000, 0.2; the MS-SSIM term is srf_ms_ssim_* below).  Images planar stacked [V,C,H,W] as the fused epilogue writes
 * them; `target_hwc` is the batch's own channel-last [V,H,W,3].  srf_loss_backward writes the four gradient maps
 * srf_views_epilogue_backward consumes, scaled by the device scalar `upstream` (NULL = 1):
 *   g_image = 2 w_mse (image - target), g_rend_dist = w_dist, g_rend_normal = -w_normal acc depth_normal,
 *   g_depth_normal = -w_normal acc rend_normal   (w_* = weight / element count).
 * srf_loss_forward's `workspace`: NULL sums with atomics; otherwise (deterministic) the per-block partial sums go to
 * `workspace` (8-byte aligned, srf_loss_deterministic_workspace_bytes) and are reduced in a fixed order, on a grid
 * that does not depend on the device.                                                                       */
int srf_loss_forward(srf_stream_t stream, int V, int image_height, int image_width, int with_reg,
                     const float* image, const float* target_hwc, const float* rend_normal, const float* depth_normal,
                     const float* acc_map, const float* rend_dist, double* sums, void* workspace);
int srf_loss_deterministic_workspace_bytes(int V, int image_height, int image_width, size_t* bytes);
int srf_loss_backward(srf_stream_t stream, int V, int image_height, int image_width, int with_reg,
                      float w_mse, float w_dist, float w_normal,
                      const float* image, const float* target_hwc, const float* rend_normal, const float* depth_normal,
                      const float* acc_map, const float* upstream,
                      float* g_image, float* g_rend_normal, float* g_depth_normal, float* g_rend_dist);
/* Both passes of LaRa's step in one launch per direction (DESIGN §3.27): V may be the B*V views of a batch
 * ([B*V,3,H,W] planar buffers of the batch render), and `image_fine` (NULL: none) is the fine pass, read against the
 * same target.  srf_loss_passes_forward then writes sums[3] = sum (image_fine - target)^2 as well (sums [4]; [3]
 * without image_fine), each target pixel read once; the fine pass has no regulariser terms, as in LaRa.  The
 * backward writes g_image_fine = 2 w_mse (image_fine - target) with the same w_mse and upstream; image_fine and
 * g_image_fine are both given or both NULL.  Buffers must be 4-byte aligned (sums and workspace 8-byte).  With
 * image_fine NULL these are srf_loss_forward / _backward (which run them), bit for bit; the deterministic workspace
 * (srf_loss_passes_deterministic_workspace_bytes, with_fine != 0 for image_fine) holds one partial per term and block,
 * so with a fine image each of the first three sums has the bits of the call without it.                     */
int srf_loss_passes_forward(srf_stream_t stream, int V, int image_height, int image_width, int with_reg,
                            const float* image, const float* image_fine, const float* target_hwc,
                            const float* rend_normal, const float* depth_normal, const float* acc_map,
                            const float* rend_dist, double* sums, void* workspace);
int srf_loss_passes_deterministic_workspace_bytes(int V, int image_height, int image_width, int with_fine,
                                                  size_t* bytes);
int srf_loss_passes_backward(srf_stream_t stream, int V, int image_height, int image_width, int with_reg,
                             float w_mse, float w_dist, float w_normal,
                             const float* image, const float* image_fine, const float* target_hwc,
                             const float* rend_normal, const float* depth_normal, const float* acc_map,
                             const float* upstream, float* g_image, float* g_image_fine, float* g_rend_normal,
                             float* g_depth_normal, float* g_rend_dist);

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
 * points, feats and g_feats may then be NULL.
 * The backward's `workspace`: NULL adds with atomics; otherwise (deterministic) the rendering gradients are summed in
 * 64-bit fixed point in `workspace` (256-byte aligned, srf_point_feats_deterministic_workspace_bytes) and then written,
 * so two calls give identical bits; the call then waits for the stream and returns an error instead of a gradient if
 * g_feats holds a non-finite value.                                                                                 */
int srf_point_feats_forward(srf_stream_t stream, int V, int n, int H, int W,
                            const float* points, const float* w2cs, const float* ixts,
                            const float* img_ref, const float* image, const float* acc, const float* depth,
                            float* feats);
int srf_point_feats_backward(srf_stream_t stream, int V, int n, int H, int W,
                             const float* points, const float* w2cs, const float* ixts,
                             const float* img_ref, const float* image, const float* acc, const float* depth,
                             const float* g_feats, float* g_points, float* g_image, float* g_acc, float* g_depth,
                             void* workspace);
int srf_point_feats_deterministic_workspace_bytes(int V, int H, int W, size_t* bytes);
/* The same over the S scenes of a batch in one launch per direction (DESIGN §3.26).  Scene s's points are
 * [offsets[s], offsets[s+1]) of the n points (`offsets`: HOST int64 [S+1], from 0, non-decreasing, ending at n, at most
 * P per scene; checked without waiting for the stream).  Point i's centre is row rows[i] of centers [S*P,3] (`rows`
 * [n] int32, the global row b*P + index; NULL: row i, with n <= S*P); a row outside [0, S*P) is never read: that
 * point's features are 0 and it gets no gradient.  Scene s's Vs source views use cameras w2cs / ixts [S*Vs,...] at
 * s*Vs + v, img_ref [S,Vs,3,H,W] at the element strides of `img_ref_addr` (host; any layout, e.g. a channel-last view),
 * and the renderings image [S*Vr,3,H,W], acc and depth [S*Vr,H,W] at view s*Vr + v, Vr >= Vs (a batch render's own
 * planar outputs).  feats [Vs,8,n] as above.  The backward writes g_centers [S*P,3] (the points' rows: their sum over
 * the views; every other row 0; no atomics) and the rendering gradients in the full [S*Vr,...] planes (0 for views
 * v >= Vs).  Per point, the float operations are those of the one-scene call; with a `workspace`
 * (srf_point_feats_scenes_deterministic_workspace_bytes(S, Vs, H, W)) each scene's rendering gradients are summed under
 * its own fixed-point scale, so they equal the one-scene call's on that scene bit for bit.  srf_point_feats_forward /
 * _backward are this with S = 1, rows NULL, Vr = V and a contiguous img_ref.  0 < S <= SRF_MAX_SCENES, S*P < 2^31. */
typedef struct srf_pf_image_addr { int64_t ss, sv, sc, sy, sx; } srf_pf_image_addr;
int srf_point_feats_scenes_forward(srf_stream_t stream, int S, int Vs, int Vr, int P, int n, int H, int W,
                                   const int64_t* offsets, const int32_t* rows, const float* centers,
                                   const float* w2cs, const float* ixts, const float* img_ref,
                                   const srf_pf_image_addr* img_ref_addr, const float* image, const float* acc,
                                   const float* depth, float* feats);
int srf_point_feats_scenes_backward(srf_stream_t stream, int S, int Vs, int Vr, int P, int n, int H, int W,
                                    const int64_t* offsets, const int32_t* rows, const float* centers,
                                    const float* w2cs, const float* ixts, const float* img_ref,
                                    const srf_pf_image_addr* img_ref_addr, const float* image, const float* acc,
                                    const float* depth, const float* g_feats, float* g_centers, float* g_image,
                                    float* g_acc, float* g_depth, void* workspace);
int srf_point_feats_scenes_deterministic_workspace_bytes(int S, int Vs, int H, int W, size_t* bytes);

/* ---- fused MS-SSIM (next-row: lightning/loss.py:44-47, pytorch-msssim 1.0.0 MS_SSIM, channel = C) -------------
 * The 5-level MS-SSIM of X (rendering) and Y (target), logical images B x C x H x W, with the library's valid 11-tap
 * Gaussian window (sigma 1.5), C1 = (0.01 data_range)^2, C2 = (0.03 data_range)^2, 2x2 average pooling with padding
 * (H % 2, W % 2) between levels and weights (0.0448, 0.2856, 0.3001, 0.2363, 0.1333).  min(H, W) must be > 160.
 * Each image is read through an srf_ms_ssim_addr (host pointer): element (b, c, y, x) lies at element offset
 *   b sb + c sc + y sy + (x / wv) sv + (x % wv) sx
 * so a strided NCHW tensor is wv = W (sv unused) and V planar [V,C,H,w] views side by side are wv = w, sv = C H w.
 * srf_ms_ssim_forward writes out[0] = mean over (b, c) (size_average != 0) or out[b] = mean over c, and keeps in the
 * workspace (srf_ms_ssim_workspace_bytes, 256-byte aligned) what srf_ms_ssim_backward needs: pass the same workspace,
 * inputs and flags to the backward.  The backward takes the upstream gradient of `out` (device, same shape) and
 * writes dL/dX through dx_addr; Y gets no gradient.  Where a level's mean is <= 0 (relu) value[b,c] is 0 and every
 * gradient through (b, c) is exactly 0.  Deterministic: no atomics.                                               */
typedef struct srf_ms_ssim_addr { int64_t sb, sc, sy, sx, sv, wv; } srf_ms_ssim_addr;
int srf_ms_ssim_workspace_bytes(int B, int C, int H, int W, size_t* bytes);
/* Host only, for tests and tooling that read the workspace after a call (lara_b200.debug.unpack_ms_ssim).
 *   regions[7]  : byte offsets of the pyramid, its gradient, the per-CTA partial sums (double), the means (double
 *                 [5][B C]), the values (double [B C]), the coefficients (float [5][B C]); then the total size
 *   levels[15]  : per level l, the element index of X_l in the pyramid (float; Y_l follows B C h_l w_l floats later),
 *                 of dX_l in the gradient pyramid (float) and of the level's partial sums (double [B C][ntx ny]);
 *                 the first two are unused at l = 0, whose X, Y and dX are the caller's tensors
 *   dims[30]    : h[5], w[5], px[5], py[5] (pooling padding to the next level), ntx[5], nty[5] (forward tiles)  */
int srf_ms_ssim_workspace_layout(int B, int C, int H, int W, size_t regions[7], size_t levels[15], int dims[30]);
int srf_ms_ssim_forward(srf_stream_t stream, int B, int C, int H, int W,
                        const float* x, const srf_ms_ssim_addr* x_addr, const float* y, const srf_ms_ssim_addr* y_addr,
                        float data_range, int size_average, void* workspace, float* out);
int srf_ms_ssim_backward(srf_stream_t stream, int B, int C, int H, int W,
                         const float* x, const srf_ms_ssim_addr* x_addr, const float* y, const srf_ms_ssim_addr* y_addr,
                         float data_range, int size_average, void* workspace, const float* upstream,
                         float* dx, const srf_ms_ssim_addr* dx_addr);
/* Both passes of a batch against one target in one launch set per direction (DESIGN §3.27): X is the coarse pass `x`
 * and, when `x_fine` is not NULL, the fine pass `x_fine`, both B x C x H x W images read through `x_addr`; Y is read
 * once per pass.  out[0] is the coarse pass's mean over (b, c), out[1] the fine pass's (out [2]; [1] without x_fine).
 * Each (scene, pass, channel) plane's value and coefficients have the bits of srf_ms_ssim_forward on that pass alone
 * (size_average = 1), which is this with x_fine NULL.  The backward takes upstream [2] (or [1]) and writes, or with
 * accumulate != 0 adds, dL/dX into dx and dx_fine through dx_addr (dx_fine given exactly when x_fine is).  Needs
 * 2 B C <= 65535 with x_fine; the workspace is srf_ms_ssim_passes_workspace_bytes(..., with_fine = x_fine != NULL). */
int srf_ms_ssim_passes_workspace_bytes(int B, int C, int H, int W, int with_fine, size_t* bytes);
int srf_ms_ssim_passes_forward(srf_stream_t stream, int B, int C, int H, int W,
                               const float* x, const float* x_fine, const srf_ms_ssim_addr* x_addr,
                               const float* y, const srf_ms_ssim_addr* y_addr, float data_range, void* workspace,
                               float* out);
int srf_ms_ssim_passes_backward(srf_stream_t stream, int B, int C, int H, int W,
                                const float* x, const float* x_fine, const srf_ms_ssim_addr* x_addr,
                                const float* y, const srf_ms_ssim_addr* y_addr, float data_range, void* workspace,
                                const float* upstream, float* dx, float* dx_fine, const srf_ms_ssim_addr* dx_addr,
                                int accumulate);

/* ---- fused single-scale SSIM (pytorch-msssim 1.0.0 ssim; evaluation.py:93 and the D-SSIM loss term) -----------------
 * Level 0 of the MS-SSIM above on its own: the same window, C1, C2, image addressing, workspace rules and determinism.
 * ssim_per_channel[b,c] = mean of the valid ssim_map, relu'd when nonnegative_ssim != 0; out[0] is its mean over (b, c)
 * (size_average != 0), else out[b] is its mean over c.  H and W must be at least 11 (the library instead skips the
 * filter along a shorter side with a warning).  The backward needs the forward's workspace and the same arguments;
 * through a plane whose relu'd value is 0 its gradient is exactly 0.                                                    */
int srf_ssim_workspace_bytes(int B, int C, int H, int W, size_t* bytes);
int srf_ssim_forward(srf_stream_t stream, int B, int C, int H, int W,
                     const float* x, const srf_ms_ssim_addr* x_addr, const float* y, const srf_ms_ssim_addr* y_addr,
                     float data_range, int size_average, int nonnegative_ssim, void* workspace, float* out);
int srf_ssim_backward(srf_stream_t stream, int B, int C, int H, int W,
                      const float* x, const srf_ms_ssim_addr* x_addr, const float* y, const srf_ms_ssim_addr* y_addr,
                      float data_range, int size_average, int nonnegative_ssim, void* workspace,
                      const float* upstream, float* dx, const srf_ms_ssim_addr* dx_addr);

/* ---- optional per-kernel timing (no reference counterpart; used by bench.py's roofline) --
 * Between srf_profile_begin() and srf_profile_end() every kernel launch made by this
 * library is bracketed by CUDA events on its launching stream.  srf_profile_end waits for
 * them and returns, per kernel id, the summed device time in ms and the launch count.
 * Kernel ids: 0 preprocess_fwd, 1 tile_scan, 2 scatter, 3 sort_small, 4 sort_big,
 * 5 render_fwd, 6 render_bwd, 7 preprocess_bwd (SRF_NUM_KERNELS entries).  Not thread-safe.
 * The forward-only blend counts as render_fwd.
 * The deterministic backward runs the blend backward twice: two render_bwd launches per call.            */
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
