// surfel_kernels.h -- internal (non-ABI) interface between the C-ABI layer (api.cu)
// and the kernel translation units.  The public boundary is include/surfel_rasterizer.h.
//
// Every kernel takes a *view* dimension: the V target views of one scene share the Gaussian set
// (reference caller loop lightning/network.py:484-497), so one launch covers all of them.  Per-view
// arrays live in per-view workspaces of identical layout; the structs carry the base pointers of view 0
// plus the byte stride from one view's workspace to the next (`*_stride`, 0 when nviews == 1).  Camera
// data (view matrix, camera position, background) are three pointers into per-view camera records
// `cam_stride` floats apart.  Images are stacked [V,C,H,W].
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace srf {

// pointer of view `v` given the pointer of view 0 and a byte stride
template <typename T>
__host__ __device__ __forceinline__ T* view_ptr(T* p, int v, size_t stride_bytes) {
    return reinterpret_cast<T*>(reinterpret_cast<uintptr_t>(p) + (size_t)v * stride_bytes);
}

struct PreprocessArgs {
    int P, D, M;
    int nviews;
    const float* means3D;        // [P,3]
    const float* scales;         // [P,2]
    const float* rotations;      // [P,4] (w,x,y,z)
    const float* opacities;      // [P]
    const float* shs;            // [P,M,3] or null
    const float* transMat_precomp;  // [P,9] or null
    const float* colors_precomp;    // [P,3] or null
    const float* viewmatrix;     // [16] column-major world->view  (per view, cam_stride floats apart)
    const float* campos;         // [3]                             (per view)
    size_t cam_stride;           // floats
    int W, H;
    float focal_x, focal_y;
    int gx, gy;                  // tile grid
    int prefiltered;
    int stage_sh;                // set by the launcher
    int raw_act;                 // inputs are LaRa's raw network outputs: opacity logits, log-scales, unnormalised quaternions
    int* radii;                  // [V,P] out
    float4* rec;                 // [P*6] out                (geom workspace)
    float* depths;               // [P] out                  (geom workspace)
    uint2* rects;                // [P] out: (x0 | y0<<16, x1 | y1<<16)   (geom workspace)
    uint32_t* tile_count;        // [ntiles * SRF_TILE_CTR_STRIDE] in/out (zeroed by the caller)   (tile workspace)
    size_t geom_stride, tile_stride;   // bytes
};

struct BinArgs {
    int P;
    int nviews;
    int ntiles;
    int gx;
    uint32_t capacity;           // number of instance slots in entries / point_list (per view)
    const float* depths;
    const uint2* rects;          // empty rect = culled
    uint32_t* tile_count;        // [ntiles * SRF_TILE_CTR_STRIDE]: word 0 count, word 1 bucket cursor
    uint2* ranges;               // [ntiles] out
    uint32_t* counters;          // [4]: num_rendered, big_count, overflow, spare
    uint32_t* count_host;        // [nviews] device-visible pinned host memory: the scan stores num_rendered there directly (or null)
    uint32_t* big_list;          // [ntiles] scratch
    uint32_t* tile_order;        // [ntiles] out: tiles by descending instance count (launch order of the blend CTAs)
    uint64_t* entries;           // [capacity] scratch: depth_bits<<32 | gaussian idx, bucketed by tile
    uint32_t* point_list;        // [capacity] out: per-tile depth-sorted gaussian indices
    size_t geom_stride, tile_stride, entries_stride, plist_stride;   // bytes
};

struct RenderFwdArgs {
    int W, H, gx, gy;
    int nviews;
    uint32_t capacity;
    const uint2* ranges;
    const uint32_t* tile_order;  // [ntiles]: CTA i renders tile tile_order[i] (heaviest first)
    const uint32_t* point_list;
    uint32_t* masks;             // [8][capacity] out: bit l = the splat at this list position was blended into
                                 //   pixel l of 8x4 block w (inside the point_list workspace, plist_stride apart)
    const float4* rec;
    const float* bg;             // [3] device (per view, cam_stride floats apart)
    float* out_color;            // [V,3,H,W]
    float* out_others;           // [V,8,H,W]
    float* accum;                // [3,H,W]: final_T, dist1, dist2      (image workspace)
    uint32_t* n_contrib;         // [2,H,W]: last contributor, median contributor
    size_t geom_stride, tile_stride, plist_stride, image_stride, cam_stride;   // bytes (cam_stride: floats)
};

struct RenderBwdArgs {
    int W, H, gx, gy;
    int nviews;
    uint32_t capacity;
    const uint2* ranges;
    const uint32_t* tile_order;
    const uint32_t* point_list;
    const uint32_t* masks;       // [8][capacity]: the forward's contribution masks (RenderFwdArgs::masks)
    const float4* rec;
    const float* bg;
    const float* accum;
    const uint32_t* n_contrib;
    const float* dL_dpix;        // [V,3,H,W]
    const float* dL_dothers;     // [V,8,H,W]
    float* ggrad;                // [P,20] zero-initialised accumulation records (per view, ggrad_stride bytes apart)
    size_t geom_stride, tile_stride, plist_stride, image_stride, cam_stride, ggrad_stride;
};

struct PreprocessBwdArgs {
    int P, D, M;
    int nviews;                  // gradients of all views are summed in registers and written once
    const float* means3D;
    const float* scales;
    const float* rotations;
    const float* shs;
    const float* viewmatrix;
    const float* campos;
    size_t cam_stride;
    int W, H;
    float focal_x, focal_y, tan_fovx, tan_fovy;
    int has_precomp_T;           // transMat_precomp was given: only dL_dtransMat is produced
    int has_precomp_color;
    int raw_act;                 // as in PreprocessArgs; gradients are then wrt the raw parameters
    const int* radii;            // [V,P]
    const float4* rec;
    const float* ggrad;          // [P,20] per view
    size_t geom_stride, ggrad_stride;
    int accumulate;              // += into the outputs instead of overwriting (view-sharded accumulation)
    int vec_ok;                  // set by the launcher: output rows are 16/8-byte aligned -> vector stores
    float* dL_dmeans3D;          // [P,3]
    float* dL_dmeans2D;          // [P,3] or null
    float* dL_dsh;               // [P,M,3] or null
    float* dL_dcolors;           // [P,3] or null
    float* dL_dopacity;          // [P]
    float* dL_dscales;           // [P,2]
    float* dL_drotations;        // [P,4]
    float* dL_dtransMat;         // [P,9] or null
};

// Fused render_img epilogue (SURVEY 8f rank 2); all images planar [V,C,H,W] fp32.
struct EpilogueArgs {
    int W, H;
    int nviews;
    float depth_ratio;
    const float* color;          // [V,3,H,W] rasterizer colour
    const float* allmap;         // [V,8,H,W] rasterizer aux maps
    const float* rays;           // [V,H,W,6] or null (then no pseudo normals)
    const float* viewmatrix;     // [16] per view, cam_stride floats apart
    size_t cam_stride;
    // forward outputs
    float* image;                // [V,3,H,W]
    float* depth;                // [V,1,H,W]
    float* acc;                  // [V,H,W]
    float* rend_normal;          // [V,3,H,W]
    float* depth_normal;         // [V,3,H,W]
    float* dist;                 // [V,H,W]
    // backward inputs (any may be null = zero) and outputs
    const float* g_image; const float* g_depth; const float* g_acc;
    const float* g_rend_normal; const float* g_depth_normal; const float* g_dist;
    float* scratch;              // [V,3,H,W]
    float* dL_dcolor;            // [V,3,H,W]
    float* dL_dallmap;           // [V,8,H,W]
};
cudaError_t launch_epilogue_fwd(const EpilogueArgs& a, cudaStream_t stream);
cudaError_t launch_epilogue_bwd(const EpilogueArgs& a, cudaStream_t stream);

// Fused loss -> dL/d(render_img outputs) producer (SURVEY 8f rank 3, lightning/loss.py:33-60).
struct LossArgs {
    int W, H, nviews;
    int with_reg;                // iter > 1000: distortion and normal-consistency terms are on
    float w_mse, w_dist, w_normal;   // weights already divided by the reference's mean() denominators
    const float* image;          // [V,3,H,W]
    const float* target;         // [V,H,W,3] channel-last, the batch's own layout
    const float* rend_normal;    // [V,3,H,W]
    const float* depth_normal;   // [V,3,H,W]
    const float* acc;            // [V,H,W]
    const float* dist;           // [V,H,W]
    double* sums;                // [3]: sum (image-target)^2, sum dist, sum (1 - <rn,dn>) acc   (zeroed by the caller); null = skip
    const float* gout;           // device scalar: upstream gradient of the loss (null = 1)
    float* g_image;              // [V,3,H,W] out (may be null: forward statistics only)
    float* g_rend_normal; float* g_depth_normal; float* g_dist;
};
cudaError_t launch_loss_fused(const LossArgs& a, cudaStream_t stream);

// Decoder epilogue (SURVEY 8f rank 4, lightning/network.py:261-278, 425-429): MLP output rows -> the five
// contiguous parameter tensors, and the mirror-image backward.
struct DecoderArgs {
    size_t total;                // B * N * K Gaussians
    int N, K, C, sh_dim;         // voxels per scene, Gaussians per voxel, floats per row (10 + sh_dim), SH floats
    float opacity_shift, scaling_shift, half_cell;
    const float* params;         // [B,N,K*C] MLP output (fp32)
    const float* group_centers;  // [N,3]
    float* centers; float* shs; float* opacity; float* scaling; float* rotation;     // forward outputs
    const float* g_centers; const float* g_shs; const float* g_opacity; const float* g_scaling; const float* g_rotation;
    float* g_params;             // [B,N,K*C] backward output
};
cudaError_t launch_decoder_layout(const DecoderArgs& a, bool backward, cudaStream_t stream);

// Fine-pass point-feature sampler (lightning/network.py:390-411, projection :182-187): n points sampled in V source
// views from the 8-channel stack img_ref | image | acc | depth; all images planar fp32.
struct PointFeatsArgs {
    int V, n, H, W;
    const float* points;         // [n,3]
    const float* w2cs;           // [V,4,4] row-major
    const float* ixts;           // [V,3,3] row-major
    const float* img_ref;        // [V,3,H,W]
    const float* image;          // [V,3,H,W]
    const float* acc;            // [V,H,W]
    const float* depth;          // [V,H,W]
    float* feats;                // [V,8,n] forward output
    const float* g_feats;        // [V,8,n] backward input
    float* g_points;             // [n,3] written (may be null)
    float* g_image; float* g_acc; float* g_depth;   // accumulated into, cleared by the caller (each may be null)
};
cudaError_t launch_point_feats(const PointFeatsArgs& a, bool backward, cudaStream_t stream);

// Optional per-kernel CUDA-event timing (srf_profile_begin/end in the C ABI); no-ops unless enabled.
enum KernelId { K_PREPROCESS_FWD = 0, K_TILE_SCAN, K_SCATTER, K_SORT_SMALL, K_SORT_BIG, K_RENDER_FWD,
                K_RENDER_BWD, K_PREPROCESS_BWD, K_COUNT };
void prof_start(int kernel, cudaStream_t stream);
void prof_stop(int kernel, cudaStream_t stream);

// number of SMs of the current device (cached per device)
int sm_count();

cudaError_t launch_preprocess_fwd(const PreprocessArgs& a, cudaStream_t stream);
cudaError_t launch_mark_visible(int P, const float* means3D, const float* viewmatrix, uint8_t* present,
                                cudaStream_t stream);
cudaError_t launch_tile_scan(const BinArgs& a, cudaStream_t stream);
cudaError_t launch_bin_and_sort(const BinArgs& a, cudaStream_t stream);
cudaError_t launch_render_fwd(const RenderFwdArgs& a, cudaStream_t stream);
cudaError_t launch_render_bwd(const RenderBwdArgs& a, cudaStream_t stream);
cudaError_t launch_preprocess_bwd(const PreprocessBwdArgs& a, cudaStream_t stream);

}  // namespace srf
