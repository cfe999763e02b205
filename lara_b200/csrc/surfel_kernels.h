// surfel_kernels.h -- internal (non-ABI) interface of the library: the rasterizer's kernel launchers, which api.cu's
// entries call, and the host helpers every translation unit's extern "C" entries share.  The public
// boundary is include/surfel_rasterizer.h (and surfel_mesh.h, surfel_fine_head.h); each fused op (epilogue, loss,
// decoder layout, point features, MS-SSIM, mesh, fine head) keeps its argument structs and entries in its own .cu.
//
// Every rasterizer kernel takes a *view* dimension: the V target views of one scene share the Gaussian set
// (reference caller loop lightning/network.py:484-497), so one launch covers all of them.  Per-view
// arrays live in per-view workspaces of identical layout; the structs carry the base pointers of view 0
// plus the byte stride from one view's workspace to the next (`*_stride`).  Camera data (view matrix,
// camera position, background) are pointers into view 0's camera record (include/surfel_rasterizer.h
// SRF_CAM_*), the records `cam_stride` floats apart.  Images are stacked [V,C,H,W].
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "../../include/surfel_rasterizer.h"

namespace srf {

// ---- host helpers of the extern "C" entries ----
// Record a failure: the text goes to the thread-local buffer srf_last_error() returns.  Returns 1, the C ABI's
// failure status.
int set_error(const char* fmt, ...) __attribute__((format(printf, 1, 2)));
// a CUDA call's failure as "<what>: <CUDA error string>"
inline int cuda_error(const char* what, cudaError_t e) { return set_error("%s: %s", what, cudaGetErrorString(e)); }
// workspaces are 256-byte aligned, and so are the regions inside them
inline bool misaligned(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 255) != 0; }
inline size_t align_up(size_t x) { return (x + 255) / 256 * 256; }
// Reads a device flag that the work enqueued so far sets (waits for the stream); set means a deterministic
// fixed-point sum overflowed, reported as a failure of `fn`.
int check_overflow_flag(const char* fn, const uint32_t* flag, cudaStream_t stream);

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
    const float* means3D;
    const float* scales;
    const float* rotations;
    const float* shs;
    const float* viewmatrix;
    const float* campos;
    size_t cam_stride;
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

// The scenes of an srf_scenes_* call (include/surfel_rasterizer.h): S scenes of Vs views each, laid out as V = S*Vs
// views; view v belongs to scene v / Vs.  One scene is S = 1.  Passed as a __grid_constant__ kernel parameter (the
// kernels index `fov` by the scene without a local copy) next to the per-view arguments, whose Gaussian pointers are
// those of scene 0.  scene_fov is the one place the focal lengths are computed.
struct SceneArgs {
    int views_per_scene;         // Vs
    const int64_t* offsets;      // [S+1] device: scene s's Gaussians are rows [offsets[s], offsets[s+1]) of the inputs
                                 //   and gradients; null: rows [s*P, (s+1)*P)
    float4 fov[SRF_MAX_SCENES];  // per scene: focal_x, focal_y, tan_fovx, tan_fovy
};

// pointer to row `row` of a `width`-float row array; null stays null
template <typename T>
__device__ __forceinline__ T* rows_at(T* p, size_t row, int width) {
    return p ? p + row * width : p;
}

// Optional per-kernel CUDA-event timing (srf_profile_begin/end in the C ABI); no-ops unless enabled.
enum KernelId { K_PREPROCESS_FWD = 0, K_TILE_SCAN, K_SCATTER, K_SORT_SMALL, K_SORT_BIG, K_RENDER_FWD,
                K_RENDER_BWD, K_PREPROCESS_BWD, K_COUNT };
void prof_start(int kernel, cudaStream_t stream);
void prof_stop(int kernel, cudaStream_t stream);

// number of SMs of the current device (cached per device)
int sm_count();

// Byte offsets inside one view's geom / tile workspaces and their per-view strides (the layout srf_state_layout
// reports), for the entries outside api.cu that read or write the forward's state.
struct StateLayout {
    size_t rec, depths, rects, geom_stride;
    size_t tile_count, counters, ranges, order, tile_stride;
    int gx, gy, ntiles;
};
StateLayout state_layout(int P, int H, int W);
// bytes from one view's point_list workspace to the next (the list, then for_backward the contribution record)
size_t plist_stride(size_t capacity, bool for_backward);
// The blend forward of V views on the state stage 1 and the binning left (ranges, launch order, point_list, records):
// the render_fwd launch of srf_scenes_forward, arguments checked by the caller.  record = false: forward-only.
int views_blend(cudaStream_t stream, int V, int P, int image_height, int image_width, size_t capacity,
                const void* geom_state, const void* tile_state, const uint32_t* point_list, void* image_state,
                const float* cams, float* out_color, float* out_others, bool record);

// Argument checks of the srf_scenes_* entries, made before they enqueue anything.  check_scenes: 0 < S <=
// SRF_MAX_SCENES, Vs > 0, S * Vs <= 65535 (views are a grid dimension).  scene_fov: finite positive tan_fov [S,2]
// (host) into s.fov.  check_offsets: reads the device array offsets [S+1] (waits for the stream) and checks that it
// starts at 0, never decreases, puts at most n_max Gaussians in a scene and, if n >= 0, ends at n.
int check_scenes(const char* fn, int S, int Vs);
int scene_fov(const char* fn, int S, const float* tan_fov, int image_height, int image_width, SceneArgs& s);
int check_offsets(const char* fn, cudaStream_t stream, int S, const int64_t* offsets, int n_max, int n);

// a.nviews = S * Vs views, each reading the Gaussian inputs of its scene in `s`
cudaError_t launch_preprocess_fwd(const PreprocessArgs& a, const SceneArgs& s, cudaStream_t stream);
cudaError_t launch_mark_visible(int P, const float* means3D, const float* viewmatrix, uint8_t* present,
                                cudaStream_t stream);
cudaError_t launch_tile_scan(const BinArgs& a, cudaStream_t stream);
cudaError_t launch_bin_and_sort(const BinArgs& a, cudaStream_t stream);
// record = false: the forward-only blend, which writes neither a.masks nor a.accum / a.n_contrib (they may be null)
cudaError_t launch_render_fwd(const RenderFwdArgs& a, bool record, cudaStream_t stream);
cudaError_t launch_render_bwd(const RenderBwdArgs& a, cudaStream_t stream);
// Deterministic blend backward (DESIGN §3.13): a.ggrad / a.ggrad_stride point at zeroed det_record_bytes() records per
// (Gaussian, view); the fp32 gradient records preprocess_bwd reads go to ggrad / ggrad_stride; *overflow (zeroed by the
// caller) is set if a partial sum was over its fixed-point budget.
size_t det_record_bytes();
cudaError_t launch_render_bwd_det(const RenderBwdArgs& a, int P, float* ggrad, size_t ggrad_stride, uint32_t* overflow,
                                  cudaStream_t stream);
// one thread per (Gaussian, scene of `s`), summing that scene's Vs views
cudaError_t launch_preprocess_bwd(const PreprocessBwdArgs& a, const SceneArgs& s, int S, cudaStream_t stream);

}  // namespace srf
