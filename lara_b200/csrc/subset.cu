// subset.cu -- render a subset of a forward's Gaussians from that forward's binning (DESIGN §3.18): LaRa's fine pass
// renders the coarse pass's Gaussians under a mask, with the same cameras and new SH coefficients.
//
// Stage 1 and the binning of a fresh forward of the gathered subset would recompute what the coarse forward already
// holds.  Every geometric quantity of a Gaussian (record words q0-q3 and q5, depth, tile rectangle, radius) depends on
// its own parameters and the camera alone, so the subset's are the coarse ones, copied; only q4, the colour, is new.
// The per-tile lists are sorted by (depth bits, Gaussian index) and the mask keeps index order, so each subset tile's
// list is the coarse list with the unmasked Gaussians removed, in the same order.  Two kernels build that state:
//   records : per (subset Gaussian j, view): copy the coarse record / depth / rect / radius of Gaussian idx[j] and
//             recompute q4 from shs[j] with the preprocess's own SH code (sh_eval.cuh); view 0 also writes the rank map
//             rank[idx[j]] = j;
//   filter  : one warp per (tile, view) walks the coarse list in order and keeps, ballot-compacted, the entries whose
//             rank is set, writing ranks (subset indices) at the coarse tile's start offset.
// Then the unchanged blend forward runs on that state (views_blend), and srf_scenes_backward with P = n_max takes its
// gradient.  Nothing is counted, sorted or read back.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "../../include/surfel_rasterizer.h"
#include "sh_eval.cuh"
#include "surfel_common.cuh"
#include "surfel_kernels.h"

namespace srf {
namespace {

constexpr uint32_t kNoRank = 0xffffffffu;

template <typename T>
T* at(const void* base, size_t off) {
    return reinterpret_cast<T*>(reinterpret_cast<uintptr_t>(base) + off);
}

struct RecordsArgs {
    int P, n, D, M;
    int n_slot, views_per_scene;   // Gaussians per view of the subset state; views per scene
    const int64_t* offsets;        // [S+1]: scene s's subset is idx[offsets[s] .. offsets[s+1]); null: one scene
    const int64_t* idx;            // [n] ascending coarse indices per scene
    const float* means3D;          // [S,P,3] coarse centers
    const float* shs;              // [n,M,3]
    const float* cams;             // [V, SRF_CAM_FLOATS]
    const int* c_radii;            // [V,P]
    const float4* c_rec;
    const float* c_depths;
    const uint2* c_rects;
    size_t c_geom_stride;
    int* radii;                    // [V,n_slot] out
    float4* rec;
    float* depths;
    uint2* rects;
    size_t geom_stride;
    uint32_t* rank;                // [S,P], kNoRank outside the subset
};

__global__ void __launch_bounds__(256) subset_records_kernel(RecordsArgs a) {
    const int j = blockIdx.x * 256 + threadIdx.x;
    const int view = blockIdx.y;
    const int scene = view / a.views_per_scene;
    const int64_t first = a.offsets ? a.offsets[scene] : 0;
    if (j >= (a.offsets ? a.offsets[scene + 1] - first : a.n)) return;
    const int64_t g = a.idx[first + j];
    if (view == scene * a.views_per_scene) a.rank[(size_t)scene * a.P + g] = (uint32_t)j;
    const int radius = a.c_radii[(size_t)view * a.P + g];
    a.radii[(size_t)view * a.n_slot + j] = radius;
    view_ptr(a.rects, view, a.geom_stride)[j] = view_ptr(a.c_rects, view, a.c_geom_stride)[g];
    if (radius == 0) return;      // culled: the preprocess writes no record and no depth either
    const float4* cq = view_ptr(a.c_rec, view, a.c_geom_stride) + (size_t)g * SRF_REC_QUADS;
    float4* q = view_ptr(a.rec, view, a.geom_stride) + (size_t)j * SRF_REC_QUADS;
    q[0] = cq[0]; q[1] = cq[1]; q[2] = cq[2]; q[3] = cq[3]; q[5] = cq[5];
    view_ptr(a.depths, view, a.geom_stride)[j] = view_ptr(a.c_depths, view, a.c_geom_stride)[g];
    // q4 exactly as preprocess_fwd_kernel writes it: normalised view direction, SH -> RGB, clamp bits
    const float* campos = a.cams + (size_t)view * SRF_CAM_FLOATS + SRF_CAM_CAMPOS;
    const float* mean = a.means3D + 3 * ((size_t)scene * a.P + g);
    const float px = mean[0], py = mean[1], pz = mean[2];
    float dx = fadd_(px, -campos[0]), dy = fadd_(py, -campos[1]), dz = fadd_(pz, -campos[2]);
    const float len = __fsqrt_rn(fma_(dz, dz, fma_(dx, dx, fmul_(dy, dy))));
    dx = __fdiv_rn(dx, len); dy = __fdiv_rn(dy, len); dz = __fdiv_rn(dz, len);
    float rgb[3];
    sh_to_rgb(a.D, a.shs + (size_t)(first + j) * 3 * a.M, dx, dy, dz, rgb);
    int clampbits = 0;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        if (rgb[c] < 0.0f) { clampbits |= (1 << c); }
        rgb[c] = fmaxf(rgb[c], 0.0f);
    }
    q[4] = make_float4(rgb[0], rgb[1], rgb[2], __int_as_float(clampbits));
}

struct FilterArgs {
    int n, ntiles;
    int P, views_per_scene;
    uint32_t capacity;
    const uint32_t* rank;          // [S,P]
    const uint2* c_ranges;
    const uint32_t* c_order;
    const uint32_t* c_counters;
    const uint32_t* c_plist;
    size_t c_tile_stride, c_plist_stride;
    uint2* ranges;
    uint32_t* order;
    uint32_t* tile_count;
    uint32_t* counters;
    uint32_t* plist;
    size_t tile_stride, plist_stride;
};

__global__ void __launch_bounds__(256) subset_filter_kernel(FilterArgs a) {
    const int t = (blockIdx.x * 256 + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    const int view = blockIdx.y;
    if (t >= a.ntiles) return;
    const uint2 cr = view_ptr(a.c_ranges, view, a.c_tile_stride)[t];
    const uint32_t* src = view_ptr(a.c_plist, view, a.c_plist_stride);
    const uint32_t* rank = a.rank + (size_t)(view / a.views_per_scene) * a.P;
    uint32_t* dst = view_ptr(a.plist, view, a.plist_stride) + cr.x;
    const uint32_t below = (1u << lane) - 1u;
    uint32_t kept = 0;
    const uint32_t end = (a.n > 0 && cr.y <= a.capacity) ? cr.y : cr.x;
    // kFilterChunks x 32 entries per trip: all list and rank loads of a trip are in flight together, then the ballots
    // append the kept ranks in list order
    constexpr int kFilterChunks = 4;
    for (uint32_t base = cr.x; base < end; base += 32 * kFilterChunks) {
        uint32_t r[kFilterChunks];
#pragma unroll
        for (int k = 0; k < kFilterChunks; ++k) {
            const uint32_t i = base + 32 * k + lane;
            r[k] = i < end ? src[i] : kNoRank;
        }
#pragma unroll
        for (int k = 0; k < kFilterChunks; ++k) r[k] = r[k] != kNoRank ? rank[r[k]] : kNoRank;
#pragma unroll
        for (int k = 0; k < kFilterChunks; ++k) {
            const uint32_t keep = __ballot_sync(0xffffffffu, r[k] != kNoRank);
            if (r[k] != kNoRank) dst[kept + __popc(keep & below)] = r[k];
            kept += __popc(keep);
        }
    }
    if (lane == 0) {
        view_ptr(a.ranges, view, a.tile_stride)[t] = kept ? make_uint2(cr.x, cr.x + kept) : make_uint2(0u, 0u);
        view_ptr(a.tile_count, view, a.tile_stride)[(size_t)t * SRF_TILE_CTR_STRIDE] = kept;
        // the coarse launch order (heaviest coarse tile first): any order of the tiles gives the same bits
        view_ptr(a.order, view, a.tile_stride)[t] = view_ptr(a.c_order, view, a.c_tile_stride)[t];
        // counters[0]: the extent of the list in use, which is the coarse one (the kept entries stay in place)
        if (t == 0) view_ptr(a.counters, view, a.tile_stride)[0] = view_ptr(a.c_counters, view, a.c_tile_stride)[0];
    }
}

size_t rank_bytes(int P) { return align_up((size_t)(P > 0 ? P : 1) * sizeof(uint32_t)); }

}  // namespace

// srf_scenes_subset_forward: S scenes of Vs views, scene s's subset idx[offsets[s] .. offsets[s+1]) of its P coarse
// Gaussians (offsets null: S = 1, the n Gaussians idx[0..n)), n_slot Gaussians per view of the subset state.  The caller
// has checked S, Vs, the offsets and n_slot.
int subset_forward(const char* fn, cudaStream_t stream, int S, int Vs, int P, int n, int n_slot, const int64_t* offsets,
                   int D, int M, const int64_t* idx, const float* means3D, const float* shs, const float* colors_precomp,
                   const float* cams, int image_height, int image_width, size_t capacity,
                   const int* coarse_radii, const void* coarse_geom_state, const void* coarse_tile_state,
                   const uint32_t* coarse_point_list, size_t coarse_capacity, int coarse_for_backward,
                   int* radii, void* geom_state, void* tile_state, uint32_t* point_list, void* image_state,
                   float* out_color, float* out_others, void* workspace, int for_backward) {
    const int V = S * Vs;
    // every check before anything is enqueued
    if (P < 0 || n < 0 || image_height <= 0 || image_width <= 0) return set_error("%s: bad sizes", fn);
    if (image_height > 16 * 65535 || image_width > 16 * 65535) return set_error("%s: image too large", fn);
    if (D < 0 || D > 3) return set_error("%s: sh degree must be in [0,3]", fn);
    if (colors_precomp) return set_error("%s: colors_precomp is not supported: the subset's colour comes from shs", fn);
    if (capacity != coarse_capacity)
        return set_error("%s: capacity %zu differs from the coarse forward's %zu: the kept entries stay at the coarse "
                         "list positions", fn, capacity, coarse_capacity);
    if (capacity > 0xfffffff0ull) return set_error("%s: capacity exceeds 32-bit instance indices", fn);
    if (!cams || !out_color || !out_others || !coarse_tile_state || !tile_state || (for_backward && !image_state))
        return set_error("%s: null required pointer", fn);
    if (capacity > 0 && (!coarse_point_list || !point_list)) return set_error("%s: null point list", fn);
    if (n > 0) {
        if (!idx || !means3D || !coarse_radii || !coarse_geom_state || !radii || !geom_state || !workspace)
            return set_error("%s: null required pointer", fn);
        if (!shs) return set_error("%s: shs is required", fn);
        if (M < (D + 1) * (D + 1)) return set_error("%s: M=%d SH coefficients < (D+1)^2 for D=%d", fn, M, D);
        if (misaligned(coarse_geom_state) || misaligned(geom_state) || misaligned(workspace))
            return set_error("%s: geom_state, coarse_geom_state and workspace must be 256-byte aligned", fn);
    }
    if (misaligned(coarse_tile_state) || misaligned(tile_state) || (for_backward && misaligned(image_state)) ||
        (capacity > 0 && (misaligned(coarse_point_list) || misaligned(point_list))))
        return set_error("%s: tile_state, point_list and image_state (and the coarse ones) must be 256-byte aligned", fn);

    const srf::StateLayout cl = srf::state_layout(P, image_height, image_width);
    const srf::StateLayout sl = srf::state_layout(n_slot, image_height, image_width);
    uint32_t* rank = static_cast<uint32_t*>(workspace);
    cudaError_t e;
    if (n > 0) {
        e = cudaMemsetAsync(rank, 0xff, (size_t)S * P * sizeof(uint32_t), stream);
        if (e != cudaSuccess) return srf::cuda_error("memset rank", e);
        srf::RecordsArgs r;
        memset(&r, 0, sizeof(r));
        r.P = P; r.n = n; r.D = D; r.M = M;
        r.n_slot = n_slot; r.views_per_scene = Vs; r.offsets = offsets;
        r.idx = idx; r.means3D = means3D; r.shs = shs; r.cams = cams;
        r.c_radii = coarse_radii;
        r.c_rec = srf::at<const float4>(coarse_geom_state, cl.rec);
        r.c_depths = srf::at<const float>(coarse_geom_state, cl.depths);
        r.c_rects = srf::at<const uint2>(coarse_geom_state, cl.rects);
        r.c_geom_stride = cl.geom_stride;
        r.radii = radii;
        r.rec = srf::at<float4>(geom_state, sl.rec);
        r.depths = srf::at<float>(geom_state, sl.depths);
        r.rects = srf::at<uint2>(geom_state, sl.rects);
        r.geom_stride = sl.geom_stride;
        r.rank = rank;
        srf::subset_records_kernel<<<dim3((n_slot + 255) / 256, V), 256, 0, stream>>>(r);
        e = cudaGetLastError();
        if (e != cudaSuccess) return srf::cuda_error("subset_records launch", e);
    }
    srf::FilterArgs f;
    memset(&f, 0, sizeof(f));
    f.n = n; f.ntiles = cl.ntiles; f.capacity = (uint32_t)capacity;
    f.P = P; f.views_per_scene = Vs;
    f.rank = rank;
    f.c_ranges = srf::at<const uint2>(coarse_tile_state, cl.ranges);
    f.c_order = srf::at<const uint32_t>(coarse_tile_state, cl.order);
    f.c_counters = srf::at<const uint32_t>(coarse_tile_state, cl.counters);
    f.c_plist = coarse_point_list;
    f.c_tile_stride = cl.tile_stride;
    f.c_plist_stride = srf::plist_stride(capacity, coarse_for_backward != 0);
    f.ranges = srf::at<uint2>(tile_state, sl.ranges);
    f.order = srf::at<uint32_t>(tile_state, sl.order);
    f.tile_count = srf::at<uint32_t>(tile_state, sl.tile_count);
    f.counters = srf::at<uint32_t>(tile_state, sl.counters);
    f.plist = point_list;
    f.tile_stride = sl.tile_stride;
    f.plist_stride = srf::plist_stride(capacity, for_backward != 0);
    srf::subset_filter_kernel<<<dim3((cl.ntiles + 7) / 8, V), 256, 0, stream>>>(f);
    e = cudaGetLastError();
    if (e != cudaSuccess) return srf::cuda_error("subset_filter launch", e);
    return srf::views_blend(stream, V, n_slot, image_height, image_width, capacity, geom_state, tile_state, point_list,
                            image_state, cams, out_color, out_others, for_backward != 0);
}

}  // namespace srf

using srf::misaligned;
using srf::set_error;

extern "C" {

int srf_views_subset_workspace_bytes(int P, size_t* bytes) {
    if (P < 0 || !bytes) return set_error("srf_views_subset_workspace_bytes: bad arguments");
    *bytes = srf::rank_bytes(P);
    return 0;
}

int srf_scenes_subset_forward(srf_stream_t stream_, int S, int Vs, int P, int n, int n_max, int D, int M,
                              const int64_t* idx, const int64_t* offsets, const float* means3D, const float* shs,
                              const float* colors_precomp, const float* cams, int image_height, int image_width,
                              size_t capacity, const int* coarse_radii, const void* coarse_geom_state,
                              const void* coarse_tile_state, const uint32_t* coarse_point_list, size_t coarse_capacity,
                              int coarse_for_backward, int* radii, void* geom_state, void* tile_state,
                              uint32_t* point_list, void* image_state, float* out_color, float* out_others,
                              void* workspace, int for_backward) {
    const char* fn = "srf_scenes_subset_forward";
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (srf::check_scenes(fn, S, Vs)) return 1;
    if (P < 0 || n < 0 || n_max < 0) return set_error("%s: bad sizes", fn);
    if (n_max > P) return set_error("%s: bad sizes: a subset of n_max = %d > P = %d Gaussians", fn, n_max, P);
    if ((size_t)S * P > 0x7fffffffull) return set_error("%s: S * P exceeds 32-bit Gaussian indices", fn);
    if (!offsets) {         // one scene, idx[0..n): nothing to read back, no wait for the stream
        if (S != 1 || n_max != n)
            return set_error("%s: null offsets need one scene and n_max == n, got S = %d, n = %d, n_max = %d", fn, S, n,
                             n_max);
    } else if (srf::check_offsets(fn, stream, S, offsets, n_max, n)) {
        return 1;
    }
    return srf::subset_forward(fn, stream, S, Vs, P, n, n_max, offsets, D, M, idx, means3D, shs, colors_precomp, cams,
                               image_height, image_width, capacity, coarse_radii, coarse_geom_state, coarse_tile_state,
                               coarse_point_list, coarse_capacity, coarse_for_backward, radii, geom_state, tile_state,
                               point_list, image_state, out_color, out_others, workspace, for_backward);
}

}  // extern "C"
