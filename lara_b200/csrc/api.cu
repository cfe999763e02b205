// api.cu -- the library-wide part of the extern "C" boundary declared in include/surfel_rasterizer.h: the ABI version,
// the last-error buffer, per-kernel profiling, the workspace layouts and the rasterizer's entries (forward, its
// stage-2 re-run, backward, srf_mark_visible).  The fused ops' entries are defined next to their kernels.
// Plain pointers and sizes in, int status out; only enqueues work on the given stream.
#include <cuda_runtime.h>
#include <math.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <mutex>
#include <vector>

#include "../../include/surfel_rasterizer.h"
#include "surfel_common.cuh"
#include "surfel_kernels.h"

using srf::align_up;
using srf::cuda_error;
using srf::misaligned;
using srf::set_error;

namespace {

thread_local char g_err[512] = "";

struct GeomLayout { size_t rec, depths, rects, total; };
struct TileLayout { size_t count, counters, ranges, big, order, total; int gx, gy, ntiles; };
struct ImageLayout { size_t accum, ncontrib, total; };

GeomLayout geom_layout(int P) {
    GeomLayout l;
    const size_t p = (size_t)(P > 0 ? P : 0);
    size_t o = 0;
    l.rec = o; o = align_up(o + p * SRF_REC_QUADS * sizeof(float4));
    l.depths = o; o = align_up(o + p * sizeof(float));
    l.rects = o; o = align_up(o + p * sizeof(uint2));
    l.total = o + 256;
    return l;
}

TileLayout tile_layout(int H, int W) {
    TileLayout l;
    l.gx = (W + SRF_TILE - 1) / SRF_TILE;
    l.gy = (H + SRF_TILE - 1) / SRF_TILE;
    l.ntiles = l.gx * l.gy;
    const size_t n = (size_t)l.ntiles;
    size_t o = 0;
    l.count = o; o += n * SRF_TILE_CTR_STRIDE * sizeof(uint32_t);   // one 256 B block per tile
    l.counters = o; o = align_up(o + 4 * sizeof(uint32_t));   // blocks+counters are zeroed by one memset
    l.ranges = o; o = align_up(o + n * sizeof(uint2));
    l.big = o; o = align_up(o + n * sizeof(uint32_t));
    l.order = o; o = align_up(o + n * sizeof(uint32_t));
    l.total = o + 256;
    return l;
}

ImageLayout image_layout(int H, int W) {
    ImageLayout l;
    const size_t npix = (size_t)H * W;
    size_t o = 0;
    l.accum = o; o = align_up(o + 3 * npix * sizeof(float));
    l.ncontrib = o; o = align_up(o + 2 * npix * sizeof(uint32_t));
    l.total = o + 256;
    return l;
}

template <typename T>
T* at(const void* base, size_t off) {
    return reinterpret_cast<T*>(reinterpret_cast<uintptr_t>(base) + off);
}

// One view's point_list workspace: the depth-sorted list (u32 [capacity]), then, for a forward a backward follows, the
// blend forward's contribution masks (u32 [8 warp blocks][capacity], indexed by list position), which the blend
// backward replays.
size_t plist_masks_offset(size_t capacity) { return align_up(capacity * sizeof(uint32_t)); }
size_t plist_stride_bytes(size_t capacity, bool for_backward) {
    if (!for_backward) return plist_masks_offset(capacity);
    return plist_masks_offset(capacity) + align_up(capacity * 8 * sizeof(uint32_t)) + 256;
}
size_t entries_stride_bytes(size_t capacity) { return align_up(capacity * sizeof(uint64_t)) + 256; }
size_t ggrad_stride_bytes(int P) { return align_up((size_t)P * SRF_GRAD_FLOATS * sizeof(float)) + 256; }

// Scratch of the deterministic backward: V fp32 gradient-record arrays (as srf_scenes_backward's scratch), then V arrays
// of fixed-point records, then the overflow flag.
size_t det_stride_bytes(int P) { return align_up((size_t)P * srf::det_record_bytes()); }
size_t det_scratch_bytes(int V, int P) { return (ggrad_stride_bytes(P) + det_stride_bytes(P)) * (size_t)V + 256; }

// ---- optional per-kernel timing --------------------------------------------------
struct ProfSpan { int kernel; cudaEvent_t start, stop; };
bool g_prof_on = false;
std::mutex g_prof_mu;      // autograd runs the backward on another host thread
std::vector<ProfSpan> g_spans;
std::vector<cudaEvent_t> g_event_pool;
cudaEvent_t g_open[srf::K_COUNT];

cudaEvent_t take_event() {
    if (!g_event_pool.empty()) { cudaEvent_t e = g_event_pool.back(); g_event_pool.pop_back(); return e; }
    cudaEvent_t e = nullptr;
    cudaEventCreate(&e);
    return e;
}

}  // namespace

namespace srf {
int set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return 1;
}

int check_overflow_flag(const char* fn, const uint32_t* flag, cudaStream_t stream) {
    uint32_t h = 0;
    cudaError_t e = cudaMemcpyAsync(&h, flag, sizeof(h), cudaMemcpyDeviceToHost, stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
    if (e != cudaSuccess) return cuda_error("deterministic overflow flag read-back", e);
    if (h) return set_error("%s: a gradient term is not finite or beyond the range of the deterministic fixed-point sum; "
                            "no gradient was produced", fn);
    return 0;
}

void prof_start(int kernel, cudaStream_t stream) {
    if (!g_prof_on) return;
    std::lock_guard<std::mutex> lk(g_prof_mu);
    g_open[kernel] = take_event();
    cudaEventRecord(g_open[kernel], stream);
}
void prof_stop(int kernel, cudaStream_t stream) {
    if (!g_prof_on) return;
    std::lock_guard<std::mutex> lk(g_prof_mu);
    ProfSpan s; s.kernel = kernel; s.start = g_open[kernel]; s.stop = take_event();
    cudaEventRecord(s.stop, stream);
    g_spans.push_back(s);
}

int sm_count() {
    // per device: a process may drive several GPUs
    static int cache[64] = {0};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
    if (cache[dev] == 0) {
        int n = 0;
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        cache[dev] = n > 0 ? n : 132;
    }
    return cache[dev];
}

StateLayout state_layout(int P, int H, int W) {
    const GeomLayout g = geom_layout(P);
    const TileLayout t = tile_layout(H, W);
    StateLayout s;
    s.rec = g.rec; s.depths = g.depths; s.rects = g.rects; s.geom_stride = g.total;
    s.tile_count = t.count; s.counters = t.counters; s.ranges = t.ranges; s.order = t.order; s.tile_stride = t.total;
    s.gx = t.gx; s.gy = t.gy; s.ntiles = t.ntiles;
    return s;
}

size_t plist_stride(size_t capacity, bool for_backward) { return plist_stride_bytes(capacity, for_backward); }

int check_scenes(const char* fn, int S, int Vs) {
    if (S <= 0 || Vs <= 0) return set_error("%s: need S > 0 scenes of Vs > 0 views, got S = %d, Vs = %d", fn, S, Vs);
    if (S > SRF_MAX_SCENES) return set_error("%s: S = %d scenes exceeds SRF_MAX_SCENES = %d", fn, S, SRF_MAX_SCENES);
    if ((int64_t)S * Vs > 65535) return set_error("%s: S * Vs = %lld views exceeds 65535", fn, (long long)S * Vs);
    return 0;
}

int scene_fov(const char* fn, int S, const float* tan_fov, int image_height, int image_width, SceneArgs& s) {
    if (!tan_fov) return set_error("%s: null tan_fov", fn);
    for (int i = 0; i < S; ++i) {
        const float tx = tan_fov[2 * i], ty = tan_fov[2 * i + 1];
        if (!isfinite(tx) || !isfinite(ty) || !(tx > 0.f) || !(ty > 0.f))
            return set_error("%s: tan_fov of scene %d is (%g, %g), not finite and positive", fn, i, tx, ty);
        // rasterizer_impl.cu:223-224; the only place the kernels' focal lengths are computed
        s.fov[i] = make_float4(image_width / (2.0f * tx), image_height / (2.0f * ty), tx, ty);
    }
    return 0;
}

int check_offsets(const char* fn, cudaStream_t stream, int S, const int64_t* offsets, int n_max, int n) {
    if (!offsets) return set_error("%s: null offsets", fn);
    int64_t h[SRF_MAX_SCENES + 1];
    cudaError_t e = cudaMemcpyAsync(h, offsets, (size_t)(S + 1) * sizeof(int64_t), cudaMemcpyDeviceToHost, stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
    if (e != cudaSuccess) return cuda_error("offsets read-back", e);
    if (h[0] != 0) return set_error("%s: offsets[0] = %lld, not 0", fn, (long long)h[0]);
    for (int i = 0; i < S; ++i) {
        if (h[i + 1] < h[i]) return set_error("%s: offsets decrease at scene %d", fn, i);
        if (h[i + 1] - h[i] > n_max)
            return set_error("%s: scene %d has %lld Gaussians, more than %d", fn, i, (long long)(h[i + 1] - h[i]), n_max);
    }
    if (n >= 0 && h[S] != n) return set_error("%s: offsets end at %lld, not at n = %d", fn, (long long)h[S], n);
    return 0;
}

int views_blend(cudaStream_t stream, int V, int P, int image_height, int image_width, size_t capacity,
                const void* geom_state, const void* tile_state, const uint32_t* point_list, void* image_state,
                const float* cams, float* out_color, float* out_others, bool record) {
    const TileLayout tl = tile_layout(image_height, image_width);
    const ImageLayout il = image_layout(image_height, image_width);
    const GeomLayout gl = geom_layout(P);
    RenderFwdArgs r;
    memset(&r, 0, sizeof(r));
    r.W = image_width; r.H = image_height; r.gx = tl.gx; r.gy = tl.gy; r.nviews = V;
    r.capacity = (uint32_t)capacity;
    r.ranges = at<uint2>(tile_state, tl.ranges);
    r.tile_order = at<uint32_t>(tile_state, tl.order);
    r.point_list = point_list;
    r.masks = record ? at<uint32_t>(point_list, plist_masks_offset(capacity)) : nullptr;
    r.rec = P > 0 ? at<float4>(geom_state, gl.rec) : nullptr;
    r.bg = cams + SRF_CAM_BG;
    r.out_color = out_color; r.out_others = out_others;
    if (record) {
        r.accum = at<float>(image_state, il.accum);
        r.n_contrib = at<uint32_t>(image_state, il.ncontrib);
        r.image_stride = il.total;
    }
    r.geom_stride = gl.total; r.tile_stride = tl.total; r.plist_stride = plist_stride_bytes(capacity, record);
    r.cam_stride = SRF_CAM_FLOATS;
    const cudaError_t e = launch_render_fwd(r, record, stream);
    if (e != cudaSuccess) return cuda_error("render_fwd launch", e);
    return 0;
}
}  // namespace srf

extern "C" {

int srf_abi_version(void) { return SRF_ABI_VERSION; }

int srf_profile_begin(void) {
    std::lock_guard<std::mutex> lk(g_prof_mu);
    for (auto& s : g_spans) { g_event_pool.push_back(s.start); g_event_pool.push_back(s.stop); }
    g_spans.clear();
    g_prof_on = true;
    return 0;
}

int srf_profile_end(float* ms_out, int* launches_out, int n) {
    g_prof_on = false;
    std::lock_guard<std::mutex> lk(g_prof_mu);
    if (n < srf::K_COUNT || !ms_out || !launches_out) return set_error("srf_profile_end: need arrays of %d entries", (int)srf::K_COUNT);
    for (int k = 0; k < n; ++k) { ms_out[k] = 0.f; launches_out[k] = 0; }
    for (auto& s : g_spans) {
        cudaError_t e = cudaEventSynchronize(s.stop);
        if (e != cudaSuccess) return cuda_error("profile event sync", e);
        float ms = 0.f;
        e = cudaEventElapsedTime(&ms, s.start, s.stop);
        if (e != cudaSuccess) return cuda_error("profile elapsed", e);
        ms_out[s.kernel] += ms;
        launches_out[s.kernel] += 1;
        g_event_pool.push_back(s.start); g_event_pool.push_back(s.stop);
    }
    g_spans.clear();
    return 0;
}
const char* srf_last_error(void) { return g_err; }

int srf_views_workspace_bytes(int V, int P, int H, int W, size_t capacity, int for_backward, size_t bytes[6]) {
    if (V <= 0 || P < 0 || H <= 0 || W <= 0 || !bytes) return set_error("srf_views_workspace_bytes: bad arguments");
    bytes[0] = geom_layout(P).total * (size_t)V;
    bytes[1] = tile_layout(H, W).total * (size_t)V;
    bytes[2] = for_backward ? image_layout(H, W).total * (size_t)V : 0;
    bytes[3] = entries_stride_bytes(capacity) * (size_t)V;
    bytes[4] = plist_stride_bytes(capacity, for_backward != 0) * (size_t)V;
    bytes[5] = for_backward ? ggrad_stride_bytes(P) * (size_t)V : 0;
    return 0;
}

int srf_state_layout(int P, int H, int W, size_t geom_off[3], size_t tile_off[5], size_t image_off[2]) {
    if (P < 0 || H <= 0 || W <= 0) return set_error("srf_state_layout: bad arguments");
    const GeomLayout g = geom_layout(P);
    const TileLayout t = tile_layout(H, W);
    const ImageLayout i = image_layout(H, W);
    if (geom_off) { geom_off[0] = g.rec; geom_off[1] = g.depths; geom_off[2] = g.rects; }
    if (tile_off) { tile_off[0] = t.count; tile_off[1] = t.counters; tile_off[2] = t.ranges; tile_off[3] = t.count + sizeof(uint32_t); tile_off[4] = t.big; }
    if (image_off) { image_off[0] = i.accum; image_off[1] = i.ncontrib; }
    return 0;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------
// Implementation of the rasterizer's entry points: V views in one launch set, each view's
// camera a record of SRF_CAM_FLOATS floats in `cams`, each view's workspaces one layout stride apart.
// ---------------------------------------------------------------------------------------------
namespace {

void fill_bin_args(srf::BinArgs& b, int V, int P, const TileLayout& tl, void* tile_state) {
    memset(&b, 0, sizeof(b));
    b.P = P; b.nviews = V; b.ntiles = tl.ntiles; b.gx = tl.gx;
    b.tile_count = at<uint32_t>(tile_state, tl.count);
    b.counters = at<uint32_t>(tile_state, tl.counters);
    b.ranges = at<uint2>(tile_state, tl.ranges);
    b.big_list = at<uint32_t>(tile_state, tl.big);
    b.tile_order = at<uint32_t>(tile_state, tl.order);
    b.tile_stride = tl.total;
}

// argument checks of stage 1, all made before it enqueues anything
int forward_preprocess_check(const char* fn, int V, int P, int D, int M,
                             const float* means3D, const float* shs, const float* colors_precomp,
                             const float* opacities, const float* scales, const float* rotations,
                             const float* transMat_precomp, int image_height, int image_width,
                             const int* radii, const void* geom_state, const void* tile_state) {
    if (V <= 0 || P < 0 || image_height <= 0 || image_width <= 0) return set_error("%s: bad sizes", fn);
    if (image_height > 16 * 65535 || image_width > 16 * 65535) return set_error("%s: image too large", fn);
    if (!tile_state || misaligned(tile_state)) return set_error("%s: tile_state must be 256-byte aligned", fn);
    if (D < 0 || D > 3) return set_error("%s: sh degree must be in [0,3]", fn);
    if (P > 0) {
        if (!means3D || !opacities || !radii) return set_error("%s: null required pointer", fn);
        if ((shs == nullptr) == (colors_precomp == nullptr))
            return set_error("Please provide excatly one of either SHs or precomputed colors!");
        if (((scales == nullptr || rotations == nullptr) && transMat_precomp == nullptr) ||
            ((scales != nullptr || rotations != nullptr) && transMat_precomp != nullptr))
            return set_error("Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!");
        if (shs && M < (D + 1) * (D + 1)) return set_error("%s: M=%d SH coefficients < (D+1)^2 for D=%d", fn, M, D);
        if (!geom_state || misaligned(geom_state)) return set_error("%s: geom_state must be 256-byte aligned", fn);
        if ((reinterpret_cast<uintptr_t>(rotations) & 15) || (reinterpret_cast<uintptr_t>(scales) & 7))
            return set_error("%s: rotations must be 16-byte and scales 8-byte aligned", fn);
    }
    return 0;
}

// stage 1: preprocess, per-tile counting, tile scan and the count read-back (arguments checked by the caller)
int forward_preprocess_impl(cudaStream_t stream, int V, int P, int D, int M,
                            const float* means3D, const float* shs, const float* colors_precomp,
                            const float* opacities, const float* scales, const float* rotations,
                            const float* transMat_precomp, const float* cams, const srf::SceneArgs& scenes,
                            int image_height, int image_width,
                            int prefiltered, int* radii, void* geom_state, void* tile_state,
                            uint32_t* num_rendered_host, int raw_activations) {
    const TileLayout tl = tile_layout(image_height, image_width);
    // tile blocks + counters of every view are zeroed by one 2-D memset
    cudaError_t e = cudaMemset2DAsync(at<char>(tile_state, tl.count), tl.total, 0,
                                      tl.counters + 4 * sizeof(uint32_t) - tl.count, (size_t)V, stream);
    if (e != cudaSuccess) return cuda_error("memset tile counters", e);

    srf::BinArgs b;
    fill_bin_args(b, V, P, tl, tile_state);

    if (P > 0) {
        const GeomLayout gl = geom_layout(P);
        srf::PreprocessArgs a;
        memset(&a, 0, sizeof(a));
        a.P = P; a.D = D; a.M = shs ? M : 0; a.nviews = V;
        a.means3D = means3D; a.scales = scales; a.rotations = rotations; a.opacities = opacities;
        a.shs = shs; a.transMat_precomp = transMat_precomp; a.colors_precomp = colors_precomp;
        a.viewmatrix = cams + SRF_CAM_VIEW; a.campos = cams + SRF_CAM_CAMPOS; a.cam_stride = SRF_CAM_FLOATS;
        a.W = image_width; a.H = image_height;
        a.gx = tl.gx; a.gy = tl.gy;
        a.prefiltered = prefiltered;
        a.raw_act = (raw_activations && !transMat_precomp) ? 1 : 0;
        a.radii = radii;
        a.rec = at<float4>(geom_state, gl.rec);
        a.depths = at<float>(geom_state, gl.depths);
        a.rects = at<uint2>(geom_state, gl.rects);
        a.tile_count = b.tile_count;
        a.geom_stride = gl.total;
        a.tile_stride = b.tile_stride;
        e = srf::launch_preprocess_fwd(a, scenes, stream);
        if (e != cudaSuccess) return cuda_error("preprocess_fwd launch", e);
    }
    // num_rendered read-back: pinned host memory is device-visible under UVA, so the scan kernel stores the counts there
    // itself (no copy-engine operation between the kernels of the stream); pageable memory falls back to an async copy
    bool zero_copy = false;
    if (num_rendered_host) {
        cudaPointerAttributes at_;
        if (cudaPointerGetAttributes(&at_, num_rendered_host) == cudaSuccess && at_.type == cudaMemoryTypeHost &&
            at_.devicePointer != nullptr) {
            b.count_host = static_cast<uint32_t*>(at_.devicePointer);
            zero_copy = true;
        } else {
            (void)cudaGetLastError();
        }
    }
    e = srf::launch_tile_scan(b, stream);
    if (e != cudaSuccess) return cuda_error("tile_scan launch", e);
    if (num_rendered_host && !zero_copy) {
        e = cudaMemcpy2DAsync(num_rendered_host, sizeof(uint32_t), b.counters, tl.total, sizeof(uint32_t), (size_t)V,
                              cudaMemcpyDeviceToHost, stream);
        if (e != cudaSuccess) return cuda_error("num_rendered copy", e);
    }
    return 0;
}

// argument checks of stage 2, all made before anything is enqueued; `record` = false (forward-only) needs no image_state
int forward_render_check(const char* fn, int V, int P, int image_height, int image_width, size_t capacity,
                         const void* geom_state, const void* tile_state, const void* entries, const uint32_t* point_list,
                         const void* image_state, const float* cams, const float* out_color, const float* out_others, bool record) {
    if (V <= 0 || P < 0 || image_height <= 0 || image_width <= 0) return set_error("%s: bad sizes", fn);
    if (!cams || !tile_state || (record && !image_state) || !out_color || !out_others)
        return set_error("%s: null required pointer", fn);
    if (capacity > 0xfffffff0ull) return set_error("%s: capacity exceeds 32-bit instance indices", fn);
    if (capacity > 0 && (!entries || !point_list)) return set_error("%s: null binning buffers", fn);
    if (P > 0 && (!geom_state || misaligned(geom_state))) return set_error("%s: geom_state must be 256-byte aligned", fn);
    if (misaligned(tile_state)) return set_error("%s: tile_state must be 256-byte aligned", fn);
    if (capacity > 0 && (misaligned(entries) || misaligned(point_list)))
        return set_error("%s: entries and point_list must be 256-byte aligned", fn);
    return 0;
}

// stage 2: scatter into tile buckets, per-tile depth sort, blend (arguments checked by the caller; record = false: the
// forward-only blend, no contribution record and no image state)
int forward_render_impl(cudaStream_t stream, int V, int P, int image_height, int image_width,
                        size_t capacity, const void* geom_state, void* tile_state,
                        void* entries, uint32_t* point_list, void* image_state,
                        const float* cams, float* out_color, float* out_others, bool record) {
    const TileLayout tl = tile_layout(image_height, image_width);
    const GeomLayout gl = geom_layout(P);

    srf::BinArgs b;
    fill_bin_args(b, V, P, tl, tile_state);
    b.capacity = (uint32_t)capacity;
    b.entries = static_cast<uint64_t*>(entries);
    b.point_list = point_list;
    b.geom_stride = gl.total;
    b.entries_stride = entries_stride_bytes(capacity);
    b.plist_stride = plist_stride_bytes(capacity, record);
    cudaError_t e;
    if (P > 0) {
        // culled Gaussians carry an empty rect, so the radii array is not needed here
        b.depths = at<float>(geom_state, gl.depths);
        b.rects = at<uint2>(geom_state, gl.rects);
        e = srf::launch_bin_and_sort(b, stream);
        if (e != cudaSuccess) return cuda_error("binning launch", e);
    }
    return srf::views_blend(stream, V, P, image_height, image_width, capacity, geom_state, tile_state, point_list,
                            image_state, cams, out_color, out_others, record);
}

int backward_impl(const char* fn, cudaStream_t stream, int V, int P, int D, int M, int image_height, int image_width,
                  size_t capacity, const float* cams,
                  const float* means3D, const float* shs, int colors_were_precomputed,
                  const float* scales, const float* rotations, int transmat_was_precomputed,
                  const int* radii,
                  const void* geom_state, const void* tile_state, const uint32_t* point_list,
                  const void* image_state,
                  const float* dL_dout_color, const float* dL_dout_others,
                  void* scratch, int accumulate,
                  float* dL_dmeans3D, float* dL_dmeans2D, float* dL_dsh, float* dL_dcolors,
                  float* dL_dopacity, float* dL_dscales, float* dL_drotations, float* dL_dtransMat,
                  int raw_activations, bool deterministic, const srf::SceneArgs& scenes, int S) {
    if (!cams) return set_error("%s: null camera records", fn);
    if (V <= 0 || P < 0 || image_height <= 0 || image_width <= 0) return set_error("%s: bad sizes", fn);
    if (P == 0) return 0;
    if (!geom_state || !tile_state || !image_state || !scratch || !radii) return set_error("%s: null state pointer", fn);
    if (!dL_dout_color || !dL_dout_others) return set_error("%s: null upstream gradient", fn);
    if (!dL_dmeans3D || !dL_dopacity || !dL_dscales || !dL_drotations)
        return set_error("%s: null required output gradient", fn);
    if (!means3D) return set_error("%s: null input pointer", fn);
    if (!transmat_was_precomputed && (!scales || !rotations)) return set_error("%s: scales/rotations required", fn);
    if (misaligned(scratch)) return set_error("%s: scratch must be 256-byte aligned", fn);
    const TileLayout tl = tile_layout(image_height, image_width);
    const ImageLayout il = image_layout(image_height, image_width);
    const GeomLayout gl = geom_layout(P);
    const size_t gstride = ggrad_stride_bytes(P);

    // deterministic: the fixed-point records and the flag behind the fp32 records are zeroed, the fp32 records written
    void* det = at<void>(scratch, gstride * (size_t)V);
    const size_t dstride = det_stride_bytes(P);
    uint32_t* overflow = at<uint32_t>(det, dstride * (size_t)V);
    cudaError_t e = deterministic ? cudaMemsetAsync(det, 0, dstride * (size_t)V + sizeof(uint32_t), stream)
                                  : cudaMemsetAsync(scratch, 0, gstride * (size_t)V, stream);
    if (e != cudaSuccess) return cuda_error("memset gradient records", e);

    srf::RenderBwdArgs r;
    memset(&r, 0, sizeof(r));
    r.W = image_width; r.H = image_height; r.gx = tl.gx; r.gy = tl.gy; r.nviews = V;
    r.capacity = (uint32_t)capacity;
    r.ranges = at<uint2>(tile_state, tl.ranges);
    r.tile_order = at<uint32_t>(tile_state, tl.order);
    r.point_list = point_list;
    r.masks = at<const uint32_t>(point_list, plist_masks_offset(capacity));
    r.rec = at<float4>(geom_state, gl.rec);
    r.bg = cams + SRF_CAM_BG;
    r.accum = at<float>(image_state, il.accum);
    r.n_contrib = at<uint32_t>(image_state, il.ncontrib);
    r.dL_dpix = dL_dout_color;
    r.dL_dothers = dL_dout_others;
    r.ggrad = static_cast<float*>(scratch);
    r.geom_stride = gl.total; r.tile_stride = tl.total; r.plist_stride = plist_stride_bytes(capacity, true);
    r.image_stride = il.total; r.ggrad_stride = gstride;
    r.cam_stride = SRF_CAM_FLOATS;
    if (deterministic) {
        srf::RenderBwdArgs rd = r;
        rd.ggrad = static_cast<float*>(det);
        rd.ggrad_stride = dstride;
        e = srf::launch_render_bwd_det(rd, P, r.ggrad, gstride, overflow, stream);
    } else {
        e = srf::launch_render_bwd(r, stream);
    }
    if (e != cudaSuccess) return cuda_error("render_bwd launch", e);

    srf::PreprocessBwdArgs p;
    memset(&p, 0, sizeof(p));
    p.P = P; p.D = D; p.M = (shs && !colors_were_precomputed) ? M : 0;
    p.means3D = means3D; p.scales = scales; p.rotations = rotations;
    p.shs = colors_were_precomputed ? nullptr : shs;
    p.viewmatrix = cams + SRF_CAM_VIEW; p.campos = cams + SRF_CAM_CAMPOS; p.cam_stride = SRF_CAM_FLOATS;
    p.has_precomp_T = transmat_was_precomputed ? 1 : 0;
    p.has_precomp_color = colors_were_precomputed ? 1 : 0;
    p.raw_act = (raw_activations && !transmat_was_precomputed) ? 1 : 0;
    p.radii = radii;
    p.rec = r.rec;
    p.ggrad = r.ggrad;
    p.geom_stride = r.geom_stride; p.ggrad_stride = r.ggrad_stride;
    p.accumulate = accumulate ? 1 : 0;
    p.dL_dmeans3D = dL_dmeans3D; p.dL_dmeans2D = dL_dmeans2D;
    p.dL_dsh = p.M > 0 ? dL_dsh : nullptr;
    p.dL_dcolors = dL_dcolors; p.dL_dopacity = dL_dopacity;
    p.dL_dscales = dL_dscales; p.dL_drotations = dL_drotations; p.dL_dtransMat = dL_dtransMat;
    e = srf::launch_preprocess_bwd(p, scenes, S, stream);
    if (e != cudaSuccess) return cuda_error("preprocess_bwd launch", e);
    return deterministic ? srf::check_overflow_flag(fn, overflow, stream) : 0;
}

}  // namespace

extern "C" {

int srf_views_forward_render(srf_stream_t stream_, int V, int P, int image_height, int image_width,
                             size_t capacity, const void* geom_state, void* tile_state,
                             void* entries, uint32_t* point_list, void* image_state,
                             const float* cams, float* out_color, float* out_others, int for_backward) {
    if (forward_render_check("srf_views_forward_render", V, P, image_height, image_width, capacity, geom_state,
                             tile_state, entries, point_list, image_state, cams, out_color, out_others, for_backward != 0))
        return 1;
    return forward_render_impl(static_cast<cudaStream_t>(stream_), V, P, image_height, image_width, capacity, geom_state,
                               tile_state, entries, point_list, image_state, cams, out_color, out_others,
                               for_backward != 0);
}

int srf_scenes_forward(srf_stream_t stream_, int S, int Vs, int P, int D, int M,
                       const float* means3D, const float* shs, const float* colors_precomp,
                       const float* opacities, const float* scales, const float* rotations,
                       const float* transMat_precomp, const float* cams, const float* tan_fov,
                       int image_height, int image_width, int prefiltered,
                       size_t capacity, int* radii, void* geom_state, void* tile_state, void* entries,
                       uint32_t* point_list, void* image_state, float* out_color, float* out_others,
                       uint32_t* num_rendered_host, void* count_event, int raw_activations, int for_backward) {
    const char* fn = "srf_scenes_forward";
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    srf::SceneArgs scenes;
    if (srf::check_scenes(fn, S, Vs) || srf::scene_fov(fn, S, tan_fov, image_height, image_width, scenes)) return 1;
    scenes.views_per_scene = Vs;
    scenes.offsets = nullptr;
    const int V = S * Vs;
    if (forward_preprocess_check(fn, V, P, D, M, means3D, shs, colors_precomp, opacities, scales, rotations,
                                 transMat_precomp, image_height, image_width, radii, geom_state, tile_state) ||
        forward_render_check(fn, V, P, image_height, image_width, capacity, geom_state, tile_state, entries, point_list,
                             image_state, cams, out_color, out_others, for_backward != 0))
        return 1;
    if ((size_t)S * P > 0x7fffffffull) return set_error("%s: S * P exceeds 32-bit Gaussian indices", fn);
    int rc = forward_preprocess_impl(stream, V, P, D, M, means3D, shs, colors_precomp, opacities, scales, rotations,
                                     transMat_precomp, cams, scenes, image_height, image_width, prefiltered, radii,
                                     geom_state, tile_state, num_rendered_host, raw_activations);
    if (rc != 0) return rc;
    if (count_event) {      // lets the caller wait for the instance counts without waiting for the blend
        cudaError_t e = cudaEventRecord(static_cast<cudaEvent_t>(count_event), stream);
        if (e != cudaSuccess) return cuda_error("count event record", e);
    }
    return forward_render_impl(stream, V, P, image_height, image_width, capacity, geom_state, tile_state, entries,
                               point_list, image_state, cams, out_color, out_others, for_backward != 0);
}

int srf_scenes_backward(srf_stream_t stream_, int S, int Vs, int P, const int64_t* offsets, int D, int M,
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
                        int raw_activations, int deterministic) {
    const char* fn = "srf_scenes_backward";
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    srf::SceneArgs scenes;
    if (srf::check_scenes(fn, S, Vs) || srf::scene_fov(fn, S, tan_fov, image_height, image_width, scenes)) return 1;
    if (P < 0) return set_error("%s: bad sizes", fn);
    if (!offsets && (size_t)S * P > 0x7fffffffull) return set_error("%s: S * P exceeds 32-bit Gaussian indices", fn);
    if (offsets && P > 0 && srf::check_offsets(fn, stream, S, offsets, P, -1)) return 1;
    scenes.views_per_scene = Vs;
    scenes.offsets = offsets;
    return backward_impl(fn, stream, S * Vs, P, D, M, image_height, image_width, capacity, cams, means3D, shs,
                         colors_were_precomputed, scales, rotations, transmat_was_precomputed, radii, geom_state,
                         tile_state, point_list, image_state, dL_dout_color, dL_dout_others, scratch, accumulate,
                         dL_dmeans3D, dL_dmeans2D, dL_dsh, dL_dcolors, dL_dopacity, dL_dscales, dL_drotations,
                         dL_dtransMat, raw_activations, deterministic != 0, scenes, S);
}

int srf_views_backward_deterministic_scratch_bytes(int V, int P, size_t* bytes) {
    if (V <= 0 || P < 0 || !bytes) return set_error("srf_views_backward_deterministic_scratch_bytes: bad arguments");
    *bytes = det_scratch_bytes(V, P);
    return 0;
}

int srf_mark_visible(srf_stream_t stream_, int P, const float* means3D,
                     const float* viewmatrix, const float* projmatrix, uint8_t* present) {
    (void)projmatrix;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (P < 0) return set_error("srf_mark_visible: bad P");
    if (P == 0) return 0;
    if (!means3D || !viewmatrix || !present) return set_error("srf_mark_visible: null pointer");
    cudaError_t e = srf::launch_mark_visible(P, means3D, viewmatrix, present, stream);
    if (e != cudaSuccess) return cuda_error("mark_visible launch", e);
    return 0;
}

}  // extern "C"
