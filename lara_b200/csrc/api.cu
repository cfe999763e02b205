// api.cu -- the extern "C" boundary declared in include/surfel_rasterizer.h.
// Plain pointers and sizes in, int status out; only enqueues work on the given stream.
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <mutex>
#include <vector>

#include "../../include/surfel_rasterizer.h"
#include "surfel_common.cuh"
#include "surfel_kernels.h"

namespace {

thread_local char g_err[512] = "";

int fail(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return 1;
}

int cuda_fail(const char* what, cudaError_t e) {
    return fail("%s: %s", what, cudaGetErrorString(e));
}

inline size_t align_up(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }

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

bool misaligned(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 255) != 0; }

// One view's point_list workspace: the depth-sorted list (u32 [capacity]), then the blend forward's contribution
// masks (u32 [8 warp blocks][capacity], indexed by list position), which the blend backward replays.
size_t plist_masks_offset(size_t capacity) { return align_up(capacity * sizeof(uint32_t)); }
size_t plist_stride_bytes(size_t capacity) {
    return plist_masks_offset(capacity) + align_up(capacity * 8 * sizeof(uint32_t)) + 256;
}

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
    if (n < srf::K_COUNT || !ms_out || !launches_out) return fail("srf_profile_end: need arrays of %d entries", (int)srf::K_COUNT);
    for (int k = 0; k < n; ++k) { ms_out[k] = 0.f; launches_out[k] = 0; }
    for (auto& s : g_spans) {
        cudaError_t e = cudaEventSynchronize(s.stop);
        if (e != cudaSuccess) return cuda_fail("profile event sync", e);
        float ms = 0.f;
        e = cudaEventElapsedTime(&ms, s.start, s.stop);
        if (e != cudaSuccess) return cuda_fail("profile elapsed", e);
        ms_out[s.kernel] += ms;
        launches_out[s.kernel] += 1;
        g_event_pool.push_back(s.start); g_event_pool.push_back(s.stop);
    }
    g_spans.clear();
    return 0;
}
const char* srf_last_error(void) { return g_err; }

int srf_geom_state_bytes(int P, size_t* bytes) {
    if (P < 0 || !bytes) return fail("srf_geom_state_bytes: bad arguments");
    *bytes = geom_layout(P).total;
    return 0;
}

int srf_tile_state_bytes(int H, int W, size_t* bytes) {
    if (H <= 0 || W <= 0 || !bytes) return fail("srf_tile_state_bytes: bad arguments");
    *bytes = tile_layout(H, W).total;
    return 0;
}

int srf_image_state_bytes(int H, int W, size_t* bytes) {
    if (H <= 0 || W <= 0 || !bytes) return fail("srf_image_state_bytes: bad arguments");
    *bytes = image_layout(H, W).total;
    return 0;
}

int srf_binning_bytes(size_t capacity, size_t* entries_bytes, size_t* point_list_bytes) {
    if (!entries_bytes || !point_list_bytes) return fail("srf_binning_bytes: bad arguments");
    *entries_bytes = align_up(capacity * sizeof(uint64_t)) + 256;
    *point_list_bytes = plist_stride_bytes(capacity);
    return 0;
}

int srf_backward_scratch_bytes(int P, size_t* bytes) {
    if (P < 0 || !bytes) return fail("srf_backward_scratch_bytes: bad arguments");
    *bytes = align_up((size_t)P * SRF_GRAD_FLOATS * sizeof(float)) + 256;
    return 0;
}

int srf_state_layout(int P, int H, int W, size_t geom_off[3], size_t tile_off[5], size_t image_off[2]) {
    if (P < 0 || H <= 0 || W <= 0) return fail("srf_state_layout: bad arguments");
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
// Implementation shared by the per-view entry points (the reference's interface, one view per call)
// and the srf_views_* entry points (all V target views of one scene in one launch set).
// ---------------------------------------------------------------------------------------------
namespace {

struct Cams {               // per-view camera data: three pointers into records `stride` floats apart
    const float* view;
    const float* campos;
    const float* bg;
    size_t stride;
};

size_t entries_stride_bytes(size_t capacity) { return align_up(capacity * sizeof(uint64_t)) + 256; }
size_t ggrad_stride_bytes(int P) { return align_up((size_t)P * SRF_GRAD_FLOATS * sizeof(float)) + 256; }

void fill_bin_args(srf::BinArgs& b, int V, int P, const TileLayout& tl, void* tile_state) {
    memset(&b, 0, sizeof(b));
    b.P = P; b.nviews = V; b.ntiles = tl.ntiles; b.gx = tl.gx;
    b.tile_count = at<uint32_t>(tile_state, tl.count);
    b.counters = at<uint32_t>(tile_state, tl.counters);
    b.ranges = at<uint2>(tile_state, tl.ranges);
    b.big_list = at<uint32_t>(tile_state, tl.big);
    b.tile_order = at<uint32_t>(tile_state, tl.order);
    b.tile_stride = V > 1 ? tl.total : 0;
}

int forward_preprocess_impl(const char* fn, cudaStream_t stream, int V, int P, int D, int M,
                            const float* means3D, const float* shs, const float* colors_precomp,
                            const float* opacities, const float* scales, const float* rotations,
                            const float* transMat_precomp, Cams cams,
                            float tan_fovx, float tan_fovy, int image_height, int image_width,
                            int prefiltered, int* radii, void* geom_state, void* tile_state,
                            uint32_t* num_rendered_host, int raw_activations) {
    if (V <= 0 || P < 0 || image_height <= 0 || image_width <= 0) return fail("%s: bad sizes", fn);
    if (image_height > 16 * 65535 || image_width > 16 * 65535) return fail("%s: image too large", fn);
    if (!tile_state || misaligned(tile_state)) return fail("%s: tile_state must be 256-byte aligned", fn);
    if (D < 0 || D > 3) return fail("%s: sh degree must be in [0,3]", fn);
    const TileLayout tl = tile_layout(image_height, image_width);
    // tile blocks + counters of every view are zeroed by one 2-D memset
    cudaError_t e = cudaMemset2DAsync(at<char>(tile_state, tl.count), tl.total, 0,
                                      tl.counters + 4 * sizeof(uint32_t) - tl.count, (size_t)V, stream);
    if (e != cudaSuccess) return cuda_fail("memset tile counters", e);

    srf::BinArgs b;
    fill_bin_args(b, V, P, tl, tile_state);

    if (P > 0) {
        if (!means3D || !opacities || !cams.view || !cams.campos || !radii)
            return fail("%s: null required pointer", fn);
        if ((shs == nullptr) == (colors_precomp == nullptr))
            return fail("Please provide excatly one of either SHs or precomputed colors!");
        if (((scales == nullptr || rotations == nullptr) && transMat_precomp == nullptr) ||
            ((scales != nullptr || rotations != nullptr) && transMat_precomp != nullptr))
            return fail("Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!");
        if (shs && M < (D + 1) * (D + 1)) return fail("%s: M=%d SH coefficients < (D+1)^2 for D=%d", fn, M, D);
        if (!geom_state || misaligned(geom_state)) return fail("%s: geom_state must be 256-byte aligned", fn);
        if ((reinterpret_cast<uintptr_t>(rotations) & 15) || (reinterpret_cast<uintptr_t>(scales) & 7))
            return fail("%s: rotations must be 16-byte and scales 8-byte aligned", fn);
        const GeomLayout gl = geom_layout(P);
        srf::PreprocessArgs a;
        memset(&a, 0, sizeof(a));
        a.P = P; a.D = D; a.M = shs ? M : 0; a.nviews = V;
        a.means3D = means3D; a.scales = scales; a.rotations = rotations; a.opacities = opacities;
        a.shs = shs; a.transMat_precomp = transMat_precomp; a.colors_precomp = colors_precomp;
        a.viewmatrix = cams.view; a.campos = cams.campos; a.cam_stride = cams.stride;
        a.W = image_width; a.H = image_height;
        a.focal_y = image_height / (2.0f * tan_fovy);   // rasterizer_impl.cu:223-224
        a.focal_x = image_width / (2.0f * tan_fovx);
        a.gx = tl.gx; a.gy = tl.gy;
        a.prefiltered = prefiltered;
        a.raw_act = (raw_activations && !transMat_precomp) ? 1 : 0;
        a.radii = radii;
        a.rec = at<float4>(geom_state, gl.rec);
        a.depths = at<float>(geom_state, gl.depths);
        a.rects = at<uint2>(geom_state, gl.rects);
        a.tile_count = b.tile_count;
        a.geom_stride = V > 1 ? gl.total : 0;
        a.tile_stride = b.tile_stride;
        e = srf::launch_preprocess_fwd(a, stream);
        if (e != cudaSuccess) return cuda_fail("preprocess_fwd launch", e);
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
    if (e != cudaSuccess) return cuda_fail("tile_scan launch", e);
    if (num_rendered_host && !zero_copy) {
        e = cudaMemcpy2DAsync(num_rendered_host, sizeof(uint32_t), b.counters, tl.total, sizeof(uint32_t), (size_t)V,
                              cudaMemcpyDeviceToHost, stream);
        if (e != cudaSuccess) return cuda_fail("num_rendered copy", e);
    }
    return 0;
}

int forward_render_impl(const char* fn, cudaStream_t stream, int V, int P, int image_height, int image_width,
                        size_t capacity, const void* geom_state, void* tile_state,
                        void* entries, uint32_t* point_list, void* image_state,
                        const float* background, size_t cam_stride, float* out_color, float* out_others) {
    if (V <= 0 || P < 0 || image_height <= 0 || image_width <= 0) return fail("%s: bad sizes", fn);
    if (!tile_state || !image_state || !background || !out_color || !out_others)
        return fail("%s: null required pointer", fn);
    if (capacity > 0xfffffff0ull) return fail("%s: capacity exceeds 32-bit instance indices", fn);
    if (capacity > 0 && (!entries || !point_list)) return fail("%s: null binning buffers", fn);
    const TileLayout tl = tile_layout(image_height, image_width);
    const ImageLayout il = image_layout(image_height, image_width);
    const GeomLayout gl = geom_layout(P);

    srf::BinArgs b;
    fill_bin_args(b, V, P, tl, tile_state);
    b.capacity = (uint32_t)capacity;
    b.entries = static_cast<uint64_t*>(entries);
    b.point_list = point_list;
    b.geom_stride = V > 1 ? gl.total : 0;
    b.entries_stride = V > 1 ? entries_stride_bytes(capacity) : 0;
    b.plist_stride = V > 1 ? plist_stride_bytes(capacity) : 0;
    cudaError_t e;
    if (P > 0) {
        if (!geom_state) return fail("%s: null geom_state", fn);
        // culled Gaussians carry an empty rect, so the radii array is not needed here
        b.depths = at<float>(geom_state, gl.depths);
        b.rects = at<uint2>(geom_state, gl.rects);
        e = srf::launch_bin_and_sort(b, stream);
        if (e != cudaSuccess) return cuda_fail("binning launch", e);
    }
    srf::RenderFwdArgs r;
    memset(&r, 0, sizeof(r));
    r.W = image_width; r.H = image_height; r.gx = tl.gx; r.gy = tl.gy; r.nviews = V;
    r.capacity = (uint32_t)capacity;
    r.ranges = b.ranges;
    r.tile_order = b.tile_order;
    r.point_list = point_list;
    r.masks = at<uint32_t>(point_list, plist_masks_offset(capacity));
    r.rec = P > 0 ? at<float4>(geom_state, gl.rec) : nullptr;
    r.bg = background;
    r.out_color = out_color; r.out_others = out_others;
    r.accum = at<float>(image_state, il.accum);
    r.n_contrib = at<uint32_t>(image_state, il.ncontrib);
    r.geom_stride = b.geom_stride; r.tile_stride = b.tile_stride; r.plist_stride = b.plist_stride;
    r.image_stride = V > 1 ? il.total : 0;
    r.cam_stride = cam_stride;
    e = srf::launch_render_fwd(r, stream);
    if (e != cudaSuccess) return cuda_fail("render_fwd launch", e);
    return 0;
}

int backward_impl(const char* fn, cudaStream_t stream, int V, int P, int D, int M, int image_height, int image_width,
                  size_t capacity, Cams cams,
                  const float* means3D, const float* shs, int colors_were_precomputed,
                  const float* scales, const float* rotations, int transmat_was_precomputed,
                  float tan_fovx, float tan_fovy, const int* radii,
                  const void* geom_state, const void* tile_state, const uint32_t* point_list,
                  const void* image_state,
                  const float* dL_dout_color, const float* dL_dout_others,
                  void* scratch, int accumulate,
                  float* dL_dmeans3D, float* dL_dmeans2D, float* dL_dsh, float* dL_dcolors,
                  float* dL_dopacity, float* dL_dscales, float* dL_drotations, float* dL_dtransMat,
                  int raw_activations) {
    if (V <= 0 || P < 0 || image_height <= 0 || image_width <= 0) return fail("%s: bad sizes", fn);
    if (P == 0) return 0;
    if (!geom_state || !tile_state || !image_state || !scratch || !radii || !cams.bg)
        return fail("%s: null state pointer", fn);
    if (!dL_dout_color || !dL_dout_others) return fail("%s: null upstream gradient", fn);
    if (!dL_dmeans3D || !dL_dopacity || !dL_dscales || !dL_drotations)
        return fail("%s: null required output gradient", fn);
    if (!means3D || !cams.view || !cams.campos) return fail("%s: null input pointer", fn);
    if (!transmat_was_precomputed && (!scales || !rotations)) return fail("%s: scales/rotations required", fn);
    if (misaligned(scratch)) return fail("%s: scratch must be 256-byte aligned", fn);
    const TileLayout tl = tile_layout(image_height, image_width);
    const ImageLayout il = image_layout(image_height, image_width);
    const GeomLayout gl = geom_layout(P);
    const size_t gstride = ggrad_stride_bytes(P);

    cudaError_t e = cudaMemsetAsync(scratch, 0, V > 1 ? gstride * (size_t)V : (size_t)P * SRF_GRAD_FLOATS * sizeof(float), stream);
    if (e != cudaSuccess) return cuda_fail("memset gradient records", e);

    srf::RenderBwdArgs r;
    memset(&r, 0, sizeof(r));
    r.W = image_width; r.H = image_height; r.gx = tl.gx; r.gy = tl.gy; r.nviews = V;
    r.capacity = (uint32_t)capacity;
    r.ranges = at<uint2>(tile_state, tl.ranges);
    r.tile_order = at<uint32_t>(tile_state, tl.order);
    r.point_list = point_list;
    r.masks = at<const uint32_t>(point_list, plist_masks_offset(capacity));
    r.rec = at<float4>(geom_state, gl.rec);
    r.bg = cams.bg;
    r.accum = at<float>(image_state, il.accum);
    r.n_contrib = at<uint32_t>(image_state, il.ncontrib);
    r.dL_dpix = dL_dout_color;
    r.dL_dothers = dL_dout_others;
    r.ggrad = static_cast<float*>(scratch);
    if (V > 1) {
        r.geom_stride = gl.total; r.tile_stride = tl.total; r.plist_stride = plist_stride_bytes(capacity);
        r.image_stride = il.total; r.ggrad_stride = gstride;
    }
    r.cam_stride = cams.stride;
    e = srf::launch_render_bwd(r, stream);
    if (e != cudaSuccess) return cuda_fail("render_bwd launch", e);

    srf::PreprocessBwdArgs p;
    memset(&p, 0, sizeof(p));
    p.P = P; p.D = D; p.M = (shs && !colors_were_precomputed) ? M : 0; p.nviews = V;
    p.means3D = means3D; p.scales = scales; p.rotations = rotations;
    p.shs = colors_were_precomputed ? nullptr : shs;
    p.viewmatrix = cams.view; p.campos = cams.campos; p.cam_stride = cams.stride;
    p.W = image_width; p.H = image_height;
    p.focal_y = image_height / (2.0f * tan_fovy);
    p.focal_x = image_width / (2.0f * tan_fovx);
    p.tan_fovx = tan_fovx; p.tan_fovy = tan_fovy;
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
    e = srf::launch_preprocess_bwd(p, stream);
    if (e != cudaSuccess) return cuda_fail("preprocess_bwd launch", e);
    return 0;
}

Cams cams_of(const float* cams) {
    Cams c;
    c.view = cams; c.campos = cams ? cams + SRF_CAM_CAMPOS : nullptr; c.bg = cams ? cams + SRF_CAM_BG : nullptr;
    c.stride = SRF_CAM_FLOATS;
    return c;
}

}  // namespace

extern "C" {

int srf_forward_preprocess(srf_stream_t stream_, int P, int D, int M,
                           const float* means3D, const float* shs, const float* colors_precomp,
                           const float* opacities, const float* scales, float scale_modifier,
                           const float* rotations, const float* transMat_precomp,
                           const float* viewmatrix, const float* projmatrix, const float* campos,
                           float tan_fovx, float tan_fovy, int image_height, int image_width,
                           int prefiltered, int* radii, void* geom_state, void* tile_state,
                           uint32_t* num_rendered_host, int raw_activations) {
    (void)scale_modifier; (void)projmatrix;
    Cams c; c.view = viewmatrix; c.campos = campos; c.bg = nullptr; c.stride = 0;
    return forward_preprocess_impl("srf_forward_preprocess", static_cast<cudaStream_t>(stream_), 1, P, D, M, means3D, shs,
                                   colors_precomp, opacities, scales, rotations, transMat_precomp, c, tan_fovx, tan_fovy,
                                   image_height, image_width, prefiltered, radii, geom_state, tile_state,
                                   num_rendered_host, raw_activations);
}

int srf_forward_render(srf_stream_t stream_, int P, int image_height, int image_width,
                       size_t capacity, const void* geom_state, void* tile_state,
                       void* entries, uint32_t* point_list, void* image_state,
                       const float* background, float* out_color, float* out_others) {
    return forward_render_impl("srf_forward_render", static_cast<cudaStream_t>(stream_), 1, P, image_height, image_width,
                               capacity, geom_state, tile_state, entries, point_list, image_state, background, 0,
                               out_color, out_others);
}

int srf_backward(srf_stream_t stream_, int P, int D, int M, int image_height, int image_width,
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
                 int raw_activations) {
    (void)projmatrix;
    Cams c; c.view = viewmatrix; c.campos = campos; c.bg = background; c.stride = 0;
    return backward_impl("srf_backward", static_cast<cudaStream_t>(stream_), 1, P, D, M, image_height, image_width, capacity, c,
                         means3D, shs, colors_were_precomputed, scales, rotations, transmat_was_precomputed,
                         tan_fovx, tan_fovy, radii, geom_state, tile_state, point_list, image_state,
                         dL_dout_color, dL_dout_others, scratch, accumulate, dL_dmeans3D, dL_dmeans2D, dL_dsh, dL_dcolors,
                         dL_dopacity, dL_dscales, dL_drotations, dL_dtransMat, raw_activations);
}

// both forward stages in one call (one host->library transition per view in the drop-in path)
int srf_forward(srf_stream_t stream_, int P, int D, int M,
                const float* means3D, const float* shs, const float* colors_precomp,
                const float* opacities, const float* scales, float scale_modifier,
                const float* rotations, const float* transMat_precomp,
                const float* viewmatrix, const float* projmatrix, const float* campos,
                float tan_fovx, float tan_fovy, int image_height, int image_width, int prefiltered,
                const float* background, size_t capacity,
                int* radii, void* geom_state, void* tile_state, void* entries, uint32_t* point_list, void* image_state,
                float* out_color, float* out_others, uint32_t* num_rendered_host, void* count_event, int raw_activations) {
    int rc = srf_forward_preprocess(stream_, P, D, M, means3D, shs, colors_precomp, opacities, scales, scale_modifier, rotations,
                                    transMat_precomp, viewmatrix, projmatrix, campos, tan_fovx, tan_fovy, image_height,
                                    image_width, prefiltered, radii, geom_state, tile_state, num_rendered_host, raw_activations);
    if (rc != 0) return rc;
    if (count_event) {      // lets the caller wait for the instance count without waiting for the blend
        cudaError_t e = cudaEventRecord(static_cast<cudaEvent_t>(count_event), static_cast<cudaStream_t>(stream_));
        if (e != cudaSuccess) return cuda_fail("count event record", e);
    }
    return srf_forward_render(stream_, P, image_height, image_width, capacity, geom_state, tile_state, entries, point_list,
                              image_state, background, out_color, out_others);
}

// ---- all V target views of one scene in one launch set (reference caller loop: lightning/network.py:484-497)
int srf_views_workspace_bytes(int V, int P, int H, int W, size_t capacity, size_t bytes[6]) {
    if (V <= 0 || P < 0 || H <= 0 || W <= 0 || !bytes) return fail("srf_views_workspace_bytes: bad arguments");
    bytes[0] = geom_layout(P).total * (size_t)V;
    bytes[1] = tile_layout(H, W).total * (size_t)V;
    bytes[2] = image_layout(H, W).total * (size_t)V;
    bytes[3] = entries_stride_bytes(capacity) * (size_t)V;
    bytes[4] = plist_stride_bytes(capacity) * (size_t)V;
    bytes[5] = ggrad_stride_bytes(P) * (size_t)V;
    return 0;
}

int srf_views_forward_preprocess(srf_stream_t stream_, int V, int P, int D, int M,
                                 const float* means3D, const float* shs, const float* colors_precomp,
                                 const float* opacities, const float* scales, const float* rotations,
                                 const float* transMat_precomp, const float* cams,
                                 float tan_fovx, float tan_fovy, int image_height, int image_width,
                                 int prefiltered, int* radii, void* geom_state, void* tile_state,
                                 uint32_t* num_rendered_host, int raw_activations) {
    if (!cams) return fail("srf_views_forward_preprocess: null camera records");
    return forward_preprocess_impl("srf_views_forward_preprocess", static_cast<cudaStream_t>(stream_), V, P, D, M, means3D,
                                   shs, colors_precomp, opacities, scales, rotations, transMat_precomp, cams_of(cams),
                                   tan_fovx, tan_fovy, image_height, image_width, prefiltered, radii, geom_state,
                                   tile_state, num_rendered_host, raw_activations);
}

int srf_views_forward_render(srf_stream_t stream_, int V, int P, int image_height, int image_width,
                             size_t capacity, const void* geom_state, void* tile_state,
                             void* entries, uint32_t* point_list, void* image_state,
                             const float* cams, float* out_color, float* out_others) {
    if (!cams) return fail("srf_views_forward_render: null camera records");
    return forward_render_impl("srf_views_forward_render", static_cast<cudaStream_t>(stream_), V, P, image_height,
                               image_width, capacity, geom_state, tile_state, entries, point_list, image_state,
                               cams + SRF_CAM_BG, SRF_CAM_FLOATS, out_color, out_others);
}

int srf_views_backward(srf_stream_t stream_, int V, int P, int D, int M, int image_height, int image_width,
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
                       int raw_activations) {
    if (!cams) return fail("srf_views_backward: null camera records");
    return backward_impl("srf_views_backward", static_cast<cudaStream_t>(stream_), V, P, D, M, image_height, image_width,
                         capacity, cams_of(cams), means3D, shs, colors_were_precomputed, scales, rotations,
                         transmat_was_precomputed, tan_fovx, tan_fovy, radii, geom_state, tile_state, point_list,
                         image_state, dL_dout_color, dL_dout_others, scratch, accumulate, dL_dmeans3D, dL_dmeans2D,
                         dL_dsh, dL_dcolors, dL_dopacity, dL_dscales, dL_drotations, dL_dtransMat, raw_activations);
}

static int epilogue_forward_impl(const char* fn, cudaStream_t stream, int V, int image_height, int image_width,
                                 float depth_ratio, const float* color, const float* allmap, const float* rays,
                                 const float* viewmatrix, size_t cam_stride, float* image, float* depth, float* acc_map,
                                 float* rend_normal, float* depth_normal, float* rend_dist) {
    if (V <= 0 || image_height <= 0 || image_width <= 0) return fail("%s: bad sizes", fn);
    if (!color || !allmap || !viewmatrix || !image || !depth || !acc_map || !rend_normal || !depth_normal || !rend_dist)
        return fail("%s: null pointer", fn);
    srf::EpilogueArgs a;
    memset(&a, 0, sizeof(a));
    a.W = image_width; a.H = image_height; a.nviews = V; a.depth_ratio = depth_ratio;
    a.color = color; a.allmap = allmap; a.rays = rays; a.viewmatrix = viewmatrix; a.cam_stride = cam_stride;
    a.image = image; a.depth = depth; a.acc = acc_map; a.rend_normal = rend_normal; a.depth_normal = depth_normal;
    a.dist = rend_dist;
    cudaError_t e = srf::launch_epilogue_fwd(a, stream);
    if (e != cudaSuccess) return cuda_fail("epilogue_fwd launch", e);
    return 0;
}

static int epilogue_backward_impl(const char* fn, cudaStream_t stream, int V, int image_height, int image_width,
                                  float depth_ratio, const float* color, const float* allmap, const float* rays,
                                  const float* viewmatrix, size_t cam_stride,
                                  const float* g_image, const float* g_depth, const float* g_acc_map,
                                  const float* g_rend_normal, const float* g_depth_normal, const float* g_rend_dist,
                                  float* scratch, float* dL_dcolor, float* dL_dallmap) {
    if (V <= 0 || image_height <= 0 || image_width <= 0) return fail("%s: bad sizes", fn);
    if (!color || !allmap || !viewmatrix || !dL_dcolor || !dL_dallmap) return fail("%s: null pointer", fn);
    if (g_depth_normal && rays && !scratch) return fail("%s: scratch [V,3,H,W] required", fn);
    srf::EpilogueArgs a;
    memset(&a, 0, sizeof(a));
    a.W = image_width; a.H = image_height; a.nviews = V; a.depth_ratio = depth_ratio;
    a.color = color; a.allmap = allmap; a.rays = rays; a.viewmatrix = viewmatrix; a.cam_stride = cam_stride;
    a.g_image = g_image; a.g_depth = g_depth; a.g_acc = g_acc_map; a.g_rend_normal = g_rend_normal;
    a.g_depth_normal = g_depth_normal; a.g_dist = g_rend_dist;
    a.scratch = scratch; a.dL_dcolor = dL_dcolor; a.dL_dallmap = dL_dallmap;
    cudaError_t e = srf::launch_epilogue_bwd(a, stream);
    if (e != cudaSuccess) return cuda_fail("epilogue_bwd launch", e);
    return 0;
}

int srf_epilogue_forward(srf_stream_t stream_, int image_height, int image_width, float depth_ratio,
                         const float* color, const float* allmap, const float* rays, const float* viewmatrix,
                         float* image, float* depth, float* acc_map, float* rend_normal, float* depth_normal,
                         float* rend_dist) {
    return epilogue_forward_impl("srf_epilogue_forward", static_cast<cudaStream_t>(stream_), 1, image_height, image_width,
                                 depth_ratio, color, allmap, rays, viewmatrix, 0, image, depth, acc_map, rend_normal,
                                 depth_normal, rend_dist);
}

int srf_epilogue_backward(srf_stream_t stream_, int image_height, int image_width, float depth_ratio,
                          const float* color, const float* allmap, const float* rays, const float* viewmatrix,
                          const float* g_image, const float* g_depth, const float* g_acc_map,
                          const float* g_rend_normal, const float* g_depth_normal, const float* g_rend_dist,
                          float* scratch, float* dL_dcolor, float* dL_dallmap) {
    return epilogue_backward_impl("srf_epilogue_backward", static_cast<cudaStream_t>(stream_), 1, image_height, image_width,
                                  depth_ratio, color, allmap, rays, viewmatrix, 0, g_image, g_depth, g_acc_map,
                                  g_rend_normal, g_depth_normal, g_rend_dist, scratch, dL_dcolor, dL_dallmap);
}

int srf_views_epilogue_forward(srf_stream_t stream_, int V, int image_height, int image_width, float depth_ratio,
                               const float* color, const float* allmap, const float* rays, const float* cams,
                               float* image, float* depth, float* acc_map, float* rend_normal, float* depth_normal,
                               float* rend_dist) {
    return epilogue_forward_impl("srf_views_epilogue_forward", static_cast<cudaStream_t>(stream_), V, image_height,
                                 image_width, depth_ratio, color, allmap, rays, cams, SRF_CAM_FLOATS, image, depth, acc_map,
                                 rend_normal, depth_normal, rend_dist);
}

int srf_views_epilogue_backward(srf_stream_t stream_, int V, int image_height, int image_width, float depth_ratio,
                                const float* color, const float* allmap, const float* rays, const float* cams,
                                const float* g_image, const float* g_depth, const float* g_acc_map,
                                const float* g_rend_normal, const float* g_depth_normal, const float* g_rend_dist,
                                float* scratch, float* dL_dcolor, float* dL_dallmap) {
    return epilogue_backward_impl("srf_views_epilogue_backward", static_cast<cudaStream_t>(stream_), V, image_height,
                                  image_width, depth_ratio, color, allmap, rays, cams, SRF_CAM_FLOATS, g_image, g_depth,
                                  g_acc_map, g_rend_normal, g_depth_normal, g_rend_dist, scratch, dL_dcolor, dL_dallmap);
}

int srf_loss_forward(srf_stream_t stream_, int V, int image_height, int image_width, int with_reg,
                     const float* image, const float* target_hwc, const float* rend_normal, const float* depth_normal,
                     const float* acc_map, const float* rend_dist, double* sums) {
    if (V <= 0 || image_height <= 0 || image_width <= 0) return fail("srf_loss_forward: bad sizes");
    if (!image || !target_hwc || !sums) return fail("srf_loss_forward: null pointer");
    if (with_reg && (!rend_normal || !depth_normal || !acc_map || !rend_dist)) return fail("srf_loss_forward: null regulariser input");
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    cudaError_t e = cudaMemsetAsync(sums, 0, 3 * sizeof(double), stream);
    if (e != cudaSuccess) return cuda_fail("memset loss sums", e);
    srf::LossArgs a;
    memset(&a, 0, sizeof(a));
    a.W = image_width; a.H = image_height; a.nviews = V; a.with_reg = with_reg ? 1 : 0;
    a.image = image; a.target = target_hwc; a.rend_normal = rend_normal; a.depth_normal = depth_normal;
    a.acc = acc_map; a.dist = rend_dist; a.sums = sums;
    e = srf::launch_loss_fused(a, stream);
    if (e != cudaSuccess) return cuda_fail("loss_sums launch", e);
    return 0;
}

int srf_loss_backward(srf_stream_t stream_, int V, int image_height, int image_width, int with_reg,
                      float w_mse, float w_dist, float w_normal,
                      const float* image, const float* target_hwc, const float* rend_normal, const float* depth_normal,
                      const float* acc_map, const float* upstream,
                      float* g_image, float* g_rend_normal, float* g_depth_normal, float* g_rend_dist) {
    if (V <= 0 || image_height <= 0 || image_width <= 0) return fail("srf_loss_backward: bad sizes");
    if (!image || !target_hwc || !g_image) return fail("srf_loss_backward: null pointer");
    if (with_reg && (!rend_normal || !depth_normal || !acc_map || !g_rend_normal || !g_depth_normal || !g_rend_dist))
        return fail("srf_loss_backward: null regulariser pointer");
    srf::LossArgs a;
    memset(&a, 0, sizeof(a));
    a.W = image_width; a.H = image_height; a.nviews = V; a.with_reg = with_reg ? 1 : 0;
    a.w_mse = w_mse; a.w_dist = w_dist; a.w_normal = w_normal;
    a.image = image; a.target = target_hwc; a.rend_normal = rend_normal; a.depth_normal = depth_normal; a.acc = acc_map;
    a.gout = upstream;
    a.g_image = g_image; a.g_rend_normal = g_rend_normal; a.g_depth_normal = g_depth_normal; a.g_dist = g_rend_dist;
    cudaError_t e = srf::launch_loss_fused(a, static_cast<cudaStream_t>(stream_));
    if (e != cudaSuccess) return cuda_fail("loss_grads launch", e);
    return 0;
}

int srf_decoder_layout_forward(srf_stream_t stream_, size_t B, int N, int K, int sh_dim,
                               float opacity_shift, float scaling_shift, float half_cell_size,
                               const float* params, const float* group_centers,
                               float* centers, float* shs, float* opacity, float* scaling, float* rotation) {
    if (N <= 0 || K <= 0 || sh_dim < 3 || sh_dim % 3 != 0) return fail("srf_decoder_layout_forward: bad sizes");
    if (!params || !group_centers || !centers || !shs || !opacity || !scaling || !rotation)
        return fail("srf_decoder_layout_forward: null pointer");
    if ((reinterpret_cast<uintptr_t>(rotation) & 15) || (reinterpret_cast<uintptr_t>(scaling) & 7) ||
        ((sh_dim & 3) == 0 && (reinterpret_cast<uintptr_t>(shs) & 15)))
        return fail("srf_decoder_layout_forward: outputs must be 16-byte aligned");
    srf::DecoderArgs a;
    memset(&a, 0, sizeof(a));
    a.total = B * (size_t)N * (size_t)K; a.N = N; a.K = K; a.C = 10 + sh_dim; a.sh_dim = sh_dim;
    a.opacity_shift = opacity_shift; a.scaling_shift = scaling_shift; a.half_cell = half_cell_size;
    a.params = params; a.group_centers = group_centers;
    a.centers = centers; a.shs = shs; a.opacity = opacity; a.scaling = scaling; a.rotation = rotation;
    cudaError_t e = srf::launch_decoder_layout(a, false, static_cast<cudaStream_t>(stream_));
    if (e != cudaSuccess) return cuda_fail("decoder_layout launch", e);
    return 0;
}

int srf_decoder_layout_backward(srf_stream_t stream_, size_t B, int N, int K, int sh_dim, float half_cell_size,
                                const float* params, const float* g_centers, const float* g_shs, const float* g_opacity,
                                const float* g_scaling, const float* g_rotation, float* g_params) {
    if (N <= 0 || K <= 0 || sh_dim < 3 || sh_dim % 3 != 0) return fail("srf_decoder_layout_backward: bad sizes");
    if (!params || !g_params) return fail("srf_decoder_layout_backward: null pointer");
    srf::DecoderArgs a;
    memset(&a, 0, sizeof(a));
    a.total = B * (size_t)N * (size_t)K; a.N = N; a.K = K; a.C = 10 + sh_dim; a.sh_dim = sh_dim;
    a.half_cell = half_cell_size;
    a.params = params;
    a.g_centers = g_centers; a.g_shs = g_shs; a.g_opacity = g_opacity; a.g_scaling = g_scaling; a.g_rotation = g_rotation;
    a.g_params = g_params;
    cudaError_t e = srf::launch_decoder_layout(a, true, static_cast<cudaStream_t>(stream_));
    if (e != cudaSuccess) return cuda_fail("decoder_layout backward launch", e);
    return 0;
}

static int point_feats_check(const char* fn, int V, int n, int H, int W, const float* points, const float* w2cs,
                             const float* ixts, const float* img_ref, const float* image, const float* acc,
                             const float* depth) {
    if (V <= 0 || n < 0 || H <= 0 || W <= 0) return fail("%s: bad sizes (V=%d, n=%d, H=%d, W=%d)", fn, V, n, H, W);
    if (H > (1 << 24) || W > (1 << 24)) return fail("%s: image too large", fn);    // pixel indices exact in fp32
    // an empty point set has no storage: points (and feats / g_feats) are only needed when n > 0
    if ((n > 0 && !points) || !w2cs || !ixts || !img_ref || !image || !acc || !depth) return fail("%s: null input pointer", fn);
    return 0;
}

int srf_point_feats_forward(srf_stream_t stream_, int V, int n, int H, int W,
                            const float* points, const float* w2cs, const float* ixts,
                            const float* img_ref, const float* image, const float* acc, const float* depth,
                            float* feats) {
    const char* fn = "srf_point_feats_forward";
    if (point_feats_check(fn, V, n, H, W, points, w2cs, ixts, img_ref, image, acc, depth)) return 1;
    if (n > 0 && !feats) return fail("%s: null output pointer", fn);
    if (n == 0) return 0;
    srf::PointFeatsArgs a;
    memset(&a, 0, sizeof(a));
    a.V = V; a.n = n; a.H = H; a.W = W;
    a.points = points; a.w2cs = w2cs; a.ixts = ixts; a.img_ref = img_ref; a.image = image; a.acc = acc; a.depth = depth;
    a.feats = feats;
    cudaError_t e = srf::launch_point_feats(a, false, static_cast<cudaStream_t>(stream_));
    if (e != cudaSuccess) return cuda_fail("point_feats_fwd launch", e);
    return 0;
}

int srf_point_feats_backward(srf_stream_t stream_, int V, int n, int H, int W,
                             const float* points, const float* w2cs, const float* ixts,
                             const float* img_ref, const float* image, const float* acc, const float* depth,
                             const float* g_feats, float* g_points, float* g_image, float* g_acc, float* g_depth) {
    const char* fn = "srf_point_feats_backward";
    if (point_feats_check(fn, V, n, H, W, points, w2cs, ixts, img_ref, image, acc, depth)) return 1;
    if (n > 0 && !g_feats) return fail("%s: null upstream gradient", fn);
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const size_t plane = (size_t)V * H * W * sizeof(float);
    cudaError_t e = cudaSuccess;
    if (g_image && (e = cudaMemsetAsync(g_image, 0, 3 * plane, stream)) != cudaSuccess) return cuda_fail("memset g_image", e);
    if (g_acc && (e = cudaMemsetAsync(g_acc, 0, plane, stream)) != cudaSuccess) return cuda_fail("memset g_acc", e);
    if (g_depth && (e = cudaMemsetAsync(g_depth, 0, plane, stream)) != cudaSuccess) return cuda_fail("memset g_depth", e);
    if (n == 0 || (!g_points && !g_image && !g_acc && !g_depth)) return 0;
    srf::PointFeatsArgs a;
    memset(&a, 0, sizeof(a));
    a.V = V; a.n = n; a.H = H; a.W = W;
    a.points = points; a.w2cs = w2cs; a.ixts = ixts; a.img_ref = img_ref; a.image = image; a.acc = acc; a.depth = depth;
    a.g_feats = g_feats; a.g_points = g_points; a.g_image = g_image; a.g_acc = g_acc; a.g_depth = g_depth;
    e = srf::launch_point_feats(a, true, stream);
    if (e != cudaSuccess) return cuda_fail("point_feats_bwd launch", e);
    return 0;
}

int srf_mark_visible(srf_stream_t stream_, int P, const float* means3D,
                     const float* viewmatrix, const float* projmatrix, uint8_t* present) {
    (void)projmatrix;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (P < 0) return fail("srf_mark_visible: bad P");
    if (P == 0) return 0;
    if (!means3D || !viewmatrix || !present) return fail("srf_mark_visible: null pointer");
    cudaError_t e = srf::launch_mark_visible(P, means3D, viewmatrix, present, stream);
    if (e != cudaSuccess) return cuda_fail("mark_visible launch", e);
    return 0;
}

}  // extern "C"
