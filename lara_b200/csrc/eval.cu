// eval.cu -- LaRa's per-scene evaluation on the GPU (evaluation.py:83-141): the novel-view metric sums and the
// turntable video's uint8 frames.  The C entries of include/surfel_eval.h are defined here.
//
// eval_metrics_kernel : a fixed grid of kGrid CTAs strides over the view range's pixels (squared colour error) and
//                       over all pixels of the depth maps (masked absolute error, count, threshold counts).  Each
//                       thread accumulates in fp64 (counts in 64-bit integers), each CTA reduces in a fixed order and
//                       writes one record of partials.
// part_sums_kernel    : sums the kGrid records in CTA order (fixed_sums.cuh).  No atomics: two identical calls give
//                       identical bits.
// video_frames_kernel : one thread per frame pixel, LaRa's rounding chain with every operation rounded on its own.
#include <math.h>
#include <string.h>

#include "../../include/surfel_eval.h"
#include "fixed_sums.cuh"
#include "surfel_common.cuh"
#include "surfel_kernels.h"

namespace srf {
namespace {

constexpr int kThreads = 256;
constexpr int kGrid = 264;                        // fixed, so that the reduction order does not depend on the device
constexpr int kSums = 3 + SRF_EVAL_MAX_THRESHOLDS;

// element (c, y, x) of a logical [1,C,H,X] image; column x lies in view x / wv at column x % wv
struct Addr { long long sc, sy, sx, sv; int wv; };

__device__ __forceinline__ long long at(const Addr& a, int c, int y, int x) {
    const int v = x / a.wv;
    return c * a.sc + y * a.sy + v * a.sv + (x - v * a.wv) * a.sx;
}

struct MetricArgs {
    int H, VW, x0, nx;            // image columns [x0, x0 + nx) of the H x VW image
    int nthr;
    float thr[SRF_EVAL_MAX_THRESHOLDS];
    const float* img; const float* tar; Addr ai, at;
    const float* dep; const float* dgt; const uint8_t* msk; Addr ad, ag, am;
    double* part;                 // [kGrid][kSums]
    double* out;
};

__global__ void __launch_bounds__(kThreads) eval_metrics_kernel(const MetricArgs a) {
    double sq = 0.0, ab = 0.0;
    unsigned long long cnt = 0, acc[SRF_EVAL_MAX_THRESHOLDS] = {};
    const long long stride = (long long)kGrid * kThreads;
    const long long nc = (long long)a.H * a.nx, nd = a.dep ? (long long)a.H * a.VW : 0;
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < nc; i += stride) {
        const int y = (int)(i / a.nx), x = a.x0 + (int)(i - (long long)y * a.nx);
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float d = __fsub_rn(__ldg(a.img + at(a.ai, c, y, x)), __ldg(a.tar + at(a.at, c, y, x)));
            sq += (double)__fmul_rn(d, d);
        }
    }
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < nd; i += stride) {
        const int y = (int)(i / a.VW), x = (int)(i - (long long)y * a.VW);
        if (!__ldg(a.msk + at(a.am, 0, y, x))) continue;
        const float e = fabsf(__fsub_rn(__ldg(a.dep + at(a.ad, 0, y, x)), __ldg(a.dgt + at(a.ag, 0, y, x))));
        ab += (double)e;
        ++cnt;
#pragma unroll
        for (int t = 0; t < SRF_EVAL_MAX_THRESHOLDS; ++t)
            if (t < a.nthr && e < a.thr[t]) ++acc[t];
    }
    double v[kSums];
    v[0] = sq; v[1] = ab; v[2] = (double)cnt;
#pragma unroll
    for (int t = 0; t < SRF_EVAL_MAX_THRESHOLDS; ++t) v[3 + t] = (double)acc[t];
    __shared__ double s_w[kThreads / 32][kSums];
#pragma unroll
    for (int k = 0; k < kSums; ++k) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
    }
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int k = 0; k < kSums; ++k) s_w[threadIdx.x >> 5][k] = v[k];
    }
    __syncthreads();
    if (threadIdx.x < kSums) {
        double s = 0.0;
#pragma unroll
        for (int w = 0; w < kThreads / 32; ++w) s += s_w[w][threadIdx.x];
        a.part[(size_t)blockIdx.x * kSums + threadIdx.x] = s;
    }
}

struct FrameArgs {
    int N, H, W;
    const float* img; const float* nrm; const float* alp;
    long long ib, nb, ab;         // frame strides
    Addr ai, an, aa;
    uint8_t* rgb; uint8_t* out_nrm;
};

// np.round (half to even) of an fp32 value, then a saturating cast to uint8 (NaN -> 0)
__device__ __forceinline__ uint8_t to_u8(float v) {
    const float r = fminf(fmaxf(rintf(v), 0.f), 255.f);
    return (uint8_t)(int)r;
}

__global__ void __launch_bounds__(kThreads) video_frames_kernel(const FrameArgs a) {
    const long long HW = (long long)a.H * a.W;
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i >= (long long)a.N * HW) return;
    const int n = (int)(i / HW), p = (int)(i - n * HW), y = p / a.W, x = p - y * a.W;
    if (a.img) {
        const float* s = a.img + n * a.ib;
#pragma unroll
        for (int c = 0; c < 3; ++c) a.rgb[3 * i + c] = to_u8(__fmul_rn(__ldg(s + at(a.ai, c, y, x)), 255.f));
    }
    if (a.nrm) {
        const float* s = a.nrm + n * a.nb;
        const float al = __ldg(a.alp + n * a.ab + at(a.aa, 0, y, x));
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            float t = __fmul_rn(__ldg(s + at(a.an, c, y, x)), al);    // normal * alpha
            t = __fadd_rn(t, 1.f);                                     // + 1
            t = __fsub_rn(t, al);                                      // - alpha
            t = __fadd_rn(t, 1.f);                                     // + 1
            t = __fmul_rn(t, 0.5f);                                    // / 2 (exact, as the division is)
            a.out_nrm[3 * i + c] = to_u8(__fmul_rn(t, 255.f));
        }
    }
}

int to_addr(const char* fn, const char* what, const void* p, const srf_ms_ssim_addr* a, int elem, Addr* out,
            long long* sb = nullptr) {
    if (!p || !a) return set_error("%s: null %s pointer", fn, what);
    if (reinterpret_cast<uintptr_t>(p) & (elem - 1)) return set_error("%s: %s must be %d-byte aligned", fn, what, elem);
    if (a->wv <= 0 || a->wv > 0x7fffffff) return set_error("%s: %s view width %lld out of range", fn, what, (long long)a->wv);
    out->sc = a->sc; out->sy = a->sy; out->sx = a->sx; out->sv = a->sv; out->wv = (int)a->wv;
    if (sb) *sb = a->sb;
    return 0;
}

}  // namespace
}  // namespace srf

using srf::set_error;

extern "C" int srf_eval_workspace_bytes(size_t* bytes) {
    if (!bytes) return set_error("srf_eval_workspace_bytes: null pointer");
    *bytes = srf::align_up((size_t)srf::kGrid * srf::kSums * sizeof(double));
    return 0;
}

extern "C" int srf_eval_metrics(srf_stream_t stream_, int V, int H, int W, int v0, int v1,
                                const float* image, const srf_ms_ssim_addr* image_addr,
                                const float* target, const srf_ms_ssim_addr* target_addr,
                                const float* depth, const srf_ms_ssim_addr* depth_addr,
                                const float* depth_gt, const srf_ms_ssim_addr* depth_gt_addr,
                                const uint8_t* mask, const srf_ms_ssim_addr* mask_addr,
                                int n_thresholds, const double* thresholds, void* workspace, double* out) {
    using namespace srf;
    const char* fn = "srf_eval_metrics";
    if (V <= 0 || H <= 0 || W <= 0) return set_error("%s: bad sizes (V=%d, H=%d, W=%d)", fn, V, H, W);
    if ((long long)V * W > 0x7fffffffLL || (long long)H * V * W * 3 > 0x7fffffffLL)
        return set_error("%s: bad sizes: 3 H V W = %lld exceeds 2^31", fn, 3LL * H * V * W);
    if (v0 < 0 || v0 > v1 || v1 > V) return set_error("%s: bad view range [%d, %d) of V = %d", fn, v0, v1, V);
    if (n_thresholds < 0 || n_thresholds > SRF_EVAL_MAX_THRESHOLDS)
        return set_error("%s: n_thresholds = %d out of [0, %d]", fn, n_thresholds, SRF_EVAL_MAX_THRESHOLDS);
    MetricArgs a;
    memset(&a, 0, sizeof(a));
    if (to_addr(fn, "image", image, image_addr, 4, &a.ai) || to_addr(fn, "target", target, target_addr, 4, &a.at))
        return 1;
    if (depth) {
        if (to_addr(fn, "depth", depth, depth_addr, 4, &a.ad) || to_addr(fn, "depth_gt", depth_gt, depth_gt_addr, 4, &a.ag)
            || to_addr(fn, "mask", mask, mask_addr, 1, &a.am))
            return 1;
        if (n_thresholds && !thresholds) return set_error("%s: null thresholds", fn);
        for (int t = 0; t < n_thresholds; ++t) a.thr[t] = (float)thresholds[t];
        a.nthr = n_thresholds;
    }
    if (!workspace || misaligned(workspace)) return set_error("%s: workspace must be 256-byte aligned", fn);
    if (!out || (reinterpret_cast<uintptr_t>(out) & 7)) return set_error("%s: out must be 8-byte aligned", fn);
    a.H = H; a.VW = V * W; a.x0 = v0 * W; a.nx = (v1 - v0) * W;
    a.img = image; a.tar = target; a.dep = depth; a.dgt = depth_gt; a.msk = mask;
    a.part = static_cast<double*>(workspace);
    a.out = out;
    const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    eval_metrics_kernel<<<kGrid, kThreads, 0, stream>>>(a);
    part_sums(stream, a.part, kGrid, kSums, seg(out, 3 + n_thresholds));
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_error("eval_metrics launch", e);
}

extern "C" int srf_video_frames(srf_stream_t stream_, int N, int H, int W,
                                const float* image, const srf_ms_ssim_addr* image_addr,
                                const float* normal, const srf_ms_ssim_addr* normal_addr,
                                const float* alpha, const srf_ms_ssim_addr* alpha_addr,
                                uint8_t* rgb, uint8_t* nrm) {
    using namespace srf;
    const char* fn = "srf_video_frames";
    if (N < 0 || H <= 0 || W <= 0) return set_error("%s: bad sizes (N=%d, H=%d, W=%d)", fn, N, H, W);
    if ((long long)N * H * W * 3 > 0x7fffffffLL) return set_error("%s: bad sizes: 3 N H W exceeds 2^31", fn);
    FrameArgs a;
    memset(&a, 0, sizeof(a));
    a.N = N; a.H = H; a.W = W;
    if (image) {
        if (to_addr(fn, "image", image, image_addr, 4, &a.ai, &a.ib)) return 1;
        if (!rgb) return set_error("%s: null rgb output", fn);
        a.img = image; a.rgb = rgb;
    }
    if (normal) {
        if (to_addr(fn, "normal", normal, normal_addr, 4, &a.an, &a.nb) ||
            to_addr(fn, "alpha", alpha, alpha_addr, 4, &a.aa, &a.ab))
            return 1;
        if (!nrm) return set_error("%s: null nrm output", fn);
        a.nrm = normal; a.alp = alpha; a.out_nrm = nrm;
    }
    const long long n = (long long)N * H * W;
    if (n == 0 || (!a.img && !a.nrm)) return 0;
    const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    video_frames_kernel<<<(unsigned)((n + kThreads - 1) / kThreads), kThreads, 0, stream>>>(a);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_error("video_frames launch", e);
}
