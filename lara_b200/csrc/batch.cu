// batch.cu -- LaRa's training batch on the GPU (dataLoader/gobjverse.py:40-141, dataLoader/utils.py:21-34): the C entry
// of include/surfel_batch.h.
//
// batch_assemble_kernel: the first `rows * chunks` CTAs each take kPix consecutive pixels of one image row (scene b,
// view n, row y), one pixel per thread.  The 12-byte colour and normal and the 24-byte ray of each pixel are staged in
// shared memory, then leave as 128-bit stores: every output run of a CTA is contiguous (tar_nrm's [H, N W, 3] layout
// keeps one view's row segment contiguous too), and the staging buffer is offset so that it has the destination's
// alignment modulo 16 bytes, leaving at most three scalar stores at each end.  The remaining CTAs write the
// H/16 x W/16 rays of tar_rays_down, one pixel per thread.
//
// Every value is rounded as LaRa's NumPy lines round it: fp32 operations through __f*_rn (no FMA contraction where
// NumPy rounds twice), the rays in fp64 with one rounding to fp32.  Each product XYZ_j * i2w[j][i] is exact in fp64
// (a half-integer of at most 24 bits times a 24-bit significand), so the rays equal NumPy's bit for bit wherever the
// three-term fp64 sum is exact, whatever order BLAS sums in.
#include <string.h>

#include "../../include/surfel_batch.h"
#include "surfel_common.cuh"
#include "surfel_kernels.h"

namespace srf {
namespace {

constexpr int kThreads = 256;
constexpr int kPix = kThreads;        // pixels per CTA of the full-resolution part
constexpr int kDown = 16;             // LaRa's tar_rays_down scale, 1/16

struct AssembleArgs {
    int N, H, W, Hd, Wd, chunks;
    long long main_ctas, n_down;      // CTAs of the full-resolution part; pixels of tar_rays_down
    const uint32_t* rgba; const uint8_t* nrm_in;
    const float* bg; const float* i2w; const float* i2w_d; const float* org; const float* rot;
    float* rgb; uint8_t* msk; float* nrm; float* rays; float* rays_d;
};

// staging buffer of `count` floats for destination `dst`: the first float sits at the index with dst's alignment
__device__ __forceinline__ int stage_shift(const float* dst) {
    return (int)((reinterpret_cast<uintptr_t>(dst) >> 2) & 3);
}

// copy s[0, n) (shared, with dst's alignment modulo 16) to dst[0, n): scalar head and tail, 128-bit body
__device__ __forceinline__ void flush(float* dst, const float* s, int n) {
    const int head = min((4 - stage_shift(dst)) & 3, n);
    const int nv = (n - head) >> 2;
    float4* d4 = reinterpret_cast<float4*>(dst + head);
    const float4* s4 = reinterpret_cast<const float4*>(s + head);
    if ((int)threadIdx.x < head) dst[threadIdx.x] = s[threadIdx.x];
    for (int i = threadIdx.x; i < nv; i += kThreads) d4[i] = s4[i];
    const int t0 = head + 4 * nv;
    if (t0 + (int)threadIdx.x < n) dst[t0 + threadIdx.x] = s[t0 + threadIdx.x];
}

// fp32(sum_j XYZ_j m[3 j + i]) for XYZ = (X, Y, 1), the products exact in fp64, summed j = 0, 1, 2
__device__ __forceinline__ float ray_dir(const float* m, int i, double X, double Y) {
    const double s = __dadd_rn(__dmul_rn(X, (double)__ldg(m + i)), __dmul_rn(Y, (double)__ldg(m + 3 + i)));
    return __double2float_rn(__dadd_rn(s, (double)__ldg(m + 6 + i)));
}

__device__ __forceinline__ float unit_u8(unsigned v) { return __fdiv_rn((float)v, 255.f); }    // fp32(v / 255)

__device__ void down_rays(const AssembleArgs& a, long long q) {
    if (q >= a.n_down) return;
    const long long HWd = (long long)a.Hd * a.Wd;
    const long long view = q / HWd;
    const int p = (int)(q - view * HWd), y = p / a.Wd, x = p - y * a.Wd;
    const float* m = a.i2w_d + view * 9;
    const float* o = a.org + view * 3;
    float* r = a.rays_d + q * 6;
    const double X = (double)x + 0.5, Y = (double)y + 0.5;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        r[i] = __ldg(o + i);
        r[3 + i] = ray_dir(m, i, X, Y);
    }
}

__global__ void __launch_bounds__(kThreads) batch_assemble_kernel(const AssembleArgs a) {
    __shared__ __align__(16) float s_rgb[kPix * 3 + 4];
    __shared__ __align__(16) float s_nrm[kPix * 3 + 4];
    __shared__ __align__(16) float s_ray[kPix * 6 + 4];
    if ((long long)blockIdx.x >= a.main_ctas) {       // uniform per CTA: no barrier below is skipped by part of it
        down_rays(a, ((long long)blockIdx.x - a.main_ctas) * kThreads + threadIdx.x);
        return;
    }
    const long long row = (long long)blockIdx.x / a.chunks;         // (view, y), view = b N + n
    const int x0 = (int)((long long)blockIdx.x - row * a.chunks) * kPix;
    const int npx = min(kPix, a.W - x0);
    const long long view = row / a.H;
    const int y = (int)(row - view * a.H);
    const long long b = view / a.N;
    const int n = (int)(view - b * a.N);
    const long long p0 = row * a.W + x0;                            // first pixel of the CTA in [B,N,H,W]

    float* d_rgb = a.rgb + p0 * 3;
    float* d_ray = a.rays + p0 * 6;
    float* d_nrm = a.nrm ? a.nrm + (((b * a.H + y) * a.N + n) * a.W + x0) * 3 : nullptr;
    float* st_rgb = s_rgb + stage_shift(d_rgb);
    float* st_ray = s_ray + stage_shift(d_ray);
    float* st_nrm = s_nrm + (d_nrm ? stage_shift(d_nrm) : 0);

    const int t = threadIdx.x;
    if (t < npx) {
        const long long p = p0 + t;
        const uint32_t px = __ldg(a.rgba + p);
        const unsigned au = px >> 24;
        const float al = unit_u8(au), om = __fsub_rn(1.f, al);
        const float* bg = a.bg + view * 3;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float col = unit_u8((px >> (8 * c)) & 255u);
            st_rgb[3 * t + c] = __fadd_rn(__fmul_rn(col, al), __fmul_rn(__ldg(bg + c), om));
        }
        a.msk[p] = au > 0;
        if (d_nrm) {
            const uint8_t* s = a.nrm_in + p * 3;
            double nv[3];
#pragma unroll
            for (int j = 0; j < 3; ++j) nv[j] = (double)__fsub_rn(__fmul_rn(unit_u8(__ldg(s + j)), 2.f), 1.f);
            const float* R = a.rot + b * 9;
#pragma unroll
            for (int i = 0; i < 3; ++i) {        // (n R^T)_i = sum_j n_j R[i][j]
                const double v = __dadd_rn(__dadd_rn(__dmul_rn(nv[0], (double)__ldg(R + 3 * i)),
                                                     __dmul_rn(nv[1], (double)__ldg(R + 3 * i + 1))),
                                           __dmul_rn(nv[2], (double)__ldg(R + 3 * i + 2)));
                st_nrm[3 * t + i] = __double2float_rn(v);
            }
        }
        const float* m = a.i2w + view * 9;
        const float* o = a.org + view * 3;
        const double X = (double)(x0 + t) + 0.5, Y = (double)y + 0.5;
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            st_ray[6 * t + i] = __ldg(o + i);
            st_ray[6 * t + 3 + i] = ray_dir(m, i, X, Y);
        }
    }
    __syncthreads();
    flush(d_rgb, st_rgb, npx * 3);
    flush(d_ray, st_ray, npx * 6);
    if (d_nrm) flush(d_nrm, st_nrm, npx * 3);
}

// One camera record per view (include/surfel_batch.h): the 4x4 inverse by cofactors of 2x2 minors, all in fp64, each
// element divided by the fp64 determinant and rounded once to fp32.
__global__ void __launch_bounds__(kThreads) batch_cameras_kernel(int n, const float* __restrict__ c2w,
                                                                 const float* __restrict__ bg, float* __restrict__ cams) {
    const int v = blockIdx.x * kThreads + threadIdx.x;
    if (v >= n) return;
    const float* m = c2w + (size_t)v * 16;
    double a[16];
    bool finite = true;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
        const float x = __ldg(m + i);
        finite = finite && isfinite(x);
        a[i] = (double)x;
    }
    const double s0 = a[0] * a[5] - a[4] * a[1], s1 = a[0] * a[6] - a[4] * a[2], s2 = a[0] * a[7] - a[4] * a[3];
    const double s3 = a[1] * a[6] - a[5] * a[2], s4 = a[1] * a[7] - a[5] * a[3], s5 = a[2] * a[7] - a[6] * a[3];
    const double c5 = a[10] * a[15] - a[14] * a[11], c4 = a[9] * a[15] - a[13] * a[11], c3 = a[9] * a[14] - a[13] * a[10];
    const double c2 = a[8] * a[15] - a[12] * a[11], c1 = a[8] * a[14] - a[12] * a[10], c0 = a[8] * a[13] - a[12] * a[9];
    const double det = s0 * c5 - s1 * c4 + s2 * c3 + s3 * c2 - s4 * c1 + s5 * c0;
    float* r = cams + (size_t)v * SRF_CAM_FLOATS;
    if (!finite || !(fabs(det) >= 1e-12)) {
        // every finite point lands at view depth -1, behind the near plane: the view renders its background only
#pragma unroll
        for (int i = 0; i < SRF_CAM_BG; ++i) r[i] = 0.f;
        r[SRF_CAM_VIEW + 14] = -1.f;
        r[SRF_CAM_VIEW + 15] = 1.f;
    } else {
        const double inv[16] = {
            a[5] * c5 - a[6] * c4 + a[7] * c3,   -a[1] * c5 + a[2] * c4 - a[3] * c3,
            a[13] * s5 - a[14] * s4 + a[15] * s3, -a[9] * s5 + a[10] * s4 - a[11] * s3,
            -a[4] * c5 + a[6] * c2 - a[7] * c1,  a[0] * c5 - a[2] * c2 + a[3] * c1,
            -a[12] * s5 + a[14] * s2 - a[15] * s1, a[8] * s5 - a[10] * s2 + a[11] * s1,
            a[4] * c4 - a[5] * c2 + a[7] * c0,   -a[0] * c4 + a[1] * c2 - a[3] * c0,
            a[12] * s4 - a[13] * s2 + a[15] * s0, -a[8] * s4 + a[9] * s2 - a[11] * s0,
            -a[4] * c3 + a[5] * c1 - a[6] * c0,  a[0] * c3 - a[1] * c1 + a[2] * c0,
            -a[12] * s3 + a[13] * s1 - a[14] * s0, a[8] * s3 - a[9] * s1 + a[10] * s0};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) r[SRF_CAM_VIEW + 4 * i + j] = __double2float_rn(inv[4 * j + i] / det);   // w2c^T
#pragma unroll
        for (int i = 0; i < 3; ++i) r[SRF_CAM_CAMPOS + i] = -__ldg(m + 4 * i + 3);
    }
#pragma unroll
    for (int i = 0; i < 3; ++i) r[SRF_CAM_BG + i] = __ldg(bg + (size_t)v * 3 + i);
#pragma unroll
    for (int i = SRF_CAM_BG + 3; i < SRF_CAM_FLOATS; ++i) r[i] = 0.f;
}

int check_ptr(const char* fn, const char* what, const void* p, int align) {
    if (!p) return set_error("%s: null %s pointer", fn, what);
    if (reinterpret_cast<uintptr_t>(p) & (align - 1)) return set_error("%s: %s must be %d-byte aligned", fn, what, align);
    return 0;
}

}  // namespace
}  // namespace srf

using srf::set_error;

extern "C" int srf_batch_assemble(srf_stream_t stream_, int B, int N, int H, int W,
                                  const uint8_t* rgba, const uint8_t* normal, const float* bg,
                                  const float* i2w, const float* i2w_down, const float* origin, const float* nrm_rot,
                                  float* tar_rgb, uint8_t* tar_msk, float* tar_nrm, float* tar_rays,
                                  float* tar_rays_down) {
    using namespace srf;
    const char* fn = "srf_batch_assemble";
    if (B <= 0 || N <= 0 || H <= 0 || W <= 0) return set_error("%s: bad sizes (B=%d, N=%d, H=%d, W=%d)", fn, B, N, H, W);
    if (H < kDown || W < kDown)
        return set_error("%s: bad sizes: H = %d and W = %d must be at least %d (the 1/%d rays would be empty)", fn, H, W,
                         kDown, kDown);
    const long long views = (long long)B * N, chunks = (W + kPix - 1) / kPix;
    const long long main_ctas = views * H * chunks, n_down = views * (H / kDown) * (W / kDown);
    const long long ctas = main_ctas + (n_down + kThreads - 1) / kThreads;
    if (views * H * W * 6 > (1LL << 40) || ctas > 0x7fffffffLL)
        return set_error("%s: bad sizes: B N H W = %lld pixels is too large", fn, views * H * W);
    if (check_ptr(fn, "rgba", rgba, 4) || check_ptr(fn, "bg", bg, 4) || check_ptr(fn, "i2w", i2w, 4) ||
        check_ptr(fn, "i2w_down", i2w_down, 4) || check_ptr(fn, "origin", origin, 4) ||
        check_ptr(fn, "tar_rgb", tar_rgb, 4) || check_ptr(fn, "tar_msk", tar_msk, 1) ||
        check_ptr(fn, "tar_rays", tar_rays, 4) || check_ptr(fn, "tar_rays_down", tar_rays_down, 4))
        return 1;
    if (normal && (check_ptr(fn, "nrm_rot", nrm_rot, 4) || check_ptr(fn, "tar_nrm", tar_nrm, 4))) return 1;
    AssembleArgs a;
    memset(&a, 0, sizeof(a));
    a.N = N; a.H = H; a.W = W; a.Hd = H / kDown; a.Wd = W / kDown; a.chunks = (int)chunks;
    a.main_ctas = main_ctas; a.n_down = n_down;
    a.rgba = reinterpret_cast<const uint32_t*>(rgba);
    a.nrm_in = normal; a.bg = bg; a.i2w = i2w; a.i2w_d = i2w_down; a.org = origin; a.rot = normal ? nrm_rot : nullptr;
    a.rgb = tar_rgb; a.msk = tar_msk; a.nrm = normal ? tar_nrm : nullptr; a.rays = tar_rays; a.rays_d = tar_rays_down;
    const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    batch_assemble_kernel<<<(unsigned)ctas, kThreads, 0, stream>>>(a);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_error("batch_assemble launch", e);
}

extern "C" int srf_batch_cameras(srf_stream_t stream_, int n, const float* c2w, const float* bg, float* cams) {
    using namespace srf;
    const char* fn = "srf_batch_cameras";
    if (n <= 0 || n > 65535) return set_error("%s: bad sizes: n = %d views must be in (0, 65535]", fn, n);
    if (check_ptr(fn, "c2w", c2w, 4) || check_ptr(fn, "bg", bg, 4) || check_ptr(fn, "cams", cams, 4)) return 1;
    const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    batch_cameras_kernel<<<(unsigned)((n + kThreads - 1) / kThreads), kThreads, 0, stream>>>(n, c2w, bg, cams);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_error("batch_cameras launch", e);
}
