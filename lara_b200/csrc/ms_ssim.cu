// ms_ssim.cu -- fused MS-SSIM of LaRa's training loss (lightning/loss.py:44-47, pytorch-msssim 1.0.0
// MS_SSIM(data_range, size_average, channel=3)), forward and backward.
//
// Per level l = 0..4 on X_l, Y_l (one (b, c) plane per blockIdx.y):
//   mu = G(.), sigma = G(. * .) - mu mu with G the separable valid 11-tap Gaussian (H pass, then W pass),
//   cs_map = (2 s_xy + C2) / (s_x + s_y + C2), ssim_map = (2 mu_x mu_y + C1) / (mu_x^2 + mu_y^2 + C1) * cs_map,
//   m_l = mean(cs_map) for l < 4, mean(ssim_map) for l = 4, then X_{l+1} = avg_pool2d(X_l, 2, padding=dims % 2).
//   value[b,c] = prod_l relu(m_l)^w_l; the result is its mean over (b, c), or over c per b.
// ms_ssim_fwd_kernel   : one CTA per 32x16 tile of one plane: stages X, Y with the 10-pixel halo, filters the five
//                        quantities (H pass into shared memory, W pass in registers), writes one partial sum per CTA
//                        and the 2x2 average pool of the pixels it owns (the next level's input).
// ms_ssim_finalize_kernel: reduces the partials in a fixed order in fp64 (fixed_sums.cuh's warp_strided_sum), applies
//                        relu / pow / prod / mean and writes the result and dvalue/dm_l per plane, already divided by
//                        the level's valid-pixel count.
// ms_ssim_bwd_kernel   : levels 4 -> 0, gather form, one thread per input pixel: recomputes the filtered maps on the
//                        outputs whose windows cover the tile (20-pixel input halo), forms the coefficient maps
//                        A = dm/dmu_x, B = dm/dG(XX), C = dm/dG(XY) (times the level's coefficient), filters them back
//                        and adds the pooling backward: dX_l = G^T A + 2 X G^T B + Y G^T C + dX_{l+1}(parent) / 4.
// No atomics anywhere: two identical calls give identical bits.  The level-0 image is read (and its gradient
// written) through MsAddr, so a channel-last tensor and V planar views side by side are read in place.
// Two sources (srf_ms_ssim_passes_*, LaRa's coarse and fine passes against one target): the batch has 2 B entries;
// at level 0 entry b < B reads X from x, entry b >= B from x2 at b - B, and both read Y at b mod B; levels >= 1 are
// planar over all 2 B C planes.  Each plane runs the same code as in a one-source call, so its value and coefficients
// have the same bits; the finalize writes one mean per source.  The backward can add its level-0 gradient into dX
// instead of writing it.
// The C entries srf_ms_ssim_* (include/surfel_rasterizer.h) are defined here, and so are srf_ssim_*: single-scale
// SSIM, the same code with a one-level pyramid (its only level is the kLast level, on the caller's image).  The
// level count changes only the size rule and the finalize's value / coefficient rule.
#include <math.h>
#include <string.h>

#include "../../include/surfel_rasterizer.h"
#include "fixed_sums.cuh"
#include "surfel_common.cuh"
#include "surfel_kernels.h"

namespace srf {

// A logical B x C x H x W image read through element strides; column x of the logical image lies in view x / wv at
// column x % wv.
struct MsAddr { long long sb, sc, sy, sx, sv; int wv; };
struct MsSsimArgs {
    int B, C, H, W;              // B: entries of all sources, nsrc * nb
    int nb, nsrc;                // entries per source, sources (1, or 2 with x2)
    int size_average;            // out[s] = mean over (b, c) of source s; else out[b] = mean over c
    float data_range;
    const float* x; const float* x2; const float* y; MsAddr ax, ay;   // x2: the second source (null: one), read via ax
    void* workspace;             // srf_ms_ssim_workspace_bytes: pyramid, its gradient, partial sums, coefficients
    float* out;                  // forward output
    const float* gout;           // backward: upstream gradient of out (device)
    float* gx; float* gx2; MsAddr ag;   // backward output, dL/dX of each source
    int accumulate;              // backward: add dL/dX into gx / gx2 instead of writing it
};

namespace {

constexpr int kTW = 32, kTH = 16;          // tile of output pixels (forward) / input pixels (backward)
constexpr int kR = 10;                     // window size - 1
constexpr int kThreads = 256;
constexpr int kLevels = 5;                 // MS-SSIM's; single-scale SSIM has 1

struct Layout {
    int levels;
    int h[kLevels], w[kLevels];
    int px[kLevels], py[kLevels];          // pooling padding from level l to l + 1 (0 at the last level)
    int ntx[kLevels], nty[kLevels];        // forward tile grid
    size_t pyr[kLevels];                   // float index of X_l (Y_l follows n_l floats later), l >= 1
    size_t gpyr[kLevels];                  // float index of dX_l, l >= 1
    size_t part[kLevels];                  // double index of level l's per-CTA partial sums
    size_t o_pyr, o_gpyr, o_part, o_mean, o_val, o_coef, total;   // byte offsets in the workspace
};

Layout make_layout(int levels, int B, int C, int H, int W) {
    Layout L;
    L.levels = levels;
    const size_t planes = (size_t)B * C;
    size_t np = 0, ng = 0, nq = 0;
    for (int l = 0; l < levels; ++l) {
        L.h[l] = l ? (L.h[l - 1] + 1) / 2 : H;      // avg_pool2d(2, padding = s % 2): floor((s + 2 (s % 2)) / 2)
        L.w[l] = l ? (L.w[l - 1] + 1) / 2 : W;
        L.px[l] = l < levels - 1 ? L.w[l] % 2 : 0;
        L.py[l] = l < levels - 1 ? L.h[l] % 2 : 0;
        L.ntx[l] = (L.w[l] + L.px[l] + kTW - 1) / kTW;
        L.nty[l] = (L.h[l] + L.py[l] + kTH - 1) / kTH;
        const size_t n = planes * L.h[l] * L.w[l];
        L.pyr[l] = np; L.gpyr[l] = ng;
        if (l) { np += 2 * n; ng += n; }
        L.part[l] = nq;
        nq += planes * L.ntx[l] * L.nty[l];
    }
    size_t o = 0;
    L.o_pyr = o;  o = align_up(o + np * sizeof(float));
    L.o_gpyr = o; o = align_up(o + ng * sizeof(float));
    L.o_part = o; o = align_up(o + nq * sizeof(double));
    L.o_mean = o; o = align_up(o + levels * planes * sizeof(double));
    L.o_val = o;  o = align_up(o + planes * sizeof(double));
    L.o_coef = o; o = align_up(o + levels * planes * sizeof(float));
    L.total = o;
    return L;
}

struct LevelArgs {
    int C, H, W;                 // planes are (b, c) = (p / C, p % C); this level's input size
    int px, py;                  // pooling padding towards the next level
    int ntx;                     // tiles per row of the grid
    float c1, c2;
    float win[kR + 1];
    const float* x; const float* y; MsAddr ax, ay;   // this level's input
    const float* x2; int nb;     // level 0 of two sources: entries b >= nb read x2 at b - nb, and Y at b - nb
    // forward
    float* nx; float* ny; int nh, nw;                // next level's planar X, Y (null at the last level)
    double* part;                // [planes][ntiles] per-CTA partial sums
    // backward
    const float* coef;           // [planes] dvalue/dm_l / count_l
    const float* gout; int gout_planes;              // upstream gradient: entry plane / gout_planes
    const float* gnext;          // planar dX_{l+1} (null at the last level)
    float* gx; float* gx2; MsAddr ag;                // dX_l (gx2: level 0's for the entries that read x2)
    int accumulate;              // add into gx / gx2

};

struct FinalArgs {
    int B, C, planes, size_average, nsrc;
    int levels;
    int nonnegative;             // one level: relu the mean (MS-SSIM always does)
    int ntiles[kLevels];
    size_t part_off[kLevels];
    double count[kLevels];       // valid output pixels per plane, (h - 10)(w - 10)
    const double* part;
    double* mean;                // [levels][planes]
    double* val;                 // [planes]
    float* coef;                 // [levels][planes]
    float* out;                  // [nsrc] or [B]
};

__device__ __forceinline__ long long addr_of(const MsAddr& a, int b, int c, int y, int x) {
    const int v = x / a.wv;
    return b * a.sb + c * a.sc + y * a.sy + v * a.sv + (x - v * a.wv) * a.sx;
}

// Level 0 of two sources: the X base of entry b, which becomes its scene b mod nb (the index of X, Y and dX).
__device__ __forceinline__ bool second_source(const LevelArgs& a, int& b) {
    if (!a.x2 || b < a.nb) return false;
    b -= a.nb;
    return true;
}

// Sum over the CTA of one double per thread, in a fixed order; the result is valid in thread 0.
__device__ __forceinline__ double block_sum(double v) {
    __shared__ double s_w[kThreads / 32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
    if (threadIdx.x == 0) {
#pragma unroll
        for (int w = 0; w < kThreads / 32; ++w) t += s_w[w];
    }
    return t;
}

template <bool kLast>
__global__ void __launch_bounds__(kThreads) ms_ssim_fwd_kernel(const LevelArgs a) {
    constexpr int IW = kTW + kR, IH = kTH + kR;
    __shared__ float s_in[2][IH][IW];
    __shared__ float s_h[5][kTH][IW];
    const int plane = blockIdx.y, c = plane % a.C;
    int b = plane / a.C;
    const float* xs = second_source(a, b) ? a.x2 : a.x;
    const int tx = blockIdx.x % a.ntx, ty = blockIdx.x / a.ntx;
    // tiles start at -padding so that each CTA owns whole 2x2 pooling cells
    const int x0 = tx * kTW - a.px, y0 = ty * kTH - a.py;
    for (int i = threadIdx.x; i < IH * IW; i += kThreads) {
        const int r = i / IW, q = i - r * IW, y = y0 + r, x = x0 + q;
        float vx = 0.f, vy = 0.f;
        if (y >= 0 && y < a.H && x >= 0 && x < a.W) {
            vx = __ldg(xs + addr_of(a.ax, b, c, y, x));
            vy = __ldg(a.y + addr_of(a.ay, b, c, y, x));
        }
        s_in[0][r][q] = vx;
        s_in[1][r][q] = vy;
    }
    __syncthreads();
    if (!kLast && threadIdx.x < (kTH / 2) * (kTW / 2)) {
        // avg_pool2d: the in-image inputs of a cell added row by row (padding adds 0), divided by 4
        const int j = threadIdx.x % (kTW / 2), k = threadIdx.x / (kTW / 2);
        const int X1 = tx * (kTW / 2) + j, Y1 = ty * (kTH / 2) + k;
        if (X1 < a.nw && Y1 < a.nh) {
            const size_t o = ((size_t)plane * a.nh + Y1) * a.nw + X1;
#pragma unroll
            for (int s = 0; s < 2; ++s) {
                float t = s_in[s][2 * k][2 * j];
                t += s_in[s][2 * k][2 * j + 1];
                t += s_in[s][2 * k + 1][2 * j];
                t += s_in[s][2 * k + 1][2 * j + 1];
                (s ? a.ny : a.nx)[o] = t * 0.25f;
            }
        }
    }
    // H pass (along y): 11 taps of x, y, x^2, y^2, xy
    for (int i = threadIdx.x; i < kTH * IW; i += kThreads) {
        const int r = i / IW, q = i - r * IW;
        float m0 = 0.f, m1 = 0.f, m2 = 0.f, m3 = 0.f, m4 = 0.f;
#pragma unroll
        for (int t = 0; t <= kR; ++t) {
            const float u = s_in[0][r + t][q], v = s_in[1][r + t][q], g = a.win[t];
            m0 = fmaf(g, u, m0);
            m1 = fmaf(g, v, m1);
            m2 = fmaf(g, u * u, m2);
            m3 = fmaf(g, v * v, m3);
            m4 = fmaf(g, u * v, m4);
        }
        s_h[0][r][q] = m0; s_h[1][r][q] = m1; s_h[2][r][q] = m2; s_h[3][r][q] = m3; s_h[4][r][q] = m4;
    }
    __syncthreads();
    // W pass in registers, then the maps
    const int lane = threadIdx.x & 31;
    double acc = 0.0;
    for (int r = threadIdx.x >> 5; r < kTH; r += kThreads / 32) {
        const int oy = y0 + r, ox = x0 + lane;
        if (oy < 0 || oy >= a.H - kR || ox < 0 || ox >= a.W - kR) continue;
        float f[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int t = 0; t <= kR; ++t) {
#pragma unroll
            for (int k = 0; k < 5; ++k) f[k] = fmaf(a.win[t], s_h[k][r][lane + t], f[k]);
        }
        const float mxx = f[0] * f[0], myy = f[1] * f[1], mxy = f[0] * f[1];
        const float sx = f[2] - mxx, sy = f[3] - myy, sxy = f[4] - mxy;
        const float cs = (2.f * sxy + a.c2) / (sx + sy + a.c2);
        if (kLast) acc += (double)((2.f * mxy + a.c1) / (mxx + myy + a.c1) * cs);
        else acc += (double)cs;
    }
    const double s = block_sum(acc);
    if (threadIdx.x == 0) a.part[(size_t)plane * gridDim.x + blockIdx.x] = s;
}

__global__ void __launch_bounds__(kThreads) ms_ssim_finalize_kernel(const FinalArgs f) {
    const double kWeights[kLevels] = {0.0448, 0.2856, 0.3001, 0.2363, 0.1333};
    const int P = f.planes;
    // one warp per (level, plane)
    for (int j = threadIdx.x >> 5; j < f.levels * P; j += kThreads / 32) {
        const int l = j / P, p = j - l * P, n = f.ntiles[l];
        const double s = warp_strided_sum(f.part + f.part_off[l] + (size_t)p * n, n, 1);
        if ((threadIdx.x & 31) == 0) f.mean[j] = s / f.count[l];
    }
    __syncthreads();
    const int per_src = P / f.nsrc;
    const double scale = 1.0 / (f.size_average ? (double)per_src : (double)f.C);
    for (int p = threadIdx.x; p < P; p += kThreads) {
        if (f.levels == 1) {
            // SSIM: the mean, optionally relu'd; relu's backward is a select, so no gradient through a mean <= 0
            const double m = f.mean[p];
            const bool pass = !f.nonnegative || m > 0.0;
            f.val[p] = pass ? m : 0.0;
            f.coef[p] = pass ? (float)(scale / f.count[0]) : 0.f;
            continue;
        }
        double m[kLevels];
        bool pos = true;
#pragma unroll
        for (int l = 0; l < kLevels; ++l) {
            m[l] = f.mean[l * P + p];
            pos = pos && m[l] > 0.0;
        }
        // relu(m) = 0 at any level: value 0 and, relu's backward being a select, no gradient through this plane
        double v = pos ? 1.0 : 0.0;
        if (pos) {
#pragma unroll
            for (int l = 0; l < kLevels; ++l) v *= pow(m[l], kWeights[l]);
        }
        f.val[p] = v;
#pragma unroll
        for (int l = 0; l < kLevels; ++l)
            f.coef[l * P + p] = pos ? (float)(kWeights[l] * v / m[l] * scale / f.count[l]) : 0.f;
    }
    __syncthreads();
    const int nout = f.size_average ? f.nsrc : f.B;
    for (int o = threadIdx.x; o < nout; o += kThreads) {
        const int np = f.size_average ? per_src : f.C, p0 = o * np;
        double s = 0.0;
        for (int p = 0; p < np; ++p) s += f.val[p0 + p];
        f.out[o] = (float)(s / np);
    }
}

template <bool kLast>
__global__ void __launch_bounds__(kThreads) ms_ssim_bwd_kernel(const LevelArgs a) {
    constexpr int IW = kTW + 2 * kR, IH = kTH + 2 * kR;   // inputs under the windows of the outputs below
    constexpr int OW = kTW + kR, OH = kTH + kR;           // outputs whose windows cover the tile
    __shared__ float s_a[2 * IH * IW];     // X, Y; then the coefficient maps [3][OH][OW]
    __shared__ float s_b[5 * OH * IW];     // H pass of the five quantities; then the H pass of G^T [3][kTH][OW]
    static_assert(3 * OH * OW <= 2 * IH * IW && 3 * kTH * OW <= 5 * OH * IW, "shared-memory aliasing");
    const int plane = blockIdx.y, c = plane % a.C;
    int b = plane / a.C;
    const bool second = second_source(a, b);
    const float* xs = second ? a.x2 : a.x;
    float* gxs = second ? a.gx2 : a.gx;
    const int x0 = (blockIdx.x % a.ntx) * kTW, y0 = (blockIdx.x / a.ntx) * kTH;
    const int lane = threadIdx.x & 31, wr = threadIdx.x >> 5;
    const float k = a.coef[plane] * __ldg(a.gout + plane / a.gout_planes);
    float ga[2] = {0.f, 0.f}, gb[2] = {0.f, 0.f}, gc[2] = {0.f, 0.f};
    if (k != 0.f) {     // uniform over the CTA
        for (int i = threadIdx.x; i < IH * IW; i += kThreads) {
            const int r = i / IW, q = i - r * IW, y = y0 - kR + r, x = x0 - kR + q;
            float vx = 0.f, vy = 0.f;
            if (y >= 0 && y < a.H && x >= 0 && x < a.W) {
                vx = __ldg(xs + addr_of(a.ax, b, c, y, x));
                vy = __ldg(a.y + addr_of(a.ay, b, c, y, x));
            }
            s_a[r * IW + q] = vx;
            s_a[IH * IW + r * IW + q] = vy;
        }
        __syncthreads();
        for (int i = threadIdx.x; i < OH * IW; i += kThreads) {
            const int r = i / IW, q = i - r * IW;
            float m0 = 0.f, m1 = 0.f, m2 = 0.f, m3 = 0.f, m4 = 0.f;
#pragma unroll
            for (int t = 0; t <= kR; ++t) {
                const float u = s_a[(r + t) * IW + q], v = s_a[IH * IW + (r + t) * IW + q], g = a.win[t];
                m0 = fmaf(g, u, m0);
                m1 = fmaf(g, v, m1);
                m2 = fmaf(g, u * u, m2);
                m3 = fmaf(g, v * v, m3);
                m4 = fmaf(g, u * v, m4);
            }
            s_b[0 * OH * IW + i] = m0; s_b[1 * OH * IW + i] = m1; s_b[2 * OH * IW + i] = m2;
            s_b[3 * OH * IW + i] = m3; s_b[4 * OH * IW + i] = m4;
        }
        __syncthreads();
        for (int i = threadIdx.x; i < OH * OW; i += kThreads) {
            const int r = i / OW, q = i - r * OW, oy = y0 - kR + r, ox = x0 - kR + q;
            float A = 0.f, Bm = 0.f, Cm = 0.f;
            if (oy >= 0 && oy < a.H - kR && ox >= 0 && ox < a.W - kR) {
                float f[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
                for (int t = 0; t <= kR; ++t) {
#pragma unroll
                    for (int j = 0; j < 5; ++j) f[j] = fmaf(a.win[t], s_b[j * OH * IW + r * IW + q + t], f[j]);
                }
                const float mx = f[0], my = f[1];
                const float mxx = mx * mx, myy = my * my, mxy = mx * my;
                const float sx = f[2] - mxx, sy = f[3] - myy, sxy = f[4] - mxy;
                const float dcs = sx + sy + a.c2;
                const float cs = (2.f * sxy + a.c2) / dcs;
                const float rd = 1.f / dcs;
                // d cs / d mu_x, d cs / d G(XX), d cs / d G(XY)
                const float cmu = 2.f * (mx * cs - my) * rd, cxx = -cs * rd, cxy = 2.f * rd;
                if (kLast) {
                    const float dl = mxx + myy + a.c1;
                    const float lum = (2.f * mxy + a.c1) / dl;
                    const float lmu = 2.f * (my - mx * lum) / dl;
                    A = k * (cs * lmu + lum * cmu);
                    Bm = k * lum * cxx;
                    Cm = k * lum * cxy;
                } else {
                    A = k * cmu;
                    Bm = k * cxx;
                    Cm = k * cxy;
                }
            }
            s_a[i] = A;
            s_a[OH * OW + i] = Bm;
            s_a[2 * OH * OW + i] = Cm;
        }
        __syncthreads();
        // G^T along y: input row y0 + r gathers the output rows y0 + r - t, local r + kR - t
        for (int i = threadIdx.x; i < kTH * OW; i += kThreads) {
            const int r = i / OW, q = i - r * OW;
            float t0 = 0.f, t1 = 0.f, t2 = 0.f;
#pragma unroll
            for (int t = 0; t <= kR; ++t) {
                const int o = (r + kR - t) * OW + q;
                const float g = a.win[t];
                t0 = fmaf(g, s_a[o], t0);
                t1 = fmaf(g, s_a[OH * OW + o], t1);
                t2 = fmaf(g, s_a[2 * OH * OW + o], t2);
            }
            s_b[i] = t0;
            s_b[kTH * OW + i] = t1;
            s_b[2 * kTH * OW + i] = t2;
        }
        __syncthreads();
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int r = wr + h * (kThreads / 32);
#pragma unroll
            for (int t = 0; t <= kR; ++t) {
                const int o = r * OW + lane + kR - t;
                ga[h] = fmaf(a.win[t], s_b[o], ga[h]);
                gb[h] = fmaf(a.win[t], s_b[kTH * OW + o], gb[h]);
                gc[h] = fmaf(a.win[t], s_b[2 * kTH * OW + o], gc[h]);
            }
        }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int y = y0 + wr + h * (kThreads / 32), x = x0 + lane;
        if (y >= a.H || x >= a.W) continue;
        float d = 0.f;
        if (k != 0.f) {
            const float vx = __ldg(xs + addr_of(a.ax, b, c, y, x)), vy = __ldg(a.y + addr_of(a.ay, b, c, y, x));
            d = fmaf(2.f * vx, gb[h], ga[h]);
            d = fmaf(vy, gc[h], d);
        }
        if (!kLast) d += 0.25f * __ldg(a.gnext + ((size_t)plane * a.nh + (y + a.py) / 2) * a.nw + (x + a.px) / 2);
        float* g = gxs + addr_of(a.ag, b, c, y, x);
        if (a.accumulate) *g += d;
        else *g = d;
    }
}

static_assert(kThreads / 32 * 2 == kTH && kTW == 32, "backward: one warp per tile row pair, one lane per column");

// a level >= 1 of the pyramid: planes (b, c) back to back, each H x W
MsAddr planar(int C, int H, int W) {
    MsAddr p;
    p.sc = (long long)H * W; p.sb = C * p.sc; p.sy = W; p.sx = 1; p.sv = 0; p.wv = W;
    return p;
}

// level l's inputs and the window / constants shared by both directions
void level_constants(LevelArgs& a, float data_range) {
    const double c1 = 0.01 * data_range, c2 = 0.03 * data_range;
    a.c1 = (float)(c1 * c1); a.c2 = (float)(c2 * c2);
    // the library's fp32 window: g = exp(-(i - 5)^2 / (2 * 1.5^2)) in fp32, g / sum(g); the sum is rounded once
    float e[kR + 1];
    double sum = 0.0;
    for (int i = 0; i <= kR; ++i) {
        const float ci = (float)(i - 5);
        e[i] = (float)exp((double)(-(ci * ci) / 4.5f));
        sum += e[i];
    }
    for (int i = 0; i <= kR; ++i) a.win[i] = e[i] / (float)sum;
}

LevelArgs level_args(const MsSsimArgs& m, const Layout& L, char* ws, int l) {
    LevelArgs a;
    memset(&a, 0, sizeof(a));
    a.C = m.C; a.H = L.h[l]; a.W = L.w[l]; a.px = L.px[l]; a.py = L.py[l];
    level_constants(a, m.data_range);
    float* pyr = reinterpret_cast<float*>(ws + L.o_pyr);
    if (l == 0) {
        a.x = m.x; a.y = m.y; a.ax = m.ax; a.ay = m.ay;
        a.x2 = m.x2; a.nb = m.nb;
    } else {
        const size_t n = (size_t)m.B * m.C * L.h[l] * L.w[l];
        a.x = pyr + L.pyr[l]; a.y = a.x + n;
        a.ax = a.ay = planar(m.C, L.h[l], L.w[l]);
    }
    if (l + 1 < L.levels) {
        a.nh = L.h[l + 1]; a.nw = L.w[l + 1];
        a.nx = pyr + L.pyr[l + 1];
        a.ny = a.nx + (size_t)m.B * m.C * a.nh * a.nw;
    }
    return a;
}

}  // namespace

}  // namespace srf

using srf::cuda_error;
using srf::set_error;


// min(H, W) > 10 * 2^(levels - 1): every level of the pyramid keeps at least one valid window
static int ms_ssim_sizes(const char* fn, int levels, int B, int C, int H, int W) {
    if (B <= 0 || C <= 0 || H <= 0 || W <= 0) return set_error("%s: bad sizes (B=%d, C=%d, H=%d, W=%d)", fn, B, C, H, W);
    if ((H < W ? H : W) <= srf::kR << (levels - 1)) {
        if (levels > 1)
            return set_error("%s: Image size should be larger than 160 due to the 4 downsamplings in ms-ssim (H=%d, W=%d)", fn, H, W);
        return set_error("%s: H and W must be at least the window size 11 (H=%d, W=%d)", fn, H, W);
    }
    if ((long long)B * C > 65535) return set_error("%s: B*C=%lld planes exceeds 65535", fn, (long long)B * C);
    return 0;
}

static int ms_ssim_addr(const char* fn, const char* what, const float* p, const srf_ms_ssim_addr* a, srf::MsAddr* out) {
    if (!p || !a) return set_error("%s: null %s pointer", fn, what);
    if (reinterpret_cast<uintptr_t>(p) & 3) return set_error("%s: %s must be 4-byte aligned", fn, what);
    if (a->wv <= 0 || a->wv > 0x7fffffff) return set_error("%s: %s view width %lld out of range", fn, what, (long long)a->wv);
    out->sb = a->sb; out->sc = a->sc; out->sy = a->sy; out->sx = a->sx; out->sv = a->sv; out->wv = (int)a->wv;
    return 0;
}

// B scenes per source; x2 (read through x_addr) null for one source
static int ms_ssim_prepare(const char* fn, int levels, int B, int C, int H, int W, const float* x, const float* x2,
                           const srf_ms_ssim_addr* x_addr, const float* y, const srf_ms_ssim_addr* y_addr,
                           float data_range, int size_average, void* workspace, srf::MsSsimArgs* a) {
    memset(a, 0, sizeof(*a));
    const int nsrc = x2 ? 2 : 1;
    if (ms_ssim_sizes(fn, levels, B, C, H, W)) return 1;
    if (nsrc > 1 && ms_ssim_sizes(fn, levels, nsrc * B, C, H, W)) return 1;
    if (ms_ssim_addr(fn, "x", x, x_addr, &a->ax) || ms_ssim_addr(fn, "y", y, y_addr, &a->ay)) return 1;
    if (x2 && (reinterpret_cast<uintptr_t>(x2) & 3)) return set_error("%s: x_fine must be 4-byte aligned", fn);
    if (!(data_range > 0.f) || !(data_range < 3.0e38f)) return set_error("%s: data_range must be positive and finite", fn);
    if (!workspace || srf::misaligned(workspace)) return set_error("%s: workspace must be 256-byte aligned", fn);
    a->B = nsrc * B; a->nb = B; a->nsrc = nsrc; a->C = C; a->H = H; a->W = W;
    a->size_average = size_average ? 1 : 0; a->data_range = data_range;
    a->x = x; a->x2 = x2; a->y = y; a->workspace = workspace;
    return 0;
}

static int ms_ssim_workspace_bytes(const char* fn, int levels, int nsrc, int B, int C, int H, int W, size_t* bytes) {
    if (ms_ssim_sizes(fn, levels, B, C, H, W)) return 1;
    if (nsrc > 1 && ms_ssim_sizes(fn, levels, nsrc * B, C, H, W)) return 1;
    if (!bytes) return set_error("%s: null pointer", fn);
    *bytes = srf::make_layout(levels, nsrc * B, C, H, W).total;
    return 0;
}

// the pyramid's levels 0 .. levels - 1, then the finalize
static int ms_ssim_forward(const char* fn, int levels, int nonnegative, srf_stream_t stream_, int B, int C, int H,
                           int W, const float* x, const float* x2, const srf_ms_ssim_addr* x_addr, const float* y,
                           const srf_ms_ssim_addr* y_addr, float data_range, int size_average, void* workspace,
                           float* out) {
    using namespace srf;
    MsSsimArgs m;
    if (ms_ssim_prepare(fn, levels, B, C, H, W, x, x2, x_addr, y, y_addr, data_range, size_average, workspace, &m))
        return 1;
    if (!out) return set_error("%s: null output pointer", fn);
    if (reinterpret_cast<uintptr_t>(out) & 3) return set_error("%s: out must be 4-byte aligned", fn);
    m.out = out;
    B = m.B;
    const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const Layout L = make_layout(levels, B, C, H, W);
    char* ws = static_cast<char*>(workspace);
    const int planes = B * C;
    for (int l = 0; l < levels; ++l) {
        LevelArgs a = level_args(m, L, ws, l);
        a.ntx = L.ntx[l];
        a.part = reinterpret_cast<double*>(ws + L.o_part) + L.part[l];
        const dim3 grid((unsigned)(L.ntx[l] * L.nty[l]), (unsigned)planes);
        if (l + 1 < levels) ms_ssim_fwd_kernel<false><<<grid, kThreads, 0, stream>>>(a);
        else ms_ssim_fwd_kernel<true><<<grid, kThreads, 0, stream>>>(a);
    }
    FinalArgs f;
    memset(&f, 0, sizeof(f));
    f.B = B; f.C = C; f.planes = planes; f.size_average = m.size_average; f.nsrc = m.nsrc;
    f.levels = levels; f.nonnegative = nonnegative ? 1 : 0;
    for (int l = 0; l < levels; ++l) {
        f.ntiles[l] = L.ntx[l] * L.nty[l];
        f.part_off[l] = L.part[l];
        f.count[l] = (double)(L.h[l] - kR) * (double)(L.w[l] - kR);
    }
    f.part = reinterpret_cast<const double*>(ws + L.o_part);
    f.mean = reinterpret_cast<double*>(ws + L.o_mean);
    f.val = reinterpret_cast<double*>(ws + L.o_val);
    f.coef = reinterpret_cast<float*>(ws + L.o_coef);
    f.out = out;
    ms_ssim_finalize_kernel<<<1, kThreads, 0, stream>>>(f);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_error(levels > 1 ? "ms_ssim_fwd launch" : "ssim_fwd launch", e);
}

// levels - 1 .. 0 with the coefficients the forward left in the workspace
static int ms_ssim_backward(const char* fn, int levels, srf_stream_t stream_, int B, int C, int H, int W,
                            const float* x, const float* x2, const srf_ms_ssim_addr* x_addr, const float* y,
                            const srf_ms_ssim_addr* y_addr, float data_range, int size_average, void* workspace,
                            const float* upstream, float* dx, float* dx2, const srf_ms_ssim_addr* dx_addr,
                            int accumulate) {
    using namespace srf;
    MsSsimArgs m;
    if (ms_ssim_prepare(fn, levels, B, C, H, W, x, x2, x_addr, y, y_addr, data_range, size_average, workspace, &m))
        return 1;
    if (!upstream) return set_error("%s: null upstream gradient", fn);
    if (reinterpret_cast<uintptr_t>(upstream) & 3) return set_error("%s: upstream must be 4-byte aligned", fn);
    if (ms_ssim_addr(fn, "dx", dx, dx_addr, &m.ag)) return 1;
    if (!x2 != !dx2) return set_error("%s: x_fine and dx_fine go together", fn);
    if (dx2 && (reinterpret_cast<uintptr_t>(dx2) & 3)) return set_error("%s: dx_fine must be 4-byte aligned", fn);
    m.gout = upstream; m.gx = dx; m.gx2 = dx2; m.accumulate = accumulate ? 1 : 0;
    B = m.B;
    const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const Layout L = make_layout(levels, B, C, H, W);
    char* ws = static_cast<char*>(workspace);
    const int planes = B * C;
    float* coef = reinterpret_cast<float*>(ws + L.o_coef);
    float* gpyr = reinterpret_cast<float*>(ws + L.o_gpyr);
    for (int l = levels - 1; l >= 0; --l) {
        LevelArgs a = level_args(m, L, ws, l);
        a.ntx = (L.w[l] + kTW - 1) / kTW;
        const int nty = (L.h[l] + kTH - 1) / kTH;
        a.coef = coef + (size_t)l * planes;
        a.gout = m.gout; a.gout_planes = m.size_average ? m.nb * C : C;
        if (l + 1 < levels) a.gnext = gpyr + L.gpyr[l + 1];
        if (l == 0) { a.gx = m.gx; a.gx2 = m.gx2; a.ag = m.ag; a.accumulate = m.accumulate; }
        else { a.gx = gpyr + L.gpyr[l]; a.ag = planar(m.C, L.h[l], L.w[l]); }
        const dim3 grid((unsigned)(a.ntx * nty), (unsigned)planes);
        if (l + 1 < levels) ms_ssim_bwd_kernel<false><<<grid, kThreads, 0, stream>>>(a);
        else ms_ssim_bwd_kernel<true><<<grid, kThreads, 0, stream>>>(a);
    }
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_error(levels > 1 ? "ms_ssim_bwd launch" : "ssim_bwd launch", e);
}

extern "C" int srf_ms_ssim_workspace_bytes(int B, int C, int H, int W, size_t* bytes) {
    return ms_ssim_workspace_bytes("srf_ms_ssim_workspace_bytes", srf::kLevels, 1, B, C, H, W, bytes);
}

extern "C" int srf_ms_ssim_workspace_layout(int B, int C, int H, int W, size_t regions[7], size_t levels[15],
                                            int dims[30]) {
    if (ms_ssim_sizes("srf_ms_ssim_workspace_layout", srf::kLevels, B, C, H, W)) return 1;
    if (!regions || !levels || !dims) return set_error("srf_ms_ssim_workspace_layout: null pointer");
    const srf::Layout L = srf::make_layout(srf::kLevels, B, C, H, W);
    const size_t r[7] = {L.o_pyr, L.o_gpyr, L.o_part, L.o_mean, L.o_val, L.o_coef, L.total};
    for (int i = 0; i < 7; ++i) regions[i] = r[i];
    for (int l = 0; l < srf::kLevels; ++l) {
        levels[l] = L.pyr[l]; levels[srf::kLevels + l] = L.gpyr[l]; levels[2 * srf::kLevels + l] = L.part[l];
        const int d[6] = {L.h[l], L.w[l], L.px[l], L.py[l], L.ntx[l], L.nty[l]};
        for (int i = 0; i < 6; ++i) dims[i * srf::kLevels + l] = d[i];
    }
    return 0;
}

extern "C" int srf_ms_ssim_forward(srf_stream_t stream, int B, int C, int H, int W, const float* x,
                                   const srf_ms_ssim_addr* x_addr, const float* y, const srf_ms_ssim_addr* y_addr,
                                   float data_range, int size_average, void* workspace, float* out) {
    return ms_ssim_forward("srf_ms_ssim_forward", srf::kLevels, 1, stream, B, C, H, W, x, nullptr, x_addr, y, y_addr,
                           data_range, size_average, workspace, out);
}

extern "C" int srf_ms_ssim_backward(srf_stream_t stream, int B, int C, int H, int W, const float* x,
                                    const srf_ms_ssim_addr* x_addr, const float* y, const srf_ms_ssim_addr* y_addr,
                                    float data_range, int size_average, void* workspace, const float* upstream,
                                    float* dx, const srf_ms_ssim_addr* dx_addr) {
    return ms_ssim_backward("srf_ms_ssim_backward", srf::kLevels, stream, B, C, H, W, x, nullptr, x_addr, y, y_addr,
                            data_range, size_average, workspace, upstream, dx, nullptr, dx_addr, 0);
}

extern "C" int srf_ms_ssim_passes_workspace_bytes(int B, int C, int H, int W, int with_fine, size_t* bytes) {
    return ms_ssim_workspace_bytes("srf_ms_ssim_passes_workspace_bytes", srf::kLevels, with_fine ? 2 : 1, B, C, H, W,
                                   bytes);
}

extern "C" int srf_ms_ssim_passes_forward(srf_stream_t stream, int B, int C, int H, int W, const float* x,
                                          const float* x_fine, const srf_ms_ssim_addr* x_addr, const float* y,
                                          const srf_ms_ssim_addr* y_addr, float data_range, void* workspace,
                                          float* out) {
    return ms_ssim_forward("srf_ms_ssim_passes_forward", srf::kLevels, 1, stream, B, C, H, W, x, x_fine, x_addr, y,
                           y_addr, data_range, 1, workspace, out);
}

extern "C" int srf_ms_ssim_passes_backward(srf_stream_t stream, int B, int C, int H, int W, const float* x,
                                           const float* x_fine, const srf_ms_ssim_addr* x_addr, const float* y,
                                           const srf_ms_ssim_addr* y_addr, float data_range, void* workspace,
                                           const float* upstream, float* dx, float* dx_fine,
                                           const srf_ms_ssim_addr* dx_addr, int accumulate) {
    return ms_ssim_backward("srf_ms_ssim_passes_backward", srf::kLevels, stream, B, C, H, W, x, x_fine, x_addr, y,
                            y_addr, data_range, 1, workspace, upstream, dx, dx_fine, dx_addr, accumulate);
}

// ---- single-scale SSIM (pytorch-msssim 1.0.0 ssim): the one-level pyramid ----

extern "C" int srf_ssim_workspace_bytes(int B, int C, int H, int W, size_t* bytes) {
    return ms_ssim_workspace_bytes("srf_ssim_workspace_bytes", 1, 1, B, C, H, W, bytes);
}

extern "C" int srf_ssim_forward(srf_stream_t stream, int B, int C, int H, int W, const float* x,
                                const srf_ms_ssim_addr* x_addr, const float* y, const srf_ms_ssim_addr* y_addr,
                                float data_range, int size_average, int nonnegative_ssim, void* workspace, float* out) {
    return ms_ssim_forward("srf_ssim_forward", 1, nonnegative_ssim, stream, B, C, H, W, x, nullptr, x_addr, y, y_addr,
                           data_range, size_average, workspace, out);
}

extern "C" int srf_ssim_backward(srf_stream_t stream, int B, int C, int H, int W, const float* x,
                                 const srf_ms_ssim_addr* x_addr, const float* y, const srf_ms_ssim_addr* y_addr,
                                 float data_range, int size_average, int nonnegative_ssim, void* workspace,
                                 const float* upstream, float* dx, const srf_ms_ssim_addr* dx_addr) {
    (void)nonnegative_ssim;      // the forward folded the relu into the coefficients it left in the workspace
    return ms_ssim_backward("srf_ssim_backward", 1, stream, B, C, H, W, x, nullptr, x_addr, y, y_addr, data_range,
                            size_average, workspace, upstream, dx, nullptr, dx_addr, 0);
}
