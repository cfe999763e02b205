// feat_volume.cu -- fused feature-volume lifting of LaRa's coarse pass (Network.build_feat_vol,
// lightning/network.py:352-379, the view-embedding concatenation of :451-452 and VolTransformer.forward's block layout
// of :145-150), DESIGN §3.17.  The C entries of include/surfel_feat_volume.h are defined here.
//
// Forward, two kernels:
//   fv_token_fwd_kernel   a CTA per tile of 64 tokens of one (scene, view): the Plücker / SH features and their SiLU
//                         into shared memory, the LayerNorm statistics (two passes over the channels), then per slice
//                         of 32 channels the 32 -> 2C product with the slice's weight rows in registers, and the
//                         modulation.  y is written channel-last into the workspace, [B V, h w, C].
//   fv_sample_kernel      a CTA per tile of 32 voxels of one (scene, view): the taps of sample_taps.cuh (shared with
//                         point_feats.cu), then each warp reads the tap rows of y along the channels and writes the
//                         output: row by row in the condition layout (with the view-embedding columns), through a
//                         shared-memory transpose in the drop-in layout.  Both layouts form the same sum.
// Backward, no float atomics:
//   fv_cell_kernel        each voxel's floor cell (fx, fy) in [-1, w-1] x [-1, h-1] and its four tap weights; cells
//                         are counted with integer atomics (exact in any order).
//   fv_scan_kernel        exclusive scan of the counts per (scene, view).
//   fv_place_kernel       stable counting sort: rounds of 1024 voxels are bitonic-sorted by (cell, voxel) in shared
//                         memory and placed after the cell's earlier voxels, so each cell lists its voxels ascending.
//   fv_gather_kernel      a warp per token: dL/dy = sum over the cells (x, y), (x-1, y), (x, y-1), (x-1, y-1), in that
//                         order, of each listed voxel's tap weight times its dL/dout row.
//   fv_token_bwd_kernel   recomputes the token forward per tile and forms the modulation and LayerNorm vjp; the
//                         parameter gradients of the tile are summed per CTA in a fixed order (per-CTA partials).
//   fv_view_embed_kernel  per-slice sums of the view-embedding columns of dL/dout.
//   part_sums_kernel      the partials summed over the CTAs in CTA order in fp64 (fixed_sums.cuh).
#include <string.h>

#include "../../include/surfel_feat_volume.h"
#include "fixed_sums.cuh"
#include "sample_taps.cuh"
#include "surfel_kernels.h"

namespace srf {
namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kTT = 64;            // tokens per tile of the token kernels
constexpr int kTokPerWarp = kTT / kWarps;
constexpr int kVT = 32;            // voxels per tile of the sample kernel
constexpr int kSH = 32;            // Plücker / SH features per token
constexpr int kRound = 1024;       // voxels per round of the placement sort (its block size)
constexpr int kVeSlices = 64;      // row slices of the view-embedding gradient
constexpr int kAcc = 2 * kSH + 4;  // per-channel accumulators of the token backward: 2 x 32 weights, 2 biases, norm w / b
constexpr float kLnEps = 1e-6f;

struct Args {
    int B, V, C, h, w, R, E, ng;          // ng: n_group, 0 = drop-in layout
    int Himg, Wimg, hw, R3, ncells, ntiles;
    const float *x, *rays, *w2c, *ixt, *grid, *ln_w, *ln_b, *mlp_w, *mlp_b, *ve;
    float* y;                             // [B V, h w, C]: y (forward), dL/dy (backward)
    float* out;                           // forward output
    const float* gout;                    // backward: dL/dout
    float* gx;                            // dL/dimg_feats [B V, C, h w]
    float4* wts;                          // [B V, R^3] tap weights nw, ne, sw, se
    int* cell;                            // [B V, R^3] floor cell, -1 = no tap
    int* count;                           // [B V, ncells] counts, then the placement cursors
    int* start;                           // [B V, ncells + 1] first list position of each cell
    int* list;                            // [B V, R^3] voxels by cell, ascending within a cell
    float* parts;                         // [B V ntiles, 2C kAcc / 2] token-backward partials
    float* ve_parts;                      // [kVeSlices, V E]
};

// Real spherical harmonics up to degree 3 (rsh_cart_3's order, index n (n+1) + m), the constants in closed form.
__device__ __forceinline__ void rsh3(float x, float y, float z, float* o) {
    const float x2 = x * x, y2 = y * y, z2 = z * z;
    o[0] = 0.28209479177387814f;                                   // 1 / (2 sqrt(pi))
    o[1] = -0.4886025119029199f * y;                               // sqrt(3 / (4 pi))
    o[2] = 0.4886025119029199f * z;
    o[3] = -0.4886025119029199f * x;
    o[4] = 1.0925484305920792f * (x * y);                          // sqrt(15 / pi) / 2
    o[5] = -1.0925484305920792f * (y * z);
    o[6] = 0.31539156525252005f * (3.0f * z2 - 1.0f);              // sqrt(5 / pi) / 4
    o[7] = -1.0925484305920792f * (x * z);
    o[8] = 0.5462742152960396f * (x2 - y2);                        // sqrt(15 / pi) / 4
    o[9] = -0.5900435899266435f * y * (3.0f * x2 - y2);            // sqrt(35 / (2 pi)) / 4
    o[10] = 2.890611442640554f * (x * y) * z;                      // sqrt(105 / pi) / 2
    o[11] = 0.4570457994644658f * y * (1.0f - 5.0f * z2);          // sqrt(21 / (2 pi)) / 4
    o[12] = 0.3731763325901154f * z * (5.0f * z2 - 3.0f);          // sqrt(7 / pi) / 4
    o[13] = 0.4570457994644658f * x * (1.0f - 5.0f * z2);
    o[14] = 1.445305721320277f * z * (x2 - y2);                    // sqrt(105 / pi) / 4
    o[15] = -0.5900435899266435f * x * (x2 - 3.0f * y2);
}

// SiLU of [rsh_cart_3(d^), rsh_cart_3(o x d^)] for the ray r = (o, d)
__device__ void token_features(const float* r, float* s) {
    const float o0 = __ldg(r), o1 = __ldg(r + 1), o2 = __ldg(r + 2);
    const float d0 = __ldg(r + 3), d1 = __ldg(r + 4), d2 = __ldg(r + 5);
    const float inv = 1.0f / fmaxf(sqrtf(d0 * d0 + d1 * d1 + d2 * d2), 1e-12f);
    const float u0 = d0 * inv, u1 = d1 * inv, u2 = d2 * inv;
    float f[kSH];
    rsh3(u0, u1, u2, f);
    rsh3(o1 * u2 - o2 * u1, o2 * u0 - o0 * u2, o0 * u1 - o1 * u0, f + 16);
#pragma unroll
    for (int i = 0; i < kSH; ++i) s[i] = f[i] / (1.0f + expf(-f[i]));
}

// Shared state of a token tile: SiLU features, LayerNorm statistics, a transposed 32-channel slice of x.
struct TokenTile {
    float S[kTT][kSH];
    float X[32][kTT + 1];
    float mean[kTT], rstd[kTT];
    float red[4][kTT];
};

__device__ void token_prologue(const Args& a, int bv, int t0, int nt, TokenTile& sm) {
    const int tid = threadIdx.x;
    if (tid < nt) token_features(a.rays + ((size_t)bv * a.hw + t0 + tid) * 6, sm.S[tid]);
    const int tok = tid % kTT, part = tid / kTT;     // 4 threads per token, channels strided by 4
    const float* xt = a.x + (size_t)bv * a.C * a.hw + t0 + tok;
    float s = 0.0f;
    if (tok < nt) {
#pragma unroll 8
        for (int c = part; c < a.C; c += 4) s += __ldg(xt + (size_t)c * a.hw);
    }
    sm.red[part][tok] = s;
    __syncthreads();
    const float mean = (sm.red[0][tok] + sm.red[1][tok] + sm.red[2][tok] + sm.red[3][tok]) / (float)a.C;
    __syncthreads();
    float v = 0.0f;
    if (tok < nt) {
#pragma unroll 8
        for (int c = part; c < a.C; c += 4) {
            const float d = __ldg(xt + (size_t)c * a.hw) - mean;
            v = fmaf(d, d, v);
        }
    }
    sm.red[part][tok] = v;
    __syncthreads();
    if (part == 0) {
        sm.mean[tok] = mean;
        sm.rstd[tok] = 1.0f / sqrtf((sm.red[0][tok] + sm.red[1][tok] + sm.red[2][tok] + sm.red[3][tok]) / (float)a.C + kLnEps);
    }
    __syncthreads();
}

__device__ __forceinline__ void load_x_slice(const Args& a, int bv, int t0, int nt, int c0, TokenTile& sm) {
    const float* xb = a.x + ((size_t)bv * a.C + c0) * a.hw + t0;
    for (int e = threadIdx.x; e < 32 * kTT; e += kThreads) {
        const int cl = e / kTT, tok = e % kTT;
        sm.X[cl][tok] = tok < nt ? __ldg(xb + (size_t)cl * a.hw + tok) : 0.0f;
    }
}

// rows c (shift) and C + c (scale) of mlp.1
__device__ __forceinline__ void load_rows(const Args& a, int c, float* ws, float* wc) {
#pragma unroll
    for (int i = 0; i < kSH; ++i) {
        ws[i] = __ldg(a.mlp_w + (size_t)c * kSH + i);
        wc[i] = __ldg(a.mlp_w + (size_t)(a.C + c) * kSH + i);
    }
}

__device__ __forceinline__ void modulation(const float* s, const float* ws, const float* wc, float& sh, float& sc) {
#pragma unroll
    for (int i = 0; i < kSH; i += 4) {
        const float4 q = *reinterpret_cast<const float4*>(s + i);
        sh = fmaf(ws[i], q.x, sh); sh = fmaf(ws[i + 1], q.y, sh); sh = fmaf(ws[i + 2], q.z, sh); sh = fmaf(ws[i + 3], q.w, sh);
        sc = fmaf(wc[i], q.x, sc); sc = fmaf(wc[i + 1], q.y, sc); sc = fmaf(wc[i + 2], q.z, sc); sc = fmaf(wc[i + 3], q.w, sc);
    }
}

__global__ void __launch_bounds__(kThreads) fv_token_fwd_kernel(Args a) {
    __shared__ __align__(16) TokenTile sm;
    const int bv = blockIdx.y, t0 = blockIdx.x * kTT, nt = min(kTT, a.hw - t0);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    token_prologue(a, bv, t0, nt, sm);
    for (int c0 = 0; c0 < a.C; c0 += 32) {
        load_x_slice(a, bv, t0, nt, c0, sm);
        const int c = c0 + lane;
        float ws[kSH], wc[kSH];
        load_rows(a, c, ws, wc);
        const float bs = __ldg(a.mlp_b + c), bc = __ldg(a.mlp_b + a.C + c);
        const float gam = __ldg(a.ln_w + c), bet = __ldg(a.ln_b + c);
        __syncthreads();
        for (int tok = warp; tok < nt; tok += kWarps) {
            float sh = bs, sc = bc;
            modulation(sm.S[tok], ws, wc, sh, sc);
            const float ln = fmaf((sm.X[lane][tok] - sm.mean[tok]) * sm.rstd[tok], gam, bet);
            a.y[((size_t)bv * a.hw + t0 + tok) * a.C + c] = fmaf(ln, 1.0f + sc, sh);
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(kThreads, 1) fv_token_bwd_kernel(Args a) {
    __shared__ __align__(16) TokenTile sm;
    __shared__ float acc_s[kAcc][33];
    __shared__ float m12[2][kTT];
    const int bv = blockIdx.y, t0 = blockIdx.x * kTT, nt = min(kTT, a.hw - t0);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, C = a.C;
    token_prologue(a, bv, t0, nt, sm);
    float s1[kTokPerWarp] = {}, s2[kTokPerWarp] = {};       // per token of this warp: sum dn, sum dn n
    float* part = a.parts + ((size_t)bv * a.ntiles + blockIdx.x) * ((size_t)C * kAcc);
    for (int c0 = 0; c0 < C; c0 += 32) {
        load_x_slice(a, bv, t0, nt, c0, sm);
        const int c = c0 + lane;
        float ws[kSH], wc[kSH];
        load_rows(a, c, ws, wc);
        const float bs = __ldg(a.mlp_b + c), bc = __ldg(a.mlp_b + C + c);
        const float gam = __ldg(a.ln_w + c), bet = __ldg(a.ln_b + c);
        float aw[kSH] = {}, ac[kSH] = {}, ab = 0.0f, abc = 0.0f, ag = 0.0f, abt = 0.0f;
        __syncthreads();
#pragma unroll
        for (int j = 0; j < kTokPerWarp; ++j) {
            const int tok = warp + j * kWarps;
            if (tok >= nt) break;
            float sh = bs, sc = bc;
            modulation(sm.S[tok], ws, wc, sh, sc);
            const float n = (sm.X[lane][tok] - sm.mean[tok]) * sm.rstd[tok];
            const float ln = fmaf(n, gam, bet);
            const float dy = a.y[((size_t)bv * a.hw + t0 + tok) * C + c];
            const float dsc = dy * ln, dln = dy * (1.0f + sc);
            ag = fmaf(dln, n, ag);
            abt += dln;
            ab += dy;
            abc += dsc;
#pragma unroll
            for (int i = 0; i < kSH; ++i) {
                aw[i] = fmaf(dy, sm.S[tok][i], aw[i]);
                ac[i] = fmaf(dsc, sm.S[tok][i], ac[i]);
            }
            const float dn = dln * gam;
            s1[j] += warp_sum(dn);
            s2[j] += warp_sum(dn * n);
            sm.X[lane][tok] = dn;
        }
        // the warps' accumulators, added in warp order
        for (int w = 0; w < kWarps; ++w) {
            if (warp == w) {
#pragma unroll
                for (int i = 0; i < kSH; ++i) {
                    acc_s[i][lane] = w ? acc_s[i][lane] + aw[i] : aw[i];
                    acc_s[kSH + i][lane] = w ? acc_s[kSH + i][lane] + ac[i] : ac[i];
                }
                const float rest[4] = {ab, abc, ag, abt};
#pragma unroll
                for (int k = 0; k < 4; ++k) acc_s[2 * kSH + k][lane] = w ? acc_s[2 * kSH + k][lane] + rest[k] : rest[k];
            }
            __syncthreads();
        }
        // dn to dL/dimg_feats (fixed up below); the slice's partials: weight rows c and C + c, biases, norm w / b
        float* gxb = a.gx + ((size_t)bv * C + c0) * a.hw + t0;
        for (int e = threadIdx.x; e < 32 * kTT; e += kThreads) {
            const int cl = e / kTT, tok = e % kTT;
            if (tok < nt) gxb[(size_t)cl * a.hw + tok] = sm.X[cl][tok];
        }
        for (int e = threadIdx.x; e < 32 * kSH; e += kThreads) {
            const int cl = e / kSH, i = e % kSH;
            part[(size_t)(c0 + cl) * kSH + i] = acc_s[i][cl];
            part[(size_t)(C + c0 + cl) * kSH + i] = acc_s[kSH + i][cl];
        }
        if (threadIdx.x < 32) {
            const int o = 2 * C * kSH;
            part[o + c] = acc_s[2 * kSH][lane];
            part[o + C + c] = acc_s[2 * kSH + 1][lane];
            part[o + 2 * C + c] = acc_s[2 * kSH + 2][lane];
            part[o + 3 * C + c] = acc_s[2 * kSH + 3][lane];
        }
        __syncthreads();
    }
    if (lane == 0) {
#pragma unroll
        for (int j = 0; j < kTokPerWarp; ++j) {
            m12[0][warp + j * kWarps] = s1[j] / (float)C;
            m12[1][warp + j * kWarps] = s2[j] / (float)C;
        }
    }
    __syncthreads();
    // dx = rstd (dn - mean(dn) - n mean(dn n)), over the dn this CTA wrote above
    for (int e = threadIdx.x; e < C * kTT; e += kThreads) {
        const int c = e / kTT, tok = e % kTT;
        if (tok >= nt) continue;
        const size_t i = ((size_t)bv * C + c) * a.hw + t0 + tok;
        const float n = (__ldg(a.x + i) - sm.mean[tok]) * sm.rstd[tok];
        a.gx[i] = sm.rstd[tok] * (a.gx[i] - m12[0][tok] - n * m12[1][tok]);
    }
}

__device__ __forceinline__ PfTaps voxel_taps(const Args& a, int bv, int g, int& cell) {
    const float* p = a.grid + 3 * (size_t)g;
    float px, py, pz, m[21];
    pf_project(a.w2c + 16 * (size_t)bv, a.ixt + 9 * (size_t)bv, __ldg(p), __ldg(p + 1), __ldg(p + 2), px, py, pz, m);
    const float ix = pf_source_coord(__fdiv_rn(px, pz), (float)a.Wimg, (float)a.w);
    const float iy = pf_source_coord(__fdiv_rn(py, pz), (float)a.Himg, (float)a.h);
    const PfTaps t = pf_taps(ix, iy, a.w, a.h);
    cell = t.any ? ((int)floorf(iy) + 1) * (a.w + 1) + (int)floorf(ix) + 1 : -1;
    return t;
}

// row of voxel g of view v of scene b in the condition layout [B g^3, V bs^3, C+E]
__device__ __forceinline__ size_t cond_row(const Args& a, int b, int v, int g) {
    const int R = a.R, ng = a.ng, bs = R / ng, bs3 = bs * bs * bs;
    const int i = g / (R * R), j = (g / R) % R, k = g % R;
    const int G = ((i / bs) * ng + j / bs) * ng + k / bs;
    const int l = ((i % bs) * bs + j % bs) * bs + k % bs;
    return ((size_t)b * ng * ng * ng + G) * ((size_t)a.V * bs3) + (size_t)v * bs3 + l;
}

__device__ __forceinline__ float sample_channel(const float* yb, const int* off, const float* w, int C, int c) {
    float s = 0.0f;
#pragma unroll
    for (int k = 0; k < 4; ++k)
        if (off[k] >= 0) s = __fmaf_rn(__ldg(yb + (size_t)off[k] * C + c), w[k], s);
    return s;
}

template <bool kCond>
__global__ void __launch_bounds__(kThreads) fv_sample_kernel(Args a) {
    __shared__ int off_s[kVT][4];
    __shared__ float w_s[kVT][4];
    __shared__ float T[32][kVT + 1];
    const int bv = blockIdx.y, g0 = blockIdx.x * kVT, nv = min(kVT, a.R3 - g0);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, C = a.C;
    if (threadIdx.x < kVT) {
        int cell;
        const PfTaps t = threadIdx.x < nv ? voxel_taps(a, bv, g0 + threadIdx.x, cell) : PfTaps{0, 0, 0, 0, {0, 0, 0, 0}, {-1, -1, -1, -1}, false};
#pragma unroll
        for (int k = 0; k < 4; ++k) { off_s[threadIdx.x][k] = t.off[k]; w_s[threadIdx.x][k] = t.w[k]; }
    }
    __syncthreads();
    const float* yb = a.y + (size_t)bv * a.hw * C;
    if (kCond) {
        const int b = bv / a.V, v = bv % a.V;
        for (int vi = warp; vi < nv; vi += kWarps) {
            float* o = a.out + cond_row(a, b, v, g0 + vi) * (size_t)(C + a.E);
            for (int c = lane; c < C; c += 32) o[c] = sample_channel(yb, off_s[vi], w_s[vi], C, c);
            for (int e = lane; e < a.E; e += 32) o[C + e] = __ldg(a.ve + (size_t)v * a.E + e);
        }
    } else {
        for (int c0 = 0; c0 < C; c0 += 32) {
            for (int vi = warp; vi < kVT; vi += kWarps)
                T[lane][vi] = vi < nv ? sample_channel(yb, off_s[vi], w_s[vi], C, c0 + lane) : 0.0f;
            __syncthreads();
            for (int cl = warp; cl < 32; cl += kWarps)
                if (lane < nv) a.out[((size_t)bv * C + c0 + cl) * a.R3 + g0 + lane] = T[cl][lane];
            __syncthreads();
        }
    }
}

__global__ void __launch_bounds__(kThreads) fv_cell_kernel(Args a) {
    const int bv = blockIdx.y, g = blockIdx.x * kThreads + threadIdx.x;
    if (g >= a.R3) return;
    int cell;
    const PfTaps t = voxel_taps(a, bv, g, cell);
    const size_t i = (size_t)bv * a.R3 + g;
    a.wts[i] = make_float4(t.w[0], t.w[1], t.w[2], t.w[3]);
    a.cell[i] = cell;
    if (cell >= 0) atomicAdd(a.count + (size_t)bv * a.ncells + cell, 1);
}

// start = exclusive scan of the counts (and a copy into count, the placement cursors)
__global__ void __launch_bounds__(1024) fv_scan_kernel(Args a) {
    __shared__ int wsum[32];
    const int bv = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int* cnt = a.count + (size_t)bv * a.ncells;
    int* st = a.start + (size_t)bv * (a.ncells + 1);
    int carry = 0;
    for (int base = 0; base < a.ncells; base += 1024) {
        const int i = base + threadIdx.x;
        const int v = i < a.ncells ? cnt[i] : 0;
        int incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int u = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += u;
        }
        if (lane == 31) wsum[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            int s = wsum[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int u = __shfl_up_sync(0xffffffffu, s, o);
                if (lane >= o) s += u;
            }
            wsum[lane] = s;
        }
        __syncthreads();
        const int ex = carry + (warp ? wsum[warp - 1] : 0) + incl - v;
        if (i < a.ncells) { st[i] = ex; cnt[i] = ex; }
        carry += wsum[31];
        __syncthreads();
    }
    if (threadIdx.x == 0) st[a.ncells] = carry;
}

__global__ void __launch_bounds__(kRound) fv_place_kernel(Args a) {
    __shared__ unsigned long long keys[kRound];
    const int bv = blockIdx.x, tid = threadIdx.x;
    int* cursor = a.count + (size_t)bv * a.ncells;
    int* list = a.list + (size_t)bv * a.R3;
    const int* cells = a.cell + (size_t)bv * a.R3;
    constexpr unsigned long long kNone = ~0ull;
    for (int r0 = 0; r0 < a.R3; r0 += kRound) {
        const int c = r0 + tid < a.R3 ? cells[r0 + tid] : -1;
        keys[tid] = c >= 0 ? ((unsigned long long)c << 10) | (unsigned)tid : kNone;
        __syncthreads();
        for (int k = 2; k <= kRound; k <<= 1) {
            for (int j = k >> 1; j > 0; j >>= 1) {
                const int p = tid ^ j;
                if (p > tid) {
                    const unsigned long long u = keys[tid], v = keys[p];
                    if ((u > v) == ((tid & k) == 0)) { keys[tid] = v; keys[p] = u; }
                }
                __syncthreads();
            }
        }
        const unsigned long long key = keys[tid];
        bool last = false;
        int rank = 0, cc = 0;
        if (key != kNone) {
            cc = (int)(key >> 10);
            int lo = 0, hi = tid;                  // first position holding cell cc
            while (lo < hi) {
                const int m = (lo + hi) >> 1;
                if ((keys[m] >> 10) < (unsigned long long)cc) lo = m + 1; else hi = m;
            }
            rank = tid - lo;
            list[cursor[cc] + rank] = r0 + (int)(key & 1023);
            last = tid == kRound - 1 || (keys[tid + 1] >> 10) != (unsigned long long)cc;
        }
        __syncthreads();
        if (last) cursor[cc] += rank + 1;
        __syncthreads();
    }
}

template <bool kCond>
__global__ void __launch_bounds__(kThreads) fv_gather_kernel(Args a) {
    const int lane = threadIdx.x & 31;
    const long long gt = (long long)blockIdx.x * kWarps + (threadIdx.x >> 5);
    if (gt >= (long long)a.B * a.V * a.hw) return;
    const int bv = (int)(gt / a.hw), t = (int)(gt % a.hw), ty = t / a.w, tx = t % a.w;
    const int b = bv / a.V, v = bv % a.V, C = a.C, nj = C / 32, W1 = a.w + 1;
    const int* st = a.start + (size_t)bv * (a.ncells + 1);
    const int* list = a.list + (size_t)bv * a.R3;
    const float4* wts = a.wts + (size_t)bv * a.R3;
    float acc[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) acc[j] = 0.0f;
    // the token is tap nw of cell (x, y), ne of (x-1, y), sw of (x, y-1), se of (x-1, y-1)
    const int cells[4] = {(ty + 1) * W1 + tx + 1, (ty + 1) * W1 + tx, ty * W1 + tx + 1, ty * W1 + tx};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int end = __ldg(st + cells[k] + 1);
        for (int p = __ldg(st + cells[k]); p < end; ++p) {
            const int g = __ldg(list + p);
            const float4 w4 = __ldg(wts + g);
            const float wk = k == 0 ? w4.x : k == 1 ? w4.y : k == 2 ? w4.z : w4.w;
            if (kCond) {
                const float* row = a.gout + cond_row(a, b, v, g) * (size_t)(C + a.E);
#pragma unroll
                for (int j = 0; j < 32; ++j)
                    if (j < nj) acc[j] = fmaf(wk, __ldg(row + lane + 32 * j), acc[j]);
            } else {
                const float* col = a.gout + (size_t)bv * C * a.R3 + g;
#pragma unroll
                for (int j = 0; j < 32; ++j)
                    if (j < nj) acc[j] = fmaf(wk, __ldg(col + (size_t)(lane + 32 * j) * a.R3), acc[j]);
            }
        }
    }
    float* dy = a.y + (size_t)gt * C;
#pragma unroll
    for (int j = 0; j < 32; ++j)
        if (j < nj) dy[lane + 32 * j] = acc[j];
}

// per-slice sums over the B R^3 rows of view v of the view-embedding columns of dL/dout (condition layout)
__global__ void __launch_bounds__(kThreads) fv_view_embed_kernel(Args a) {
    __shared__ float red[kWarps][32];
    const int v = blockIdx.x, e = blockIdx.y * 32 + (threadIdx.x & 31), grp = threadIdx.x >> 5;
    const int bs = a.R / a.ng, bs3 = bs * bs * bs;
    const long long n = (long long)a.B * a.R3;
    const long long lo = n * blockIdx.z / kVeSlices, hi = n * (blockIdx.z + 1) / kVeSlices;
    float s = 0.0f;
    if (e < a.E)
        for (long long j = lo + grp; j < hi; j += kWarps) {
            const long long row = (j / bs3 * a.V + v) * bs3 + j % bs3;
            s += __ldg(a.gout + row * (a.C + a.E) + a.C + e);
        }
    red[grp][threadIdx.x & 31] = s;
    __syncthreads();
    if (grp == 0 && e < a.E) {
        float t = 0.0f;
#pragma unroll
        for (int q = 0; q < kWarps; ++q) t += red[q][threadIdx.x];
        a.ve_parts[((size_t)blockIdx.z * a.V + v) * a.E + e] = t;
    }
}

struct WsLayout { size_t y, wts, cell, count, start, list, parts, ve_parts, total; };

WsLayout ws_layout(int B, int V, int C, int h, int w, int R, int E) {
    const size_t BV = (size_t)B * V, hw = (size_t)h * w, R3 = (size_t)R * R * R, ncells = (size_t)(h + 1) * (w + 1);
    const size_t ntiles = (hw + kTT - 1) / kTT;
    WsLayout l;
    l.y = 0;
    l.wts = align_up(l.y + sizeof(float) * BV * hw * C);
    l.cell = align_up(l.wts + sizeof(float4) * BV * R3);
    l.count = align_up(l.cell + sizeof(int) * BV * R3);
    l.start = align_up(l.count + sizeof(int) * BV * ncells);
    l.list = align_up(l.start + sizeof(int) * BV * (ncells + 1));
    l.parts = align_up(l.list + sizeof(int) * BV * R3);
    l.ve_parts = align_up(l.parts + sizeof(float) * BV * ntiles * C * kAcc);
    l.total = align_up(l.ve_parts + sizeof(float) * kVeSlices * V * E);
    return l;
}

int check_sizes(const char* fn, int B, int V, int C, int h, int w, int R, int E) {
    if (B < 1 || V < 1 || V > 8 || (long long)B * V > 65535)
        return set_error("%s: bad sizes (B=%d, V=%d): need B >= 1, 1 <= V <= 8 and B*V <= 65535", fn, B, V);
    if (C < 32 || C > 1024 || C % 32 != 0)
        return set_error("%s: bad sizes (C=%d): need a multiple of 32 up to 1024", fn, C);
    if (h < 1 || w < 1 || h > (1 << 24) || w > (1 << 24) || (long long)(h + 1) * (w + 1) > INT32_MAX)
        return set_error("%s: bad sizes (h=%d, w=%d): need h, w >= 1 and (h+1)(w+1) < 2^31", fn, h, w);
    if (R < 1 || R > 64) return set_error("%s: bad sizes (R=%d): need 1 <= R <= 64", fn, R);
    if (E < 0 || E > 128) return set_error("%s: bad sizes (E=%d): need 0 <= E <= 128", fn, E);
    return 0;
}

int check_call(const char* fn, int B, int V, int C, int h, int w, int R, int E, int Vmax, int H_img, int W_img,
               int n_group) {
    if (check_sizes(fn, B, V, C, h, w, R, E)) return 1;
    if (E > 0 && Vmax < V) return set_error("%s: bad sizes (Vmax=%d, V=%d): view_embed has fewer rows than views", fn, Vmax, V);
    if (H_img < 1 || W_img < 1) return set_error("%s: bad sizes (H_img=%d, W_img=%d)", fn, H_img, W_img);
    if (n_group < 0 || (n_group > 0 && R % n_group != 0))
        return set_error("%s: bad layout (n_group=%d): need 0 (drop-in) or a divisor of R=%d", fn, n_group, R);
    if (n_group == 0 && E != 0) return set_error("%s: bad layout: the drop-in layout has no view embedding (E=%d)", fn, E);
    return 0;
}

Args make_args(int B, int V, int C, int h, int w, int R, int E, int H_img, int W_img, int n_group,
               const float* img_feats, const float* rays, const float* w2c, const float* ixt, const float* grid,
               const float* norm_w, const float* norm_b, const float* mlp_w, const float* mlp_b, void* workspace) {
    Args a;
    memset(&a, 0, sizeof(a));
    a.B = B; a.V = V; a.C = C; a.h = h; a.w = w; a.R = R; a.E = E; a.ng = n_group; a.Himg = H_img; a.Wimg = W_img;
    a.hw = h * w; a.R3 = R * R * R; a.ncells = (h + 1) * (w + 1); a.ntiles = (a.hw + kTT - 1) / kTT;
    a.x = img_feats; a.rays = rays; a.w2c = w2c; a.ixt = ixt; a.grid = grid;
    a.ln_w = norm_w; a.ln_b = norm_b; a.mlp_w = mlp_w; a.mlp_b = mlp_b;
    const WsLayout l = ws_layout(B, V, C, h, w, R, E);
    char* ws = static_cast<char*>(workspace);
    a.y = reinterpret_cast<float*>(ws + l.y);
    a.wts = reinterpret_cast<float4*>(ws + l.wts);
    a.cell = reinterpret_cast<int*>(ws + l.cell);
    a.count = reinterpret_cast<int*>(ws + l.count);
    a.start = reinterpret_cast<int*>(ws + l.start);
    a.list = reinterpret_cast<int*>(ws + l.list);
    a.parts = reinterpret_cast<float*>(ws + l.parts);
    a.ve_parts = reinterpret_cast<float*>(ws + l.ve_parts);
    return a;
}

}  // namespace
}  // namespace srf

using srf::cuda_error;
using srf::set_error;

extern "C" int srf_feat_volume_workspace_bytes(int B, int V, int C, int h, int w, int R, int E, size_t* bytes) {
    const char* fn = "srf_feat_volume_workspace_bytes";
    if (srf::check_sizes(fn, B, V, C, h, w, R, E)) return 1;
    if (!bytes) return set_error("%s: null output", fn);
    *bytes = srf::ws_layout(B, V, C, h, w, R, E).total;
    return 0;
}

extern "C" int srf_feat_volume_forward(void* stream_, int B, int V, int C, int h, int w, int R, int E, int Vmax,
                                       int H_img, int W_img, int n_group, const float* img_feats, const float* rays,
                                       const float* w2c, const float* ixt, const float* grid, const float* norm_w,
                                       const float* norm_b, const float* mlp_w, const float* mlp_b,
                                       const float* view_embed, void* workspace, float* out) {
    const char* fn = "srf_feat_volume_forward";
    if (srf::check_call(fn, B, V, C, h, w, R, E, Vmax, H_img, W_img, n_group)) return 1;
    if (!img_feats || !rays || !w2c || !ixt || !grid) return set_error("%s: null input pointer", fn);
    if (!norm_w || !norm_b || !mlp_w || !mlp_b) return set_error("%s: null weight pointer", fn);
    if (E > 0 && !view_embed) return set_error("%s: null view_embed with E=%d", fn, E);
    if (!out) return set_error("%s: null output pointer", fn);
    if (!workspace || srf::misaligned(workspace)) return set_error("%s: workspace must be 256-byte aligned", fn);
    srf::Args a = srf::make_args(B, V, C, h, w, R, E, H_img, W_img, n_group, img_feats, rays, w2c, ixt, grid, norm_w,
                                 norm_b, mlp_w, mlp_b, workspace);
    a.ve = view_embed;
    a.out = out;
    const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const unsigned BV = (unsigned)(B * V);
    srf::fv_token_fwd_kernel<<<dim3((unsigned)a.ntiles, BV), srf::kThreads, 0, stream>>>(a);
    const dim3 sgrid((unsigned)((a.R3 + srf::kVT - 1) / srf::kVT), BV);
    if (n_group > 0) srf::fv_sample_kernel<true><<<sgrid, srf::kThreads, 0, stream>>>(a);
    else srf::fv_sample_kernel<false><<<sgrid, srf::kThreads, 0, stream>>>(a);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_error("feat_volume forward launch", e);
}

extern "C" int srf_feat_volume_backward(void* stream_, int B, int V, int C, int h, int w, int R, int E, int Vmax,
                                        int H_img, int W_img, int n_group, const float* img_feats, const float* rays,
                                        const float* w2c, const float* ixt, const float* grid, const float* norm_w,
                                        const float* norm_b, const float* mlp_w, const float* mlp_b,
                                        const float* dL_dout, void* workspace, float* dL_dimg_feats, float* d_norm_w,
                                        float* d_norm_b, float* d_mlp_w, float* d_mlp_b, float* d_view_embed) {
    const char* fn = "srf_feat_volume_backward";
    if (srf::check_call(fn, B, V, C, h, w, R, E, Vmax, H_img, W_img, n_group)) return 1;
    if (!img_feats || !rays || !w2c || !ixt || !grid) return set_error("%s: null input pointer", fn);
    if (!norm_w || !norm_b || !mlp_w || !mlp_b) return set_error("%s: null weight pointer", fn);
    if (!dL_dout) return set_error("%s: null upstream gradient", fn);
    if (!dL_dimg_feats || !d_norm_w || !d_norm_b || !d_mlp_w || !d_mlp_b || (E > 0 && !d_view_embed))
        return set_error("%s: null gradient pointer", fn);
    if (!workspace || srf::misaligned(workspace)) return set_error("%s: workspace must be 256-byte aligned", fn);
    srf::Args a = srf::make_args(B, V, C, h, w, R, E, H_img, W_img, n_group, img_feats, rays, w2c, ixt, grid, norm_w,
                                 norm_b, mlp_w, mlp_b, workspace);
    a.gout = dL_dout;
    a.gx = dL_dimg_feats;
    const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const unsigned BV = (unsigned)(B * V);
    cudaError_t e = cudaMemsetAsync(a.count, 0, sizeof(int) * (size_t)BV * a.ncells, stream);
    if (e != cudaSuccess) return cuda_error("memset feat_volume counts", e);
    if (E > 0 && (e = cudaMemsetAsync(d_view_embed, 0, sizeof(float) * (size_t)Vmax * E, stream)) != cudaSuccess)
        return cuda_error("memset d_view_embed", e);
    srf::fv_cell_kernel<<<dim3((unsigned)((a.R3 + srf::kThreads - 1) / srf::kThreads), BV), srf::kThreads, 0, stream>>>(a);
    srf::fv_scan_kernel<<<BV, 1024, 0, stream>>>(a);
    srf::fv_place_kernel<<<BV, srf::kRound, 0, stream>>>(a);
    const unsigned ggrid = (unsigned)(((long long)BV * a.hw + srf::kWarps - 1) / srf::kWarps);
    if (n_group > 0) srf::fv_gather_kernel<true><<<ggrid, srf::kThreads, 0, stream>>>(a);
    else srf::fv_gather_kernel<false><<<ggrid, srf::kThreads, 0, stream>>>(a);
    srf::fv_token_bwd_kernel<<<dim3((unsigned)a.ntiles, BV), srf::kThreads, 0, stream>>>(a);
    srf::part_sums(stream, a.parts, (int)BV * a.ntiles, (size_t)C * srf::kAcc,
                   srf::seg(d_mlp_w, 2 * C * srf::kSH), srf::seg(d_mlp_b, 2 * C), srf::seg(d_norm_w, C),
                   srf::seg(d_norm_b, C));
    if (E > 0) {
        srf::fv_view_embed_kernel<<<dim3((unsigned)V, (unsigned)((E + 31) / 32), srf::kVeSlices), srf::kThreads, 0,
                                    stream>>>(a);
        srf::part_sums(stream, a.ve_parts, srf::kVeSlices, (size_t)V * E, srf::seg(d_view_embed, V * E));
    }
    e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_error("feat_volume backward launch", e);
}
