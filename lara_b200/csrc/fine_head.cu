// fine_head.cu -- fused fine-pass decoder head of LaRa (Decoder.forward_fine, lightning/network.py:280-284, with the
// mask gathers and residual of :508-512), DESIGN §3.16.  The C entries of include/surfel_fine_head.h are defined here.
//
// Per point p (fp32), with the head algebra reassociated (DESIGN §3.16 says why):
//   x   = LayerNorm(vf)                                  vf = volume_feat[row(p)], eps 1e-5, affine
//   r   = A x,          A_h  = s Wk_h^T Wq_h  [8, D]     64 values: per head the query seen in the 8-dim key space
//   s_hj = r_h . f_j;   a_h = softmax_j(s_h)            max subtracted, as SDPA does
//   c_h = sum_j a_hj f_j                                 64 values
//   z   = W1c c + b1,   W1c = W1 Wo blockdiag(Wv_h)  [64, 64]
//   sh  = W2 relu(z) + b2 (+ shs_coarse[idx(p)])
// A and W1c are composed per CTA in fp64 and rounded once.  The per-point products run as register-tiled SIMT FMA
// loops over a tile of kTP points whose activations sit in shared memory feature-major ([feature][kTP]).
//
// The backward recomputes the forward per tile and keeps nothing else.  The weight gradients of the composed
// matrices (dA = sum dr x^T, dW1c = sum dz c^T, ...) are summed per CTA in shared memory, each element by one thread
// in tile order, written as per-CTA partials, then summed over the CTAs in fp64 in a fixed order; the gradients of
// Wq, Wk, Wv, Wo and W1 follow from dA and dW1c by the chain rule through the compositions, in fp64.  The voxel-row
// gradient of the gather mode is a gather over the per-point rows (idx is strictly increasing).  No atomics.
#include "../../include/surfel_fine_head.h"
#include "fixed_sums.cuh"
#include "surfel_kernels.h"

namespace srf {
namespace {

constexpr int kTP = 32;             // points per tile
constexpr int kThreads = 256;       // = kTP * 8 heads: the attention steps run one thread per (point, head)
constexpr int kHeads = 8, kCond = 8, kHid = 64, kHK = kHeads * kCond;   // kHK = 64: (head, cond) pairs
constexpr int kTS = kTP + 1;        // row stride of the padded transpose buffer
constexpr float kEps = 1e-5f;
static_assert(kThreads == kTP * kHeads, "one thread per (point, head)");

struct Args {
    int n, V, D, S, Sp, K;           // Sp: sh_dim rounded up to 4
    long long NK;                    // N * K rows of shs_coarse (gather mode)
    const float* vf;                 // [N or n, D]
    const int* idx;                  // [n] or null (plain mode: row p, no residual)
    const float* pf;                 // [V, 8, n]
    const float* shs;                // [N*K, S] or null
    const float *ln_w, *ln_b, *wq, *wk, *wv, *wo, *w1, *b1, *w2, *b2;
    float* out;                      // forward: [n, S]
    const float* g;                  // backward: [n, S]
    float* g_rows;                   // [n, D]: per-point volume-feature gradient (the output in plain mode)
    float* g_pf;                     // [V, 8, n]
    float* g_shs;                    // [N*K, S] (rows not in idx zeroed by the caller) or null
    float* partials;                 // [gridDim.x, nacc]
};

// shared-memory layout in floats; every region starts on a 16-byte boundary
struct Layout {
    int A, W1c, W2, b1, b2, lw, lb;                  // weights
    int XH, X, F, R, PA, C, Z, G, E, red, rstd;      // tile activations ([rows][kTP]); T aliases F..E
    int acc;                                         // backward: weight-gradient accumulators (nacc)
    int dA, dW1c, dW2, db1, db2, dlw, dlb, nacc;     // offsets inside acc
    int fwd_floats, bwd_floats;
};

__host__ __device__ inline Layout layout(int D, int Sp) {
    Layout l;
    int o = 0;
    l.A = o; o += kHK * D;
    l.W1c = o; o += kHid * kHK;
    l.W2 = o; o += Sp * kHid;
    l.b1 = o; o += kHid;
    l.b2 = o; o += Sp;
    l.lw = o; o += D;
    l.lb = o; o += D;
    l.XH = o; o += D * kTP;
    l.X = o; o += D * kTP;
    l.F = o; o += 64 * kTP;
    l.R = o; o += 64 * kTP;
    l.PA = o; o += 64 * kTP;
    l.C = o; o += 64 * kTP;
    l.Z = o; o += 64 * kTP;
    l.G = o; o += 64 * kTP;
    l.E = o; o += 64 * kTP;
    l.red = o; o += 2 * 8 * kTP;
    l.rstd = o; o += kTP;
    l.fwd_floats = o;
    l.acc = o;
    int a = 0;
    l.dA = a; a += kHK * D;
    l.dW1c = a; a += kHid * kHK;
    l.dW2 = a; a += Sp * kHid;
    l.db1 = a; a += kHid;
    l.db2 = a; a += Sp;
    l.dlw = a; a += D;
    l.dlb = a; a += D;
    l.nacc = a;
    l.bwd_floats = o + a;
    return l;
}

// out[o][p] = sum_i W[o so + i si] in'[i][p] (+ bias[o]) for o < No; in' = relu(in) if RELU; with `mask`, out is 0
// where mask[o][p] <= 0.  Each thread computes 2 outputs x 4 points; the sum over i runs in order.
template <bool RELU>
__device__ __forceinline__ void tile_gemm(float* out, const float* in, const float* W, int so, int si, int No, int Ni,
                                          const float* bias, const float* mask) {
    const int nb = (No / 2) * (kTP / 4);
    for (int b = threadIdx.x; b < nb; b += kThreads) {
        const int pb = (b % (kTP / 4)) * 4, ob = (b / (kTP / 4)) * 2;
        float acc[2][4] = {};
        const float* w = W + ob * so;
        for (int i = 0; i < Ni; ++i) {
            float4 x = *reinterpret_cast<const float4*>(in + i * kTP + pb);
            if (RELU) { x.x = fmaxf(x.x, 0.f); x.y = fmaxf(x.y, 0.f); x.z = fmaxf(x.z, 0.f); x.w = fmaxf(x.w, 0.f); }
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const float wr = w[i * si + r * so];
                acc[r][0] = fmaf(wr, x.x, acc[r][0]); acc[r][1] = fmaf(wr, x.y, acc[r][1]);
                acc[r][2] = fmaf(wr, x.z, acc[r][2]); acc[r][3] = fmaf(wr, x.w, acc[r][3]);
            }
        }
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const int o = ob + r;
            if (bias) {
#pragma unroll
                for (int c = 0; c < 4; ++c) acc[r][c] += bias[o];
            }
            if (mask) {
#pragma unroll
                for (int c = 0; c < 4; ++c) acc[r][c] = mask[o * kTP + pb + c] > 0.f ? acc[r][c] : 0.f;
            }
            *reinterpret_cast<float4*>(out + o * kTP + pb) = make_float4(acc[r][0], acc[r][1], acc[r][2], acc[r][3]);
        }
    }
}

// acc[o Ni + i] += sum_p a[o][p] b'[i][p] over the tile (b' = relu(b) if RELU); 4 x 4 outputs per thread, each
// output owned by one thread, the tile's sum formed in point order and then added.
template <bool RELU>
__device__ __forceinline__ void tile_outer_acc(float* acc, const float* a, const float* b, int No, int Ni) {
    const int nib = Ni / 4, nb = (No / 4) * nib;
    for (int blk = threadIdx.x; blk < nb; blk += kThreads) {
        const int ob = (blk / nib) * 4, ib = (blk % nib) * 4;
        float s[4][4] = {};
        for (int p = 0; p < kTP; p += 4) {
            float4 av[4], bv[4];
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                av[r] = *reinterpret_cast<const float4*>(a + (ob + r) * kTP + p);
                bv[r] = *reinterpret_cast<const float4*>(b + (ib + r) * kTP + p);
                if (RELU) {
                    bv[r].x = fmaxf(bv[r].x, 0.f); bv[r].y = fmaxf(bv[r].y, 0.f);
                    bv[r].z = fmaxf(bv[r].z, 0.f); bv[r].w = fmaxf(bv[r].w, 0.f);
                }
            }
#pragma unroll
            for (int r = 0; r < 4; ++r)
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    s[r][c] = fmaf(av[r].x, bv[c].x, s[r][c]); s[r][c] = fmaf(av[r].y, bv[c].y, s[r][c]);
                    s[r][c] = fmaf(av[r].z, bv[c].z, s[r][c]); s[r][c] = fmaf(av[r].w, bv[c].w, s[r][c]);
                }
        }
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
            for (int c = 0; c < 4; ++c) acc[(ob + r) * Ni + ib + c] += s[r][c];
    }
}

// acc[o] += sum_p a[o][p] (b ? b[o][p] : 1) for o < No
__device__ __forceinline__ void tile_row_acc(float* acc, const float* a, const float* b, int No) {
    for (int o = threadIdx.x; o < No; o += kThreads) {
        float s = 0.f;
        for (int p = 0; p < kTP; ++p) s = b ? fmaf(a[o * kTP + p], b[o * kTP + p], s) : s + a[o * kTP + p];
        acc[o] += s;
    }
}

// Weights into shared memory, with A and W1c composed in fp64 (the composition scratch aliases the activations).
__device__ void load_weights(const Args& a, const Layout& l, float* sm) {
    const int D = a.D, hd = D / kHeads;
    const double scale = 1.0 / sqrt((double)hd);
    for (int e = threadIdx.x; e < kHK * D; e += kThreads) {          // A[h8+k][d] = s sum_i Wk[h hd+i][k] Wq[h hd+i][d]
        const int hk = e / D, d = e % D, h = hk / kCond, k = hk % kCond;
        double s = 0.0;
        for (int i = 0; i < hd; ++i)
            s += (double)__ldg(a.wk + (h * hd + i) * kCond + k) * (double)__ldg(a.wq + (size_t)(h * hd + i) * D + d);
        sm[l.A + e] = (float)(s * scale);
    }
    double* B = reinterpret_cast<double*>(sm + l.XH);                 // B[d][h8+k] = sum_i Wo[d][h hd+i] Wv[h hd+i][k]
    for (int e = threadIdx.x; e < D * kHK; e += kThreads) {
        const int d = e / kHK, hk = e % kHK, h = hk / kCond, k = hk % kCond;
        double s = 0.0;
        for (int i = 0; i < hd; ++i)
            s += (double)__ldg(a.wo + (size_t)d * D + h * hd + i) * (double)__ldg(a.wv + (h * hd + i) * kCond + k);
        B[e] = s;
    }
    for (int e = threadIdx.x; e < a.Sp * kHid; e += kThreads)
        sm[l.W2 + e] = e / kHid < a.S ? __ldg(a.w2 + e) : 0.f;
    for (int e = threadIdx.x; e < kHid; e += kThreads) sm[l.b1 + e] = __ldg(a.b1 + e);
    for (int e = threadIdx.x; e < a.Sp; e += kThreads) sm[l.b2 + e] = e < a.S ? __ldg(a.b2 + e) : 0.f;
    for (int e = threadIdx.x; e < D; e += kThreads) {
        sm[l.lw + e] = __ldg(a.ln_w + e);
        sm[l.lb + e] = __ldg(a.ln_b + e);
    }
    __syncthreads();
    for (int e = threadIdx.x; e < kHid * kHK; e += kThreads) {       // W1c[m][hk] = sum_d W1[m][d] B[d][hk]
        const int m = e / kHK, hk = e % kHK;
        double s = 0.0;
        for (int d = 0; d < D; ++d) s += (double)__ldg(a.w1 + (size_t)m * D + d) * B[d * kHK + hk];
        sm[l.W1c + e] = (float)s;
    }
    __syncthreads();
}

__device__ __forceinline__ long long row_of(const Args& a, int p) {
    if (!a.idx) return p;
    const int id = __ldg(a.idx + p);
    return (id >= 0 && id < a.NK) ? id / a.K : -1;          // an index out of range reads a zero row
}

// Tile forward up to z = W1c c + b1 in Z; leaves xhat (XH), x (X), f (F), r (R), a (PA), c (C) and rstd.
__device__ void tile_forward(const Args& a, const Layout& l, float* sm, int p0) {
    const int D = a.D, V = a.V, tid = threadIdx.x;
    float* T = sm + l.F;                                       // padded transpose buffer [D][kTS]
    for (int e = tid; e < kTP * D; e += kThreads) {            // rows read along d (coalesced)
        const int p = e / D, d = e % D;
        const long long row = p0 + p < a.n ? row_of(a, p0 + p) : -1;
        T[d * kTS + p] = row >= 0 ? __ldg(a.vf + row * D + d) : 0.f;
    }
    __syncthreads();
    {   // LayerNorm: 8 slices of d per point, two passes (mean, then the centred variance)
        const int p = tid % kTP, sub = tid / kTP;
        float* red = sm + l.red;
        float s = 0.f;
        for (int d = sub; d < D; d += 8) s += T[d * kTS + p];
        red[sub * kTP + p] = s;
        __syncthreads();
        s = 0.f;
#pragma unroll
        for (int q = 0; q < 8; ++q) s += red[q * kTP + p];
        const float mean = s / (float)D;
        float v = 0.f;
        for (int d = sub; d < D; d += 8) {
            const float t = T[d * kTS + p] - mean;
            v = fmaf(t, t, v);
        }
        red[8 * kTP + sub * kTP + p] = v;
        __syncthreads();
        v = 0.f;
#pragma unroll
        for (int q = 0; q < 8; ++q) v += red[8 * kTP + q * kTP + p];
        const float rstd = 1.0f / sqrtf(v / (float)D + kEps);
        if (sub == 0) sm[l.rstd + p] = rstd;
        for (int d = sub; d < D; d += 8) {
            const float xh = (T[d * kTS + p] - mean) * rstd;
            sm[l.XH + d * kTP + p] = xh;
            sm[l.X + d * kTP + p] = fmaf(xh, sm[l.lw + d], sm[l.lb + d]);
        }
    }
    __syncthreads();                                           // T is dead: F overwrites it
    for (int e = tid; e < V * kCond * kTP; e += kThreads) {
        const int jk = e / kTP, p = e % kTP;
        sm[l.F + e] = p0 + p < a.n ? __ldg(a.pf + (size_t)jk * a.n + p0 + p) : 0.f;
    }
    tile_gemm<false>(sm + l.R, sm + l.X, sm + l.A, D, 1, kHK, D, nullptr, nullptr);
    __syncthreads();
    {   // attention, one thread per (point, head)
        const int p = tid % kTP, h = tid / kTP;
        float r[kCond], s[8];
#pragma unroll
        for (int k = 0; k < kCond; ++k) r[k] = sm[l.R + (h * kCond + k) * kTP + p];
        float m = -INFINITY;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            if (j < V) {
                float t = 0.f;
#pragma unroll
                for (int k = 0; k < kCond; ++k) t = fmaf(r[k], sm[l.F + (j * kCond + k) * kTP + p], t);
                s[j] = t;
                m = fmaxf(m, t);
            }
        }
        float sum = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j)
            if (j < V) { s[j] = expf(s[j] - m); sum += s[j]; }
        float c[kCond] = {};
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            if (j < V) {
                const float aj = s[j] / sum;
                sm[l.PA + (h * V + j) * kTP + p] = aj;
#pragma unroll
                for (int k = 0; k < kCond; ++k) c[k] = fmaf(aj, sm[l.F + (j * kCond + k) * kTP + p], c[k]);
            }
        }
#pragma unroll
        for (int k = 0; k < kCond; ++k) sm[l.C + (h * kCond + k) * kTP + p] = c[k];
    }
    __syncthreads();
    tile_gemm<false>(sm + l.Z, sm + l.C, sm + l.W1c, kHK, 1, kHid, kHK, sm + l.b1, nullptr);
    __syncthreads();
}

__global__ void __launch_bounds__(kThreads, 1) fine_head_fwd_kernel(Args a) {
    extern __shared__ __align__(16) float sm[];
    const Layout l = layout(a.D, a.Sp);
    load_weights(a, l, sm);
    const int ntiles = (a.n + kTP - 1) / kTP;
    for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const int p0 = t * kTP;
        tile_forward(a, l, sm, p0);
        tile_gemm<true>(sm + l.G, sm + l.Z, sm + l.W2, kHid, 1, a.Sp, kHid, sm + l.b2, nullptr);
        __syncthreads();
        for (int e = threadIdx.x; e < kTP * a.S; e += kThreads) {
            const int p = e / a.S, s = e % a.S;
            if (p0 + p >= a.n) break;
            float v = sm[l.G + s * kTP + p];
            if (a.shs) {
                const int id = __ldg(a.idx + p0 + p);
                if (id >= 0 && id < a.NK) v += __ldg(a.shs + (size_t)id * a.S + s);
            }
            a.out[(size_t)(p0 + p) * a.S + s] = v;
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(kThreads, 1) fine_head_bwd_kernel(Args a) {
    extern __shared__ __align__(16) float sm[];
    const Layout l = layout(a.D, a.Sp);
    const int D = a.D, V = a.V, tid = threadIdx.x;
    float* acc = sm + l.acc;
    for (int e = tid; e < l.nacc; e += kThreads) acc[e] = 0.f;
    load_weights(a, l, sm);
    const int ntiles = (a.n + kTP - 1) / kTP;
    for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const int p0 = t * kTP;
        tile_forward(a, l, sm, p0);
        // upstream gradient (0 for the padding rows and points), and the residual's gradient
        for (int e = tid; e < 64 * kTP; e += kThreads) {
            const int s = e / kTP, p = e % kTP;
            sm[l.G + e] = (s < a.S && p0 + p < a.n) ? __ldg(a.g + (size_t)(p0 + p) * a.S + s) : 0.f;
        }
        if (a.g_shs) {
            for (int e = tid; e < kTP * a.S; e += kThreads) {
                const int p = e / a.S, s = e % a.S;
                if (p0 + p >= a.n) break;
                const int id = __ldg(a.idx + p0 + p);
                if (id >= 0 && id < a.NK) a.g_shs[(size_t)id * a.S + s] = __ldg(a.g + (size_t)(p0 + p) * a.S + s);
            }
        }
        __syncthreads();
        // sh = W2 relu(z) + b2
        tile_outer_acc<true>(acc + l.dW2, sm + l.G, sm + l.Z, a.Sp, kHid);
        tile_row_acc(acc + l.db2, sm + l.G, nullptr, a.Sp);
        tile_gemm<false>(sm + l.E, sm + l.G, sm + l.W2, 1, kHid, kHid, a.Sp, nullptr, sm + l.Z);     // dz
        __syncthreads();
        // z = W1c c + b1
        tile_outer_acc<false>(acc + l.dW1c, sm + l.E, sm + l.C, kHid, kHK);
        tile_row_acc(acc + l.db1, sm + l.E, nullptr, kHid);
        tile_gemm<false>(sm + l.Z, sm + l.E, sm + l.W1c, 1, kHK, kHK, kHid, nullptr, nullptr);       // dc -> Z
        __syncthreads();
        {   // attention backward, one thread per (point, head): dr -> C, ds -> G
            const int p = tid % kTP, h = tid / kTP;
            float dc[kCond], dr[kCond] = {};
#pragma unroll
            for (int k = 0; k < kCond; ++k) dc[k] = sm[l.Z + (h * kCond + k) * kTP + p];
            float da[8], aj[8], dot = 0.f;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                if (j < V) {
                    float t = 0.f;
#pragma unroll
                    for (int k = 0; k < kCond; ++k) t = fmaf(dc[k], sm[l.F + (j * kCond + k) * kTP + p], t);
                    da[j] = t;
                    aj[j] = sm[l.PA + (h * V + j) * kTP + p];
                    dot = fmaf(aj[j], t, dot);
                }
            }
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                if (j < V) {
                    const float ds = aj[j] * (da[j] - dot);
                    sm[l.G + (h * V + j) * kTP + p] = ds;
#pragma unroll
                    for (int k = 0; k < kCond; ++k) dr[k] = fmaf(ds, sm[l.F + (j * kCond + k) * kTP + p], dr[k]);
                }
            }
#pragma unroll
            for (int k = 0; k < kCond; ++k) sm[l.C + (h * kCond + k) * kTP + p] = dr[k];
        }
        __syncthreads();
        // dL/df_j = sum_h a_hj dc_h + ds_hj r_h
        for (int e = tid; e < V * kCond * kTP; e += kThreads) {
            const int jk = e / kTP, p = e % kTP, j = jk / kCond, k = jk % kCond;
            float s = 0.f;
#pragma unroll
            for (int h = 0; h < kHeads; ++h) {
                s = fmaf(sm[l.PA + (h * V + j) * kTP + p], sm[l.Z + (h * kCond + k) * kTP + p], s);
                s = fmaf(sm[l.G + (h * V + j) * kTP + p], sm[l.R + (h * kCond + k) * kTP + p], s);
            }
            if (p0 + p < a.n) a.g_pf[(size_t)jk * a.n + p0 + p] = s;
        }
        // r = A x
        tile_outer_acc<false>(acc + l.dA, sm + l.C, sm + l.X, kHK, D);
        __syncthreads();
        tile_gemm<false>(sm + l.X, sm + l.C, sm + l.A, 1, D, D, kHK, nullptr, nullptr);              // dx -> X
        __syncthreads();
        tile_row_acc(acc + l.dlw, sm + l.X, sm + l.XH, D);
        tile_row_acc(acc + l.dlb, sm + l.X, nullptr, D);
        {   // LayerNorm backward: dvf = rstd (dxh - mean(dxh) - xh mean(dxh xh)), dxh = dx w
            const int p = tid % kTP, sub = tid / kTP;
            float* red = sm + l.red;
            float s1 = 0.f, s2 = 0.f;
            for (int d = sub; d < D; d += 8) {
                const float dxh = sm[l.X + d * kTP + p] * sm[l.lw + d];
                s1 += dxh;
                s2 = fmaf(dxh, sm[l.XH + d * kTP + p], s2);
            }
            red[sub * kTP + p] = s1;
            red[8 * kTP + sub * kTP + p] = s2;
            __syncthreads();
            s1 = 0.f; s2 = 0.f;
#pragma unroll
            for (int q = 0; q < 8; ++q) { s1 += red[q * kTP + p]; s2 += red[8 * kTP + q * kTP + p]; }
            const float m1 = s1 / (float)D, m2 = s2 / (float)D, rstd = sm[l.rstd + p];
            float* T = sm + l.F;
            for (int d = sub; d < D; d += 8) {
                const float dxh = sm[l.X + d * kTP + p] * sm[l.lw + d];
                T[d * kTS + p] = rstd * (dxh - m1 - sm[l.XH + d * kTP + p] * m2);
            }
        }
        __syncthreads();
        for (int e = tid; e < kTP * D; e += kThreads) {       // rows written along d (coalesced)
            const int p = e / D, d = e % D;
            if (p0 + p >= a.n) break;
            a.g_rows[(size_t)(p0 + p) * D + d] = sm[l.F + d * kTS + p];
        }
        __syncthreads();
    }
    float* part = a.partials + (size_t)blockIdx.x * l.nacc;
    for (int e = tid; e < l.nacc; e += kThreads) part[e] = acc[e];
}

struct GradArgs {
    int D, S, Sp;
    const double* tot;               // reduced accumulators (Layout offsets)
    double* B; double* dB;           // [D][64]
    const float *wq, *wk, *wv, *wo, *w1;
    float *d_lw, *d_lb, *d_wq, *d_wk, *d_wv, *d_wo, *d_w1, *d_b1, *d_w2, *d_b2;
};

// stage 0: the direct gradients, dWq, dWk, B and dB; stage 1: dW1, dWo, dWv (from B and dB).  fp64 throughout.
__global__ void fine_head_grads_kernel(GradArgs g, int stage) {
    const int D = g.D, hd = D / kHeads;
    const Layout l = layout(D, g.Sp);
    const double scale = 1.0 / sqrt((double)hd);
    const double* dA = g.tot + l.dA;
    const double* dW1c = g.tot + l.dW1c;
    int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (stage == 0) {
        if (e < D) { g.d_lw[e] = (float)g.tot[l.dlw + e]; g.d_lb[e] = (float)g.tot[l.dlb + e]; return; }
        e -= D;
        if (e < kHid) { g.d_b1[e] = (float)g.tot[l.db1 + e]; return; }
        e -= kHid;
        if (e < g.S) { g.d_b2[e] = (float)g.tot[l.db2 + e]; return; }
        e -= g.S;
        if (e < g.S * kHid) { g.d_w2[e] = (float)g.tot[l.dW2 + e]; return; }
        e -= g.S * kHid;
        if (e < D * D) {             // dWq[h hd+i][d] = s sum_k Wk[h hd+i][k] dA[h8+k][d]
            const int row = e / D, d = e % D, h = row / hd;
            double s = 0.0;
            for (int k = 0; k < kCond; ++k) s += (double)g.wk[row * kCond + k] * dA[(h * kCond + k) * D + d];
            g.d_wq[e] = (float)(s * scale);
            return;
        }
        e -= D * D;
        if (e < D * kCond) {         // dWk[h hd+i][k] = s sum_d Wq[h hd+i][d] dA[h8+k][d]
            const int row = e / kCond, k = e % kCond, h = row / hd;
            double s = 0.0;
            for (int d = 0; d < D; ++d) s += (double)g.wq[(size_t)row * D + d] * dA[(h * kCond + k) * D + d];
            g.d_wk[e] = (float)(s * scale);
            return;
        }
        e -= D * kCond;
        if (e < D * kHK) {           // B[d][hk] = sum_i Wo[d][h hd+i] Wv[h hd+i][k];  dB[d][hk] = sum_m W1[m][d] dW1c[m][hk]
            const int d = e / kHK, hk = e % kHK, h = hk / kCond, k = hk % kCond;
            double s = 0.0, t = 0.0;
            for (int i = 0; i < hd; ++i) s += (double)g.wo[(size_t)d * D + h * hd + i] * (double)g.wv[(h * hd + i) * kCond + k];
            for (int m = 0; m < kHid; ++m) t += (double)g.w1[(size_t)m * D + d] * dW1c[m * kHK + hk];
            g.B[e] = s;
            g.dB[e] = t;
        }
        return;
    }
    if (e < kHid * D) {              // dW1[m][d] = sum_hk dW1c[m][hk] B[d][hk]
        const int m = e / D, d = e % D;
        double s = 0.0;
        for (int hk = 0; hk < kHK; ++hk) s += dW1c[m * kHK + hk] * g.B[d * kHK + hk];
        g.d_w1[e] = (float)s;
        return;
    }
    e -= kHid * D;
    if (e < D * D) {                 // dWo[d][h hd+i] = sum_k dB[d][h8+k] Wv[h hd+i][k]
        const int d = e / D, col = e % D, h = col / hd;
        double s = 0.0;
        for (int k = 0; k < kCond; ++k) s += g.dB[d * kHK + h * kCond + k] * (double)g.wv[col * kCond + k];
        g.d_wo[e] = (float)s;
        return;
    }
    e -= D * D;
    if (e < D * kCond) {             // dWv[h hd+i][k] = sum_d Wo[d][h hd+i] dB[d][h8+k]
        const int row = e / kCond, k = e % kCond, h = row / hd;
        double s = 0.0;
        for (int d = 0; d < D; ++d) s += (double)g.wo[(size_t)d * D + row] * g.dB[d * kHK + h * kCond + k];
        g.d_wv[e] = (float)s;
    }
}

// dL/dvolume_feat[row] = sum of the rows of the points with idx / K == row (adjacent: idx is strictly increasing)
__global__ void fine_head_row_gather_kernel(const float* rows, const int* idx, int n, int N, int K, int D, float* out) {
    const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (size_t)N * D) return;
    const int row = (int)(e / D), d = (int)(e % D);
    const long long lo = (long long)row * K, hi = lo + K;
    int a = 0, b = n;                                          // first p with idx[p] >= lo
    while (a < b) {
        const int m = (a + b) >> 1;
        if (__ldg(idx + m) < lo) a = m + 1; else b = m;
    }
    float s = 0.f;
    for (int p = a; p < n && __ldg(idx + p) < hi; ++p) s += rows[(size_t)p * D + d];
    out[e] = s;
}

struct WsLayout { size_t parts, tot, B, dB, rows, total; };

int grid_for(int n) {
    const int tiles = (n + kTP - 1) / kTP;
    return tiles < sm_count() ? tiles : sm_count();
}

WsLayout ws_layout(int n, int D, int Sp, bool gather) {
    const Layout l = layout(D, Sp);
    WsLayout w;
    w.parts = 0;
    w.tot = align_up(w.parts + sizeof(float) * (size_t)grid_for(n) * l.nacc);
    w.B = align_up(w.tot + sizeof(double) * l.nacc);
    w.dB = align_up(w.B + sizeof(double) * D * kHK);
    w.rows = align_up(w.dB + sizeof(double) * D * kHK);
    w.total = align_up(w.rows + (gather ? sizeof(float) * (size_t)n * D : 0));
    return w;
}

int check_sizes(const char* fn, int n, int V, int D, int sh_dim, int K, int N, bool gather) {
    if (n < 0 || V < 1 || V > 8 || D < 8 || D > 128 || D % 8 != 0)
        return set_error("%s: bad sizes (n=%d, V=%d, D=%d): need n >= 0, 1 <= V <= 8 and D a multiple of 8 up to 128",
                         fn, n, V, D);
    if (sh_dim != 3 && sh_dim != 12 && sh_dim != 27 && sh_dim != 48)
        return set_error("%s: bad sizes (sh_dim=%d): need 3, 12, 27 or 48", fn, sh_dim);
    if (gather && (K < 1 || N < 0 || (long long)N * K > INT32_MAX || n > (long long)N * K))
        return set_error("%s: bad sizes (K=%d, N=%d, n=%d): need K >= 1, N >= 0, N*K < 2^31 and n <= N*K", fn, K, N, n);
    if ((long long)n * 64 > INT32_MAX) return set_error("%s: bad sizes (n=%d): too many points", fn, n);
    return 0;
}

void fill_common(Args& a, int n, int V, int D, int sh_dim, int K, int N, const float* vf, const int* idx,
                 const float* pf, const float* ln_w, const float* ln_b, const float* wq, const float* wk,
                 const float* wv, const float* wo, const float* w1, const float* b1, const float* w2, const float* b2) {
    a.n = n; a.V = V; a.D = D; a.S = sh_dim; a.Sp = (sh_dim + 3) / 4 * 4; a.K = idx ? K : 1;
    a.NK = idx ? (long long)N * K : 0;
    a.vf = vf; a.idx = idx; a.pf = pf;
    a.ln_w = ln_w; a.ln_b = ln_b; a.wq = wq; a.wk = wk; a.wv = wv; a.wo = wo; a.w1 = w1; a.b1 = b1; a.w2 = w2; a.b2 = b2;
}

}  // namespace
}  // namespace srf

using srf::cuda_error;
using srf::set_error;

extern "C" int srf_fine_head_workspace_bytes(int n, int V, int D, int sh_dim, int gather, size_t* bytes) {
    const char* fn = "srf_fine_head_workspace_bytes";
    if (srf::check_sizes(fn, n, V, D, sh_dim, 1, n, false)) return 1;
    if (!bytes) return set_error("%s: null output", fn);
    *bytes = srf::ws_layout(n, D, (sh_dim + 3) / 4 * 4, gather != 0).total;
    return 0;
}

extern "C" int srf_fine_head_forward(void* stream, int n, int V, int D, int sh_dim, int K, int N,
                                     const float* volume_feat, const int32_t* idx, const float* point_feats,
                                     const float* shs_coarse, const float* norm_w, const float* norm_b,
                                     const float* wq, const float* wk, const float* wv, const float* wo,
                                     const float* w1, const float* b1, const float* w2, const float* b2,
                                     float* sh_out) {
    const char* fn = "srf_fine_head_forward";
    if (srf::check_sizes(fn, n, V, D, sh_dim, K, N, idx != nullptr)) return 1;
    if (!norm_w || !norm_b || !wq || !wk || !wv || !wo || !w1 || !b1 || !w2 || !b2)
        return set_error("%s: null weight pointer", fn);
    if (shs_coarse && !idx) return set_error("%s: shs_coarse needs idx (the residual is added in gather mode only)", fn);
    if (n == 0) return 0;
    if (!volume_feat || !point_feats) return set_error("%s: null input pointer", fn);
    if (!sh_out) return set_error("%s: null output pointer", fn);
    srf::Args a = {};
    srf::fill_common(a, n, V, D, sh_dim, K, N, volume_feat, idx, point_feats, norm_w, norm_b, wq, wk, wv, wo, w1, b1,
                     w2, b2);
    a.shs = shs_coarse;
    a.out = sh_out;
    const size_t smem = sizeof(float) * srf::layout(D, a.Sp).fwd_floats;
    cudaError_t e = cudaFuncSetAttribute(srf::fine_head_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return cuda_error("fine_head_fwd shared memory", e);
    srf::fine_head_fwd_kernel<<<srf::grid_for(n), srf::kThreads, smem, (cudaStream_t)stream>>>(a);
    e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_error("fine_head_fwd launch", e);
}

extern "C" int srf_fine_head_backward(void* stream_, int n, int V, int D, int sh_dim, int K, int N,
                                      const float* volume_feat, const int32_t* idx, const float* point_feats,
                                      const float* norm_w, const float* norm_b,
                                      const float* wq, const float* wk, const float* wv, const float* wo,
                                      const float* w1, const float* b1, const float* w2, const float* b2,
                                      const float* dL_dsh, void* workspace,
                                      float* dL_dvolume_feat, float* dL_dpoint_feats, float* dL_dshs_coarse,
                                      float* d_norm_w, float* d_norm_b, float* d_wq, float* d_wk, float* d_wv,
                                      float* d_wo, float* d_w1, float* d_b1, float* d_w2, float* d_b2) {
    const char* fn = "srf_fine_head_backward";
    const bool gather = idx != nullptr;
    if (srf::check_sizes(fn, n, V, D, sh_dim, K, N, gather)) return 1;
    if (!norm_w || !norm_b || !wq || !wk || !wv || !wo || !w1 || !b1 || !w2 || !b2)
        return set_error("%s: null weight pointer", fn);
    if (!d_norm_w || !d_norm_b || !d_wq || !d_wk || !d_wv || !d_wo || !d_w1 || !d_b1 || !d_w2 || !d_b2)
        return set_error("%s: null weight-gradient pointer", fn);
    if (dL_dshs_coarse && !gather) return set_error("%s: dL_dshs_coarse needs idx (gather mode)", fn);
    if (!workspace || srf::misaligned(workspace)) return set_error("%s: workspace must be 256-byte aligned", fn);
    const int rows = gather ? N : n;
    if (rows > 0 && !dL_dvolume_feat) return set_error("%s: null dL_dvolume_feat", fn);
    if (n > 0 && (!volume_feat || !point_feats)) return set_error("%s: null input pointer", fn);
    if (n > 0 && (!dL_dsh || !dL_dpoint_feats)) return set_error("%s: null upstream gradient or dL_dpoint_feats", fn);
    const cudaStream_t stream = (cudaStream_t)stream_;
    srf::Args a = {};
    srf::fill_common(a, n, V, D, sh_dim, K, N, volume_feat, idx, point_feats, norm_w, norm_b, wq, wk, wv, wo, w1, b1,
                     w2, b2);
    const srf::Layout l = srf::layout(D, a.Sp);
    const srf::WsLayout w = srf::ws_layout(n, D, a.Sp, gather);
    char* ws = static_cast<char*>(workspace);
    a.g = dL_dsh;
    a.g_pf = dL_dpoint_feats;
    a.g_shs = dL_dshs_coarse;
    a.g_rows = gather ? reinterpret_cast<float*>(ws + w.rows) : dL_dvolume_feat;
    a.partials = reinterpret_cast<float*>(ws + w.parts);
    cudaError_t e;
    if (dL_dshs_coarse && N > 0) {
        e = cudaMemsetAsync(dL_dshs_coarse, 0, sizeof(float) * (size_t)N * K * sh_dim, stream);
        if (e != cudaSuccess) return cuda_error("memset dL_dshs_coarse", e);
    }
    const int grid = srf::grid_for(n);
    if (grid > 0) {
        const size_t smem = sizeof(float) * l.bwd_floats;
        e = cudaFuncSetAttribute(srf::fine_head_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return cuda_error("fine_head_bwd shared memory", e);
        srf::fine_head_bwd_kernel<<<grid, srf::kThreads, smem, stream>>>(a);
        if ((e = cudaGetLastError()) != cudaSuccess) return cuda_error("fine_head_bwd launch", e);
    }
    double* tot = reinterpret_cast<double*>(ws + w.tot);
    srf::part_sums(stream, a.partials, grid, (size_t)l.nacc, srf::seg(tot, l.nacc));   // in CTA order, in fp64
    srf::GradArgs g = {D, sh_dim, a.Sp, tot, reinterpret_cast<double*>(ws + w.B), reinterpret_cast<double*>(ws + w.dB),
                       wq, wk, wv, wo, w1, d_norm_w, d_norm_b, d_wq, d_wk, d_wv, d_wo, d_w1, d_b1, d_w2, d_b2};
    const int n0 = D + 64 + sh_dim + sh_dim * 64 + D * D + D * 8 + D * 64, n1 = 64 * D + D * D + D * 8;
    srf::fine_head_grads_kernel<<<(n0 + 127) / 128, 128, 0, stream>>>(g, 0);
    srf::fine_head_grads_kernel<<<(n1 + 127) / 128, 128, 0, stream>>>(g, 1);
    if (gather && N > 0) {
        const size_t total = (size_t)N * D;
        srf::fine_head_row_gather_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(a.g_rows, idx, n, N, K, D,
                                                                                             dL_dvolume_feat);
    }
    e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_error("fine_head backward launch", e);
}
