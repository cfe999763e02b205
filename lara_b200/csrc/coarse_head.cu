// coarse_head.cu -- fused coarse-pass decoder head of LaRa (Decoder.forward_coarse, lightning/network.py:259-278: the
// three Linear layers of mlp_coarse and the decoder layout, optionally with get_offseted_pt), DESIGN §3.20.  The C
// entries of include/surfel_coarse_head.h are defined here.
//
// Per row: h1 = relu(W0 x + b0), h2 = relu(W1 h1 + b1), y = W2 h2 + b2, then decoder_layout.cuh on y's K Gaussians.
// Every product runs on the tensor cores as 3xTF32 mma.sync.m16n8k8: each fp32 operand is split into hi = tf32(v) and
// lo = tf32(v - hi), and a b is accumulated in fp32 as lo_a hi_b + hi_a lo_b + hi_a hi_b.  A warp owns 16 rows.  The
// activations stay in registers from layer to layer: the accumulator fragment of one layer is the A fragment of the
// next when the k index inside each 8-wide step is permuted (k = t <-> column 2t, k = t + 4 <-> column 2t + 1); the B
// fragments are read in the same permuted order.
//
// The backward recomputes the forward per tile of 128 rows (64 when the weights are read through L1), stages h1, h2 and dL/dy of the tile in shared memory (dz1
// and dz0 overwrite h2 and h1 once their weight gradients are formed, and x is read again for dW0), and writes dL/dx
// per row.  The weight and
// bias gradients of a tile (dW = dz^T h over the tile's rows, again 3xTF32) are added to per-CTA partials in global
// memory, each element by one fixed thread; the partials are summed over the CTAs in CTA order in fp64.  No atomics.
//
// The weights sit in shared memory, rows padded to D + 8 floats (fragment loads without bank conflicts), when they fit
// next to the staging buffers; otherwise (D >= 112 with a wide output) they are read through the L1 cache.
#include <stdint.h>

#include "../../include/surfel_coarse_head.h"
#include "decoder_layout.cuh"
#include "fixed_sums.cuh"
#include "surfel_kernels.h"

namespace srf {
namespace {

constexpr int kWarpRows = 16;                        // rows per warp (the MMA's m)
constexpr int kFwdWarps = 8;
// backward warps: 8 (tiles of 128 rows) with the weights in shared memory, 4 (64 rows) when they are read through L1,
// which keeps the staging of the widest outputs within the shared memory
__host__ __device__ constexpr int bwd_warps(bool wsmem) { return wsmem ? 8 : 4; }

struct Args {
    int rows, D, O, Op;          // O = K*C outputs per row, Op = O rounded up to 16
    bool centers;                // get_offseted_pt form
    const float* x;              // [rows, D]
    const float *w0, *b0, *w1, *b1, *w2, *b2;
    DecoderArgs lay;             // layout outputs (forward) / upstream gradients (backward)
    float* dx;                   // [rows, D]
    float* partials;             // [gridDim.x][nacc]: dW0 db0 dW1 db1 dW2 db2
};

// shared-memory layout in floats; every region starts on a 16-byte boundary
struct Layout {
    int w0, w1, w2, b0, b1, b2;  // weights (w* only when they are in shared memory), biases
    int stage;                   // forward: per warp [16][ldx] + [16][ldy]; backward: A, B [rows][ldx], Y [rows][ldy]
    int ldx, ldy, floats;
};

__host__ __device__ inline Layout layout(int D, int Op, bool wsmem, bool bwd) {
    Layout l;
    l.ldx = D + 8; l.ldy = Op + 8;                   // = 8 mod 16: conflict-free fragment loads
    int o = 0;
    l.w0 = o; o += wsmem ? D * l.ldx : 0;
    l.w1 = o; o += wsmem ? D * l.ldx : 0;
    l.w2 = o; o += wsmem ? Op * l.ldx : 0;
    l.b0 = o; o += D;
    l.b1 = o; o += D;
    l.b2 = o; o += Op;
    l.stage = o;
    o += bwd ? bwd_warps(wsmem) * kWarpRows * (2 * l.ldx + l.ldy) : kFwdWarps * kWarpRows * (l.ldx + l.ldy);
    l.floats = o;
    return l;
}

__host__ __device__ inline int nacc_of(int D, int O) { return 2 * D * D + 2 * D + O * D + O; }

__device__ __forceinline__ uint32_t tf32(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return r;
}

__device__ __forceinline__ void split(float x, uint32_t& hi, uint32_t& lo) {
    hi = tf32(x);
    lo = tf32(x - __uint_as_float(hi));
}

__device__ __forceinline__ void mma(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// c += a b in 3xTF32, the small cross terms first
__device__ __forceinline__ void mma3(float (&c)[4], const uint32_t (&ah)[4], const uint32_t (&al)[4], float b0, float b1) {
    uint32_t bh0, bl0, bh1, bl1;
    split(b0, bh0, bl0);
    split(b1, bh1, bl1);
    mma(c, al, bh0, bh1);
    mma(c, ah, bl0, bl1);
    mma(c, ah, bh0, bh1);
}

// A fragment (permuted k) of an accumulator tile c, split
__device__ __forceinline__ void a_frag(const float (&c)[4], uint32_t (&ah)[4], uint32_t (&al)[4]) {
    split(c[0], ah[0], al[0]);
    split(c[2], ah[1], al[1]);
    split(c[1], ah[2], al[2]);
    split(c[3], ah[3], al[3]);
}

// one weight element: shared memory (pad rows are zero there) or the L1 path (rows >= nrows read as 0)
template <bool WS>
__device__ __forceinline__ float wld(const float* p, bool ok) { return WS ? *p : (ok ? __ldg(p) : 0.f); }

// the split A fragment (permuted k) of columns k0 .. k0+8 of a [16][ld] block of shared memory
__device__ __forceinline__ void a_frag_smem(const float* s, int ld, int k0, uint32_t (&ah)[4], uint32_t (&al)[4]) {
    const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const float2 p = *reinterpret_cast<const float2*>(s + g * ld + k0 + 2 * t);
    const float2 q = *reinterpret_cast<const float2*>(s + (g + 8) * ld + k0 + 2 * t);
    const float c[4] = {p.x, p.y, q.x, q.y};
    a_frag(c, ah, al);
}

// acc[j] = bias + in W^T for the n-tiles j < nt of columns n0 + 8j: in is [16][8 KT] in shared memory (row stride
// ldi), W [out][in] with row stride ld and nrows valid rows.
template <bool WS, int NT>
__device__ __forceinline__ void layer_fwd(float (&acc)[NT][4], const float* in, int ldi, int KT, const float* W, int ld,
                                          int nrows, int n0, int nt, const float* bias) {
    const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
#pragma unroll
    for (int j = 0; j < NT; ++j) {
        const float b0 = j < nt ? bias[n0 + 8 * j + 2 * t] : 0.f, b1 = j < nt ? bias[n0 + 8 * j + 2 * t + 1] : 0.f;
        acc[j][0] = b0; acc[j][1] = b1; acc[j][2] = b0; acc[j][3] = b1;
    }
#pragma unroll 1
    for (int ks = 0; ks < KT; ++ks) {
        uint32_t ah[4], al[4];
        a_frag_smem(in, ldi, 8 * ks, ah, al);
#pragma unroll
        for (int j = 0; j < NT; ++j) {
            if (j < nt) {
                const int n = n0 + 8 * j + g;
                const float* wp = W + (size_t)n * ld + 8 * ks + 2 * t;
                float2 b;
                if (WS) b = *reinterpret_cast<const float2*>(wp);
                else b = n < nrows ? __ldg(reinterpret_cast<const float2*>(wp)) : make_float2(0.f, 0.f);
                mma3(acc[j], ah, al, b.x, b.y);
            }
        }
    }
}

// acc = in W: the vjp of a layer, in [16][8 KT] in shared memory (row stride ldi), W [out][in] with row stride ld and
// nrows valid rows (the k index)
template <bool WS, int NT>
__device__ __forceinline__ void layer_bwd(float (&acc)[NT][4], const float* in, int ldi, int KT, const float* W, int ld,
                                          int nrows) {
    const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
#pragma unroll
    for (int j = 0; j < NT; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
#pragma unroll 1
    for (int ks = 0; ks < KT; ++ks) {
        uint32_t ah[4], al[4];
        a_frag_smem(in, ldi, 8 * ks, ah, al);
        const int k = 8 * ks + 2 * t;
        const float* w = W + (size_t)k * ld + g;
#pragma unroll
        for (int j = 0; j < NT; ++j)
            mma3(acc[j], ah, al, wld<WS>(w + 8 * j, k < nrows), wld<WS>(w + ld + 8 * j, k + 1 < nrows));
    }
}

template <int NT>
__device__ __forceinline__ void relu(float (&v)[NT][4]) {
#pragma unroll
    for (int j = 0; j < NT; ++j)
#pragma unroll
        for (int c = 0; c < 4; ++c) v[j][c] = fmaxf(v[j][c], 0.f);
}

// accumulator tiles <-> a [16][ld] block of shared memory
template <int NT>
__device__ __forceinline__ void store_tiles(float* s, int ld, const float (&v)[NT][4], int n0 = 0, int nt = NT) {
    const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
#pragma unroll
    for (int j = 0; j < NT; ++j) {
        if (j < nt) {
            *reinterpret_cast<float2*>(s + g * ld + n0 + 8 * j + 2 * t) = make_float2(v[j][0], v[j][1]);
            *reinterpret_cast<float2*>(s + (g + 8) * ld + n0 + 8 * j + 2 * t) = make_float2(v[j][2], v[j][3]);
        }
    }
}

template <int NT>
__device__ __forceinline__ void load_tiles(float (&v)[NT][4], const float* s, int ld) {
    const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
#pragma unroll
    for (int j = 0; j < NT; ++j) {
        const float2 a = *reinterpret_cast<const float2*>(s + g * ld + 8 * j + 2 * t);
        const float2 b = *reinterpret_cast<const float2*>(s + (g + 8) * ld + 8 * j + 2 * t);
        v[j][0] = a.x; v[j][1] = a.y; v[j][2] = b.x; v[j][3] = b.y;
    }
}

// v *= (s > 0) elementwise, s a [16][ld] block: the ReLU's vjp from its output
template <int NT>
__device__ __forceinline__ void relu_mask(float (&v)[NT][4], const float* s, int ld) {
    float m[NT][4];
    load_tiles(m, s, ld);
#pragma unroll
    for (int j = 0; j < NT; ++j)
#pragma unroll
        for (int c = 0; c < 4; ++c) v[j][c] = m[j][c] > 0.f ? v[j][c] : 0.f;
}

// 16 rows of x from r0 into s [16][ld] (zero past rows), 128-bit loads
template <int D>
__device__ __forceinline__ void stage_x(float* s, int ld, const float* x, int r0, int rows) {
    const int lane = threadIdx.x & 31;
    for (int e = lane; e < kWarpRows * D / 4; e += 32) {
        const int r = e / (D / 4), c = 4 * (e % (D / 4));
        const float4 v = r0 + r < rows ? __ldg(reinterpret_cast<const float4*>(x + (size_t)(r0 + r) * D + c))
                                       : make_float4(0.f, 0.f, 0.f, 0.f);
        *reinterpret_cast<float4*>(s + r * ld + c) = v;
    }
}

template <bool WS>
__device__ void load_weights(const Args& a, const Layout& l, float* sm) {
    const int D = a.D;
    if (WS) {
        for (int e = threadIdx.x; e < D * D; e += blockDim.x) {
            sm[l.w0 + (e / D) * l.ldx + e % D] = __ldg(a.w0 + e);
            sm[l.w1 + (e / D) * l.ldx + e % D] = __ldg(a.w1 + e);
        }
        for (int e = threadIdx.x; e < a.Op * D; e += blockDim.x)
            sm[l.w2 + (e / D) * l.ldx + e % D] = e < a.O * D ? __ldg(a.w2 + e) : 0.f;
    }
    for (int e = threadIdx.x; e < D; e += blockDim.x) {
        sm[l.b0 + e] = __ldg(a.b0 + e);
        sm[l.b1 + e] = __ldg(a.b1 + e);
    }
    for (int e = threadIdx.x; e < a.Op; e += blockDim.x) sm[l.b2 + e] = e < a.O ? __ldg(a.b2 + e) : 0.f;
}

struct Weights { const float *w0, *w1, *w2; int ld; };

template <bool WS>
__device__ __forceinline__ Weights weights(const Args& a, const Layout& l, const float* sm) {
    if (WS) return {sm + l.w0, sm + l.w1, sm + l.w2, l.ldx};
    return {a.w0, a.w1, a.w2, a.D};
}

// The MLP of 16 rows: x in xs, h1 to h1s, h2 to h2s (each [16][ldx]; the forward passes one buffer for all three),
// y = W2 h2 + b2 to ys [16][ldy].
template <int D, bool WS>
__device__ __forceinline__ void mlp_rows(const Args& a, const Layout& l, const float* sm, const Weights& w,
                                         const float* xs, float* h1s, float* h2s, float* ys) {
    constexpr int KT = D / 8;
    float z[KT][4];
    layer_fwd<WS>(z, xs, l.ldx, KT, w.w0, w.ld, D, 0, KT, sm + l.b0);
    relu(z);
    __syncwarp();
    store_tiles(h1s, l.ldx, z);
    __syncwarp();
    layer_fwd<WS>(z, h1s, l.ldx, KT, w.w1, w.ld, D, 0, KT, sm + l.b1);
    relu(z);
    __syncwarp();
    store_tiles(h2s, l.ldx, z);
    __syncwarp();
    for (int n0 = 0; n0 < a.Op; n0 += 64) {
        const int nt = min(8, (a.Op - n0) / 8);
        float y[8][4];
        layer_fwd<WS>(y, h2s, l.ldx, KT, w.w2, w.ld, a.O, n0, nt, sm + l.b2);
        store_tiles(ys, l.ldy, y, n0, nt);
    }
}

template <int D, bool WS>
__global__ void __launch_bounds__(kFwdWarps * 32, 1) coarse_head_fwd_kernel(Args a) {
    extern __shared__ __align__(16) float sm[];
    const Layout l = layout(D, a.Op, WS, false);
    load_weights<WS>(a, l, sm);
    __syncthreads();
    const Weights w = weights<WS>(a, l, sm);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, K = a.lay.K, C = a.lay.C;
    float* st = sm + l.stage + warp * kWarpRows * (l.ldx + l.ldy);
    float* ys = st + kWarpRows * l.ldx;
    const int ntiles = (a.rows + kWarpRows - 1) / kWarpRows;
    for (int tile = blockIdx.x * kFwdWarps + warp; tile < ntiles; tile += gridDim.x * kFwdWarps) {
        const int r0 = tile * kWarpRows;
        stage_x<D>(st, l.ldx, a.x, r0, a.rows);
        __syncwarp();
        mlp_rows<D, WS>(a, l, sm, w, st, st, st, ys);
        __syncwarp();
        for (int e = lane; e < kWarpRows * K; e += 32) {
            const int r = e / K, k = e % K;
            if (r0 + r >= a.rows) break;
            const size_t g = (size_t)(r0 + r) * K + k;
            if (a.centers) layout_store<true>(a.lay, ys + r * l.ldy + k * C, g);
            else layout_store<false>(a.lay, ys + r * l.ldy + k * C, g);
        }
        __syncwarp();
    }
}

// dW[o][i] += sum over the tile's NW*16 rows of dz[r][o] h[r][i] (o < Mv), db[o] += sum dz[r][o]: dz [rows][lda] (Mp
// columns, a multiple of 16), h [rows][ldb].  The warps take units of 16 x 16 outputs in turn; each element is owned by one
// thread, its tile sum formed in row order.
template <int D, int NW>
__device__ __forceinline__ void weight_grads(const float* dz, int lda, int Mp, int Mv, const float* h, int ldb, float* pw,
                                             float* pb) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int nng = D / 16;
    for (int u = warp; u < (Mp / 16) * nng; u += NW) {
        const int o0 = (u / nng) * 16, i0 = (u % nng) * 16;
        float acc[2][4] = {};
#pragma unroll 4
        for (int ks = 0; ks < NW * 2; ++ks) {
            const float* ar = dz + (ks * 8 + t) * lda + o0 + g;
            const float* br = h + (ks * 8 + t) * ldb + i0 + g;
            uint32_t ah[4], al[4];
            split(ar[0], ah[0], al[0]);
            split(ar[8], ah[1], al[1]);
            split(ar[4 * lda], ah[2], al[2]);
            split(ar[4 * lda + 8], ah[3], al[3]);
#pragma unroll
            for (int j = 0; j < 2; ++j) mma3(acc[j], ah, al, br[8 * j], br[4 * ldb + 8 * j]);
        }
        const int o = o0 + g;
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int i = i0 + 8 * j + 2 * t;
            if (o < Mv) { pw[o * D + i] += acc[j][0]; pw[o * D + i + 1] += acc[j][1]; }
            if (o + 8 < Mv) { pw[(o + 8) * D + i] += acc[j][2]; pw[(o + 8) * D + i + 1] += acc[j][3]; }
        }
    }
    for (int o = threadIdx.x; o < Mv; o += blockDim.x) {
        float s = 0.f;
        for (int r = 0; r < NW * kWarpRows; ++r) s += dz[r * lda + o];
        pb[o] += s;
    }
}

template <int D, bool WS>
__global__ void __launch_bounds__(bwd_warps(WS) * 32, 1) coarse_head_bwd_kernel(Args a) {
    extern __shared__ __align__(16) float sm[];
    constexpr int KT = D / 8, NW = bwd_warps(WS), kBwdRows = NW * kWarpRows;
    const Layout l = layout(D, a.Op, WS, true);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
    const int K = a.lay.K, C = a.lay.C, O = a.O, Op = a.Op;
    float* part = a.partials + (size_t)blockIdx.x * nacc_of(D, O);
    float *pw0 = part, *pb0 = pw0 + D * D, *pw1 = pb0 + D, *pb1 = pw1 + D * D, *pw2 = pb1 + D, *pb2 = pw2 + O * D;
    for (int e = tid; e < nacc_of(D, O); e += blockDim.x) part[e] = 0.f;
    load_weights<WS>(a, l, sm);
    __syncthreads();
    const Weights w = weights<WS>(a, l, sm);
    // A holds x, then h2, then dz1, then x again; B holds h1, then dz0
    float* As = sm + l.stage;
    float* Bs = As + kBwdRows * l.ldx;
    float* Ys = Bs + kBwdRows * l.ldx;
    const int wr = warp * kWarpRows;             // this warp's rows in the tile
    float* aw = As + wr * l.ldx; float* bw = Bs + wr * l.ldx; float* yw = Ys + wr * l.ldy;
    const int ntiles = (a.rows + kBwdRows - 1) / kBwdRows;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int r0 = tile * kBwdRows + wr;
        stage_x<D>(aw, l.ldx, a.x, r0, a.rows);
        __syncwarp();
        mlp_rows<D, WS>(a, l, sm, w, aw, bw, aw, yw);
        __syncwarp();
        // dL/dy through the layout (0 for the rows past the end and the pad columns)
        for (int e = lane; e < kWarpRows * K; e += 32) {
            const int r = e / K, k = e % K;
            float* row = yw + r * l.ldy + k * C;
            if (r0 + r < a.rows) layout_grad_row(a.lay, [&](int c) { return row[c]; }, row, (size_t)(r0 + r) * K + k);
            else for (int c = 0; c < C; ++c) row[c] = 0.f;
        }
        for (int e = lane; e < kWarpRows * (Op - O); e += 32) yw[(e / (Op - O)) * l.ldy + O + e % (Op - O)] = 0.f;
        __syncthreads();
        weight_grads<D, NW>(Ys, l.ldy, Op, O, As, l.ldx, pw2, pb2);
        float d[KT][4];                          // dz1 = (dy W2) relu'(z1)
        layer_bwd<WS>(d, yw, l.ldy, Op / 8, w.w2, w.ld, O);
        relu_mask(d, aw, l.ldx);
        __syncthreads();
        store_tiles(aw, l.ldx, d);
        __syncthreads();
        weight_grads<D, NW>(As, l.ldx, D, D, Bs, l.ldx, pw1, pb1);
        layer_bwd<WS>(d, aw, l.ldx, KT, w.w1, w.ld, D);       // dz0 = (dz1 W1) relu'(z0)
        relu_mask(d, bw, l.ldx);
        __syncthreads();
        store_tiles(bw, l.ldx, d);
        stage_x<D>(aw, l.ldx, a.x, r0, a.rows);  // x again (an L2 hit), for dW0
        __syncthreads();
        weight_grads<D, NW>(Bs, l.ldx, D, D, As, l.ldx, pw0, pb0);
        layer_bwd<WS>(d, bw, l.ldx, KT, w.w0, w.ld, D);       // dL/dx = dz0 W0
#pragma unroll
        for (int j = 0; j < KT; ++j) {
            const int i = 8 * j + 2 * t;
            if (r0 + g < a.rows) *reinterpret_cast<float2*>(a.dx + (size_t)(r0 + g) * D + i) = make_float2(d[j][0], d[j][1]);
            if (r0 + g + 8 < a.rows)
                *reinterpret_cast<float2*>(a.dx + (size_t)(r0 + g + 8) * D + i) = make_float2(d[j][2], d[j][3]);
        }
        __syncthreads();
    }
}

using Kernel = void (*)(Args);

template <int D>
Kernel pick(bool bwd, bool ws) {
    if (bwd) return ws ? coarse_head_bwd_kernel<D, true> : coarse_head_bwd_kernel<D, false>;
    return ws ? coarse_head_fwd_kernel<D, true> : coarse_head_fwd_kernel<D, false>;
}

Kernel kernel_for(int D, bool bwd, bool ws) {
    switch (D) {
        case 16: return pick<16>(bwd, ws);
        case 32: return pick<32>(bwd, ws);
        case 48: return pick<48>(bwd, ws);
        case 64: return pick<64>(bwd, ws);
        case 80: return pick<80>(bwd, ws);
        case 96: return pick<96>(bwd, ws);
        case 112: return pick<112>(bwd, ws);
        default: return pick<128>(bwd, ws);
    }
}

int max_smem() {
    int dev = 0, v = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess)
        return 48 * 1024;
    return v;
}

int op_of(int K, int sh_dim) { return (K * (10 + sh_dim) + 15) / 16 * 16; }

// the weights in shared memory when they fit
bool wsmem(int D, int Op, bool bwd) { return sizeof(float) * layout(D, Op, true, bwd).floats <= (size_t)max_smem(); }

// CTAs of the backward: one per tile, at most one per SM
int bwd_grid(int rows, bool ws) {
    const int tile = bwd_warps(ws) * kWarpRows, tiles = (rows + tile - 1) / tile;
    return tiles < sm_count() ? tiles : sm_count();
}

int check_sizes(const char* fn, int rows, int N, int D, int K, int sh_dim) {
    if (rows < 0 || N < 1 || rows % N != 0)
        return set_error("%s: bad sizes (rows=%d, N=%d): need N >= 1 and rows a non-negative multiple of N", fn, rows, N);
    if (D < 16 || D > 128 || D % 16 != 0 || K < 1 || K > 4)
        return set_error("%s: bad sizes (D=%d, K=%d): need D a multiple of 16 in [16, 128] and 1 <= K <= 4", fn, D, K);
    if (sh_dim != 3 && sh_dim != 12 && sh_dim != 27 && sh_dim != 48)
        return set_error("%s: bad sizes (sh_dim=%d): need 3, 12, 27 or 48", fn, sh_dim);
    if ((long long)rows * K > INT32_MAX) return set_error("%s: bad sizes (rows=%d, K=%d): rows*K over 2^31", fn, rows, K);
    return 0;
}

void fill(Args& a, int rows, int N, int D, int K, int sh_dim, float half_cell, bool centers, const float* feats,
          const float* group_centers, const float* w0, const float* b0, const float* w1, const float* b1,
          const float* w2, const float* b2) {
    a.rows = rows; a.D = D; a.O = K * (10 + sh_dim); a.Op = op_of(K, sh_dim); a.centers = centers;
    a.x = feats; a.w0 = w0; a.b0 = b0; a.w1 = w1; a.b1 = b1; a.w2 = w2; a.b2 = b2;
    a.lay.total = (size_t)rows * K; a.lay.N = N; a.lay.K = K; a.lay.C = 10 + sh_dim; a.lay.sh_dim = sh_dim;
    a.lay.half_cell = centers ? half_cell : 1.0f;          // the offset form's vjp has no cell scale
    a.lay.group_centers = group_centers;
}

bool unaligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) != 0; }

}  // namespace
}  // namespace srf

using srf::cuda_error;
using srf::set_error;

extern "C" int srf_coarse_head_workspace_bytes(int rows, int D, int K, int sh_dim, size_t* bytes) {
    const char* fn = "srf_coarse_head_workspace_bytes";
    if (srf::check_sizes(fn, rows, 1, D, K, sh_dim)) return 1;
    if (!bytes) return set_error("%s: null output", fn);
    const bool ws = srf::wsmem(D, srf::op_of(K, sh_dim), true);
    *bytes = srf::align_up(sizeof(float) * (size_t)srf::bwd_grid(rows, ws) * srf::nacc_of(D, K * (10 + sh_dim)));
    return 0;
}

extern "C" int srf_coarse_head_forward(void* stream, int rows, int N, int D, int K, int sh_dim,
                                       float opacity_shift, float scaling_shift, float half_cell,
                                       const float* feats, const float* group_centers,
                                       const float* w0, const float* b0, const float* w1, const float* b1,
                                       const float* w2, const float* b2,
                                       float* centers_or_offset, float* shs, float* opacity, float* scaling,
                                       float* rotation) {
    const char* fn = "srf_coarse_head_forward";
    if (srf::check_sizes(fn, rows, N, D, K, sh_dim)) return 1;
    if (!w0 || !b0 || !w1 || !b1 || !w2 || !b2) return set_error("%s: null weight pointer", fn);
    if (rows == 0) return 0;
    if (!feats) return set_error("%s: null input pointer", fn);
    if (!centers_or_offset || !shs || !opacity || !scaling || !rotation) return set_error("%s: null output pointer", fn);
    if (srf::unaligned16(feats) || srf::unaligned16(rotation) || (reinterpret_cast<uintptr_t>(scaling) & 7) ||
        ((sh_dim & 3) == 0 && srf::unaligned16(shs)))
        return set_error("%s: feats, shs and rotation must be 16-byte aligned, scaling 8-byte aligned", fn);
    srf::Args a = {};
    srf::fill(a, rows, N, D, K, sh_dim, half_cell, group_centers != nullptr, feats, group_centers, w0, b0, w1, b1, w2, b2);
    a.lay.opacity_shift = opacity_shift; a.lay.scaling_shift = scaling_shift;
    a.lay.centers = centers_or_offset; a.lay.shs = shs; a.lay.opacity = opacity; a.lay.scaling = scaling;
    a.lay.rotation = rotation;
    const bool ws = srf::wsmem(D, a.Op, false);
    const srf::Kernel kern = srf::kernel_for(D, false, ws);
    const size_t smem = sizeof(float) * srf::layout(D, a.Op, ws, false).floats;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return cuda_error("coarse_head_fwd shared memory", e);
    const int units = (rows + srf::kWarpRows * srf::kFwdWarps - 1) / (srf::kWarpRows * srf::kFwdWarps);
    const int grid = units < srf::sm_count() ? units : srf::sm_count();
    kern<<<grid, srf::kFwdWarps * 32, smem, (cudaStream_t)stream>>>(a);
    e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_error("coarse_head_fwd launch", e);
}

extern "C" int srf_coarse_head_backward(void* stream_, int rows, int N, int D, int K, int sh_dim, float half_cell,
                                        const float* feats, const float* group_centers,
                                        const float* w0, const float* b0, const float* w1, const float* b1,
                                        const float* w2, const float* b2,
                                        const float* dL_dcenters_or_offset, const float* dL_dshs,
                                        const float* dL_dopacity, const float* dL_dscaling, const float* dL_drotation,
                                        void* workspace, float* dL_dfeats, float* d_w0, float* d_b0, float* d_w1,
                                        float* d_b1, float* d_w2, float* d_b2) {
    const char* fn = "srf_coarse_head_backward";
    if (srf::check_sizes(fn, rows, N, D, K, sh_dim)) return 1;
    if (!w0 || !b0 || !w1 || !b1 || !w2 || !b2) return set_error("%s: null weight pointer", fn);
    if (!d_w0 || !d_b0 || !d_w1 || !d_b1 || !d_w2 || !d_b2) return set_error("%s: null weight-gradient pointer", fn);
    if (rows > 0 && (!workspace || srf::misaligned(workspace)))
        return set_error("%s: workspace must be 256-byte aligned", fn);
    if (rows > 0 && (!feats || !dL_dfeats)) return set_error("%s: null feats or dL_dfeats", fn);
    if (rows > 0 && srf::unaligned16(feats)) return set_error("%s: feats must be 16-byte aligned", fn);
    const cudaStream_t stream = (cudaStream_t)stream_;
    srf::Args a = {};
    srf::fill(a, rows, N, D, K, sh_dim, half_cell, group_centers != nullptr, feats, group_centers, w0, b0, w1, b1, w2, b2);
    a.lay.g_centers = dL_dcenters_or_offset; a.lay.g_shs = dL_dshs; a.lay.g_opacity = dL_dopacity;
    a.lay.g_scaling = dL_dscaling; a.lay.g_rotation = dL_drotation;
    a.dx = dL_dfeats;
    a.partials = static_cast<float*>(workspace);
    const bool ws = srf::wsmem(D, a.Op, true);
    const int grid = srf::bwd_grid(rows, ws);
    cudaError_t e;
    if (grid > 0) {
        const srf::Kernel kern = srf::kernel_for(D, true, ws);
        const size_t smem = sizeof(float) * srf::layout(D, a.Op, ws, true).floats;
        e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return cuda_error("coarse_head_bwd shared memory", e);
        kern<<<grid, srf::bwd_warps(ws) * 32, smem, stream>>>(a);
        if ((e = cudaGetLastError()) != cudaSuccess) return cuda_error("coarse_head_bwd launch", e);
    }
    // the six parameter gradients: the per-CTA partials summed over the CTAs, in CTA order, in fp64
    const int O = a.O;
    srf::part_sums(stream, a.partials, grid, (size_t)srf::nacc_of(D, O), srf::seg(d_w0, D * D), srf::seg(d_b0, D),
                   srf::seg(d_w1, D * D), srf::seg(d_b1, D), srf::seg(d_w2, O * D), srf::seg(d_b2, O));
    e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_error("coarse_head backward launch", e);
}
