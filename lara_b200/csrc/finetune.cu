// finetune.cu -- per-scene refinement of LaRa's predicted Gaussians (configs/infer.yaml `finetuning`): the C entry of
// include/surfel_finetune.h, one Adam step over the five tensors of the Gaussian record.
//
// gaussian_adam_kernel: the five tensors are five segments of one 1D grid; CTA b belongs to the segment whose
// [block_start[s], block_start[s + 1]) holds b, and each thread takes kIlp elements kThreads apart, loads all of them
// first, then updates them.  Every access is a coalesced 4-byte one: the segments' lengths (3n, 3Mn, n, 2n, 4n) and
// therefore the moment buffer's segment offsets have no alignment a wider access could rely on.
//
// Rounding follows torch.optim.Adam's single-tensor path on CUDA op by op (include/surfel_finetune.h): each torch op
// writes its result to memory, so each is rounded on its own here, and where torch's kernel source reads a + b c it is
// compiled to one fma, which the intrinsics below pin whatever nvcc's -fmad setting is.
#include <math.h>
#include <string.h>

#include "../../include/surfel_finetune.h"
#include "surfel_common.cuh"
#include "surfel_kernels.h"

namespace srf {
namespace {

constexpr int kThreads = 256;
constexpr int kIlp = 4;
constexpr int kSegs = 5;
constexpr long long kPerCta = (long long)kThreads * kIlp;

struct AdamArgs {
    float* p[kSegs]; float* g[kSegs]; float* m[kSegs]; float* v[kSegs];
    long long len[kSegs];
    long long block_start[kSegs + 1];
    float step[SRF_ADAM_GROUPS];          // fp32(-(lr / bias_correction1)) per group
    float w, omw;                         // fp32(1 - beta1) and fp32(1 - w), the lerp weight and its complement
    float b2, a2;                         // fp32(beta2), fp32(1 - beta2)
    float inv_bc2;                        // fp32(1 / bias_correction2_sqrt), the reciprocal taken in fp64
    float eps;
    int M, small_w, zero;
};

__device__ __forceinline__ float adam_one(const AdamArgs& a, float& p, float g, float& m, float v, float step) {
    const float d = __fsub_rn(g, m);
    m = a.small_w ? __fmaf_rn(a.w, d, m) : __fmaf_rn(-d, a.omw, g);                 // exp_avg.lerp_(grad, 1 - beta1)
    v = __fmaf_rn(a.a2, __fmul_rn(g, g), __fmul_rn(v, a.b2));                       // .mul_(beta2).addcmul_(g, g, 1 - b2)
    const float den = __fadd_rn(__fmul_rn(__fsqrt_rn(v), a.inv_bc2), a.eps);        // (sqrt(v) / bc2_sqrt).add_(eps)
    p = __fmaf_rn(step, __fdiv_rn(m, den), p);                                      // param.addcdiv_(m, den, -step_size)
    return v;
}

__global__ void __launch_bounds__(kThreads) gaussian_adam_kernel(const AdamArgs a) {
    const long long b = blockIdx.x;
    int s = 0;
#pragma unroll
    for (int k = 1; k < kSegs; ++k) s += b >= a.block_start[k];
    const long long len = a.len[s];
    const long long i0 = (b - a.block_start[s]) * kPerCta + threadIdx.x;
    float* P = a.p[s]; float* G = a.g[s]; float* Mm = a.m[s]; float* Vv = a.v[s];
    float p[kIlp], g[kIlp], m[kIlp], v[kIlp];
#pragma unroll
    for (int k = 0; k < kIlp; ++k) {
        const long long i = i0 + k * kThreads;
        if (i < len) { p[k] = P[i]; g[k] = G[i]; m[k] = Mm[i]; v[k] = Vv[i]; }
    }
    const int stride = 3 * a.M;           // shs row: M coefficients of 3 channels; f_dc is the first 3 floats
#pragma unroll
    for (int k = 0; k < kIlp; ++k) {
        const long long i = i0 + k * kThreads;
        if (i >= len) continue;
        const int grp = s == 0 ? SRF_ADAM_XYZ
                      : s == 1 ? ((int)(i % stride) < 3 ? SRF_ADAM_F_DC : SRF_ADAM_F_REST)
                               : s + 1;  // opacity, scaling, rotation
        v[k] = adam_one(a, p[k], g[k], m[k], v[k], a.step[grp]);
        P[i] = p[k]; Mm[i] = m[k]; Vv[i] = v[k];
        if (a.zero) G[i] = 0.f;
    }
}

}  // namespace
}  // namespace srf

using srf::set_error;

extern "C" int srf_gaussian_adam_step(srf_stream_t stream_, int n, int M, float* const params[5],
                                      float* const grads[5], float* moments, const double lr[6], double beta1,
                                      double beta2, double eps, double bias_correction1,
                                      double bias_correction2_sqrt, int zero_grads) {
    using namespace srf;
    const char* fn = "srf_gaussian_adam_step";
    if (n < 0) return set_error("%s: bad size n = %d", fn, n);
    if (M != 1 && M != 4 && M != 9 && M != 16) return set_error("%s: M = %d is not 1, 4, 9 or 16", fn, M);
    if (n == 0) return 0;                 // nothing to update: empty tensors may carry null pointers
    if (!params || !grads || !lr) return set_error("%s: null params, grads or lr array", fn);
    if (!(beta1 >= 0.0 && beta1 < 1.0) || !(beta2 >= 0.0 && beta2 < 1.0) || !(eps >= 0.0))
        return set_error("%s: bad hyper-parameters (beta1 = %g, beta2 = %g, eps = %g)", fn, beta1, beta2, eps);
    if (!(bias_correction1 > 0.0) || !(bias_correction2_sqrt > 0.0))
        return set_error("%s: bias corrections must be positive (%g, %g)", fn, bias_correction1, bias_correction2_sqrt);
    static const char* names[kSegs] = {"centers", "shs", "opacity", "scaling", "rotation"};
    for (int k = 0; k < kSegs; ++k) {
        if (!params[k]) return set_error("%s: null %s pointer", fn, names[k]);
        if (!grads[k]) return set_error("%s: null %s gradient pointer", fn, names[k]);
    }
    if (!moments) return set_error("%s: null moments pointer", fn);
    AdamArgs a;
    memset(&a, 0, sizeof(a));
    const long long N = n;
    const long long len[kSegs] = {3 * N, 3LL * M * N, N, 2 * N, 4 * N};
    const long long row = (10LL + 3LL * M) * N;             // one moment
    long long off = 0;
    a.block_start[0] = 0;
    for (int k = 0; k < kSegs; ++k) {
        a.p[k] = params[k]; a.g[k] = grads[k];
        a.m[k] = moments + off; a.v[k] = moments + row + off;
        a.len[k] = len[k];
        off += len[k];
        a.block_start[k + 1] = a.block_start[k] + (len[k] + kPerCta - 1) / kPerCta;
    }
    if (a.block_start[kSegs] > 0x7fffffffLL) return set_error("%s: n = %d is too large", fn, n);
    for (int k = 0; k < SRF_ADAM_GROUPS; ++k) a.step[k] = (float)(-(lr[k] / bias_correction1));
    a.w = (float)(1.0 - beta1);
    a.omw = 1.0f - a.w;
    a.small_w = fabsf(a.w) < 0.5f;
    a.b2 = (float)beta2;
    a.a2 = (float)(1.0 - beta2);
    a.inv_bc2 = (float)(1.0 / bias_correction2_sqrt);
    a.eps = (float)eps;
    a.M = M;
    a.zero = zero_grads ? 1 : 0;
    const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    gaussian_adam_kernel<<<(unsigned)a.block_start[kSegs], kThreads, 0, stream>>>(a);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_error("gaussian_adam launch", e);
}
