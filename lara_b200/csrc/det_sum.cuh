// det_sum.cuh -- order-independent sums of fp32 terms in 64-bit fixed point (the deterministic backward, DESIGN §3.13).
// Compiles for the device and, as plain C++, for the host (tests/test_deterministic.py checks it there).
//
// A sum of n fp32 terms x_i with |x_i| <= m (m known before the sum starts) is taken as
//     k  = scale_exp(bits(m), L),  L = ceil(log2 n)       so that m 2^k < 2^(kSumBits - 1 - L)
//     q_i = round_nearest_even(x_i 2^k)                   (exact scaling in double, then one rounding)
//     S  = sum of q_i in wrapping 64-bit integer arithmetic, in any order
//     result = fp32(S) 2^-k                               (one rounding; a second one only if the result is subnormal)
// Integer addition is associative, so S, and with it the result, does not depend on the order of the terms.  Each
// |q_i| is held to the budget 2^(kSumBits - L) -- twice what m implies, so a term computed by a separately compiled
// instantiation may differ from the one the bound was taken from by an ulp -- and then the true sum
// |S| <= n 2^(kSumBits - L) <= 2^62 < 2^63 is exact even if partial sums wrap.  A term over its budget (or not finite)
// is reported, never summed.
// Error: |result - sum x_i| <= n 2^-(k+1) (the q_i roundings) + 2^-24 |result| (the final rounding); with
// 2^-k <= 2 n m 2^-61 the first part is at most n^2 m 2^-61.
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#define SRF_DET_HD __host__ __device__ __forceinline__
#else
#define SRF_DET_HD static inline
#endif

namespace srf {
namespace det {

constexpr int kSumBits = 62;

// ceil(log2(n)); 0 for n <= 1
SRF_DET_HD int ceil_log2(uint64_t n) {
    if (n <= 1) return 0;
#if defined(__CUDA_ARCH__)
    return 64 - __clzll((long long)(n - 1));
#else
    return 64 - __builtin_clzll(n - 1);
#endif
}

// 2^k as a double, -1022 <= k <= 1023
SRF_DET_HD double pow2(int k) {
    const uint64_t b = (uint64_t)(1023 + k) << 52;
#if defined(__CUDA_ARCH__)
    return __longlong_as_double((long long)b);
#else
    double d;
    memcpy(&d, &b, sizeof(d));
    return d;
#endif
}

// Scale exponent for terms bounded by the float with bit pattern `bound_bits` (sign bit clear), of which there are at
// most 2^L: m < 2^E with E the bound's binary exponent + 1, and k = kSumBits - 1 - L - E.  An infinite or NaN bound
// gives a k at which no term is scaled up; the non-finite term itself fails quantize().  Range: -132 <= k <= 186.
SRF_DET_HD int scale_exp(uint32_t bound_bits, int L) {
    const int e = (int)(bound_bits >> 23);
    const int E = (e == 0 ? 1 : e) - 126;
    return (kSumBits - 1) - L - E;
}

// q = round_nearest_even(x 2^k); false (q = 0) if |x 2^k| > 2^(kSumBits - L) or x is not finite
SRF_DET_HD bool quantize(float x, int k, int L, long long& q) {
    const double s = (double)x * pow2(k);          // exact: a float times a power of two, far from over/underflow
    if (!(fabs(s) <= pow2(kSumBits - L))) {
        q = 0;
        return false;
    }
#if defined(__CUDA_ARCH__)
    q = __double2ll_rn(s);
#else
    q = llrint(s);
#endif
    return true;
}

// the sum S of the quantised terms back to fp32: one rounding of S, then an exact scaling by 2^-k unless the result is
// subnormal or beyond the fp32 range
SRF_DET_HD float to_float(long long S, int k) {
#if defined(__CUDA_ARCH__)
    const float f = __ll2float_rn(S);
#else
    const float f = (float)S;
#endif
    return (float)((double)f * pow2(-k));
}

// magnitude bits of x: ordered like |x| for every non-NaN x, above +inf for NaN
SRF_DET_HD uint32_t abs_bits(float x) {
    uint32_t u;
#if defined(__CUDA_ARCH__)
    u = __float_as_uint(x);
#else
    memcpy(&u, &x, sizeof(u));
#endif
    return u & 0x7fffffffu;
}

}  // namespace det
}  // namespace srf
