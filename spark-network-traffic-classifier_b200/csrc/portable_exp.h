// exp(x) that gives the same bits on the device and on the host (GBTClassifier's LogLoss residual and probability,
// DESIGN.md §5e).  CUDA's exp and libm's differ in the last bit on some inputs, and a residual that differs by one ulp puts a
// record into another histogram cell of the next tree; so both sides use this restatement, built only from IEEE-754
// round-to-nearest +, -, *, /, rint and exact scaling by powers of two assembled from their bits.
//
// Algorithm (Cody-Waite reduction + a Remez rational form, as in the classic fdlibm exp; error below 1 ulp):
//   k  = rint(x / ln2),  hi = x - k * LN2_HI (exact: LN2_HI has 21 trailing zero bits, |k| <= 1076),  lo = k * LN2_LO,
//   r  = hi - lo,  t = r * r,  c = r - t * (P1 + t * (P2 + t * (P3 + t * (P4 + t * P5)))),
//   y  = 1 - ((lo - (r * c) / (2 - c)) - hi)   ~ exp(r),   exp(x) = y * 2^k.
// Overflow (x > 709.78...) gives +inf, underflow below -745.13... gives +0, subnormal results are rounded once in the last
// scaling.  exp(+-0) = 1 exactly, exp(+inf) = +inf, exp(-inf) = +0, exp(NaN) = NaN.
// Every caller must be compiled without FMA contraction (nvcc -fmad=false, g++ -ffp-contract=off): a fused r - t*(...)
// rounds differently.  tests/test_gbt.py checks the host build against math.exp (within 1 ulp) and against the Python
// restatement in tests/gbt_oracle.py (bit for bit).
#pragma once
#include <stdint.h>
#include <string.h>
#include <math.h>

#if defined(__CUDACC__)
#define B2F_EXP_HD __host__ __device__ __forceinline__
#else
#define B2F_EXP_HD static inline
#endif

namespace b200flow {

B2F_EXP_HD double pexp_pow2(int k) {                   // 2^k for -1022 <= k <= 1023, from its bits
    const uint64_t b = (uint64_t)(k + 1023) << 52;
    double d;
    memcpy(&d, &b, 8);
    return d;
}

B2F_EXP_HD double portable_exp(double x) {
    const double O_THRESHOLD = 7.09782712893383973096e+02;   // largest x with a finite exp(x)
    const double U_THRESHOLD = -7.45133219101941108420e+02;  // below: exp(x) rounds to +0
    const double INV_LN2 = 1.44269504088896338700e+00;
    const double LN2_HI = 6.93147180369123816490e-01;        // 0x3fe62e42fee00000
    const double LN2_LO = 1.90821492927058770002e-10;        // 0x3dea39ef35793c76
    const double P1 = 1.66666666666666019037e-01, P2 = -2.77777777770155933842e-03, P3 = 6.61375632143793436117e-05,
                 P4 = -1.65339022054652515390e-06, P5 = 4.13813679705723846039e-08;
    if (x != x) return x + x;                                 // NaN
    if (x > O_THRESHOLD) return INFINITY;
    if (x < U_THRESHOLD) return 0.0;
    const double kd = rint(x * INV_LN2);
    const int k = (int)kd;
    const double hi = x - kd * LN2_HI;
    const double lo = kd * LN2_LO;
    const double r = hi - lo;
    const double t = r * r;
    const double c = r - t * (P1 + t * (P2 + t * (P3 + t * (P4 + t * P5))));
    const double y = 1.0 - ((lo - (r * c) / (2.0 - c)) - hi);
    if (k > 1023) return (y * pexp_pow2(1023)) * pexp_pow2(k - 1023);
    if (k < -1021) return (y * pexp_pow2(k + 1000)) * pexp_pow2(-1000);   // one rounding, into the subnormals
    return y * pexp_pow2(k);
}

}  // namespace b200flow
