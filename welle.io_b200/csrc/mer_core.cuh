// mer_core.cuh — modulation error ratio of the FIC softbits (dabb_set_mer, tap 14): the per-carrier sums, the carrier-group map and the
// record's derived value.  Compiles for the device (mer.cu) and as host C++ (api.cu builds the group table with it,
// tests/host_emul/emul_mer.cpp checks it), so host and device compute the same bits.
//
// The reference demap makes a carrier's softbits a = trunc(-Re r1 127 / l1), b = trunc(-Im r1 127 / l1), l1 = |Re r1| + |Im r1|: their
// magnitudes carry the angle of r1 and nothing of its level.  With u = |a| + |b| and v = |a| - |b|, v / u = tan(pi/4 - theta) for theta
// the angle of r1 folded into its quadrant, so v^2 is the squared distance of the unit-normalised product from its nearest DQPSK point
// and u^2 that point's power (both scaled by the same u^2 / 2).
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define MER_HD __host__ __device__ __forceinline__
#else
#define MER_HD inline
#endif

namespace dabb_mer {

constexpr int GROUPS = 64;                       // DABB_MER_GROUPS
constexpr int GROUP_CARRIERS = 24;               // carriers per group: 1536 / 64
constexpr int SYMBOLS = 3;                       // the FIC's data symbols l = 1, 2, 3
constexpr int CARRIERS = 1536;

// the group of physical carrier k (-768 .. 768 without 0): 24 carriers each, lowest frequency first
MER_HD int group_of(int k) { return (k + 768 - (k > 0 ? 1 : 0)) / GROUP_CARRIERS; }

// one point: softbits a (Re) and b (Im) of one carrier; u^2 and v^2
MER_HD void point(int8_t a, int8_t b, int32_t& u2, int32_t& v2)
{
    const int32_t x = a < 0 ? -(int32_t)a : (int32_t)a, y = b < 0 ? -(int32_t)b : (int32_t)b;
    const int32_t u = x + y, v = x - y;
    u2 = u * u; v2 = v * v;
}

// double arithmetic rounded after every operation (no contraction into fused multiply-adds on either side)
MER_HD double dmul(double a, double b)
{
#if defined(__CUDA_ARCH__)
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}
MER_HD double dadd(double a, double b)
{
#if defined(__CUDA_ARCH__)
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}
MER_HD double ddiv(double a, double b)
{
#if defined(__CUDA_ARCH__)
    return __ddiv_rn(a, b);
#else
    return a / b;
#endif
}

// ln x for a finite x > 0, the same bits on host and device: x = m 2^e with m in [sqrt(1/2), sqrt(2)), ln m = 2 atanh(z) with
// z = (m - 1) / (m + 1), |z| <= 0.172, summed to z^25 (the next term is below 2^-60 relative); within a few ulp of the exact value
MER_HD double ln_pos(double x)
{
    int e;
    double m = frexp(x, &e);
    if (m < 0.70710678118654752440) { m = m * 2.0; e -= 1; }
    const double z = ddiv(dadd(m, -1.0), dadd(m, 1.0)), w = dmul(z, z);
    double s = 2.0 / 25.0;
    for (int k = 11; k >= 0; k--) s = dadd(dmul(s, w), 2.0 / (2 * k + 1));
    return dadd(dmul((double)e, 0.69314718055994530942), dmul(s, z));
}

// the record's mer_db: 10 log10(sig / err) rounded to float; +inf when err == 0 < sig, 0 when sig == 0
MER_HD float mer_db(int64_t sig, int64_t err)
{
    if (sig <= 0) return 0.f;
    if (err <= 0) return INFINITY;
    return (float)dmul(ln_pos(ddiv((double)sig, (double)err)), 4.3429448190325182765);     // 10 / ln 10
}

} // namespace dabb_mer
