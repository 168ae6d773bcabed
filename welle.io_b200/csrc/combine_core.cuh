// combine_core.cuh — diversity reception (dabb_set_combining): the arithmetic that adds the differential products of the streams of one
// group (the antennas of one capture) before the demap.  Plain C++ plus the DABB_HD building blocks of ofdm_core.cuh, so that the host
// test (tests/host_emul/emul_combine.cpp) compiles exactly what combine_kernel and null_power_kernel run.
//
// Post-detection combining: DQPSK is differential, so a timing offset inside the guard interval and a carrier phase both cancel in
// r1 = X_l conj(X_{l-1}); each antenna keeps its own synchronisation and the products are added per carrier, each weighted by the inverse
// of its antenna's noise power N_b (the mean |y|^2 of the null symbol that ends its frame window):
//     R[k] = sum over the contributing members b, in ascending stream order, of r1_b[k] / N_b       (fp32, each operation rounded)
// and the leader's softbits are the context's demap of R.  Every order of summation is fixed, so the result does not depend on the
// batch size or the launch configuration.
#pragma once
#include "ofdm_core.cuh"

namespace dabb_comb {

using dabb::LevelSum;

constexpr int MAX_BRANCHES = 8;          // DABB_MAX_BRANCHES: members of a group, leader included
constexpr int MAX_OFFSET = 504;          // |A_b - A_L| a contributing member's phase reference symbol may be off the leader's (T_g)
constexpr int NULL_THREADS = 256;        // null_power_kernel: thread t sums the null samples t, t + 256, ...
constexpr int COMB_THREADS = 128;        // combine_kernel: thread t combines the logical carriers t + 128 j, j = 0 .. 11
constexpr int COMB_PER_THREAD = dabb::KC / COMB_THREADS;

DABB_HD float fdiv(float a, float b)
{
#if defined(__CUDA_ARCH__)
    return __fdiv_rn(a, b);
#else
    return a / b;
#endif
}

// ---- noise power of one member: the TNULL samples y of its null symbol (NCO applied, tap 3)
// thread t's partial sum: |y_i|^2 = Re^2 + Im^2 (each product and sum rounded) over i = t, t + NULL_THREADS, ... in ascending order
DABB_HD float null_partial(const float2* y, int t)
{
    float s = 0.f;
    for (int i = t; i < dabb::TNULL; i += NULL_THREADS)
        s = dabb::fadd_<true>(s, dabb::fadd_<true>(dabb::fmul_<true>(y[i].x, y[i].x), dabb::fmul_<true>(y[i].y, y[i].y)));
    return s;
}
// N from the NULL_THREADS partial sums, added in thread order, divided by TNULL
DABB_HD float null_noise(const float* part)
{
    float s = 0.f;
    for (int t = 0; t < NULL_THREADS; t++) s = dabb::fadd_<true>(s, part[t]);
    return fdiv(s, (float)dabb::TNULL);
}
// a member with N == 0, inf or NaN does not contribute
DABB_HD bool noise_ok(float n) { return n > 0.f && n <= 3.40282347e38f; }

// ---- contributors of one group in one step.  Member i (ascending stream order) decoded a frame in the step (`decoded`), its phase
// reference symbol is at absolute position a[i] of the shared sample axis, its noise is noise[i]; lpos is the leader's position.
// Bit i of the result: member i contributes.  0 when the leader decoded no frame; only the leader's bit when its own noise is unusable.
DABB_HD uint32_t contributors(int n, int lpos, const int32_t* decoded, const int64_t* a, const float* noise)
{
    if (!decoded[lpos]) return 0u;
    if (!noise_ok(noise[lpos])) return 1u << lpos;
    uint32_t m = 0u;
    for (int i = 0; i < n; i++) {
        const int64_t d = a[i] - a[lpos];
        if (i == lpos || (decoded[i] && noise_ok(noise[i]) && d <= MAX_OFFSET && d >= -MAX_OFFSET)) m |= 1u << i;
    }
    return m;
}
DABB_HD int popcount(uint32_t m) { int c = 0; for (; m; m &= m - 1) c++; return c; }

// R += r1 / N
DABB_HD void acc(float2& R, float2 r1, float n)
{
    R.x = dabb::fadd_<true>(R.x, fdiv(r1.x, n));
    R.y = dabb::fadd_<true>(R.y, fdiv(r1.y, n));
}

// ---- the demap of the combined products.  DABB_DEMAP_REFERENCE: dabb::demap_r1.  DABB_DEMAP_WEIGHTED: G over the combined levels,
// from per-thread level sums (thread t: carriers t + 128 j in ascending j) added in thread order.
DABB_HD LevelSum level_partial(const float2* R /* COMB_PER_THREAD */)
{
    LevelSum a{0, 0.f};
    for (int j = 0; j < COMB_PER_THREAD; j++) dabb::level_acc(a, dabb::level_l1(R[j]));
    return a;
}
DABB_HD float level_total(const LevelSum* part /* COMB_THREADS */)
{
    LevelSum a{0, 0.f};
    for (int t = 0; t < COMB_THREADS; t++) { a.e += part[t].e; a.m = dabb::fadd_<true>(a.m, part[t].m); }
    return dabb::level_gmean(a);
}

} // namespace dabb_comb
