// acq_core.cuh — robust acquisition (dabb_options.acquisition = DABB_ACQ_ROBUST): the arithmetic of the spectral null-symbol search
// (acq_level_kernel, acq_decide_kernel in acq.cu) and of the interferer excision in the phase reference correlation
// (find_index_excise_kernel in ofdm.cu).  Plain C++ plus the DABB_HD building blocks of ofdm_core.cuh, so that the host test
// (tests/host_emul/emul_acq.cpp) compiles exactly what the kernels run; every operation is rounded on its own and every sum runs in a
// fixed order, so the device and the host build give the same bits.
//
// The level of a block of 256 samples is the mean of log2 of the Hann-windowed power spectrum over the bins within 700 kHz of the
// centre: the log of the geometric mean of the in-band bin powers.  The null symbol (2656 samples) holds nine whole blocks at any
// alignment; during it the level drops by the signal-to-noise ratio in dB (about 3.6 dB at 0 dB SNR).  A narrowband interferer lifts a
// handful of bins, which barely moves a mean of logs, so unlike the reference's 50-sample envelope dip the search still sees the null.
#pragma once
#include "ofdm_core.cuh"
#include <string.h>

namespace dabb_acq {

constexpr int BLK = 256;                 // samples per block; blocks are aligned to the search start
constexpr int HALF = 87;                 // in-band bins: |k| <= 87, |k| * 8 kHz <= 700 kHz
constexpr int NBIN = 2 * HALF + 1;       // 175
constexpr int WIN = 9;                   // blocks of a window: 9 * 256 = 2304 <= 2656 - 255, wholly inside the null at any alignment
constexpr int NB_MAX = 784;              // blocks per search: 200 704 samples, one frame period plus a null and some slack
constexpr int CHUNK = 8;                 // blocks per CTA of acq_level_kernel, one warp each
constexpr int MIN_BLOCKS = 32;           // fewer samples than this many blocks: the stream does not search in this step
constexpr int EDGE = 2;                  // a found window must end at least this many blocks before the span does
constexpr int KEEP = 11;                 // a search that finds nothing keeps its last KEEP blocks for the next one
constexpr int NULL_END = 2480;           // estimated null end after the best window's first sample (midpoint of 2304 .. 2656)
constexpr int LEAD = 256;                // tracking starts this many samples before the estimated null end
constexpr float DEPTH_DB = 1.2f;         // D: a null is found when its window is at least this far below the span's median level
constexpr float DB_PER_LOG2 = 3.01029996f;   // 10 log10(2)
constexpr float TINY = 1.17549435e-38f;  // 2^-126: the smallest power a level reads
constexpr float HUGE_P = 3.40282347e38f;
// excision in the phase reference correlation: bins whose power exceeds T times the geometric mean of the in-band bin powers, and
// their EXC_NEIGH neighbours on each side, are zeroed before the multiply by conj(PRS)
constexpr float LOG2_T = 4.32192809f;    // log2(20): T = 20
constexpr int EXC_NEIGH = 2;
constexpr int EXC_THREADS = 128;         // find_index_kernel's CTA: thread t owns the bins t + 128 c, c = 0 .. 15
constexpr int EXC_INBAND = 1536;         // bins 1 .. 768 and 1280 .. 2047

using dabb::fmul_; using dabb::fadd_; using dabb::fsub_;

DABB_HD uint32_t bits_of(float x)
{
#if defined(__CUDA_ARCH__)
    return __float_as_uint(x);
#else
    uint32_t u; memcpy(&u, &x, 4); return u;
#endif
}
DABB_HD float from_bits(uint32_t u)
{
#if defined(__CUDA_ARCH__)
    return __uint_as_float(u);
#else
    float x; memcpy(&x, &u, 4); return x;
#endif
}
DABB_HD float fdiv(float a, float b)
{
#if defined(__CUDA_ARCH__)
    return __fdiv_rn(a, b);
#else
    return a / b;
#endif
}

// the power a level reads: max(P, 2^-126) clipped to FLT_MAX (NaN reads as 2^-126, +inf as FLT_MAX), so every level is finite
DABB_HD float clamp_power(float p) { return fminf(fmaxf(p, TINY), HUGE_P); }

// log2 of a finite x >= 2^-126: x = m 2^e with m in [sqrt(1/2), sqrt(2)), log2 m = (2 / ln 2) atanh((m - 1) / (m + 1)) from its odd
// series to t^9 (|t| <= 0.1716: truncation below 2e-9), each operation rounded; within 3e-7 of log2 x
DABB_HD float log2_pos(float x)
{
    const uint32_t b = bits_of(x);
    int e = (int)(b >> 23) - 127;
    float m = from_bits((b & 0x7FFFFFu) | 0x3F800000u);
    if (m > 1.41421356f) { m = fmul_<true>(m, 0.5f); e++; }
    const float t = fdiv(fsub_<true>(m, 1.f), fadd_<true>(m, 1.f));
    const float t2 = fmul_<true>(t, t);
    float p = fadd_<true>(fmul_<true>(t2, 0.111111111f), 0.142857143f);
    p = fadd_<true>(fmul_<true>(p, t2), 0.2f);
    p = fadd_<true>(fmul_<true>(p, t2), 0.333333333f);
    p = fadd_<true>(fmul_<true>(p, t2), 1.f);
    return fadd_<true>((float)e, fmul_<true>(fmul_<true>(fmul_<true>(2.f, t), p), 1.44269504f));
}

// ---- block level ---------------------------------------------------------------------------------------------------------------
// cos_tab[n] = (float)cos(2 pi n / 256), n = 0 .. 255, rounded from double on the host (make_cos_table) and uploaded
inline void make_cos_table(float* tab)
{
    for (int n = 0; n < BLK; n++) tab[n] = (float)cos(6.283185307179586476925 * n / BLK);
}
// periodic Hann window w[n] = sin^2(pi n / 256) = 0.5 - 0.5 cos(2 pi n / 256)
DABB_HD float hann(const float* cos_tab, int n) { return fsub_<true>(0.5f, fmul_<true>(0.5f, cos_tab[n])); }
DABB_HD int bitrev8(int n)
{
    n = ((n & 0x0F) << 4) | ((n & 0xF0) >> 4);
    n = ((n & 0x33) << 2) | ((n & 0xCC) >> 2);
    return ((n & 0x55) << 1) | ((n & 0xAA) >> 1);
}
// butterfly q (0 .. 127) of the radix-2 decimation-in-time stage with half-size h (1, 2, 4, ... 128) on x in bit-reversed input order:
// i = (q / h) 2h + q mod h, W = exp(-2 pi i (q mod h) (128 / h) / 256); x[i] = a + W b, x[i + h] = a - W b
DABB_HD void butterfly(float2* x, const float* cos_tab, int h, int q)
{
    const int j = q & (h - 1), i = ((q - j) << 1) + j;
    const int k = j * (128 / h);
    const float2 w = make_float2(cos_tab[k], -cos_tab[(k + 192) & 255]);       // sin(2 pi k / 256) = cos(2 pi (k - 64) / 256)
    const float2 a = x[i], b = dabb::cmul_<true>(x[i + h], w);
    x[i] = dabb::cadd_<true>(a, b);
    x[i + h] = dabb::csub_<true>(a, b);
}
// lane t's partial sum of the log2 powers of the in-band bins j = t, t + 32, ... (j = 0 .. 174, bin k = j - 87) in ascending order
DABB_HD float level_partial(const float2* X, int t)
{
    float s = 0.f;
    for (int j = t; j < NBIN; j += 32) {
        const float2 v = X[(j - HALF + BLK) & (BLK - 1)];
        s = fadd_<true>(s, log2_pos(clamp_power(fadd_<true>(fmul_<true>(v.x, v.x), fmul_<true>(v.y, v.y)))));
    }
    return s;
}
// the block's level from the 32 partials, added in lane order, divided by 175
DABB_HD float level_total(const float* part)
{
    float s = 0.f;
    for (int t = 0; t < 32; t++) s = fadd_<true>(s, part[t]);
    return fdiv(s, (float)NBIN);
}
// |Re| + |Im| of a (mixed) sample, summed per lane over n = t, t + 32, ... and then in lane order: the block's envelope sum
DABB_HD float l1_of(float2 y) { return fadd_<true>(fabsf(y.x), fabsf(y.y)); }

// ---- the decision over a span of nb blocks -------------------------------------------------------------------------------------
// W[b] = level[b] + ... + level[b + 8] (ascending); the best window is the last b with the smallest W, so that in a run of digital
// silence (equal levels) tracking starts where the silence ends
DABB_HD float window_sum(const float* level, int b)
{
    float s = 0.f;
    for (int i = 0; i < WIN; i++) s = fadd_<true>(s, level[b + i]);
    return s;
}
// depth (dB) of a window below the span's median level M (the ((nb - 1) / 2)-th smallest level, counted from 0)
DABB_HD float depth_db(float median, float wsum)
{
    return fmul_<true>(fsub_<true>(median, fdiv(wsum, (float)WIN)), DB_PER_LOG2);
}
DABB_HD bool is_found(float depth, int best, int nb) { return depth >= DEPTH_DB && best + WIN + EDGE <= nb; }

// ---- interferer excision ------------------------------------------------------------------------------------------------------
DABB_HD bool in_band(int bin) { return bin != 0 && (bin <= 768 || bin >= 2048 - 768); }
// thread t's partial sum of log2 of the clamped powers of its in-band bins t + 128 c, c ascending
DABB_HD float exc_partial(const float* pw, int t)
{
    float s = 0.f;
    for (int c = 0; c < 16; c++) { const int bin = t + EXC_THREADS * c; if (in_band(bin)) s = fadd_<true>(s, log2_pos(clamp_power(pw[bin]))); }
    return s;
}
// log2 G + log2 T from the 128 partials added in thread order: a bin is an interferer when log2 of its clamped power exceeds this
DABB_HD float exc_limit(const float* part)
{
    float s = 0.f;
    for (int t = 0; t < EXC_THREADS; t++) s = fadd_<true>(s, part[t]);
    return fadd_<true>(fdiv(s, (float)EXC_INBAND), LOG2_T);
}
DABB_HD bool exc_over(float p, int bin, float limit) { return in_band(bin) && log2_pos(clamp_power(p)) > limit; }

} // namespace dabb_acq
