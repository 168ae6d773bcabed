// chan_core.cuh — the wideband channelizer's arithmetic, shared by the device kernel (chan.cu), the library's host code (api.cu) and a
// host C++ build (tests/host_emul/emul_chan.cpp) that runs the same code on the CPU.  Also the per-sample RAW conversion that
// convert_iq_kernel uses.
//
// Definition (include/dab_b200.h, DESIGN.md 3.5).  Input rate R Hz, 2 048 000 / R = L / M in lowest terms.  One Kaiser-windowed-sinc
// prototype h of L*T taps at rate L*R (cutoff 856 kHz, 72 dB design, beta = 0.1102 (72 - 8.7),
// T = ceil((72 - 7.95) / (14.36 * 176 000 / R)) + 1, designed in double, scaled to sum L, rounded to float).  Output m of a channel at
// offset f Hz on input x, with n_m = floor(m M / L) and p_m = (m M) mod L:
//   y[m] = sum_{j < T} h[p_m + j L] x[n_m - j] exp(-2 pi i k(n_m - j) / R),   k(n) = (f n) mod R, exact in integers
// An output depends on m and the input samples [n_m - T + 1, n_m] only: the channelizer keeps no state between calls.
// Evaluation order (the same in both builds, so that any cut of a run into calls gives the same bits): each input sample is converted,
// mixed with the float phase -2 ks / R (ks = k reduced to (-R/2, R/2]) through sincospi, then every output sums its taps in groups of
// four, j = 4q .. 4q + 3 in ascending q (the last group cut at T), into two accumulators (even j, odd j) with fused multiply-adds, and
// adds the two at the end.  The packed tap table is zero-padded to TP = a multiple of 4 so that every group is one aligned 16-byte load.
#pragma once
#include <math.h>
#include <stdint.h>
#include "../../include/dab_b200.h"

#if defined(__CUDACC__)
#define CHAN_HD __host__ __device__ __forceinline__
#else
#define CHAN_HD inline
#endif

namespace dabb_channel {

constexpr int64_t OUT_RATE = 2048000;
constexpr int64_t MIN_RATE = 2048000, MAX_RATE = 64000000;
constexpr int MAX_L = 1024;
constexpr int64_t HALF_BAND = 768000;                // edge of the 1536 carriers
constexpr int MAX_CHANNELS = 4096;
constexpr int64_t MAX_OUT_INDEX = int64_t(1) << 45;  // out_start + out_len at most this: m * M stays below 2^61

struct cf { float x, y; };

// ---- raw sample formats, value for value like CRAWFile::convertSamples (input/raw_file.cpp:336-363): u8 (b-128)/128, s8 b/128,
// "s16le"/"s16be" unscaled with the byte order the reference applies to each name.  Sample i of a raw (not cf32) buffer.
struct alignas(2) u8x2 { uint8_t x, y; };
struct alignas(2) s8x2 { int8_t x, y; };
struct alignas(4) u8x4 { uint8_t x, y, z, w; };
CHAN_HD cf raw_sample(const uint8_t* raw, int64_t i, int fmt)
{
    float re, im;
    if (fmt == DABB_IQ_U8) { const u8x2 b = reinterpret_cast<const u8x2*>(raw)[i]; re = (float)((int)b.x - 128) / 128.0f; im = (float)((int)b.y - 128) / 128.0f; }
    else if (fmt == DABB_IQ_S8) { const s8x2 b = reinterpret_cast<const s8x2*>(raw)[i]; re = (float)b.x / 128.0f; im = (float)b.y / 128.0f; }
    else {
        const u8x4 b = reinterpret_cast<const u8x4*>(raw)[i];
        int16_t I, Q;
        if (fmt == DABB_IQ_S16LE) { I = (int16_t)((b.x << 8) | b.y); Q = (int16_t)((b.z << 8) | b.w); }
        else { I = (int16_t)((b.y << 8) | b.x); Q = (int16_t)((b.w << 8) | b.z); }
        re = (float)I; im = (float)Q;
    }
    return cf{re, im};
}
CHAN_HD cf in_sample(const uint8_t* raw, int64_t i, int fmt)
{
    if (fmt == DABB_IQ_CF32) return reinterpret_cast<const cf*>(raw)[i];
    return raw_sample(raw, i, fmt);
}
CHAN_HD int bytes_per_sample(int fmt) { return fmt == DABB_IQ_CF32 ? 8 : ((fmt == DABB_IQ_U8 || fmt == DABB_IQ_S8) ? 2 : 4); }

// ---- exact index arithmetic
CHAN_HD int64_t floor_div(int64_t a, int64_t b) { const int64_t q = a / b; return (a % b != 0 && ((a < 0) != (b < 0))) ? q - 1 : q; }
CHAN_HD int64_t floor_mod(int64_t a, int64_t b) { const int64_t r = a % b; return r < 0 ? r + b : r; }
// k(n) = (f n) mod R with fm = f mod R: both factors below 2^26, so the product is exact in 64 bits for every n
CHAN_HD int64_t phase_index(int64_t fm, int64_t n, int64_t R) { return (fm * floor_mod(n, R)) % R; }
// the float phase (in half turns) of the mixer at phase index k: exp(-2 pi i k / R) = (cospi(a), sinpi(a)), a = -2 ks / R
CHAN_HD float mixer_arg(int64_t k, int64_t R, float inv_r) { const int64_t ks = 2 * k > R ? k - R : k; return (float)(int32_t)(-2 * ks) * inv_r; }
CHAN_HD cf mix(cf x, float s, float c) { return cf{fmaf(x.x, c, -(x.y * s)), fmaf(x.x, s, x.y * c)}; }

// output m -> last input sample n_m and the polyphase branch p_m
CHAN_HD int64_t last_input(int64_t m, int L, int M) { return floor_div(m * M, L); }

// ---- geometry and filter design (host)
struct Geometry { int64_t R; int L, M, T, TP; };

inline int64_t gcd64(int64_t a, int64_t b) { while (b) { const int64_t t = a % b; a = b; b = t; } return a; }

// DABB_OK, DABB_E_UNSUPPORTED (rate outside [2 048 000, 64 000 000] or L > 1024)
inline int geometry(int64_t R, Geometry& g)
{
    if (R < MIN_RATE || R > MAX_RATE) return DABB_E_UNSUPPORTED;
    const int64_t d = gcd64(OUT_RATE, R);
    if (OUT_RATE / d > MAX_L) return DABB_E_UNSUPPORTED;
    g.R = R; g.L = (int)(OUT_RATE / d); g.M = (int)(R / d);
    g.T = (int)ceil((72.0 - 7.95) / (14.36 * 176000.0 / (double)R)) + 1;
    g.TP = (g.T + 3) & ~3;
    return DABB_OK;
}

// an offset is accepted when the channel's 1536 carriers lie inside the input band: |f| + 768 000 <= R / 2
inline bool offset_ok(int64_t R, int64_t f) { return f > -R && f < R && 2 * ((f < 0 ? -f : f) + HALF_BAND) <= R; }

inline double bessel_i0(double x)
{
    double sum = 1.0, term = 1.0;
    const double q = 0.25 * x * x;
    for (int k = 1; k < 500; k++) {
        term *= q / ((double)k * (double)k);
        sum += term;
        if (term < 1e-17 * sum) break;
    }
    return sum;
}

// the prototype h[0 .. L*T) in float: windowed sinc in double, scaled so that the taps sum to L, rounded once
inline void design_taps(const Geometry& g, float* h)
{
    const int64_t N = (int64_t)g.L * g.T;
    const double beta = 0.1102 * (72.0 - 8.7), i0b = bessel_i0(beta), c = 0.5 * (double)(N - 1);
    const double fc = 856000.0 / ((double)g.L * (double)g.R);      // cutoff in cycles per prototype sample
    const double pi = 3.14159265358979323846;
    double* t = new double[(size_t)N];
    double sum = 0.0;
    for (int64_t n = 0; n < N; n++) {
        const double u = (double)n - c;
        const double arg = 2.0 * fc * u;
        const double s = u == 0.0 ? 1.0 : sin(pi * arg) / (pi * arg);
        const double r = c > 0.0 ? u / c : 0.0;
        const double w = bessel_i0(beta * sqrt(fmax(0.0, 1.0 - r * r))) / i0b;
        t[n] = 2.0 * fc * s * w;
        sum += t[n];
    }
    for (int64_t n = 0; n < N; n++) h[n] = (float)(t[n] * (double)g.L / sum);
    delete[] t;
}

// the taps as the kernel reads them: [TP / 4][L] groups of four, entry (q, r) = h[p + (4q + e) L] for e < 4 (0 past T), where
// p = (r M) mod L is the branch of every output m with m mod L = r (consecutive outputs read consecutive groups)
inline void pack_taps(const Geometry& g, const float* h, float* packed)
{
    for (int q = 0; q < g.TP / 4; q++)
        for (int r = 0; r < g.L; r++) {
            const int p = (int)(((int64_t)r * g.M) % g.L);
            for (int e = 0; e < 4; e++) {
                const int j = 4 * q + e;
                packed[((size_t)q * g.L + r) * 4 + e] = j < g.T ? h[(int64_t)p + (int64_t)j * g.L] : 0.0f;
            }
        }
}

// one output from mixed input: xs[0] is x[n_m] and xs[-j] is x[n_m - j]; taps4 = the packed groups + (m mod L), group q at taps4[q L].
// Only the T defined taps are summed (the last group's padding is skipped), so the output reads exactly [n_m - T + 1, n_m]
struct alignas(16) f4 { float x, y, z, w; };
CHAN_HD cf dot(const cf* xs, const f4* taps4, int L, int T)
{
    float ar = 0.f, ai = 0.f, br = 0.f, bi = 0.f;
    const int full = T / 4, rest = T % 4;
#if defined(__CUDA_ARCH__)
#pragma unroll 4
#endif
    for (int q = 0; q < full; q++) {
        const f4 h = taps4[(size_t)q * L];
        const cf x0 = xs[-4 * q], x1 = xs[-4 * q - 1], x2 = xs[-4 * q - 2], x3 = xs[-4 * q - 3];
        ar = fmaf(h.x, x0.x, ar); ai = fmaf(h.x, x0.y, ai);
        br = fmaf(h.y, x1.x, br); bi = fmaf(h.y, x1.y, bi);
        ar = fmaf(h.z, x2.x, ar); ai = fmaf(h.z, x2.y, ai);
        br = fmaf(h.w, x3.x, br); bi = fmaf(h.w, x3.y, bi);
    }
    if (rest) {
        const f4 h = taps4[(size_t)full * L];
        const cf x0 = xs[-4 * full];
        ar = fmaf(h.x, x0.x, ar); ai = fmaf(h.x, x0.y, ai);
        if (rest > 1) { const cf x1 = xs[-4 * full - 1]; br = fmaf(h.y, x1.x, br); bi = fmaf(h.y, x1.y, bi); }
        if (rest > 2) { const cf x2 = xs[-4 * full - 2]; ar = fmaf(h.z, x2.x, ar); ai = fmaf(h.z, x2.y, ai); }
    }
    return cf{ar + br, ai + bi};
}

} // namespace dabb_channel
