// clock_core.cuh — sample-clock tracking (dabb_options.sample_clock = DABB_CLOCK_TRACK): the per-stream estimate of the recording's
// sample-clock error and the per-carrier phasor that removes the phase ramp it puts on the differential products.
//
// A recording whose clock runs fast by eps holds 2.048 M (1 + eps) samples per second of air time.  Every frame then ends T_F eps samples
// later than the receiver expects, so the time synchronisation finds the phase reference symbol that much behind T_g: over frames the
// mean of start_index - 504 is T_F eps (the placement's own bias telescopes, the rounding of idx carries over into the next frame's
// position).  Within a frame each symbol's FFT window is eps T_s samples earlier relative to its symbol than the one before, which
// rotates carrier k's differential product by -2 pi k eps T_s / T_u; the demodulator multiplies it back.
//
// Everything here is __host__ __device__ so tests/host_emul runs the identical arithmetic on the CPU.
#pragma once
#include "ofdm_core.cuh"

namespace dabb_clock {

constexpr int REF_INDEX = dabb::TG;     // start_index of a frame that ends exactly where the previous one said
constexpr int D_MAX = 64;               // |start_index - 504| counted: 64 samples per frame = 325 ppm; beyond it a placement jump or re-sync
constexpr int N_APPLY = 8;              // frames counted before the estimate is applied
constexpr int N_AVG = 32;               // running mean over the first 32 counted frames, then an exponential average of 32 frames

// one stream's estimator (StreamState in api.cu)
struct State {
    double e;           // ppm
    int32_t n;          // frames counted, saturating at INT32_MAX
    int32_t prev;       // 1: the previous active step of the stream decoded a frame (with the option TRACK)
};

DABB_HD double dadd(double a, double b)
{
#if defined(__CUDA_ARCH__)
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}
DABB_HD double ddiv(double a, double b)
{
#if defined(__CUDA_ARCH__)
    return __ddiv_rn(a, b);
#else
    return a / b;
#endif
}

// a frame decoded with TRACK at start_index: e <- e + (1e6 d / T_F - e) / min(n, 32) when it counts
DABB_HD void update(State& s, int32_t start_index)
{
    const int d = start_index - REF_INDEX;
    if (s.prev && d >= -D_MAX && d <= D_MAX) {
        if (s.n < 0x7FFFFFFF) s.n++;
        const double x = ddiv(1e6 * (double)d, (double)dabb::TF);
        s.e = dadd(s.e, ddiv(dadd(x, -s.e), (double)(s.n < N_AVG ? s.n : N_AVG)));
    }
    s.prev = 1;
}

// the value a frame is derotated with: the estimate from before the frame, once N_APPLY frames have been counted
DABB_HD double applied(const State& s) { return s.n >= N_APPLY ? s.e : 0.0; }

// e^{i pi x}
DABB_HD float2 unit_halfturns(double x)
{
#if defined(__CUDA_ARCH__)
    double sn, cs;
    sincospi(x, &sn, &cs);
#else
    const double sn = sin(3.14159265358979323846 * x), cs = cos(3.14159265358979323846 * x);
#endif
    return make_float2((float)cs, (float)sn);
}
// half turns per carrier of the ramp removed at ppm: 2 ppm 1e-6 T_s / T_u
DABB_HD double halfturns_per_carrier(float ppm) { return 2e-6 * (double)ppm * (double)dabb::TS / (double)dabb::TU; }

// a * b with explicitly rounded fused operations (the same bits on host and device)
DABB_HD float2 cmul(float2 a, float2 b)
{
#if defined(__CUDA_ARCH__)
    return make_float2(__fmaf_rn(a.x, b.x, -__fmul_rn(a.y, b.y)), __fmaf_rn(a.x, b.y, __fmul_rn(a.y, b.x)));
#else
    return make_float2(fmaf(a.x, b.x, -(a.y * b.y)), fmaf(a.x, b.y, a.y * b.x));
#endif
}

// Phasor of carrier k (-768..768) at ppm: e^{+2 pi i k ppm 1e-6 T_s / T_u} as the product of two float factors, P[k & 127] Q[k >> 7]
// (k = t + 128 j, the bins a thread of the demodulator owns share t), each rounded from double: every component is within 2^-22 of the
// exact value.  The demodulator keeps P of its thread in registers and Q[-6..6] in shared memory (Q[-j] = conj(Q[j])).
DABB_HD float2 factor_p(int t, float ppm) { return unit_halfturns(halfturns_per_carrier(ppm) * (double)t); }
DABB_HD float2 factor_q(int j, float ppm)
{
    const float2 q = unit_halfturns(halfturns_per_carrier(ppm) * (double)(128 * (j < 0 ? -j : j)));
    return j < 0 ? make_float2(q.x, -q.y) : q;
}
DABB_HD float2 phasor(int k, float ppm) { return cmul(factor_p(k & 127, ppm), factor_q(k >> 7, ppm)); }

} // namespace dabb_clock
