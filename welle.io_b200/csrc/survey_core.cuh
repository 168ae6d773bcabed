// survey_core.cuh — the spectrum survey's arithmetic (dabb_survey, survey.cu) and the candidate detector (dabb_survey_candidates), shared
// by the device kernel, the library's host code (api.cu) and a host C++ build (tests/host_emul/emul_survey.cpp, the CPU test double of
// batch_decode --scan) that runs the same code on the CPU.
//
// Spectrum (include/dab_b200.h, DESIGN.md 3.6).  Welch segments of nfft samples with 50 % overlap, S = floor((in_len - nfft) / (nfft/2)) + 1
// of them, segment s starting at sample s nfft/2; periodic Hann window w[n] = sin^2(pi n / nfft); for bin j (frequency (j - nfft/2) R / nfft)
//   P[j] = (1/S) sum_s |sum_n w[n] x[s nfft/2 + n] exp(-2 pi i k n / nfft)|^2 / sum_n w[n]^2,   k = (j + nfft/2) mod nfft,
// with sum_n w[n]^2 = 3 nfft / 8 exactly.  Evaluation: every sample is converted (chan_core.cuh's in_sample), multiplied by the float
// window, and the segment is transformed in place by radix-2 decimation in frequency (natural order in, bit-reversed order out), the
// twiddles exp(-2 pi i m / 16384) and the window sin^2(pi n / 16384) rounded once from double; a smaller nfft reads every
// (16384 / nfft)-th entry of both tables.  The segments are cut into chunks of `chunk_segments` consecutive segments: each chunk adds its
// segments' |X|^2 in float in ascending order, then the chunk sums of every bin are added in double in ascending chunk order and scaled
// by 1 / (S 3 nfft / 8).  No atomics: the same call gives the same bits.
//
// Detector: see candidates() below; plain host C++, exact integer bin membership, double sums in ascending bin order.
#pragma once
#include <math.h>
#include <stdint.h>
#include "../../include/dab_b200.h"
#include "chan_core.cuh"

#if defined(__CUDACC__)
#define SURVEY_HD __host__ __device__ __forceinline__
#else
#define SURVEY_HD inline
#endif

namespace dabb_spectrum {

using dabb_channel::cf;

constexpr int LOG2_MIN_NFFT = 10, LOG2_MAX_NFFT = 14;
constexpr int MAX_NFFT = 1 << LOG2_MAX_NFFT;
constexpr int MAX_INPUTS = 4096;
constexpr int64_t MAX_LEN = int64_t(1) << 60;

// log2(nfft) for a power of two in [1024, 16384], else -1
inline int log2_nfft(int64_t nfft)
{
    for (int l = LOG2_MIN_NFFT; l <= LOG2_MAX_NFFT; l++) if (nfft == (int64_t(1) << l)) return l;
    return -1;
}
inline int64_t n_segments(int64_t in_len, int nfft) { return (in_len - nfft) / (nfft / 2) + 1; }
// segments per chunk: about 2048 chunks over all inputs, at least 4 and at most 64 segments each (and no more than S)
inline int64_t chunk_segments(int64_t S, int n_inputs)
{
    int64_t c = (S * n_inputs + 2047) / 2048;
    c = c < 4 ? 4 : (c > 64 ? 64 : c);
    return c < S ? c : S;
}

// the tables: tw[m] = exp(-2 pi i m / 16384) for m < 8192, win[n] = sin^2(pi n / 16384) for n < 16384
inline void make_tables(cf* tw, float* win)
{
    const double pi = 3.14159265358979323846;
    for (int m = 0; m < MAX_NFFT / 2; m++) tw[m] = cf{(float)cos(-2.0 * pi * m / MAX_NFFT), (float)sin(-2.0 * pi * m / MAX_NFFT)};
    for (int n = 0; n < MAX_NFFT; n++) { const double s = sin(pi * n / MAX_NFFT); win[n] = (float)(s * s); }
}

// sample n of a segment, windowed; `in` points at the segment's first sample
SURVEY_HD cf windowed(const uint8_t* in, int64_t n, int fmt, const float* win, int log2n)
{
    const cf x = dabb_channel::in_sample(in, n, fmt);
    const float w = win[n << (LOG2_MAX_NFFT - log2n)];
    return cf{x.x * w, x.y * w};
}

// butterfly b (0 <= b < nfft/2) of the decimation-in-frequency stage with half-size h = 2^lh: (a[i0], a[i1]) <- (u + v, (u - v) tw)
SURVEY_HD void butterfly(cf* a, int lh, int b, const cf* tw, int log2n)
{
    const int h = 1 << lh, pos = b & (h - 1);
    const int i0 = ((b >> lh) << (lh + 1)) + pos, i1 = i0 + h;
    const cf u = a[i0], v = a[i1];
    const cf t = tw[pos << (LOG2_MAX_NFFT - 1 - lh)];
    const float dx = u.x - v.x, dy = u.y - v.y;
    a[i0] = cf{u.x + v.x, u.y + v.y};
    a[i1] = cf{dx * t.x - dy * t.y, dx * t.y + dy * t.x};
}

// the storage position of transform bin k after the stages (bit reversal of log2n bits)
SURVEY_HD int bin_position(int k, int log2n)
{
#if defined(__CUDA_ARCH__)
    return (int)(__brev((unsigned)k) >> (32 - log2n));
#else
    unsigned r = 0;
    for (int i = 0; i < log2n; i++) r |= (((unsigned)k >> i) & 1u) << (log2n - 1 - i);
    return (int)r;
#endif
}

// ---- candidate detector (host).  With f_j = (j - nfft/2) R / nfft and L_j = 10 log10(max(P_j, 1e-12 max P)) in double:
//   a centre bin c is considered when |f_c| + 768 000 <= R/2;
//   I = {j : |f_j - f_c| <= 700 000}; G- = {j : 784 000 <= f_c - f_j <= 896 000}, G+ = {j : 784 000 <= f_j - f_c <= 896 000}, each
//   clipped to |f_j| <= R/2 - R/nfft (1 <= j <= nfft - 1); a side is present when it keeps at least ceil(56 000 nfft / R) bins, and c is
//   skipped when neither is;
//   score(c) = mean_I L - max over present sides of mean_G L (each mean a double sum in ascending j, divided by the count);
//   every maximal run of consecutive considered bins with score >= min_score_db is one candidate at the run's midpoint
//   ((c_first + c_last - nfft) R) / (2 nfft), rounded to the nearest Hz (ties away from zero), scored with the run's largest score.
// All membership tests are exact integer comparisons of |j - c| R against multiples of nfft.
constexpr int64_t IN_BAND_HZ = 700000, GUARD_LO_HZ = 784000, GUARD_HI_HZ = 896000, GUARD_MIN_HZ = 56000;

inline int64_t round_div_away(int64_t num, int64_t den)       // num / den rounded to nearest, ties away from zero (den > 0)
{
    const int64_t a = num < 0 ? -num : num;
    const int64_t q = (2 * a + den) / (2 * den);
    return num < 0 ? -q : q;
}

// DABB_OK, or DABB_E_ARG for a bad pointer, nfft, rate or cap
inline int candidates(const float* psd, int32_t nfft, int64_t R, float min_score_db, dabb_survey_candidate* out, int32_t cap, int32_t* n_found)
{
    if (!psd || !n_found || log2_nfft(nfft) < 0 || R < 1 || R > dabb_channel::MAX_RATE || cap < 0 || (cap > 0 && !out)) return DABB_E_ARG;
    *n_found = 0;
    double pmax = 0.0;
    for (int j = 0; j < nfft; j++) if ((double)psd[j] > pmax) pmax = (double)psd[j];
    if (!(pmax > 0.0)) return DABB_OK;
    const double floor_p = 1e-12 * pmax;
    double* L = new double[(size_t)nfft];
    for (int j = 0; j < nfft; j++) { const double p = (double)psd[j]; L[j] = 10.0 * log10(p > floor_p ? p : floor_p); }
    const int64_t N = nfft, half = N / 2;
    const int64_t min_bins = (GUARD_MIN_HZ * N + R - 1) / R;
    const double thr = (double)min_score_db;
    int found = 0;
    bool in_run = false; int64_t run_first = 0, run_last = 0; double run_best = 0.0;
    auto close_run = [&]() {
        if (!in_run) return;
        if (found < cap) {
            out[found].offset_hz = round_div_away((run_first + run_last - N) * R, 2 * N);
            out[found].score_db = (float)run_best;
            out[found].reserved = 0;
        }
        found++;
        in_run = false;
    };
    for (int64_t c = 0; c < N; c++) {
        const int64_t dc = c - half;
        bool ok = 2 * (dc < 0 ? -dc : dc) * R + 2 * dabb_channel::HALF_BAND * N <= R * N;
        double score = 0.0;
        if (ok) {
            double si = 0.0; int64_t ni = 0;
            double sg[2] = {0.0, 0.0}; int64_t ng[2] = {0, 0};
            for (int64_t j = 1; j < N; j++) {           // j = 0 is -R/2: outside |f_j| <= R/2 - R/nfft, and never within 700 kHz of a centre
                const int64_t d = j - c, ad = (d < 0 ? -d : d) * R;
                if (ad <= IN_BAND_HZ * N) { si += L[j]; ni++; }
                else if (ad >= GUARD_LO_HZ * N && ad <= GUARD_HI_HZ * N) { const int side = d > 0; sg[side] += L[j]; ng[side]++; }
            }
            bool any = false; double g = 0.0;
            for (int side = 0; side < 2; side++)
                if (ng[side] >= min_bins) { const double m = sg[side] / (double)ng[side]; if (!any || m > g) g = m; any = true; }
            ok = any && ni > 0;
            if (ok) score = si / (double)ni - g;
        }
        if (ok && score >= thr) {
            if (!in_run) { in_run = true; run_first = c; run_best = score; }
            else if (score > run_best) run_best = score;
            run_last = c;
        } else close_run();
    }
    close_run();
    delete[] L;
    *n_found = found;
    return DABB_OK;
}

} // namespace dabb_spectrum
