// tii_core.cuh — transmitter identification (TII) analysis of one stream, shared by the device kernels (tii.cu) and a host C++ build
// (tests/host_emul/emul_tii.cpp) that runs the same code on the CPU.
//
// Input per analysed frame: the two 2048-point spectra of tii_spectra_kernel (phase reference symbol p, last T_u samples of the null
// symbol that follows it n), natural bin order.  What TIIDecoder does with them (tii-decoder.cpp:236-383), restated for data-parallel
// evaluation:
//   - pair products mult[i] = sum over the blocks {1280, 1664, 1, 385} of n[k + 2i] conj(n[k + 2i + 1]), i < 192; pair i is active
//     when |mult[i]| > 0.4 |p[1 + 2i]|^2.  Pair i = c + 24 b is carrier 1 + 2c + 48b, so comb c has an 8-bit active mask A_c (bit 7 - b).
//   - votes in closed form: a pattern is an 8-bit word with four ones, so it collects >= 4 votes of comb c exactly when it is a subset
//     of A_c; the frame has sum_c C(popcount A_c, 4) likely combinations and is skipped at 10 or more.  The at most 9 others are
//     analysed in ascending (comb, pattern) order.
//   - phase-error table: for the 32 sorted carriers k_j of a combination and every delay err = -4 .. 499,
//     absErr = sum_j |arg(n[k_j] polar(1, 2 pi err k_j / 2048)) - arg(p[k_{j & ~1}])|, accumulated per (comb, pattern) with the
//     reference's uint64_t += float (truncation at every addition); the 5th analysis reports the smallest sum and starts over.
// Arithmetic: every float product and sum is rounded on its own (no contraction), as in the reference's x86-64 build.  |z| and std::norm
// are evaluated the way glibc's hypotf does (double squares and sum, double square root, one rounding), so the activity decisions are
// the reference's.  sin, cos and atan2 are evaluated in double and rounded once to float in both builds; glibc's float functions may
// differ from that in the last bit, which can move an error sum by one (DESIGN.md 5).
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define TII_HD __host__ __device__ __forceinline__
#else
#define TII_HD inline
#endif

namespace dabb_tii {

constexpr int N_PAIRS = 192;
constexpr int N_ERR = 504;          // delay hypotheses -4 .. 499 samples
constexpr int ERR_FIRST = -4;
constexpr int MAX_JOBS = 9;         // a frame with 10 or more likely combinations is skipped
constexpr int N_SLOTS = 32;         // open (comb, pattern) accumulators per stream
constexpr int N_MEAS = 5;           // analyses per report

struct cf { float x, y; };

// one open accumulator: the sums live beside it in a [N_SLOTS][N_ERR] table of the stream
struct Slot {
    int16_t comb, pattern;
    uint8_t valid, count;           // count: analyses since the last report
    uint8_t cleared, pad;           // cleared: reported at least once (its map has been cleared: the second iteration order applies)
    uint32_t stamp;                 // frame number of the last analysis (least recently analysed = evicted first)
};
struct StreamHdr {
    Slot slot[N_SLOTS];
    uint32_t frame;                 // decoded frames seen while TII was on (0 after a reset)
    uint32_t pad;
};
// one (comb, pattern) analysis of the current frame
struct Job {
    int16_t slot, comb, pattern, word;
    uint8_t start;                  // first analysis since the last report: the sums start from 0
    uint8_t table;                  // iteration-order table for the arg-min: 0 fresh map, 1 after clear()
    int8_t out;                     // index of the measurement in the step's record when this analysis reports, else -1
    uint8_t pad;
};
struct FrameSummary { int njobs, nmeas, skipped, evicted; };

// ---- arithmetic -------------------------------------------------------------------------------------------------------------------
TII_HD float fmul(float a, float b)
{
#if defined(__CUDA_ARCH__)
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}
TII_HD float fadd(float a, float b)
{
#if defined(__CUDA_ARCH__)
    return __fadd_rn(a, b);
#else
    return a + b;
#endif
}
TII_HD float fsub(float a, float b)
{
#if defined(__CUDA_ARCH__)
    return __fsub_rn(a, b);
#else
    return a - b;
#endif
}
// glibc hypotf: (float) sqrt((double) x * x + (double) y * y); the squares of floats are exact in double, so only the sum and the root round
TII_HD float abs_f(cf z)
{
    const double x = z.x, y = z.y;
#if defined(__CUDA_ARCH__)
    return (float)__dsqrt_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)));
#else
    return (float)sqrt(x * x + y * y);
#endif
}
// libstdc++ std::norm(complex<float>) = abs(z) * abs(z)
TII_HD float norm_f(cf z) { const float a = abs_f(z); return fmul(a, a); }
TII_HD float arg_f(cf z) { return (float)atan2((double)z.y, (double)z.x); }
TII_HD cf polar1_f(float theta)
{
    double s, c;
#if defined(__CUDA_ARCH__)
    sincos((double)theta, &s, &c);
#else
    s = sin((double)theta); c = cos((double)theta);
#endif
    return cf{(float)c, (float)s};
}
// std::complex<float> product a * b without contraction: (ac - bd, ad + bc)
TII_HD cf cmul(cf a, cf b) { return cf{fsub(fmul(a.x, b.x), fmul(a.y, b.y)), fadd(fmul(a.x, b.y), fmul(a.y, b.x))}; }
TII_HD cf cadd(cf a, cf b) { return cf{fadd(a.x, b.x), fadd(a.y, b.y)}; }

TII_HD int popcount8(unsigned w) { int n = 0; for (int b = 0; b < 8; b++) n += (w >> b) & 1; return n; }
TII_HD int choose4(int n) { return n < 4 ? 0 : n * (n - 1) * (n - 2) * (n - 3) / 24; }
// pattern p is the p-th 8-bit word with four ones in ascending order (EN 300 401 clause 14.8.1 table)
TII_HD unsigned pattern_word(int pattern) { for (unsigned w = 0, p = 0; w < 256; w++) if (popcount8(w) == 4 && (int)p++ == pattern) return w; return 0; }
TII_HD int bin_of(int k) { return k < 0 ? 2048 + k : k; }

// ---- pair products and activity ------------------------------------------------------------------------------------------------
// mult[i] of the reference's block loop; `null` and `prs` are the two spectra
TII_HD bool pair_active(const cf* null, const cf* prs, int i)
{
    const int starts[4] = {2048 - 768, 2048 - 384, 1, 385};
    cf m{0.f, 0.f};
    for (int q = 0; q < 4; q++) {
        const cf a = null[starts[q] + 2 * i], b = null[starts[q] + 2 * i + 1];
        m = cadd(m, cmul(a, cf{b.x, -b.y}));
    }
    return abs_f(m) > fmul(norm_f(prs[1 + 2 * i]), 0.4f);
}
// comb masks from the 192 activity flags: bit 7 - b of mask[c] = pair c + 24 b
TII_HD void comb_masks(const uint8_t* active, uint8_t* mask)
{
    for (int c = 0; c < 24; c++) {
        unsigned m = 0;
        for (int b = 0; b < 8; b++) if (active[c + 24 * b]) m |= 1u << (7 - b);
        mask[c] = (uint8_t)m;
    }
}

// ---- the analysis plan of one frame: likely combinations, accumulator slots, which analyses report --------------------------------
// Updates the stream's accumulator headers; jobs[0 .. njobs) in ascending (comb, pattern) order.
TII_HD FrameSummary plan_frame(StreamHdr& h, const uint8_t* mask, Job* jobs)
{
    FrameSummary r{0, 0, 0, 0};
    int likely = 0;
    for (int c = 0; c < 24; c++) likely += choose4(popcount8(mask[c]));
    h.frame++;
    if (likely >= 10) { r.skipped = 1; return r; }
    for (int c = 0; c < 24; c++) {
        const unsigned A = mask[c];
        if (popcount8(A) < 4) continue;
        for (unsigned w = 0, next_p = 0; w < 256; w++) {
            if (popcount8(w) != 4) continue;
            const int p = (int)next_p++;          // the pattern number of w
            if (w & ~A) continue;
            int s = -1;
            for (int q = 0; q < N_SLOTS && s < 0; q++) if (h.slot[q].valid && h.slot[q].comb == c && h.slot[q].pattern == p) s = q;
            if (s < 0) {
                for (int q = 0; q < N_SLOTS && s < 0; q++) if (!h.slot[q].valid) s = q;
                if (s < 0) {            // every slot is open: the least recently analysed one (lowest slot on a tie) starts over (DESIGN.md 5)
                    s = 0;
                    for (int q = 1; q < N_SLOTS; q++) if (h.slot[q].stamp < h.slot[s].stamp) s = q;
                    r.evicted++;
                }
                Slot z{}; z.comb = (int16_t)c; z.pattern = (int16_t)p; z.valid = 1;
                h.slot[s] = z;
            }
            Slot& z = h.slot[s];
            Job& j = jobs[r.njobs++];
            j.slot = (int16_t)s; j.comb = (int16_t)c; j.pattern = (int16_t)p; j.word = (int16_t)w;
            j.start = z.count == 0; j.table = z.cleared; j.out = -1; j.pad = 0;
            z.stamp = h.frame;
            if (++z.count >= N_MEAS) { j.out = (int8_t)r.nmeas++; z.count = 0; z.cleared = 1; }
        }
    }
    return r;
}

// ---- phase-error table ------------------------------------------------------------------------------------------------------------
// carrier j (0..31) of a combination in ascending order (CombPattern::generateCarriers sorted): four blocks of eight, each block the
// pairs k + off, k + off + 1 of the pattern's groups b in ascending order, k = 1 + 2 comb + 48 b
TII_HD int carrier(int comb, unsigned word, int j)
{
    const int offs[4] = {-769, -385, 0, 384};
    const int q = j >> 3, g = (j & 7) >> 1;
    int b = 0;
    for (int seen = -1; b < 8; b++) if (((word >> (7 - b)) & 1) && ++seen == g) break;
    return 1 + 2 * comb + 48 * b + offs[q] + (j & 1);
}
// absErr of one delay hypothesis; nv[j] = null[bin_of(k_j)], ph[j] = arg(prs[bin_of(k_{j & ~1})])
TII_HD float abs_err(const cf* nv, const float* ph, const int* car, int err)
{
    const float two_pi = fmul(2.0f, (float)M_PI);
    float acc = 0.f;
    for (int j = 0; j < 32; j++) {
        const float theta = fmul(fmul(fmul(two_pi, (float)err), (float)car[j]), 1.0f / 2048.0f);     // = the reference's / 2048.0f (a power of two)
        const float delta = fsub(arg_f(cmul(nv[j], polar1_f(theta))), ph[j]);
        acc = fadd(acc, fabsf(delta));
    }
    return acc;
}
// uint64_t += float of the reference: the sum goes to float, is added to, and is truncated back
TII_HD uint32_t accumulate(uint32_t sum, bool start, float abs_err_v) { return (uint32_t)fadd((float)(start ? 0u : sum), abs_err_v); }
// arg-min key: smallest sum first, then the entry std::min_element meets first (rank in the map's iteration order); err index in the low bits
TII_HD uint64_t argmin_key(uint32_t sum, int rank, int e) { return ((uint64_t)sum << 32) | ((uint64_t)rank << 16) | (uint64_t)e; }

} // namespace dabb_tii

#include <unordered_map>
namespace dabb_tii {
// rank[t][e]: position of key (float)(e - 4) in the iteration order of the reference's std::unordered_map<float, uint64_t> after it has
// been filled for err = -4 .. 499 in that order - t = 0 a fresh map (504 inserts with rehashes), t = 1 the same map after clear() (bucket
// count kept) filled again.  Built with the host's libstdc++, so the order is the one the reference's build iterates in.
inline void build_rank_tables(uint16_t rank[2][N_ERR])
{
    std::unordered_map<float, uint64_t> m;
    for (int t = 0; t < 2; t++) {
        if (t) m.clear();
        for (int e = 0; e < N_ERR; e++) m[(float)(e + ERR_FIRST)] += 0;
        int pos = 0;
        for (const auto& kv : m) rank[t][(int)kv.first - ERR_FIRST] = (uint16_t)pos++;
    }
}
} // namespace dabb_tii
