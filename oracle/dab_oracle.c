/*
 * dab_oracle.c — plain-C CPU restatement of the welle.io DAB/DAB+ PHY decode path (Mode I).
 *
 * TEST INFRASTRUCTURE ONLY — see dab_oracle.h.  Written from the behaviour of the reference
 * (/root/reference/src, cited per function as file:line); no reference source is copied.  Float stages keep
 * the reference's operation order so that, compiled without FMA contraction (-ffp-contract=off, see
 * oracle/Makefile), results are bit-identical to the reference's KISS-FFT build (oracle/_ref/libwelle_ref.so).
 * Parity status: PINNED by tests/test_oracle_vs_ref.py and tests/golden/.
 */
#include "dab_oracle.h"
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <stdio.h>

#ifndef M_PI
#define M_PI 3.14159265358979323846
#endif

typedef struct { float r, i; } cf;

/* ============================================================================================
 * Tables
 * ========================================================================================== */

/* ETSI EN 300 401 §14.6 frequency interleaver as built by backend/freq-interleaver.cpp:35-59:
 * Pi(0)=0, Pi(i)=(13*Pi(i-1)+511) mod 2048; keep 256<=Pi<=1792, Pi!=1024; carrier = Pi-1024. */
void orc_perm_table(int16_t out[ORC_K])
{
    int pi = 0, n = 0;
    for (int i = 0; i < ORC_TU; i++) {
        if (i > 0) pi = (13 * pi + 511) % ORC_TU;
        if (pi == ORC_TU / 2 || pi < 256 || pi > 256 + ORC_K) continue;
        out[n++] = (int16_t)(pi - ORC_TU / 2);
    }
}

/* ETSI EN 300 401 Table 39 (Mode I) as encoded in backend/phasetable.cpp:24-75: 48 blocks of 32 carriers.
 * Block b<24 covers k = -768+32b .. -737+32b, block b>=24 covers k = 1+32(b-24) .. 32+32(b-24).
 * Each block has (i, n): phi_k = pi/2 * (h[i][k - kmin] + n).  */
static const uint8_t PRS_I[48] = {
    0,1,2,3, 0,1,2,3, 0,1,2,3, 0,1,2,3, 0,1,2,3, 0,1,2,3,
    0,3,2,1, 0,3,2,1, 0,3,2,1, 0,3,2,1, 0,3,2,1, 0,3,2,1 };
static const uint8_t PRS_N[48] = {
    1,2,0,1, 3,2,2,3, 2,1,2,3, 1,2,3,3, 2,2,2,1, 1,3,1,2,
    3,1,1,1, 2,2,1,0, 2,2,3,3, 0,2,1,3, 3,3,3,0, 3,0,1,1 };
/* ETSI Table 38 h_{i,j}, j = 0..15 (period 16; phasetable.cpp:138-152 stores 32 entries) */
static const uint8_t PRS_H[4][16] = {
    {0,2,0,0,0,0,1,1,2,0,0,0,2,2,1,1},
    {0,3,2,3,0,1,3,0,2,1,2,3,2,3,3,0},
    {0,0,0,2,0,2,1,3,2,2,0,2,2,0,1,3},
    {0,1,2,1,0,3,3,2,2,3,2,1,2,1,3,2} };

/* PhaseTable::get_Phi (phasetable.cpp:172-183) returns DSPFLOAT: the double product is rounded to float. */
static float prs_phi(int k)
{
    int b, kmin;
    if (k < 0) { b = (k + 768) / 32; kmin = -768 + 32 * b; }
    else       { b = 24 + (k - 1) / 32; kmin = 1 + 32 * (b - 24); }
    int h = PRS_H[PRS_I[b]][(k - kmin) & 15];
    return (float)(M_PI / 2.0f * (h + PRS_N[b]));
}

/* PhaseReference ctor, phasereference.cpp:45-51: refTable[i] = (cos phi_i, sin phi_i), refTable[T_u-i] for -i.
 * phi_k is a float; the unqualified cos/sin there resolve to the float overloads. */
void orc_prs_table(float out[2 * ORC_TU])
{
    memset(out, 0, sizeof(float) * 2 * ORC_TU);
    for (int i = 1; i <= ORC_K / 2; i++) {
        float p = prs_phi(i);
        out[2 * i] = cosf(p); out[2 * i + 1] = sinf(p);
        p = prs_phi(-i);
        out[2 * (ORC_TU - i)] = cosf(p); out[2 * (ORC_TU - i) + 1] = sinf(p);
    }
}

/* ETSI Table 13 puncturing vectors PI_1..PI_24 (backend/protTables.cpp:25-51).  Rule: every 4-bit group
 * starts as 1000; PI_p switches on one more bit per step, visiting the 8 groups in the order 0,4,2,6,1,5,3,7,
 * second column for p=1..8, third for p=9..16, fourth for p=17..24. */
void orc_pcodes(int8_t out[24 * 32])
{
    static const int order[8] = {0, 4, 2, 6, 1, 5, 3, 7};
    for (int p = 1; p <= 24; p++) {
        int8_t* v = out + 32 * (p - 1);
        for (int g = 0; g < 8; g++) { v[4 * g] = 1; v[4 * g + 1] = v[4 * g + 2] = v[4 * g + 3] = 0; }
        for (int q = 1; q <= p; q++) v[4 * order[(q - 1) & 7] + 1 + (q - 1) / 8] = 1;
    }
}

static const uint8_t PI_TAIL[24] = {1,1,0,0,1,1,0,0,1,1,0,0,1,1,0,0,1,1,0,0,1,1,0,0};   /* fic-handler.cpp:39-42 */

/* PRBS x^9+x^5+1, all-ones start: fic-handler.cpp:62-71 and energy_dispersal.h:40-49 */
void orc_prbs(uint8_t* out, int n)
{
    unsigned reg = 0x1FF;
    for (int i = 0; i < n; i++) {
        unsigned b = ((reg >> 8) ^ (reg >> 4)) & 1;
        reg = ((reg << 1) | b) & 0x1FF;
        out[i] = (uint8_t)b;
    }
}

/* ============================================================================================
 * FFT — restatement of libs/kiss_fft/kiss_fft.c for power-of-two sizes.
 * kf_factor (kiss_fft.c:309-330) peels radix 4 while divisible, then radix 2: 2048 = 4*4*4*4*4*2.
 * kf_work (:243-302) is a decimation-in-time recursion; butterflies kf_bfly2 (:22-43), kf_bfly4 (:45-91).
 * Twiddles: (float)cos / (float)sin of the double phase -2*pi*i/n (:356-364).  Complex multiply is
 * r = ar*br - ai*bi, i = ar*bi + ai*br (_kiss_fft_guts.h C_MUL).
 * ========================================================================================== */
typedef struct { int n, inverse; cf* tw; int fac[64]; } fftplan;

static void plan_init(fftplan* p, int n, int inverse)
{
    p->n = n; p->inverse = inverse;
    p->tw = (cf*)malloc(sizeof(cf) * n);
    for (int i = 0; i < n; i++) {
        const double pi = 3.141592653589793238462643383279502884197169399375105820974944;
        double ph = -2 * pi * i / n;
        if (inverse) ph *= -1;
        p->tw[i].r = (float)cos(ph); p->tw[i].i = (float)sin(ph);
    }
    int m = n, k = 0, r = 4;
    while (m > 1) {
        while (m % r) r = 2;
        m /= r; p->fac[k++] = r; p->fac[k++] = m;
    }
}

static inline cf cmul(cf a, cf b) { cf m; m.r = a.r * b.r - a.i * b.i; m.i = a.r * b.i + a.i * b.r; return m; }
static inline cf cadd(cf a, cf b) { cf m; m.r = a.r + b.r; m.i = a.i + b.i; return m; }
static inline cf csub(cf a, cf b) { cf m; m.r = a.r - b.r; m.i = a.i - b.i; return m; }

static void fft_rec(const fftplan* p, cf* out, const cf* f, int fstride, const int* fac)
{
    const int radix = fac[0], m = fac[1];
    if (m == 1) {
        for (int q = 0; q < radix; q++) out[q] = f[(size_t)q * fstride];
    } else {
        for (int q = 0; q < radix; q++) fft_rec(p, out + (size_t)q * m, f + (size_t)q * fstride, fstride * radix, fac + 2);
    }
    if (radix == 2) {
        for (int k = 0; k < m; k++) {
            cf t = cmul(out[m + k], p->tw[(size_t)k * fstride]);
            out[m + k] = csub(out[k], t);
            out[k] = cadd(out[k], t);
        }
    } else { /* radix 4 */
        for (int k = 0; k < m; k++) {
            cf s0 = cmul(out[k + m], p->tw[(size_t)k * fstride]);
            cf s1 = cmul(out[k + 2 * m], p->tw[(size_t)k * fstride * 2]);
            cf s2 = cmul(out[k + 3 * m], p->tw[(size_t)k * fstride * 3]);
            cf s5 = csub(out[k], s1);
            out[k] = cadd(out[k], s1);
            cf s3 = cadd(s0, s2);
            cf s4 = csub(s0, s2);
            out[k + 2 * m] = csub(out[k], s3);
            out[k] = cadd(out[k], s3);
            if (p->inverse) {
                out[k + m].r = s5.r - s4.i;     out[k + m].i = s5.i + s4.r;
                out[k + 3 * m].r = s5.r + s4.i; out[k + 3 * m].i = s5.i - s4.r;
            } else {
                out[k + m].r = s5.r + s4.i;     out[k + m].i = s5.i - s4.r;
                out[k + 3 * m].r = s5.r - s4.i; out[k + 3 * m].i = s5.i + s4.r;
            }
        }
    }
}

static fftplan g_fwd2048, g_inv2048;
static int g_plans_ready = 0;
static void ensure_plans(void)
{
    if (!g_plans_ready) { plan_init(&g_fwd2048, ORC_TU, 0); plan_init(&g_inv2048, ORC_TU, 1); g_plans_ready = 1; }
}

void orc_fft(int n, const float* in, float* out, int inverse)
{
    fftplan local; const fftplan* p;
    ensure_plans();
    if (n == ORC_TU) p = inverse ? &g_inv2048 : &g_fwd2048;
    else { plan_init(&local, n, inverse); p = &local; }
    cf* tmp = (cf*)malloc(sizeof(cf) * n);
    fft_rec(p, tmp, (const cf*)in, 1, p->fac);
    memcpy(out, tmp, sizeof(cf) * n);
    free(tmp);
    if (p == &local) free(local.tw);
}

/* fft::Backward::do_IFFT, various/fft.cpp:146-158: factor = 1.0f/N, every entry *= factor */
void orc_ifft_scaled(int n, const float* in, float* out)
{
    orc_fft(n, in, out, 1);
    const float factor = 1.0f / (float)n;
    for (int i = 0; i < 2 * n; i++) out[i] *= factor;
}

/* ============================================================================================
 * Time sync — PhaseReference::findIndex, phasereference.cpp:73-97 + ThresholdBeforePeak :212-253
 * ========================================================================================== */
static float g_prs[2 * ORC_TU];
static int16_t g_perm[ORC_K];
static int g_tables_ready = 0;
static void ensure_tables(void)
{
    if (!g_tables_ready) { orc_prs_table(g_prs); orc_perm_table(g_perm); g_tables_ready = 1; }
}

int orc_find_index(const float* v, float* cir_out)
{
    ensure_tables();
    const int Tu = ORC_TU;
    cf* spec = (cf*)malloc(sizeof(cf) * Tu);
    cf* res = (cf*)malloc(sizeof(cf) * Tu);
    float* cir = (float*)malloc(sizeof(float) * Tu);
    float* pk = (float*)calloc(Tu, sizeof(float));
    orc_fft(Tu, v, (float*)spec, 0);
    /* res = fft * conj(ref)  (std::complex product: re = a*c - b*(-d), im = a*(-d) + b*c) */
    for (int i = 0; i < Tu; i++) {
        float a = spec[i].r, b = spec[i].i, c = g_prs[2 * i], d = -g_prs[2 * i + 1];
        res[i].r = a * c - b * d;
        res[i].i = a * d + b * c;
    }
    orc_ifft_scaled(Tu, (const float*)res, (float*)res);
    float sum = 0;
    for (int i = 0; i < Tu; i++) { float a = hypotf(res[i].r, res[i].i); cir[i] = a; sum += a; }
    if (cir_out) memcpy(cir_out, cir, sizeof(float) * Tu);
    const int W = 100;
    float gmax = -10000;
    for (int i = 0; i + W < Tu; i++) {
        float mx = -10000;
        for (int j = 0; j < W; j++) if (cir[i + j] > mx) mx = cir[i + j];
        pk[i] = mx;
        if (mx > gmax) gmax = mx;
    }
    int ret = -1;
    if (gmax > 3 * sum / Tu) {
        const float thresh = gmax / 2;
        for (int i = 0; i + W < Tu; i++) if (pk[i + W] > thresh) { ret = i; break; }
    }
    free(spec); free(res); free(cir); free(pk);
    return ret;
}

/* The two non-default FFT placements of PhaseReference::findIndex (phasereference.cpp:93-211) */
int orc_find_index_m(const float* v, float* cir_out, int placement)
{
    if (placement == 0) return orc_find_index(v, cir_out);
    ensure_tables();
    const int Tu = ORC_TU;
    cf* spec = (cf*)malloc(sizeof(cf) * Tu);
    cf* res = (cf*)malloc(sizeof(cf) * Tu);
    float* cir = (float*)calloc(Tu, sizeof(float));
    orc_fft(Tu, v, (float*)spec, 0);
    for (int i = 0; i < Tu; i++) {
        float a = spec[i].r, b = spec[i].i, c = g_prs[2 * i], d = -g_prs[2 * i + 1];
        res[i].r = a * c - b * d;
        res[i].i = a * d + b * c;
    }
    orc_ifft_scaled(Tu, (const float*)res, (float*)res);
    int ret = -1;
    if (placement == 1) {
        /* StrongestPeak (:93-123): running sum and first maximum in one pass */
        float sum = 0, max = -10000; int maxIndex = -1;
        for (int i = 0; i < Tu; i++) {
            const float value = hypotf(res[i].r, res[i].i);
            sum += value; cir[i] = value;
            if (value > max) { maxIndex = i; max = value; }
        }
        if (sum == 0) ret = -1;
        else if (max < 3.0f * sum / (float)Tu) ret = (int)(-fabsf(max * (float)Tu / sum) - 1);
        else ret = maxIndex;
    } else {
        /* EarliestPeakWithBinning (:124-211): peaks of 20-sample bins (the last 8 samples are never looked at), the four
         * strongest bins within 500 samples of the strongest, those above 3 x mean, the earliest of them.
         * std::sort is not stable: bins of exactly equal value may come out in another order than here (ties broken
         * towards the earlier bin). */
        enum { BIN = 20, KEEP = 4, MAXB = 128 };
        int idx[MAXB]; float val[MAXB]; int nb = 0;
        float mean = 0;
        for (int i = 0; i + BIN < Tu; i += BIN) {
            int pi = -1; float pv = 0;
            for (int j = 0; j < BIN; j++) {
                const float value = hypotf(res[i + j].r, res[i + j].i);
                mean += value; cir[i + j] = value;
                if (value > pv) { pv = value; pi = i + j; }
            }
            idx[nb] = pi; val[nb] = pv; nb++;
        }
        mean /= (float)Tu;
        /* descending selection, stable */
        int order[MAXB]; char used[MAXB]; memset(used, 0, sizeof used);
        for (int k = 0; k < nb; k++) {
            int best = -1;
            for (int b = 0; b < nb; b++) if (!used[b] && (best < 0 || val[b] > val[best])) best = b;
            used[best] = 1; order[k] = best;
        }
        const int peak_index = idx[order[0]];
        int kept[KEEP], nk = 0;
        for (int k = 0; k < nb && nk < KEEP; k++) if (abs(idx[order[k]] - peak_index) <= 500) kept[nk++] = order[k];
        const float thresh = 3 * mean;
        int earliest = -1, have = 0;
        for (int k = 0; k < nk; k++) {
            if (val[kept[k]] < thresh) continue;
            if (!have || idx[kept[k]] < earliest) { earliest = idx[kept[k]]; have = 1; }
        }
        ret = have ? earliest : -1;
    }
    if (cir_out) memcpy(cir_out, cir, sizeof(float) * Tu);
    free(spec); free(res); free(cir);
    return ret;
}

/* OFDMProcessor::processPRS, FreqsyncMethod::PatternOfZeros, ofdm-processor.cpp:582-613.
 * std::arg -> atan2f.  IMPORTANT: in that translation unit the unqualified `abs` applied to a float or a double resolves
 * to the C library's `int abs(int)` (libstdc++'s <cmath> only declares the floating overloads inside namespace std, and
 * nothing there says `using namespace std`), so every `abs(arg(..))` TRUNCATES its argument to int first — verified with the
 * reference's own headers (typeid(abs(0.7f)) is int) and pinned against the compiled reference (ref_process_prs).
 * The metric is therefore a small integer: a1, a2, b1 are 1 unless the argument is exactly +-(float)pi, the other six terms
 * are trunc|arg| in 0..3.  Returns carrier offset, 100 = "no estimate". */
static float argprod(const cf* s, int i, int j)
{
    const int Tu = ORC_TU;
    cf a = s[i % Tu], b = s[j % Tu];
    float c = b.r, d = -b.i;
    float re = a.r * c - a.i * d, im = a.r * d + a.i * c;
    return atan2f(im, re);
}
static int iabs_f(float x) { int v = (int)x; return v < 0 ? -v : v; }           /* abs(float)  -> int abs(int) */
static int iabs_pi(float x) { int v = (int)((double)x / M_PI); v = v < 0 ? -v : v; v -= 1; return v < 0 ? -v : v; }   /* abs(abs(x / M_PI) - 1) */
int orc_coarse_pattern_of_zeros(const float* prs)
{
    const int Tu = ORC_TU, RANGE2 = 72;
    cf* s = (cf*)malloc(sizeof(cf) * Tu);
    orc_fft(Tu, prs, (float*)s, 0);
    int index = 100;
    float Mmin = 1000;
    for (int i = Tu - RANGE2 / 2; i < Tu + RANGE2 / 2; i++) {
        float a1 = (float)iabs_pi(argprod(s, i + 1, i + 2));
        float a2 = (float)iabs_pi(argprod(s, i + 2, i + 3));
        float a3 = (float)iabs_f(argprod(s, i + 3, i + 4));
        float a4 = (float)iabs_f(argprod(s, i + 4, i + 5));
        float a5 = (float)iabs_f(argprod(s, i + 5, i + 6));
        float b1 = (float)iabs_pi(argprod(s, i + 16 + 1, i + 16 + 3));
        float b2 = (float)iabs_f(argprod(s, i + 16 + 3, i + 16 + 4));
        float b3 = (float)iabs_f(argprod(s, i + 16 + 4, i + 16 + 5));
        float b4 = (float)iabs_f(argprod(s, i + 16 + 5, i + 16 + 6));
        float sum = a1 + a2 + a3 + a4 + a5 + b1 + b2 + b3 + b4;
        if (sum < Mmin) { Mmin = sum; index = i; }
    }
    free(s);
    return index - Tu;   /* :612 returns index - T_u unconditionally */
}

/* FreqsyncMethod::GetMiddle (ofdm-processor.cpp:617-644, including its `sum = oldMax` assignment) and
 * FreqsyncMethod::CorrelatePRS (:546-581; refArg from the ctor :96-101) */
int orc_coarse(const float* prs, int method)
{
    if (method == 0) return orc_coarse_pattern_of_zeros(prs);
    ensure_tables();
    const int Tu = ORC_TU, K = ORC_K;
    cf* s = (cf*)malloc(sizeof(cf) * Tu);
    orc_fft(Tu, prs, (float*)s, 0);
    int ret;
    if (method == 1) {
        float sum = 0, oldMax = 0; int maxIndex = 0;
        for (int i = 40; i < K + 40; i++) { const cf z = s[(Tu / 2 + i) % Tu]; sum += hypotf(z.r, z.i); }
        for (int i = 40; i < Tu - (K - 40); i++) {
            const cf a = s[(Tu / 2 + i) % Tu], b = s[(Tu / 2 + i + K) % Tu];
            sum -= hypotf(a.r, a.i);
            sum += hypotf(b.r, b.i);
            if (sum > oldMax) { sum = oldMax; maxIndex = i; }
        }
        ret = (int16_t)(maxIndex - (Tu - K) / 2);
    } else {
        enum { SEARCH = 72, CORR = 24 };
        float refArg[CORR], cv[SEARCH + CORR];
        const cf* ref = (const cf*)g_prs;
        for (int i = 0; i < CORR; i++) {
            const cf a = ref[(Tu + i) % Tu], b = ref[(Tu + i + 1) % Tu];
            const float c = b.r, d = -b.i;
            refArg[i] = atan2f(a.r * d + a.i * c, a.r * c - a.i * d);
        }
        for (int i = 0; i < SEARCH + CORR; i++) cv[i] = argprod(s, Tu - SEARCH / 2 + i, Tu - SEARCH / 2 + i + 1);
        float MMax = 0; int index = 100;
        for (int i = 0; i < SEARCH; i++) {
            float sum = 0;
            for (int j = 0; j < CORR; j++) {
                sum += (float)iabs_f(refArg[j] * cv[i + j]);       /* `abs` is int abs(int) here too, see above */
                if (sum > MMax) { MMax = sum; index = i; }
            }
        }
        ret = (int16_t)(Tu - SEARCH / 2 + index - Tu);
    }
    free(s);
    return ret;
}

/* ============================================================================================
 * OFDM demod — OfdmDecoder::processPRS / decodeDataSymbol, ofdm-decoder.cpp:144-230
 * ========================================================================================== */
static void demap_symbol(const cf* X, cf* ref, int8_t* soft, float* r1s)
{
    for (int i = 0; i < ORC_K; i++) {
        int idx = g_perm[i];
        if (idx < 0) idx += ORC_TU;
        float a = X[idx].r, b = X[idx].i, c = ref[idx].r, d = -ref[idx].i;
        float re = a * c - b * d, im = a * d + b * c;   /* X * conj(ref) */
        ref[idx] = X[idx];
        float ab1 = 127.0f / (fabsf(re) + fabsf(im));
        soft[i] = (int8_t)(-re * ab1);           /* float -> int8: truncation toward zero */
        soft[ORC_K + i] = (int8_t)(-im * ab1);
        if (r1s) { r1s[2 * i] = re; r1s[2 * i + 1] = im; }
    }
}

int orc_snr(const float* spec);
void orc_ofdm_demod_frame2(const float* prs, const float* syms, int8_t* soft, float* r1s, int* snr);
void orc_ofdm_demod_frame(const float* prs, const float* syms, int8_t* soft, float* r1s) { orc_ofdm_demod_frame2(prs, syms, soft, r1s, NULL); }

/* also returns OfdmDecoder::get_snr(fft_buffer, 1) of the phase reference symbol's spectrum (ofdm-decoder.cpp:144-160) */
void orc_ofdm_demod_frame2(const float* prs, const float* syms, int8_t* soft, float* r1s, int* snr)
{
    ensure_tables();
    cf ref[ORC_TU], X[ORC_TU];
    orc_fft(ORC_TU, prs, (float*)ref, 0);
    if (snr) *snr = orc_snr((const float*)ref);
    for (int l = 1; l < ORC_L; l++) {
        orc_fft(ORC_TU, syms + 2 * ((size_t)(l - 1) * ORC_TS + ORC_TG), (float*)X, 0);
        demap_symbol(X, ref, soft + (size_t)(l - 1) * 2 * ORC_K, r1s ? r1s + (size_t)(l - 1) * 2 * ORC_K : NULL);
    }
}

/* OfdmDecoder::get_snr method 1 (ofdm-decoder.cpp:240-265); get_db_over_256 MathHelper.h:43-46.
 * Returns the int16 the reference returns (float dB difference truncated). */
int orc_snr(const float* spec)
{
    const cf* v = (const cf*)spec;
    const int Tu = ORC_TU, K = ORC_K;
    int low = Tu / 2 - K / 2, high = low + K;
    float noise = 0, signal = 0;
    for (int i = 70; i < low - 20; i++) noise += hypotf(v[(Tu / 2 + i) % Tu].r, v[(Tu / 2 + i) % Tu].i);
    for (int i = high + 20; i < high + 120; i++) noise += hypotf(v[(Tu / 2 + i) % Tu].r, v[(Tu / 2 + i) % Tu].i);
    noise /= (low - 90 + 100);
    for (int i = Tu / 2 - K / 4; i < Tu / 2 + K / 4; i++) signal += hypotf(v[(Tu / 2 + i) % Tu].r, v[(Tu / 2 + i) % Tu].i);
    float dbs = 20 * log10f((signal / (K / 2) + 1.0f) / 256.0f);
    float dbn = 20 * log10f((noise + 1.0f) / 256.0f);
    return (int16_t)(dbs - dbn);
}

/* ============================================================================================
 * Viterbi — backend/viterbi.cpp.  K=7, polys 0155 0117 0123 0155 (:35-36), soft symbol = clamp(s+127,0,255)
 * (:232-237), branch table Branchtab[k*32+s] = parity(2s & poly_k) ? 255 : 0 (:165-171), butterfly (:248-279),
 * start metrics 63 / 0 (:342-354), renormalisation (:104-120), traceback from state 0 (:313-339).
 * ========================================================================================== */
static const int POLYS[4] = {0155, 0117, 0123, 0155};
static int parity32(unsigned x) { x ^= x >> 16; x ^= x >> 8; x ^= x >> 4; x ^= x >> 2; x ^= x >> 1; return x & 1; }

void orc_conv_encode(const uint8_t* bits, int nbits, uint8_t* out)
{
    unsigned sr = 0;
    for (int i = 0; i < nbits + 6; i++) {
        unsigned b = i < nbits ? (bits[i] & 1) : 0;
        sr = ((sr << 1) | b) & 0x7F;
        for (int k = 0; k < 4; k++) *out++ = (uint8_t)parity32(sr & POLYS[k]);
    }
}

void orc_viterbi(int nbits, const int8_t* in, uint8_t* out)
{
    const int steps = nbits + 6;
    uint16_t btab[4][32];
    for (int s = 0; s < 32; s++)
        for (int k = 0; k < 4; k++) btab[k][s] = parity32((2 * s) & POLYS[k]) ? 255 : 0;
    uint64_t* dec = (uint64_t*)calloc(steps, sizeof(uint64_t));
    uint16_t ma[64], mb[64], *old = ma, *nw = mb;
    for (int i = 0; i < 64; i++) old[i] = 63;
    old[0] = 0;
    for (int t = 0; t < steps; t++) {
        uint16_t sym[4];
        for (int k = 0; k < 4; k++) {
            int v = (int)in[4 * t + k] + 127;
            if (v < 0) v = 0;
            if (v > 255) v = 255;
            sym[k] = (uint16_t)v;
        }
        uint64_t d = 0;
        for (int i = 0; i < 32; i++) {
            uint16_t metric = 0;
            for (int k = 0; k < 4; k++) metric += btab[k][i] ^ sym[k];
            const uint16_t mx = 1020;
            uint16_t m0 = old[i] + metric, m1 = old[i + 32] + (mx - metric);
            uint16_t m2 = old[i] + (mx - metric), m3 = old[i + 32] + metric;
            int d0 = ((int32_t)(m0 - m1)) > 0, d1 = ((int32_t)(m2 - m3)) > 0;
            nw[2 * i] = d0 ? m1 : m0;
            nw[2 * i + 1] = d1 ? m3 : m2;
            d |= ((uint64_t)(d0 | (d1 << 1))) << (2 * i);
        }
        dec[t] = d;
        if (nw[0] > 137) {
            uint16_t mn = nw[0];
            for (int i = 0; i < 64; i++) if (nw[i] < mn) mn = nw[i];
            for (int i = 0; i < 64; i++) nw[i] -= mn;
        }
        uint16_t* tmp = old; old = nw; nw = tmp;
    }
    /* traceback: state kept left-aligned in a byte (ADDSHIFT = 2), viterbi.cpp:313-339 */
    unsigned end = 0;
    for (int t = nbits - 1; t >= 0; t--) {
        unsigned st = end >> 2;
        unsigned k = (unsigned)(dec[t + 6] >> st) & 1;
        end = (end >> 1) | (k << 7);
        out[t] = (uint8_t)k;
    }
    free(dec);
}

/* ============================================================================================
 * FIC — fic-handler.cpp:111-230
 * ========================================================================================== */
/* MathHelper.h:53-80: CRC-CCITT over one-bit-per-byte data, register preset to ones, last 16 bits inverted */
int orc_check_crc_bits(const uint8_t* in, int n)
{
    unsigned reg = 0xFFFF;
    for (int i = 0; i < n; i++) {
        unsigned d = in[i] & 1;
        if (i >= n - 16) d ^= 1;
        unsigned fb = ((reg >> 15) & 1) ^ d;
        reg = (reg << 1) & 0xFFFF;
        if (fb) reg ^= 0x1021;
    }
    return reg == 0;
}

static int8_t g_pc[24 * 32];
static uint8_t g_prbs768[768];
static int g_fic_ready = 0;

void orc_fic_decode(const int8_t* soft, uint8_t* fib_bits, uint8_t* crc_ok)
{
    if (!g_fic_ready) { orc_pcodes(g_pc); orc_prbs(g_prbs768, 768); g_fic_ready = 1; }
    const int8_t* PI16 = g_pc + 32 * 15; const int8_t* PI15 = g_pc + 32 * 14;
    for (int blk = 0; blk < 4; blk++) {
        const int8_t* in = soft + 2304 * blk;   /* 9216 softbits cut into 4 x 2304 across symbol boundaries (:111-127) */
        int8_t mother[3072 + 24];
        memset(mother, 0, sizeof mother);
        int ic = 0, pos = 0;
        for (int i = 0; i < 21 * 128; i++, pos++) if (PI16[i & 31]) mother[pos] = in[ic++];
        for (int i = 0; i < 3 * 128; i++, pos++) if (PI15[i & 31]) mother[pos] = in[ic++];
        for (int i = 0; i < 24; i++, pos++) if (PI_TAIL[i]) mother[pos] = in[ic++];
        uint8_t bits[768];
        orc_viterbi(768, mother, bits);
        for (int i = 0; i < 768; i++) bits[i] ^= g_prbs768[i];
        for (int f = 0; f < 3; f++) {
            memcpy(fib_bits + 256 * (3 * blk + f), bits + 256 * f, 256);
            crc_ok[3 * blk + f] = (uint8_t)orc_check_crc_bits(bits + 256 * f, 256);
        }
    }
}

/* ============================================================================================
 * MSC protection profiles
 * ========================================================================================== */
int orc_prot_eep(int b, int profile_a, int level, orc_prot_t* p)
{
    memset(p, 0, sizeof *p);
    p->bitrate = b; p->nblk = 2;
    if (profile_a) {   /* eep-protection.cpp:37-78 */
        switch (level) {
            case 1: p->L[0] = 6 * b / 8 - 3; p->L[1] = 3; p->PI[0] = 24; p->PI[1] = 23; break;
            case 2:
                if (b == 8) { p->L[0] = 5; p->L[1] = 1; p->PI[0] = 13; p->PI[1] = 12; }
                else { p->L[0] = 2 * b / 8 - 3; p->L[1] = 4 * b / 8 + 3; p->PI[0] = 14; p->PI[1] = 13; }
                break;
            case 3: p->L[0] = 6 * b / 8 - 3; p->L[1] = 3; p->PI[0] = 8; p->PI[1] = 7; break;
            case 4: p->L[0] = 4 * b / 8 - 3; p->L[1] = 2 * b / 8 + 3; p->PI[0] = 3; p->PI[1] = 2; break;
            default: return -1;
        }
    } else {           /* eep-protection.cpp:80-112 */
        p->L[0] = 24 * b / 32 - 3; p->L[1] = 3;
        switch (level) {
            case 1: p->PI[0] = 10; p->PI[1] = 9; break;
            case 2: p->PI[0] = 6; p->PI[1] = 5; break;
            case 3: p->PI[0] = 4; p->PI[1] = 3; break;
            case 4: p->PI[0] = 2; p->PI[1] = 1; break;
            default: return -1;
        }
    }
    int8_t pc[24 * 32]; orc_pcodes(pc);
    int n = 12;   /* tail: 12 of 24 kept */
    for (int k = 0; k < p->nblk; k++) { int ones = 0; for (int j = 0; j < 32; j++) ones += pc[32 * (p->PI[k] - 1) + j]; n += 4 * ones * p->L[k]; }
    p->in_bits = n;
    return 0;
}

/* uep-protection.cpp:38-118 — the reference's table (bitrate, level, L1..L4, PI1..PI4).  These are the values
 * the reference uses (a few rows differ from ETSI Table 15; parity is with the reference).  PI4 = 0: unused. */
static const int16_t UEP_ROWS[][10] = {
    {32,5,3,4,17,0,5,3,2,0},{32,4,3,3,18,0,11,6,5,0},{32,3,3,4,14,3,15,9,6,8},{32,2,3,4,14,3,22,13,8,13},{32,1,3,5,13,3,24,17,12,17},
    {48,5,4,3,26,3,5,4,2,3},{48,4,3,4,26,3,9,6,4,6},{48,3,3,4,26,3,15,10,6,9},{48,2,3,4,26,3,24,14,8,15},{48,1,3,5,25,3,24,18,13,18},
    {56,5,6,10,23,3,5,4,2,3},{56,4,6,10,23,3,9,6,4,5},{56,3,6,12,21,3,16,7,6,9},{56,2,6,10,23,3,23,13,8,13},
    {64,5,6,9,31,2,5,3,2,3},{64,4,6,9,33,0,11,6,5,0},{64,3,6,12,27,3,16,8,6,9},{64,2,6,10,29,3,23,13,8,13},{64,1,6,11,28,3,24,18,12,18},
    {80,5,6,10,41,3,6,3,2,3},{80,4,6,10,41,3,11,6,5,6},{80,3,6,11,40,3,16,8,6,7},{80,2,6,10,41,3,23,13,8,13},{80,1,6,10,41,3,24,7,12,18},
    {96,5,7,9,53,3,5,4,2,4},{96,4,7,10,52,3,9,6,4,6},{96,3,6,12,51,3,16,9,6,10},{96,2,6,10,53,3,22,12,9,12},{96,1,6,13,50,3,24,18,13,19},
    {112,5,14,17,50,3,5,4,2,5},{112,4,11,21,49,3,9,6,4,8},{112,3,11,23,47,3,16,8,6,9},{112,2,11,21,49,3,23,12,9,14},
    {128,5,12,19,62,3,5,3,2,4},{128,4,11,21,61,3,11,6,5,7},{128,3,11,22,60,3,16,9,6,10},{128,2,11,21,61,3,22,12,9,14},{128,1,11,20,62,3,24,17,13,19},
    {160,5,11,19,87,3,5,4,2,4},{160,4,11,23,83,3,11,6,5,9},{160,3,11,24,82,3,16,8,6,11},{160,2,11,21,85,3,22,11,9,13},{160,1,11,22,84,3,24,18,12,19},
    {192,5,11,20,110,3,6,4,2,5},{192,4,11,22,108,3,10,6,4,9},{192,3,11,24,106,3,16,10,6,11},{192,2,11,20,110,3,22,13,9,13},{192,1,11,21,109,3,24,20,13,24},
    {224,5,12,22,131,3,8,6,2,6},{224,4,12,26,127,3,12,8,4,11},{224,3,11,20,134,3,16,10,7,9},{224,2,11,22,132,3,24,16,10,15},{224,1,11,24,130,3,24,20,12,20},
    {256,5,11,24,154,3,6,5,2,5},{256,4,11,24,154,3,12,9,5,10},{256,3,11,27,151,3,16,10,7,10},{256,2,11,22,156,3,24,14,10,13},{256,1,11,26,152,3,24,19,14,18},
    {320,5,11,26,200,3,8,5,2,6},{320,4,11,25,201,3,13,9,5,10},{320,2,11,26,200,3,24,17,9,17},
    {384,5,11,27,247,3,8,6,2,7},{384,3,11,24,250,3,16,9,7,10},{384,1,12,28,245,3,24,20,14,23},
};

int orc_prot_uep(int b, int level, orc_prot_t* p)
{
    memset(p, 0, sizeof *p);
    const int nrows = (int)(sizeof UEP_ROWS / sizeof UEP_ROWS[0]);
    int idx = -1;
    for (int i = 0; i < nrows; i++) if (UEP_ROWS[i][0] == b && UEP_ROWS[i][1] == level) { idx = i; break; }
    if (idx < 0) idx = 1;   /* uep-protection.cpp:152-155: unknown combination falls back to row 1 */
    p->bitrate = b; p->nblk = 4;
    for (int k = 0; k < 4; k++) { p->L[k] = UEP_ROWS[idx][2 + k]; p->PI[k] = UEP_ROWS[idx][6 + k]; }
    int8_t pc[24 * 32]; orc_pcodes(pc);
    int n = 12;
    for (int k = 0; k < 4; k++) { if (!p->L[k]) continue; if (!p->PI[k]) return -1; int ones = 0; for (int j = 0; j < 32; j++) ones += pc[32 * (p->PI[k] - 1) + j]; n += 4 * ones * p->L[k]; }
    p->in_bits = n;
    return 0;
}

int orc_eep_bitrate(int len, int profile_a, int level)   /* dab-constants.cpp:404-440 */
{
    static const int da[5] = {0, 12, 8, 6, 4}, db[5] = {0, 27, 21, 18, 15};
    if (level < 1 || level > 4) return -1;
    return profile_a ? len / da[level] * 8 : len / db[level] * 32;
}

void orc_msc_deconvolve(const orc_prot_t* p, const int8_t* in, uint8_t* outbits)
{
    int8_t pc[24 * 32]; orc_pcodes(pc);
    const int nb = 24 * p->bitrate;
    int8_t* mother = (int8_t*)calloc((size_t)nb * 4 + 24, 1);
    int ic = 0, pos = 0;
    for (int k = 0; k < p->nblk; k++) {
        const int8_t* pi = pc + 32 * (p->PI[k] - 1);
        for (int i = 0; i < p->L[k] * 128; i++, pos++) if (pi[i & 31]) mother[pos] = in[ic++];
    }
    for (int i = 0; i < 24; i++, pos++) if (PI_TAIL[i]) mother[pos] = in[ic++];
    orc_viterbi(nb, mother, outbits);
    free(mother);
}

void orc_dedisperse(uint8_t* bits, int n)
{
    uint8_t* pr = (uint8_t*)malloc(n);
    orc_prbs(pr, n);
    for (int i = 0; i < n; i++) bits[i] ^= pr[i];
    free(pr);
}

void orc_pack_bits(const uint8_t* bits, int nbytes, uint8_t* out)
{
    for (int i = 0; i < nbytes; i++) {
        unsigned b = 0;
        for (int j = 0; j < 8; j++) b = (b << 1) | (bits[8 * i + j] & 1);
        out[i] = (uint8_t)b;
    }
}

/* ---- time de-interleaver: dab-audio.cpp:113-149 ---- */
static const int DEINT_MAP[16] = {0, 8, 4, 12, 2, 10, 6, 14, 1, 9, 5, 13, 3, 11, 7, 15};

orc_deint_t* orc_deint_new(int fragment)
{
    orc_deint_t* d = (orc_deint_t*)calloc(1, sizeof *d);
    d->fragment = fragment;
    d->hist = (int8_t*)calloc((size_t)16 * fragment, 1);
    return d;
}
void orc_deint_free(orc_deint_t* d) { if (d) { free(d->hist); free(d); } }

int orc_deint_push(orc_deint_t* d, const int8_t* in, int8_t* out)
{
    const int F = d->fragment;
    for (int i = 0; i < F; i++) {
        out[i] = d->hist[(size_t)((d->index + DEINT_MAP[i & 15]) & 15) * F + i];
        d->hist[(size_t)d->index * F + i] = in[i];
    }
    d->index = (d->index + 1) & 15;
    if (d->count <= 15) { d->count++; return 0; }
    return 1;
}

/* ============================================================================================
 * Reed-Solomon (120,110) over GF(2^8), field poly 0x11D, fcr 0, prim 1, 10 roots, shortened by 135
 * (dabplus_decoder.cpp:316-321).  Decoder follows libs/fec/decode_rs.h:71-298 (syndromes, Berlekamp-Massey,
 * Chien search, Forney) so that behaviour on uncorrectable words matches too.  Polynomial-form arithmetic
 * with explicit gf_mul instead of the library's index-form bookkeeping; the algebra is the same.
 * ========================================================================================== */
static uint8_t gf_exp[512], gf_log[256];
static int gf_ready = 0;
static void gf_init(void)
{
    if (gf_ready) return;
    unsigned x = 1;
    for (int i = 0; i < 255; i++) { gf_exp[i] = (uint8_t)x; gf_log[x] = (uint8_t)i; x <<= 1; if (x & 0x100) x ^= 0x11D; }
    for (int i = 255; i < 512; i++) gf_exp[i] = gf_exp[i - 255];
    gf_ready = 1;
}
static inline uint8_t gf_mul(uint8_t a, uint8_t b) { return (a && b) ? gf_exp[gf_log[a] + gf_log[b]] : 0; }
static inline uint8_t gf_div(uint8_t a, uint8_t b) { return a ? gf_exp[gf_log[a] + 255 - gf_log[b]] : 0; }
static inline uint8_t gf_pow_alpha(int e) { e %= 255; if (e < 0) e += 255; return gf_exp[e]; }

enum { RS_NROOTS = 10, RS_NN = 255, RS_PAD = 135, RS_LEN = 120 };

/* encode_rs.h:33-58: systematic LFSR division by g(x) = prod_{i=0}^{9} (x - alpha^i) */
void orc_rs_encode(const uint8_t data[110], uint8_t parity[10])
{
    gf_init();
    uint8_t g[RS_NROOTS + 1] = {1};
    for (int i = 0; i < RS_NROOTS; i++) {
        uint8_t root = gf_pow_alpha(i);
        g[i + 1] = 1;
        for (int j = i; j > 0; j--) g[j] = g[j - 1] ^ gf_mul(g[j], root);
        g[0] = gf_mul(g[0], root);
    }
    memset(parity, 0, RS_NROOTS);
    for (int i = 0; i < RS_LEN - RS_NROOTS; i++) {
        uint8_t fb = data[i] ^ parity[0];
        for (int j = 0; j < RS_NROOTS - 1; j++) parity[j] = parity[j + 1] ^ gf_mul(fb, g[RS_NROOTS - 1 - j]);
        parity[RS_NROOTS - 1] = gf_mul(fb, g[0]);
    }
}

int orc_rs_decode_codeword(uint8_t data[120], int corr_pos[10])
{
    gf_init();
    uint8_t s[RS_NROOTS];
    /* syndromes S_i = r(alpha^i), Horner over the 120 received symbols (decode_rs.h:86-98) */
    int any = 0;
    for (int i = 0; i < RS_NROOTS; i++) {
        uint8_t acc = data[0], a = gf_pow_alpha(i);
        for (int j = 1; j < RS_LEN; j++) acc = data[j] ^ gf_mul(acc, a);
        s[i] = acc; any |= acc;
    }
    if (!any) return 0;
    /* Berlekamp-Massey (decode_rs.h:152-193), no erasures */
    uint8_t lambda[RS_NROOTS + 1] = {1}, b[RS_NROOTS + 1] = {1}, t[RS_NROOTS + 1];
    int el = 0;
    for (int r = 1; r <= RS_NROOTS; r++) {
        uint8_t discr = 0;
        for (int i = 0; i < r; i++) discr ^= gf_mul(lambda[i], s[r - i - 1]);
        if (discr == 0) {
            memmove(b + 1, b, RS_NROOTS); b[0] = 0;
        } else {
            t[0] = lambda[0];
            for (int i = 0; i < RS_NROOTS; i++) t[i + 1] = lambda[i + 1] ^ gf_mul(discr, b[i]);
            if (2 * el <= r - 1) {
                el = r - el;
                for (int i = 0; i <= RS_NROOTS; i++) b[i] = gf_div(lambda[i], discr);
            } else {
                memmove(b + 1, b, RS_NROOTS); b[0] = 0;
            }
            memcpy(lambda, t, RS_NROOTS + 1);
        }
    }
    int deg_lambda = 0;
    for (int i = 0; i <= RS_NROOTS; i++) if (lambda[i]) deg_lambda = i;
    /* Chien search over all 255 locations (decode_rs.h:204-231): root index i = 1..255, location k = i-1 stepping
     * by iprim = 1: k = (i - 1); X^{-1} = alpha^i */
    int root[RS_NROOTS], loc[RS_NROOTS], count = 0;
    for (int i = 1, k = 0; i <= RS_NN; i++, k = (k + 1) % RS_NN) {
        uint8_t q = 1;
        for (int j = deg_lambda; j > 0; j--) q ^= gf_mul(lambda[j], gf_pow_alpha(j * i));
        if (q) continue;
        root[count] = i; loc[count] = k;
        if (++count == deg_lambda) break;
    }
    if (deg_lambda != count) return -1;
    /* omega(x) = s(x) lambda(x) mod x^NROOTS, degree deg_lambda-1 (decode_rs.h:243-256) */
    uint8_t omega[RS_NROOTS + 1];
    int deg_omega = deg_lambda - 1;
    for (int i = 0; i <= deg_omega; i++) {
        uint8_t tmp = 0;
        for (int j = i; j >= 0; j--) tmp ^= gf_mul(s[i - j], lambda[j]);
        omega[i] = tmp;
    }
    /* Forney (decode_rs.h:262-289): fcr = 0 -> num2 = X^{-(fcr-1)} = alpha^{-root}... computed as alpha^(root*(fcr-1)+NN) */
    for (int j = count - 1; j >= 0; j--) {
        uint8_t num1 = 0;
        for (int i = deg_omega; i >= 0; i--) num1 ^= gf_mul(omega[i], gf_pow_alpha(i * root[j]));
        uint8_t num2 = gf_pow_alpha(root[j] * (0 - 1) + RS_NN);
        uint8_t den = 0;
        int top = (deg_lambda < RS_NROOTS - 1 ? deg_lambda : RS_NROOTS - 1) & ~1;
        for (int i = top; i >= 0; i -= 2) den ^= gf_mul(lambda[i + 1], gf_pow_alpha(i * root[j]));
        if (num1 != 0 && loc[j] >= RS_PAD) data[loc[j] - RS_PAD] ^= gf_div(gf_mul(num1, num2), den);
    }
    if (corr_pos) for (int i = 0; i < count; i++) corr_pos[i] = loc[i];
    return count;
}

/* RSDecoder::DecodeSuperframe, dabplus_decoder.cpp:326-359 */
void orc_rs_decode_superframe(uint8_t* sf, int sf_len, int* corr, int* uncorr)
{
    const int S = sf_len / 120;
    int total = 0, unc = 0;
    for (int i = 0; i < S; i++) {
        uint8_t cw[120]; int pos[10];
        for (int p = 0; p < 120; p++) cw[p] = sf[p * S + i];
        int c = orc_rs_decode_codeword(cw, pos);
        if (c == -1) unc = 1; else total += c;
        for (int j = 0; j < c; j++) { int p = pos[j] - RS_PAD; if (p < 0) continue; sf[p * S + i] = cw[p]; }
    }
    *corr = total; *uncorr = unc;
}

/* CalcCRC, tools.cpp:35-73 / tools.h:70-89: MSB-first CRC-16 */
unsigned orc_crc16(const uint8_t* d, int n, unsigned poly, int init_invert, int final_invert)
{
    unsigned crc = init_invert ? 0xFFFF : 0;
    for (int i = 0; i < n; i++) {
        crc ^= (unsigned)d[i] << 8;
        for (int b = 0; b < 8; b++) crc = (crc & 0x8000) ? ((crc << 1) ^ poly) & 0xFFFF : (crc << 1) & 0xFFFF;
    }
    return final_invert ? (~crc) & 0xFFFF : crc;
}
unsigned orc_crc_fire(const uint8_t* d, int n) { return orc_crc16(d, n, 0x782F, 0, 0); }
unsigned orc_crc_ccitt(const uint8_t* d, int n) { return orc_crc16(d, n, 0x1021, 1, 1); }

/* ---- SuperframeFilter::Feed / CheckSync, dabplus_decoder.cpp:49-142,171-215 ---- */
orc_sff_t* orc_sff_new(void) { return (orc_sff_t*)calloc(1, sizeof(orc_sff_t)); }
void orc_sff_free(orc_sff_t* f) { if (f) { free(f->sf_raw); free(f->sf); free(f); } }

static int sff_check_sync(orc_sff_t* f)
{
    const uint8_t* sf = f->sf;
    if (sf[3] == 0 && sf[4] == 0) return 0;
    unsigned stored = (sf[0] << 8) | sf[1];
    if (stored != orc_crc_fire(sf + 2, 9)) return 0;
    int dac = sf[2] & 0x40, sbr = sf[2] & 0x20;
    f->num_aus = dac ? (sbr ? 3 : 6) : (sbr ? 2 : 4);
    f->au_start[0] = dac ? (sbr ? 6 : 11) : (sbr ? 5 : 8);
    f->au_start[f->num_aus] = f->sf_len / 120 * 110;
    f->au_start[1] = sf[3] << 4 | sf[4] >> 4;
    if (f->num_aus >= 3) f->au_start[2] = (sf[4] & 0x0F) << 8 | sf[5];
    if (f->num_aus >= 4) f->au_start[3] = sf[6] << 4 | sf[7] >> 4;
    if (f->num_aus == 6) { f->au_start[4] = (sf[7] & 0x0F) << 8 | sf[8]; f->au_start[5] = sf[9] << 4 | sf[10] >> 4; }
    for (int i = 0; i < f->num_aus; i++) if (f->au_start[i] >= f->au_start[i + 1]) return 0;
    return 1;
}

void orc_sff_feed(orc_sff_t* f, const uint8_t* frame, int len, orc_sff_result_t* res, uint8_t* sf_out)
{
    memset(res, 0, sizeof *res);
    if (f->frame_len) { if (f->frame_len != len) return; }
    else {
        if (len < 10 || (5 * len) % 120) return;
        f->frame_len = len; f->sf_len = 5 * len;
        f->sf_raw = (uint8_t*)calloc(f->sf_len, 1); f->sf = (uint8_t*)calloc(f->sf_len, 1);
    }
    if (f->frame_count == 5) memmove(f->sf_raw, f->sf_raw + len, (size_t)4 * len);
    else f->frame_count++;
    memcpy(f->sf_raw + (size_t)(f->frame_count - 1) * len, frame, len);
    if (f->frame_count < 5) return;
    memcpy(f->sf, f->sf_raw, f->sf_len);
    res->attempted = 1;
    orc_rs_decode_superframe(f->sf, f->sf_len, &res->corr, &res->uncorr);
    if (!sff_check_sync(f)) return;
    res->sync_ok = 1; res->num_aus = f->num_aus;
    for (int i = 0; i < f->num_aus; i++) {
        const uint8_t* au = f->sf + f->au_start[i];
        int alen = f->au_start[i + 1] - f->au_start[i];
        unsigned stored = au[alen - 2] << 8 | au[alen - 1];
        if (stored == orc_crc_ccitt(au, alen - 2)) res->au_crc_ok_mask |= 1 << i;
    }
    if (sf_out) memcpy(sf_out, f->sf, f->sf_len);
    f->frame_count = 0;
}

/* ============================================================================================
 * Closed-loop receiver — OFDMProcessor::run, ofdm-processor.cpp:235-501, with the decode chain inline.
 * The reference runs the decoder on a second thread; FicHandler::getFicDecodeRatioPercent() read at :397 races
 * with it.  Here frame n is fully decoded before frame n+1's PRS is examined.
 * ========================================================================================== */
struct orc_rx {
    orc_rx_cfg_t cfg;
    float* osc;            /* 2 048 000-entry oscillator, ofdm-processor.cpp:92-94 */
    int32_t coarse; int16_t fine; int32_t local_phase; float slevel;
    int fic_ratio;         /* saturating 0..10, fic-handler.cpp:222-228 */
    long nfib_total; long nframes;
    int msc_active;
    int8_t cif[864 * 64];
    orc_deint_t* deint; orc_sff_t* sff;
    int acquired;          /* 0 = must run the null search, 1 = tracking */
    int started;
};

orc_rx_t* orc_rx_new(const orc_rx_cfg_t* cfg)
{
    orc_rx_t* r = (orc_rx_t*)calloc(1, sizeof *r);
    r->cfg = *cfg;
    r->osc = (float*)malloc(sizeof(float) * 2 * ORC_INPUT_RATE);
    for (int i = 0; i < ORC_INPUT_RATE; i++) {
        r->osc[2 * i] = (float)cos(2.0 * M_PI * i / ORC_INPUT_RATE);
        r->osc[2 * i + 1] = (float)sin(2.0 * M_PI * i / ORC_INPUT_RATE);
    }
    if (cfg->subch_len_cu > 0) { r->deint = orc_deint_new(cfg->subch_len_cu * 64); r->sff = orc_sff_new(); }
    return r;
}
void orc_rx_free(orc_rx_t* r) { if (r) { free(r->osc); orc_deint_free(r->deint); orc_sff_free(r->sff); free(r); } }

typedef struct { const cf* iq; long n, pos; } src_t;

/* getSample / getSamples, ofdm-processor.cpp:145-224: NCO mix + sLevel IIR. returns 0 when input is exhausted */
static int rx_get(orc_rx_t* r, src_t* s, cf* out, int n, int32_t phase)
{
    if (s->pos + n > s->n) return 0;
    for (int i = 0; i < n; i++) {
        cf v = s->iq[s->pos + i];
        r->local_phase -= phase;
        r->local_phase = (r->local_phase + ORC_INPUT_RATE) % ORC_INPUT_RATE;
        cf o; o.r = r->osc[2 * r->local_phase]; o.i = r->osc[2 * r->local_phase + 1];
        cf m; m.r = v.r * o.r - v.i * o.i; m.i = v.r * o.i + v.i * o.r;
        out[i] = m;
        r->slevel = (float)(0.00001 * (double)(fabsf(m.r) + fabsf(m.i)) + (1 - 0.00001) * (double)r->slevel);
    }
    s->pos += n;
    return 1;
}

long orc_rx_run(orc_rx_t* r, const float* iq, long nsamples,
                uint8_t* fibs, long fib_cap, long* n_fibs,
                uint8_t* msc, long msc_cap, long* n_msc,
                int* rs_events, long rs_cap, long* n_rs,
                orc_frame_info_t* finfo, long finfo_cap,
                int8_t* soft_tap, long soft_cap_frames)
{
    ensure_tables();
    src_t src = { (const cf*)iq, nsamples, 0 };
    long nf = 0, nfib = 0, nmsc = 0, nrs = 0;
    cf* prsbuf = (cf*)malloc(sizeof(cf) * ORC_TU);
    cf* syms = (cf*)malloc(sizeof(cf) * 75 * ORC_TS);
    cf* nullsym = (cf*)malloc(sizeof(cf) * ORC_TNULL);
    int8_t* soft = (int8_t*)malloc(75 * 3072);
    float* env = (float*)calloc(32768, sizeof(float));
    const int mask = 32767;
    cf one;
    const int frag = r->cfg.subch_len_cu * 64;
    int8_t* dtmp = frag ? (int8_t*)malloc(frag) : NULL;
    uint8_t* obits = frag ? (uint8_t*)malloc(24 * r->cfg.prot.bitrate) : NULL;
    const int flen = 3 * r->cfg.prot.bitrate;
    uint8_t* fr = frag ? (uint8_t*)malloc(flen) : NULL;

    if (!r->started) {
        r->started = 1;
        r->slevel = 0;
        for (int i = 0; i < ORC_TF / 2; i++) if (!rx_get(r, &src, &one, 1, 0)) goto done;
    }
    for (;;) {
        if (!r->acquired) {
        not_synced:;
            int idx = 0, counter;
            float cur = 0;
            for (int i = 0; i < 50; i++) {
                if (!rx_get(r, &src, &one, 1, 0)) goto done;
                env[idx] = fabsf(one.r) + fabsf(one.i); cur += env[idx]; idx++;
            }
            counter = 0;
            while ((double)(cur / 50) > 0.50 * (double)r->slevel) {
                if (!rx_get(r, &src, &one, 1, r->coarse + r->fine)) goto done;
                env[idx] = fabsf(one.r) + fabsf(one.i);
                cur += env[idx] - env[(idx - 50) & mask];
                idx = (idx + 1) & mask;
                if (++counter > ORC_TF) goto not_synced;
            }
            counter = 0;
            while ((double)(cur / 50) < 0.75 * (double)r->slevel) {
                if (!rx_get(r, &src, &one, 1, r->coarse + r->fine)) goto done;
                env[idx] = fabsf(one.r) + fabsf(one.i);
                cur += env[idx] - env[(idx - 50) & mask];
                idx = (idx + 1) & mask;
                if (++counter > ORC_TNULL + 50) goto not_synced;
            }
            r->acquired = 1;
        }
        /* SyncOnPhase */
        long fpos = src.pos;
        if (!rx_get(r, &src, prsbuf, ORC_TU, r->coarse + r->fine)) goto done;
        int start = orc_find_index_m((const float*)prsbuf, NULL, r->cfg.fft_placement);
        if (start < 0) { r->acquired = 0; continue; }
        memmove(prsbuf, prsbuf + start, sizeof(cf) * (ORC_TU - start));
        if (!rx_get(r, &src, prsbuf + (ORC_TU - start), start, r->coarse + r->fine)) goto done;
        if (!r->cfg.disable_coarse && r->fic_ratio * 10 < 50) {
            int corr = orc_coarse((const float*)prsbuf, r->cfg.freqsync_method);
            if (corr != 100) {
                r->coarse += corr * ORC_CARRIER_DIFF;
                if (abs(r->coarse) > 35000) r->coarse = 0;
            }
        }
        cf fc = {0, 0};
        for (int sym = 1; sym < ORC_L; sym++) {
            cf* b = syms + (size_t)(sym - 1) * ORC_TS;
            if (!rx_get(r, &src, b, ORC_TS, r->coarse + r->fine)) goto done;
            for (int i = ORC_TU; i < ORC_TS; i++) {
                float a = b[i].r, bb = b[i].i, c = b[i - ORC_TU].r, d = -b[i - ORC_TU].i;
                fc.r += a * c - bb * d;
                fc.i += a * d + bb * c;
            }
        }
        /* ---- decoder thread work for this frame (ofdm-decoder.cpp:93-130) ---- */
        int snr_raw = 0;
        orc_ofdm_demod_frame2((const float*)prsbuf, (const float*)syms, soft, NULL, &snr_raw);
        if (soft_tap && nf < soft_cap_frames) memcpy(soft_tap + (size_t)nf * 75 * 3072, soft, 75 * 3072);
        {
            uint8_t fb[12 * 256], ok[12];
            orc_fic_decode(soft, fb, ok);
            for (int f = 0; f < 12; f++) {
                if (nfib < fib_cap) { fibs[33 * nfib] = ok[f]; orc_pack_bits(fb + 256 * f, 32, fibs + 33 * nfib + 1); }
                nfib++; r->nfib_total++;
                if (ok[f]) { if (r->fic_ratio < 10) r->fic_ratio++; } else if (r->fic_ratio > 0) r->fic_ratio--;
            }
        }
        if (frag && !r->msc_active && r->nframes >= r->cfg.select_after_frames) r->msc_active = 1;
        if (frag && r->msc_active) {
            for (int c = 0; c < 4; c++) {
                memcpy(r->cif, soft + (size_t)(3 + 18 * c) * 3072, 18 * 3072);   /* symbols 4+18c .. 21+18c, msc-handler.cpp:136-139 */
                if (orc_deint_push(r->deint, r->cif + r->cfg.subch_start_cu * 64, dtmp)) {
                    orc_msc_deconvolve(&r->cfg.prot, dtmp, obits);
                    orc_dedisperse(obits, 24 * r->cfg.prot.bitrate);
                    orc_pack_bits(obits, flen, fr);
                    if (nmsc + flen <= msc_cap) memcpy(msc + nmsc, fr, flen);
                    nmsc += flen;
                    if (r->cfg.dabplus) {
                        orc_sff_result_t res;
                        orc_sff_feed(r->sff, fr, flen, &res, NULL);
                        if (res.attempted) { if (nrs < rs_cap) { rs_events[2 * nrs] = res.uncorr; rs_events[2 * nrs + 1] = res.corr; } nrs++; }
                    }
                }
            }
        }
        /* ---- back on the OFDM thread ---- */
        r->fine = (int16_t)((double)r->fine + 0.1 * (double)atan2f(fc.i, fc.r) / M_PI * (ORC_CARRIER_DIFF / 2));
        if (finfo && nf < finfo_cap) { finfo[nf].start_index = start; finfo[nf].fine = r->fine; finfo[nf].coarse = r->coarse; finfo[nf].snr_raw = snr_raw; finfo[nf].frame_pos = fpos; }
        nf++; r->nframes++;
        if (!rx_get(r, &src, nullsym, ORC_TNULL, r->coarse + r->fine)) goto done;
        if (r->fine > ORC_CARRIER_DIFF / 2) { r->coarse += ORC_CARRIER_DIFF; r->fine -= ORC_CARRIER_DIFF; }
        else if (r->fine < -ORC_CARRIER_DIFF / 2) { r->coarse -= ORC_CARRIER_DIFF; r->fine += ORC_CARRIER_DIFF; }
    }
done:
    free(prsbuf); free(syms); free(nullsym); free(soft); free(env); free(dtmp); free(obits); free(fr);
    if (n_fibs) *n_fibs = nfib;
    if (n_msc) *n_msc = nmsc;
    if (n_rs) *n_rs = nrs;
    return nf;
}
