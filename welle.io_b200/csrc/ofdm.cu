// ofdm.cu — OFDM front-end kernels for sm_90a:
//   ofdm_demod_kernel   NCO mix (optional) + 2048-point FFT per symbol + differential-QPSK demap with the frequency
//                       de-interleaver scatter + guard-interval correlation (fine AFC) + PRS SNR estimate.
//                       Replaces OFDMProcessor::getSamples mix loop (ofdm-processor.cpp:211-214), the CP correlation
//                       (:436-442), OfdmDecoder::processPRS/decodeDataSymbol (ofdm-decoder.cpp:144-230), get_snr (:240-265)
//   find_index_kernel   PhaseReference::findIndex, ThresholdBeforePeak (phasereference.cpp:73-97,212-253)
//
// HBM-bound by design: every input sample is read exactly once straight into registers with coalesced float2 loads
// (the digit-reversed first pass makes lane-consecutive addresses), each softbit is written exactly once through a
// 3 KB shared staging buffer with 16-byte stores.  Algorithmic bytes per frame: 76*2048*8 (+75*504*8 guard) in,
// 75*3072 out (see DESIGN.md).  One 128-thread CTA walks `sym_per_cta` consecutive symbols of one frame and keeps
// the previous symbol's spectrum in registers (differential demodulation needs only that).
#include "common.cuh"
#include "osc_factors.h"
#include <cstdlib>

namespace dabb {

namespace {

struct __align__(16) OfdmSmem {
    float2 xbuf[TU];                 // 16 KB swizzled exchange buffer
    float2 tw[TwLayout::C4];         // 1 KB: twiddles of passes A and B (pass C reads its 15 KB through L1 with __ldg)
};

// pass C with both stages' twiddles read through the read-only path (lane-consecutive, L1 resident across CTAs)
template <bool EXACT, bool INV>
__device__ __forceinline__ void passC_ldg(float2 v[16], int t, const float2* __restrict__ tw_c5)
{
    const float2* tw_c4 = tw_c5 - 384;
    const float2 w1 = __ldg(tw_c4 + t), w2 = __ldg(tw_c4 + 128 + t), w3 = __ldg(tw_c4 + 256 + t);
#pragma unroll
    for (int b = 0; b < 4; b++) bfly4<EXACT, INV>(v[4 * b], v[4 * b + 1], v[4 * b + 2], v[4 * b + 3], w1, w2, w3);
#pragma unroll
    for (int a = 0; a < 4; a++) {
        const int k5 = t + 128 * a;
        bfly4<EXACT, INV>(v[a], v[a + 4], v[a + 8], v[a + 12], __ldg(tw_c5 + k5), __ldg(tw_c5 + 512 + k5), __ldg(tw_c5 + 1024 + k5));
    }
}

// ---- NCO (ofdm-processor.cpp:211-214): sample idx of the frame is multiplied by osc[(lp0 - idx*ph) mod 2 048 000].
// Per symbol one 64-bit modulo gives the phase of the thread's first sample; the other samples follow by modular
// subtraction of per-CTA constants (stride 128 and 256 samples).  `mix` is CTA-uniform; lp0 == ph == 0 means the
// oscillator is (1, 0) for every sample and the multiplication is skipped.
struct Nco {
    int32_t lp0, ph, d128, d256, u2048;   // d = (stride * ph) mod RATE; u2048 = (-2048 * ph) mod RATE
    bool mix;
};
__device__ __forceinline__ int32_t mod_rate64(int64_t v) { v %= INPUT_RATE; if (v < 0) v += INPUT_RATE; return (int32_t)v; }
__device__ __forceinline__ Nco make_nco(int32_t lp0, int32_t ph)
{
    Nco n; n.lp0 = lp0; n.ph = ph; n.mix = (lp0 != 0) || (ph != 0);
    n.d128 = n.mix ? mod_rate64(128 * (int64_t)ph) : 0; n.d256 = n.mix ? mod_rate64(256 * (int64_t)ph) : 0; n.u2048 = n.mix ? mod_rate64(-2048 * (int64_t)ph) : 0;
    return n;
}
__device__ __forceinline__ int32_t sub_mod(int32_t a, int32_t d) { a -= d; return a < 0 ? a + INPUT_RATE : a; }
// oscillator sample m without the table (osc_factors.h): one 16-byte load that is the same for (nearly) all lanes of a warp
// replaces a scattered 8-byte gather per lane.  Every operation is explicitly rounded so that every kernel - and the start-up
// verification against the reference's table - executes the identical arithmetic.
struct OscDevOps {
    static __device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
    static __device__ __forceinline__ double fma(double a, double b, double c) { return __fma_rn(a, b, c); }
    static __device__ __forceinline__ float to_float(double a) { return __double2float_rn(a); }
};
__device__ __forceinline__ float2 osc_onthefly(const DevTables& tb, int32_t m)
{
    const double2 h = __ldg(tb.osc_hi + (m >> OSC_LO_BITS));
    const double r = __dsub_rn(__hiloint2double(0x43300000, m & ((1 << OSC_LO_BITS) - 1)), 4503599627370496.0);     // exact int -> double without a conversion instruction
    float2 o;
    osc_formula<OscDevOps>(h.x, h.y, r, tb.osc_theta, o.x, o.y);
    return o;
}
__device__ __forceinline__ float2 osc_value(const DevTables& tb, int32_t m)
{
    return tb.osc_mode ? osc_onthefly(tb, m) : __ldg(tb.osc + m);          // kernel-uniform
}
__device__ __forceinline__ float2 mix_sample(float2 v, const DevTables& tb, int32_t lp)
{
    return cmul_<true>(v, osc_value(tb, lp));   // std::complex product, separately rounded
}

// ---- tolerance-mode oscillator (DABB_NCO_FAST): fp32 sincospi of the exact integer phase.  osc(m) = e^{j 2 pi m / 2 048 000}
// = (cospi, sinpi)(m / 1 024 000); m < 2^21 is exact in fp32, the quotient is rounded once (<= 6e-8 relative -> <= 4e-7 rad), sincospif
// adds ~1e-7: every oscillator sample is within ~1e-6 of the reference's table value (north_star: soft intermediates within 1e-4).
__device__ __forceinline__ float2 osc_fast(int32_t m)
{
    float s, c;
    sincospif(__fmul_rn((float)m, 1.0f / 1024000.0f), &s, &c);
    return make_float2(c, s);
}
__device__ __forceinline__ float2 cmul_fast(float2 a, float2 b) { return make_float2(fmaf(a.x, b.x, -(a.y * b.y)), fmaf(a.x, b.y, a.y * b.x)); }

__device__ __forceinline__ float block_sum(float v, float* red, int t)
{
    // fixed-order reduction: lane tree, then the four warp results added in warp order
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((t & 31) == 0) red[t >> 5] = v;
    __syncthreads();
    return red[0] + red[1] + red[2] + red[3];
}

// the CTA's sum of the per-thread level sums (DABB_DEMAP_WEIGHTED) in the fixed order of block_sum
__device__ __forceinline__ LevelSum block_level_sum(LevelSum a, float* red, int t)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { a.e += __shfl_down_sync(0xffffffffu, a.e, o); a.m += __shfl_down_sync(0xffffffffu, a.m, o); }
    __syncthreads();
    if ((t & 31) == 0) { red[t >> 5] = a.m; red[4 + (t >> 5)] = __int_as_float(a.e); }
    __syncthreads();
    LevelSum r;
    r.m = red[0] + red[1] + red[2] + red[3];
    r.e = __float_as_int(red[4]) + __float_as_int(red[5]) + __float_as_int(red[6]) + __float_as_int(red[7]);
    return r;
}

// per-thread loop-invariant shared-memory indices of the exchange buffer (see swz() in ofdm_core.cuh)
struct XIdx {
    int a[2];     // pass A: swz(8 * rev(n0)) for the two blocks; element e lives at a[h] ^ e
    int b[4];     // pass B: swz(base) ^ 8a; element (a, b) lives at b[a] + 32 b
    int kk;
};
__device__ __forceinline__ XIdx make_xidx(int t)
{
    XIdx x;
    x.a[0] = swz(8 * rev4x4(t)); x.a[1] = swz(8 * rev4x4(t + 128));
    x.kk = t & 7;
    const int sb = swz(128 * (t >> 3) + x.kk);
#pragma unroll
    for (int a = 0; a < 4; a++) x.b[a] = sb ^ (8 * a);
    return x;
}
// pass C: position t + 128 c -> (t ^ X(c)) + 128 c with the compile-time constant X(c) = swizzle bits of 128 c
__device__ __forceinline__ constexpr int xc_of(int c) { return ((c & 1) << 3) | (((c >> 1) & 1) << 2) | ((c >> 2) & 3); }

// FFT of the 2048 samples at src[w0 .. w0+2048) -> v[a+4b] = X[t + 128a + 512b], exact arithmetic.  Contains two __syncthreads.
__device__ __forceinline__ void fft2048_from_global(const float2* __restrict__ src, int64_t w0, float2 v[16], OfdmSmem& sm, int t, const XIdx& xi,
                                                    const DevTables& tb, const Nco& nco, const float2* __restrict__ tw_c5)
{
    // pass A: two blocks n0 = t, t+128; loads are lane-consecutive for each c
    float2 x[16];
    const float2* p = src + w0 + t;
#pragma unroll
    for (int h = 0; h < 2; h++)
#pragma unroll
        for (int c = 0; c < 8; c++) x[8 * h + c] = __ldg(p + 128 * h + 256 * c);
    if (nco.mix) {
        int32_t lp = mod_rate64((int64_t)nco.lp0 - (w0 + t) * (int64_t)nco.ph);
#pragma unroll
        for (int c = 0; c < 8; c++) {
            x[c] = mix_sample(x[c], tb, lp);
            x[8 + c] = mix_sample(x[8 + c], tb, sub_mod(lp, nco.d128));
            lp = sub_mod(lp, nco.d256);
        }
    }
#pragma unroll
    for (int h = 0; h < 2; h++) {
        float2 y[8];
        passA_block<true, false>(x + 8 * h, y, sm.tw);
#pragma unroll
        for (int e = 0; e < 8; e++) sm.xbuf[xi.a[h] ^ e] = y[e];
    }
    __syncthreads();
    // pass B
    {
#pragma unroll
        for (int b = 0; b < 4; b++)
#pragma unroll
            for (int a = 0; a < 4; a++) v[a + 4 * b] = sm.xbuf[xi.b[a] + 32 * b];
        passB<true, false>(v, xi.kk, sm.tw);
#pragma unroll
        for (int b = 0; b < 4; b++)
#pragma unroll
            for (int a = 0; a < 4; a++) sm.xbuf[xi.b[a] + 32 * b] = v[a + 4 * b];
    }
    __syncthreads();
    // pass C
#pragma unroll
    for (int c = 0; c < 16; c++) v[c] = sm.xbuf[(t ^ xc_of(c)) + 128 * c];
    passC_ldg<true, false>(v, t, tw_c5);
}

// ---- TMA / mbarrier helpers (SASS: UBLKCP, SYNCS) ----
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count)); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity)
{
    asm volatile("{\n.reg .pred p;\nWAIT_LOOP:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@p bra DONE;\nbra WAIT_LOOP;\nDONE:\n}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// one term of the fine-AFC correlation, fc += x conj(b), rounded as the contracted form the kernel always compiled to (so the transformed
// and the light symbols of ofdm_demod_kernel round identically)
__device__ __forceinline__ void afc_acc(float2& fc, float2 x, float2 b)
{
    fc.x = __fadd_rn(fc.x, __fmaf_rn(x.x, b.x, __fmul_rn(x.y, b.y)));
    fc.y = __fadd_rn(fc.y, __fmaf_rn(x.y, b.x, -__fmul_rn(x.x, b.y)));
}
// |re| + |im| of a thread's first (mixed) window sample: the sub-sampled input of the running signal level (see advance_kernel)
__device__ __forceinline__ float level_sample(float2 x) { return fabsf(x.x) + fabsf(x.y); }

// (1 - 1e-5)^2552: what the reference's level tracker sLevel = 1e-5 |v|_1 + (1 - 1e-5) sLevel (ofdm-processor.cpp:166,215) forgets per symbol
constexpr float LEVEL_DECAY_SYM = 0.97480279f;
constexpr int IN_CAP = 2560;     // staged samples per symbol: 2552 + 1 (16-byte alignment shift) + 1 (round-up), padded
constexpr int SB_DUMMY = 1536;   // softbit staging as (re, im) byte pairs indexed by logical carrier: [0,1536) real entries, then one private
                                 // dummy entry per thread for its unused bin
struct __align__(16) DemodSmem {
    float2 inbuf[IN_CAP];            // 20 KB: one symbol, guard interval first, filled by one cp.async.bulk (TMA)
    float2 xbuf[TU];                 // 16 KB swizzled exchange buffer
    float2 tw[TwLayout::C4];         // 1 KB: twiddles of passes A and B (pass C reads its 15 KB through L1 with __ldg)
    uint16_t sbuf[1536 + 128];        // (re | im << 8) per logical carrier: one 16-bit scatter store per carrier
    float2 rtab[2][16];              // DABB_NCO_FAST: e^{-j theta((128 h + 256 c) Hz)} for the PRS / the data symbols
    float red[16];
    uint64_t full;                   // a transformed symbol's copy, or a light symbol's in the first half of inbuf
    uint64_t half1;                  // a light symbol's copy in the second half of inbuf
    uint8_t kind[NSYM];              // per symbol of the frame: SYM_LIGHT, SYM_FFT or SYM_DEMAP (from the frame's symbol mask)
};

// A symbol that no decoder reads and that is no demapped symbol's reference is "light": it contributes only its fine-AFC terms and its
// level sample, which need the guard interval, the last T_g samples and the first OFDM_THREADS window samples - the symbol's samples
// [0, LIGHT_A) and [T_u, T_s), 9.1 instead of 20.4 KB.  Two light symbols are staged at once, one in each half of inbuf: the first span
// at the half's start, the second LIGHT_B samples later (each with the transformed symbol's 16-byte alignment shift).
enum : uint8_t { SYM_LIGHT = 0, SYM_FFT = 1, SYM_DEMAP = 2 };
constexpr int IN_HALF = IN_CAP / 2, LIGHT_A = TG + OFDM_THREADS, LIGHT_B = 640;
static_assert(LIGHT_B >= LIGHT_A + 2 && LIGHT_B % 2 == 0 && LIGHT_B + TG + 2 <= IN_HALF, "light symbol staging");
// sample-clock derotation (the CLOCK instances): the frame's factors Q[1..6] of dabb_clock::phasor live in the six entries of inbuf past
// the largest copy (a transformed symbol: T_s samples + the alignment shift, rounded up to an even count), which no copy writes
constexpr int CLK_Q = TS + 2;
static_assert(CLK_Q + 6 <= IN_CAP, "clock factors behind the symbol copy");

// a light symbol at lb (= the half's start + the alignment shift): exactly the per-thread fine-AFC terms and level sample the transformed
// path (fft2048_from_smem) takes for it, in the same order and with the same oscillator phases; window sample n >= T_u - T_g is at
// lb[LIGHT_B + n - (T_u - T_g)], its partner T_u earlier at lb[n - (T_u - T_g)], window sample t at lb[T_g + t]
template <bool FASTNCO>
__device__ __forceinline__ void light_symbol(const float2* lb, int64_t idx0, int t, const DevTables& tb, const Nco& nco, float2& fc, const float2* rtab, float& l1_first)
{
    const float2* tail = lb + LIGHT_B;
    if (FASTNCO && nco.mix) {
        // raw samples for the correlation (the frame's sum is rotated once at the end of the kernel)
#pragma unroll
        for (int h = 0; h < 2; h++)
#pragma unroll
            for (int c = 6; c < 8; c++) {
                const int n = t + 128 * h + 256 * c;
                if (n >= TU - TG) afc_acc(fc, tail[n - (TU - TG)], lb[n - (TU - TG)]);
            }
        const float2 o0 = osc_fast(mod_rate64((int64_t)nco.lp0 - (idx0 + t) * (int64_t)nco.ph));
        l1_first = level_sample(cmul_fast(lb[TG + t], cmul_fast(o0, rtab[0])));
        return;
    }
    if (nco.mix) {
#pragma unroll
        for (int h = 0; h < 2; h++)
#pragma unroll
            for (int c = 6; c < 8; c++) {
                const int n = t + 128 * h + 256 * c;
                if (n >= TU - TG) {
                    const int32_t l = mod_rate64((int64_t)nco.lp0 - (idx0 + n) * (int64_t)nco.ph);
                    afc_acc(fc, mix_sample(tail[n - (TU - TG)], tb, l), mix_sample(lb[n - (TU - TG)], tb, sub_mod(l, nco.u2048)));
                }
            }
        l1_first = level_sample(mix_sample(lb[TG + t], tb, mod_rate64((int64_t)nco.lp0 - (idx0 + t) * (int64_t)nco.ph)));
        return;
    }
#pragma unroll
    for (int h = 0; h < 2; h++)
#pragma unroll
        for (int c = 6; c < 8; c++) {
            const int n = t + 128 * h + 256 * c;
            if (n >= TU - TG) afc_acc(fc, tail[n - (TU - TG)], lb[n - (TU - TG)]);
        }
    l1_first = level_sample(lb[TG + t]);
}

// one symbol's samples, already in shared memory at in[0..], -> spectrum in registers (same pass structure as
// fft2048_from_global); idx0 = frame-relative index of in[0] for the NCO phase

// With afc: also accumulates the fine-AFC correlation of this symbol, sum x[i] * conj(x[i - T_u]) over its last 504 samples
// (ofdm-processor.cpp:436-442): those are the transform inputs n = 1544..2047, which the owning thread has just mixed, so only
// the guard-interval partner (T_u samples earlier, at in[n - 2048]) is loaded and mixed here.
template <bool EXACT, bool FASTNCO>
__device__ __forceinline__ void fft2048_from_smem(const float2* in, int64_t idx0, float2 v[16], DemodSmem& sm, int t, const XIdx& xi,
                                                  const float2* __restrict__ tw_c5, const DevTables& tb, const Nco& nco, bool afc, float2& fc, const float2* rtab, float& l1_first)
{
    // l1_first: |re| + |im| of the thread's first (mixed) sample, the sub-sampled input of the running signal level (see advance_kernel)
    if (FASTNCO && nco.mix) {
        // sample n = t + 128 h + 256 c gets osc(lp - (128 h + 256 c) Hz) = osc(lp) * rtab[8 h + c]; the guard-interval correlation is
        // taken on the raw samples: mixing multiplies every term x[i] conj(x[i - T_u]) by the same e^{-j theta(2048 Hz)}, applied
        // once to the frame's sum at the end of the kernel
        const float2 o0 = osc_fast(mod_rate64((int64_t)nco.lp0 - (idx0 + t) * (int64_t)nco.ph));
#pragma unroll
        for (int h = 0; h < 2; h++) {
            float2 x[8];
#pragma unroll
            for (int c = 0; c < 8; c++) x[c] = in[t + 128 * h + 256 * c];
            if (afc) {
#pragma unroll
                for (int c = 6; c < 8; c++) {
                    const int n = t + 128 * h + 256 * c;
                    if (n >= TU - TG) afc_acc(fc, x[c], in[n - TU]);
                }
            }
#pragma unroll
            for (int c = 0; c < 8; c++) x[c] = cmul_fast(x[c], cmul_fast(o0, rtab[8 * h + c]));
            if (h == 0) l1_first = level_sample(x[0]);
            float2 y[8];
            passA_block<EXACT, false>(x, y, sm.tw);
#pragma unroll
            for (int e = 0; e < 8; e++) sm.xbuf[xi.a[h] ^ e] = y[e];
        }
        return;
    }
    // one 8-point block at a time (load, oscillator, radix-2 + radix-4, store): keeps 8 instead of 16 inputs live while the
    // oscillator's double-precision temporaries are
    int32_t lp = 0;
    if (nco.mix) lp = mod_rate64((int64_t)nco.lp0 - (idx0 + t) * (int64_t)nco.ph);
#pragma unroll
    for (int h = 0; h < 2; h++) {
        float2 x[8];
#pragma unroll
        for (int c = 0; c < 8; c++) x[c] = in[t + 128 * h + 256 * c];
        if (nco.mix) {
            int32_t l = h ? sub_mod(lp, nco.d128) : lp;
#pragma unroll
            for (int c = 0; c < 8; c++) {
                x[c] = mix_sample(x[c], tb, l);
                if (c >= 6 && afc) {
                    const int n = t + 128 * h + 256 * c;
                    if (n >= TU - TG) afc_acc(fc, x[c], mix_sample(in[n - TU], tb, sub_mod(l, nco.u2048)));     // phase of the sample T_u earlier
                }
                l = sub_mod(l, nco.d256);
            }
        } else if (afc) {
#pragma unroll
            for (int c = 6; c < 8; c++) {
                const int n = t + 128 * h + 256 * c;
                if (n >= TU - TG) afc_acc(fc, x[c], in[n - TU]);
            }
        }
        if (h == 0) l1_first = level_sample(x[0]);
        float2 y[8];
        passA_block<EXACT, false>(x, y, sm.tw);
#pragma unroll
        for (int e = 0; e < 8; e++) sm.xbuf[xi.a[h] ^ e] = y[e];
    }
}
template <bool EXACT>
__device__ __forceinline__ void fft2048_finish(float2 v[16], DemodSmem& sm, int t, const XIdx& xi, const float2* __restrict__ tw_c5, const TwB2& b2)
{
#pragma unroll
    for (int b = 0; b < 4; b++)
#pragma unroll
        for (int a = 0; a < 4; a++) v[a + 4 * b] = sm.xbuf[xi.b[a] + 32 * b];
    passB_w<EXACT, false>(v, xi.kk, sm.tw, b2);
#pragma unroll
    for (int b = 0; b < 4; b++)
#pragma unroll
        for (int a = 0; a < 4; a++) sm.xbuf[xi.b[a] + 32 * b] = v[a + 4 * b];
    __syncthreads();
#pragma unroll
    for (int c = 0; c < 16; c++) v[c] = sm.xbuf[(t ^ xc_of(c)) + 128 * c];
    passC_ldg<EXACT, false>(v, t, tw_c5);
}

template <bool EXACT, bool TAP, bool FASTNCO, bool WEIGHTED, bool CLOCK>
__global__ void __launch_bounds__(OFDM_THREADS, 5)
ofdm_demod_kernel(DevTables tb, OfdmParams p)
{
    extern __shared__ __align__(16) unsigned char smraw[];
    DemodSmem& sm = *reinterpret_cast<DemodSmem*>(smraw);
    const int t = threadIdx.x;
    // ---- once per CTA
    if (t == 0) { mbar_init(&sm.full, 1); mbar_init(&sm.half1, 1); asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
    if (t < TwLayout::C4) sm.tw[t] = tb.tw_fwd[t];
    const float2* tw_c5 = tb.tw_fwd + TwLayout::C5;
    const XIdx xi = make_xidx(t);
    const TwB2 b2 = load_twb2(tb.tw_fwd, xi.kk);
    // loop-invariant: staging offset of each owned bin's softbits (unused bins write to a dummy area)
    int sidx[NSLOT];
#pragma unroll
    for (int s = 0; s < NSLOT; s++) { const int iv = tb.invperm[TU + t + 128 * slot_c(s)]; sidx[s] = iv >= 0 ? iv : SB_DUMMY + t; }   // exactly one unused slot per thread -> a private dummy byte
    // the reader's two 16-byte chunks (logical chunks t and t + 96) sit in these slots of the staging area (tables.cpp: kChunkSlot)
    // (bits 0-7 / 8-15: slot, bit 16 / 17: halves stored swapped)
    const int rslot = t < 96 ? (((int)tb.invperm[2 * TU + t] & 0xFF) | (((int)tb.invperm[2 * TU + t + 96] & 0xFF) << 8) |
                               (((int)tb.invperm[2 * TU + t] >> 8) << 16) | (((int)tb.invperm[2 * TU + t + 96] >> 8) << 17)) : 0;
    __syncthreads();

    // One CTA per work item: the first n_full frames are walked by `groups` items each; the remaining (tail) frames are cut into
    // tail_groups short items, which come last and fill the slots the long ones free one by one at the end of the launch.
    const int item = blockIdx.x;
    if (item >= p.n_full * p.groups + (p.n_frames - p.n_full) * p.tail_groups) return;
    [&]() {     // the body stays a lambda: as a plain block, ptxas spills more in three of the eight instances
    int f, g, spc, ng;
    if (item < p.n_full * p.groups) { f = item / p.groups; g = item % p.groups; spc = p.sym_per_cta; ng = p.groups; }
    else { const int r = item - p.n_full * p.groups; f = p.n_full + r / p.tail_groups; g = r % p.tail_groups; spc = 75 / p.tail_groups; ng = p.tail_groups; }
    if (p.active && !p.active[f]) return;
    const unsigned long long trace_t0 = p.trace.rec ? trace_now() : 0ull;

    const float2* src = p.iq + (int64_t)f * p.stride + p.prs_start[f];
    const int l_first = 1 + g * spc, l_last = l_first + spc;   // data symbols [l_first, l_last)

    // sample range of symbol l relative to the first useful PRS sample: the PRS is [0,2048); symbol l >= 1 (guard first)
    // starts at 2048 + (l-1)*2552, its FFT window 504 samples later (ofdm-decoder.cpp:178-180)
    auto issue = [&](int l) {
        const int64_t s0 = (l == 0) ? 0 : (int64_t)TU + (int64_t)(l - 1) * TS;
        const int count = (l == 0) ? TU : TS;
        const float2* g0 = src + s0;
        const int shift = (int)((reinterpret_cast<uintptr_t>(g0) >> 3) & 1);     // cp.async.bulk needs 16-byte aligned addresses
        const uint32_t bytes = (uint32_t)(((count + shift + 1) & ~1) * 8);
        mbar_expect_tx(&sm.full, bytes);
        bulk_g2s(sm.inbuf, g0 - shift, bytes, &sm.full);
    };
    // a light symbol (l >= 1) into half h of inbuf: its samples [0, LIGHT_A) and [T_u, T_s), on that half's barrier
    auto issue_light = [&](int l, int h) {
        const float2* g0 = src + (int64_t)TU + (int64_t)(l - 1) * TS;
        const int shift = (int)((reinterpret_cast<uintptr_t>(g0) >> 3) & 1);
        const uint32_t ba = (uint32_t)(((LIGHT_A + shift + 1) & ~1) * 8), bb = (uint32_t)(((TG + shift + 1) & ~1) * 8);
        uint64_t* bar = h ? &sm.half1 : &sm.full;
        mbar_expect_tx(bar, ba + bb);
        bulk_g2s(sm.inbuf + IN_HALF * h, g0 - shift, ba, bar);
        bulk_g2s(sm.inbuf + IN_HALF * h + LIGHT_B, g0 + TU - shift, bb, bar);
    };
    // what each symbol of the frame needs (CTA-uniform): transformed when it is the phase reference symbol, demapped, or the reference of
    // a demapped symbol; light otherwise.  No mask: every symbol is transformed and demapped.
    if (t < NSYM) {
        const uint32_t* m = p.symmask ? p.symmask + (int64_t)f * OFDM_MASK_WORDS : nullptr;
        const bool dm = !m || ((m[t >> 5] >> (t & 31)) & 1u), dm1 = !m || (t + 1 < NSYM && ((m[(t + 1) >> 5] >> ((t + 1) & 31)) & 1u));
        sm.kind[t] = (t > 0 && dm) ? SYM_DEMAP : ((t == 0 || dm1) ? SYM_FFT : SYM_LIGHT);
    }

    // nco[f] = {phase applied to PRS sample 0, Hz for the PRS, phase at index 0 extrapolated for the data symbols, Hz}
    const Nco ncoP = make_nco(p.nco ? p.nco[4 * f] : 0, p.nco ? p.nco[4 * f + 1] : 0);
    const Nco ncoS = make_nco(p.nco ? p.nco[4 * f + 2] : 0, p.nco ? p.nco[4 * f + 3] : 0);
    if (FASTNCO && t < 32) {
        const Nco& n = (t >> 4) ? ncoS : ncoP;
        const int k = t & 15;
        sm.rtab[t >> 4][k] = osc_fast(mod_rate64(-(int64_t)(128 * (k >> 3) + 256 * (k & 7)) * n.ph));
    }
    __syncthreads();
    // CLOCK: the frame's ppm (CTA-uniform); 0 leaves r1 untouched.  Carrier k = t + 128 j of this thread is derotated by P * Q[j]
    // (dabb_clock::phasor): P in registers, Q[1..6] in shared memory, written here and first read after barrier (1) of the first symbol
    float2 ckp = make_float2(1.f, 0.f);
    bool rot = false;
    if (CLOCK) {
        const float a = p.clock[f];
        rot = a != 0.f;
        if (rot) {
            ckp = dabb_clock::factor_p(t, a);
            if (t < 6) sm.inbuf[CLK_Q + t] = dabb_clock::factor_q(t + 1, a);
        }
    }
    // the phasor of slot s: bin t + 128 slot_c(s), carrier j = slot_c(s) (< 7) or slot_c(s) - 16
    auto clk_phasor = [&](int s) -> float2 {
        const int c = slot_c(s), j = c < 7 ? c : c - 16;
        if (j == 0) return ckp;
        const float2 q = sm.inbuf[CLK_Q - 1 + (j < 0 ? -j : j)];
        return dabb_clock::cmul(ckp, j < 0 ? make_float2(q.x, -q.y) : q);
    };

    // TAP: where symbol l's r1 goes (CTA-uniform), nullptr for nowhere.  Without r1_row, row f * 75 + l - 1 (the constellation tap);
    // with it, row r1_row[f] (< 0: the frame stores nothing) plus the symbol's column: l - 1 without r1_lmask, else its rank among the
    // symbols r1_lmask[f] marks (a diversity group's leader's symbols, combine.cu), nothing for the symbols it does not mark
    auto r1_dst = [&](int l) -> float2* {
        if (!p.r1_row) return p.r1 + ((int64_t)f * 75 + (l - 1)) * KC;
        const int32_t b = p.r1_row[f];
        if (b < 0) return nullptr;
        if (!p.r1_lmask) return p.r1 + ((int64_t)b + (l - 1)) * KC;
        const uint32_t* m = p.r1_lmask + (int64_t)f * OFDM_MASK_WORDS;
        if (!((m[l >> 5] >> (l & 31)) & 1u)) return nullptr;
        int c = __popc(m[l >> 5] & ((1u << (l & 31)) - 1u));
        for (int w = 0; w < (l >> 5); w++) c += __popc(m[w]);
        return p.r1 + ((int64_t)b + c) * KC;
    };

    // Staging: inbuf holds one transformed symbol or two light ones.  Symbols are copied in order, each as soon as its space is free
    // (a transformed one needs both halves); light symbols alternate between the halves.  The reference symbol l_first - 1 of a later
    // item is staged only when it is transformed: a light one contributes nothing to this item.
    auto kind_of = [&](int l) -> int { return sm.kind[l]; };
    const int l_begin = (l_first > 1 && kind_of(l_first - 1) == SYM_LIGHT) ? l_first : l_first - 1;
    int nxt = l_begin;                    // next symbol to copy
    int used = 0, ih = 0, ch = 0;         // halves in use; half of the next light copy, of the next light symbol to consume
    uint32_t parity = 0;                  // bit h: phase parity of the barrier of half h (half 0's is also the transformed symbols')
    auto fill = [&]() {
        while (nxt < l_last) {
            const int need = kind_of(nxt) == SYM_LIGHT ? 1 : 2;
            if (used + need > 2) break;
            if (t == 0) {
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                if (need == 2) issue(nxt); else issue_light(nxt, ih);
            }
            if (need == 1) ih ^= 1;
            used += need; nxt++;
        }
    };
    fill();

    float2 prev[NSLOT];
    float2 fc = make_float2(0.f, 0.f);
    float lvl = 0.f;                                  // decayed sum of one sample magnitude per symbol and thread (signal level estimate)

    for (int l = l_begin; l < l_last; l++) {
        const int64_t s0 = (l == 0) ? 0 : (int64_t)TU + (int64_t)(l - 1) * TS;
        const int goff = (l == 0) ? 0 : TG;
        const int shift = (int)((reinterpret_cast<uintptr_t>(src + s0) >> 3) & 1);
        const int kind = kind_of(l);
        if (kind == SYM_LIGHT) {               // l >= l_first: its fine-AFC terms and level sample only
            mbar_wait(ch ? &sm.half1 : &sm.full, (parity >> ch) & 1); parity ^= 1u << ch;
            float l1s;
            light_symbol<FASTNCO>(sm.inbuf + IN_HALF * ch + shift, s0 + TG, t, tb, ncoS, fc, sm.rtab[1], l1s);
            lvl = fmaf(lvl, LEVEL_DECAY_SYM, l1s);
            ch ^= 1;
            __syncthreads();                   // the half is consumed
            used -= 1; fill();
            continue;
        }
        const Nco& nco = l == 0 ? ncoP : ncoS;
        mbar_wait(&sm.full, parity & 1); parity ^= 1;
        const float2* in = sm.inbuf + shift;
        float2 v[16];
        float l1s;
        fft2048_from_smem<EXACT, FASTNCO>(in + goff, s0 + goff, v, sm, t, xi, tw_c5, tb, nco, l >= l_first, fc, sm.rtab[l == 0 ? 0 : 1], l1s);
        if (l >= l_first || l == 0) lvl = fmaf(lvl, LEVEL_DECAY_SYM, l1s);
        __syncthreads();                       // (1) inbuf fully consumed, pass-A results in xbuf
        used = 0; fill();                      // prefetch the next symbol(s) while passes B, C and the demap run
        fft2048_finish<EXACT>(v, sm, t, xi, tw_c5, b2);   // contains barrier (2)

        if (l >= l_first && kind == SYM_DEMAP) {
            if (WEIGHTED) {
                // DABB_DEMAP_WEIGHTED: r1 of every owned bin into v[] (its spectrum moves to prev[]), the symbol's geometric-mean carrier
                // level G from one block reduction, then the demap against max(l1, G) (ofdm_core.cuh: level_acc, level_gmean)
                LevelSum ls{0, 0.f};
                float2* const r1d = TAP ? r1_dst(l) : nullptr;
#pragma unroll
                for (int s = 0; s < NSLOT; s++) {
                    const float2 X = v[slot_c(s)];
                    v[slot_c(s)] = diff_one<EXACT>(X, prev[s]);
                    if (CLOCK && rot) v[slot_c(s)] = dabb_clock::cmul(v[slot_c(s)], clk_phasor(s));
                    prev[s] = X;
                    if (sidx[s] < SB_DUMMY) level_acc(ls, level_l1(v[slot_c(s)]));
                }
                const LevelSum tot = block_level_sum(ls, sm.red, t);
                const float G = level_gmean(tot), rG = q127(G);
#pragma unroll
                for (int s = 0; s < NSLOT; s++) {
                    const float2 r1 = v[slot_c(s)];
                    int8_t sre, sim;
                    demap_weighted(r1, G, rG, sre, sim);
                    sm.sbuf[sidx[s]] = (uint16_t)((uint8_t)sre | ((uint16_t)(uint8_t)sim << 8));
                    if (TAP && r1d) { const int c0 = tb.invperm[t + 128 * slot_c(s)]; if (c0 >= 0) r1d[c0] = r1; }
                }
            } else {
            // demap owned bins against the previous symbol, scatter softbits into logical order (branch free)
            float2* const r1d = TAP ? r1_dst(l) : nullptr;
#pragma unroll
            for (int s = 0; s < NSLOT; s++) {
                const float2 X = v[slot_c(s)];
                int8_t sre, sim; float2 r1;
                if (CLOCK) {
                    r1 = diff_one<EXACT>(X, prev[s]);
                    if (rot) r1 = dabb_clock::cmul(r1, clk_phasor(s));
                    demap_r1(r1, sre, sim);
                } else demap_one<EXACT>(X, prev[s], sre, sim, r1);
                sm.sbuf[sidx[s]] = (uint16_t)((uint8_t)sre | ((uint16_t)(uint8_t)sim << 8));
                if (TAP && r1d) { const int c0 = tb.invperm[t + 128 * slot_c(s)]; if (c0 >= 0) r1d[c0] = r1; }
                prev[s] = X;
            }
            }
            __syncthreads();                   // (3)
            // de-interleave the pairs into the reference's layout (1536 Re bits, then 1536 Im bits): thread t < 96 takes the 16-byte
            // chunks t and t + 96 of the staging area (lane-consecutive: conflict-free; 8 carriers each) and stores 8 bytes per chunk and half
            if (t < 96) {
                const uint4* s4 = reinterpret_cast<const uint4*>(sm.sbuf);
                uint2* dst = reinterpret_cast<uint2*>(p.soft + (int64_t)f * p.soft_stride + (int64_t)(l - 1) * 3072);
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    const uint4 a = s4[(rslot >> (8 * h)) & 0xFF];
                    const bool sw = (rslot >> (16 + h)) & 1;
                    const uint32_t lo0 = sw ? a.z : a.x, lo1 = sw ? a.w : a.y, hi0 = sw ? a.x : a.z, hi1 = sw ? a.y : a.w;
                    uint2 re, im;
                    re.x = __byte_perm(lo0, lo1, 0x6420); im.x = __byte_perm(lo0, lo1, 0x7531);
                    re.y = __byte_perm(hi0, hi1, 0x6420); im.y = __byte_perm(hi0, hi1, 0x7531);
                    dst[t + 96 * h] = re;               // carriers 8 (t + 96 h) .. + 7
                    dst[192 + t + 96 * h] = im;
                }
            }
        } else {
            // a reference only (the PRS when l == 0, or a symbol no decoder reads before one they do): keep its spectrum, estimate SNR from the PRS
#pragma unroll
            for (int s = 0; s < NSLOT; s++) prev[s] = v[slot_c(s)];
            __syncthreads();                   // (3') every thread is done reading xbuf before the next symbol's pass A overwrites it
            if (l == 0 && p.snr) {
                // OfdmDecoder::get_snr method 1 (ofdm-decoder.cpp:246-265): noise bins 1094..1259 and 788..887,
                // signal bins 1664..2047 and 0..383
                float noise = 0.f, signal = 0.f;
#pragma unroll
                for (int c = 0; c < 16; c++) {
                    const int bin = t + 128 * c;
                    const float mag = (float)sqrt((double)v[c].x * (double)v[c].x + (double)v[c].y * (double)v[c].y);
                    if ((bin >= 1094 && bin < 1260) || (bin >= 788 && bin < 888)) noise += mag;
                    if (bin >= 1664 || bin < 384) signal += mag;
                }
                noise = block_sum(noise, sm.red, t);
                signal = block_sum(signal, sm.red, t);
                if (t == 0) {
                    noise /= 266.f;
                    const float dbs = 20.f * log10f((signal / 768.f + 1.0f) / 256.0f), dbn = 20.f * log10f((noise + 1.0f) / 256.0f);
                    p.snr[f] = (int32_t)(int16_t)(dbs - dbn);
                }
            }
        }
    }
    if (p.freqcorr) {
        const float sx = block_sum(fc.x, sm.red, t), sy = block_sum(fc.y, sm.red, t);
        float2 sum = make_float2(sx, sy);
        if (FASTNCO && ncoS.mix) sum = cmul_fast(sum, osc_fast(ncoS.u2048));      // x[i] conj(x[i - T_u]) of the mixed samples
        if (t == 0) p.freqcorr[(int64_t)f * p.fc_pitch + g] = sum;
        if (g == 0 && t > 0 && t < p.fc_pitch - ng + 1) p.freqcorr[(int64_t)f * p.fc_pitch + ng - 1 + t] = make_float2(0.f, 0.f);   // unused partial slots
    }
    if (p.level) {
        // this CTA's share of the frame's level estimate, referred to the end of symbol 75: mean over the 128 sampled positions, decayed
        // by the symbols that follow this CTA's last one
        const float s = block_sum(lvl, sm.red, t);
        if (t == 0) p.level[(int64_t)f * p.fc_pitch + g] = s * (1.0f / 128.0f) * powf(LEVEL_DECAY_SYM, (float)(76 - l_last));
        if (g == 0 && t > 0 && t < p.fc_pitch - ng + 1) p.level[(int64_t)f * p.fc_pitch + ng - 1 + t] = 0.f;
    }
    if (p.trace.rec && t == 0) trace_put(p.trace, 1u, trace_t0);
    }();
}

// ------------------------------------------------------------------------------------------------------------
// findIndex: FFT -> * conj(refTable) -> IFFT/2048 -> |.| (find_index_kernel, one CTA per window), then the placement search
// (find_search_tbp_kernel, find_search_kernel).  The sum of |.| is accumulated sequentially by one thread in index order like the
// CPU loop (phasereference.cpp:216-220) so that the `max > 3*sum/Tu` decision sees the same float.
// ------------------------------------------------------------------------------------------------------------
struct __align__(16) SyncSmem {
    OfdmSmem o;
    float cir[TU];
    float2 spec[128];
    float cand[128];
    float cv[96]; float refarg[24];
    float wmax[4]; int wmin[4];
    float sum;
};

// coarse frequency estimate of one aligned PRS = the T_u samples at src[off ..]; collective over the CTA, result via *out
__device__ __forceinline__ void coarse_estimate(const DevTables& tb, SyncSmem& sm, const float2* __restrict__ src, int64_t off, const Nco& nco, const XIdx& xi,
                                                int t, int freqsync, int32_t* out)
{
    // ---- coarse AFC (OFDMProcessor::processPRS, ofdm-processor.cpp:537-644): FFT of the aligned PRS (window start + index).
    // NOTE on `abs`: in the reference's translation unit the unqualified abs() of a float/double is the C library's
    // int abs(int) - the argument is truncated to int first (see oracle/dab_oracle.c, pinned against the compiled reference).
    float2 v[16];
    __syncthreads();
    if (t < TwLayout::C4) sm.o.tw[t] = tb.tw_fwd[t];
    __syncthreads();
    // the PRS useful part starts `off` samples into the window; its samples continue the NCO phase sequence
    fft2048_from_global(src, off, v, sm.o, t, xi, tb, nco, tb.tw_fwd + TwLayout::C5);
    if (freqsync == 1) {
        // ---- GetMiddle (:617-644), including its `sum = oldMax` assignment: moving sum of |X| over K carriers
#pragma unroll
        for (int c = 0; c < 16; c++) {
            const int bin = t + 128 * (c & 3) + 512 * (c >> 2);
            const double m = __dsqrt_rn(__dadd_rn(__dmul_rn((double)v[c].x, (double)v[c].x), __dmul_rn((double)v[c].y, (double)v[c].y)));
            sm.cir[bin] = (float)m;
        }
        __syncthreads();
        if (t == 0) {
            float sum = 0.f, oldMax = 0.f; int maxIndex = 0;
            for (int i = 40; i < 1536 + 40; i++) sum = __fadd_rn(sum, sm.cir[(TU / 2 + i) % TU]);
            for (int i = 40; i < TU - (1536 - 40); i++) {
                sum = __fsub_rn(sum, sm.cir[(TU / 2 + i) % TU]);
                sum = __fadd_rn(sum, sm.cir[(TU / 2 + i + 1536) % TU]);
                if (sum > oldMax) { sum = oldMax; maxIndex = i; }
            }
            *out = (int16_t)(maxIndex - (TU - 1536) / 2);
        }
        return;
    }
    // bins 2012..2047 and 0..63 in natural order
    float2* spec = sm.spec;     // [0..35] = bins 2012..2047, [36..99] = bins 0..63
    if (t < 64) spec[36 + t] = v[0];
    if (t >= 92) spec[t - 92] = v[15];
    __syncthreads();
    auto ap = [&](int a, int b) -> float {       // arg(X[a] * conj(X[b]))
        const float2 A = spec[a], B = spec[b];
        const float c = B.x, d = -B.y;
        const float re = __fsub_rn(__fmul_rn(A.x, c), __fmul_rn(A.y, d)), im = __fadd_rn(__fmul_rn(A.x, d), __fmul_rn(A.y, c));
        return atan2f(im, re);
    };
    auto iabs_f = [](float x) -> float { return (float)abs(__float2int_rz(x)); };                       // abs(float) -> int abs(int)
    auto iabs_pi = [](float x) -> float {                                                                 // abs(abs(x / M_PI) - 1)
        const int q = abs(__double2int_rz(__ddiv_rn((double)x, 3.14159265358979323846)));
        return (float)abs(q - 1);
    };
    if (freqsync == 2) {
        // ---- CorrelatePRS (:546-581): phase differences of adjacent carriers against those of the reference table
        if (t < 24) {
            const float2 A = tb.prs_ref[t], B = tb.prs_ref[t + 1];
            const float c = B.x, d = -B.y;
            sm.refarg[t] = atan2f(__fadd_rn(__fmul_rn(A.x, d), __fmul_rn(A.y, c)), __fsub_rn(__fmul_rn(A.x, c), __fmul_rn(A.y, d)));
        }
        if (t < 96) sm.cv[t] = ap(t, t + 1);
        __syncthreads();
        float mysum = 0.f;
        if (t < 72) for (int j = 0; j < 24; j++) mysum = __fadd_rn(mysum, iabs_f(__fmul_rn(sm.refarg[j], sm.cv[t + j])));
        sm.cand[t] = mysum;
        __syncthreads();
        if (t == 0) {
            // the partial sums only grow, so `sum > MMax` inside the j loop is decided by the full sum: first strict maximum
            float MMax = 0.f; int index = 100;
            for (int i = 0; i < 72; i++) if (sm.cand[i] > MMax) { MMax = sm.cand[i]; index = i; }
            *out = (int16_t)(TU - 36 + index - TU);
        }
        return;
    }
    // ---- PatternOfZeros (:582-613) over +-36 carriers
    float mysum = 1e30f;
    if (t < 72) {
        // candidate i = Tu - 36 + t; fft_buffer[(i + k) % Tu] = spec[t + k]
        const float a1 = iabs_pi(ap(t + 1, t + 2)), a2 = iabs_pi(ap(t + 2, t + 3));
        const float a3 = iabs_f(ap(t + 3, t + 4)), a4 = iabs_f(ap(t + 4, t + 5)), a5 = iabs_f(ap(t + 5, t + 6));
        const float b1 = iabs_pi(ap(t + 17, t + 19));
        const float b2 = iabs_f(ap(t + 19, t + 20)), b3 = iabs_f(ap(t + 20, t + 21)), b4 = iabs_f(ap(t + 21, t + 22));
        mysum = __fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(a1, a2), a3), a4), a5), b1), b2), b3), b4);
    }
    sm.cand[t] = mysum;
    __syncthreads();
    if (t == 0) {
        float mmin = 1000.f; int index = 100;      // sequential first-minimum like the CPU loop
        for (int i = 0; i < 72; i++) if (sm.cand[i] < mmin) { mmin = sm.cand[i]; index = TU - 36 + i; }
        *out = index - TU;
    }
}

// TII diagnostics (TIIDecoder::run, tii-decoder.cpp:197-214): the two transforms the decoder starts from - the phase reference symbol
// (the aligned T_u samples, oscillator applied) and the last T_u samples of the null symbol that follows the frame (already mixed by
// null_tap_kernel).  One CTA per (stream, which); spectra in natural bin order, bit-identical to the reference's fft::Forward.
__global__ void __launch_bounds__(OFDM_THREADS, 5)
tii_spectra_kernel(DevTables tb, const float2* iq, int64_t stride, const int64_t* prs_start, const int32_t* nco_frame, const int32_t* active,
                   const float2* nulls, float2* out)
{
    extern __shared__ __align__(16) unsigned char smraw[];
    OfdmSmem& sm = *reinterpret_cast<OfdmSmem*>(smraw);
    const int t = threadIdx.x, f = blockIdx.x >> 1, which = blockIdx.x & 1;
    float2* dst = out + ((int64_t)f * 2 + which) * TU;
    if (active && !active[f]) { for (int c = 0; c < 16; c++) dst[t + 128 * c] = make_float2(0.f, 0.f); return; }
    if (t < TwLayout::C4) sm.tw[t] = tb.tw_fwd[t];
    __syncthreads();
    const XIdx xi = make_xidx(t);
    float2 v[16];
    if (which == 0) {
        const Nco nco = make_nco(nco_frame[4 * f], nco_frame[4 * f + 1]);
        fft2048_from_global(iq + (int64_t)f * stride + prs_start[f], 0, v, sm, t, xi, tb, nco, tb.tw_fwd + TwLayout::C5);
    } else {
        const Nco nco = make_nco(0, 0);
        fft2048_from_global(nulls + (int64_t)f * TNULL, TNULL - TU, v, sm, t, xi, tb, nco, tb.tw_fwd + TwLayout::C5);
    }
#pragma unroll
    for (int c = 0; c < 16; c++) dst[t + 128 * c] = v[c];
}

// stage-level processPRS: one CTA per aligned PRS
__global__ void __launch_bounds__(OFDM_THREADS, 5)
coarse_kernel(DevTables tb, const float2* iq, int64_t stride, const int64_t* prs_start, int freqsync, int32_t* out)
{
    extern __shared__ __align__(16) unsigned char smraw[];
    SyncSmem& sm = *reinterpret_cast<SyncSmem*>(smraw);
    const int t = threadIdx.x, f = blockIdx.x;
    const Nco nco = make_nco(0, 0);
    const XIdx xi = make_xidx(t);
    coarse_estimate(tb, sm, iq + (int64_t)f * stride, prs_start[f], nco, xi, t, freqsync, out + f);
}

// interferer excision (DABB_ACQ_ROBUST, acq_core.cuh) on the window's spectrum, bins t + 128 c in v[c]: G is the geometric mean of the
// in-band bin powers (per thread in ascending c, the 128 partials in thread order); every in-band bin with power above T G and its
// EXC_NEIGH neighbours on each side (circular) are zeroed.  A window with no such bin is left untouched, bit for bit.  Thread 0 writes
// the number of zeroed bins.
__device__ __forceinline__ void excise_bins(float2 (&v)[16], int t, int32_t* excised)
{
    using namespace dabb_acq;
    __shared__ float part[EXC_THREADS];
    __shared__ uint32_t mark[TU / 32];
    __shared__ int total;
    float pw[16];
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < 16; c++) {
        pw[c] = __fadd_rn(__fmul_rn(v[c].x, v[c].x), __fmul_rn(v[c].y, v[c].y));
        if (in_band(t + 128 * c)) s = __fadd_rn(s, log2_pos(clamp_power(pw[c])));        // exc_partial
    }
    part[t] = s;
    if (t < TU / 32) mark[t] = 0u;
    if (t == 0) total = 0;
    __syncthreads();
    const float limit = exc_limit(part);
    bool any = false;
#pragma unroll
    for (int c = 0; c < 16; c++) {
        const int bin = t + 128 * c;
        if (exc_over(pw[c], bin, limit)) {
            any = true;
            for (int d = -EXC_NEIGH; d <= EXC_NEIGH; d++) { const int b = (bin + d) & (TU - 1); atomicOr(&mark[b >> 5], 1u << (b & 31)); }
        }
    }
    if (!__syncthreads_or(any)) { if (t == 0) *excised = 0; return; }      // CTA-uniform: nothing to excise
    int n = 0;
#pragma unroll
    for (int c = 0; c < 16; c++) {
        const int bin = t + 128 * c;
        if ((mark[bin >> 5] >> (bin & 31)) & 1u) { v[c] = make_float2(0.f, 0.f); n++; }
    }
    atomicAdd(&total, n);
    __syncthreads();
    if (t == 0) *excised = total;
}

template <bool NCO, bool EXCISE>
__device__ __forceinline__ void find_index_body(const DevTables& tb, const SyncParams& p, int32_t* excised)
{
    extern __shared__ __align__(16) unsigned char smraw[];
    SyncSmem& sm = *reinterpret_cast<SyncSmem*>(smraw);
    const int t = threadIdx.x, f = blockIdx.x;
    if (p.active && !p.active[f]) return;
    if (t < TwLayout::C4) sm.o.tw[t] = tb.tw_fwd[t];
    __syncthreads();
    const float2* src = p.iq + (int64_t)f * p.stride + p.win_start[f];
    const Nco nco = make_nco((NCO && p.nco) ? p.nco[2 * f] : 0, (NCO && p.nco) ? p.nco[2 * f + 1] : 0);
    const XIdx xi = make_xidx(t);
    float2 v[16];
    fft2048_from_global(src, 0, v, sm.o, t, xi, tb, nco, tb.tw_fwd + TwLayout::C5);
    if constexpr (EXCISE) excise_bins(v, t, excised + f);
    // res = X * conj(ref), written in natural order into the exchange buffer (free between the two transforms)
    float2* scratch = sm.o.xbuf;
    __syncthreads();             // pass C of the forward transform has read xbuf
#pragma unroll
    for (int c = 0; c < 16; c++) {
        const int bin = t + 128 * c;
        const float2 r = tb.prs_ref[bin];
        const float cc = r.x, d = -r.y;
        scratch[bin] = make_float2(fsub_<true>(fmul_<true>(v[c].x, cc), fmul_<true>(v[c].y, d)),
                                   fadd_<true>(fmul_<true>(v[c].x, d), fmul_<true>(v[c].y, cc)));
    }
    __syncthreads();
    if (t < TwLayout::C4) sm.o.tw[t] = tb.tw_inv[t];
    // inverse FFT reading its input from shared memory: same pass structure (load pattern n0 + 256 c)
    {
        float2 x[16];
#pragma unroll
        for (int h = 0; h < 2; h++)
#pragma unroll
            for (int c = 0; c < 8; c++) x[8 * h + c] = scratch[t + 128 * h + 256 * c];
        __syncthreads();   // twiddles loaded, scratch consumed
#pragma unroll
        for (int h = 0; h < 2; h++) {
            float2 y[8];
            passA_block<true, true>(x + 8 * h, y, sm.o.tw);
#pragma unroll
            for (int e = 0; e < 8; e++) sm.o.xbuf[xi.a[h] ^ e] = y[e];
        }
        __syncthreads();
#pragma unroll
        for (int b = 0; b < 4; b++)
#pragma unroll
            for (int a = 0; a < 4; a++) v[a + 4 * b] = sm.o.xbuf[xi.b[a] + 32 * b];
        passB<true, true>(v, xi.kk, sm.o.tw);
#pragma unroll
        for (int b = 0; b < 4; b++)
#pragma unroll
            for (int a = 0; a < 4; a++) sm.o.xbuf[xi.b[a] + 32 * b] = v[a + 4 * b];
        __syncthreads();
#pragma unroll
        for (int c = 0; c < 16; c++) v[c] = sm.o.xbuf[(t ^ xc_of(c)) + 128 * c];
        passC_ldg<true, true>(v, t, tb.tw_inv + TwLayout::C5);
    }
    // scale by 1/2048 (fft.cpp:146-158) and take the magnitude the way glibc's hypotf does (double sqrt, narrowed); the magnitudes go to
    // global memory: the search over them (find_search_tbp_kernel, find_search_kernel) is a different kind of work - a 2048-step
    // sequential sum beside a few short parallel phases - and runs as its own kernel at a much higher residency than this
    // register-heavy transform kernel
    const float factor = 1.0f / 2048.0f;
    float* cw = p.cir_work + (int64_t)f * TU;
#pragma unroll
    for (int c = 0; c < 16; c++) {
        const float re = fmul_<true>(v[c].x, factor), im = fmul_<true>(v[c].y, factor);
        const double m = __dsqrt_rn(__dadd_rn(__dmul_rn((double)re, (double)re), __dmul_rn((double)im, (double)im)));
        cw[t + 128 * c] = (float)m;
    }
}

template <bool NCO>
__global__ void __launch_bounds__(OFDM_THREADS, 5)
find_index_kernel(DevTables tb, SyncParams p)
{
    find_index_body<NCO, false>(tb, p, nullptr);
}

// the same with the interferer excision of DABB_ACQ_ROBUST; excised[f]: the bins zeroed in window f
template <bool NCO>
__global__ void __launch_bounds__(OFDM_THREADS, 5)
find_index_excise_kernel(DevTables tb, SyncParams p, int32_t* excised)
{
    find_index_body<NCO, true>(tb, p, excised);
}

// findIndex, second part: the placement search over the 2048 magnitudes of one window (phasereference.cpp:93-211) for the
// StrongestPeak and EarliestPeakWithBinning placements (ThresholdBeforePeak, the default: find_search_tbp_kernel).  One 128-thread CTA
// per window, 24 KB of shared memory and few registers: many windows per SM hide the sequential sum each of them carries.
struct __align__(16) SearchSmem {
    float cir[TU];
    float m2[2 * TU];
    float wmax[4]; int wmin[4];
    float sum;
};
__global__ void __launch_bounds__(OFDM_THREADS)
find_search_kernel(SyncParams p)
{
    __shared__ SearchSmem sm;
    const int t = threadIdx.x, f = blockIdx.x;
    if (p.active && !p.active[f]) return;
    {
        const float4* src4 = reinterpret_cast<const float4*>(p.cir_work + (int64_t)f * TU);
        float4* dst4 = reinterpret_cast<float4*>(sm.cir);
#pragma unroll
        for (int c = 0; c < 4; c++) dst4[t + 128 * c] = src4[t + 128 * c];
    }
    __syncthreads();
    // the binning placement never computes the last 8 magnitudes (loop bound i + 20 < Tu, phasereference.cpp:148)
    if (p.cir_out) for (int i = t; i < TU; i += OFDM_THREADS) p.cir_out[(int64_t)f * TU + i] = (p.placement == 2 && i >= 2040) ? 0.f : sm.cir[i];
    float* ma = sm.m2;
    float* mb = ma + TU;
    // the sequential float sum of the magnitudes in index order (the CPU loop's order, so the same float): 16-byte loads, and the loop
    // unrolled so that the loads run ahead of the dependent adds
    auto seq_sum = [&](float acc, int q0, int nq) {
        const float4* c4 = reinterpret_cast<const float4*>(sm.cir);
#pragma unroll 8
        for (int q = q0; q < q0 + nq; q++) {
            const float4 x = c4[q];
            acc = __fadd_rn(acc, x.x); acc = __fadd_rn(acc, x.y); acc = __fadd_rn(acc, x.z); acc = __fadd_rn(acc, x.w);
        }
        return acc;
    };
    int result;                 // what findIndex returns: >= 0 sample index, < 0 no synchronisation
    if (p.placement == 1) {
        // ---- StrongestPeak (:93-123): sequential sum, first maximum (strict >), negative score when below 3 x mean
        float mx = -10000.f; int mi = -1;
#pragma unroll
        for (int c = 0; c < 16; c++) { const int i = t + 128 * c; const float val = sm.cir[i]; if (val > mx) { mx = val; mi = i; } }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_down_sync(0xffffffffu, mx, o); const int oi = __shfl_down_sync(0xffffffffu, mi, o);
            if (ov > mx || (ov == mx && oi < mi)) { mx = ov; mi = oi; }
        }
        if ((t & 31) == 0) { sm.wmax[t >> 5] = mx; sm.wmin[t >> 5] = mi; }
        if (t == 32) sm.sum = seq_sum(0.f, 0, TU / 4);
        __syncthreads();
        mx = sm.wmax[0]; mi = sm.wmin[0];
#pragma unroll
        for (int w = 1; w < 4; w++) if (sm.wmax[w] > mx || (sm.wmax[w] == mx && sm.wmin[w] < mi)) { mx = sm.wmax[w]; mi = sm.wmin[w]; }
        const float sum = sm.sum;
        if (sum == 0.f) result = -1;
        else if (mx < __fdiv_rn(__fmul_rn(3.0f, sum), 2048.0f)) result = (int)__fsub_rn(-fabsf(__fdiv_rn(__fmul_rn(mx, 2048.0f), sum)), 1.0f);
        else result = mi;
    } else {
        // ---- EarliestPeakWithBinning (:124-211): 102 bins of 20 samples; the 4 strongest bins within 500 samples of the
        // strongest one; of those above 3 x mean, the earliest.  Bins of exactly equal value are ordered by position
        // (the reference's std::sort leaves that order unspecified).
        float* bval = ma; int* bidx = reinterpret_cast<int*>(mb);
        constexpr int NB = 102;
        if (t < NB) {
            float pv = 0.f; int pi = -1;
            for (int j = 0; j < 20; j++) { const float val = sm.cir[20 * t + j]; if (val > pv) { pv = val; pi = 20 * t + j; } }
            bval[t] = pv; bidx[t] = pi;
        }
        if (t == 127) sm.sum = __fdiv_rn(seq_sum(0.f, 0, 20 * NB / 4), 2048.0f);
        __syncthreads();
        if (t == 0) {
            int top = 0;
            for (int b = 1; b < NB; b++) if (bval[b] > bval[top]) top = b;
            const int peak_index = bidx[top];
            const float thresh = __fmul_rn(3.0f, sm.sum);
            unsigned long long used0 = 0, used1 = 0;      // 102 flags
            int earliest = -1; bool have = false;
            for (int k = 0; k < 4; k++) {
                int best = -1;
                for (int b = 0; b < NB; b++) {
                    const bool u = b < 64 ? (used0 >> b) & 1 : (used1 >> (b - 64)) & 1;
                    if (u || abs(bidx[b] - peak_index) > 500) continue;
                    if (best < 0 || bval[b] > bval[best]) best = b;
                }
                if (best < 0) break;
                if (best < 64) used0 |= 1ull << best; else used1 |= 1ull << (best - 64);
                if (bval[best] < thresh) continue;
                if (!have || bidx[best] < earliest) { earliest = bidx[best]; have = true; }
            }
            sm.wmin[0] = have ? earliest : -1;
        }
        __syncthreads();
        result = sm.wmin[0];
    }
    if (t == 0) {
        p.index_out[f] = result;
        if (p.coarse_out) p.coarse_out[f] = 100;          // 100 = not evaluated (OFDMProcessor::processPRS returns 100 for "no estimate" too)
    }
}

// ThresholdBeforePeak (the default placement, phasereference.cpp:212-253) without the sliding maximum.  The reference takes
// pk[i] = max(cir[i .. i+99]) for i + 100 < T_u (0 beyond), gmax = max pk, and - if gmax > 3 sum / T_u - returns the first i with
// pk[i + 100] > gmax / 2.  Since max() is exact: gmax = max(cir[0 .. T_u - 2]); and a window [j, j + 99], j >= 100, holds a value above
// the threshold exactly when j >= k* - 99 for the first k* >= 100 with cir[k*] > gmax / 2, so the first such window starts at
// j = max(100, k* - 99) (always < T_u - 100 for k* <= T_u - 2) and the result is j - 100.  What is left per window is the sequential
// float sum (one lane, 2048 dependent adds - the CPU loop's order, so the same float), one maximum and one first-above-threshold
// search: one WARP per window, four windows per CTA, 8 KB of shared memory each, so ~28 sums are in flight per SM.
__global__ void __launch_bounds__(OFDM_THREADS)
find_search_tbp_kernel(SyncParams p)
{
    __shared__ __align__(16) float cir_s[OFDM_THREADS / 32][TU];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int f = blockIdx.x * (OFDM_THREADS / 32) + w;
    if (f >= p.n) return;                                   // warp-uniform from here on
    if (p.active && !p.active[f]) return;
    float* cir = cir_s[w];
    const float4* src4 = reinterpret_cast<const float4*>(p.cir_work + (int64_t)f * TU);
    float gmax = -10000.f;
    float4 x[16];
#pragma unroll
    for (int c = 0; c < 16; c++) x[c] = src4[lane + 32 * c];
#pragma unroll
    for (int c = 0; c < 16; c++) {
        reinterpret_cast<float4*>(cir)[lane + 32 * c] = x[c];
        if (p.cir_out) reinterpret_cast<float4*>(p.cir_out + (int64_t)f * TU)[lane + 32 * c] = x[c];
        gmax = fmaxf(gmax, fmaxf(fmaxf(x[c].x, x[c].y), x[c].z));
        if (!(c == 15 && lane == 31)) gmax = fmaxf(gmax, x[c].w);          // index T_u - 1 is in no window
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) gmax = fmaxf(gmax, __shfl_xor_sync(0xffffffffu, gmax, o));
    const float thresh = gmax / 2;
    int kstar = 1 << 30;
#pragma unroll
    for (int c = 15; c >= 0; c--) {
        const int k0 = 4 * (lane + 32 * c);
        if (k0 + 3 <= TU - 2 && k0 + 3 >= 100 && x[c].w > thresh) kstar = k0 + 3;
        if (k0 + 2 >= 100 && x[c].z > thresh) kstar = k0 + 2;
        if (k0 + 1 >= 100 && x[c].y > thresh) kstar = k0 + 1;
        if (k0 >= 100 && x[c].x > thresh) kstar = k0;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) kstar = min(kstar, __shfl_xor_sync(0xffffffffu, kstar, o));
    __syncwarp();
    float sum = 0.f;
    if (lane == 0) {
        const float4* c4 = reinterpret_cast<const float4*>(cir);
#pragma unroll 8
        for (int q = 0; q < TU / 4; q++) {
            const float4 v = c4[q];
            sum = __fadd_rn(sum, v.x); sum = __fadd_rn(sum, v.y); sum = __fadd_rn(sum, v.z); sum = __fadd_rn(sum, v.w);
        }
    }
    sum = __shfl_sync(0xffffffffu, sum, 0);
    if (lane == 0) {
        int result = -1;
        // `3 * sum / Tu`: float 3*sum, then / (size_t Tu converted to float)
        if (gmax > __fdiv_rn(__fmul_rn(3.0f, sum), 2048.0f) && kstar != (1 << 30)) result = max(100, kstar - 99) - 100;
        p.index_out[f] = result;
        if (p.coarse_out) p.coarse_out[f] = 100;          // 100 = not evaluated
    }
}

// findIndex, third part: the coarse frequency estimate for the windows whose FIC success counter is low (ofdm-processor.cpp:397);
// every other CTA leaves at once
template <bool NCO>
__global__ void __launch_bounds__(OFDM_THREADS, 5)
find_coarse_kernel(DevTables tb, SyncParams p)
{
    extern __shared__ __align__(16) unsigned char smraw[];
    SyncSmem& sm = *reinterpret_cast<SyncSmem*>(smraw);
    const int t = threadIdx.x, f = blockIdx.x;
    if (p.active && !p.active[f]) return;
    const int result = p.index_out[f];
    if (result < 0 || p.fic_ratio[f] * 10 >= 50) return;      // CTA-uniform
    const float2* src = p.iq + (int64_t)f * p.stride + p.win_start[f];
    const Nco nco = make_nco((NCO && p.nco) ? p.nco[2 * f] : 0, (NCO && p.nco) ? p.nco[2 * f + 1] : 0);
    const XIdx xi = make_xidx(t);
    coarse_estimate(tb, sm, src, result, nco, xi, t, p.freqsync, &p.coarse_out[f]);
}

} // namespace

// ------------------------------------------------------------------------------------------------------------
template <typename K> static void set_smem(K k, size_t bytes)
{
    // every template instantiation is its own function: set the attribute per launch (it is a cheap host-side call)
    cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    // always the largest shared-memory carve-out: with a smaller one (chosen by the driver from this kernel's own footprint) the CTAs of
    // the other lane's kernels cannot be placed beside this kernel's on the same SM even when registers and bytes would allow it
    cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared);
}

namespace {
__global__ void osc_verify_kernel(DevTables tb, int32_t* count)
{
    const int m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= INPUT_RATE) return;
    const float2 a = osc_onthefly(tb, m), b = tb.osc[m];
    if (__float_as_uint(a.x) != __float_as_uint(b.x) || __float_as_uint(a.y) != __float_as_uint(b.y)) atomicAdd(count, 1);
}
} // namespace

int launch_osc_verify(const DevTables& tb, cudaStream_t st)
{
    int32_t* d = nullptr;
    if (cudaMalloc((void**)&d, sizeof(int32_t)) != cudaSuccess) return -1;
    cudaMemsetAsync(d, 0, sizeof(int32_t), st);
    osc_verify_kernel<<<(INPUT_RATE + 255) / 256, 256, 0, st>>>(tb, d);
    int32_t h = -1;
    if (cudaMemcpyAsync(&h, d, sizeof h, cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess) h = -1;
    cudaFree(d);
    return h;
}

void launch_ofdm_demod(const DevTables& tb, const OfdmParams& p_in, int fft_mode, cudaStream_t st)
{
    OfdmParams p = p_in;
    if (p.tail_groups < 1 || 75 % p.tail_groups) { p.tail_groups = 1; }
    if (p.n_full < 0 || p.n_full > p.n_frames || p.tail_groups == 1) p.n_full = p.n_frames;
    if (p.fc_pitch < 1) p.fc_pitch = p.groups > p.tail_groups ? p.groups : p.tail_groups;
    const size_t sm = sizeof(DemodSmem);
    const dim3 grid(p.n_full * p.groups + (p.n_frames - p.n_full) * p.tail_groups), block(OFDM_THREADS);
    const bool tap = p.r1 != nullptr, fast = p.nco_fast != 0 && p.nco != nullptr;
#define LAUNCH(E, T, F, W, C) do { set_smem(ofdm_demod_kernel<E, T, F, W, C>, sm); ofdm_demod_kernel<E, T, F, W, C><<<grid, block, sm, st>>>(tb, p); } while (0)
#define LAUNCH_C(E, T, F, W) do { if (p.clock) LAUNCH(E, T, F, W, true); else LAUNCH(E, T, F, W, false); } while (0)
#define LAUNCH_W(E, T, F) do { if (p.weighted) LAUNCH_C(E, T, F, true); else LAUNCH_C(E, T, F, false); } while (0)
#define LAUNCH_F(E, T) do { if (fast) LAUNCH_W(E, T, true); else LAUNCH_W(E, T, false); } while (0)
    if (fft_mode == 0) { if (tap) LAUNCH_F(true, true); else LAUNCH_F(true, false); }
    else { if (tap) LAUNCH_F(false, true); else LAUNCH_F(false, false); }
#undef LAUNCH_F
#undef LAUNCH_W
#undef LAUNCH_C
#undef LAUNCH
}

// how many frames of a launch of n frames (one CTA per frame) to cut into short CTAs: about half a residency's worth, so that the
// short CTAs fill the slots the long ones leave as they finish (0 when the launch is too small for that to matter)
int ofdm_tail_frames(int n_frames)
{
    static int resident = 0;
    if (!resident) {
        int dev = 0, sms = 0, per_sm = 0;
        cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        set_smem(ofdm_demod_kernel<true, false, false, false, false>, sizeof(DemodSmem));
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, ofdm_demod_kernel<true, false, false, false, false>, OFDM_THREADS, sizeof(DemodSmem));
        resident = sms * (per_sm > 0 ? per_sm : 1);
    }
    if (n_frames < 2 * resident) return 0;
    return resident / 2;
}

void launch_tii_spectra(const DevTables& tb, const float2* iq, int64_t stride, const int64_t* prs_start, const int32_t* nco_frame, const int32_t* active,
                        const float2* nulls, float2* out, int n, cudaStream_t st)
{
    tii_spectra_kernel<<<2 * n, OFDM_THREADS, sizeof(OfdmSmem), st>>>(tb, iq, stride, prs_start, nco_frame, active, nulls, out);
}

void launch_coarse(const DevTables& tb, const float2* iq, int64_t stride, const int64_t* prs_start, int n, int freqsync, int32_t* out, cudaStream_t st)
{
    set_smem(coarse_kernel, sizeof(SyncSmem));
    coarse_kernel<<<n, OFDM_THREADS, sizeof(SyncSmem), st>>>(tb, iq, stride, prs_start, freqsync, out);
}

// part: 0 transforms -> magnitudes, 1 placement search -> index, 2 coarse estimate where the FIC counter asks for it, -1 all three
// Time sync always uses the exact arithmetic, whatever the context's fft_mode: its integer result feeds the closed loop.
// excised (or nullptr): the transforms excise interferers (DABB_ACQ_ROBUST) and record the zeroed bins per window
void launch_find_index(const DevTables& tb, const SyncParams& p, cudaStream_t st, int part, int32_t* excised)
{
    const dim3 grid(p.n), block(OFDM_THREADS);
    const bool nco = p.nco != nullptr;
    if ((part < 0 || part == 0) && excised) {
        const size_t sm = sizeof(OfdmSmem);
        if (nco) { set_smem(find_index_excise_kernel<true>, sm); find_index_excise_kernel<true><<<grid, block, sm, st>>>(tb, p, excised); }
        else { set_smem(find_index_excise_kernel<false>, sm); find_index_excise_kernel<false><<<grid, block, sm, st>>>(tb, p, excised); }
    } else if (part < 0 || part == 0) {
        const size_t sm = sizeof(OfdmSmem);
        if (nco) { set_smem(find_index_kernel<true>, sm); find_index_kernel<true><<<grid, block, sm, st>>>(tb, p); }
        else { set_smem(find_index_kernel<false>, sm); find_index_kernel<false><<<grid, block, sm, st>>>(tb, p); }
    }
    if (part < 0 || part == 1) {
        if (p.placement == 0) {
            cudaFuncSetAttribute(find_search_tbp_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared);
            find_search_tbp_kernel<<<(p.n + OFDM_THREADS / 32 - 1) / (OFDM_THREADS / 32), block, 0, st>>>(p);
        } else {
            cudaFuncSetAttribute(find_search_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared);
            find_search_kernel<<<grid, block, 0, st>>>(p);
        }
    }
    if ((part < 0 || part == 2) && p.coarse_out) {
        const size_t sc = sizeof(SyncSmem);
        if (nco) { set_smem(find_coarse_kernel<true>, sc); find_coarse_kernel<true><<<grid, block, sc, st>>>(tb, p); }
        else { set_smem(find_coarse_kernel<false>, sc); find_coarse_kernel<false><<<grid, block, sc, st>>>(tb, p); }
    }
}

} // namespace dabb
