// viterbi_core.cuh — per-thread K=7 rate-1/4 Viterbi add-compare-select, one codeword per thread, all 64 path
// metrics in 32 registers as packed signed 16-bit pairs (VIADDMNMX.S16x2 on sm_90a).
//
// Semantics reproduced from the reference (backend/viterbi.cpp): polynomials 0155 0117 0123 0155 (:35-36); branch
// metric = sum_k (sym_k or 255 - sym_k) (:248-261); new[2i] = min(old[i] + m, old[i+32] + 1020 - m),
// new[2i+1] = min(old[i] + 1020 - m, old[i+32] + m) with the decision bit (m_a - m_b) > 0, i.e. ties keep the old[i]
// branch (:263-275); decision bit n of step t belongs to new state n (:276-278); start metrics 63 / 0 (:342-354).
// The reference's renormalisation (:104-120) subtracts a uniform value and cannot change a decision; here the
// minimum is subtracted every 24 steps so that metrics stay inside [0, 32767).
//
// Register layout.  Layout L_b pairs, in one 32-bit register, the two states that differ in bit b (low half: bit
// b = 0).  An ACS step maps L_b -> L_{b+1} with plain SIMD (two butterflies per pair of registers, no data movement);
// L_5 pairs butterfly partners, so that step swaps halves with PRMT and lands in L_0.  Six consecutive steps
// (nsteps = nbits + 6 is always a multiple of 6) are unrolled with compile-time register indices.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define VIT_HD __host__ __device__ __forceinline__
#else
#define VIT_HD inline
#endif

namespace dabb {

#define VIT_POLY0 0155
#define VIT_POLY1 0117
#define VIT_POLY2 0123   /* fourth polynomial == first */

VIT_HD constexpr int vit_parity(unsigned x) { x ^= x >> 4; x ^= x >> 2; x ^= x >> 1; return (int)(x & 1u); }
// branch pattern of butterfly i (0..31): bit k = parity((2i) & poly_k), k = 0,1,2 (poly_3 == poly_0)
VIT_HD constexpr int vit_pat(int i) { return vit_parity((2 * i) & VIT_POLY0) | (vit_parity((2 * i) & VIT_POLY1) << 1) | (vit_parity((2 * i) & VIT_POLY2) << 2); }
VIT_HD constexpr int vit_remove_bit(int s, int b) { return ((s >> (b + 1)) << b) | (s & ((1 << b) - 1)); }
VIT_HD constexpr int vit_insert_zero(int j, int b) { return ((j >> b) << (b + 1)) | (j & ((1 << b) - 1)); }

// per-half signed 16-bit minimum; pl/ph = (a_half <= b_half)
VIT_HD uint32_t vibmin16(uint32_t a, uint32_t b, bool& ph, bool& pl)
{
#if defined(__CUDA_ARCH__)
    return __vibmin_s16x2(a, b, &ph, &pl);
#else
    const int16_t al = (int16_t)(a & 0xFFFF), ah = (int16_t)(a >> 16), bl = (int16_t)(b & 0xFFFF), bh = (int16_t)(b >> 16);
    pl = al <= bl; ph = ah <= bh;
    return (uint32_t)(uint16_t)(pl ? al : bl) | ((uint32_t)(uint16_t)(ph ? ah : bh) << 16);
#endif
}
VIT_HD uint32_t swap16(uint32_t r)
{
#if defined(__CUDA_ARCH__)
    return __byte_perm(r, 0, 0x1032);
#else
    return (r >> 16) | (r << 16);
#endif
}
VIT_HD uint32_t vminu16x2(uint32_t a, uint32_t b)
{
#if defined(__CUDA_ARCH__)
    return __vminu2(a, b);
#else
    const uint32_t al = a & 0xFFFF, ah = a >> 16, bl = b & 0xFFFF, bh = b >> 16;
    return (al < bl ? al : bl) | ((ah < bh ? ah : bh) << 16);
#endif
}

// per-half signed 16-bit minimum (SASS: VIMNMX.S16x2)
VIT_HD uint32_t vmin16(uint32_t a, uint32_t b)
{
#if defined(__CUDA_ARCH__)
    uint32_t r; asm("min.s16x2 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r;
#else
    bool ph, pl; return vibmin16(a, b, ph, pl);
#endif
}
// per-half min(a + b, c), the sums wrapping within their half (SASS: VIADDMNMX.S16x2)
VIT_HD uint32_t vaddmin16(uint32_t a, uint32_t b, uint32_t c)
{
#if defined(__CUDA_ARCH__)
    return __viaddmin_s16x2(a, b, c);
#else
    const uint32_t s = ((a + b) & 0xFFFFu) | (((a >> 16) + (b >> 16)) << 16);
    return vmin16(s, c);
#endif
}
// bytes (sign(t1 bit 15), sign(t2 bit 15), sign(t1 bit 31), sign(t2 bit 31)) as 0x00 / 0xFF: PRMT in sign-replicating mode
VIT_HD uint32_t vit_signbytes(uint32_t t1, uint32_t t2)
{
#if defined(__CUDA_ARCH__)
    uint32_t r;        // generic prmt: selector nibble = byte index 0..7 of {t2, t1} | 8 = replicate that byte's sign bit
    asm("prmt.b32 %0, %1, %2, 0xFBD9;" : "=r"(r) : "r"(t1), "r"(t2));
    return r;
#else
    return ((t1 >> 15) & 1u ? 0xFFu : 0u) | ((t2 >> 15) & 1u ? 0xFF00u : 0u) | ((t1 >> 31) ? 0xFF0000u : 0u) | ((t2 >> 31) ? 0xFF000000u : 0u);
#endif
}
// where vit_acs<B> stores the decision of NEW state n: bit position 0..63 in the step's decision pair (x = bits 0..31, y = 32..63)
template <int B> VIT_HD uint32_t vit_dec_pos(uint32_t n)
{
    if constexpr (B < 5) {
        const uint32_t h = n >> 1;                                                    // butterfly index with its bit B = lane bit 1
        const uint32_t j = ((h >> (B + 1)) << B) | (h & ((1u << B) - 1u));           // ... removed: group 0..15
        return (j & 7u) | ((n & 1u) << 3) | (((n >> (B + 1)) & 1u) << 4) | ((j >> 3) << 5);
    } else {
        const uint32_t g = n >> 2;                                                    // lanes: 4g, 4g + 2, 4g + 1, 4g + 3
        return (g & 7u) | (((n >> 1) & 1u) << 3) | ((n & 1u) << 4) | ((g >> 3) << 5);
    }
}

// branch metrics for the eight patterns from one step's four symbols (bytes s0..s3 of w, each 0..255)
VIT_HD void vit_metrics(uint32_t w, uint32_t E[8])
{
    const uint32_t s0 = w & 0xFF, s1 = (w >> 8) & 0xFF, s2 = (w >> 16) & 0xFF, s3 = w >> 24;
    const uint32_t A = s0 + s3, B = s1, C = s2;
    const uint32_t a[2] = {A, 510u - A}, b[2] = {B, 255u - B}, c[2] = {C, 255u - C};
#pragma unroll
    for (int p = 0; p < 8; p++) E[p] = a[p & 1] + b[(p >> 1) & 1] + c[(p >> 2) & 1];
}

// The eight packed branch-metric words of one step for a layout whose SIMD partner differs by pattern DELTA:
// MC[p] = E[p] | E[p ^ DELTA] << 16.  Built directly in packed form: with A = s0 + s3, B = s1, C = s2 (one dot-product
// instruction each) the pair (x, x) or (x, max - x) is one multiply-add, its complement (max, max) - pair one subtract, and
// MC[p] = PA[p & 1] + PB[(p >> 1) & 1] + PC[p >> 2] (no carry between the halves: every sum is <= 1020).
// KM[p] = MC[p] + KOFF, the decision offsets of vit_acs (KOFF's halves <= 0x8000: every half of KM stays below 0x10000).
template <int DELTA, uint32_t KOFF> VIT_HD void vit_mc(uint32_t w, uint32_t (&MC)[8], uint32_t (&KM)[8])
{
#if defined(__CUDA_ARCH__)
    const uint32_t A = __dp4a(w, 0x01000001u, 0u), B = __dp4a(w, 0x00000100u, 0u), C = __dp4a(w, 0x00010000u, 0u);
#else
    const uint32_t A = (w & 0xFF) + (w >> 24), B = (w >> 8) & 0xFF, C = (w >> 16) & 0xFF;
#endif
    // (x, x) = x * 0x10001;  (x, max - x) = x * (1 - 65536) + (max << 16)   (mod 2^32)
    const uint32_t PA0 = (DELTA & 1) ? A * 0xFFFF0001u + (510u << 16) : A * 0x00010001u;
    const uint32_t PB0 = (DELTA & 2) ? B * 0xFFFF0001u + (255u << 16) : B * 0x00010001u;
    const uint32_t PC0 = (DELTA & 4) ? C * 0xFFFF0001u + (255u << 16) : C * 0x00010001u;
    const uint32_t PA[2] = {PA0, 0x01FE01FEu - PA0}, PB[2] = {PB0, 0x00FF00FFu - PB0}, PC[2] = {PC0, 0x00FF00FFu - PC0};
    const uint32_t PK[2] = {PC[0] + KOFF, PC[1] + KOFF};
    uint32_t AB[4];
#pragma unroll
    for (int q = 0; q < 4; q++) AB[q] = PA[q & 1] + PB[q >> 1];
#pragma unroll
    for (int p = 0; p < 8; p++) { MC[p] = AB[p & 3] + PC[p >> 2]; KM[p] = AB[p & 3] + PK[p >> 2]; }
}

// The multiplicative inverse of 255 modulo 2^32.  A word of 0x00 / 0xFF bytes is 255 x the same word with 0x00 / 0x01 bytes, so
// bytes * (VIT_INV255 << g) is that word shifted to bit g of every byte: one IMAD (FMA pipe) masks and places four decisions, and
// summing such terms for distinct g is the OR of them.
constexpr uint32_t VIT_INV255 = 0xFEFEFEFFu;

// One ACS step from layout L_B to L_{(B+1)%6}.  Q: 32 packed metric registers; dlo/dhi: decision bits of new states
// 0..31 / 32..63.
template <int B> VIT_HD void vit_acs(uint32_t (&Q)[32], const uint32_t w, uint32_t& dlo, uint32_t& dhi)
{
    uint32_t N[32];
    // A packed minimum min(a + m, c) of candidate pairs is one VIADDMNMX: of the four candidate sums of a butterfly pair only the
    // two that are a minimum's second operand are formed.
    // Decisions without predicates.  For a packed pair (a, b) of candidate metrics (every half in [0, 0x7FFF]) t = a + 0x7FFF7FFF - b has
    // bit 15 / 31 set exactly where b wins strictly ((a - b) > 0: ties keep the a = old[i] branch, viterbi.cpp:263-275) and no carry
    // crosses the halves.  With a = q + MC[p], that is t = q + KM[p] - b: one IADD3 from the old metric and the candidate b the
    // minimum needs anyway, so a is never formed.  One PRMT in sign-replicating mode turns the two sign bits of two such words
    // into four 0x00 / 0xFF bytes, and one IMAD with VIT_INV255 << g moves them to bit g of every byte and adds them into the step's
    // decision word.  (A predicated form - VIMNMX with two predicate outputs + two predicated adds - made the scheduler park
    // predicates in general registers: ~45 extra instructions per step.)
    // Decision layout of a step: group g (0..15) = the two packed minima that share their input registers, byte lane l (0..3) as listed
    // below; decision bit at word g >> 3, bit 8 l + (g & 7) (vit_dec_pos<B> is the inverse map for the traceback).
    uint32_t W[2] = {0u, 0u};
#define VIT_PUT(g, t1, t2) do { W[(g) >> 3] += vit_signbytes(t1, t2) * (VIT_INV255 << ((g) & 7)); } while (0)
    if constexpr (B < 5) {
        constexpr int delta = vit_pat(1 << B);   // pattern change when butterfly bit B flips
        uint32_t MC[8], KM[8];
        vit_mc<delta, 0x7FFF7FFFu>(w, MC, KM);
#pragma unroll
        for (int j = 0; j < 16; j++) {
            const int ilo = vit_insert_zero(j, B);            // butterfly with bit B = 0; its SIMD partner is ilo + (1<<B)
            const int ra = vit_remove_bit(ilo, B), rb = vit_remove_bit(ilo + 32, B);
            const int p = vit_pat(ilo);
            // candidates m0 = Q[ra] + MC[p], m1 = Q[rb] + MC[p ^ 7], m2 = Q[ra] + MC[p ^ 7], m3 = Q[rb] + MC[p]
            const uint32_t m1 = Q[rb] + MC[p ^ 7], m3 = Q[rb] + MC[p];
            const int ne = 2 * ilo;                           // new states: (ne, ne + (2 << B)) from (m0, m1), (ne + 1, ne + 1 + (2 << B)) from (m2, m3)
            N[vit_remove_bit(ne, B + 1)] = vaddmin16(Q[ra], MC[p], m1);
            N[vit_remove_bit(ne + 1, B + 1)] = vaddmin16(Q[ra], MC[p ^ 7], m3);
            VIT_PUT(j, Q[ra] + KM[p] - m1, Q[ra] + KM[p ^ 7] - m3);   // lanes: ne, ne + 1, ne + (2 << B), ne + 1 + (2 << B)
        }
    } else {
        // L_5: register i = (old[i], old[i+32]); result register i = (new[2i], new[2i+1]) = layout L_0.  With m = E[p] of butterfly i,
        // a = Q[i] + (m, m) = (old[i] + m, old[i+32] + m) and b = swap(Q[i]) + (1020 - m, 1020 - m) = (old[i+32] + 1020 - m, old[i] + 1020 - m)
        // hold the candidates of new[2i] in their low and of new[2i+1] in their high halves: N[i] = min(a, b).  In the high half the old[i]
        // candidate is b's, so t = a - b + 0x80007FFF has bit 31 set where old[i+32] does NOT win strictly; XOR-ing the decision words
        // with 0xFFFF0000 (byte lanes 2, 3) turns those bits into decisions.
        uint32_t EE[8], KE[8];
        vit_mc<0, 0x80007FFFu>(w, EE, KE);                     // EE[p] = (E[p], E[p]); EE[p ^ 7] = (1020 - E[p], 1020 - E[p])
#pragma unroll
        for (int g = 0; g < 16; g++) {
            uint32_t t[2];
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const int i = 2 * g + h, p = vit_pat(i);
                const uint32_t b = swap16(Q[i]) + EE[p ^ 7];
                N[i] = vaddmin16(Q[i], EE[p], b);              // (new[2i], new[2i+1])
                t[h] = Q[i] + KE[p] - b;
            }
            VIT_PUT(g, t[0], t[1]);                             // lanes: 4g, 4g + 2, 4g + 1, 4g + 3
        }
        W[0] ^= 0xFFFF0000u; W[1] ^= 0xFFFF0000u;
    }
#undef VIT_PUT
    dlo = W[0]; dhi = W[1];
#pragma unroll
    for (int r = 0; r < 32; r++) Q[r] = N[r];
}

// start metrics in layout L_0: register r = (state 2r, state 2r+1); 63 everywhere, 0 for state 0
VIT_HD void vit_init(uint32_t (&Q)[32])
{
#pragma unroll
    for (int r = 0; r < 32; r++) Q[r] = 63u | (63u << 16);
    Q[0] = 0u | (63u << 16);
}

// subtract the minimum over all 64 states from every state (uniform shift: no decision changes)
VIT_HD void vit_normalize(uint32_t (&Q)[32])
{
    uint32_t m = Q[0];
#pragma unroll
    for (int r = 1; r < 32; r++) m = vminu16x2(m, Q[r]);
    const uint32_t lo = m & 0xFFFF, hi = m >> 16;
    const uint32_t mn = lo < hi ? lo : hi;
    const uint32_t sub = mn | (mn << 16);
#pragma unroll
    for (int r = 0; r < 32; r++) Q[r] -= sub;
}

// six steps: words w[0..5] hold the symbols, dec[2*s], dec[2*s+1] receive the decision words
VIT_HD void vit_six_steps(uint32_t (&Q)[32], const uint32_t w[6], uint32_t dec[12])
{
    vit_acs<0>(Q, w[0], dec[0], dec[1]);
    vit_acs<1>(Q, w[1], dec[2], dec[3]);
    vit_acs<2>(Q, w[2], dec[4], dec[5]);
    vit_acs<3>(Q, w[3], dec[6], dec[7]);
    vit_acs<4>(Q, w[4], dec[8], dec[9]);
    vit_acs<5>(Q, w[5], dec[10], dec[11]);
}

// ---- de-puncturing inside the decoder kernel -------------------------------------------------------------------------------
// The kernel reads the PUNCTURED softbits of a codeword (consecutive bytes) and expands them itself.  Everything about the expansion
// but the data is the same for all codewords of a launch: per trellis step a byte selector over an 8-byte window of the stream, a
// byte mask (punctured positions -> softbit 0) and whether the window moves on by one word afterwards.
struct vit_u2 { uint32_t x, y; };                  // layout of uint2
constexpr int VIT_STAGE_STEPS = 24;                // steps per staging unit: <= 96 softbits + 15 bytes of alignment slack < 128

// symbol word of one step: four softbits picked from the window (w0 = lower addresses), punctured -> 0, then s + 127 = (s ^ 0x80) - 1
// per byte (softbits are >= -127, so no byte borrows): the reference's clamp(s + 127, 0, 255) (viterbi.cpp:232-237)
VIT_HD uint32_t vit_expand_step(uint32_t w0, uint32_t w1, uint32_t sel, uint32_t mask)
{
#if defined(__CUDA_ARCH__)
    const uint32_t x = __byte_perm(w0, w1, sel);
#else
    const uint64_t win = (uint64_t)w0 | ((uint64_t)w1 << 32);
    uint32_t x = 0;
    for (int k = 0; k < 4; k++) x |= (uint32_t)((win >> (8 * ((sel >> (4 * k)) & 7))) & 0xFF) << (8 * k);
#endif
    return ((x & mask) ^ 0x80808080u) - 0x01010101u;
}

// Expansion tables from a de-puncturing map (4 entries per trellis step: >= 0 present - the punctured softbits are consumed in
// order - or < 0 punctured).  steps[t] = {selector | advance flag << 16, mask}; stage_off[s] = index of the first softbit consumed
// by stage s (VIT_STAGE_STEPS steps; the kernel stages the aligned 128 bytes from there), stage_off[nstages] = total consumed.
template <class StepVec, class OffVec>
inline void build_vit_tables(const int16_t* map, int nsteps, StepVec& steps, OffVec& stage_off)
{
    steps.clear(); stage_off.clear();
    int cursor = 0, pos = 0;
    for (int t = 0; t < nsteps; t++) {
        if (t % VIT_STAGE_STEPS == 0) { stage_off.push_back((uint32_t)cursor); pos = cursor & 3; }
        uint32_t sel = 0, mask = 0; int n = 0;
        for (int k = 0; k < 4; k++)
            if (map[4 * t + k] >= 0) { sel |= (uint32_t)(pos + n) << (4 * k); mask |= 0xFFu << (8 * k); n++; cursor++; }
        pos += n;
        uint32_t adv = 0;
        if (pos >= 4) { pos -= 4; adv = 1; }
        typename StepVec::value_type e; e.x = sel | (adv << 16); e.y = mask;
        steps.push_back(e);
    }
    stage_off.push_back((uint32_t)cursor);
}

// ---- traceback ------------------------------------------------------------------------------------------------------------------
// From state 0 after the last step, skipping the 6 tail steps (viterbi.cpp:313-339): bit = decision[t + 6][state],
// state = (state >> 1) | (bit << 5).  The decoded bit enters the state at bit 5 and moves down one position per step, so after six
// steps the state IS the six decoded bits, earliest first from bit 5: the output is assembled six bits at a time.
// One call handles 24 steps: d[k] = decision words of the times T0 + k (T0 + 23 first); acc[3] collects a 96-bit big-endian string
// of the times tb .. tb + 95 (acc[2] bit 31 = time tb); q = which quarter (T0 = tb + 24 q).
template <int PH> VIT_HD void vit_tb_step(uint32_t& state, const vit_u2& d)
{
    // decision of the state reached by step PH (mod 6) of a six-step group: forward step s used vit_acs<s % 6>
    const uint32_t pos = vit_dec_pos<PH>(state);
    const uint32_t word = (pos & 32u) ? d.y : d.x;
#if defined(__CUDA_ARCH__)
    const uint32_t rot = __funnelshift_r(word, word, pos - 5u);       // bit (pos & 31) of the word rotated to bit 5
#else
    const uint32_t sh = (pos - 5u) & 31u;
    const uint32_t rot = sh ? ((word >> sh) | (word << (32 - sh))) : word;
#endif
    state = (rot & 32u) | (state >> 1);
}
template <int Q24> VIT_HD void vit_traceback24(uint32_t& state, const vit_u2 (&d)[24], uint32_t (&acc)[3])
{
    // d[k] belongs to trellis step tb + 24 Q24 + k + 6, a multiple of 6 plus k: its layout phase is k mod 6
#pragma unroll
    for (int h = 3; h >= 0; h--) {
        vit_tb_step<5>(state, d[6 * h + 5]); vit_tb_step<4>(state, d[6 * h + 4]); vit_tb_step<3>(state, d[6 * h + 3]);
        vit_tb_step<2>(state, d[6 * h + 2]); vit_tb_step<1>(state, d[6 * h + 1]); vit_tb_step<0>(state, d[6 * h + 0]);
        // state = the bits of the times T .. T+5 (T = tb + 24 Q24 + 6 h), time T at bit 5
        const int lo = 96 - (24 * Q24 + 6 * h + 6);        // offset of time T+5 in the 96-bit string (0 = time tb + 95)
        acc[lo >> 5] |= state << (lo & 31);
        if ((lo & 31) > 26) acc[(lo >> 5) + 1] |= state >> (32 - (lo & 31));
    }
}
// the 32 decoded bits of acc (first time at bit 31) -> output word: bit t MSB-first in byte t / 8, bytes in memory order
VIT_HD uint32_t vit_pack_be(uint32_t a)
{
#if defined(__CUDA_ARCH__)
    return __byte_perm(a, 0, 0x0123);
#else
    return (a >> 24) | ((a >> 8) & 0xFF00u) | ((a << 8) & 0xFF0000u) | (a << 24);
#endif
}

// soft bit (int8, 0 = punctured) -> decoder symbol clamp(s + 127, 0, 255)  (viterbi.cpp:232-237)
VIT_HD uint32_t vit_sym(int s) { int v = s + 127; return (uint32_t)(v < 0 ? 0 : (v > 255 ? 255 : v)); }

} // namespace dabb
