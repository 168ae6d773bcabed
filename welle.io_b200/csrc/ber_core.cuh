// ber_core.cuh — channel bit errors of one codeword: the decoded bits are convolutionally re-encoded and compared, at the transmitted
// positions, with the signs of the punctured softbits the decoder read.  Compiles for the device (ber.cu) and as host C++
// (tests/host_emul/emul_ber.cpp).
//
// A codeword of nbits decoded bits has 4 (nbits + 6) mother-code bits.  They are counted in chunks of 32 (8 trellis steps): every (L, PI)
// block of a protection profile covers L x 128 mother-code bits, so each of its 4 L chunks is punctured with the same 32-bit vector PI and
// reads popcount(PI) consecutive softbits; the 24 tail bits (6 steps, 12 transmitted) are one more chunk.  Per chunk: the expected code
// bits come from a 14-bit window of the decoded bits, the softbits' signs and zeros are deposited onto the PI positions, and XOR +
// popcount give the errors.  A softbit s > 0 votes for a 1 (the decoder's convention), s == 0 is an erasure.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define BER_HD __host__ __device__ __forceinline__
#else
#define BER_HD inline
#endif

namespace dabb_ber {

constexpr int MAX_BLOCKS = 5;                   // up to four (L, PI) blocks, then the tail
constexpr uint32_t TAIL_MASK = 0x00333333u;     // PI_TAIL 1100 x 6 over the 6 tail steps
// the four generator polynomials (octal 155, 117, 123, 155) bit-reversed over 7 bits, so that code bit k of step t0 + d is the parity of
// rev_poly(k) & (V >> d), V bit p = decoded bit t0 - 6 + p
BER_HD constexpr uint32_t rev_poly(int k) { return k == 1 ? 0171u : (k == 2 ? 0145u : 0133u); }

// a run of chunks punctured with one vector
struct Block {
    int32_t first_chunk;    // index of the run's first chunk in the codeword
    int32_t first_soft;     // fragment softbit of the run's first transmitted bit
    uint32_t mask;          // bit i: mother-code bit 32 chunk + i is transmitted
    int32_t pop;            // popcount(mask): softbits per chunk
    uint32_t mv[5];         // the masks of the bit deposit onto `mask` (expand_masks)
};

// the puncturing of one protection profile (or of the FIC) as the counting reads it
struct Profile {
    int32_t nbits;          // decoded bits per codeword (a multiple of 32)
    int32_t nchunks;        // nbits / 8 + 1: the last chunk is the tail
    int32_t in_bits;        // transmitted bits = softbits the decoder reads
    int32_t nblk;           // blocks in use, the tail included
    const uint32_t* prbs;   // energy-dispersal words packed like the decoder output (bit t in byte t / 8, MSB first)
    Block blk[MAX_BLOCKS];
};

BER_HD int popc(uint32_t x)
{
#if defined(__CUDA_ARCH__)
    return __popc(x);
#else
    return __builtin_popcount(x);
#endif
}

// Hacker's Delight 7-5 (expand): the five move masks that deposit the low popcount(m) bits of a word onto the set bits of m
BER_HD void expand_masks(uint32_t m, uint32_t mv[5])
{
    uint32_t mk = ~m << 1;
    for (int i = 0; i < 5; i++) {
        uint32_t mp = mk ^ (mk << 1);
        mp ^= mp << 2; mp ^= mp << 4; mp ^= mp << 8; mp ^= mp << 16;
        const uint32_t v = mp & m;
        mv[i] = v;
        m = (m ^ v) | (v >> (1 << i));
        mk &= ~mp;
    }
}
BER_HD uint32_t expand(uint32_t x, uint32_t m, const uint32_t mv[5])
{
#pragma unroll
    for (int i = 4; i >= 0; i--) x = (x & ~mv[i]) | ((x << (1 << i)) & mv[i]);
    return x & m;
}

// a profile from its blocks: L[k] x 128 mother-code bits punctured with the 32-bit vector mask[k] (bit i = PI entry i); blocks with
// L = 0 are skipped.  Returns the transmitted bits per codeword.
inline int build_profile(int nblk, const int* L, const uint32_t* mask, int nbits, Profile& p)
{
    p = Profile{};
    p.nbits = nbits; p.nchunks = nbits / 8 + 1;
    int chunk = 0, soft = 0, n = 0;
    auto add = [&](int chunks, uint32_t m) {
        Block& b = p.blk[n++];
        b.first_chunk = chunk; b.first_soft = soft; b.mask = m; b.pop = popc(m);
        expand_masks(m, b.mv);
        chunk += chunks; soft += chunks * b.pop;
    };
    for (int k = 0; k < nblk; k++) if (L[k] > 0) add(4 * L[k], mask[k]);
    add(1, TAIL_MASK);
    p.nblk = n; p.in_bits = soft;
    return soft;
}

// bit q of a byte flag word: byte q of w satisfies the test
BER_HD uint32_t flags4(uint32_t bytemask) { return (((bytemask & 0x01010101u) * 0x01020408u) >> 24) & 0xFu; }
BER_HD uint32_t positive4(uint32_t w)
{
#if defined(__CUDA_ARCH__)
    return flags4(__vcmpgts4(w, 0u));
#else
    uint32_t r = 0;
    for (int q = 0; q < 4; q++) r |= (uint32_t)((int8_t)(w >> (8 * q)) > 0) << q;
    return r;
#endif
}
BER_HD uint32_t zero4(uint32_t w)
{
#if defined(__CUDA_ARCH__)
    return flags4(__vcmpeq4(w, 0u));
#else
    uint32_t r = 0;
    for (int q = 0; q < 4; q++) r |= (uint32_t)(((w >> (8 * q)) & 0xFFu) == 0) << q;
    return r;
#endif
}
BER_HD uint32_t brev(uint32_t x)
{
#if defined(__CUDA_ARCH__)
    return __brev(x);
#else
    uint32_t r = 0;
    for (int i = 0; i < 32; i++) r |= ((x >> i) & 1u) << (31 - i);
    return r;
#endif
}
// bit d of an 8-bit value to bit 4 d
BER_HD uint32_t spread4(uint32_t x)
{
    x = (x | (x << 12)) & 0x000F000Fu;
    x = (x | (x << 6)) & 0x03030303u;
    return (x | (x << 3)) & 0x11111111u;
}

// the 32 mother-code bits of the chunk starting at step t0 = 8 j; V bit p = decoded bit t0 - 6 + p (p < 14), 0 outside the codeword
BER_HD uint32_t encode_chunk(uint32_t V)
{
    uint32_t c = 0;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        uint32_t acc = 0;
#pragma unroll
        for (int q = 0; q < 7; q++) if ((rev_poly(k) >> q) & 1u) acc ^= V >> q;
        c |= spread4(acc & 0xFFu) << k;
    }
    return c;
}

struct Counts { uint32_t bits, errors, erasures; };

// chunk j of one codeword.  soft: the codeword's punctured softbits (4-byte aligned, readable 3 bytes past its last one); out: its
// decoded bytes after energy dispersal (nbits / 8 of them); prbs: p.prbs
BER_HD void count_chunk(const Profile& p, int j, const int8_t* soft, const uint8_t* out, Counts& c)
{
    int k = 0;
    for (int i = 1; i < p.nblk; i++) if (j >= p.blk[i].first_chunk) k = i;
    const Block& b = p.blk[k];
    const int off = b.first_soft + (j - b.first_chunk) * b.pop;
    // flags of the softbits [off, off + pop): aligned words, then shifted to the first one
    const uint32_t* w = reinterpret_cast<const uint32_t*>(soft + (off & ~3));
    const int sh = off & 3, nw = (sh + b.pop + 3) >> 2;
    uint64_t P = 0, Z = 0;
    for (int q = 0; q < nw; q++) {
        const uint32_t v = w[q];
        P |= (uint64_t)positive4(v) << (4 * q);
        Z |= (uint64_t)zero4(v) << (4 * q);
    }
    const uint32_t low = b.pop >= 32 ? ~0u : (1u << b.pop) - 1u;      // the chunk's own softbits only
    const uint32_t rx = expand((uint32_t)(P >> sh) & low, b.mask, b.mv), er = expand((uint32_t)(Z >> sh) & low, b.mask, b.mv);
    // decoded bits t0 - 8 .. t0 + 7 as a 16-bit MSB-first word: byte j - 1 and byte j of out ^ prbs (zero outside the codeword)
    const int nbytes = p.nbits >> 3;
    const uint8_t* pr = reinterpret_cast<const uint8_t*>(p.prbs);
    const uint32_t hi = j >= 1 ? (uint32_t)(out[j - 1] ^ pr[j - 1]) : 0u, lo = j < nbytes ? (uint32_t)(out[j] ^ pr[j]) : 0u;
    const uint32_t V = brev((hi << 8) | lo) >> 18;
    const uint32_t code = encode_chunk(V);
    c.bits += (uint32_t)b.pop;
    c.erasures += (uint32_t)popc(er);
    c.errors += (uint32_t)popc((rx ^ code) & b.mask & ~er);
}

} // namespace dabb_ber
