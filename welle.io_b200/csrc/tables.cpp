// tables.cpp — host-side construction of the constant tables the kernels use.
// All values are derived from the ETSI EN 300 401 rules the reference implements; each builder cites the
// reference file:line whose behaviour it reproduces.  (Independent of oracle/: the product never links it.)
#include "common.cuh"
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include "osc_factors.h"
#include <cmath>
#include <cstring>

namespace dabb {

static void fill_twiddles(float2* lay, bool inverse)
{
    // tw[i] = ((float)cos(ph), (float)sin(ph)), ph = -2 pi i / 2048 as a double (libs/kiss_fft/kiss_fft.c:356-364)
    static float2 tw[TU];
    const double pi = 3.141592653589793238462643383279502884197169399375105820974944;
    for (int i = 0; i < TU; i++) {
        double ph = -2 * pi * i / TU;
        if (inverse) ph *= -1;
        tw[i].x = (float)cos(ph);
        tw[i].y = (float)sin(ph);
    }
    memset(lay, 0, sizeof(float2) * TwLayout::TOTAL);
    for (int j = 0; j < 3; j++) lay[TwLayout::A3 + j] = tw[256 * (j + 1)];
    for (int j = 0; j < 3; j++) for (int k = 0; k < 8; k++) lay[TwLayout::B2 + 8 * j + k] = tw[64 * k * (j + 1)];
    for (int j = 0; j < 3; j++) for (int k = 0; k < 32; k++) lay[TwLayout::B3 + 32 * j + k] = tw[16 * k * (j + 1)];
    for (int j = 0; j < 3; j++) for (int k = 0; k < 128; k++) lay[TwLayout::C4 + 128 * j + k] = tw[4 * k * (j + 1)];
    for (int j = 0; j < 3; j++) for (int k = 0; k < 512; k++) lay[TwLayout::C5 + 512 * j + k] = tw[k * (j + 1)];
}

// ETSI Table 39 / 38 (Mode I) — the phase reference symbol (phasetable.cpp:24-75,138-183)
// softbit staging layout of ofdm_demod_kernel (scripts/opt_scatter_layout.py; used in build_host_tables below)
static const uint8_t kChunkSlot[192] = {
    13, 182, 24, 35, 33, 76, 63, 186, 165, 131, 25, 92, 151, 128, 146, 38, 31, 20, 161, 48, 101, 171, 114, 54, 107, 72, 12, 185, 22, 181, 90, 167,
    50, 8, 140, 51, 125, 7, 6, 41, 124, 139, 18, 16, 65, 94, 119, 141, 95, 142, 189, 84, 169, 75, 58, 144, 132, 83, 121, 45, 88, 127, 66, 86,
    108, 39, 43, 150, 40, 133, 122, 49, 2, 79, 4, 153, 155, 62, 32, 149, 154, 112, 89, 100, 71, 117, 99, 126, 148, 80, 9, 85, 174, 34, 175, 91,
    106, 172, 29, 30, 81, 184, 147, 159, 27, 152, 73, 28, 190, 53, 98, 47, 129, 60, 74, 59, 23, 37, 96, 118, 135, 104, 67, 109, 156, 42, 46, 113,
    77, 36, 111, 130, 110, 123, 160, 137, 55, 105, 93, 56, 68, 187, 178, 158, 179, 97, 5, 138, 180, 136, 183, 14, 3, 134, 15, 64, 61, 116, 57, 170,
    19, 78, 168, 177, 162, 69, 87, 188, 44, 103, 0, 166, 26, 17, 11, 21, 143, 82, 70, 1, 176, 163, 52, 157, 10, 191, 115, 120, 102, 173, 145, 164,
};
static const uint8_t kChunkSwap[192] = {
    1, 1, 0, 0, 0, 1, 0, 0, 1, 0, 1, 0, 1, 0, 0, 0, 1, 1, 0, 0, 1, 0, 0, 1, 1, 1, 1, 0, 1, 0, 0, 1,
    1, 0, 1, 1, 1, 1, 0, 0, 0, 1, 0, 1, 0, 1, 0, 0, 1, 1, 0, 0, 1, 1, 0, 0, 0, 1, 1, 1, 1, 1, 1, 0,
    1, 1, 1, 0, 1, 0, 0, 1, 1, 1, 1, 1, 1, 0, 0, 1, 1, 1, 1, 0, 1, 1, 0, 1, 1, 1, 0, 0, 1, 1, 0, 0,
    1, 0, 1, 1, 1, 0, 0, 1, 0, 1, 1, 1, 1, 0, 0, 1, 0, 0, 1, 1, 0, 0, 0, 0, 0, 1, 1, 1, 1, 0, 1, 1,
    1, 1, 1, 1, 0, 1, 1, 1, 0, 0, 0, 0, 1, 1, 0, 0, 1, 1, 0, 1, 1, 0, 0, 1, 1, 1, 0, 0, 1, 0, 0, 1,
    1, 0, 0, 1, 1, 0, 1, 1, 0, 1, 0, 1, 0, 1, 1, 1, 1, 0, 1, 1, 0, 1, 1, 0, 0, 0, 1, 0, 0, 0, 1, 0,
};
static const uint8_t kPrsI[48] = {0,1,2,3,0,1,2,3,0,1,2,3,0,1,2,3,0,1,2,3,0,1,2,3, 0,3,2,1,0,3,2,1,0,3,2,1,0,3,2,1,0,3,2,1,0,3,2,1};
static const uint8_t kPrsN[48] = {1,2,0,1,3,2,2,3,2,1,2,3,1,2,3,3,2,2,2,1,1,3,1,2, 3,1,1,1,2,2,1,0,2,2,3,3,0,2,1,3,3,3,3,0,3,0,1,1};
static const uint8_t kPrsH[4][16] = {{0,2,0,0,0,0,1,1,2,0,0,0,2,2,1,1},{0,3,2,3,0,1,3,0,2,1,2,3,2,3,3,0},
                                      {0,0,0,2,0,2,1,3,2,2,0,2,2,0,1,3},{0,1,2,1,0,3,3,2,2,3,2,1,2,1,3,2}};
static float prs_phi(int k)
{
    int b, kmin;
    if (k < 0) { b = (k + 768) / 32; kmin = -768 + 32 * b; }
    else { b = 24 + (k - 1) / 32; kmin = 1 + 32 * (b - 24); }
    // PhaseTable::get_Phi returns a float: pi/2 * (h + n) evaluated in double then narrowed (phasetable.cpp:172-183)
    return (float)(M_PI / 2.0f * (kPrsH[kPrsI[b]][(k - kmin) & 15] + kPrsN[b]));
}

void build_host_tables(HostTables& t)
{
    fill_twiddles(t.tw_fwd, false);
    fill_twiddles(t.tw_inv, true);
    // the literals of ofdm_core.cuh's tw_a3() must be the table's values
    for (int j = 0; j < 3; j++) {
        const float2 f = tw_a3<false>(j), i = tw_a3<true>(j);
        if (memcmp(&f, &t.tw_fwd[TwLayout::A3 + j], sizeof f) != 0 || memcmp(&i, &t.tw_inv[TwLayout::A3 + j], sizeof i) != 0) { fprintf(stderr, "libdab_b200: twiddle literal %d differs from the table\n", j); abort(); }
    }
    // frequency interleaver (freq-interleaver.cpp:35-59)
    {
        int pi = 0, n = 0;
        for (int i = 0; i < TU; i++) t.invperm[i] = -1;
        for (int i = 0; i < TU; i++) {
            if (i > 0) pi = (13 * pi + 511) % TU;
            if (pi == TU / 2 || pi < 256 || pi > 256 + KC) continue;
            int carrier = pi - TU / 2;
            t.perm[n] = (int16_t)carrier;
            t.invperm[carrier < 0 ? carrier + TU : carrier] = (int16_t)n;
            n++;
        }
    }
    // softbit staging layout of ofdm_demod_kernel: logical chunk c (carriers 8c .. 8c+7, 16 bytes of (re, im) pairs) sits in slot
    // kChunkSlot[c] of the staging area; the permutation was found offline (scripts/opt_scatter_layout.py) so that the 16-bit scatter
    // stores of a warp spread over the shared-memory banks (3.29 -> 1.92 wavefronts per store instruction)
    {
        bool seen[192] = {false};
        for (int c = 0; c < 192; c++) { if (kChunkSlot[c] >= 192 || seen[kChunkSlot[c]]) { fprintf(stderr, "libdab_b200: kChunkSlot is not a permutation\n"); abort(); } seen[kChunkSlot[c]] = true; }
        // kChunkSwap[c] = 1: the chunk's two 8-byte halves are stored swapped (carriers 8c+4 .. 8c+7 first)
        for (int b = 0; b < TU; b++) {
            const int pos = t.invperm[b];
            t.invperm[TU + b] = pos < 0 ? (int16_t)-1 : (int16_t)(8 * kChunkSlot[pos >> 3] + (((pos & 7) + 4 * kChunkSwap[pos >> 3]) & 7));
        }
        for (int c = 0; c < 192; c++) t.invperm[2 * TU + c] = (int16_t)(kChunkSlot[c] | (kChunkSwap[c] << 8));
    }
    // phase reference (phasereference.cpp:45-51): float phase, float cos/sin
    memset(t.prs_ref, 0, sizeof t.prs_ref);
    for (int i = 1; i <= KC / 2; i++) {
        float p = prs_phi(i);
        t.prs_ref[i] = make_float2(cosf(p), sinf(p));
        p = prs_phi(-i);
        t.prs_ref[TU - i] = make_float2(cosf(p), sinf(p));
    }
    // puncturing vectors PI_1..PI_24 (protTables.cpp:25-51): groups of 4 start as 1000; bits are switched on
    // group by group in the order 0,4,2,6,1,5,3,7, one column per eight steps
    {
        static const int order[8] = {0, 4, 2, 6, 1, 5, 3, 7};
        for (int p = 1; p <= 24; p++) {
            int8_t* v = t.pcodes[p - 1];
            for (int g = 0; g < 8; g++) { v[4 * g] = 1; v[4 * g + 1] = v[4 * g + 2] = v[4 * g + 3] = 0; }
            for (int q = 1; q <= p; q++) v[4 * order[(q - 1) & 7] + 1 + (q - 1) / 8] = 1;
        }
    }
    // FIC de-puncturing map: 21 blocks PI_16, 3 blocks PI_15, tail 1100 x6 (fic-handler.cpp:39-42,158-191)
    {
        int pos = 0, ic = 0;
        for (int i = 0; i < 21 * 128; i++, pos++) t.fic_map[pos] = t.pcodes[15][i & 31] ? (int16_t)ic++ : (int16_t)-1;
        for (int i = 0; i < 3 * 128; i++, pos++) t.fic_map[pos] = t.pcodes[14][i & 31] ? (int16_t)ic++ : (int16_t)-1;
        for (int i = 0; i < 24; i++, pos++) t.fic_map[pos] = ((i & 3) < 2) ? (int16_t)ic++ : (int16_t)-1;
    }
    // GF(2^8), field polynomial 0x11D (dabplus_decoder.cpp:317, libs/fec/init_rs.h:54-64)
    {
        unsigned x = 1;
        memset(t.gf_log, 0, sizeof t.gf_log);
        for (int i = 0; i < 255; i++) { t.gf_exp[i] = (uint8_t)x; t.gf_log[x] = (uint8_t)i; x <<= 1; if (x & 0x100) x ^= 0x11D; }
        for (int i = 255; i < 512; i++) t.gf_exp[i] = t.gf_exp[i - 255];
    }
}

void build_osc_table(float2* osc) { build_osc_table_t(osc); }

// factors of the on-the-fly oscillator (osc_factors.h)
void build_osc_factors(const float2* osc_table, double2* hi, double* theta, int* patched) { build_osc_factors_t(osc_table, hi, theta, patched); }

// UEP profiles exactly as the reference applies them (uep-protection.cpp:38-118): bitrate, level, L1..L4, PI1..PI4.
// (Rows 80/1 and a few others differ from ETSI Table 15; bit-parity is with the reference.)  PI = 0: block unused.
static const int16_t kUep[][10] = {
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

int make_prot_profile(int b, int short_form, int uep_level, int eep_profile_a, int eep_level, ProtProfile& p)
{
    memset(&p, 0, sizeof p);
    p.bitrate = b;
    if (short_form) {
        const int n = (int)(sizeof kUep / sizeof kUep[0]);
        int idx = -1;
        for (int i = 0; i < n; i++) if (kUep[i][0] == b && kUep[i][1] == uep_level) { idx = i; break; }
        if (idx < 0) idx = 1;   // uep-protection.cpp:152-155
        p.nblk = 4;
        for (int k = 0; k < 4; k++) { p.L[k] = kUep[idx][2 + k]; p.PI[k] = kUep[idx][6 + k]; }
    } else if (eep_profile_a) {   // eep-protection.cpp:37-78
        p.nblk = 2;
        switch (eep_level) {
            case 1: p.L[0] = 6 * b / 8 - 3; p.L[1] = 3; p.PI[0] = 24; p.PI[1] = 23; break;
            case 2: if (b == 8) { p.L[0] = 5; p.L[1] = 1; p.PI[0] = 13; p.PI[1] = 12; }
                    else { p.L[0] = 2 * b / 8 - 3; p.L[1] = 4 * b / 8 + 3; p.PI[0] = 14; p.PI[1] = 13; } break;
            case 3: p.L[0] = 6 * b / 8 - 3; p.L[1] = 3; p.PI[0] = 8; p.PI[1] = 7; break;
            case 4: p.L[0] = 4 * b / 8 - 3; p.L[1] = 2 * b / 8 + 3; p.PI[0] = 3; p.PI[1] = 2; break;
            default: return -1;
        }
    } else {                      // eep-protection.cpp:80-112
        p.nblk = 2; p.L[0] = 24 * b / 32 - 3; p.L[1] = 3;
        switch (eep_level) {
            case 1: p.PI[0] = 10; p.PI[1] = 9; break;
            case 2: p.PI[0] = 6; p.PI[1] = 5; break;
            case 3: p.PI[0] = 4; p.PI[1] = 3; break;
            case 4: p.PI[0] = 2; p.PI[1] = 1; break;
            default: return -1;
        }
    }
    int total_blocks = 0;
    for (int k = 0; k < p.nblk; k++) { if (p.L[k] < 0) return -1; if (p.L[k] > 0 && (p.PI[k] < 1 || p.PI[k] > 24)) return -1; total_blocks += p.L[k]; }
    if (total_blocks * 128 != 4 * 24 * b) return -1;   // the (L, PI) blocks must tile the 4*24*bitrate mother-code positions
    // number of punctured bits: ones(PI) * 4 per block of 128, + 12 tail bits
    int n = 12;
    for (int k = 0; k < p.nblk; k++) n += p.L[k] * 4 * (8 + p.PI[k]);
    p.in_bits = n;
    return n;
}

void build_msc_map(const HostTables& t, const ProtProfile& p, int16_t* map)
{
    // build_vit_tables reads only the sign (the softbits are consumed in order), so the index saturates instead of wrapping negative:
    // EEP 1-A above 341 kbit/s has more than 32767 softbits per codeword
    int pos = 0, ic = 0;
    auto next = [&ic]() { const int v = ic++; return (int16_t)(v < 32767 ? v : 32767); };
    for (int k = 0; k < p.nblk; k++)
        for (int i = 0; i < p.L[k] * 128; i++, pos++) map[pos] = t.pcodes[p.PI[k] - 1][i & 31] ? next() : (int16_t)-1;
    for (int i = 0; i < 24; i++, pos++) map[pos] = ((i & 3) < 2) ? next() : (int16_t)-1;
}

void build_ber_profile(const HostTables& t, int nblk, const int* L, const int* PI, int nbits, dabb_ber::Profile& out)
{
    // the same vectors build_msc_map and the FIC map expand (bit i of a mask = entry i of PI_n)
    uint32_t mask[4] = {0, 0, 0, 0};
    for (int k = 0; k < nblk; k++)
        if (L[k] > 0) for (int i = 0; i < 32; i++) mask[k] |= (uint32_t)(t.pcodes[PI[k] - 1][i] != 0) << i;
    dabb_ber::build_profile(nblk, L, mask, nbits, out);
}

void build_prbs_words(int nbits, uint32_t* w)
{
    // PRBS x^9 + x^5 + 1, all-ones preset (fic-handler.cpp:62-71, energy_dispersal.h:40-49), run for the block's own length: an MSC
    // logical frame has up to 24 x 1824 bits.  Packed like the decoder output: bit t in byte t/8 (MSB first), bytes little-endian in the word
    memset(w, 0, sizeof(uint32_t) * (size_t)((nbits + 31) / 32));
    unsigned reg = 0x1FF;
    for (int t = 0; t < nbits; t++) {
        const unsigned b = ((reg >> 8) ^ (reg >> 4)) & 1;
        reg = ((reg << 1) | b) & 0x1FF;
        if (b) w[t >> 5] |= 1u << (8 * ((t >> 3) & 3) + 7 - (t & 7));
    }
}

} // namespace dabb
