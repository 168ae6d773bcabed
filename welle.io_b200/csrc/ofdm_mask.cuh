// ofdm_mask.cuh — the OFDM symbols of a frame whose softbits a stream's decoders read.  Plain C++ without CUDA types, so that the host
// test (tests/host_emul/emul_ofdm_mask.cpp) builds the same code.
//
// The FIC reads the softbits of data symbols 1-3 (bytes [0, 3 * 3072) of the frame's softbits).  A sub-channel of start_cu, length_cu
// reads in each CIF c = 0..3 the bytes [(3 + 18 c) 3072 + 64 start_cu, + 64 length_cu) (msc_collect_kernel), i.e. data symbols
// 4 + 18 c + [64 start_cu / 3072, (64 (start_cu + length_cu) - 1) / 3072].  Those symbols are demapped; a demapped symbol and the one
// before it (its differential reference) are transformed, and so is the phase reference symbol (its SNR estimate).  ofdm_demod_kernel
// takes only the guard-interval correlation and the level sample of every other symbol, which need no transform.
#pragma once
#include <stdint.h>

namespace dabb {

constexpr int OFDM_MASK_WORDS = 4;       // per stream: bit l (l = 1..75) of the 128-bit mask = data symbol l is demapped

// one sub-channel slot of a stream as the mask sees it
struct OfdmMaskSlot {
    int32_t enabled, start_cu, length_cu;
};

inline bool ofdm_mask_demap(const uint32_t* m, int l) { return l >= 1 && l <= 75 && ((m[l >> 5] >> (l & 31)) & 1u); }
inline bool ofdm_mask_transform(const uint32_t* m, int l) { return l == 0 || ofdm_mask_demap(m, l) || ofdm_mask_demap(m, l + 1); }

// the mask of a stream whose slots are slots[0 .. n_slots); disabled slots read nothing
inline void build_ofdm_mask(const OfdmMaskSlot* slots, int n_slots, uint32_t* mask /* OFDM_MASK_WORDS */)
{
    for (int w = 0; w < OFDM_MASK_WORDS; w++) mask[w] = 0;
    auto set = [&](int l) { mask[l >> 5] |= 1u << (l & 31); };
    for (int l = 1; l <= 3; l++) set(l);
    for (int k = 0; k < n_slots; k++) {
        const OfdmMaskSlot& s = slots[k];
        if (!s.enabled || s.length_cu < 1) continue;
        const int a = 64 * s.start_cu / 3072, b = (64 * (s.start_cu + s.length_cu) - 1) / 3072;
        for (int c = 0; c < 4; c++)
            for (int d = a; d <= b; d++) set(4 + 18 * c + d);
    }
}

} // namespace dabb
