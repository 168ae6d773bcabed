// CPU build of the per-stream OFDM symbol mask (welle.io_b200/csrc/ofdm_mask.cuh) that dabb_select_subchannel / dabb_remove_subchannel
// rebuild for a stream (tests/test_ofdm_symbol_mask.py).
#include "../../welle.io_b200/csrc/ofdm_mask.cuh"
#include <stddef.h>

using namespace dabb;

extern "C" {

// slots[n_streams][n_slots][3] = {enabled, start_cu, length_cu}; masks_out[n_streams][OFDM_MASK_WORDS];
// flags_out[n_streams][76] = demap | transform << 1 of every symbol, as the two accessors report them
void emul_ofdm_mask(const int32_t* slots, int n_streams, int n_slots, uint32_t* masks_out, uint8_t* flags_out)
{
    for (int s = 0; s < n_streams; s++) {
        uint32_t* m = masks_out + (size_t)s * OFDM_MASK_WORDS;
        build_ofdm_mask(reinterpret_cast<const OfdmMaskSlot*>(slots + (size_t)s * n_slots * 3), n_slots, m);
        for (int l = 0; l < 76; l++) flags_out[(size_t)s * 76 + l] = (uint8_t)(ofdm_mask_demap(m, l) | (ofdm_mask_transform(m, l) << 1));
    }
}

int emul_ofdm_mask_words(void) { return OFDM_MASK_WORDS; }

}
