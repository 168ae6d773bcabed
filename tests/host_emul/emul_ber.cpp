// CPU build of the channel bit-error count (welle.io_b200/csrc/ber_core.cuh) with the library's own profile tables (tables.cpp is host
// code in a CUDA translation unit: compile with nvcc -x cu; no device is involved).  tests/test_ber_emul.py
#include "../../welle.io_b200/csrc/tables.cpp"
#include "../../include/dab_b200.h"
#include <vector>
using namespace dabb;

// the counts of n codewords of one protection profile (fic = 1: the FIC).  soft: n rows of soft_pitch punctured softbits (4-byte aligned
// rows, readable 3 bytes past the profile's length); out: n rows of out_pitch decoded bytes after energy dispersal.  counts: [n][3] bits,
// errors, erasures.  Returns the profile's transmitted bits per codeword, or -1 for a profile the library does not know.
extern "C" int emul_ber_count(int fic, int bitrate, int short_form, int uep_level, int eep_profile_a, int eep_level,
                              const int8_t* soft, int soft_pitch, const uint8_t* out, int out_pitch, int n, int32_t* counts)
{
    static HostTables* t = nullptr;
    if (!t) { t = new HostTables; build_host_tables(*t); }
    dabb_ber::Profile p;
    int nbits;
    if (fic) {
        const int L[2] = {21, 3}, PI[2] = {16, 15};
        nbits = 768;
        build_ber_profile(*t, 2, L, PI, nbits, p);
    } else {
        ProtProfile pp;
        if (make_prot_profile(bitrate, short_form, uep_level, eep_profile_a, eep_level, pp) < 0) return -1;
        nbits = 24 * bitrate;
        build_ber_profile(*t, pp.nblk, pp.L, pp.PI, nbits, p);
        if (p.in_bits != pp.in_bits) return -2;
    }
    std::vector<uint32_t> w((size_t)(nbits + 31) / 32);
    build_prbs_words(nbits, w.data());
    p.prbs = w.data();
    for (int i = 0; i < n; i++) {
        dabb_ber::Counts c{0u, 0u, 0u};
        for (int j = 0; j < p.nchunks; j++) dabb_ber::count_chunk(p, j, soft + (size_t)i * soft_pitch, out + (size_t)i * out_pitch, c);
        counts[3 * i] = (int32_t)c.bits; counts[3 * i + 1] = (int32_t)c.errors; counts[3 * i + 2] = (int32_t)c.erasures;
    }
    return p.in_bits;
}

extern "C" void emul_ber_sizes(int32_t* out)
{
    out[0] = (int32_t)sizeof(dabb_options); out[1] = (int32_t)sizeof(dabb_ber_result); out[2] = (int32_t)sizeof(dabb_config);
    out[3] = (int32_t)sizeof(dabb_subchannel); out[4] = (int32_t)sizeof(dabb_frame_result);
}
