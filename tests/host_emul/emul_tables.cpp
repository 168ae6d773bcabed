// The library's own de-puncturing maps on the CPU (welle.io_b200/csrc/tables.cpp is host code): what dabb_fic_decode, dabb_msc_decode and
// dabb_select_subchannel hand to build_vit_tables.
#include "../../welle.io_b200/csrc/tables.cpp"
using namespace dabb;
// map: 4 * (nbits + 6) entries (>= 0 present, < 0 punctured); returns the number of punctured softbits a codeword consumes, or -1
extern "C" int emul_prot_map(int fic, int bitrate, int short_form, int uep_level, int eep_profile_a, int eep_level, int16_t* map)
{
    static HostTables* t = nullptr;
    if (!t) { t = new HostTables; build_host_tables(*t); }
    if (fic) { memcpy(map, t->fic_map, sizeof t->fic_map); return 2304; }
    ProtProfile p;
    if (make_prot_profile(bitrate, short_form, uep_level, eep_profile_a, eep_level, p) < 0) return -1;
    build_msc_map(*t, p, map);
    return p.in_bits;
}
// the energy-dispersal words add_profile and dabb_msc_decode give the decoder for a profile: w [(24 * bitrate + 31) / 32]; returns their number
extern "C" int emul_prot_prbs_words(int bitrate, uint32_t* w)
{
    const int nbits = 24 * bitrate;
    build_prbs_words(nbits, w);
    return (nbits + 31) / 32;
}
