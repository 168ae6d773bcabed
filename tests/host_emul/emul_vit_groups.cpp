// CPU build of the grouped Viterbi schedule (welle.io_b200/csrc/vit_groups.cuh) that dabb_select_subchannel / dabb_remove_subchannel
// rebuild for a slot (tests/test_vit_groups.py).
#include "../../welle.io_b200/csrc/vit_groups.cuh"
#include <string.h>

using namespace dabb;

extern "C" {

// groups_out[cap][5]: profile, first, count, dec_off (low, high 32 bits); list_out: at least 4 * n_streams entries.
// Returns the number of CTAs (-1: more than cap); *n_list and *dec_words as built.
int emul_vit_schedule(const int32_t* prof_of, int n_streams, const int32_t* nsteps, int n_profiles, int32_t* groups_out, int cap,
                      int32_t* list_out, int32_t* n_list, int64_t* dec_words)
{
    VitSchedule s;
    build_vit_schedule(prof_of, n_streams, nsteps, n_profiles, s);
    if ((int)s.groups.size() > cap) return -1;
    for (size_t i = 0; i < s.groups.size(); i++) {
        const VitGroup& g = s.groups[i];
        int32_t* o = groups_out + 5 * i;
        o[0] = g.profile; o[1] = g.first; o[2] = g.count; o[3] = (int32_t)(g.dec_off & 0xFFFFFFFF); o[4] = (int32_t)(g.dec_off >> 32);
    }
    if (!s.list.empty()) memcpy(list_out, s.list.data(), s.list.size() * sizeof(int32_t));
    *n_list = (int32_t)s.list.size();
    *dec_words = s.dec_words;
    return (int)s.groups.size();
}

}
