// vit_groups.cuh — the codeword schedule of a sub-channel slot's Viterbi launch when its streams use different protection profiles.
// Plain C++ without CUDA types, so that the host test (tests/host_emul/emul_vit_groups.cpp) builds the same code.
//
// The decoder kernel runs one codeword per thread and 128 codewords per CTA, and a CTA needs ONE puncturing pattern (its warps share
// the expansion table, advance their softbit windows together and run the same number of trellis steps).  So a slot with several
// profiles is decoded by one launch whose CTAs each hold codewords of one profile: CTA b reads descriptor b, and its thread t decodes
// codeword list[first + t] of that descriptor's profile.  CTAs of longer codewords come first, so that they do not form the tail of
// the launch.  For a slot whose streams are all enabled with one profile the schedule is the identity: CTA b holds codewords
// 128 b .. 128 b + 127 and its decisions start where the ungrouped launch puts them.
#pragma once
#include <stdint.h>
#include <algorithm>
#include <vector>

namespace dabb {

constexpr int VIT_GROUP_CW = 128;        // codewords per CTA of the decoder kernel (viterbi.cu defines VIT_THREADS as this)

// one CTA of a grouped launch
struct VitGroup {
    int32_t profile;                     // index into the context's protection-profile table
    int32_t first, count;                // codewords list[first .. first + count), count <= VIT_GROUP_CW (0: the CTA does nothing)
    int32_t pad;
    int64_t dec_off;                     // the CTA's decision words start at dec + dec_off (8-byte words, nsteps * 128 of them)
};

struct VitSchedule {
    std::vector<VitGroup> groups;
    std::vector<int32_t> list;           // codeword 4 stream + c of every enabled stream, grouped by profile
    int64_t dec_words = 0;               // decision words the launch needs (sum over CTAs of nsteps * 128)
};

// prof_of[s]: the profile stream s decodes in the slot, or -1 when it is not enabled there; nsteps[p]: trellis steps of profile p.
// Profiles are taken in descending nsteps (ties: ascending index), each profile's codewords in ascending order, 128 per CTA.
// A slot without enabled streams gets one empty CTA, so that its launch stays a valid grid.
inline void build_vit_schedule(const int32_t* prof_of, int n_streams, const int32_t* nsteps, int n_profiles, VitSchedule& out)
{
    out.groups.clear(); out.list.clear(); out.dec_words = 0;
    std::vector<std::vector<int32_t>> by_prof((size_t)n_profiles);
    for (int s = 0; s < n_streams; s++) {
        const int p = prof_of[s];
        if (p < 0 || p >= n_profiles) continue;
        for (int c = 0; c < 4; c++) by_prof[(size_t)p].push_back(4 * s + c);
    }
    std::vector<int32_t> order;
    for (int p = 0; p < n_profiles; p++) if (!by_prof[(size_t)p].empty()) order.push_back(p);
    std::stable_sort(order.begin(), order.end(), [&](int32_t a, int32_t b) { return nsteps[a] > nsteps[b]; });
    for (const int32_t p : order) {
        const std::vector<int32_t>& cws = by_prof[(size_t)p];
        for (size_t i = 0; i < cws.size(); i += VIT_GROUP_CW) {
            VitGroup g{};
            g.profile = p; g.first = (int32_t)out.list.size(); g.count = (int32_t)std::min<size_t>(VIT_GROUP_CW, cws.size() - i);
            out.list.insert(out.list.end(), cws.begin() + (ptrdiff_t)i, cws.begin() + (ptrdiff_t)(i + (size_t)g.count));
            g.dec_off = out.dec_words;
            out.dec_words += (int64_t)nsteps[p] * VIT_GROUP_CW;
            out.groups.push_back(g);
        }
    }
    if (out.groups.empty()) out.groups.push_back(VitGroup{0, 0, 0, 0, 0});
}

} // namespace dabb
