// CPU build of the device TII analysis (welle.io_b200/csrc/tii_core.cuh): one stream, frame by frame, the way tii_plan_kernel and
// tii_phase_kernel run it (tests/test_tii_emul.py).  Compile with -ffp-contract=off.
#include "../../welle.io_b200/csrc/tii_core.cuh"
#include <stdint.h>
#include <string.h>
#include <vector>

using namespace dabb_tii;

namespace {
uint16_t g_rank[2][N_ERR];
bool g_rank_ok = false;
const uint16_t* ranks()
{
    if (!g_rank_ok) { build_rank_tables(g_rank); g_rank_ok = true; }
    return &g_rank[0][0];
}
}

extern "C" {

// n frames of spectra (natural bin order, 2048 complex floats each); out: 5 floats per measurement (frame, comb, pattern, delay_samples,
// error), each frame's in the order of the step's record; info[4 f ..]: analyses, measurements, skipped, evicted of frame f.
// Returns the number of measurements.
int emul_tii_run(const float* null_specs, const float* prs_specs, int n, float* out, int cap, int32_t* info)
{
    StreamHdr h;
    memset(&h, 0, sizeof h);
    std::vector<uint32_t> sums((size_t)N_SLOTS * N_ERR, 0u);
    const uint16_t* rank = ranks();
    int k = 0;
    for (int f = 0; f < n; f++) {
        const cf* nul = reinterpret_cast<const cf*>(null_specs) + (size_t)f * 2048;
        const cf* prs = reinterpret_cast<const cf*>(prs_specs) + (size_t)f * 2048;
        uint8_t act[N_PAIRS], mask[24];
        for (int i = 0; i < N_PAIRS; i++) act[i] = pair_active(nul, prs, i);
        comb_masks(act, mask);
        Job jobs[MAX_JOBS];
        const FrameSummary r = plan_frame(h, mask, jobs);
        if (info) { info[4 * f] = r.njobs; info[4 * f + 1] = r.nmeas; info[4 * f + 2] = r.skipped; info[4 * f + 3] = r.evicted; }
        std::vector<float> rec((size_t)5 * r.nmeas);
        for (int j = 0; j < r.njobs; j++) {
            const Job& jb = jobs[j];
            cf nv[32]; float ph[32]; int car[32];
            for (int t = 0; t < 32; t++) {
                car[t] = carrier(jb.comb, (unsigned)jb.word, t);
                nv[t] = nul[bin_of(car[t])];
                ph[t] = arg_f(prs[bin_of(carrier(jb.comb, (unsigned)jb.word, t & ~1))]);
            }
            uint64_t best = ~0ull;
            for (int e = 0; e < N_ERR; e++) {
                uint32_t& s = sums[(size_t)jb.slot * N_ERR + e];
                s = accumulate(s, jb.start, abs_err(nv, ph, car, e + ERR_FIRST));
                const uint64_t key = argmin_key(s, rank[jb.table * N_ERR + e], e);
                if (key < best) best = key;
            }
            if (jb.out >= 0) {
                float* o = rec.data() + 5 * jb.out;
                o[0] = (float)f; o[1] = (float)jb.comb; o[2] = (float)jb.pattern; o[3] = (float)((int)(best & 0xFFFF) + ERR_FIRST); o[4] = (float)(uint32_t)(best >> 32);
            }
        }
        for (int m = 0; m < r.nmeas; m++, k++)
            if (k < cap) memcpy(out + 5 * k, rec.data() + 5 * m, 5 * sizeof(float));
    }
    return k;
}

// rank tables [2][504] (0: fresh map, 1: after clear())
void emul_tii_rank(uint16_t* out) { memcpy(out, ranks(), sizeof g_rank); }

// the delay the arg-min picks from 504 sums with rank table `table`
int emul_tii_argmin(const uint32_t* sums, int table)
{
    const uint16_t* rank = ranks();
    uint64_t best = ~0ull;
    for (int e = 0; e < N_ERR; e++) { const uint64_t key = argmin_key(sums[e], rank[table * N_ERR + e], e); if (key < best) best = key; }
    return (int)(best & 0xFFFF) + ERR_FIRST;
}

// the 32 sorted carriers of (comb, pattern)
void emul_tii_carriers(int comb, int pattern, int32_t* out)
{
    const unsigned w = pattern_word(pattern);
    for (int j = 0; j < 32; j++) out[j] = carrier(comb, w, j);
}

} // extern "C"
