// CPU build of sample-clock tracking (DABB_CLOCK_TRACK) of welle.io_b200/csrc/clock_core.cuh: the estimator update, the applied-value
// rule and the per-carrier phasor (tests/test_clock_emul.py).  emul_clock_step applies them per stream the way advance_kernel and
// post_sync_kernel do (welle.io_b200/csrc/api.cu).  Compile with -ffp-contract=off.
#include "../../welle.io_b200/csrc/clock_core.cuh"
#include <stdint.h>
#include <string.h>

extern "C" {

int emul_clock_state_size(void) { return (int)sizeof(dabb_clock::State); }

void emul_clock_reset(dabb_clock::State* st, int first, int count) { memset(st + first, 0, sizeof(dabb_clock::State) * (size_t)count); }

// one step of S streams with the option `mode` and the step's status / start_index per stream: tap 11's fields
void emul_clock_step(dabb_clock::State* st, int S, int mode, const int32_t* status, const int32_t* start_index, float* ppm, float* applied, int32_t* frames)
{
    for (int s = 0; s < S; s++) {
        dabb_clock::State& z = st[s];
        ppm[s] = 0.f; applied[s] = 0.f; frames[s] = 0;
        if (mode != 1) { z.prev = 0; continue; }
        if (status[s] == 0) {
            applied[s] = (float)dabb_clock::applied(z);
            dabb_clock::update(z, start_index[s]);
        } else if (status[s] == 2 || status[s] == 3) z.prev = 0;
        ppm[s] = (float)z.e; frames[s] = z.n;
    }
}

// the phasor of carriers k = -768 .. 768 at ppm: out[2 (k + 768)], out[2 (k + 768) + 1]
void emul_clock_phasors(float ppm, float* out)
{
    for (int k = -768; k <= 768; k++) {
        const float2 v = dabb_clock::phasor(k, ppm);
        out[2 * (k + 768)] = v.x; out[2 * (k + 768) + 1] = v.y;
    }
}

} // extern "C"
