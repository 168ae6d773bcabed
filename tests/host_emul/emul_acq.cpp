// CPU build of robust acquisition (dabb_options.acquisition = DABB_ACQ_ROBUST) of welle.io_b200/csrc/acq_core.cuh: the block levels
// as acq_level_kernel (acq.cu) computes them, the decision of acq_decide_kernel (api.cu) and the interferer excision of
// find_index_excise_kernel (ofdm.cu), applied the way the kernels apply them (tests/test_acq_emul.py, tests/test_gpu_acq.py).
// Compile with -ffp-contract=off.
#include "../../welle.io_b200/csrc/acq_core.cuh"
#include <algorithm>
#include <stdint.h>
#include <vector>

using namespace dabb_acq;

extern "C" {

// levels and envelope sums of nb blocks of 256 (already mixed) samples y[nb * 256]
void emul_acq_levels(const float2* y, int nb, float* level, float* l1sum)
{
    float cs[BLK];
    make_cos_table(cs);
    for (int b = 0; b < nb; b++) {
        const float2* src = y + (int64_t)b * BLK;
        float2 x[BLK];
        float l1[32];
        for (int lane = 0; lane < 32; lane++) {
            l1[lane] = 0.f;
            for (int r = 0; r < BLK / 32; r++) {
                const int n = lane + 32 * r;
                l1[lane] = l1[lane] + l1_of(src[n]);
                const float h = hann(cs, n);
                x[bitrev8(n)] = make_float2(src[n].x * h, src[n].y * h);
            }
        }
        for (int h = 1; h < BLK; h <<= 1)
            for (int q = 0; q < BLK / 2; q++) butterfly(x, cs, h, q);
        float part[32];
        for (int lane = 0; lane < 32; lane++) part[lane] = level_partial(x, lane);
        level[b] = level_total(part);
        float es = 0.f;
        for (int lane = 0; lane < 32; lane++) es = es + l1[lane];
        l1sum[b] = es;
    }
}

// the decision over nb levels: out = {found, best}, fout = {depth_db, median}
void emul_acq_decide(const float* level, int nb, int32_t* out, float* fout)
{
    std::vector<float> v(level, level + nb);
    std::nth_element(v.begin(), v.begin() + (nb - 1) / 2, v.end());
    const float med = v[(nb - 1) / 2];
    int best = 0; float wmin = window_sum(level, 0);
    for (int b = 1; b + WIN <= nb; b++) { const float w = window_sum(level, b); if (w <= wmin) { wmin = w; best = b; } }
    const float depth = depth_db(med, wmin);
    out[0] = is_found(depth, best, nb); out[1] = best;
    fout[0] = depth; fout[1] = med;
}

// excision of one window's spectrum X[2048] (natural bin order): zeroed[bin] = 1 for every bin set to 0; returns their count
int emul_acq_excise(const float2* X, uint8_t* zeroed)
{
    float pw[2048];
    for (int k = 0; k < 2048; k++) pw[k] = X[k].x * X[k].x + X[k].y * X[k].y;
    float part[EXC_THREADS];
    for (int t = 0; t < EXC_THREADS; t++) part[t] = exc_partial(pw, t);
    const float limit = exc_limit(part);
    int n = 0;
    for (int k = 0; k < 2048; k++) zeroed[k] = 0;
    for (int k = 0; k < 2048; k++)
        if (exc_over(pw[k], k, limit))
            for (int d = -EXC_NEIGH; d <= EXC_NEIGH; d++) zeroed[(k + d) & 2047] = 1;
    for (int k = 0; k < 2048; k++) n += zeroed[k];
    return n;
}

float emul_acq_log2(float x) { return log2_pos(x); }

} // extern "C"
