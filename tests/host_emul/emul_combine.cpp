// CPU build of diversity combining (dabb_set_combining) of welle.io_b200/csrc/combine_core.cuh: the noise power of a null symbol, the
// contributor rule and the combination + demap of one symbol, applied the way null_power_kernel (api.cu) and combine_kernel
// (combine.cu) apply them (tests/test_combine_emul.py, tests/test_gpu_combine.py).  Compile with -ffp-contract=off.
#include "../../welle.io_b200/csrc/combine_core.cuh"
#include <stdint.h>

extern "C" {

// N of n null symbols y[n][TNULL]
void emul_combine_noise(const float2* y, int n, float* out)
{
    for (int f = 0; f < n; f++) {
        float part[dabb_comb::NULL_THREADS];
        for (int t = 0; t < dabb_comb::NULL_THREADS; t++) part[t] = dabb_comb::null_partial(y + (int64_t)f * dabb::TNULL, t);
        out[f] = dabb_comb::null_noise(part);
    }
}

uint32_t emul_combine_select(int n, int lpos, const int32_t* decoded, const int64_t* a, const float* noise)
{
    return dabb_comb::contributors(n, lpos, decoded, a, noise);
}

// one symbol: the members' r1[n][KC] (logical carrier order, ascending stream order), their noise, the contributor mask -> the
// leader's softbits [3072] (1536 Re, then 1536 Im) as combine_kernel writes them (the caller keeps the leader's own softbits when fewer
// than two members contribute)
void emul_combine_symbol(const float2* r1, int n, const float* noise, uint32_t mask, int weighted, int8_t* soft)
{
    using namespace dabb_comb;
    float2 R[COMB_THREADS][COMB_PER_THREAD];
    for (int t = 0; t < COMB_THREADS; t++)
        for (int j = 0; j < COMB_PER_THREAD; j++) {
            R[t][j] = make_float2(0.f, 0.f);
            for (int i = 0; i < n; i++)
                if ((mask >> i) & 1u) acc(R[t][j], r1[(int64_t)i * dabb::KC + t + COMB_THREADS * j], noise[i]);
        }
    float G = 0.f, rG = 0.f;
    if (weighted) {
        LevelSum part[COMB_THREADS];
        for (int t = 0; t < COMB_THREADS; t++) part[t] = level_partial(R[t]);
        G = level_total(part); rG = dabb::q127(G);
    }
    for (int t = 0; t < COMB_THREADS; t++)
        for (int j = 0; j < COMB_PER_THREAD; j++) {
            int8_t sre, sim;
            if (weighted) dabb::demap_weighted(R[t][j], G, rG, sre, sim);
            else dabb::demap_r1(R[t][j], sre, sim);
            soft[t + COMB_THREADS * j] = sre;
            soft[dabb::KC + t + COMB_THREADS * j] = sim;
        }
}

} // extern "C"
