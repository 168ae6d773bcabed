// combine.cu — diversity reception on the device (dabb_set_combining, combine_core.cuh).  combine_kernel runs on lane A after the OFDM
// kernel, advance_kernel and null_power_kernel (api.cu) of a step: one CTA per (group, symbol the leader's decoders read).  Every thread
// selects the group's contributors from the step's statuses, phase reference positions and noise powers, adds the members' r1 rows in
// ascending stream order, demaps the sum, and the CTA overwrites the leader's softbits of that symbol.  A leader without another
// contributor keeps its own softbits.
#include "../../include/dab_b200.h"
#include "common.cuh"

namespace dabb {

namespace {

template <bool WEIGHTED>
__global__ void __launch_bounds__(dabb_comb::COMB_THREADS)
combine_kernel(CombParams p)
{
    using namespace dabb_comb;
    __shared__ LevelSum lsum[COMB_THREADS];
    __shared__ float gsh[2];
    const int t = threadIdx.x;
    const CombItem it = p.items ? p.items[blockIdx.x] : CombItem{(int)blockIdx.x / 75, (int)blockIdx.x % 75 + 1, (int)blockIdx.x % 75, blockIdx.x % 75 == 0};
    const CombGroup& g = p.groups[it.group];
    dabb_combine_result* res = reinterpret_cast<dabb_combine_result*>(p.res);
    int32_t dec[MAX_BRANCHES]; int64_t a[MAX_BRANCHES]; float nz[MAX_BRANCHES];
    const int n = g.n, lpos = g.lpos;
    for (int i = 0; i < n; i++) {
        const int s = g.stream[i];
        dec[i] = p.active[s] != 0;
        a[i] = p.buf_start[s] + p.prs[s];
        nz[i] = res[s].noise;
    }
    const uint32_t sel = contributors(n, lpos, dec, a, nz);
    const int leader = g.stream[lpos];
    if (it.first && t == 0) { res[leader].members = popcount(sel); res[leader].mask = sel; }
    if (popcount(sel) < 2) return;                   // CTA-uniform: the leader decodes alone
    float2 R[COMB_PER_THREAD];
#pragma unroll
    for (int j = 0; j < COMB_PER_THREAD; j++) R[j] = make_float2(0.f, 0.f);
    for (int i = 0; i < n; i++) {
        if (!((sel >> i) & 1u)) continue;
        const float2* r = p.r1 + ((int64_t)g.row[i] + it.col) * KC + t;
        const float ni = nz[i];
#pragma unroll
        for (int j = 0; j < COMB_PER_THREAD; j++) acc(R[j], __ldg(r + COMB_THREADS * j), ni);
    }
    float G = 0.f, rG = 0.f;
    if (WEIGHTED) {
        lsum[t] = level_partial(R);
        __syncthreads();
        if (t == 0) { const float g0 = level_total(lsum); gsh[0] = g0; gsh[1] = q127(g0); }
        __syncthreads();
        G = gsh[0]; rG = gsh[1];
    }
    int8_t* dst = p.soft + (int64_t)leader * p.soft_stride + (int64_t)(it.sym - 1) * 3072;
#pragma unroll
    for (int j = 0; j < COMB_PER_THREAD; j++) {
        int8_t sre, sim;
        if (WEIGHTED) demap_weighted(R[j], G, rG, sre, sim);
        else demap_r1(R[j], sre, sim);
        dst[t + COMB_THREADS * j] = sre;
        dst[KC + t + COMB_THREADS * j] = sim;
    }
}

} // namespace

void launch_combine(const CombParams& p, cudaStream_t st)
{
    if (p.n_items < 1) return;
    if (p.weighted) combine_kernel<true><<<p.n_items, dabb_comb::COMB_THREADS, 0, st>>>(p);
    else combine_kernel<false><<<p.n_items, dabb_comb::COMB_THREADS, 0, st>>>(p);
}

} // namespace dabb
