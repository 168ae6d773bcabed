// tii.cu — transmitter identification (TII) analysis of every stream on the device, behind tii_spectra_kernel (ofdm.cu).  The arithmetic
// and the per-stream bookkeeping are in tii_core.cuh, which the host emulation compiles too; these kernels only spread it over the GPU:
//   tii_plan_kernel:  one CTA per stream, one thread per carrier pair: activity flags, comb masks, then one thread plans the frame
//                     (likely combinations, accumulator slots, which analyses report) and zeroes the stream's result record
//   tii_phase_kernel: one CTA per (stream, likely combination), one thread per delay hypothesis: the 32-carrier phase error, the
//                     accumulation into the combination's table and, on its fifth analysis, the arg-min into the result record
#include "../../include/dab_b200.h"
#include "common.cuh"
#include <string.h>

namespace dabb {
namespace {

using namespace dabb_tii;

__global__ void __launch_bounds__(N_PAIRS)
tii_plan_kernel(TiiParams p)
{
    const int s = blockIdx.x, t = threadIdx.x;
    __shared__ uint8_t act[N_PAIRS];
    dabb_tii_result* res = reinterpret_cast<dabb_tii_result*>(p.res) + s;
    if (!p.active[s]) {           // only decoded frames are analysed (the reference feeds TIIDecoder after a successful frame)
        if (t == 0) { dabb_tii_result z; memset(&z, 0, sizeof z); *res = z; p.njobs[s] = 0; }
        return;
    }
    const cf* prs = reinterpret_cast<const cf*>(p.spectra + (int64_t)s * 2 * TU);
    const cf* nul = prs + TU;
    act[t] = pair_active(nul, prs, t);
    __syncthreads();
    if (t) return;
    uint8_t mask[24];
    comb_masks(act, mask);
    const FrameSummary r = plan_frame(p.hdr[s], mask, p.jobs + (int64_t)s * MAX_JOBS);
    p.njobs[s] = r.njobs;
    dabb_tii_result z; memset(&z, 0, sizeof z);
    z.count = r.nmeas; z.evicted = r.evicted; z.skipped = r.skipped;
    *res = z;
}

constexpr int PHASE_THREADS = 512;

__global__ void __launch_bounds__(PHASE_THREADS)
tii_phase_kernel(TiiParams p)
{
    const int s = blockIdx.x, j = blockIdx.y, t = threadIdx.x;
    if (j >= p.njobs[s]) return;
    const Job jb = p.jobs[(int64_t)s * MAX_JOBS + j];
    const cf* prs = reinterpret_cast<const cf*>(p.spectra + (int64_t)s * 2 * TU);
    const cf* nul = prs + TU;
    __shared__ cf nv[32];
    __shared__ float ph[32];
    __shared__ int car[32];
    __shared__ unsigned long long red[PHASE_THREADS / 32];
    if (t < 32) {
        car[t] = carrier(jb.comb, (unsigned)jb.word, t);
        nv[t] = nul[bin_of(car[t])];
        ph[t] = arg_f(prs[bin_of(carrier(jb.comb, (unsigned)jb.word, t & ~1))]);     // both carriers of a pair take the first one's PRS phase
    }
    __syncthreads();
    unsigned long long key = ~0ull;
    if (t < N_ERR) {
        uint32_t* sum = p.sums + ((int64_t)s * N_SLOTS + jb.slot) * N_ERR + t;
        const uint32_t v = accumulate(jb.start ? 0u : *sum, jb.start, abs_err(nv, ph, car, t + ERR_FIRST));
        *sum = v;
        key = argmin_key(v, p.rank[jb.table * N_ERR + t], t);
    }
    if (jb.out < 0) return;       // the same for the whole CTA
    for (int o = 16; o; o >>= 1) { const unsigned long long k = __shfl_xor_sync(0xffffffffu, key, o); key = k < key ? k : key; }
    if ((t & 31) == 0) red[t >> 5] = key;
    __syncthreads();
    if (t >= 32) return;
    key = t < PHASE_THREADS / 32 ? red[t] : ~0ull;
    for (int o = 16; o; o >>= 1) { const unsigned long long k = __shfl_xor_sync(0xffffffffu, key, o); key = k < key ? k : key; }
    if (t) return;
    auto& m = reinterpret_cast<dabb_tii_result*>(p.res)[s].m[jb.out];
    m.comb = jb.comb; m.pattern = jb.pattern; m.delay_samples = (int)(key & 0xFFFF) + ERR_FIRST; m.error = (float)(uint32_t)(key >> 32);
}

} // namespace

void launch_tii_plan(const TiiParams& p, cudaStream_t st) { tii_plan_kernel<<<p.n, N_PAIRS, 0, st>>>(p); }
void launch_tii_phase(const TiiParams& p, cudaStream_t st) { tii_phase_kernel<<<dim3(p.n, MAX_JOBS), PHASE_THREADS, 0, st>>>(p); }

} // namespace dabb
