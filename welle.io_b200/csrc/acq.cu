// acq.cu — robust acquisition on the device (dabb_options.acquisition = DABB_ACQ_ROBUST, acq_core.cuh).  acq_level_kernel runs on
// lane A between acq_plan_kernel and acq_decide_kernel (api.cu), in place of acquire_kernel: one warp per block of 256 samples, eight
// blocks per CTA.  Each warp mixes its block with the stream's NCO, windows it, transforms it (radix-2, in shared memory) and writes the
// block's level and envelope sum.  The CTAs take (stream, chunk) items in a grid-stride loop, so that a step in which few streams search
// does not launch a CTA per chunk of every stream.
#include "../../include/dab_b200.h"
#include "common.cuh"

namespace dabb {

namespace {

constexpr int ACQ_THREADS = 32 * dabb_acq::CHUNK;
constexpr int ACQ_CHUNKS = dabb_acq::NB_MAX / dabb_acq::CHUNK;

__device__ __forceinline__ int32_t acq_mod_rate(int64_t v) { v %= INPUT_RATE; if (v < 0) v += INPUT_RATE; return (int32_t)v; }

__global__ void __launch_bounds__(ACQ_THREADS)
acq_level_kernel(const AcqJob* __restrict__ job, const float2* __restrict__ iq, int64_t stride, const float2* __restrict__ osc,
                 const float* __restrict__ cos_tab, int S, float* __restrict__ level, float* __restrict__ l1sum)
{
    using namespace dabb_acq;
    __shared__ float2 buf[CHUNK][BLK];
    __shared__ float cs[BLK];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    for (int i = threadIdx.x; i < BLK; i += ACQ_THREADS) cs[i] = cos_tab[i];
    __syncthreads();
    float2* x = buf[w];
    for (int64_t item = blockIdx.x; item < (int64_t)S * ACQ_CHUNKS; item += gridDim.x) {
        const int s = (int)(item / ACQ_CHUNKS), b = (int)(item % ACQ_CHUNKS) * CHUNK + w;
        const AcqJob j = job[s];
        if (b >= j.nb) continue;                                    // warp-uniform
        const float2* src = iq + (int64_t)s * stride + j.rel + (int64_t)b * BLK;
        const bool mix = j.lp != 0 || j.phase != 0;
        float l1 = 0.f;
#pragma unroll
        for (int r = 0; r < BLK / 32; r++) {
            const int n = lane + 32 * r;
            float2 y = src[n];
            if (mix) {
                const float2 o = osc[acq_mod_rate((int64_t)j.lp - ((int64_t)b * BLK + n + 1) * j.phase)];
                y = make_float2(__fsub_rn(__fmul_rn(y.x, o.x), __fmul_rn(y.y, o.y)), __fadd_rn(__fmul_rn(y.x, o.y), __fmul_rn(y.y, o.x)));
            }
            l1 = __fadd_rn(l1, l1_of(y));
            const float h = hann(cs, n);
            x[bitrev8(n)] = make_float2(__fmul_rn(y.x, h), __fmul_rn(y.y, h));
        }
        __syncwarp();
        for (int h = 1; h < BLK; h <<= 1) {
#pragma unroll
            for (int r = 0; r < 4; r++) butterfly(x, cs, h, lane + 32 * r);
            __syncwarp();
        }
        const float part = level_partial(x, lane);
        float lv = 0.f, es = 0.f;                                   // level_total and the envelope sum, both in lane order
        for (int t = 0; t < 32; t++) {
            lv = __fadd_rn(lv, __shfl_sync(0xffffffffu, part, t));
            es = __fadd_rn(es, __shfl_sync(0xffffffffu, l1, t));
        }
        if (lane == 0) {
            level[(int64_t)s * NB_MAX + b] = __fdiv_rn(lv, (float)NBIN);
            l1sum[(int64_t)s * NB_MAX + b] = es;
        }
        __syncwarp();                                               // x is rewritten by the next item
    }
}

} // namespace

void launch_acq_levels(const AcqJob* job, const float2* iq, int64_t stride, const float2* osc, const float* cos_tab, int S,
                       float* level, float* l1sum, cudaStream_t st)
{
    static int ctas = 0;
    if (!ctas) {
        int dev = 0, sms = 0, per_sm = 0;
        cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, acq_level_kernel, ACQ_THREADS, 0);
        ctas = sms * (per_sm > 0 ? per_sm : 1);
    }
    const int64_t items = (int64_t)S * ACQ_CHUNKS;
    acq_level_kernel<<<(unsigned)(items < ctas ? items : ctas), ACQ_THREADS, 0, st>>>(job, iq, stride, osc, cos_tab, S, level, l1sum);
}

} // namespace dabb
