// chan.cu — the wideband channelizer (dabb_channelize): one CTA per (channel, block of consecutive outputs).  The CTA converts and mixes
// the block's input span [n_first - TP + 1, n_last] into shared memory once, then every thread sums the TP taps of its outputs from
// there, the taps read as groups of four from the packed table (chan_core.cuh: consecutive outputs read consecutive groups, so a warp's
// tap loads are contiguous; with L = 1 they are one broadcast).  The arithmetic is chan_core.cuh's, shared with the host build.
#include "common.cuh"
#include "chan_core.cuh"

namespace dabb {

using namespace dabb_channel;

__global__ void __launch_bounds__(CHAN_THREADS) chan_kernel(const ChanParams p)
{
    extern __shared__ cf xs[];
    const int c = blockIdx.y;
    const int64_t b0 = (int64_t)blockIdx.x * p.block_out;
    const int nb = (int)min((int64_t)p.block_out, p.out_len - b0);
    const int64_t m0 = p.out_start[c] + b0;
    const int64_t n_lo = last_input(m0, p.L, p.M) - (p.TP - 1);
    const int span = (int)(last_input(m0 + nb - 1, p.L, p.M) - n_lo + 1);
    const int i = p.input_of[c];
    const uint8_t* in = p.in + (size_t)i * (size_t)p.in_stride * (size_t)bytes_per_sample(p.fmt);
    const int64_t first = p.in_start[i], end = first + p.in_len;
    // the mixer's phase index advances by fm per sample: exact integers, one 64-bit remainder per thread
    const int64_t fm = p.fmod[c], R = p.R, step = (fm * CHAN_THREADS) % R;
    int64_t k = phase_index(fm, n_lo + threadIdx.x, R);
    for (int s = threadIdx.x; s < span; s += CHAN_THREADS) {
        const int64_t n = n_lo + s;
        cf v{0.f, 0.f};
        if (n >= first && n < end) {        // the TP - T samples in front of the first output's span may lie outside the buffer; no output reads them
            float sn, cs;
            sincospif(mixer_arg(k, R, p.inv_r), &sn, &cs);
            v = mix(in_sample(in, n - first, p.fmt), sn, cs);
        }
        xs[s] = v;
        k += step;
        if (k >= R) k -= R;
    }
    __syncthreads();
    float2* out = p.out + (size_t)c * (size_t)p.out_stride + b0;
    for (int o = threadIdx.x; o < nb; o += CHAN_THREADS) {
        const int64_t m = m0 + o;
        const cf y = dot(xs + (last_input(m, p.L, p.M) - n_lo), p.taps + floor_mod(m, p.L), p.L, p.T);
        out[o] = make_float2(y.x, y.y);
    }
}

int chan_block_outputs(int L, int M, int TP)
{
    for (int opt = 4; opt > 1; opt /= 2)
        if (chan_span_cap(opt * CHAN_THREADS, L, M, TP) * (int64_t)sizeof(cf) <= 64 * 1024) return opt * CHAN_THREADS;
    return CHAN_THREADS;
}

int64_t chan_span_cap(int block_out, int L, int M, int TP) { return ((int64_t)(block_out - 1) * M) / L + 1 + TP; }

cudaError_t launch_chan(const ChanParams& p, int n_channels, cudaStream_t st)
{
    const size_t smem = (size_t)chan_span_cap(p.block_out, p.L, p.M, p.TP) * sizeof(cf);
    const cudaError_t e = cudaFuncSetAttribute(chan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    const dim3 grid((unsigned)((p.out_len + p.block_out - 1) / p.block_out), (unsigned)n_channels);
    chan_kernel<<<grid, CHAN_THREADS, smem, st>>>(p);
    return cudaSuccess;
}

} // namespace dabb
