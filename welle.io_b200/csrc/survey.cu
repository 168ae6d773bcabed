// survey.cu — the spectrum survey (dabb_survey): one CTA per (chunk of consecutive Welch segments, input).  For each segment the CTA
// converts and windows the nfft samples into shared memory (natural order, coalesced loads), runs the log2(nfft) radix-2 stages in place,
// and every thread adds |X|^2 of its own nfft / SURVEY_THREADS storage positions into registers; the chunk's sums go to its row of the
// partial buffer in storage (bit-reversed) order.  survey_sum_kernel then adds the rows of each input in ascending chunk order in double,
// un-reverses and shifts the bins, and scales.  The arithmetic is survey_core.cuh's, shared with the host build.
#include "common.cuh"
#include "survey_core.cuh"

namespace dabb {

using namespace dabb_spectrum;

template <int LOG2N>
__global__ void __launch_bounds__(SURVEY_THREADS) survey_kernel(const SurveyParams p)
{
    constexpr int N = 1 << LOG2N, PER = N / SURVEY_THREADS;
    extern __shared__ cf a[];
    const int input = blockIdx.y;
    const int64_t s0 = (int64_t)blockIdx.x * p.chunk;
    const int64_t s1 = min(s0 + p.chunk, p.S);
    const uint8_t* in = p.in + (size_t)input * (size_t)p.in_stride * (size_t)dabb_channel::bytes_per_sample(p.fmt);
    float acc[PER];
#pragma unroll
    for (int q = 0; q < PER; q++) acc[q] = 0.f;
    for (int64_t s = s0; s < s1; s++) {
        const uint8_t* seg = in + (size_t)(s * (N / 2)) * (size_t)dabb_channel::bytes_per_sample(p.fmt);
#pragma unroll
        for (int q = 0; q < PER; q++) { const int n = threadIdx.x + q * SURVEY_THREADS; a[n] = windowed(seg, n, p.fmt, p.win, LOG2N); }
        __syncthreads();
        for (int lh = LOG2N - 1; lh >= 0; lh--) {
#pragma unroll
            for (int q = 0; q < PER / 2; q++) butterfly(a, lh, threadIdx.x + q * SURVEY_THREADS, p.tw, LOG2N);
            __syncthreads();
        }
#pragma unroll
        for (int q = 0; q < PER; q++) { const cf x = a[threadIdx.x + q * SURVEY_THREADS]; acc[q] += x.x * x.x + x.y * x.y; }
        __syncthreads();
    }
    float* row = p.part + ((size_t)input * gridDim.x + blockIdx.x) * N;
#pragma unroll
    for (int q = 0; q < PER; q++) row[threadIdx.x + q * SURVEY_THREADS] = acc[q];
}

// one thread per (input, storage position): the chunk rows are read in storage order (coalesced), and only the final store goes to the
// bin's shifted position
__global__ void survey_sum_kernel(const float* part, int64_t n_chunks, int log2n, int n_inputs, double scale, float* psd)
{
    const int n = 1 << log2n;
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (int64_t)n * n_inputs) return;
    const int input = (int)(t >> log2n), pos = (int)(t & (n - 1));
    const float* col = part + (size_t)input * (size_t)n_chunks * n + pos;
    double sum = 0.0;
    for (int64_t c = 0; c < n_chunks; c++) sum += (double)col[(size_t)c * n];
    psd[(size_t)input * n + (bin_position(pos, log2n) ^ (n / 2))] = (float)(sum * scale);
}

template <int LOG2N> static cudaError_t launch_one(const SurveyParams& p, int n_chunks, int n_inputs, cudaStream_t st)
{
    const size_t smem = sizeof(cf) << LOG2N;
    const cudaError_t e = cudaFuncSetAttribute(survey_kernel<LOG2N>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    survey_kernel<LOG2N><<<dim3((unsigned)n_chunks, (unsigned)n_inputs), SURVEY_THREADS, smem, st>>>(p);
    return cudaSuccess;
}

cudaError_t launch_survey(const SurveyParams& p, int log2n, int64_t n_chunks, int n_inputs, cudaStream_t st)
{
    switch (log2n) {
        case 10: return launch_one<10>(p, (int)n_chunks, n_inputs, st);
        case 11: return launch_one<11>(p, (int)n_chunks, n_inputs, st);
        case 12: return launch_one<12>(p, (int)n_chunks, n_inputs, st);
        case 13: return launch_one<13>(p, (int)n_chunks, n_inputs, st);
        case 14: return launch_one<14>(p, (int)n_chunks, n_inputs, st);
        default: return cudaErrorInvalidValue;
    }
}

void launch_survey_sum(const float* part, int64_t n_chunks, int log2n, int n_inputs, double scale, float* psd, cudaStream_t st)
{
    const int64_t total = (int64_t)n_inputs << log2n;
    survey_sum_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(part, n_chunks, log2n, n_inputs, scale, psd);
}

} // namespace dabb
