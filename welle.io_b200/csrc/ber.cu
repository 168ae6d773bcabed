// ber.cu — channel bit errors of the step's decoded codewords (dabb_options.count_bit_errors, tap 10), arithmetic in ber_core.cuh.
//
//   ber_kernel   one CTA per (stream, part): part 0 = the frame's four FIC codewords, part 1 + k = the logical frames slot k decoded.
//                The CTA's threads take the 32-bit chunks of those codewords in order (adjacent threads read adjacent softbits and
//                decoded bytes), and the CTA writes its sums into the stream's record: every field of every record is written every
//                step, so nothing is cleared beforehand and no atomics are needed.
#include "../../include/dab_b200.h"
#include "common.cuh"
#include "viterbi.cuh"

namespace dabb {

namespace {

static_assert(DABB_MAX_SUBCH == 4, "BerParams::slot has one entry per slot");
static_assert(sizeof(dabb_ber_result) == 80, "dabb_ber_result");
constexpr int BER_THREADS = 128;

__global__ void __launch_bounds__(BER_THREADS) ber_kernel(BerParams p)
{
    __shared__ dabb_ber::Profile prof;
    __shared__ uint32_t red[BER_THREADS / 32][3];
    const int s = blockIdx.x, part = blockIdx.y, t = threadIdx.x;
    int32_t* rec = reinterpret_cast<int32_t*>(static_cast<dabb_ber_result*>(p.res) + s) + 4 * part;   // fic_* or subch[part - 1]
    // the part's codewords (cw_mask bit c: codeword c was decoded in this step) and their profile
    int profile = -1;
    uint32_t cw_mask = 0;
    const int8_t* soft0 = nullptr; int64_t soft_step = 0;
    const uint8_t* out0 = nullptr; int64_t out_step = 0;
    if (part == 0) {
        if (p.active[s]) { profile = p.fic_profile; cw_mask = 0xFu; }
        soft0 = p.soft + (int64_t)s * p.soft_stride; soft_step = 2304;
        out0 = p.fibs + (int64_t)s * 4 * 96; out_step = 96;
    } else if (part - 1 < p.n_slots && p.slot[part - 1].frag) {
        const BerSlot sl = p.slot[part - 1];
        for (int c = 0; c < 4; c++) if (sl.valid[s * 4 + c]) cw_mask |= 1u << c;
        if (cw_mask) profile = p.slots[s * p.n_slots + part - 1].profile;
        soft0 = sl.frag + (int64_t)s * 4 * sl.frag_pitch; soft_step = sl.frag_pitch;
        out0 = sl.logical + (int64_t)s * 4 * sl.logical_stride; out_step = sl.logical_stride;
    }
    if (profile < 0) {                              // nothing decoded: all zero
        if (t < 4) rec[t] = 0;
        return;
    }
    {
        const uint32_t* src = reinterpret_cast<const uint32_t*>(p.profiles + profile);
        for (int i = t; i < (int)(sizeof(dabb_ber::Profile) / 4); i += BER_THREADS) reinterpret_cast<uint32_t*>(&prof)[i] = src[i];
    }
    __syncthreads();
    const int n_cw = __popc(cw_mask), nch = prof.nchunks, total = n_cw * nch;
    dabb_ber::Counts cnt{0u, 0u, 0u};
    for (int idx = t; idx < total; idx += BER_THREADS) {
        const int i = idx / nch, j = idx - i * nch;
        const int c = (int)__fns(cw_mask, 0, i + 1);       // the i-th decoded codeword
        dabb_ber::count_chunk(prof, j, soft0 + c * soft_step, out0 + c * out_step, cnt);
    }
    uint32_t v[3] = {cnt.bits, cnt.errors, cnt.erasures};
#pragma unroll
    for (int q = 0; q < 3; q++) v[q] = __reduce_add_sync(0xFFFFFFFFu, v[q]);
    if ((t & 31) == 0) for (int q = 0; q < 3; q++) red[t >> 5][q] = v[q];
    __syncthreads();
    if (t == 0) {
        uint32_t sum[3] = {0u, 0u, 0u};
        for (int w = 0; w < BER_THREADS / 32; w++) for (int q = 0; q < 3; q++) sum[q] += red[w][q];
        if (part == 0) { rec[0] = (int32_t)sum[0]; rec[1] = (int32_t)sum[1]; rec[2] = (int32_t)sum[2]; rec[3] = 0; }
        else { rec[0] = n_cw; rec[1] = (int32_t)sum[0]; rec[2] = (int32_t)sum[1]; rec[3] = (int32_t)sum[2]; }
    }
}

} // namespace

void launch_ber(const BerParams& p, cudaStream_t st)
{
    ber_kernel<<<dim3((unsigned)p.n_streams, 1 + DABB_MAX_SUBCH), BER_THREADS, 0, st>>>(p);
}

} // namespace dabb
