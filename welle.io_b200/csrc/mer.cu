// mer.cu — modulation error ratio of each stream's FIC softbits (dabb_set_mer, tap 14), arithmetic in mer_core.cuh.
//
//   mer_kernel   one CTA per stream, 288 threads: thread t reads 16 carriers (16 (t mod 96) ..) of data symbol 1 + t / 96 as one 16-byte
//                load of their Re softbits and one of their Im softbits, and adds u^2 and v^2 into its carriers' groups in shared memory.
//                The sums are integers, so the order of the additions changes nothing.  Every field of every record is written every step
//                (zeros for a stream that decoded no frame), so nothing is cleared beforehand.
#include "../../include/dab_b200.h"
#include "common.cuh"
#include "mer_core.cuh"

namespace dabb {

namespace {

static_assert(sizeof(dabb_mer_result) == 536, "dabb_mer_result");
static_assert(DABB_MER_GROUPS == dabb_mer::GROUPS, "DABB_MER_GROUPS");
constexpr int MER_CHUNKS = dabb_mer::CARRIERS / 16;            // 16-carrier chunks per symbol
constexpr int MER_THREADS = dabb_mer::SYMBOLS * MER_CHUNKS;     // 288

__device__ __forceinline__ int8_t byte_of(const uint4& q, int j)
{
    const uint32_t w = j < 4 ? q.x : (j < 8 ? q.y : (j < 12 ? q.z : q.w));
    return (int8_t)(w >> (8 * (j & 3)));
}

__global__ void __launch_bounds__(MER_THREADS) mer_kernel(MerParams p)
{
    __shared__ int32_t gsig[dabb_mer::GROUPS], gerr[dabb_mer::GROUPS], npoints;
    const int s = blockIdx.x, t = threadIdx.x;
    dabb_mer_result* rec = static_cast<dabb_mer_result*>(p.res) + s;
    if (!p.active[s]) {                             // no frame decoded: all zero
        int32_t* w = reinterpret_cast<int32_t*>(rec);
        for (int i = t; i < (int)(sizeof(dabb_mer_result) / 4); i += MER_THREADS) w[i] = 0;
        return;
    }
    if (t < dabb_mer::GROUPS) { gsig[t] = 0; gerr[t] = 0; }
    if (t == 0) npoints = 0;
    __syncthreads();
    const int sym = t / MER_CHUNKS, c = t - sym * MER_CHUNKS;
    const int8_t* row = p.soft + (int64_t)s * p.soft_stride + (int64_t)sym * (2 * dabb_mer::CARRIERS) + 16 * c;
    const uint4 re = __ldg(reinterpret_cast<const uint4*>(row));
    const uint4 im = __ldg(reinterpret_cast<const uint4*>(row + dabb_mer::CARRIERS));
    const uint4 grp = __ldg(reinterpret_cast<const uint4*>(p.group + 16 * c));
    int n = 0;
#pragma unroll
    for (int j = 0; j < 16; j++) {
        int32_t u2, v2;
        dabb_mer::point(byte_of(re, j), byte_of(im, j), u2, v2);
        const int g = (uint8_t)byte_of(grp, j);
        n += u2 > 0;
        atomicAdd(&gsig[g], u2);
        atomicAdd(&gerr[g], v2);
    }
    n = (int)__reduce_add_sync(0xFFFFFFFFu, (unsigned)n);
    if ((t & 31) == 0) atomicAdd(&npoints, n);
    __syncthreads();
    if (t < dabb_mer::GROUPS) { rec->group[t].sig = gsig[t]; rec->group[t].err = gerr[t]; }
    if (t == 0) {
        int64_t sig = 0, err = 0;
        for (int g = 0; g < dabb_mer::GROUPS; g++) { sig += gsig[g]; err += gerr[g]; }
        rec->points = npoints; rec->mer_db = dabb_mer::mer_db(sig, err); rec->sig = sig; rec->err = err;
    }
}

} // namespace

void launch_mer(const MerParams& p, cudaStream_t st)
{
    mer_kernel<<<p.n_streams, MER_THREADS, 0, st>>>(p);
}

} // namespace dabb
