// viterbi.cu — batched K=7 rate-1/4 Viterbi for FIC and MSC codewords on sm_90a, plus the de-puncturing /
// time-de-interleaving kernels that feed it.
//
//   msc_collect_kernel   MscHandler::processMscBlock CIF slicing (msc-handler.cpp:129-158) into a residue-major ring
//   msc_gather_kernel    DabAudio::run time de-interleaver (dab-audio.cpp:113-149): the punctured fragment of one CIF, contiguous
//   viterbi_kernel       de-puncturing (fic-handler.cpp:144-191, eep-protection.cpp:115-152, uep-protection.cpp:169-239) +
//                        Viterbi::deconvolve (viterbi.cpp:227-339) + energy de-dispersal (energy_dispersal.h:35-54,
//                        fic-handler.cpp:199-201) + MSB-first byte pack (decoder_adapter.cpp:57-67)
//   fic_crc_kernel       check_CRC_bits per FIB (MathHelper.h:53-80)
//
// viterbi_kernel: one codeword per thread, 64 path metrics packed 2x16 bit in 32 registers (viterbi_core.cuh).  The kernel reads
// the PUNCTURED softbits (FIC: straight from the OFDM kernel's output; MSC: the gathered fragment): per 24 trellis steps every
// thread stages the 16-byte aligned 128 bytes that hold its next <= 96 softbits into shared memory with cp.async.bulk (TMA,
// completion on an mbarrier, 3-stage ring) and expands them itself - the puncturing pattern is the same for every codeword of a
// CTA (of the launch, or of the CTA's profile in a grouped MSC launch, vit_groups.cuh), so the byte selector / mask /
// window-advance flag of each step come from one small table (build_vit_tables) and the expansion of a step is PRMT + LOP3 + IADD.  Decision words go to HBM/L2 as 8 bytes per step per codeword and are read back by
// the same thread for the traceback.  Issue-slot bound (integer ACS).
#include "common.cuh"
#include "viterbi_core.cuh"
#include "viterbi.cuh"
#include <vector>

namespace dabb {

namespace {

// ------------------------------------------------------------------------------------------------ helpers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ------------------------------------------------------------------------------------------------ prep kernels
// MSC collect: copy the sub-channel's slice of each of this frame's 4 CIFs into the de-interleaver ring, residue-major:
// ring[(stream*slots + slot)][cif mod 20][r][j] = softbit (start_cu*64 + r + 16 j) of that CIF.
// One thread per capacity unit (64 softbits = 4 values of j for each of the 16 residues): four 16-byte loads, a 4x4 byte
// transpose per word with PRMT, sixteen 4-byte stores that are lane-consecutive in j.
__global__ void __launch_bounds__(128)
msc_collect_kernel(MscCollectParams p)
{
    const int s = blockIdx.x / 4, c = blockIdx.x % 4, t = threadIdx.x;
    if (p.active && !p.active[s]) return;
    const MscSlotState st = p.slots[s * p.n_slots + p.slot];
    if (!st.enabled) return;
    const int frag = st.frag, per = frag / 16;
    // CIF c of this frame = symbols 4+18c .. 21+18c -> softbits [(3+18c)*3072, +55296)
    const uint4* src = reinterpret_cast<const uint4*>(p.soft + (int64_t)s * p.soft_stride + (int64_t)(3 + 18 * c) * 3072 + (int64_t)st.start_cu * 64);
    const int slice = (int)((st.cif_count + c) % MSC_RING);
    uint32_t* dst = reinterpret_cast<uint32_t*>(p.ring + ((int64_t)s * MSC_RING + slice) * p.ring_pitch);
    const int per_w = per / 4;
    for (int jq = t; jq < per_w; jq += 128) {
        const uint4 a0 = __ldg(src + 4 * jq), a1 = __ldg(src + 4 * jq + 1), a2 = __ldg(src + 4 * jq + 2), a3 = __ldg(src + 4 * jq + 3);
        const uint32_t w0[4] = {a0.x, a0.y, a0.z, a0.w}, w1[4] = {a1.x, a1.y, a1.z, a1.w}, w2[4] = {a2.x, a2.y, a2.z, a2.w}, w3[4] = {a3.x, a3.y, a3.z, a3.w};
#pragma unroll
        for (int q = 0; q < 4; q++) {
            const uint32_t t0 = __byte_perm(w0[q], w1[q], 0x5140), t1 = __byte_perm(w2[q], w3[q], 0x5140);
            const uint32_t t2 = __byte_perm(w0[q], w1[q], 0x7362), t3 = __byte_perm(w2[q], w3[q], 0x7362);
            dst[(4 * q + 0) * per_w + jq] = __byte_perm(t0, t1, 0x5410);
            dst[(4 * q + 1) * per_w + jq] = __byte_perm(t0, t1, 0x7632);
            dst[(4 * q + 2) * per_w + jq] = __byte_perm(t2, t3, 0x5410);
            dst[(4 * q + 3) * per_w + jq] = __byte_perm(t2, t3, 0x7632);
        }
    }
}

// MSC gather: one CTA per (stream, CIF c).  Copies the 16 residue rows of the time-de-interleaved fragment
// (out[i] = CIF[n - (16 - map[i & 15])][i], dab-audio.cpp:113-143) from the ring into shared memory, still residue-major
// (row r at word stride `sw`, odd so that the 16 rows start in different banks), and writes the fragment in natural order
// (softbit i of the fragment sits at (i & 15) * 4 sw + (i >> 4) in shared memory) as one 4-byte store per thread and word.
__constant__ int c_deint_delay[16] = {16, 8, 12, 4, 14, 6, 10, 2, 15, 7, 11, 3, 13, 5, 9, 1};   // 16 - map[r]
__global__ void __launch_bounds__(128)
msc_gather_kernel(MscPrepParams p)
{
    extern __shared__ __align__(16) int8_t frag_s[];
    const int s = blockIdx.x / 4, c = blockIdx.x % 4, t = threadIdx.x;
    if (p.active && !p.active[s]) return;
    const MscSlotState st = p.slots[s * p.n_slots + p.slot];
    if (!st.enabled) return;
    const int64_t n = st.cif_count + c;           // index (since selection) of the CIF being completed
    if (n < 16) return;                           // de-interleaver not yet filled (dab-audio.cpp:146-149)
    const int frag = st.frag, per_w = frag / 64, sw = per_w | 1;
    const int8_t* ring = p.ring + (int64_t)s * MSC_RING * p.ring_pitch;
    uint32_t* frag_w = reinterpret_cast<uint32_t*>(frag_s);
    const int nm = (int)(n % MSC_RING);           // one 64-bit modulo; the 16 slices follow with 32-bit arithmetic
    // phase 1: the 16 residue rows, flattened over the CTA (16 per_w words; every thread has all its loads in flight at once)
    const int total = 16 * per_w;
    const uint32_t magic = 0xFFFFFFFFu / (uint32_t)per_w + 1u;      // idx / per_w = umulhi(idx, magic) for idx < 2^16
#pragma unroll 4
    for (int idx = t; idx < total; idx += 128) {
        const int r = (int)__umulhi((uint32_t)idx, magic), j = idx - r * per_w;
        int slice = nm - c_deint_delay[r];        // delay <= 16 < MSC_RING
        if (slice < 0) slice += MSC_RING;
        frag_w[r * sw + j] = __ldg(reinterpret_cast<const uint32_t*>(ring + (int64_t)slice * p.ring_pitch) + r * per_w + j);
    }
    __syncthreads();
    // phase 2: natural order.  Word j of row r holds softbits r + 16 (4j .. 4j+3); output word q = bytes 4q .. 4q+3 = residues
    // 4 (q & 3) .. +3 of column q >> 2.  One thread per column word j: four 4x4 byte transposes (PRMT, as in msc_collect_kernel)
    // turn its 16 row words into the 16 consecutive output words 16 j .. 16 j + 15 (four 16-byte stores).
    const int cw = s * 4 + c;
    uint4* dst = reinterpret_cast<uint4*>(p.frag_out + (int64_t)cw * p.frag_pitch);
    for (int j = t; j < per_w; j += 128) {
        uint32_t o[4][4];        // [column m][residue group g]
#pragma unroll
        for (int g = 0; g < 4; g++) {
            const uint32_t w0 = frag_w[(4 * g + 0) * sw + j], w1 = frag_w[(4 * g + 1) * sw + j], w2 = frag_w[(4 * g + 2) * sw + j], w3 = frag_w[(4 * g + 3) * sw + j];
            const uint32_t t0 = __byte_perm(w0, w1, 0x5140), t1 = __byte_perm(w2, w3, 0x5140);
            const uint32_t t2 = __byte_perm(w0, w1, 0x7362), t3 = __byte_perm(w2, w3, 0x7362);
            o[0][g] = __byte_perm(t0, t1, 0x5410); o[1][g] = __byte_perm(t0, t1, 0x7632);
            o[2][g] = __byte_perm(t2, t3, 0x5410); o[3][g] = __byte_perm(t2, t3, 0x7632);
        }
#pragma unroll
        for (int m = 0; m < 4; m++) dst[4 * j + m] = make_uint4(o[m][0], o[m][1], o[m][2], o[m][3]);
    }
    if (t == 0 && p.valid) p.valid[cw] = 1;
}

// stage-level API helper: copy with -128 -> -127 (both are symbol 0 after the reference's clamp, viterbi.cpp:232-237), so that the
// decoder kernel may form symbols without a saturating subtract
__global__ void clamp_copy_kernel(const int8_t* src, int8_t* dst, int64_t n)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) { const int8_t v = src[i]; dst[i] = v == -128 ? (int8_t)-127 : v; }
}

// ------------------------------------------------------------------------------------------------ the decoder
constexpr int VIT_THREADS = VIT_GROUP_CW;     // codewords per CTA (vit_groups.cuh: the grouped schedule's descriptors hold as many)
// Three CTAs per SM (168 registers a thread) rather than four (128): a launch of up to 396 CTAs (50 688 codewords) is still one wave, and
// the headline batch's FIC and MSC launches (128 CTAs) are one CTA per SM either way.  At 128 registers the add-compare-select's per-step
// constants spilled the fragment address and left ptxas little room to overlap the butterflies of a step; at 168 the same launches run
// 5-9 % faster.
constexpr int VIT_MIN_CTAS = 3;
constexpr int VIT_ROW_PITCH = 144;      // 128 B of softbits + 16 B pad (rows stay 16-byte aligned for the bulk copies)
constexpr int VIT_STAGE_BYTES = VIT_THREADS * VIT_ROW_PITCH;
constexpr int VIT_STAGES = 3;           // depth of the staging ring: stage s + 3 is requested while stage s is decoded

constexpr int VIT_WARPS = VIT_THREADS / 32;
constexpr int VIT_TAB_BYTES = VIT_STAGE_STEPS * 8;      // one stage's expansion entries (24 x 8 bytes = 12 x 16)
struct __align__(16) VitSmem {
    unsigned char stage[VIT_STAGES][VIT_STAGE_BYTES];        // per thread: the 128 bytes that hold its next <= 96 softbits
    unsigned char tab[VIT_STAGES][VIT_WARPS][VIT_TAB_BYTES]; // per warp: the stage's expansion entries
};

// per-thread asynchronous copy global -> shared, 16 bytes (SASS: LDGSTS); completion by commit / wait groups of the issuing thread
__device__ __forceinline__ void cp_async16(void* dst_smem, const void* src_gmem)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst_smem)), "l"(src_gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// What one CTA decodes.  Ungrouped: codewords 128 b .. 128 b + 127 (below n_cw) with the launch's tables.  Grouped: the codewords and
// the profile of descriptor b (vit_groups.cuh); every CTA still has one profile, so all the warp-uniform structure below holds.
struct VitJob {
    const uint2* steptab; const uint32_t* stage_off;
    int nsteps;
    int cw; bool have;               // this thread's codeword (a valid index even where have is false)
    uint2* dec;                      // this thread's first decision word
    const VitProfile* prof;          // grouped: the CTA's profile (its energy-dispersal words are read for the traceback)
};
template <bool GROUPED>
__device__ __forceinline__ bool viterbi_job(const ViterbiParams& p, const int block, const int t, VitJob& j)
{
    if constexpr (GROUPED) {
        const VitGroup g = p.groups[block];
        if (g.count == 0) return false;                              // a slot without enabled streams
        j.prof = p.profiles + g.profile;
        j.steptab = j.prof->steptab; j.stage_off = j.prof->stage_off; j.nsteps = j.prof->nsteps;
        j.have = t < g.count;
        j.cw = __ldg(p.cw_list + g.first + (j.have ? t : 0));
        j.dec = p.dec + g.dec_off + t;
    } else {
        j.steptab = p.steptab; j.stage_off = p.stage_off; j.nsteps = p.nsteps; j.prof = nullptr;
        const int cw = block * VIT_THREADS + t;
        j.have = cw < p.n_cw;
        j.cw = j.have ? cw : 0;
        j.dec = p.dec + (int64_t)block * p.nsteps * VIT_THREADS + t;
    }
    return true;
}
// the output length and dispersal words of the job's codewords, read after the forward pass
template <bool GROUPED> __device__ __forceinline__ int vit_job_nbits(const ViterbiParams& p, const VitJob& j) { return GROUPED ? j.prof->nbits : p.nbits; }
template <bool GROUPED> __device__ __forceinline__ const uint32_t* vit_job_prbs(const ViterbiParams& p, const VitJob& j) { return GROUPED ? j.prof->prbs_words : p.prbs_words; }

// traceback of one codeword (vit_traceback24): 96 steps (nbits is a multiple of 96) give three output words; the decision words are read
// in batches of 24 independent loads (their addresses do not depend on the path).  dec: this thread's first decision word (stride
// VIT_THREADS per step)
__device__ __forceinline__ void viterbi_traceback(const ViterbiParams& p, const int cw, const uint2* dec, const int nbits, const uint32_t* prbs)
{
    if (p.valid && !p.valid[cw]) return;
    uint32_t state = 0;
    uint32_t* out = reinterpret_cast<uint32_t*>(p.out + (int64_t)cw * p.out_stride);
    for (int tb = nbits - 96; tb >= 0; tb -= 96) {
        uint32_t acc[3] = {0, 0, 0};
        vit_u2 d[24];
        // the decision words of a 32 768-codeword launch (0.6 GB) have mostly left the L2 by the time the traceback wants them: the batch
        // after next (48 steps further down) is requested into the L2 while this one is walked
#define VIT_TB_QUARTER(Q) do { \
            _Pragma("unroll") for (int k = 0; k < 24; k++) { const uint2 v = dec[(int64_t)(tb + 24 * (Q) + k + 6) * VIT_THREADS]; d[k].x = v.x; d[k].y = v.y; } \
            if (tb + 24 * (Q) - 48 + 6 >= 0) { _Pragma("unroll") for (int k = 0; k < 24; k++) asm volatile("prefetch.global.L2 [%0];" ::"l"(dec + (int64_t)(tb + 24 * (Q) - 48 + k + 6) * VIT_THREADS)); } \
            vit_traceback24<(Q)>(state, d, acc); } while (0)
        VIT_TB_QUARTER(3); VIT_TB_QUARTER(2); VIT_TB_QUARTER(1); VIT_TB_QUARTER(0);
#undef VIT_TB_QUARTER
#pragma unroll
        for (int j = 0; j < 3; j++) {
            const uint32_t v = vit_pack_be(acc[2 - j]);          // acc[2 - j]: the times tb + 32 j .. tb + 32 j + 31
            const int wi = (tb >> 5) + j;
            out[wi] = prbs ? v ^ prbs[wi] : v;
        }
    }
}

// Staging.  Every thread owns one codeword and reads only ITS OWN row of a stage buffer, so its data needs no CTA-wide barrier: it
// copies the 16-byte aligned 128 bytes that cover the stage's softbits with eight per-thread cp.async, three stages ahead, and waits
// for its own copy groups.  (Round 1 / the first version of this round used one cp.async.bulk per thread: the bulk engine takes its
// addresses from uniform registers, so the compiler emitted a 32-iteration lane loop per warp and stage - ncu: 10 % of the samples.)
// The stage's expansion entries (the same for all codewords) are copied once per WARP by twelve of its lanes into a warp-private
// area and read after a __syncwarp: no __syncthreads in the loop at all.
template <bool GROUPED>
__device__ __forceinline__ void viterbi_cta(const ViterbiParams& p, const int block)
{
    extern __shared__ __align__(16) unsigned char smraw[];
    VitSmem& sm = *reinterpret_cast<VitSmem*>(smraw);
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const unsigned long long trace_t0 = p.trace.rec ? trace_now() : 0ull;
    VitJob job;
    if (!viterbi_job<GROUPED>(p, block, t, job)) return;
    const int cw = job.cw;
    const bool have = job.have;
    const int groups = job.nsteps / 6;               // 6 steps per group, 4 groups per stage
    const int nstages = (groups + 3) / 4;
    const uint32_t* stage_off = job.stage_off;
    const unsigned char* frag = reinterpret_cast<const unsigned char*>(p.frag) + (int64_t)(cw / p.cw_div) * p.outer_stride + (int64_t)(cw % p.cw_div) * p.inner_stride;
    const unsigned char* tabsrc = reinterpret_cast<const unsigned char*>(job.steptab);

    // stage s needs the softbits [stage_off[s], stage_off[s+1]) of the fragment; always one commit group per call
    auto issue = [&](int s, int buf) {
        if (s < nstages) {
            const unsigned char* src = frag + (__ldg(stage_off + s) & ~15u);
            unsigned char* dst = &sm.stage[buf][t * VIT_ROW_PITCH];
#pragma unroll
            for (int k = 0; k < 8; k++) cp_async16(dst + 16 * k, src + 16 * k);
            if (lane < VIT_TAB_BYTES / 16) cp_async16(&sm.tab[buf][warp][16 * lane], tabsrc + (size_t)s * VIT_TAB_BYTES + 16 * lane);   // table is padded to whole stages
        }
        cp_async_commit();
    };
    for (int s = 0; s < VIT_STAGES; s++) issue(s, s);

    uint32_t Q[32];
    vit_init(Q);
    uint2* dec = job.dec;

    for (int s = 0; s < nstages; s++) {
        const int buf = s % VIT_STAGES;
        cp_async_wait<VIT_STAGES - 1>();            // this thread's copies of stage s have landed ...
        __syncwarp();                               // ... and so have the other lanes' parts of the warp's table
        vit_normalize(Q);
        // 8-byte window (w0, w1) over the thread's row; everything about the window but its content is the same for all threads
        const uint32_t* my = reinterpret_cast<const uint32_t*>(&sm.stage[buf][t * VIT_ROW_PITCH]);
        const uint2* tab = reinterpret_cast<const uint2*>(&sm.tab[buf][warp][0]);
        int nx = (int)((__ldg(stage_off + s) & 15u) >> 2);
        uint32_t w0 = my[nx], w1 = my[nx + 1];
        nx += 2;
        // the expansion of group g + 1 (table loads, window loads) is issued before the add-compare-select of group g: independent work
        // the scheduler interleaves, so that the window's load latency does not sit in front of every six steps
        auto expand = [&](int gq, uint32_t (&wo)[6]) {
#pragma unroll
            for (int k = 0; k < 6; k++) {
                const uint2 e = tab[6 * gq + k];                         // {byte selector | advance << 16, byte mask}: a broadcast read
                wo[k] = vit_expand_step(w0, w1, e.x, e.y);
                if (e.x & 0x10000u) { w0 = w1; w1 = my[nx]; nx++; }       // warp-uniform
            }
        };
        uint32_t wn[6];
        if (4 * s < groups) expand(0, wn);
#pragma unroll 1
        for (int gq = 0; gq < 4; gq++) {
            const int g = 4 * s + gq;
            if (g >= groups) break;
            uint32_t w[6];
#pragma unroll
            for (int k = 0; k < 6; k++) w[k] = wn[k];
            if (gq < 3 && g + 1 < groups) expand(gq + 1, wn);
            uint32_t d[12];
            vit_six_steps(Q, w, d);
            if (have) {
#pragma unroll
                for (int k = 0; k < 6; k++) dec[(int64_t)(6 * g + k) * VIT_THREADS] = make_uint2(d[2 * k], d[2 * k + 1]);
            }
        }
        __syncwarp();                               // every lane is done with the warp's table of this buffer before it is refilled
        issue(s + VIT_STAGES, buf);
    }
    cp_async_wait<0>();
    if (p.trace.rec && t == 0) trace_put(p.trace, p.trace_kind, trace_t0);       // forward pass of thread 0 done
    if (!have) return;
    viterbi_traceback(p, cw, dec, vit_job_nbits<GROUPED>(p, job), vit_job_prbs<GROUPED>(p, job));
    if (p.trace.rec && t == 0) trace_put(p.trace, p.trace_kind + 10u, trace_t0);  // ... and its traceback
}

// GROUPED: the MSC launch of a sub-channel slot (ViterbiParams::groups); the FIC and the stage-level entry points use the plain form
template <bool GROUPED>
__global__ void __launch_bounds__(VIT_THREADS, VIT_MIN_CTAS)
viterbi_kernel(ViterbiParams p) { viterbi_cta<GROUPED>(p, blockIdx.x); }


// CRC of the 12 FIBs of a frame (x^16 + x^12 + x^5 + 1, preset ones, inverted remainder; MathHelper.h:53-80): one thread per FIB, 16
// lanes per frame (12 used), the frame's mask assembled with a ballot
__global__ void fic_crc_kernel(const uint8_t* __restrict__ fibs, const int32_t* __restrict__ active, int n_frames, int32_t* __restrict__ mask_out)
{
    const int gt = blockIdx.x * blockDim.x + threadIdx.x;
    const int f = gt >> 4, fib = gt & 15;
    bool ok = false;
    if (f < n_frames && fib < 12 && !(active && !active[f])) {
        const uint4* b4 = reinterpret_cast<const uint4*>(fibs + ((int64_t)f * 12 + fib) * 32);
        const uint4 lo = __ldg(b4), hi = __ldg(b4 + 1);
        const uint32_t w[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
        uint32_t reg = 0xFFFF;
#pragma unroll
        for (int i = 0; i < 32; i++) {
            uint32_t byte = (w[i >> 2] >> (8 * (i & 3))) & 0xFFu;
            if (i >= 30) byte ^= 0xFF;
            reg ^= byte << 8;
#pragma unroll
            for (int k = 0; k < 8; k++) reg = (reg & 0x8000) ? ((reg << 1) ^ 0x1021) & 0xFFFF : (reg << 1) & 0xFFFF;
        }
        ok = reg == 0;
    }
    const uint32_t bits = __ballot_sync(0xFFFFFFFFu, ok);
    if (f < n_frames && fib == 0) mask_out[f] = (int32_t)((bits >> (threadIdx.x & 16)) & 0xFFFu);      // inactive frames: 0
}

// packed bytes -> one bit per byte (stage-level API output format of Viterbi::deconvolve)
__global__ void unpack_bits_kernel(const uint8_t* __restrict__ bytes, int64_t stride, int n_cw, int nbits, uint8_t* __restrict__ bits)
{
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (int64_t)n_cw * nbits) return;
    const int cw = (int)(idx / nbits), b = (int)(idx % nbits);
    bits[idx] = (bytes[(int64_t)cw * stride + (b >> 3)] >> (7 - (b & 7))) & 1;
}

} // namespace

void build_vit_tables_u2(const int16_t* map, int nsteps, std::vector<uint2>& steps, std::vector<uint32_t>& stage_off)
{
    build_vit_tables(map, nsteps, steps, stage_off);     // viterbi_core.cuh
    while (steps.size() % VIT_STAGE_STEPS) steps.push_back(make_uint2(0, 0));      // the kernel copies whole stages of the table
}

void launch_clamp_copy(const int8_t* src, int8_t* dst, int64_t n, cudaStream_t st)
{
    clamp_copy_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(src, dst, n);
}

void launch_msc_collect(const MscCollectParams& p, int n_streams, cudaStream_t st) { msc_collect_kernel<<<n_streams * 4, 128, 0, st>>>(p); }
void launch_msc_gather(const MscPrepParams& p, int n_streams, cudaStream_t st)
{
    const int smem = p.ring_pitch + 64;      // 16 residue rows, each padded to an odd word count
    if (smem > 48 * 1024) cudaFuncSetAttribute(msc_gather_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    msc_gather_kernel<<<n_streams * 4, 128, smem, st>>>(p);
}

template <bool GROUPED> void launch_viterbi_t(const ViterbiParams& p, const int blocks, cudaStream_t st)
{
    cudaFuncSetAttribute(viterbi_kernel<GROUPED>, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared);
    cudaFuncSetAttribute(viterbi_kernel<GROUPED>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(VitSmem));
    viterbi_kernel<GROUPED><<<blocks, VIT_THREADS, sizeof(VitSmem), st>>>(p);
}

void launch_viterbi(const ViterbiParams& p, cudaStream_t st)
{
    if (p.groups) launch_viterbi_t<true>(p, p.n_groups, st);
    else launch_viterbi_t<false>(p, (p.n_cw + VIT_THREADS - 1) / VIT_THREADS, st);
}

size_t vit_dec_bytes(int n_cw, int nsteps) { return (size_t)((n_cw + VIT_THREADS - 1) / VIT_THREADS) * nsteps * VIT_THREADS * sizeof(uint2); }

void launch_fic_crc(const uint8_t* fibs, const int32_t* active, int n_frames, int32_t* mask_out, cudaStream_t st)
{
    fic_crc_kernel<<<(n_frames * 16 + 127) / 128, 128, 0, st>>>(fibs, active, n_frames, mask_out);
}

void launch_unpack_bits(const uint8_t* bytes, int64_t stride, int n_cw, int nbits, uint8_t* bits, cudaStream_t st)
{
    const int64_t total = (int64_t)n_cw * nbits;
    unpack_bits_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(bytes, stride, n_cw, nbits, bits);
}

} // namespace dabb
