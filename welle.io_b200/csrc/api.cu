// api.cu — the C ABI of include/dab_b200.h: context, per-stream receiver state, the per-frame pipeline and the
// stage-level entry points.  Host code here only sequences kernels on the context's stream; all signal processing
// is in ofdm.cu / viterbi.cu / rs.cu and the small state-machine kernels below.  There is no CPU fallback.
#include "../../include/dab_b200.h"
#include "common.cuh"
#include "viterbi.cuh"
#include "survey_core.cuh"
#include "mer_core.cuh"
#include <cmath>
#include <cstdio>
#include <cstring>
#include <algorithm>
#include <memory>
#include <string>
#include <vector>

using namespace dabb;

namespace {

// per-stream receiver state (device resident), the variables OFDMProcessor carries between frames
// (ofdm-processor.h: coarseCorrector, fineCorrector, localPhase, sLevel) + FicHandler::fic_decode_success_ratio
struct StreamState {
    int64_t pos;            // logical sample index of the next sample to read
    int32_t coarse, fine;   // Hz; fine has int16 semantics
    int32_t local_phase;    // localPhase after the last sample read
    int32_t acq_failed;     // failed null searches since the last result record (acquire_kernel counts, advance_kernel hands over)
    int32_t acquired;       // 0: null search needed, 1: tracking
    int32_t started;        // 0: sLevel warm-up (T_F/2 samples) not done yet
    float slevel;
    int32_t start_index;    // last findIndex
    int64_t nframes;
    dabb_clock::State clk;  // sample-clock estimate (DABB_CLOCK_TRACK, clock_core.cuh): kept through a sync loss, cleared by dabb_stream_reset
};

struct StepScratch {        // per stream, rewritten every step
    int64_t win_start;      // T_u window for findIndex, relative to the stream buffer
    int32_t nco_frame[4];
    int32_t active;         // this stream decodes a frame in this step
    int32_t status;
    // receiver state after this frame, filled by advance_kernel for the result record
    int32_t r_start_index, r_fine, r_coarse;
    float r_fx, r_fy, r_slevel;
    int64_t r_next_pos;
    int64_t null_pos;       // logical index of the first sample of the null symbol that follows this frame
    int32_t null_lp, null_ph;   // NCO phase before that sample, and the increment the null is read with
    int32_t r_acq_failed, pad1;
};

std::string g_create_error;

// Sole owner of one device or pinned host allocation of n elements, freed when the holder is reallocated, reassigned or destroyed.
// It converts to T*, so kernels and copies take it where they take a raw pointer.
template <typename T, bool Pinned> class Owned {
public:
    Owned() = default;
    Owned(const Owned&) = delete;
    Owned& operator=(const Owned&) = delete;
    Owned(Owned&& o) noexcept : p_(o.p_), n_(o.n_) { o.p_ = nullptr; o.n_ = 0; }
    Owned& operator=(Owned&& o) noexcept { if (this != &o) { reset(); p_ = o.p_; n_ = o.n_; o.p_ = nullptr; o.n_ = 0; } return *this; }
    ~Owned() { reset(); }
    // frees the old buffer first; an empty request still gets 16 bytes, so that a successful allocation is never null
    cudaError_t alloc(size_t n)
    {
        reset();
        void* q = nullptr;
        const size_t bytes = n * sizeof(T) > 0 ? n * sizeof(T) : 16;
        const cudaError_t e = Pinned ? cudaHostAlloc(&q, bytes, cudaHostAllocDefault) : cudaMalloc(&q, bytes);
        if (e == cudaSuccess) { p_ = (T*)q; n_ = n; }
        return e;
    }
    void reset() { if (p_) { if (Pinned) cudaFreeHost(p_); else cudaFree(p_); } p_ = nullptr; n_ = 0; }
    T* get() const { return p_; }
    operator T*() const { return p_; }
    size_t size() const { return n_; }
private:
    T* p_ = nullptr;
    size_t n_ = 0;
};
template <typename T> using DevBuf = Owned<T, false>;
template <typename T> using HostBuf = Owned<T, true>;

// where a step's outputs go in the caller's memory (the output half of dabb_io, or a tap's buffer); any pointer may be null
struct StepOut {
    dabb_frame_result* results; uint8_t* fibs; uint8_t* msc; int64_t msc_stride; uint8_t* sf; int64_t sf_stride;
};

// The optional analyses.  Each holds all its device buffers, is built whole when it is first enabled (a failed build leaves the context
// without it) and lives until dabb_destroy; `res` is its tap's records of the last step.
// TII (tii.cu): the null symbol when keep_taps has no tap for it, the spectra (tap 4), each stream's open combinations and their
// phase-error sums, the step's analyses and the tie-order tables
struct Tii {
    DevBuf<float2> null, spectra; DevBuf<dabb_tii::StreamHdr> hdr; DevBuf<dabb_tii::Job> jobs; DevBuf<int32_t> njobs;
    DevBuf<uint32_t> sums; DevBuf<uint16_t> rank; DevBuf<dabb_tii_result> res;
};
// channel bit-error count (ber.cu): the puncturing of every protection profile, then of the FIC, as the count reads it
struct Ber { DevBuf<dabb_ber::Profile> prof; DevBuf<dabb_ber_result> res; };
// sample-clock tracking: [2][S] the ppm each frame of a step is derotated with, double buffered by step parity like the other scratch
struct Clock { DevBuf<float> frame; DevBuf<dabb_clock_result> res; };
// robust acquisition (acq.cu): the cosine table of the block transform, each stream's search span, the block levels and envelope sums
// [S][NB_MAX], the bins the excising find_index instance zeroed [S] (tap 13's `excised`, merged when it is read)
struct Acq { DevBuf<float> cos, level, l1; DevBuf<AcqJob> job; DevBuf<int32_t> exc; DevBuf<dabb_acq_result> res; };
// modulation error ratio (mer.cu): each logical carrier's group [KC]
struct Mer { DevBuf<uint8_t> group; DevBuf<dabb_mer_result> res; };
// diversity combining (combine.cu): the tables of one grouping, built whole by rebuild_comb.  Per group its members and their r1 rows
// (groups) and the (group, symbol) items of combine_kernel; per stream its group or -1 (gid).  Without keep_taps the OFDM kernel stores
// the grouped streams' r1 of their leader's symbols in r1 (row[s], the symbols lmask[s] marks); with it combine_kernel reads tap 2.
struct CombTables {
    std::shared_ptr<const std::vector<int32_t>> leader;     // the leader table they were built from
    int n_items = 0;
    DevBuf<CombGroup> groups; DevBuf<CombItem> items; DevBuf<int32_t> gid, row; DevBuf<uint32_t> lmask; DevBuf<float2> r1;
};
// tab: the current grouping, null while no group of two or more exists
struct Combining { DevBuf<dabb_combine_result> res; std::unique_ptr<CombTables> tab; };

} // namespace

struct dabb_ctx {
    int device = 0; cudaStream_t stream = nullptr; cudaStream_t streamB = nullptr; cudaEvent_t evA[2] = {nullptr, nullptr}, evB[2] = {nullptr, nullptr}; bool evB_valid[2] = {false, false};
    int64_t step = 0; int last_parity = 0; DevBuf<int32_t> d_fic_ratio, d_coarse;
    cudaStream_t stream2 = nullptr; cudaEvent_t ev_ofdm = nullptr, ev_fic = nullptr; DevBuf<uint2> d_dec_fic; int S = 0; int fft_mode = 0; int disable_coarse = 0; int keep_taps = 0; int placement = 0; int freqsync = 0;
    // the optional analyses, null until first enabled, and the options that run them in a step (combining runs while comb->tab exists)
    std::unique_ptr<Tii> tii; std::unique_ptr<Ber> ber; std::unique_ptr<Clock> clock; std::unique_ptr<Acq> acq; std::unique_ptr<Combining> comb;
    std::unique_ptr<Mer> mer;
    int decode_tii = 0, count_ber = 0, sample_clock = DABB_CLOCK_OFF, acquisition = DABB_ACQ_REFERENCE, measure_mer = 0;
    TraceBuf trace{nullptr, nullptr, 0}; std::string trace_path; int n_slots = 1; int max_cu = 144; int ring_pitch = 0;
    DevBuf<unsigned long long> d_trace_rec; DevBuf<unsigned int> d_trace_count;      // what `trace` points into
    std::string err; int64_t launches = 0; int osc_mismatches = -1; int osc_patched = 0; std::vector<float2> h_osc;
    HostTables* host = nullptr; DevTables dev{};
    DevBuf<float2> d_tw_fwd, d_tw_inv, d_prs_ref, d_osc; DevBuf<int16_t> d_invperm, d_fic_map; DevBuf<uint8_t> d_gf_exp, d_gf_log; DevBuf<double2> d_osc_hi;   // what `dev` points into
    DevBuf<StreamState> d_state; DevBuf<StepScratch> d_scr; DevBuf<MscSlotState> d_slots;
    DevBuf<int64_t> d_buf_start, d_win, d_prs; DevBuf<int32_t> d_nco_sync, d_nco_frame;
    DevBuf<int32_t> d_active, d_index; DevBuf<float> d_cir, d_cir_work; DevBuf<float2> d_r1, d_null; DevBuf<int32_t> d_snr; DevBuf<float2> d_fc; DevBuf<float> d_lvl;
    DevBuf<int8_t> d_soft; DevBuf<uint2> d_fic_steptab; DevBuf<uint32_t> d_fic_stage_off; DevBuf<uint2> d_dec; DevBuf<uint8_t> d_fibs; DevBuf<int32_t> d_crc;
    DevBuf<dabb_frame_result> d_results;
    // the protection-profile table: one entry per distinct ProtProfile a select call has met, built the first time it is selected and
    // kept until dabb_destroy (MscSlotState::profile indexes it); d_profiles holds their device tables for the grouped Viterbi launch
    struct Profile {
        ProtProfile prof{}; int nsteps = 0, nbits = 0, flen = 0, flen_pad = 0;
        DevBuf<uint2> d_steptab; DevBuf<uint32_t> d_stage_off, d_prbs_words;
        dabb_ber::Profile ber{};        // its puncturing as the bit-error count reads it (d_ber_prof)
    };
    std::vector<Profile> profiles; DevBuf<VitProfile> d_profiles;
    // per slot: the buffers of the streams that decode a sub-channel in it.  Rows of d_logical / d_window / d_sf are flen_pad bytes
    // (x 1 / 5 / 5), the largest flen_pad the slot has held, so that a stream keeps its row when another stream's geometry changes;
    // flen is the largest logical frame among the slot's enabled streams (0: none).  The MSC Viterbi launch runs the grouped schedule
    // d_groups / d_cw_list (vit_groups.cuh), rebuilt by every select and remove call.
    struct Slot {
        bool configured = false; int frag_pitch = 0, flen = 0, flen_pad = 0, n_groups = 0;
        DevBuf<int8_t> d_frag; DevBuf<int32_t> d_valid;
        DevBuf<uint8_t> d_logical; DevBuf<uint2> d_dec; DevBuf<uint8_t> d_window, d_sf; DevBuf<int32_t> d_info;
        DevBuf<VitGroup> d_groups; DevBuf<int32_t> d_cw_list;
    } slot[DABB_MAX_SUBCH];
    DevBuf<int8_t> d_ring[DABB_MAX_SUBCH];     // per slot: the time de-interleaver's history, kept when the slot's geometry changes
    DevBuf<uint32_t> d_fic_prbs_words;
    std::vector<MscSlotState> h_slots;
    DevBuf<float2> d_iq_stage; DevBuf<uint8_t> d_raw_stage;
    // pipelined host-buffer path (dabb_submit / dabb_collect): copy stream, two device staging slots, two result slots in pinned memory
    cudaStream_t streamC = nullptr; cudaEvent_t evH2D[2] = {nullptr, nullptr}, evStageFree[2] = {nullptr, nullptr}; bool stageFreeValid[2] = {false, false};
    DevBuf<uint8_t> d_stage2[2];
    int stage_last_fmt = -1; int64_t stage_last_len = 0; std::vector<int64_t> stage_last_start;     // the previous dabb_submit's window (carry_samples)
    // one step's outputs on their way to the caller: device -> pinned copies, complete at `done`, then scattered into `out`
    struct Pending {
        cudaEvent_t done = nullptr; StepOut out{};
        HostBuf<dabb_frame_result> h_res; HostBuf<uint8_t> h_fibs, h_logical, h_superframe;
        int flen_pad[DABB_MAX_SUBCH] = {0, 0, 0, 0}; size_t msc_off[DABB_MAX_SUBCH] = {0, 0, 0, 0}, sf_off[DABB_MAX_SUBCH] = {0, 0, 0, 0};    // flen_pad 0: slot not configured
        std::vector<int32_t> flen;      // [slot][stream] the stream's logical frame length when the step was enqueued (0: nothing to deliver)
    } pend[2], pend_sync;     // the two dabb_submit slots; dabb_process and taps 7 / 8, which never leave a step outstanding
    int pend_head = 0, pend_count = 0; int64_t submits = 0;
    int groups = 1; int fc_pitch = 1; int tail_frames = 0; int nco_fast = 0; int soft_demap = DABB_DEMAP_REFERENCE;
    DevBuf<const int32_t*> d_info_tab;
    // optional per-kernel timing: one event after every launch, durations = differences of consecutive events
    bool prof = false; std::vector<cudaEvent_t> prof_ev; std::vector<const char*> prof_name; size_t prof_used = 0;
    std::vector<std::pair<std::string, std::pair<double, long>>> prof_acc;
    // spectrum survey (survey.cu), allocated by the first dabb_survey: twiddle and window tables, host input staging, per-chunk sums, spectra
    DevBuf<dabb_channel::cf> d_svy_tw; DevBuf<float> d_svy_win; DevBuf<uint8_t> d_svy_stage; DevBuf<float> d_svy_part, d_svy_psd;
    // without keep_taps: [S][OFDM_MASK_WORDS] the OFDM symbols each stream's decoders read (ofdm_mask.cuh), rebuilt by every select and
    // remove call; the OFDM launch of the last step, which tap 0 repeats over every symbol when soft_partial says it skipped some
    DevBuf<uint32_t> d_symmask; OfdmParams soft_op{}; bool soft_partial = false;
    // the combine launch of the last step (n_items 0: it had no group) and the leader table it ran with, from which tap 0 builds the rows
    // of every symbol when it repeats that step, whatever grouping has replaced it since
    CombParams comb_op{}; std::shared_ptr<const std::vector<int32_t>> comb_leader;
};

namespace {

#define CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { ctx->err = std::string(#call) + ": " + cudaGetErrorString(e_); return DABB_E_CUDA; } } while (0)

template <typename T, bool Pinned> int alloc(dabb_ctx* ctx, Owned<T, Pinned>& b, size_t n)
{
    const cudaError_t e = b.alloc(n);
    if (e == cudaSuccess) return 0;
    ctx->err = std::string(Pinned ? "pinned host" : "device") + " allocation of " + std::to_string(n * sizeof(T)) + " bytes failed: " + cudaGetErrorString(e);
    return DABB_E_NOMEM;
}

// a device buffer, zero-filled on the context's stream unless `zero` is false
template <typename T> int dalloc(dabb_ctx* ctx, DevBuf<T>& b, size_t n, bool zero = true)
{
    const int rc = alloc(ctx, b, n);
    if (!rc && zero) cudaMemsetAsync(b.get(), 0, n * sizeof(T), ctx->stream);
    return rc;
}

// an analysis's records of a step that did not run it: zeros
template <typename T> int clear_records(dabb_ctx* ctx, const DevBuf<T>& res, cudaStream_t st)
{
    CK(cudaMemsetAsync(res, 0, sizeof(T) * ctx->S, st));
    return DABB_OK;
}

// the S records of an analysis's last step into `out` (at most `bytes`); refused while it was never enabled
template <typename A> int read_records(dabb_ctx* ctx, const std::unique_ptr<A>& a, const char* refusal, void* out, size_t bytes)
{
    if (!a) { ctx->err = refusal; return DABB_E_STATE; }
    const size_t n = sizeof(*a->res.get()) * ctx->S;
    CK(cudaMemcpy(out, a->res, bytes < n ? bytes : n, cudaMemcpyDeviceToHost));
    return DABB_OK;
}

CombTables* comb_tab(const dabb_ctx* ctx) { return ctx->comb ? ctx->comb->tab.get() : nullptr; }

void prof_mark(dabb_ctx* ctx, const char* what)
{
    if (!ctx->prof) return;
    if (ctx->prof_used == ctx->prof_ev.size()) {
        if (ctx->prof_ev.size() >= 16384) return;
        cudaEvent_t e; if (cudaEventCreate(&e) != cudaSuccess) return;
        ctx->prof_ev.push_back(e); ctx->prof_name.push_back(what);
    }
    ctx->prof_name[ctx->prof_used] = what;
    cudaEventRecord(ctx->prof_ev[ctx->prof_used++], ctx->stream);
}

int check_launch(dabb_ctx* ctx, const char* what)
{
    ctx->launches++;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { ctx->err = std::string(what) + ": " + cudaGetErrorString(e); return DABB_E_CUDA; }
    prof_mark(ctx, what);
    return 0;
}

void prof_collect(dabb_ctx* ctx)
{
    if (ctx->prof_used < 2) { ctx->prof_used = 0; return; }
    cudaStreamSynchronize(ctx->stream);
    for (size_t i = 1; i < ctx->prof_used; i++) {
        const char* nm = ctx->prof_name[i];
        if (!strcmp(nm, "__step_begin")) continue;
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, ctx->prof_ev[i - 1], ctx->prof_ev[i]) != cudaSuccess) continue;
        bool found = false;
        for (auto& a : ctx->prof_acc) if (a.first == nm) { a.second.first += ms; a.second.second++; found = true; break; }
        if (!found) ctx->prof_acc.push_back({nm, {ms, 1}});
    }
    ctx->prof_used = 0;
}

// ---------------------------------------------------------------------------------------------------------------
// state-machine kernels (one thread per stream)
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int32_t mod_rate(int64_t v) { v %= INPUT_RATE; if (v < 0) v += INPUT_RATE; return (int32_t)v; }

// Initial / re-acquisition: OFDMProcessor::run up to SyncOnPhase (ofdm-processor.cpp:248-323): sLevel warm-up over
// T_F/2 samples, then the 50-sample envelope dip search.  Strictly sequential per stream, exact arithmetic order
// (double IIR), only runs while a stream is not tracking.
__global__ void acquire_kernel(StreamState* st, const float2* iq, int64_t stride, const int64_t* buf_start, int64_t buf_len, const float2* osc, int S)
{
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S) return;
    StreamState z = st[s];
    if (z.acquired) return;
    const float2* src = iq + (int64_t)s * stride;
    int64_t pos = z.pos - buf_start[s];            // physical index
    const int64_t end = buf_len;
    int32_t lp = z.local_phase; float sl = z.slevel;
    if (pos < 0) return;
    auto get = [&](int32_t phase, float& l1) -> bool {
        if (pos >= end) return false;
        float2 v = src[pos++];
        lp -= phase; lp = (lp + INPUT_RATE) % INPUT_RATE;
        const float2 o = osc[lp];
        const float re = __fsub_rn(__fmul_rn(v.x, o.x), __fmul_rn(v.y, o.y)), im = __fadd_rn(__fmul_rn(v.x, o.y), __fmul_rn(v.y, o.x));
        l1 = __fadd_rn(fabsf(re), fabsf(im));
        sl = (float)__dadd_rn(__dmul_rn(0.00001, (double)l1), __dmul_rn(1 - 0.00001, (double)sl));
        return true;
    };
    float l1;
    // Progress is kept: the state is written back at every point from which the search can be resumed exactly (after the warm-up and
    // at the start of every attempt), so a buffer that ends in the middle of an attempt costs only that attempt, and eight failed
    // attempts (no signal) end the call with the position advanced - the reference's notSynced loop keeps running the same way
    // (ofdm-processor.cpp:253-323).
    auto checkpoint = [&]() { z.started = 1; z.pos = pos + buf_start[s]; z.local_phase = lp; z.slevel = sl; st[s] = z; };
    if (!z.started) {
        sl = 0.f;
        for (int i = 0; i < TF / 2; i++) if (!get(0, l1)) return;   // not enough samples for the warm-up: state untouched
        checkpoint();
    }
    const int32_t phase = z.coarse + z.fine;
    // local ring of the last 64 envelope values is enough for the 50-tap moving sum
    float env[64];
    for (int attempt = 0; attempt < 8; attempt++) {
        checkpoint();
        int idx = 0; float cur = 0.f;
        for (int i = 0; i < 50; i++) { if (!get(0, l1)) return; env[idx & 63] = l1; cur = __fadd_rn(cur, l1); idx++; }
        int counter = 0; bool fail = false;
        while ((double)__fdiv_rn(cur, 50.f) > __dmul_rn(0.50, (double)sl)) {
            if (!get(phase, l1)) return;
            env[idx & 63] = l1; cur = __fadd_rn(cur, __fsub_rn(l1, env[(idx - 50) & 63])); idx++;
            if (++counter > TF) { fail = true; break; }
        }
        if (fail) { z.acq_failed++; continue; }
        counter = 0;
        while ((double)__fdiv_rn(cur, 50.f) < __dmul_rn(0.75, (double)sl)) {
            if (!get(phase, l1)) return;
            env[idx & 63] = l1; cur = __fadd_rn(cur, __fsub_rn(l1, env[(idx - 50) & 63])); idx++;
            if (++counter > TNULL + 50) { fail = true; break; }
        }
        if (fail) { z.acq_failed++; continue; }
        z.acquired = 1;
        break;
    }
    checkpoint();      // acquired: tracking starts here; not acquired: the next call continues the search from here
}

// Robust acquisition (DABB_ACQ_ROBUST, acq_core.cuh), in place of acquire_kernel: the span each searching stream analyses in this step,
// from its position to the end of its buffer, at most NB_MAX blocks; fewer than MIN_BLOCKS: no search
__global__ void acq_plan_kernel(const StreamState* st, const int64_t* buf_start, int64_t buf_len, int S, AcqJob* job)
{
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S) return;
    const StreamState z = st[s];
    AcqJob j{};
    j.rel = z.pos - buf_start[s];
    if (!z.acquired && j.rel >= 0 && j.rel < buf_len) {
        const int64_t nb = (buf_len - j.rel) / dabb_acq::BLK;
        j.nb = nb < dabb_acq::MIN_BLOCKS ? 0 : (int32_t)(nb < dabb_acq::NB_MAX ? nb : dabb_acq::NB_MAX);
    }
    j.lp = z.local_phase; j.phase = z.coarse + z.fine;
    job[s] = j;
}

// the decision of one searching stream (one CTA): the first window of WIN blocks with the smallest level sum, its depth below the span's
// median level, and the hand-off to time synchronisation.  Every stream's tap-13 record of the step is written here.
__global__ void __launch_bounds__(256)
acq_decide_kernel(StreamState* st, const AcqJob* job, const int64_t* buf_start, const float* level, const float* l1sum, dabb_acq_result* res)
{
    using namespace dabb_acq;
    __shared__ float lv[NB_MAX];
    __shared__ float med;
    const int s = blockIdx.x, t = threadIdx.x;
    const AcqJob j = job[s];
    if (!j.nb) { if (t == 0) res[s] = dabb_acq_result{0, 0, 0.f, 0, -1}; return; }
    const int nb = j.nb;
    for (int i = t; i < nb; i += blockDim.x) lv[i] = level[(int64_t)s * NB_MAX + i];
    __syncthreads();
    // median: the level with exactly k = (nb - 1) / 2 levels below it (levels are finite, so the value is well defined)
    const int k = (nb - 1) / 2;
    for (int i = t; i < nb; i += blockDim.x) {
        int less = 0, leq = 0;
        for (int m = 0; m < nb; m++) { less += lv[m] < lv[i]; leq += lv[m] <= lv[i]; }
        if (less <= k && k < leq) med = lv[i];
    }
    __syncthreads();
    if (t) return;
    int best = 0; float wmin = window_sum(lv, 0);
    for (int b = 1; b + WIN <= nb; b++) { const float w = window_sum(lv, b); if (w <= wmin) { wmin = w; best = b; } }     // last of equal minima
    const float depth = depth_db(med, wmin);
    const bool found = is_found(depth, best, nb);
    double env = 0.0;
    for (int b = 0; b < nb; b++) env += (double)l1sum[(int64_t)s * NB_MAX + b];
    StreamState z = st[s];
    const int64_t skip = found ? (int64_t)best * BLK + NULL_END - LEAD : (int64_t)(nb - KEEP) * BLK;
    z.pos += skip;
    z.local_phase = mod_rate((int64_t)z.local_phase - skip * j.phase);
    z.started = 1;
    z.slevel = (float)(env / ((double)nb * BLK));
    if (found) z.acquired = 1; else z.acq_failed++;
    st[s] = z;
    res[s] = dabb_acq_result{1, nb, depth, 0, found ? buf_start[s] + j.rel + (int64_t)best * BLK + NULL_END : -1};
}

__global__ void plan_kernel(StreamState* st, StepScratch* scr, const int64_t* buf_start, int64_t buf_len, int S,
                            int64_t* win, int32_t* nco_sync, int32_t* active)
{
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S) return;
    const StreamState z = st[s];
    StepScratch c{};
    int32_t lp = 0, p1 = 0;
    const int64_t rel = z.pos - buf_start[s];
    const int64_t need = (int64_t)TU + (TU - 1) + 75 * (int64_t)TS + TNULL;
    if (!z.acquired) { c.active = 0; c.status = DABB_FRAME_ACQUIRING; }
    else if (rel < 0 || rel + need > buf_len) { c.active = 0; c.status = DABB_FRAME_NEED_SAMPLES; }
    else {
        c.active = 1; c.status = DABB_FRAME_DECODED; c.win_start = rel;
        p1 = z.coarse + z.fine;
        lp = mod_rate((int64_t)z.local_phase - p1);
    }
    scr[s] = c;
    win[s] = c.win_start; nco_sync[2 * s] = lp; nco_sync[2 * s + 1] = p1; active[s] = c.active;
}

// clock_frame (DABB_CLOCK_TRACK, else nullptr): the ppm the OFDM kernel derotates the frame with, the estimate from before the frame
__global__ void post_sync_kernel(StreamState* st, StepScratch* scr, const int32_t* index, const int32_t* coarse_corr, int S, int64_t* prs, int32_t* nco_frame, int32_t* active,
                                 float* clock_frame)
{
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S) return;
    StepScratch c = scr[s];
    if (!c.active) return;
    StreamState z = st[s];
    const int32_t p1 = z.coarse + z.fine;
    const int idx = index[s];
    z.start_index = idx;
    if (idx < 0) {
        // SyncOnPhase failed: the T_u samples are consumed and the null search starts over (ofdm-processor.cpp:347-350)
        z.pos += TU; z.local_phase = mod_rate((int64_t)z.local_phase - (int64_t)TU * p1); z.acquired = 0;
        c.active = 0; c.status = DABB_FRAME_NO_SYNC;
        st[s] = z; scr[s] = c; active[s] = 0;
        return;
    }
    // phase applied to PRS sample 0 (the (idx+1)-th sample read in this frame)
    const int32_t lp_prs0 = mod_rate((int64_t)z.local_phase - (int64_t)(idx + 1) * p1);
    // coarse corrector (ofdm-processor.cpp:397-409): find_index_kernel evaluated processPRS where the FIC ratio asked for it
    if (coarse_corr) {
        const int corr = coarse_corr[s];
        if (corr != 100) { z.coarse += corr * 1000; if (abs(z.coarse) > 35000) z.coarse = 0; }     // 100: not evaluated / no estimate (:404-408)
    }
    const int32_t p2 = z.coarse + z.fine;
    // phase applied to the first data-symbol sample = lp after 2048+idx samples, minus p2; expressed at index 2048
    const int32_t lp_after_prs = mod_rate((int64_t)z.local_phase - (int64_t)(TU + idx) * p1);
    const int32_t lp_sym0 = mod_rate((int64_t)lp_after_prs - p2 + (int64_t)TU * p2);   // so that lp(i) = lp_sym0 - i*p2 for i >= 2048
    c.nco_frame[0] = lp_prs0; c.nco_frame[1] = p1; c.nco_frame[2] = lp_sym0; c.nco_frame[3] = p2;
    scr[s] = c; st[s] = z;
    prs[s] = c.win_start + idx;
    nco_frame[4 * s] = lp_prs0; nco_frame[4 * s + 1] = p1; nco_frame[4 * s + 2] = lp_sym0; nco_frame[4 * s + 3] = p2;
    if (clock_frame) clock_frame[s] = (float)dabb_clock::applied(z.clk);
}

// lane A, right after the OFDM kernel: the part of OFDMProcessor::run that feeds the next frame's synchronisation
// (fine corrector update :450-451, consumed samples, NCO phase, corrector wrap :478-486)
// clock_track: the sample-clock estimator counts this step's frame (clock_core.cuh); clk_res (tap 11, or nullptr): the step's records
__global__ void advance_kernel(StreamState* st, StepScratch* scr, int S, int groups /* partial sums per frame */, const float2* fc_part, const float* lvl_part,
                               int clock_track, dabb_clock_result* clk_res)
{
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S) return;
    StepScratch c = scr[s];
    StreamState z = st[s];
    // sample clock: a decoded frame updates the estimate (with the value post_sync_kernel handed the demodulator recorded first); a step
    // without sync, or with the option off, breaks the chain of consecutive frames; NEED_SAMPLES leaves it
    dabb_clock_result cr{};
    const bool clk_break = z.clk.prev && (!clock_track || c.status == DABB_FRAME_NO_SYNC || c.status == DABB_FRAME_ACQUIRING);
    if (clock_track && c.active) {
        cr.applied_ppm = (float)dabb_clock::applied(z.clk);
        dabb_clock::update(z.clk, z.start_index);
    }
    if (clk_break) { z.clk.prev = 0; if (!c.active) st[s].clk.prev = 0; }
    if (clock_track) { cr.ppm = (float)z.clk.e; cr.frames = z.clk.n; }
    if (clk_res) clk_res[s] = cr;
    c.r_start_index = z.start_index; c.r_fx = 0.f; c.r_fy = 0.f;
    c.r_acq_failed = z.acq_failed;
    if (z.acq_failed) { z.acq_failed = 0; if (!c.active) st[s].acq_failed = 0; }
    if (c.active) {
        float fx = 0.f, fy = 0.f;      // FreqCorr: partial sums in group order
        for (int g = 0; g < groups; g++) { fx += fc_part[(int64_t)s * groups + g].x; fy += fc_part[(int64_t)s * groups + g].y; }
        const int idx = z.start_index;
        const int32_t p1 = c.nco_frame[1], p2 = c.nco_frame[3];
        // fineCorrector += 0.1 * arg(FreqCorr) / M_PI * (carrierDiff / 2), int16 store (ofdm-processor.cpp:450-451)
        const double upd = 0.1 * (double)(float)atan2((double)fy, (double)fx) / 3.14159265358979323846 * 500;
        z.fine = (int32_t)(int16_t)((double)z.fine + upd);
        const int32_t p3 = z.coarse + z.fine;
        const int64_t lpn = (int64_t)z.local_phase - (int64_t)(TU + idx) * p1 - (int64_t)75 * TS * p2;
        c.null_pos = z.pos + (int64_t)TU + idx + 75 * (int64_t)TS; c.null_lp = mod_rate(lpn); c.null_ph = p3;
        const int64_t lp = lpn - (int64_t)TNULL * p3;
        z.local_phase = mod_rate(lp);
        z.pos += (int64_t)TU + idx + 75 * (int64_t)TS + TNULL;
        if (z.fine > 500) { z.coarse += 1000; z.fine -= 1000; }
        else if (z.fine < -500) { z.coarse -= 1000; z.fine += 1000; }
        // sLevel (ofdm-processor.cpp:166,215) is an IIR over EVERY sample read: exact while a stream searches (acquire_kernel), and
        // while it tracks it follows the same recursion on a sub-sample (one magnitude per symbol and thread of the OFDM kernel,
        // decayed per symbol) - only a re-acquisition after a sync loss ever reads it (DESIGN.md 5v)
        if (lvl_part) {
            float est = 0.f;
            for (int g = 0; g < groups; g++) est += lvl_part[(int64_t)s * groups + g];
            const float ln1ma = -1.000005e-5f;          // ln(1 - 1e-5)
            const float n_frame = (float)(TU + idx + 75 * TS + TNULL);
            z.slevel = z.slevel * expf(n_frame * ln1ma) + est * (1.0f - expf((float)TS * ln1ma)) * expf((float)TNULL * ln1ma);
        }
        z.nframes++;
        c.r_fx = fx; c.r_fy = fy;
        st[s] = z;
    }
    c.r_fine = z.fine; c.r_coarse = z.coarse; c.r_next_pos = z.pos; c.r_slevel = z.slevel;
    scr[s] = c;
}

// sample i of the null symbol that follows stream s's frame, read with the NCO at coarse + fine (after this frame's fine update); 0 when
// the stream decoded no frame or the sample is outside its buffer (p0: the null symbol's first sample relative to the buffer)
__device__ __forceinline__ float2 null_sample(const StepScratch& c, const float2* iq, int64_t stride, int s, int64_t p0, int64_t buf_len, const float2* osc, bool mix, int i)
{
    float2 v = make_float2(0.f, 0.f);
    if (c.active && p0 >= 0 && p0 + i < buf_len) {
        v = iq[(int64_t)s * stride + p0 + i];
        if (mix) {
            const float2 o = osc[mod_rate((int64_t)c.null_lp - (int64_t)(i + 1) * c.null_ph)];
            v = make_float2(__fsub_rn(__fmul_rn(v.x, o.x), __fmul_rn(v.y, o.y)), __fadd_rn(__fmul_rn(v.x, o.y), __fmul_rn(v.y, o.x)));
        }
    }
    return v;
}

// diagnostics tap: the null symbol as OFDMProcessor::run hands it to onNewNullSymbol (ofdm-processor.cpp:462-469): T_null
// samples read with the NCO at coarse + fine (after this frame's fine update)
__global__ void null_tap_kernel(const StepScratch* scr, const float2* iq, int64_t stride, const int64_t* buf_start, int64_t buf_len, const float2* osc, float2* out)
{
    const int s = blockIdx.x;
    const StepScratch c = scr[s];
    float2* dst = out + (int64_t)s * TNULL;
    const int64_t p0 = c.null_pos - buf_start[s];
    const bool mix = c.null_lp != 0 || c.null_ph != 0;
    for (int i = threadIdx.x; i < TNULL; i += blockDim.x) dst[i] = null_sample(c, iq, stride, s, p0, buf_len, osc, mix, i);
}

// diversity combining, lane A after advance_kernel: the noise power N (combine_core.cuh) of every grouped stream that decoded a frame,
// from the same null-symbol samples as tap 3; every stream's tap-12 record of the step starts as {0, 0, N or 0}
__global__ void __launch_bounds__(dabb_comb::NULL_THREADS)
null_power_kernel(const StepScratch* scr, const int32_t* gid, const float2* iq, int64_t stride, const int64_t* buf_start, int64_t buf_len, const float2* osc,
                  dabb_combine_result* res)
{
    __shared__ float part[dabb_comb::NULL_THREADS];
    const int s = blockIdx.x, t = threadIdx.x;
    const StepScratch c = scr[s];
    if (gid[s] < 0 || !c.active) { if (t == 0) res[s] = dabb_combine_result{0, 0u, 0.f, 0}; return; }
    const int64_t p0 = c.null_pos - buf_start[s];
    const bool mix = c.null_lp != 0 || c.null_ph != 0;
    float a = 0.f;
    for (int i = t; i < TNULL; i += dabb_comb::NULL_THREADS) {
        const float2 v = null_sample(c, iq, stride, s, p0, buf_len, osc, mix, i);
        a = __fadd_rn(a, __fadd_rn(__fmul_rn(v.x, v.x), __fmul_rn(v.y, v.y)));       // dabb_comb::null_partial
    }
    part[t] = a;
    __syncthreads();
    if (t == 0) res[s] = dabb_combine_result{0, 0u, dabb_comb::null_noise(part), 0};
}

// lane B, after FIC / MSC / RS of the frame: decoder-side state and the result record
__global__ void finalize_kernel(const StepScratch* scr, MscSlotState* slots, int n_slots, int S, int32_t* fic_ratio,
                                const int32_t* snr, const int32_t* crc, const int32_t* const* slot_info, dabb_frame_result* res)
{
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S) return;
    const StepScratch c = scr[s];
    dabb_frame_result r;
    memset(&r, 0, sizeof r);
    r.status = c.status;
    int ratio = fic_ratio[s];
    if (c.active) {
        // FIC success counter, one saturating update per FIB in order (fic-handler.cpp:214-229)
        const int mask = crc[s];
        for (int f = 0; f < 12; f++) { if ((mask >> f) & 1) { if (ratio < 10) ratio++; } else if (ratio > 0) ratio--; }
        fic_ratio[s] = ratio;
        r.snr_raw = snr[s]; r.fib_crc_mask = mask;
        for (int k = 0; k < n_slots; k++) {
            MscSlotState& m = slots[s * n_slots + k];
            if (!m.enabled) continue;
            m.cif_count += 4;
            const int32_t* inf = slot_info[k] + (int64_t)s * 16;
            r.n_logical[k] = inf[0]; r.n_rs_events[k] = inf[1]; r.rs_uncorr_mask[k] = inf[2];
            for (int e = 0; e < 4; e++) r.rs_corr[k][e] = inf[3 + e];
            r.sf_ready[k] = inf[7]; r.sf_au_count[k] = inf[8]; r.sf_au_crc_mask[k] = inf[9];
        }
    }
    r.start_index = c.r_start_index; r.freq_corr_re = c.r_fx; r.freq_corr_im = c.r_fy;
    r.fine_corr = c.r_fine; r.coarse_corr = c.r_coarse; r.fic_ratio = ratio; r.next_pos = c.r_next_pos; r.slevel = c.r_slevel; r.acq_failed = c.r_acq_failed;
    res[s] = r;
}

__global__ void reset_kernel(StreamState* st, MscSlotState* slots, int n_slots, int first, int count, int64_t pos, int32_t* fic_ratio)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    StreamState z{}; z.pos = pos; z.start_index = -1;
    st[first + i] = z; fic_ratio[first + i] = 0;
    for (int k = 0; k < n_slots; k++) { MscSlotState& m = slots[(first + i) * n_slots + k]; m.cif_count = 0; m.sf_frame_count = 0; }
}

__global__ void set_slot_kernel(MscSlotState* slots, int n_slots, int slot, int first, int count, MscSlotState v)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    slots[(first + i) * n_slots + slot] = v;
}

void sync_all(dabb_ctx* ctx)
{
    if (ctx->stream) cudaStreamSynchronize(ctx->stream);
    if (ctx->streamB) cudaStreamSynchronize(ctx->streamB);
    if (ctx->stream2) cudaStreamSynchronize(ctx->stream2);
    if (ctx->streamC) cudaStreamSynchronize(ctx->streamC);
}

// raw file formats -> cf32, value for value like CRAWFile::convertSamples (dabb_channel::raw_sample, shared with the channelizer)
__global__ void convert_iq_kernel(const uint8_t* __restrict__ raw, int64_t raw_stride_samples, int fmt, float2* __restrict__ out, int64_t out_stride, int64_t len, int S)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int s = blockIdx.y;
    if (i >= len || s >= S) return;
    const dabb_channel::cf v = dabb_channel::raw_sample(raw, (int64_t)s * raw_stride_samples + i, fmt);
    out[(int64_t)s * out_stride + i] = make_float2(v.x, v.y);
}

// an analysis switched on (`on`) for the first time: `build` fills a new instance, which the context takes only when every allocation and
// upload succeeded
template <typename A, typename F> int enable(dabb_ctx* ctx, bool on, std::unique_ptr<A>& owner, F build)
{
    if (!on || owner) return DABB_OK;
    cudaSetDevice(ctx->device);
    sync_all(ctx);
    auto a = std::make_unique<A>();
    int rc;
    if ((rc = build(*a))) return rc;
    CK(cudaStreamSynchronize(ctx->stream));
    owner = std::move(a);
    return DABB_OK;
}

// makes b hold at least n elements, without keeping its contents; the device finishes with the old buffer first
template <typename T> int grow(dabb_ctx* ctx, DevBuf<T>& b, size_t n)
{
    if (n <= b.size()) return 0;
    sync_all(ctx);
    return alloc(ctx, b, n);
}

using dabb_channel::bytes_per_sample;

// ---- step outputs ---------------------------------------------------------------------------------------------------------------
// Every way a step's outputs reach the caller (dabb_process, dabb_submit + dabb_collect, taps 7 / 8) runs the same three routines:
// prepare_pending sizes a Pending's pinned buffers for the configured slots, enqueue_readback copies the device buffers whole into it
// behind the step, and deliver writes them into the caller's layout [S][MAX_SUBCH][4][msc_stride] / [S][MAX_SUBCH][sf_stride].
// check_strides runs before any of them and before the step, so that a refused call has enqueued nothing.

StepOut step_out(const dabb_io& io) { return StepOut{io.results, io.fibs, io.msc, io.msc_stride, io.sf, io.sf_stride}; }

int check_strides(dabb_ctx* ctx, const StepOut& o)
{
    for (int k = 0; k < ctx->n_slots; k++) {
        const auto& sl = ctx->slot[k];
        if (!sl.configured) continue;
        if (o.msc && o.msc_stride < sl.flen) { ctx->err = "msc_stride smaller than the logical frame"; return DABB_E_ARG; }
        if (o.sf && o.sf_stride < 5 * sl.flen) { ctx->err = "sf_stride smaller than the superframe"; return DABB_E_ARG; }
    }
    return DABB_OK;
}

// p must not have copies in flight (collected, or never used)
int prepare_pending(dabb_ctx* ctx, dabb_ctx::Pending& p)
{
    const int S = ctx->S;
    int rc;
    if (!p.done) CK(cudaEventCreateWithFlags(&p.done, cudaEventDisableTiming));
    if (!p.h_res && (rc = alloc(ctx, p.h_res, S))) return rc;
    if (!p.h_fibs && (rc = alloc(ctx, p.h_fibs, (size_t)S * 12 * 32))) return rc;
    size_t msc = 0, sf = 0;
    p.flen.assign((size_t)ctx->n_slots * S, 0);
    for (int k = 0; k < ctx->n_slots; k++) {
        const auto& sl = ctx->slot[k];
        p.flen_pad[k] = sl.configured ? sl.flen_pad : 0;
        if (!sl.configured) continue;
        p.msc_off[k] = msc; p.sf_off[k] = sf;
        msc += (size_t)S * 4 * sl.flen_pad; sf += (size_t)S * 5 * sl.flen_pad;
        for (int s = 0; s < S; s++) {       // the geometry the step runs with: a select call before dabb_collect does not change it
            const MscSlotState& m = ctx->h_slots[(size_t)s * ctx->n_slots + k];
            p.flen[(size_t)k * S + s] = m.enabled ? 3 * m.bitrate : 0;
        }
    }
    if (msc > p.h_logical.size() && (rc = alloc(ctx, p.h_logical, msc))) return rc;
    if (sf > p.h_superframe.size() && (rc = alloc(ctx, p.h_superframe, sf))) return rc;
    return DABB_OK;
}

// the outputs `o` asks for, device -> p, on lane B (the main stream while profiling) behind the last step's result record
int enqueue_readback(dabb_ctx* ctx, dabb_ctx::Pending& p, const StepOut& o)
{
    const int S = ctx->S;
    cudaStream_t B = ctx->prof ? ctx->stream : ctx->streamB;
    if (o.results) CK(cudaMemcpyAsync(p.h_res, ctx->d_results, sizeof(dabb_frame_result) * S, cudaMemcpyDeviceToHost, B));
    if (o.fibs) CK(cudaMemcpyAsync(p.h_fibs, ctx->d_fibs, (size_t)S * 12 * 32, cudaMemcpyDeviceToHost, B));
    for (int k = 0; k < ctx->n_slots; k++) {
        if (!p.flen_pad[k]) continue;
        const auto& sl = ctx->slot[k];
        if (o.msc) CK(cudaMemcpyAsync(p.h_logical + p.msc_off[k], sl.d_logical, (size_t)S * 4 * p.flen_pad[k], cudaMemcpyDeviceToHost, B));
        if (o.sf) CK(cudaMemcpyAsync(p.h_superframe + p.sf_off[k], sl.d_sf, (size_t)S * 5 * p.flen_pad[k], cudaMemcpyDeviceToHost, B));
    }
    CK(cudaEventRecord(p.done, B));
    p.out = o;
    return DABB_OK;
}

int deliver(dabb_ctx* ctx, dabb_ctx::Pending& p)
{
    CK(cudaEventSynchronize(p.done));
    const int S = ctx->S;
    const StepOut& o = p.out;
    if (o.results) memcpy(o.results, p.h_res, sizeof(dabb_frame_result) * S);
    if (o.fibs) memcpy(o.fibs, p.h_fibs, (size_t)S * 12 * 32);
    for (int k = 0; k < ctx->n_slots; k++) {
        const size_t fp = p.flen_pad[k];
        if (!fp) continue;
        for (int s = 0; s < S; s++) {    // each stream's own frame length; streams not enabled in the slot keep the caller's bytes
            const size_t flen = p.flen[(size_t)k * S + s];
            if (!flen) continue;
            if (o.msc)   // pinned rows [S*4][fp] -> caller [S][MAX_SUBCH][4][msc_stride]
                for (int c = 0; c < 4; c++)
                    memcpy(o.msc + (((size_t)s * DABB_MAX_SUBCH + k) * 4 + c) * o.msc_stride, p.h_logical + p.msc_off[k] + ((size_t)s * 4 + c) * fp, flen);
            if (o.sf) memcpy(o.sf + ((size_t)s * DABB_MAX_SUBCH + k) * o.sf_stride, p.h_superframe + p.sf_off[k] + (size_t)s * 5 * fp, 5 * flen);
        }
    }
    return DABB_OK;
}

// ---- sub-channel slots ----------------------------------------------------------------------------------------------------------
// a new entry of the protection-profile table: the de-puncturing expansion tables and dispersal words of its code geometry
int add_profile(dabb_ctx* ctx, const ProtProfile& prof)
{
    dabb_ctx::Profile pf;
    pf.prof = prof; pf.nbits = 24 * prof.bitrate; pf.nsteps = pf.nbits + 6; pf.flen = 3 * prof.bitrate; pf.flen_pad = (pf.flen + 15) & ~15;
    std::vector<int16_t> map((size_t)pf.nsteps * 4);
    build_msc_map(*ctx->host, prof, map.data());
    std::vector<uint2> steps; std::vector<uint32_t> soff;
    build_vit_tables_u2(map.data(), pf.nsteps, steps, soff);
    std::vector<uint32_t> w((size_t)(pf.nbits + 31) / 32); build_prbs_words(pf.nbits, w.data());
    int rc;
    if ((rc = dalloc(ctx, pf.d_steptab, steps.size(), false)) || (rc = dalloc(ctx, pf.d_stage_off, soff.size(), false)) || (rc = dalloc(ctx, pf.d_prbs_words, w.size(), false))) return rc;
    VitProfile e{pf.d_steptab, pf.d_stage_off, pf.d_prbs_words, pf.nsteps, pf.nbits};
    CK(cudaMemcpyAsync(pf.d_steptab, steps.data(), steps.size() * sizeof(uint2), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(pf.d_stage_off, soff.data(), soff.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(pf.d_prbs_words, w.data(), w.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(ctx->d_profiles + ctx->profiles.size(), &e, sizeof e, cudaMemcpyHostToDevice, ctx->stream));
    build_ber_profile(*ctx->host, prof.nblk, prof.L, prof.PI, pf.nbits, pf.ber); pf.ber.prbs = pf.d_prbs_words;
    if (ctx->ber) CK(cudaMemcpyAsync(ctx->ber->prof + ctx->profiles.size(), &pf.ber, sizeof pf.ber, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    ctx->profiles.push_back(std::move(pf));
    return DABB_OK;
}

// b: rows of old_pitch bytes -> rows of new_pitch bytes (> old_pitch), contents kept, the new bytes zero
int repitch(dabb_ctx* ctx, DevBuf<uint8_t>& b, size_t rows, size_t old_pitch, size_t new_pitch)
{
    DevBuf<uint8_t> nb;
    int rc;
    if ((rc = dalloc(ctx, nb, rows * new_pitch))) return rc;
    CK(cudaMemcpy2DAsync(nb, new_pitch, b, old_pitch, old_pitch, rows, cudaMemcpyDeviceToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    b = std::move(nb);
    return DABB_OK;
}

// the symbols stream s's own decoders read (ofdm_mask.cuh), from its slots (h_slots)
void own_symmask(dabb_ctx* ctx, int s, uint32_t* m)
{
    const int ns = ctx->n_slots;
    OfdmMaskSlot sl[DABB_MAX_SUBCH];
    for (int k = 0; k < ns; k++) {
        const MscSlotState& st = ctx->h_slots[(size_t)s * ns + k];
        sl[k] = OfdmMaskSlot{st.enabled, st.start_cu, st.frag / 64};
    }
    build_ofdm_mask(sl, ns, m);
}

// the symbol masks of streams [first, first + count), uploaded on the context's stream; the caller synchronises it before the host vector
// is gone (the copy is from pageable memory, so it is staged before cudaMemcpyAsync returns anyway).  While streams are grouped every
// stream's mask is rebuilt: a member also transforms the symbols its leader reads, so that combine_kernel has their products.
int upload_symmask(dabb_ctx* ctx, int first, int count)
{
    if (!ctx->d_symmask) return DABB_OK;
    const CombTables* ct = comb_tab(ctx);
    if (ct) { first = 0; count = ctx->S; }
    std::vector<uint32_t> m((size_t)count * OFDM_MASK_WORDS);
    for (int i = 0; i < count; i++) own_symmask(ctx, first + i, m.data() + (size_t)i * OFDM_MASK_WORDS);
    if (ct) {
        std::vector<uint32_t> own(m);
        for (int s = 0; s < ctx->S; s++) {
            const int L = (*ct->leader)[(size_t)s];
            for (int w = 0; w < OFDM_MASK_WORDS; w++) m[(size_t)s * OFDM_MASK_WORDS + w] |= own[(size_t)L * OFDM_MASK_WORDS + w];
        }
    }
    CK(cudaMemcpyAsync(ctx->d_symmask + (size_t)first * OFDM_MASK_WORDS, m.data(), m.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream));
    return DABB_OK;
}

template <typename T> int upload(dabb_ctx* ctx, DevBuf<T>& b, const std::vector<T>& h)
{
    int rc;
    if ((rc = alloc(ctx, b, h.size()))) return rc;
    if (!h.empty()) CK(cudaMemcpyAsync(b, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice, ctx->stream));
    return DABB_OK;
}

// every data symbol (1..75), as the mask of a group that combines them all
void all_symbols(int, uint32_t* m) { for (int l = 1; l <= 75; l++) m[l >> 5] |= 1u << (l & 31); }

// The groups of two or more streams that a leader table forms, in leader order with their members in stream order.  mask(L, m) marks the
// data symbols the group of leader L combines: one item of combine_kernel each, and one r1 row each for every member, the members' rows
// one after the other and the groups' too (`rows` in all).  Per stream its group (gid, -1: none), first row and its group's mask.
struct Grouping { std::vector<CombGroup> groups; std::vector<CombItem> items; std::vector<int32_t> gid, row; std::vector<uint32_t> lmask; int64_t rows = 0; };
template <typename F> Grouping group_streams(const std::vector<int32_t>& leader, F mask)
{
    const int S = (int)leader.size(), W = OFDM_MASK_WORDS;
    std::vector<std::vector<int32_t>> members((size_t)S);
    for (int s = 0; s < S; s++) members[(size_t)leader[(size_t)s]].push_back(s);
    Grouping gr;
    gr.gid.assign((size_t)S, -1); gr.row.assign((size_t)S, -1); gr.lmask.assign((size_t)S * W, 0u);
    for (int L = 0; L < S; L++) {
        const auto& mb = members[(size_t)L];
        if (mb.size() < 2) continue;
        uint32_t m[OFDM_MASK_WORDS] = {0u, 0u, 0u, 0u};
        mask(L, m);
        const int gi = (int)gr.groups.size();
        int nsym = 0;
        for (int l = 1; l <= 75; l++)
            if ((m[l >> 5] >> (l & 31)) & 1u) { gr.items.push_back(CombItem{gi, l, nsym, nsym == 0}); nsym++; }
        CombGroup g{};
        g.n = (int32_t)mb.size();
        for (int i = 0; i < g.n; i++) {
            const int s = mb[(size_t)i];
            if (s == L) g.lpos = i;
            g.stream[i] = s; g.row[i] = (int32_t)(gr.rows + (int64_t)i * nsym);
            gr.gid[(size_t)s] = gi; gr.row[(size_t)s] = g.row[i];
            for (int w = 0; w < W; w++) gr.lmask[(size_t)s * W + w] = m[w];
        }
        gr.rows += (int64_t)g.n * nsym;
        gr.groups.push_back(g);
    }
    return gr;
}

// The tables of diversity combining for a leader table that forms at least one group, built whole and then swapped into c (the caller
// has run sync_all).  Each group combines the data symbols its leader's decoders read; with keep_taps every symbol, from tap 2's rows.
// A failure leaves c's tables as they were: the last step, which cannot fail, takes over their r1 buffer when it is neither too small
// nor more than twice the size needed.
int rebuild_comb(dabb_ctx* ctx, Combining& c, std::shared_ptr<const std::vector<int32_t>> leader)
{
    const bool taps = !ctx->d_symmask;
    Grouping gr = group_streams(*leader, [&](int L, uint32_t* m) { if (taps) all_symbols(L, m); else own_symmask(ctx, L, m); });
    if (taps) for (CombGroup& g : gr.groups) for (int i = 0; i < g.n; i++) g.row[i] = 75 * g.stream[i];
    auto t = std::make_unique<CombTables>();
    t->leader = std::move(leader); t->n_items = (int)gr.items.size();
    const size_t need = (size_t)gr.rows * KC;
    const bool keep_r1 = !taps && c.tab && need <= c.tab->r1.size() && 2 * need >= c.tab->r1.size();
    int rc;
    if ((rc = upload(ctx, t->groups, gr.groups)) || (rc = upload(ctx, t->items, gr.items)) || (rc = upload(ctx, t->gid, gr.gid))) return rc;
    if (!taps && ((rc = upload(ctx, t->row, gr.row)) || (rc = upload(ctx, t->lmask, gr.lmask)) || (!keep_r1 && (rc = alloc(ctx, t->r1, need))))) return rc;
    CK(cudaStreamSynchronize(ctx->stream));
    if (keep_r1) t->r1 = std::move(c.tab->r1);
    c.tab = std::move(t);
    return DABB_OK;
}

// streams [first, first + count) of `slot` take state v (v.enabled = 0: removed).  The slot's grouped Viterbi schedule, its decision
// buffer and its largest frame length follow the new membership; the new buffers are allocated and filled before any is replaced, so
// that a failed allocation leaves the slot as it was.  Every other stream's state and buffers are untouched.  (The caller has run
// sync_all: nothing on the device uses the buffers replaced here.)
int set_slot_streams(dabb_ctx* ctx, int slot, int first, int count, const MscSlotState& v)
{
    const int S = ctx->S, ns = ctx->n_slots;
    auto& sl = ctx->slot[slot];
    int rc;
    if (sl.configured) {
        std::vector<int32_t> prof_of((size_t)S), nsteps(ctx->profiles.size());
        int flen = 0;
        for (int s = 0; s < S; s++) {
            const MscSlotState& m = (s >= first && s < first + count) ? v : ctx->h_slots[(size_t)s * ns + slot];
            prof_of[(size_t)s] = m.enabled ? m.profile : -1;
            if (m.enabled) flen = std::max(flen, 3 * m.bitrate);
        }
        for (size_t i = 0; i < ctx->profiles.size(); i++) nsteps[i] = ctx->profiles[i].nsteps;
        VitSchedule sch;
        build_vit_schedule(prof_of.data(), S, nsteps.data(), (int)nsteps.size(), sch);
        DevBuf<uint2> dec; DevBuf<VitGroup> groups; DevBuf<int32_t> list;
        if (((size_t)sch.dec_words > sl.d_dec.size() && (rc = alloc(ctx, dec, (size_t)sch.dec_words))) ||
            (rc = alloc(ctx, groups, sch.groups.size())) || (rc = alloc(ctx, list, sch.list.size())))
            return rc;
        CK(cudaMemcpyAsync(groups, sch.groups.data(), sch.groups.size() * sizeof(VitGroup), cudaMemcpyHostToDevice, ctx->stream));
        if (!sch.list.empty()) CK(cudaMemcpyAsync(list, sch.list.data(), sch.list.size() * sizeof(int32_t), cudaMemcpyHostToDevice, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        if (dec) sl.d_dec = std::move(dec);
        sl.d_groups = std::move(groups); sl.d_cw_list = std::move(list); sl.n_groups = (int)sch.groups.size(); sl.flen = flen;
    }
    set_slot_kernel<<<(count + 127) / 128, 128, 0, ctx->stream>>>(ctx->d_slots, ns, slot, first, count, v);
    for (int i = first; i < first + count; i++) ctx->h_slots[(size_t)i * ns + slot] = v;
    if ((rc = upload_symmask(ctx, first, count)) || (comb_tab(ctx) && (rc = rebuild_comb(ctx, *ctx->comb, comb_tab(ctx)->leader)))) return rc;
    { int rc_ = check_launch(ctx, "set_slot_kernel"); cudaStreamSynchronize(ctx->stream); return rc_; }
}

} // namespace

// =====================================================================================================================
extern "C" {

int dabb_abi_version(void) { return DABB_ABI_VERSION; }

const char* dabb_last_error(const dabb_ctx* ctx) { return ctx ? ctx->err.c_str() : g_create_error.c_str(); }

int dabb_create(const dabb_config* cfg, dabb_ctx** out)
{
    if (!cfg || !out) { g_create_error = "null argument"; return DABB_E_ARG; }
    if (cfg->abi_version != DABB_ABI_VERSION) { g_create_error = "ABI version mismatch"; return DABB_E_ARG; }
    if (cfg->transmission_mode != 1 && cfg->transmission_mode != 0) { g_create_error = "only transmission mode I is supported"; return DABB_E_UNSUPPORTED; }
    if (cfg->n_streams < 1) { g_create_error = "n_streams < 1"; return DABB_E_ARG; }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { g_create_error = "no CUDA device: this library has no CPU fallback"; return DABB_E_NODEVICE; }
    if (cfg->device < 0 || cfg->device >= ndev) { g_create_error = "bad device ordinal"; return DABB_E_ARG; }
    dabb_ctx* ctx = new dabb_ctx();
    ctx->device = cfg->device; ctx->S = cfg->n_streams; ctx->fft_mode = cfg->fft_mode; ctx->disable_coarse = cfg->disable_coarse; ctx->keep_taps = cfg->keep_taps; ctx->placement = cfg->fft_placement; ctx->freqsync = cfg->freqsync_method;
    ctx->n_slots = cfg->n_subch_slots > 0 ? (cfg->n_subch_slots > DABB_MAX_SUBCH ? DABB_MAX_SUBCH : cfg->n_subch_slots) : 1;
    ctx->max_cu = cfg->max_subch_cu > 0 ? std::min(cfg->max_subch_cu, 864) : 144;     // no sub-channel is larger than the MSC's 864 CUs
    ctx->groups = cfg->ofdm_groups > 0 ? cfg->ofdm_groups : (ctx->S >= 1024 ? 1 : (ctx->S >= 64 ? 5 : 25));
    if (75 % ctx->groups) ctx->groups = 1;
    ctx->nco_fast = cfg->nco_mode == DABB_NCO_FAST;
    auto fail = [&](int code) { g_create_error = ctx->err; dabb_destroy(ctx); return code; };
    if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return fail(DABB_E_CUDA); }
    // Two lanes (enqueue_step): lane A (ctx->stream: time sync + OFDM of frame n+1) and lane B (streamB: MSC + RS of frame n, with its
    // FIC chain on stream2, which overlaps the MSC chain; both only depend on the OFDM kernel) become runnable at the same moment.  Lane B
    // gets the higher priority and runs first, in a burst: its CTAs take every slot the OFDM launch frees.  (Sharing the SMs instead, with
    // the OFDM kernel capped so that a Viterbi CTA fits beside it, slowed the OFDM kernel by as much as the two overlapped; DESIGN.md 3.3.)
    int prio_lo = 0, prio_hi = 0; cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);
    if (cudaStreamCreateWithPriority(&ctx->stream, cudaStreamNonBlocking, prio_lo) != cudaSuccess ||
        cudaStreamCreateWithPriority(&ctx->streamB, cudaStreamNonBlocking, prio_hi) != cudaSuccess ||
        cudaStreamCreateWithPriority(&ctx->stream2, cudaStreamNonBlocking, prio_hi) != cudaSuccess) { ctx->err = "cudaStreamCreate failed"; return fail(DABB_E_CUDA); }
    for (int i = 0; i < 2; i++) if (cudaEventCreateWithFlags(&ctx->evA[i], cudaEventDisableTiming) != cudaSuccess || cudaEventCreateWithFlags(&ctx->evB[i], cudaEventDisableTiming) != cudaSuccess) { ctx->err = "event creation failed"; return fail(DABB_E_CUDA); }
    if ( cudaEventCreateWithFlags(&ctx->ev_ofdm, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&ctx->ev_fic, cudaEventDisableTiming) != cudaSuccess) { ctx->err = "stream/event creation failed"; return fail(DABB_E_CUDA); }
    ctx->host = new HostTables();
    build_host_tables(*ctx->host);
    const int S = ctx->S;
    int rc = 0;
    ctx->tail_frames = (cfg->ofdm_tail_split == 0 && ctx->groups == 1) ? ofdm_tail_frames(S) : 0;
    ctx->fc_pitch = ctx->tail_frames ? OFDM_TAIL_GROUPS : ctx->groups;
    // tables
    auto& tf = ctx->d_tw_fwd; auto& ti = ctx->d_tw_inv; auto& pr = ctx->d_prs_ref; auto& osc = ctx->d_osc; auto& ip = ctx->d_invperm; auto& fm = ctx->d_fic_map;
    auto& ge = ctx->d_gf_exp; auto& gl = ctx->d_gf_log;
    if ((rc = dalloc(ctx, tf, TwLayout::TOTAL)) || (rc = dalloc(ctx, ti, TwLayout::TOTAL)) || (rc = dalloc(ctx, pr, TU)) || (rc = dalloc(ctx, osc, INPUT_RATE, false)) ||
        (rc = dalloc(ctx, ip, sizeof ctx->host->invperm / sizeof(int16_t))) || (rc = dalloc(ctx, fm, 3096)) || (rc = dalloc(ctx, ge, 512)) || (rc = dalloc(ctx, gl, 256)))
        return fail(rc);
    {
        ctx->h_osc.resize(INPUT_RATE);
        build_osc_table(ctx->h_osc.data());
        cudaMemcpyAsync(osc, ctx->h_osc.data(), sizeof(float2) * INPUT_RATE, cudaMemcpyHostToDevice, ctx->stream);
        cudaMemcpyAsync(tf, ctx->host->tw_fwd, sizeof(float2) * TwLayout::TOTAL, cudaMemcpyHostToDevice, ctx->stream);
        cudaMemcpyAsync(ti, ctx->host->tw_inv, sizeof(float2) * TwLayout::TOTAL, cudaMemcpyHostToDevice, ctx->stream);
        cudaMemcpyAsync(pr, ctx->host->prs_ref, sizeof(float2) * TU, cudaMemcpyHostToDevice, ctx->stream);
        cudaMemcpyAsync(ip, ctx->host->invperm, sizeof ctx->host->invperm, cudaMemcpyHostToDevice, ctx->stream);
        cudaMemcpyAsync(fm, ctx->host->fic_map, sizeof(int16_t) * 3096, cudaMemcpyHostToDevice, ctx->stream);
        cudaMemcpyAsync(ge, ctx->host->gf_exp, 512, cudaMemcpyHostToDevice, ctx->stream);
        cudaMemcpyAsync(gl, ctx->host->gf_log, 256, cudaMemcpyHostToDevice, ctx->stream);
        if (cudaStreamSynchronize(ctx->stream) != cudaSuccess) { ctx->err = "table upload failed"; return fail(DABB_E_CUDA); }
    }
    ctx->dev.tw_fwd = tf; ctx->dev.tw_inv = ti; ctx->dev.prs_ref = pr; ctx->dev.osc = osc; ctx->dev.invperm = ip; ctx->dev.fic_map = fm;
    ctx->dev.gf_exp = ge; ctx->dev.gf_log = gl;
    {
        // on-the-fly oscillator: upload the factors, compare against the table for every index on the device, adopt it only when
        // nothing differs (else the kernels keep the table lookups)
        auto& hi = ctx->d_osc_hi;
        if ((rc = dalloc(ctx, hi, 2000))) return fail(rc);
        std::vector<double2> h_hi(2000);
        build_osc_factors(ctx->h_osc.data(), h_hi.data(), &ctx->dev.osc_theta, &ctx->osc_patched);
        cudaMemcpyAsync(hi, h_hi.data(), sizeof(double2) * 2000, cudaMemcpyHostToDevice, ctx->stream);
        cudaStreamSynchronize(ctx->stream);
        ctx->dev.osc_hi = hi; ctx->dev.osc_mode = 0;
        ctx->osc_mismatches = launch_osc_verify(ctx->dev, ctx->stream);
        if (ctx->osc_mismatches == 0) ctx->dev.osc_mode = 1;
        std::vector<float2>().swap(ctx->h_osc);
    }
    {
        std::vector<uint32_t> w(768 / 32); build_prbs_words(768, w.data());
        if ((rc = dalloc(ctx, ctx->d_fic_prbs_words, w.size()))) return fail(rc);
        cudaMemcpy(ctx->d_fic_prbs_words, w.data(), w.size() * 4, cudaMemcpyHostToDevice);
        // expansion tables of the decoder kernel for the FIC puncturing (fic-handler.cpp:144-191)
        std::vector<uint2> steps; std::vector<uint32_t> soff;
        build_vit_tables_u2(ctx->host->fic_map, 774, steps, soff);
        if ((rc = dalloc(ctx, ctx->d_fic_steptab, steps.size())) || (rc = dalloc(ctx, ctx->d_fic_stage_off, soff.size()))) return fail(rc);
        cudaMemcpy(ctx->d_fic_steptab, steps.data(), steps.size() * sizeof(uint2), cudaMemcpyHostToDevice);
        cudaMemcpy(ctx->d_fic_stage_off, soff.data(), soff.size() * 4, cudaMemcpyHostToDevice);
    }
    if (getenv("DABB_TRACE")) {
        ctx->trace_path = getenv("DABB_TRACE"); ctx->trace.cap = 1u << 20;
        if ((rc = dalloc(ctx, ctx->d_trace_rec, (size_t)3 * ctx->trace.cap)) || (rc = dalloc(ctx, ctx->d_trace_count, 1))) return fail(rc);
        ctx->trace.rec = ctx->d_trace_rec; ctx->trace.count = ctx->d_trace_count;
    }
    ctx->ring_pitch = ctx->max_cu * 64;
    if ((rc = dalloc(ctx, ctx->d_state, S)) || (rc = dalloc(ctx, ctx->d_scr, 2 * (size_t)S)) || (rc = dalloc(ctx, ctx->d_fic_ratio, S)) || (rc = dalloc(ctx, ctx->d_coarse, S)) || (rc = dalloc(ctx, ctx->d_slots, (size_t)S * ctx->n_slots)) ||
        (rc = dalloc(ctx, ctx->d_buf_start, S)) || (rc = dalloc(ctx, ctx->d_win, 2 * (size_t)S)) || (rc = dalloc(ctx, ctx->d_prs, 2 * (size_t)S)) ||
        (rc = dalloc(ctx, ctx->d_nco_sync, 4 * (size_t)S)) || (rc = dalloc(ctx, ctx->d_nco_frame, 8 * (size_t)S)) || (rc = dalloc(ctx, ctx->d_active, 2 * (size_t)S)) ||
        (rc = dalloc(ctx, ctx->d_index, 2 * (size_t)S)) || (rc = dalloc(ctx, ctx->d_snr, 2 * (size_t)S)) || (rc = dalloc(ctx, ctx->d_fc, 2 * (size_t)S * ctx->fc_pitch)) || (rc = dalloc(ctx, ctx->d_lvl, 2 * (size_t)S * ctx->fc_pitch)) ||
        (rc = dalloc(ctx, ctx->d_soft, 2 * (size_t)S * DABB_SOFT_PER_FRAME + VIT_FRAG_SLACK, false)) ||
        (rc = dalloc(ctx, ctx->d_fibs, (size_t)S * 12 * 32)) || (rc = dalloc(ctx, ctx->d_crc, S)) || (rc = dalloc(ctx, ctx->d_results, S)) ||
        (rc = dalloc(ctx, ctx->d_info_tab, DABB_MAX_SUBCH)) || (rc = dalloc(ctx, ctx->d_cir_work, (size_t)S * TU, false)))
        return fail(rc);
    if (ctx->keep_taps && ((rc = dalloc(ctx, ctx->d_cir, (size_t)S * TU)) || (rc = dalloc(ctx, ctx->d_r1, (size_t)S * 75 * 1536)) || (rc = dalloc(ctx, ctx->d_null, (size_t)S * TNULL)))) return fail(rc);
    if ((rc = dalloc(ctx, ctx->d_dec, vit_dec_bytes(S * 4, 774) / sizeof(uint2), false)) || (rc = dalloc(ctx, ctx->d_dec_fic, vit_dec_bytes(S * 4, 774) / sizeof(uint2), false))) return fail(rc);
    ctx->h_slots.assign((size_t)S * ctx->n_slots, MscSlotState{});
    // keep_taps exposes every symbol's softbits and constellation, so only a context without it skips the symbols nothing reads
    if (!ctx->keep_taps && ((rc = dalloc(ctx, ctx->d_symmask, (size_t)S * OFDM_MASK_WORDS)) || (rc = upload_symmask(ctx, 0, S)))) return fail(rc);
    ctx->profiles.reserve(DABB_MAX_PROFILES);
    if ((rc = dalloc(ctx, ctx->d_profiles, DABB_MAX_PROFILES))) return fail(rc);
    // info arrays of unconfigured slots are never read (finalize skips disabled slots)
    if ((rc = prepare_pending(ctx, ctx->pend_sync))) return fail(rc);
    {
        reset_kernel<<<(S + 127) / 128, 128, 0, ctx->stream>>>(ctx->d_state, ctx->d_slots, ctx->n_slots, 0, S, 0, ctx->d_fic_ratio);
        ctx->launches++;
    }
    if (cudaStreamSynchronize(ctx->stream) != cudaSuccess) { ctx->err = std::string("init failed: ") + cudaGetErrorString(cudaGetLastError()); return fail(DABB_E_CUDA); }
    *out = ctx;
    return DABB_OK;
}

void dabb_destroy(dabb_ctx* ctx)
{
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    sync_all(ctx);
    if (ctx->trace.rec && !ctx->trace_path.empty()) {       // CTA timeline: kind, sm, start ns, end ns per line
        unsigned int n = 0; cudaMemcpy(&n, ctx->trace.count, 4, cudaMemcpyDeviceToHost);
        if (n > ctx->trace.cap) n = ctx->trace.cap;
        std::vector<unsigned long long> h((size_t)3 * n);
        cudaMemcpy(h.data(), ctx->trace.rec, h.size() * 8, cudaMemcpyDeviceToHost);
        if (FILE* f = fopen(ctx->trace_path.c_str(), "w")) { for (unsigned int i = 0; i < n; i++) fprintf(f, "%llu %llu %llu %llu\n", h[3 * i] >> 32, h[3 * i] & 0xFFFFFFFFull, h[3 * i + 1], h[3 * i + 2]); fclose(f); }
    }
    for (cudaEvent_t e : ctx->prof_ev) cudaEventDestroy(e);
    for (int i = 0; i < 2; i++) {
        if (ctx->evH2D[i]) cudaEventDestroy(ctx->evH2D[i]);
        if (ctx->evStageFree[i]) cudaEventDestroy(ctx->evStageFree[i]);
        if (ctx->pend[i].done) cudaEventDestroy(ctx->pend[i].done);
    }
    if (ctx->pend_sync.done) cudaEventDestroy(ctx->pend_sync.done);
    if (ctx->streamC) cudaStreamDestroy(ctx->streamC);
    if (ctx->ev_ofdm) cudaEventDestroy(ctx->ev_ofdm);
    if (ctx->ev_fic) cudaEventDestroy(ctx->ev_fic);
    for (int i = 0; i < 2; i++) { if (ctx->evA[i]) cudaEventDestroy(ctx->evA[i]); if (ctx->evB[i]) cudaEventDestroy(ctx->evB[i]); }
    if (ctx->streamB) cudaStreamDestroy(ctx->streamB);
    if (ctx->stream2) cudaStreamDestroy(ctx->stream2);
    if (ctx->stream) cudaStreamDestroy(ctx->stream);
    delete ctx->host;
    delete ctx;         // frees every device and pinned buffer
}

void* dabb_cuda_stream(dabb_ctx* ctx) { return ctx ? (void*)ctx->stream : nullptr; }
int64_t dabb_kernel_launches(const dabb_ctx* ctx) { return ctx ? ctx->launches : 0; }
int dabb_sync(dabb_ctx* ctx) { if (!ctx) return DABB_E_ARG; cudaSetDevice(ctx->device); CK(cudaStreamSynchronize(ctx->stream)); CK(cudaStreamSynchronize(ctx->streamB)); CK(cudaStreamSynchronize(ctx->stream2)); if (ctx->prof) prof_collect(ctx); return 0; }

int dabb_join_lanes(dabb_ctx* ctx)
{
    if (!ctx) return DABB_E_ARG;
    cudaSetDevice(ctx->device);
    if (ctx->prof || !ctx->evB_valid[ctx->last_parity]) return DABB_OK;       // serial mode: everything is on the main stream already
    CK(cudaStreamWaitEvent(ctx->stream, ctx->evB[ctx->last_parity], 0));       // lane B's last record follows the FIC stream's join
    return DABB_OK;
}

int dabb_stream_reset(dabb_ctx* ctx, int32_t first, int32_t count, int64_t pos)
{
    if (!ctx || first < 0 || count < 0 || first + count > ctx->S) return DABB_E_ARG;
    if (!count) return 0;
    cudaSetDevice(ctx->device);
    sync_all(ctx);
    reset_kernel<<<(count + 127) / 128, 128, 0, ctx->stream>>>(ctx->d_state, ctx->d_slots, ctx->n_slots, first, count, pos, ctx->d_fic_ratio);
    if (ctx->tii) CK(cudaMemsetAsync(ctx->tii->hdr + first, 0, sizeof(dabb_tii::StreamHdr) * count, ctx->stream));     // no open TII combinations
    for (int i = first; i < first + count; i++) for (int k = 0; k < ctx->n_slots; k++) { ctx->h_slots[(size_t)i * ctx->n_slots + k].cif_count = 0; ctx->h_slots[(size_t)i * ctx->n_slots + k].sf_frame_count = 0; }
    { int rc_ = check_launch(ctx, "reset_kernel"); cudaStreamSynchronize(ctx->stream); ctx->evB_valid[0] = ctx->evB_valid[1] = false; return rc_; }
}

int dabb_select_subchannel(dabb_ctx* ctx, int32_t first, int32_t count, int32_t slot, const dabb_subchannel* sc)
{
    if (!ctx || !sc || first < 0 || count < 1 || first + count > ctx->S || slot < 0 || slot >= ctx->n_slots) return DABB_E_ARG;
    cudaSetDevice(ctx->device);
    sync_all(ctx);
    ProtProfile prof;
    if (make_prot_profile(sc->bitrate, sc->short_form, sc->uep_level, sc->eep_profile_a, sc->eep_level, prof) < 0) { ctx->err = "unsupported protection profile"; return DABB_E_UNSUPPORTED; }
    if (sc->length_cu < 1 || sc->length_cu > ctx->max_cu || sc->start_cu < 0 || sc->start_cu + sc->length_cu > 864) { ctx->err = "sub-channel does not fit (raise dabb_config.max_subch_cu)"; return DABB_E_ARG; }
    if (prof.in_bits > sc->length_cu * 64) { ctx->err = "protection profile needs more bits than the sub-channel holds"; return DABB_E_ARG; }
    if (sc->dabplus && sc->bitrate / 8 > 64) { ctx->err = "DAB+ sub-channels above 512 kbit/s are not supported"; return DABB_E_UNSUPPORTED; }
    int pi = -1;
    for (size_t i = 0; i < ctx->profiles.size(); i++) if (!memcmp(&ctx->profiles[i].prof, &prof, sizeof prof)) pi = (int)i;
    if (pi < 0 && ctx->profiles.size() >= (size_t)DABB_MAX_PROFILES) {
        ctx->err = "more than " + std::to_string(DABB_MAX_PROFILES) + " distinct protection profiles in one context"; return DABB_E_UNSUPPORTED;
    }
    int rc = 0;
    if (pi < 0 && (rc = add_profile(ctx, prof))) return rc;
    if (pi < 0) pi = (int)ctx->profiles.size() - 1;
    const auto& pf = ctx->profiles[(size_t)pi];
    auto& sl = ctx->slot[slot];
    const int S = ctx->S;
    const bool fresh = !sl.configured;
    if (fresh) {
        sl.frag_pitch = ctx->ring_pitch; sl.flen_pad = pf.flen_pad;
        if ((rc = dalloc(ctx, sl.d_frag, (size_t)S * 4 * sl.frag_pitch + VIT_FRAG_SLACK)) ||
            (rc = dalloc(ctx, sl.d_valid, (size_t)S * 4)) || (rc = dalloc(ctx, sl.d_logical, (size_t)S * 4 * sl.flen_pad)) ||
            (rc = dalloc(ctx, sl.d_window, (size_t)S * 5 * sl.flen_pad)) || (rc = dalloc(ctx, sl.d_sf, (size_t)S * 5 * sl.flen_pad)) ||
            (rc = dalloc(ctx, sl.d_info, (size_t)S * 16)))
            { sl = dabb_ctx::Slot{}; return rc; }
        if (!ctx->d_ring[slot] && (rc = dalloc(ctx, ctx->d_ring[slot], (size_t)S * MSC_RING * ctx->ring_pitch))) { sl = dabb_ctx::Slot{}; return rc; }
        sl.configured = true;
    } else if (pf.flen_pad > sl.flen_pad) {
        // wider rows: every stream's logical frames, superframe window and last superframe move into the new layout unchanged
        const size_t o = (size_t)sl.flen_pad, n = (size_t)pf.flen_pad;
        if ((rc = repitch(ctx, sl.d_logical, (size_t)S * 4, o, n)) || (rc = repitch(ctx, sl.d_window, S, 5 * o, 5 * n)) || (rc = repitch(ctx, sl.d_sf, S, 5 * o, 5 * n))) return rc;
        sl.flen_pad = pf.flen_pad;
    }
    MscSlotState v{}; v.enabled = 1; v.start_cu = sc->start_cu; v.frag = sc->length_cu * 64; v.bitrate = sc->bitrate; v.dabplus = sc->dabplus; v.profile = pi; v.cif_count = 0; v.sf_frame_count = 0;
    if ((rc = set_slot_streams(ctx, slot, first, count, v))) { if (fresh) sl = dabb_ctx::Slot{}; return rc; }
    return DABB_OK;
}

int dabb_remove_subchannel(dabb_ctx* ctx, int32_t first, int32_t count, int32_t slot)
{
    if (!ctx || first < 0 || count < 1 || first + count > ctx->S || slot < 0 || slot >= ctx->n_slots) return DABB_E_ARG;
    cudaSetDevice(ctx->device);
    sync_all(ctx);
    return set_slot_streams(ctx, slot, first, count, MscSlotState{});
}

int dabb_set_combining(dabb_ctx* ctx, const int32_t* leader, int32_t n)
{
    if (!ctx) return DABB_E_ARG;
    const int S = ctx->S;
    bool grouped = false;       // some stream is not its own leader: a group of two or more forms
    if (leader) {
        if (n != S) { ctx->err = "dabb_set_combining: the table needs n_streams entries"; return DABB_E_ARG; }
        std::vector<int> size((size_t)S, 0);
        for (int s = 0; s < S; s++) {
            const int32_t v = leader[s];
            if (v < 0 || v >= S) { ctx->err = "dabb_set_combining: leader[" + std::to_string(s) + "] is not a stream"; return DABB_E_ARG; }
            if (leader[v] != v) { ctx->err = "dabb_set_combining: leader[" + std::to_string(s) + "] is not a leader (leader[leader[s]] != leader[s])"; return DABB_E_ARG; }
            if (++size[(size_t)v] > DABB_MAX_BRANCHES) { ctx->err = "dabb_set_combining: a group has more than DABB_MAX_BRANCHES members"; return DABB_E_ARG; }
            grouped |= v != s;
        }
    }
    cudaSetDevice(ctx->device);
    sync_all(ctx);
    const bool was = comb_tab(ctx) != nullptr;
    int rc;
    if (grouped) {
        // a group of two or more: its tables, with tap 12's records when this is the first group the context forms
        std::unique_ptr<Combining> fresh;
        if (!ctx->comb) { fresh = std::make_unique<Combining>(); if ((rc = dalloc(ctx, fresh->res, (size_t)S))) return rc; }
        if ((rc = rebuild_comb(ctx, fresh ? *fresh : *ctx->comb, std::make_shared<const std::vector<int32_t>>(leader, leader + S)))) return rc;
        if (fresh) ctx->comb = std::move(fresh);
    } else if (ctx->comb)
        ctx->comb->tab = nullptr;       // no group: every table is freed, tap 12's records stay
    if ((was || comb_tab(ctx)) && (rc = upload_symmask(ctx, 0, S))) return rc;
    CK(cudaStreamSynchronize(ctx->stream));
    return DABB_OK;
}


static int run_fic(dabb_ctx* ctx, const int8_t* soft, int64_t soft_stride, const int32_t* active, int n_frames, uint8_t* fibs, int32_t* crc, cudaStream_t st, uint2* dec)
{
    int rc;
    // FIC codeword (frame f, block b) = softbits [2304 b, 2304 b + 2304) of the frame's first three symbols (fic-handler.cpp:111-127):
    // the decoder kernel reads them where the OFDM kernel wrote them and de-punctures on the fly
    ViterbiParams vp{};
    vp.frag = soft; vp.cw_div = 4; vp.outer_stride = soft_stride; vp.inner_stride = 2304; vp.steptab = ctx->d_fic_steptab; vp.stage_off = ctx->d_fic_stage_off;
    vp.n_cw = n_frames * 4; vp.nsteps = 774; vp.nbits = 768;
    vp.dec = dec; vp.out = fibs; vp.out_stride = 96; vp.prbs_words = ctx->d_fic_prbs_words; vp.valid = nullptr;
    vp.trace = ctx->trace; vp.trace_kind = 2;
    launch_viterbi(vp, st);
    if ((rc = check_launch(ctx, "viterbi_kernel(FIC)"))) return rc;
    launch_fic_crc(fibs, active, n_frames, crc, st);
    return check_launch(ctx, "fic_crc_kernel");
}

static int enqueue_step(dabb_ctx* ctx, const dabb_io* io, const float2* iq, int64_t stride);

// cf32 samples in d_iq_stage from raw-format samples on the device (stream s at raw + s * raw_stride samples), converted on lane A
static int convert_to_stage(dabb_ctx* ctx, const uint8_t* raw, int64_t raw_stride, int fmt, int64_t len)
{
    const int S = ctx->S;
    int rc;
    if ((rc = grow(ctx, ctx->d_iq_stage, (size_t)S * len))) return rc;
    const dim3 grid((unsigned)((len + 255) / 256), (unsigned)S);
    convert_iq_kernel<<<grid, 256, 0, ctx->stream>>>(raw, raw_stride, fmt, ctx->d_iq_stage, len, len, S);
    return check_launch(ctx, "convert_iq_kernel");
}

int dabb_process_async(dabb_ctx* ctx, const dabb_io* io)
{
    if (!ctx || !io || !io->iq || !io->buf_start) return DABB_E_ARG;
    cudaSetDevice(ctx->device);
    const int S = ctx->S;
    int rc;
    cudaStream_t A = ctx->stream;
    const float2* iq = reinterpret_cast<const float2*>(io->iq);
    int64_t stride = io->stride_samples;
    const int fmt = io->iq_format;
    if (fmt < 0 || fmt > DABB_IQ_S16BE) { ctx->err = "unknown iq_format"; return DABB_E_ARG; }
    if (io->iq_is_host || fmt != DABB_IQ_CF32) {
        const size_t need = (size_t)S * io->buf_len, bps = (size_t)bytes_per_sample(fmt);
        if (fmt == DABB_IQ_CF32) {
            if ((rc = grow(ctx, ctx->d_iq_stage, need))) return rc;
            CK(cudaMemcpy2DAsync(ctx->d_iq_stage, (size_t)io->buf_len * bps, io->iq, (size_t)stride * bps, (size_t)io->buf_len * bps, S, cudaMemcpyHostToDevice, A));
        } else {
            const uint8_t* raw = reinterpret_cast<const uint8_t*>(io->iq);
            int64_t raw_stride = stride;
            if (io->iq_is_host) {
                if ((rc = grow(ctx, ctx->d_raw_stage, need * bps))) return rc;
                CK(cudaMemcpy2DAsync(ctx->d_raw_stage, (size_t)io->buf_len * bps, io->iq, (size_t)stride * bps, (size_t)io->buf_len * bps, S, cudaMemcpyHostToDevice, A));
                raw = ctx->d_raw_stage; raw_stride = io->buf_len;
            }
            if ((rc = convert_to_stage(ctx, raw, raw_stride, fmt, io->buf_len))) return rc;
        }
        iq = ctx->d_iq_stage; stride = io->buf_len;
    }
    return enqueue_step(ctx, io, iq, stride);
}

// one decode step on device-resident cf32 samples (stream s at iq + s * stride)
static int enqueue_step(dabb_ctx* ctx, const dabb_io* io, const float2* iq, int64_t stride)
{
    const int S = ctx->S;
    int rc;
    // Two lanes: A = acquisition, time sync, OFDM demod and the sync-state update of frame n; B = FIC, MSC, RS and the
    // result record of frame n.  Lane A of frame n+1 only needs lane A of frame n, so B(n) overlaps A(n+1); the per-frame
    // scratch and the softbits are double buffered by frame parity.  With per-kernel profiling on everything runs
    // serially on the main stream.
    const int par = (int)(ctx->step & 1);
    const bool serial = ctx->prof;
    cudaStream_t A = ctx->stream, B = serial ? ctx->stream : ctx->streamB;
    StepScratch* scr = ctx->d_scr + (size_t)par * S;
    int64_t* d_win = ctx->d_win + (size_t)par * S; int64_t* d_prs = ctx->d_prs + (size_t)par * S;
    int32_t* d_nco_sync = ctx->d_nco_sync + (size_t)par * 2 * S; int32_t* d_nco_frame = ctx->d_nco_frame + (size_t)par * 4 * S;
    int32_t* d_active = ctx->d_active + (size_t)par * S; int32_t* d_index = ctx->d_index + (size_t)par * S; int32_t* d_snr = ctx->d_snr + (size_t)par * S;
    float2* d_fc = ctx->d_fc + (size_t)par * S * ctx->fc_pitch; float* d_lvl = ctx->d_lvl + (size_t)par * S * ctx->fc_pitch;
    int8_t* d_soft = ctx->d_soft + (size_t)par * S * DABB_SOFT_PER_FRAME;

    // the buffers of this parity were last used by lane B two frames ago
    if (!serial && ctx->evB_valid[par]) CK(cudaStreamWaitEvent(A, ctx->evB[par], 0));
    CK(cudaMemcpyAsync(ctx->d_buf_start, io->buf_start, sizeof(int64_t) * S, cudaMemcpyHostToDevice, A));
    prof_mark(ctx, "__step_begin");
    const int tb = 128, gb = (S + tb - 1) / tb;
    // ---------------- lane A
    const bool robust = ctx->acquisition == DABB_ACQ_ROBUST;
    Acq* aq = ctx->acq.get();
    if (robust) {       // the spectral null search of every stream that is not tracking, then the same hand-off to time sync
        if ((rc = clear_records(ctx, aq->exc, A))) return rc;
        acq_plan_kernel<<<gb, tb, 0, A>>>(ctx->d_state, ctx->d_buf_start, io->buf_len, S, aq->job);
        if ((rc = check_launch(ctx, "acq_plan_kernel"))) return rc;
        launch_acq_levels(aq->job, iq, stride, ctx->dev.osc, aq->cos, S, aq->level, aq->l1, A);
        if ((rc = check_launch(ctx, "acq_level_kernel"))) return rc;
        acq_decide_kernel<<<S, 256, 0, A>>>(ctx->d_state, aq->job, ctx->d_buf_start, aq->level, aq->l1, aq->res);
        if ((rc = check_launch(ctx, "acq_decide_kernel"))) return rc;
    } else {
        if (aq && ((rc = clear_records(ctx, aq->res, A)) || (rc = clear_records(ctx, aq->exc, A)))) return rc;     // tap 13: nothing searched robustly
        acquire_kernel<<<(S + 31) / 32, 32, 0, A>>>(ctx->d_state, iq, stride, ctx->d_buf_start, io->buf_len, ctx->dev.osc, S);
        if ((rc = check_launch(ctx, "acquire_kernel"))) return rc;
    }
    plan_kernel<<<gb, tb, 0, A>>>(ctx->d_state, scr, ctx->d_buf_start, io->buf_len, S, d_win, d_nco_sync, d_active);
    if ((rc = check_launch(ctx, "plan_kernel"))) return rc;
    SyncParams sp{}; sp.iq = iq; sp.stride = stride; sp.win_start = d_win; sp.nco = d_nco_sync; sp.active = d_active; sp.index_out = d_index; sp.cir_out = ctx->d_cir; sp.n = S;
    sp.fic_ratio = ctx->d_fic_ratio; sp.coarse_out = ctx->disable_coarse ? nullptr : ctx->d_coarse.get(); sp.placement = ctx->placement; sp.freqsync = ctx->freqsync;
    sp.cir_work = ctx->d_cir_work;
    launch_find_index(ctx->dev, sp, A, 0, robust ? aq->exc.get() : nullptr);
    if ((rc = check_launch(ctx, robust ? "find_index_excise_kernel" : "find_index_kernel"))) return rc;
    launch_find_index(ctx->dev, sp, A, 1);
    if ((rc = check_launch(ctx, "find_search_kernel"))) return rc;
    if (sp.coarse_out) {
        launch_find_index(ctx->dev, sp, A, 2);
        if ((rc = check_launch(ctx, "find_coarse_kernel"))) return rc;
    }
    const bool track = ctx->sample_clock == DABB_CLOCK_TRACK;
    float* d_clock_frame = track ? ctx->clock->frame + (size_t)par * S : nullptr;
    post_sync_kernel<<<gb, tb, 0, A>>>(ctx->d_state, scr, d_index, ctx->disable_coarse ? nullptr : ctx->d_coarse.get(), S, d_prs, d_nco_frame, d_active, d_clock_frame);
    if ((rc = check_launch(ctx, "post_sync_kernel"))) return rc;
    const CombTables* ct = comb_tab(ctx);
    OfdmParams op{}; op.iq = iq; op.stride = stride; op.prs_start = d_prs; op.nco = d_nco_frame; op.active = d_active; op.soft = d_soft; op.soft_stride = DABB_SOFT_PER_FRAME;
    op.r1 = ctx->d_r1; op.freqcorr = d_fc; op.level = d_lvl; op.snr = d_snr; op.n_frames = S; op.groups = ctx->groups; op.sym_per_cta = 75 / ctx->groups;
    op.trace = ctx->trace;
    op.n_full = S - ctx->tail_frames; op.tail_groups = ctx->tail_frames ? OFDM_TAIL_GROUPS : 1; op.fc_pitch = ctx->fc_pitch; op.nco_fast = ctx->nco_fast; op.weighted = ctx->soft_demap == DABB_DEMAP_WEIGHTED;
    op.symmask = ctx->d_symmask; op.clock = d_clock_frame;
    if (ct && !ctx->keep_taps) { op.r1 = ct->r1; op.r1_row = ct->row; op.r1_lmask = ct->lmask; }     // the grouped streams' r1 of their leader's symbols
    launch_ofdm_demod(ctx->dev, op, ctx->fft_mode, A);
    ctx->soft_op = op; ctx->soft_partial = op.symmask != nullptr;
    if ((rc = check_launch(ctx, "ofdm_demod_kernel"))) return rc;
    advance_kernel<<<gb, tb, 0, A>>>(ctx->d_state, scr, S, ctx->fc_pitch, d_fc, d_lvl, track, ctx->clock ? ctx->clock->res.get() : nullptr);
    if ((rc = check_launch(ctx, "advance_kernel"))) return rc;
    // the null symbol: tap 3 with keep_taps, else (TII only) an internal buffer
    Tii* tii = ctx->decode_tii ? ctx->tii.get() : nullptr;
    float2* d_null = ctx->d_null ? ctx->d_null.get() : (tii ? tii->null.get() : nullptr);
    if (d_null) {
        null_tap_kernel<<<S, 256, 0, A>>>(scr, iq, stride, ctx->d_buf_start, io->buf_len, ctx->dev.osc, d_null);
        if ((rc = check_launch(ctx, "null_tap_kernel"))) return rc;
        if (tii) {
            launch_tii_spectra(ctx->dev, iq, stride, d_prs, d_nco_frame, d_active, d_null, tii->spectra, S, A);
            if ((rc = check_launch(ctx, "tii_spectra_kernel"))) return rc;
            TiiParams tp{}; tp.spectra = tii->spectra; tp.active = d_active; tp.hdr = tii->hdr; tp.jobs = tii->jobs; tp.njobs = tii->njobs;
            tp.sums = tii->sums; tp.rank = tii->rank; tp.res = tii->res.get(); tp.n = S;
            launch_tii_plan(tp, A);
            if ((rc = check_launch(ctx, "tii_plan_kernel"))) return rc;
            launch_tii_phase(tp, A);
            if ((rc = check_launch(ctx, "tii_phase_kernel"))) return rc;
        }
    }
    if (!tii && ctx->tii && (rc = clear_records(ctx, ctx->tii->res, A))) return rc;     // tap 9: nothing analysed in this step
    // diversity combining: the members' noise powers, then the leaders' softbits from their groups' products.  The step's combine launch
    // and leader table are kept for the tap-0 repeat.
    ctx->comb_op = CombParams{}; ctx->comb_leader = nullptr;
    if (ct) {
        null_power_kernel<<<S, dabb_comb::NULL_THREADS, 0, A>>>(scr, ct->gid, iq, stride, ctx->d_buf_start, io->buf_len, ctx->dev.osc, ctx->comb->res);
        if ((rc = check_launch(ctx, "null_power_kernel"))) return rc;
        CombParams cp{}; cp.groups = ct->groups; cp.items = ct->items; cp.n_items = ct->n_items; cp.r1 = ctx->keep_taps ? ctx->d_r1.get() : ct->r1.get();
        cp.active = d_active; cp.prs = d_prs; cp.buf_start = ctx->d_buf_start; cp.res = ctx->comb->res.get(); cp.soft = d_soft; cp.soft_stride = DABB_SOFT_PER_FRAME;
        cp.weighted = ctx->soft_demap == DABB_DEMAP_WEIGHTED;
        launch_combine(cp, A);
        if ((rc = check_launch(ctx, "combine_kernel"))) return rc;
        ctx->comb_op = cp; ctx->comb_leader = ct->leader;
    } else if (ctx->comb && (rc = clear_records(ctx, ctx->comb->res, A))) return rc;     // tap 12: no group in this step
    if (!serial) { CK(cudaEventRecord(ctx->evA[par], A)); CK(cudaStreamWaitEvent(B, ctx->evA[par], 0)); }
    // ---------------- lane B: FIC chain forked onto its own stream, MSC chain per slot (longest first), then the result record.
    // (One fused Viterbi launch over FIC + MSC codewords was measured slower: 1.44 ms vs 0.34 + 1.02 ms.)
    cudaStream_t F = serial ? ctx->stream : ctx->stream2;
    if (!serial) { CK(cudaEventRecord(ctx->ev_ofdm, B)); CK(cudaStreamWaitEvent(F, ctx->ev_ofdm, 0)); }
    if ((rc = run_fic(ctx, d_soft, DABB_SOFT_PER_FRAME, d_active, S, ctx->d_fibs, ctx->d_crc, F, ctx->d_dec_fic))) return rc;
    // the MER of the softbits the FIC decoder has just read, behind the same wait for lane A and before ev_fic, which guards their reuse
    if (ctx->measure_mer) {
        MerParams mp{}; mp.soft = d_soft; mp.soft_stride = DABB_SOFT_PER_FRAME; mp.active = d_active; mp.group = ctx->mer->group; mp.res = ctx->mer->res.get(); mp.n_streams = S;
        launch_mer(mp, F);
        if ((rc = check_launch(ctx, "mer_kernel"))) return rc;
    } else if (ctx->mer && (rc = clear_records(ctx, ctx->mer->res, F))) return rc;     // tap 14: nothing measured in this step
    if (!serial) CK(cudaEventRecord(ctx->ev_fic, F));
    const int32_t* h_info[DABB_MAX_SUBCH] = {nullptr, nullptr, nullptr, nullptr};
    for (int k = 0; k < ctx->n_slots; k++) {
        auto& sl = ctx->slot[k];
        h_info[k] = sl.d_info;
        if (!sl.configured) continue;
        CK(cudaMemsetAsync(sl.d_valid, 0, sizeof(int32_t) * S * 4, B));
        MscCollectParams cp{}; cp.soft = d_soft; cp.soft_stride = DABB_SOFT_PER_FRAME; cp.active = d_active; cp.slots = ctx->d_slots; cp.n_slots = ctx->n_slots; cp.slot = k; cp.ring = ctx->d_ring[k]; cp.ring_pitch = ctx->ring_pitch;
        launch_msc_collect(cp, S, B);
        if ((rc = check_launch(ctx, "msc_collect_kernel"))) return rc;
        MscPrepParams pp{}; pp.active = d_active; pp.slots = ctx->d_slots; pp.n_slots = ctx->n_slots; pp.slot = k; pp.ring = ctx->d_ring[k]; pp.ring_pitch = ctx->ring_pitch;
        pp.frag_out = sl.d_frag; pp.frag_pitch = sl.frag_pitch; pp.valid = sl.d_valid;
        launch_msc_gather(pp, S, B);
        if ((rc = check_launch(ctx, "msc_gather_kernel"))) return rc;
        // one launch for all the slot's profiles: each CTA decodes codewords of one profile (vit_groups.cuh)
        ViterbiParams vp{}; vp.frag = sl.d_frag; vp.cw_div = 1; vp.outer_stride = sl.frag_pitch; vp.inner_stride = 0;
        vp.groups = sl.d_groups; vp.cw_list = sl.d_cw_list; vp.profiles = ctx->d_profiles; vp.n_groups = sl.n_groups;
        vp.n_cw = S * 4; vp.dec = sl.d_dec; vp.out = sl.d_logical; vp.out_stride = sl.flen_pad; vp.valid = sl.d_valid;
        vp.trace = ctx->trace; vp.trace_kind = 3;
        launch_viterbi(vp, B);
        if ((rc = check_launch(ctx, "viterbi_kernel(MSC)"))) return rc;
        SuperframeParams fp{}; fp.active = d_active; fp.slots = ctx->d_slots; fp.n_slots = ctx->n_slots; fp.slot = k; fp.n_streams = S; fp.logical = sl.d_logical; fp.logical_stride = sl.flen_pad;
        fp.valid = sl.d_valid; fp.window = sl.d_window; fp.window_pitch = 5 * sl.flen_pad; fp.sf_out = sl.d_sf; fp.sf_pitch = 5 * sl.flen_pad; fp.info = sl.d_info; fp.gf_exp = ctx->dev.gf_exp; fp.gf_log = ctx->dev.gf_log;
        launch_superframe(fp, B);
        if ((rc = check_launch(ctx, "superframe_kernel"))) return rc;
    }
    if (!serial) CK(cudaStreamWaitEvent(B, ctx->ev_fic, 0));
    // the channel bit errors of the step's FIC and logical frames, while its FIBs, fragments and logical frames are all in place
    if (ctx->count_ber) {
        BerParams bp{}; bp.soft = d_soft; bp.soft_stride = DABB_SOFT_PER_FRAME; bp.fibs = ctx->d_fibs; bp.active = d_active; bp.slots = ctx->d_slots; bp.n_slots = ctx->n_slots;
        for (int k = 0; k < ctx->n_slots; k++) {
            const auto& sl = ctx->slot[k];
            if (sl.configured) bp.slot[k] = BerSlot{sl.d_frag, sl.frag_pitch, sl.d_valid, sl.d_logical, sl.flen_pad};
        }
        bp.profiles = ctx->ber->prof; bp.fic_profile = DABB_MAX_PROFILES; bp.res = ctx->ber->res.get(); bp.n_streams = S;
        launch_ber(bp, B);
        if ((rc = check_launch(ctx, "ber_kernel"))) return rc;
    } else if (ctx->ber && (rc = clear_records(ctx, ctx->ber->res, B))) return rc;     // tap 10: nothing counted in this step
    CK(cudaMemcpyAsync((void*)ctx->d_info_tab, h_info, sizeof(void*) * DABB_MAX_SUBCH, cudaMemcpyHostToDevice, B));
    finalize_kernel<<<gb, tb, 0, B>>>(scr, ctx->d_slots, ctx->n_slots, S, ctx->d_fic_ratio, d_snr, ctx->d_crc, ctx->d_info_tab, ctx->d_results);
    if ((rc = check_launch(ctx, "finalize_kernel"))) return rc;
    if (!serial) { CK(cudaEventRecord(ctx->evB[par], B)); ctx->evB_valid[par] = true; }
    ctx->last_parity = par; ctx->step++;
    return DABB_OK;
}

int dabb_process(dabb_ctx* ctx, const dabb_io* io)
{
    if (!ctx || !io) return DABB_E_ARG;
    cudaSetDevice(ctx->device);
    const StepOut o = step_out(*io);
    int rc;
    if ((rc = check_strides(ctx, o)) || (rc = prepare_pending(ctx, ctx->pend_sync)) || (rc = dabb_process_async(ctx, io)) || (rc = enqueue_readback(ctx, ctx->pend_sync, o)))
        return rc;
    CK(cudaStreamSynchronize(ctx->stream));
    return deliver(ctx, ctx->pend_sync);
}

// ---- pipelined host-buffer path -------------------------------------------------------------------------------------------------
// dabb_submit: H2D of the step's samples on a copy stream into one of two device staging slots, the kernels on the lanes, D2H of the
// results into one of two pinned result slots on lane B - and return.  dabb_collect: wait for the OLDEST outstanding step and hand
// its results to the pointers given at submit.  With two steps outstanding the copy of step n+1 overlaps the kernels of step n and
// the result read-back of step n-1.
int dabb_submit(dabb_ctx* ctx, const dabb_io* io)
{
    if (!ctx || !io || !io->iq || !io->buf_start || !io->iq_is_host) return DABB_E_ARG;
    if (ctx->prof) { ctx->err = "dabb_submit is not available while per-kernel profiling is on"; return DABB_E_STATE; }
    if (ctx->pend_count == 2) { ctx->err = "two steps are outstanding: call dabb_collect first"; return DABB_E_STATE; }
    cudaSetDevice(ctx->device);
    const int S = ctx->S, fmt = io->iq_format;
    if (fmt < 0 || fmt > DABB_IQ_S16BE) { ctx->err = "unknown iq_format"; return DABB_E_ARG; }
    const StepOut o = step_out(*io);
    int rc;
    if ((rc = check_strides(ctx, o))) return rc;
    if (!ctx->streamC) {
        CK(cudaStreamCreateWithFlags(&ctx->streamC, cudaStreamNonBlocking));
        for (int i = 0; i < 2; i++) { CK(cudaEventCreateWithFlags(&ctx->evH2D[i], cudaEventDisableTiming)); CK(cudaEventCreateWithFlags(&ctx->evStageFree[i], cudaEventDisableTiming)); }
    }
    const int slot = (int)(ctx->submits & 1);
    dabb_ctx::Pending& p = ctx->pend[(ctx->pend_head + ctx->pend_count) & 1];
    if ((rc = prepare_pending(ctx, p))) return rc;
    cudaStream_t A = ctx->stream, Cs = ctx->streamC;
    const size_t bps = (size_t)bytes_per_sample(fmt);
    const size_t need = (size_t)S * io->buf_len * bps;
    if (need > ctx->d_stage2[slot].size()) {
        if ((rc = grow(ctx, ctx->d_stage2[slot], need))) return rc;
        ctx->stageFreeValid[slot] = false;
    }
    // the staging slot was last read by the step submitted two calls ago
    if (ctx->stageFreeValid[slot]) CK(cudaStreamWaitEvent(Cs, ctx->evStageFree[slot], 0));
    // carry_samples: the head of every window is the tail of the previous one, which still lies in the other staging slot
    const int64_t carry = io->carry_samples;
    if (carry) {
        if (carry < 0 || carry >= io->buf_len || ctx->submits == 0 || ctx->stage_last_fmt != fmt || carry > ctx->stage_last_len || !ctx->d_stage2[slot ^ 1]) {
            ctx->err = "carry_samples needs a previous dabb_submit of the same format with a window at least that long"; return DABB_E_ARG;
        }
        for (int s = 0; s < S; s++)
            if (io->buf_start[s] != ctx->stage_last_start[s] + ctx->stage_last_len - carry) { ctx->err = "carry_samples: a window does not start where the previous one ended minus the carry"; return DABB_E_ARG; }
        const uint8_t* prev = ctx->d_stage2[slot ^ 1];
        CK(cudaMemcpy2DAsync(ctx->d_stage2[slot], (size_t)io->buf_len * bps, prev + (size_t)(ctx->stage_last_len - carry) * bps, (size_t)ctx->stage_last_len * bps,
                             (size_t)carry * bps, S, cudaMemcpyDeviceToDevice, Cs));          // same stream as the copy that filled the other slot
    }
    CK(cudaMemcpy2DAsync(ctx->d_stage2[slot] + (size_t)carry * bps, (size_t)io->buf_len * bps,
                         reinterpret_cast<const unsigned char*>(io->iq) + (size_t)carry * bps, (size_t)io->stride_samples * bps, (size_t)(io->buf_len - carry) * bps, S, cudaMemcpyHostToDevice, Cs));
    ctx->stage_last_fmt = fmt; ctx->stage_last_len = io->buf_len; ctx->stage_last_start.assign(io->buf_start, io->buf_start + S);
    CK(cudaEventRecord(ctx->evH2D[slot], Cs));
    CK(cudaStreamWaitEvent(A, ctx->evH2D[slot], 0));
    const float2* iq = reinterpret_cast<const float2*>(ctx->d_stage2[slot].get());
    if (fmt != DABB_IQ_CF32) {
        if ((rc = convert_to_stage(ctx, ctx->d_stage2[slot], io->buf_len, fmt, io->buf_len))) return rc;
        CK(cudaEventRecord(ctx->evStageFree[slot], A)); ctx->stageFreeValid[slot] = true;       // the raw bytes are consumed
        iq = ctx->d_iq_stage;
    }
    if ((rc = enqueue_step(ctx, io, iq, io->buf_len))) return rc;
    if (fmt == DABB_IQ_CF32) { CK(cudaEventRecord(ctx->evStageFree[slot], A)); ctx->stageFreeValid[slot] = true; }   // lane A has read the samples
    if ((rc = enqueue_readback(ctx, p, o))) return rc;
    ctx->pend_count++; ctx->submits++;
    return DABB_OK;
}

int dabb_collect(dabb_ctx* ctx)
{
    if (!ctx) return DABB_E_ARG;
    if (ctx->pend_count == 0) { ctx->err = "nothing outstanding"; return DABB_E_STATE; }
    cudaSetDevice(ctx->device);
    int rc;
    if ((rc = deliver(ctx, ctx->pend[ctx->pend_head]))) return rc;
    ctx->pend_head ^= 1; ctx->pend_count--;
    return DABB_OK;
}

int dabb_profile(dabb_ctx* ctx, int32_t enable)
{
    if (!ctx) return DABB_E_ARG;
    cudaSetDevice(ctx->device);
    if (!enable && ctx->prof) prof_collect(ctx);
    if (enable && !ctx->prof) { ctx->prof_acc.clear(); ctx->prof_used = 0; }
    ctx->prof = enable != 0;
    return 0;
}

int dabb_profile_read(dabb_ctx* ctx, char* out, size_t cap)
{
    if (!ctx || !out || cap < 3) return DABB_E_ARG;
    cudaSetDevice(ctx->device);
    prof_collect(ctx);
    std::string j = "{";
    for (size_t i = 0; i < ctx->prof_acc.size(); i++) {
        char b[256];
        snprintf(b, sizeof b, "%s\"%s\": {\"ms\": %.6f, \"n\": %ld}", i ? ", " : "", ctx->prof_acc[i].first.c_str(), ctx->prof_acc[i].second.first, ctx->prof_acc[i].second.second);
        j += b;
    }
    j += "}";
    if (j.size() + 1 > cap) return DABB_E_ARG;
    memcpy(out, j.c_str(), j.size() + 1);
    return 0;
}

int dabb_read_tap(dabb_ctx* ctx, int32_t what, void* host_out, size_t bytes)
{
    if (!ctx || !host_out) return DABB_E_ARG;
    cudaSetDevice(ctx->device);
    sync_all(ctx);
    if (what == 0 && ctx->soft_partial) {
        // the last step demapped only the symbols its decoders read: repeat its OFDM launch over every symbol, from the same input and
        // per-frame parameters, writing nothing but the softbits (the symbols it did demap get the same bytes again)
        OfdmParams op = ctx->soft_op;
        op.symmask = nullptr; op.r1 = nullptr; op.r1_row = nullptr; op.r1_lmask = nullptr; op.freqcorr = nullptr; op.level = nullptr; op.snr = nullptr; op.trace = TraceBuf{nullptr, nullptr, 0};
        // a step that combined: the grouped streams' r1 of every symbol into a temporary, then the combination over every symbol, with
        // tables built from the leader table that step ran with (each member holds 75 rows, in group order)
        const bool comb = ctx->comb_op.n_items > 0;
        const Grouping gr = comb ? group_streams(*ctx->comb_leader, all_symbols) : Grouping{};
        DevBuf<CombGroup> groups; DevBuf<int32_t> rows; DevBuf<float2> full;
        if (comb) {
            int rc;
            if ((rc = upload(ctx, groups, gr.groups)) || (rc = upload(ctx, rows, gr.row)) || (rc = alloc(ctx, full, (size_t)gr.rows * KC))) return rc;
            op.r1 = full; op.r1_row = rows;
        }
        launch_ofdm_demod(ctx->dev, op, ctx->fft_mode, ctx->stream);
        CK(cudaGetLastError());
        if (comb) {
            CombParams cp = ctx->comb_op; cp.groups = groups; cp.items = nullptr; cp.n_items = (int)gr.groups.size() * 75; cp.r1 = full;
            launch_combine(cp, ctx->stream);
            CK(cudaGetLastError());
        }
        CK(cudaStreamSynchronize(ctx->stream));
        ctx->soft_partial = false;
    }
    if (what == 0) { const size_t n = (size_t)ctx->S * DABB_SOFT_PER_FRAME; CK(cudaMemcpy(host_out, ctx->d_soft + (size_t)ctx->last_parity * n, bytes < n ? bytes : n, cudaMemcpyDeviceToHost)); return 0; }
    if (what == 1 && ctx->d_cir) { const size_t n = (size_t)ctx->S * TU * 4; CK(cudaMemcpy(host_out, ctx->d_cir, bytes < n ? bytes : n, cudaMemcpyDeviceToHost)); return 0; }
    if (what == 2 && ctx->d_r1) {      // every 96th logical carrier of every data symbol (constellationDecimation, ofdm-decoder.h:87)
        const size_t n = (size_t)ctx->S * 75 * 16;
        if (bytes < n * 8) { ctx->err = "constellation tap needs n_streams * 1200 * 8 bytes"; return DABB_E_ARG; }
        CK(cudaMemcpy2D(host_out, 8, ctx->d_r1, 96 * 8, 8, n, cudaMemcpyDeviceToHost));
        return 0;
    }
    if (what == 9) return read_records(ctx, ctx->tii, "tap 9 needs dabb_options.decode_tii to have been set", host_out, bytes);
    if (what == 10) return read_records(ctx, ctx->ber, "tap 10 needs dabb_options.count_bit_errors to have been set", host_out, bytes);
    if (what == 11) return read_records(ctx, ctx->clock, "tap 11 needs dabb_options.sample_clock to have been set", host_out, bytes);
    if (what == 12) return read_records(ctx, ctx->comb, "tap 12 needs dabb_set_combining to have formed a group", host_out, bytes);
    if (what == 14) return read_records(ctx, ctx->mer, "tap 14 needs dabb_set_mer to have been called with enable = 1", host_out, bytes);
    if (what == 13) {
        std::vector<dabb_acq_result> r(ctx->S); std::vector<int32_t> exc(ctx->S);
        int rc;
        if ((rc = read_records(ctx, ctx->acq, "tap 13 needs dabb_options.acquisition to have been set to DABB_ACQ_ROBUST", r.data(), sizeof(dabb_acq_result) * ctx->S))) return rc;
        CK(cudaMemcpy(exc.data(), ctx->acq->exc, sizeof(int32_t) * ctx->S, cudaMemcpyDeviceToHost));
        for (int s = 0; s < ctx->S; s++) r[s].excised = exc[s];
        const size_t n = sizeof(dabb_acq_result) * ctx->S; memcpy(host_out, r.data(), bytes < n ? bytes : n); return 0;
    }
    if (what == 4 && ctx->d_null && ctx->decode_tii) { const size_t n = (size_t)ctx->S * 2 * TU * 8; CK(cudaMemcpy(host_out, ctx->tii->spectra, bytes < n ? bytes : n, cudaMemcpyDeviceToHost)); return 0; }
    if (what == 3 && ctx->d_null) { const size_t n = (size_t)ctx->S * TNULL * 8; CK(cudaMemcpy(host_out, ctx->d_null, bytes < n ? bytes : n, cudaMemcpyDeviceToHost)); return 0; }
    if (what == 5) { const size_t n = sizeof(dabb_frame_result) * ctx->S; CK(cudaMemcpy(host_out, ctx->d_results, bytes < n ? bytes : n, cudaMemcpyDeviceToHost)); return 0; }
    if (what == 6) { const size_t n = (size_t)ctx->S * 12 * 32; CK(cudaMemcpy(host_out, ctx->d_fibs, bytes < n ? bytes : n, cudaMemcpyDeviceToHost)); return 0; }
    if (what == 7 || what == 8) {      // the layouts of dabb_io.msc / dabb_io.sf, the stride implied by `bytes`
        const int64_t per = (int64_t)ctx->S * DABB_MAX_SUBCH * (what == 7 ? 4 : 1), stride = (int64_t)(bytes / (size_t)per);
        uint8_t* out = (uint8_t*)host_out;
        const StepOut o = what == 7 ? StepOut{nullptr, nullptr, out, stride, nullptr, 0} : StepOut{nullptr, nullptr, nullptr, 0, out, stride};
        int rc;
        if ((rc = check_strides(ctx, o)) || (rc = prepare_pending(ctx, ctx->pend_sync)) || (rc = enqueue_readback(ctx, ctx->pend_sync, o))) return rc;
        return deliver(ctx, ctx->pend_sync);
    }
    ctx->err = "tap not available (keep_taps = 0?)";
    return DABB_E_STATE;
}

// ------------------------------------------------------------------------------------------------ stage-level API
int dabb_ofdm_demod(dabb_ctx* ctx, const float* iq, int64_t stride, const int64_t* prs_start, int32_t n, const int32_t* nco, int8_t* soft, float* r1, float* fc)
{
    return dabb_ofdm_demod_ex(ctx, iq, stride, prs_start, n, nco, nullptr, soft, r1, fc);
}

int dabb_ofdm_demod_ex(dabb_ctx* ctx, const float* iq, int64_t stride, const int64_t* prs_start, int32_t n, const int32_t* nco, const float* clock_ppm,
                       int8_t* soft, float* r1, float* fc)
{
    if (!ctx || !iq || !prs_start || !soft || n < 1) return DABB_E_ARG;
    cudaSetDevice(ctx->device);
    sync_all(ctx);
    OfdmParams op{}; op.iq = reinterpret_cast<const float2*>(iq); op.stride = stride; op.prs_start = prs_start; op.active = nullptr; op.soft = soft; op.soft_stride = DABB_SOFT_PER_FRAME;
    op.r1 = reinterpret_cast<float2*>(r1); op.freqcorr = reinterpret_cast<float2*>(fc); op.snr = nullptr; op.n_frames = n;
    op.groups = (fc || n >= 1024) ? 1 : (n >= 64 ? 5 : 25); op.sym_per_cta = 75 / op.groups; op.n_full = n; op.tail_groups = 1; op.fc_pitch = op.groups; op.nco_fast = ctx->nco_fast; op.weighted = ctx->soft_demap == DABB_DEMAP_WEIGHTED;
    op.clock = clock_ppm;
    DevBuf<int32_t> nco4;
    int rc;
    if (nco) {
        // expand {lp applied to PRS sample 0, Hz} to the 4-entry form of the pipeline (same increment for PRS and symbols)
        std::vector<int32_t> h(2 * (size_t)n), h4(4 * (size_t)n);
        CK(cudaMemcpy(h.data(), nco, sizeof(int32_t) * 2 * n, cudaMemcpyDeviceToHost));
        for (int i = 0; i < n; i++) { h4[4 * i] = h[2 * i]; h4[4 * i + 1] = h[2 * i + 1]; h4[4 * i + 2] = h[2 * i]; h4[4 * i + 3] = h[2 * i + 1]; }
        if ((rc = dalloc(ctx, nco4, 4 * (size_t)n, false))) return rc;
        CK(cudaMemcpy(nco4, h4.data(), sizeof(int32_t) * 4 * n, cudaMemcpyHostToDevice));
        op.nco = nco4;
    }
    launch_ofdm_demod(ctx->dev, op, ctx->fft_mode, ctx->stream);
    rc = check_launch(ctx, "ofdm_demod_kernel");
    if (nco4) cudaStreamSynchronize(ctx->stream);
    return rc;
}

int dabb_find_index_ex(dabb_ctx* ctx, const float* iq, int64_t stride, const int64_t* win_start, int32_t n, int32_t placement, int32_t* index_out, float* cir_out)
{
    if (!ctx || !iq || !win_start || !index_out || n < 1 || placement < 0 || placement > 2) return DABB_E_ARG;
    cudaSetDevice(ctx->device);
    sync_all(ctx);
    SyncParams sp{}; sp.iq = reinterpret_cast<const float2*>(iq); sp.stride = stride; sp.win_start = win_start; sp.nco = nullptr; sp.active = nullptr; sp.index_out = index_out; sp.cir_out = cir_out; sp.n = n; sp.fic_ratio = nullptr; sp.coarse_out = nullptr; sp.placement = placement; sp.freqsync = 0;
    // magnitudes between the transform and the search kernel: the context's buffer when the batch fits, else a temporary
    DevBuf<float> temp;
    int rc;
    if (n > ctx->S && (rc = dalloc(ctx, temp, (size_t)n * TU, false))) return rc;
    sp.cir_work = temp ? temp.get() : ctx->d_cir_work.get();
    launch_find_index(ctx->dev, sp, ctx->stream);
    rc = check_launch(ctx, "find_index_kernel");
    if (temp) cudaStreamSynchronize(ctx->stream);
    return rc;
}

int dabb_find_index(dabb_ctx* ctx, const float* iq, int64_t stride, const int64_t* win_start, int32_t n, int32_t* index_out, float* cir_out)
{
    return dabb_find_index_ex(ctx, iq, stride, win_start, n, DABB_PLACEMENT_THRESHOLD_BEFORE_PEAK, index_out, cir_out);
}

int dabb_coarse_estimate(dabb_ctx* ctx, const float* iq, int64_t stride, const int64_t* prs_start, int32_t n, int32_t method, int32_t* offset_out)
{
    if (!ctx || !iq || !prs_start || !offset_out || n < 1 || method < 0 || method > 2) return DABB_E_ARG;
    cudaSetDevice(ctx->device);
    sync_all(ctx);
    launch_coarse(ctx->dev, reinterpret_cast<const float2*>(iq), stride, prs_start, n, method, offset_out, ctx->stream);
    return check_launch(ctx, "coarse_kernel");
}

int dabb_get_info(dabb_ctx* ctx, int32_t what, int64_t* out)
{
    if (!ctx || !out) return DABB_E_ARG;
    switch (what) {
        case DABB_INFO_OSC_MODE: *out = ctx->dev.osc_mode; return DABB_OK;
        case DABB_INFO_OSC_MISMATCHES: *out = ctx->osc_mismatches; return DABB_OK;
        case DABB_INFO_OSC_PATCHED: *out = ctx->osc_patched; return DABB_OK;
        default: return DABB_E_ARG;
    }
}

int dabb_set_options(dabb_ctx* ctx, const dabb_options* opt)
{
    if (!ctx || !opt || opt->fft_placement < 0 || opt->fft_placement > 2 || opt->freqsync_method < 0 || opt->freqsync_method > 2
        || (opt->soft_demap != DABB_DEMAP_REFERENCE && opt->soft_demap != DABB_DEMAP_WEIGHTED)
        || (opt->sample_clock != DABB_CLOCK_OFF && opt->sample_clock != DABB_CLOCK_TRACK)
        || (opt->acquisition != DABB_ACQ_REFERENCE && opt->acquisition != DABB_ACQ_ROBUST)) return DABB_E_ARG;
    const size_t S = (size_t)ctx->S;
    int rc;
    if ((rc = enable(ctx, opt->decode_tii, ctx->tii, [&](Tii& t) -> int {        // zeroed: no open combinations
            uint16_t rank[2][dabb_tii::N_ERR];
            dabb_tii::build_rank_tables(rank);
            if ((!ctx->d_null && (rc = dalloc(ctx, t.null, S * TNULL))) || (rc = dalloc(ctx, t.spectra, S * 2 * TU)) || (rc = dalloc(ctx, t.hdr, S)) ||
                (rc = dalloc(ctx, t.jobs, S * dabb_tii::MAX_JOBS)) || (rc = dalloc(ctx, t.njobs, S)) || (rc = dalloc(ctx, t.sums, S * dabb_tii::N_SLOTS * dabb_tii::N_ERR)) ||
                (rc = dalloc(ctx, t.rank, 2 * dabb_tii::N_ERR)) || (rc = dalloc(ctx, t.res, S)))
                return rc;
            CK(cudaMemcpyAsync(t.rank, rank, sizeof rank, cudaMemcpyHostToDevice, ctx->stream));
            return DABB_OK;
        })) ||
        (rc = enable(ctx, opt->count_bit_errors, ctx->ber, [&](Ber& b) -> int {        // the puncturing of every profile so far and of the FIC
            if ((rc = dalloc(ctx, b.prof, DABB_MAX_PROFILES + 1)) || (rc = dalloc(ctx, b.res, S))) return rc;
            for (size_t i = 0; i < ctx->profiles.size(); i++) CK(cudaMemcpyAsync(b.prof + i, &ctx->profiles[i].ber, sizeof(dabb_ber::Profile), cudaMemcpyHostToDevice, ctx->stream));
            dabb_ber::Profile fic{}; const int fic_L[2] = {21, 3}, fic_PI[2] = {16, 15};
            build_ber_profile(*ctx->host, 2, fic_L, fic_PI, 768, fic); fic.prbs = ctx->d_fic_prbs_words;
            CK(cudaMemcpyAsync(b.prof + DABB_MAX_PROFILES, &fic, sizeof fic, cudaMemcpyHostToDevice, ctx->stream));
            return DABB_OK;
        })) ||
        (rc = enable(ctx, opt->sample_clock == DABB_CLOCK_TRACK, ctx->clock, [&](Clock& c) { return (rc = dalloc(ctx, c.frame, 2 * S)) ? rc : dalloc(ctx, c.res, S); })) ||
        (rc = enable(ctx, opt->acquisition == DABB_ACQ_ROBUST, ctx->acq, [&](Acq& a) -> int {
            float cos_tab[dabb_acq::BLK];
            dabb_acq::make_cos_table(cos_tab);
            if ((rc = dalloc(ctx, a.cos, dabb_acq::BLK)) || (rc = dalloc(ctx, a.job, S)) || (rc = dalloc(ctx, a.level, S * dabb_acq::NB_MAX)) ||
                (rc = dalloc(ctx, a.l1, S * dabb_acq::NB_MAX)) || (rc = dalloc(ctx, a.exc, S)) || (rc = dalloc(ctx, a.res, S)))
                return rc;
            CK(cudaMemcpyAsync(a.cos, cos_tab, sizeof cos_tab, cudaMemcpyHostToDevice, ctx->stream));
            return DABB_OK;
        })))
        return rc;
    ctx->disable_coarse = opt->disable_coarse != 0; ctx->placement = opt->fft_placement; ctx->freqsync = opt->freqsync_method; ctx->decode_tii = opt->decode_tii != 0;
    ctx->count_ber = opt->count_bit_errors != 0; ctx->soft_demap = opt->soft_demap; ctx->sample_clock = opt->sample_clock;
    ctx->acquisition = opt->acquisition;
    return DABB_OK;
}

int dabb_set_mer(dabb_ctx* ctx, int32_t on)
{
    if (!ctx) return DABB_E_ARG;
    int rc;
    if ((rc = enable(ctx, on != 0, ctx->mer, [&](Mer& m) -> int {        // each logical carrier's group
            uint8_t g[KC];
            for (int i = 0; i < KC; i++) g[i] = (uint8_t)dabb_mer::group_of(ctx->host->perm[i]);
            if ((rc = dalloc(ctx, m.group, KC, false)) || (rc = dalloc(ctx, m.res, (size_t)ctx->S))) return rc;
            CK(cudaMemcpyAsync(m.group, g, sizeof g, cudaMemcpyHostToDevice, ctx->stream));
            return DABB_OK;
        })))
        return rc;
    ctx->measure_mer = on != 0;
    return DABB_OK;
}

// stage-level helper: the decoder kernel on n codewords of `frag` punctured softbits each (device, any alignment / values): the input
// is copied into a padded 16-byte pitched buffer with -128 mapped to -127 (same symbol after the reference's clamp)
static int run_stage_viterbi(dabb_ctx* ctx, const int8_t* soft, int n_cw, int64_t in_stride, int frag, const int16_t* map, int nsteps, int nbits,
                             const uint32_t* d_prbs_words, uint8_t* out, int64_t out_stride)
{
    std::vector<uint2> steps; std::vector<uint32_t> soff;
    build_vit_tables_u2(map, nsteps, steps, soff);
    if ((int)soff.back() > frag) { ctx->err = "de-puncturing map consumes more softbits than provided"; return DABB_E_ARG; }
    const int pitch = (frag + 15) & ~15;
    DevBuf<uint2> d_steps; DevBuf<uint32_t> d_soff; DevBuf<int8_t> tmp;
    int rc;
    if ((rc = dalloc(ctx, d_steps, steps.size(), false)) || (rc = dalloc(ctx, d_soff, soff.size(), false)) || (rc = dalloc(ctx, tmp, (size_t)n_cw * pitch + VIT_FRAG_SLACK, false))) return rc;
    CK(cudaMemcpyAsync(d_steps, steps.data(), steps.size() * sizeof(uint2), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(d_soff, soff.data(), soff.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemsetAsync(tmp, 0, (size_t)n_cw * pitch + VIT_FRAG_SLACK, ctx->stream));
    if (pitch == frag && in_stride == frag) { launch_clamp_copy(soft, tmp, (int64_t)n_cw * frag, ctx->stream); rc = check_launch(ctx, "clamp_copy_kernel"); }
    else {
        CK(cudaMemcpy2DAsync(tmp, pitch, soft, (size_t)in_stride, frag, n_cw, cudaMemcpyDeviceToDevice, ctx->stream));
        launch_clamp_copy(tmp, tmp, (int64_t)n_cw * pitch, ctx->stream); rc = check_launch(ctx, "clamp_copy_kernel");
    }
    if (!rc) rc = grow(ctx, ctx->d_dec, vit_dec_bytes(n_cw, nsteps) / sizeof(uint2));
    if (!rc) {
        ViterbiParams vp{}; vp.frag = tmp; vp.cw_div = 1; vp.outer_stride = pitch; vp.inner_stride = 0; vp.steptab = d_steps; vp.stage_off = d_soff;
        vp.n_cw = n_cw; vp.nsteps = nsteps; vp.nbits = nbits; vp.dec = ctx->d_dec; vp.out = out; vp.out_stride = out_stride; vp.prbs_words = d_prbs_words; vp.valid = nullptr;
        launch_viterbi(vp, ctx->stream);
        rc = check_launch(ctx, "viterbi_kernel");
    }
    cudaStreamSynchronize(ctx->stream);
    return rc;
}

int dabb_viterbi(dabb_ctx* ctx, const int8_t* soft, int32_t n_cw, int32_t nbits, uint8_t* bits_out)
{
    if (!ctx || !soft || !bits_out || n_cw < 1 || nbits < 32 || (nbits % 32) || ((nbits + 6) % 6)) return DABB_E_ARG;
    cudaSetDevice(ctx->device);
    sync_all(ctx);
    const int nsteps = nbits + 6, ob = nbits / 8;
    DevBuf<uint8_t> bytes;
    int rc;
    if ((rc = dalloc(ctx, bytes, (size_t)n_cw * ob, false))) return rc;
    std::vector<int16_t> map((size_t)nsteps * 4);
    std::fill(map.begin(), map.end(), (int16_t)0);                      // >= 0 = present: nothing punctured, the caller's zeros are softbit 0
    rc = run_stage_viterbi(ctx, soft, n_cw, (int64_t)nsteps * 4, nsteps * 4, map.data(), nsteps, nbits, nullptr, bytes, ob);
    if (!rc) { launch_unpack_bits(bytes, ob, n_cw, nbits, bits_out, ctx->stream); rc = check_launch(ctx, "unpack_bits_kernel"); }
    cudaStreamSynchronize(ctx->stream);
    return rc;
}

int dabb_fic_decode(dabb_ctx* ctx, const int8_t* soft, int32_t n_frames, uint8_t* fib_out, int32_t* crc_mask_out)
{
    if (!ctx || !soft || !fib_out || !crc_mask_out || n_frames < 1) return DABB_E_ARG;
    cudaSetDevice(ctx->device);
    sync_all(ctx);
    // codeword (f, b) = softbits [9216 f + 2304 b, +2304)
    int rc = run_stage_viterbi(ctx, soft, n_frames * 4, 2304, 2304, ctx->host->fic_map, 774, 768, ctx->d_fic_prbs_words, fib_out, 96);
    if (!rc) { launch_fic_crc(fib_out, nullptr, n_frames, crc_mask_out, ctx->stream); rc = check_launch(ctx, "fic_crc_kernel"); }
    cudaStreamSynchronize(ctx->stream);
    return rc;
}

int dabb_msc_decode(dabb_ctx* ctx, const dabb_subchannel* sc, const int8_t* soft, int32_t n, uint8_t* bytes_out)
{
    if (!ctx || !sc || !soft || !bytes_out || n < 1) return DABB_E_ARG;
    cudaSetDevice(ctx->device);
    sync_all(ctx);
    ProtProfile prof;
    if (make_prot_profile(sc->bitrate, sc->short_form, sc->uep_level, sc->eep_profile_a, sc->eep_level, prof) < 0) { ctx->err = "unsupported protection profile"; return DABB_E_UNSUPPORTED; }
    const int frag = sc->length_cu * 64, nbits = 24 * prof.bitrate, nsteps = nbits + 6, flen = 3 * prof.bitrate;
    if (prof.in_bits > frag) { ctx->err = "protection profile needs more bits than the sub-channel holds"; return DABB_E_ARG; }
    std::vector<int16_t> map((size_t)nsteps * 4);
    build_msc_map(*ctx->host, prof, map.data());
    std::vector<uint32_t> w((size_t)(nbits + 31) / 32); build_prbs_words(nbits, w.data());
    DevBuf<uint32_t> d_w;
    int rc;
    if ((rc = dalloc(ctx, d_w, w.size(), false))) return rc;
    CK(cudaMemcpy(d_w, w.data(), w.size() * 4, cudaMemcpyHostToDevice));
    // output rows are 3*bitrate bytes (a multiple of 4)
    rc = run_stage_viterbi(ctx, soft, n, frag, frag, map.data(), nsteps, nbits, d_w, bytes_out, flen);
    cudaStreamSynchronize(ctx->stream);
    return rc;
}

int dabb_rs_superframes(dabb_ctx* ctx, uint8_t* sf, int32_t n, int32_t sf_len, int32_t* info)
{
    if (!ctx || !sf || !info || n < 1 || sf_len < 120 || (sf_len % 120)) return DABB_E_ARG;
    if (sf_len / 120 > 64) { ctx->err = "superframes above 512 kbit/s (64 interleaved codewords) are not supported"; return DABB_E_UNSUPPORTED; }
    cudaSetDevice(ctx->device);
    sync_all(ctx);
    launch_rs_superframes(sf, n, sf_len, info, ctx->dev.gf_exp, ctx->dev.gf_log, ctx->stream);
    return check_launch(ctx, "rs_superframes_kernel");
}

int dabb_dev_alloc(dabb_ctx* ctx, size_t bytes, void** out) { if (!ctx || !out) return DABB_E_ARG; cudaSetDevice(ctx->device); CK(cudaMalloc(out, bytes)); return 0; }
int dabb_dev_free(dabb_ctx* ctx, void* p) { if (!ctx) return DABB_E_ARG; cudaSetDevice(ctx->device); CK(cudaStreamSynchronize(ctx->stream)); CK(cudaFree(p)); return 0; }
int dabb_memcpy_h2d(dabb_ctx* ctx, void* d, const void* s, size_t n) { if (!ctx) return DABB_E_ARG; cudaSetDevice(ctx->device); CK(cudaMemcpyAsync(d, s, n, cudaMemcpyHostToDevice, ctx->stream)); CK(cudaStreamSynchronize(ctx->stream)); return 0; }
int dabb_memcpy_d2h(dabb_ctx* ctx, void* d, const void* s, size_t n) { if (!ctx) return DABB_E_ARG; cudaSetDevice(ctx->device); CK(cudaStreamSynchronize(ctx->stream)); CK(cudaMemcpy(d, s, n, cudaMemcpyDeviceToHost)); return 0; }

} // extern "C"

// ---------------------------------------------------------------------------------------------------------------
// wideband channelizer (chan.cu, chan_core.cuh): the filter, the channel table and per-call staging, owned by one context

struct dabb_chan {
    dabb_ctx* ctx = nullptr;
    dabb_channel::Geometry g{}; int fmt = 0, n_in = 0, n_ch = 0, block_out = 0; float inv_r = 0.f;
    std::vector<int32_t> input_of;
    DevBuf<dabb_channel::f4> d_taps; DevBuf<int32_t> d_input_of; DevBuf<int64_t> d_fmod;
    DevBuf<int64_t> d_starts;           // per call: out_start [n_ch], then in_start [n_in]
    DevBuf<uint8_t> d_stage;            // host inputs, copied to the device
};

namespace {
constexpr int64_t CHAN_MAX_INDEX = int64_t(1) << 60;      // |in_start| and in_len bounds: index sums stay far from overflow

int chan_range(const dabb_chan* ch, int64_t out_start, int64_t out_len, int64_t& first, int64_t& end)
{
    if (out_start < 0 || out_len < 1 || out_len > dabb_channel::MAX_OUT_INDEX || out_start > dabb_channel::MAX_OUT_INDEX - out_len) return DABB_E_ARG;
    first = dabb_channel::last_input(out_start, ch->g.L, ch->g.M) - ch->g.T + 1;
    end = dabb_channel::last_input(out_start + out_len - 1, ch->g.L, ch->g.M) + 1;
    return DABB_OK;
}
} // namespace

extern "C" {

int dabb_chan_create(dabb_ctx* ctx, const dabb_chan_config* cfg, dabb_chan** out)
{
    if (!ctx || !cfg || !out) return DABB_E_ARG;
    *out = nullptr;
    dabb_channel::Geometry g{};
    if (dabb_channel::geometry(cfg->rate_hz, g) != DABB_OK) {
        ctx->err = "channelizer: rate " + std::to_string(cfg->rate_hz) + " Hz is outside 2048000 .. 64000000 or 2048000 / rate does not reduce to L / M with L <= 1024";
        return DABB_E_UNSUPPORTED;
    }
    const int nc = cfg->n_channels, ni = cfg->n_inputs;
    if (cfg->iq_format < DABB_IQ_CF32 || cfg->iq_format > DABB_IQ_S16BE || ni < 1 || ni > dabb_channel::MAX_CHANNELS || nc < 1 || nc > dabb_channel::MAX_CHANNELS
        || !cfg->input_of_channel || !cfg->offset_hz) { ctx->err = "channelizer: bad format, input count, channel count or NULL channel table"; return DABB_E_ARG; }
    for (int c = 0; c < nc; c++) {
        if (cfg->input_of_channel[c] < 0 || cfg->input_of_channel[c] >= ni) { ctx->err = "channelizer: channel " + std::to_string(c) + " names no input"; return DABB_E_ARG; }
        if (!dabb_channel::offset_ok(g.R, cfg->offset_hz[c])) { ctx->err = "channelizer: offset of channel " + std::to_string(c) + " leaves the input band (|f| + 768000 > R / 2)"; return DABB_E_ARG; }
    }
    cudaSetDevice(ctx->device);
    std::unique_ptr<dabb_chan> ch(new dabb_chan);
    ch->ctx = ctx; ch->g = g; ch->fmt = cfg->iq_format; ch->n_in = ni; ch->n_ch = nc;
    ch->block_out = chan_block_outputs(g.L, g.M, g.TP); ch->inv_r = (float)(1.0 / (double)g.R);
    ch->input_of.assign(cfg->input_of_channel, cfg->input_of_channel + nc);
    std::vector<float> h((size_t)g.L * g.T), packed((size_t)g.L * g.TP);
    dabb_channel::design_taps(g, h.data());
    dabb_channel::pack_taps(g, h.data(), packed.data());
    std::vector<int64_t> fm((size_t)nc);
    for (int c = 0; c < nc; c++) fm[(size_t)c] = dabb_channel::floor_mod(cfg->offset_hz[c], g.R);
    int rc;
    if ((rc = alloc(ctx, ch->d_taps, packed.size() / 4)) || (rc = alloc(ctx, ch->d_input_of, (size_t)nc)) || (rc = alloc(ctx, ch->d_fmod, (size_t)nc))
        || (rc = alloc(ctx, ch->d_starts, (size_t)(nc + ni)))) return rc;
    CK(cudaMemcpy(ch->d_taps, packed.data(), packed.size() * sizeof(float), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(ch->d_input_of, ch->input_of.data(), (size_t)nc * sizeof(int32_t), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(ch->d_fmod, fm.data(), (size_t)nc * sizeof(int64_t), cudaMemcpyHostToDevice));
    *out = ch.release();
    return DABB_OK;
}

void dabb_chan_destroy(dabb_chan* ch)
{
    if (!ch) return;
    cudaSetDevice(ch->ctx->device);
    cudaStreamSynchronize(ch->ctx->stream);
    delete ch;          // frees its device buffers
}

int dabb_chan_input_range(const dabb_chan* ch, int64_t out_start, int64_t out_len, int64_t* in_first, int64_t* in_end)
{
    if (!ch || !in_first || !in_end) return DABB_E_ARG;
    int64_t f, e;
    const int rc = chan_range(ch, out_start, out_len, f, e);
    if (rc) return rc;
    *in_first = f; *in_end = e;
    return DABB_OK;
}

int dabb_channelize(dabb_chan* ch, const dabb_chan_io* io)
{
    if (!ch) return DABB_E_ARG;
    dabb_ctx* ctx = ch->ctx;
    if (!io || !io->in || !io->in_start || !io->out || !io->out_start) { ctx->err = "dabb_channelize: NULL argument"; return DABB_E_ARG; }
    if ((io->in_is_host != 0 && io->in_is_host != 1) || io->in_len < 1 || io->in_len > CHAN_MAX_INDEX || io->in_stride < io->in_len || io->out_len < 1
        || io->out_stride < io->out_len) { ctx->err = "dabb_channelize: bad in_is_host, length or stride"; return DABB_E_ARG; }
    for (int i = 0; i < ch->n_in; i++)
        if (io->in_start[i] < -CHAN_MAX_INDEX || io->in_start[i] > CHAN_MAX_INDEX) { ctx->err = "dabb_channelize: in_start out of range"; return DABB_E_ARG; }
    for (int c = 0; c < ch->n_ch; c++) {
        int64_t f, e;
        const int i = ch->input_of[(size_t)c];
        if (chan_range(ch, io->out_start[c], io->out_len, f, e) || f < io->in_start[i] || e > io->in_start[i] + io->in_len) {
            ctx->err = "dabb_channelize: channel " + std::to_string(c) + " needs input samples its buffer does not hold (see dabb_chan_input_range)";
            return DABB_E_ARG;
        }
    }
    cudaSetDevice(ctx->device);
    cudaStream_t st = ctx->stream;
    const size_t bps = (size_t)bytes_per_sample(ch->fmt);
    std::vector<int64_t> starts((size_t)(ch->n_ch + ch->n_in));
    std::copy(io->out_start, io->out_start + ch->n_ch, starts.begin());
    std::copy(io->in_start, io->in_start + ch->n_in, starts.begin() + ch->n_ch);
    CK(cudaMemcpyAsync(ch->d_starts, starts.data(), starts.size() * sizeof(int64_t), cudaMemcpyHostToDevice, st));
    const uint8_t* in = static_cast<const uint8_t*>(io->in);
    int64_t in_stride = io->in_stride;
    if (io->in_is_host) {
        int rc;
        if ((rc = grow(ctx, ch->d_stage, (size_t)ch->n_in * (size_t)io->in_len * bps))) return rc;
        CK(cudaMemcpy2DAsync(ch->d_stage, (size_t)io->in_len * bps, io->in, (size_t)io->in_stride * bps, (size_t)io->in_len * bps, (size_t)ch->n_in, cudaMemcpyHostToDevice, st));
        in = ch->d_stage; in_stride = io->in_len;
    }
    prof_mark(ctx, "__step_begin");
    ChanParams p{};
    p.in = in; p.in_stride = in_stride; p.fmt = ch->fmt; p.in_start = ch->d_starts + ch->n_ch; p.in_len = io->in_len;
    p.input_of = ch->d_input_of; p.fmod = ch->d_fmod; p.out_start = ch->d_starts;
    p.out_len = io->out_len; p.out = reinterpret_cast<float2*>(io->out); p.out_stride = io->out_stride;
    p.taps = ch->d_taps; p.R = ch->g.R; p.L = ch->g.L; p.M = ch->g.M; p.T = ch->g.T; p.TP = ch->g.TP; p.inv_r = ch->inv_r; p.block_out = ch->block_out;
    CK(launch_chan(p, ch->n_ch, st));
    return check_launch(ctx, "chan_kernel");
}

} // extern "C"

// ---------------------------------------------------------------------------------------------------------------
// spectrum survey (survey.cu, survey_core.cuh) and the candidate detector

extern "C" {

int dabb_survey(dabb_ctx* ctx, const dabb_survey_io* io)
{
    if (!ctx) return DABB_E_ARG;
    if (!io || !io->in || !io->psd) { ctx->err = "dabb_survey: NULL argument"; return DABB_E_ARG; }
    const int log2n = dabb_spectrum::log2_nfft(io->nfft);
    if (log2n < 0) { ctx->err = "dabb_survey: nfft must be a power of two from 1024 to 16384"; return DABB_E_ARG; }
    if ((io->in_is_host != 0 && io->in_is_host != 1) || io->iq_format < DABB_IQ_CF32 || io->iq_format > DABB_IQ_S16BE || io->n_inputs < 1
        || io->n_inputs > dabb_spectrum::MAX_INPUTS || io->in_len < io->nfft || io->in_len > dabb_spectrum::MAX_LEN || io->in_stride < io->in_len) {
        ctx->err = "dabb_survey: bad in_is_host, format, input count, length or stride"; return DABB_E_ARG;
    }
    cudaSetDevice(ctx->device);
    cudaStream_t st = ctx->stream;
    int rc;
    if (!ctx->d_svy_tw) {
        std::vector<dabb_channel::cf> tw(dabb_spectrum::MAX_NFFT / 2); std::vector<float> win(dabb_spectrum::MAX_NFFT);
        dabb_spectrum::make_tables(tw.data(), win.data());
        if ((rc = alloc(ctx, ctx->d_svy_win, win.size())) || (rc = alloc(ctx, ctx->d_svy_tw, tw.size()))) { ctx->d_svy_tw.reset(); return rc; }
        // pageable sources: each copy has read its source when it returns.  d_svy_tw is what marks the tables as present, so a failed
        // copy leaves none
        cudaError_t e = cudaMemcpyAsync(ctx->d_svy_win, win.data(), win.size() * sizeof(float), cudaMemcpyHostToDevice, st);
        if (e == cudaSuccess) e = cudaMemcpyAsync(ctx->d_svy_tw, tw.data(), tw.size() * sizeof(dabb_channel::cf), cudaMemcpyHostToDevice, st);
        if (e != cudaSuccess) { ctx->d_svy_tw.reset(); ctx->d_svy_win.reset(); ctx->err = std::string("dabb_survey: table upload: ") + cudaGetErrorString(e); return DABB_E_CUDA; }
    }
    const int n_in = io->n_inputs, nfft = io->nfft;
    const size_t bps = (size_t)bytes_per_sample(io->iq_format);
    const int64_t S = dabb_spectrum::n_segments(io->in_len, nfft), chunk = dabb_spectrum::chunk_segments(S, n_in), n_chunks = (S + chunk - 1) / chunk;
    const int64_t used = (S + 1) * (nfft / 2);          // the samples the segments read
    const uint8_t* in = static_cast<const uint8_t*>(io->in);
    int64_t in_stride = io->in_stride;
    if (io->in_is_host) {
        if ((rc = grow(ctx, ctx->d_svy_stage, (size_t)n_in * (size_t)used * bps))) return rc;
        CK(cudaMemcpy2DAsync(ctx->d_svy_stage, (size_t)used * bps, io->in, (size_t)io->in_stride * bps, (size_t)used * bps, (size_t)n_in, cudaMemcpyHostToDevice, st));
        in = ctx->d_svy_stage; in_stride = used;
    }
    if ((rc = grow(ctx, ctx->d_svy_part, (size_t)n_in * (size_t)n_chunks * (size_t)nfft)) || (rc = grow(ctx, ctx->d_svy_psd, (size_t)n_in * (size_t)nfft))) return rc;
    prof_mark(ctx, "__step_begin");
    SurveyParams p{};
    p.in = in; p.in_stride = in_stride; p.fmt = io->iq_format; p.S = S; p.chunk = chunk; p.tw = ctx->d_svy_tw; p.win = ctx->d_svy_win; p.part = ctx->d_svy_part;
    CK(launch_survey(p, log2n, n_chunks, n_in, st));
    if ((rc = check_launch(ctx, "survey_kernel"))) return rc;
    launch_survey_sum(ctx->d_svy_part, n_chunks, log2n, n_in, 1.0 / ((double)S * (3.0 * nfft / 8.0)), ctx->d_svy_psd, st);
    if ((rc = check_launch(ctx, "survey_sum_kernel"))) return rc;
    CK(cudaMemcpyAsync(io->psd, ctx->d_svy_psd, (size_t)n_in * (size_t)nfft * sizeof(float), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return DABB_OK;
}

int dabb_survey_candidates(const float* psd, int32_t nfft, int64_t rate_hz, float min_score_db, dabb_survey_candidate* out, int32_t cap, int32_t* n_found)
{
    return dabb_spectrum::candidates(psd, nfft, rate_hz, min_score_db, out, cap, n_found);
}

} // extern "C"
