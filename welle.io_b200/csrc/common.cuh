// common.cuh — shared declarations of the libdab_b200 CUDA sources
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string>
#include "ofdm_core.cuh"
#include "tii_core.cuh"
#include "ber_core.cuh"
#include "chan_core.cuh"
#include "ofdm_mask.cuh"
#include "clock_core.cuh"
#include "combine_core.cuh"
#include "acq_core.cuh"

namespace dabb {

// ---- device tables (built on the host by tables.cpp, uploaded once per context) ----
struct DevTables {
    const float2* tw_fwd;      // TwLayout::TOTAL entries, forward transform
    const float2* tw_inv;      // inverse transform
    const int16_t* invperm;    // [2048] bin -> logical carrier index 0..1535, -1 for unused bins (freq-interleaver.cpp:35-91);
                               // [2048 + bin] its index in ofdm_demod_kernel's softbit staging area, [4096 + c] the slot of logical chunk c there
    const float2* prs_ref;     // [2048] PhaseReference::refTable (phasereference.cpp:45-51)
    const float2* osc;         // [2 048 000] oscillator table (ofdm-processor.cpp:92-94)
    // the same values computed on the fly (osc_mode = 1): osc[m] == float(H[m >> 10] * exp(j theta (m & 1023))) in double, the small
    // rotation from its Taylor polynomial; verified for all 2 048 000 m at context creation (else osc_mode stays 0)
    const double2* osc_hi;     // [2000] exp(j 2 pi 1024 a / 2 048 000), correctly rounded doubles - except at the quarter turns, where
                               // the reference's own double angle is an ulp off and the factor is the table value itself
    double osc_theta;          // 2 pi / 2 048 000, correctly rounded
    int32_t osc_mode;          // 0: table lookups (a scattered 8-byte gather per sample), 1: on the fly
    const int16_t* fic_map;    // [3096] mother-code position -> index into the 2304 punctured softbits or -1
    const uint8_t* gf_exp;     // [512]
    const uint8_t* gf_log;     // [256]
};

// ---- optional CTA timeline (environment DABB_TRACE=<file>): every CTA of the two hot kernels records {kind, SM, start, end} (global
// nanosecond timer) so that the overlap of the two lanes can be drawn; off (nullptr) in normal operation
struct TraceBuf { unsigned long long* rec; unsigned int* count; unsigned int cap; };
#if defined(__CUDACC__)
__device__ __forceinline__ unsigned long long trace_now() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
__device__ __forceinline__ unsigned int trace_smid() { unsigned int s; asm volatile("mov.u32 %0, %%smid;" : "=r"(s)); return s; }
__device__ __forceinline__ void trace_put(const TraceBuf& tb, unsigned int kind, unsigned long long t0)
{
    const unsigned int i = atomicAdd(tb.count, 1u);
    if (i < tb.cap) { tb.rec[3 * i] = ((unsigned long long)kind << 32) | trace_smid(); tb.rec[3 * i + 1] = t0; tb.rec[3 * i + 2] = trace_now(); }
}
#endif

// ---- OFDM demod launch parameters ----
struct OfdmParams {
    const float2* iq; int64_t stride;            // complex samples
    const int64_t* prs_start;                    // [n] first useful PRS sample, relative to iq + f*stride
    const int32_t* nco;                          // [n][4] or nullptr: {phase applied to PRS sample 0, Hz (PRS), phase extrapolated to index 0 for the data symbols, Hz}
    const int32_t* active;                       // [n] or nullptr: 0 = skip frame
    int8_t* soft; int64_t soft_stride;           // per frame stride in bytes (>= 75*3072)
    float2* r1;                                  // optional tap [n][75][1536]
    float2* freqcorr;                            // optional [n][fc_pitch] partial CP correlation sums
    float* level;                                // optional [n][fc_pitch] partial signal-level estimates (see advance_kernel in api.cu)
    int32_t* snr;                                // optional [n] get_snr value of the PRS
    int n_frames; int groups; int sym_per_cta;   // groups * sym_per_cta == 75
    int n_full; int tail_groups;                 // frames >= n_full are cut into tail_groups CTAs each (tail_groups divides 75; 1 / 0 = off)
    int fc_pitch;                                // freqcorr entries per frame (>= groups, tail_groups); 0 -> the larger of the two
    int nco_fast;                                // DABB_NCO_FAST: fp32 oscillator (tolerance mode)
    int weighted;                                // DABB_DEMAP_WEIGHTED: softbits against max(carrier level, the symbol's geometric-mean level)
    const uint32_t* symmask;                     // [n][OFDM_MASK_WORDS] the symbols each frame demaps (ofdm_mask.cuh), or nullptr: all of them
    TraceBuf trace;                              // rec == nullptr: off
    const float* clock;                          // [n] sample-clock ppm whose phase ramp the demap removes (clock_core.cuh), or nullptr: none
    // where the TAP instances store r1 (see r1_dst in ofdm.cu): nullptr = the constellation tap's layout [n][75][1536]; else a row index per
    // frame (< 0: none) and optionally [n][OFDM_MASK_WORDS] the symbols that get a row (diversity combining, combine.cu)
    const int32_t* r1_row;
    const uint32_t* r1_lmask;
};

struct SyncParams {
    const float2* iq; int64_t stride;
    const int64_t* win_start;                    // [n]
    const int32_t* nco;                          // [n][2] or nullptr
    const int32_t* active;
    int32_t* index_out; float* cir_out; int n;
    float* cir_work;                             // [n][T_u] magnitudes between the transform kernel and the search kernel
    // coarse frequency corrector (OFDMProcessor::processPRS, PatternOfZeros): evaluated for streams whose FIC success
    // counter is below 5 (ofdm-processor.cpp:397); result = carrier offset, or 100 when not evaluated / no estimate
    const int32_t* fic_ratio; int32_t* coarse_out;
    int placement;      // DABB_PLACEMENT_*: 0 ThresholdBeforePeak, 1 StrongestPeak, 2 EarliestPeakWithBinning
    int freqsync;       // DABB_FREQSYNC_*: 0 PatternOfZeros, 1 GetMiddle, 2 CorrelatePRS
};

void launch_ofdm_demod(const DevTables& tb, const OfdmParams& p, int fft_mode, cudaStream_t st);
int ofdm_tail_frames(int n_frames);
constexpr int OFDM_TAIL_GROUPS = 5;              // CTAs per tail frame (15 data symbols each): the best of 5 / 15 / 25 before the port to H100
void launch_find_index(const DevTables& tb, const SyncParams& p, cudaStream_t st, int part = -1, int32_t* excised = nullptr);
void launch_tii_spectra(const DevTables& tb, const float2* iq, int64_t stride, const int64_t* prs_start, const int32_t* nco_frame, const int32_t* active,
                        const float2* nulls, float2* out, int n, cudaStream_t st);
void launch_coarse(const DevTables& tb, const float2* iq, int64_t stride, const int64_t* prs_start, int n, int freqsync, int32_t* out, cudaStream_t st);

// ---- diversity combining (combine.cu, combine_core.cuh) ----
// one group of streams of a context (dabb_set_combining): members in ascending stream order, the leader at lpos; member i's r1 of the
// leader's j-th combined symbol is row row[i] + j of CombParams::r1
struct CombGroup {
    int32_t n, lpos;
    int32_t stream[dabb_comb::MAX_BRANCHES];
    int32_t row[dabb_comb::MAX_BRANCHES];
};
// one CTA of combine_kernel: data symbol sym (1..75) of a group, in column col of the members' rows; `first`: the group's first item,
// which writes the leader's tap-12 record
struct CombItem { int32_t group, sym, col, first; };
struct CombParams {
    const CombGroup* groups;
    const CombItem* items; int n_items;          // items == nullptr: every symbol of every group, item i = (i / 75, i % 75 + 1, i % 75)
    const float2* r1;                            // rows of KC products (logical carrier order)
    const int32_t* active;                       // [S] the step decoded a frame
    const int64_t* prs; const int64_t* buf_start;   // [S] the phase reference symbol, relative to the buffer; the buffer's first sample
    void* res;                                   // [S] dabb_combine_result (tap 12): noise in, members and mask out
    int8_t* soft; int64_t soft_stride;           // the step's softbits: the leaders' rows are overwritten
    int weighted;                                // DABB_DEMAP_WEIGHTED
};
void launch_combine(const CombParams& p, cudaStream_t st);

// ---- modulation error ratio (mer.cu, mer_core.cuh) ----
struct MerParams {
    const int8_t* soft; int64_t soft_stride;     // the step's softbits (the FIC decoder's input)
    const int32_t* active;                       // [S] the step decoded a frame
    const uint8_t* group;                        // [1536] each logical carrier's group (dabb_mer::group_of of its physical carrier)
    void* res;                                   // [S] dabb_mer_result (tap 14)
    int n_streams;
};
void launch_mer(const MerParams& p, cudaStream_t st);

// ---- TII analysis (tii.cu, tii_core.cuh) ----
struct TiiParams {
    const float2* spectra;                       // [n][2][T_u] from tii_spectra_kernel: phase reference symbol, null symbol
    const int32_t* active;                       // [n] 1 = the stream decoded a frame in this step
    dabb_tii::StreamHdr* hdr;                    // [n] open combinations
    dabb_tii::Job* jobs; int32_t* njobs;         // [n][MAX_JOBS], [n]: this step's analyses (tii_plan_kernel -> tii_phase_kernel)
    uint32_t* sums;                              // [n][N_SLOTS][N_ERR] accumulated phase errors
    const uint16_t* rank;                        // [2][N_ERR] arg-min tie order (dabb_tii::build_rank_tables)
    void* res;                                   // [n] dabb_tii_result
    int n;
};
void launch_tii_plan(const TiiParams& p, cudaStream_t st);
void launch_tii_phase(const TiiParams& p, cudaStream_t st);

// ---- wideband channelizer (chan.cu, chan_core.cuh) ----
constexpr int CHAN_THREADS = 256;
struct ChanParams {
    const uint8_t* in; int64_t in_stride; int fmt; // input i at in + i * in_stride samples of format fmt (DABB_IQ_*)
    const int64_t* in_start; int64_t in_len;     // [n_inputs] absolute index of each buffer's first sample; samples per buffer
    const int32_t* input_of;                     // [n_channels] input of each channel
    const int64_t* fmod;                         // [n_channels] offset_hz mod R
    const int64_t* out_start;                    // [n_channels] absolute output index of each row's first sample
    int64_t out_len; float2* out; int64_t out_stride;
    const dabb_channel::f4* taps;                   // [TP / 4][L] (dabb_channel::pack_taps)
    int64_t R; int L, M, T, TP; float inv_r;     // inv_r = 1 / R rounded to float
    int block_out;                               // outputs per CTA (chan_block_outputs)
};
// outputs per CTA: 4, 2 or 1 per thread, the most whose input span fits 64 KB of shared memory
int chan_block_outputs(int L, int M, int TP);
// input samples a CTA of block_out outputs stages, at most
int64_t chan_span_cap(int block_out, int L, int M, int TP);
cudaError_t launch_chan(const ChanParams& p, int n_channels, cudaStream_t st);

// ---- spectrum survey (survey.cu, survey_core.cuh) ----
constexpr int SURVEY_THREADS = 512;
struct SurveyParams {
    const uint8_t* in; int64_t in_stride; int fmt;  // input i at in + i * in_stride samples of format fmt (DABB_IQ_*)
    int64_t S, chunk;                            // segments per input, segments per CTA (the last CTA of an input may have fewer)
    const dabb_channel::cf* tw; const float* win;   // dabb_spectrum::make_tables
    float* part;                                 // [n_inputs][n_chunks][nfft] per-chunk sums, storage order
};
cudaError_t launch_survey(const SurveyParams& p, int log2n, int64_t n_chunks, int n_inputs, cudaStream_t st);
// psd[i][j] = scale * sum over the chunks of input i of part at bin j (double, ascending chunk order)
void launch_survey_sum(const float* part, int64_t n_chunks, int log2n, int n_inputs, double scale, float* psd, cudaStream_t st);

// ---- robust acquisition (acq.cu, acq_core.cuh): the span one searching stream analyses in a step (acq_plan_kernel in api.cu) ----
struct AcqJob {
    int64_t rel;            // the search start (the stream's position) relative to its buffer
    int32_t nb;             // blocks of 256 samples analysed (0: the stream does not search in this step)
    int32_t lp, phase;      // NCO: sample i of the span is mixed with osc[(lp - (i + 1) phase) mod 2 048 000]; none when both are 0
    int32_t pad;
};
// levels [S][NB_MAX] and envelope sums [S][NB_MAX] of every analysed block; cos_tab: dabb_acq::make_cos_table
void launch_acq_levels(const AcqJob* job, const float2* iq, int64_t stride, const float2* osc, const float* cos_tab, int S,
                       float* level, float* l1sum, cudaStream_t st);

// ---- host-side table builders (tables.cpp) ----
struct HostTables {
    float2 tw_fwd[TwLayout::TOTAL], tw_inv[TwLayout::TOTAL];
    int16_t perm[KC]; int16_t invperm[TU + TU + 192];   // [0, T_u) bin -> logical carrier; [T_u, 2 T_u) bin -> softbit staging index; then the staging slot of each 16-byte chunk
    float2 prs_ref[TU];
    int16_t fic_map[3096];
    uint8_t gf_exp[512], gf_log[256];
    int8_t pcodes[24][32];
};
void build_host_tables(HostTables& t);
void build_osc_table(float2* osc /* INPUT_RATE entries */);
void build_osc_factors(const float2* osc_table, double2* hi /* 2000 */, double* theta, int* patched);
// compares the on-the-fly oscillator with the table for every index on the device; returns the number of differing entries
int launch_osc_verify(const DevTables& tb, cudaStream_t st);

// protection profile -> (L, PI) blocks; returns punctured length or -1
struct ProtProfile { int bitrate; int nblk; int L[4]; int PI[4]; int in_bits; };
int make_prot_profile(int bitrate, int short_form, int uep_level, int eep_profile_a, int eep_level, ProtProfile& out);
// mother-code map: for each of 4*(24*bitrate+6) positions the index into the punctured input (saturating at 32767) or -1
void build_msc_map(const HostTables& t, const ProtProfile& p, int16_t* map);
// energy-dispersal words of an nbits-bit block ((nbits + 31) / 32 of them), packed like the decoder output
void build_prbs_words(int nbits, uint32_t* w);
// the puncturing of nbits-bit codewords with blocks (L[k], PI[k]) and the tail, as the bit-error count reads it (ber_core.cuh); the
// dispersal words (Profile::prbs) are the caller's
void build_ber_profile(const HostTables& t, int nblk, const int* L, const int* PI, int nbits, dabb_ber::Profile& out);

} // namespace dabb
