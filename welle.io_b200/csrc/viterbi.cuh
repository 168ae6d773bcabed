// viterbi.cuh — parameter blocks and launchers of viterbi.cu / rs.cu
#pragma once
#include "common.cuh"
#include "vit_groups.cuh"
#include <vector>

namespace dabb {

constexpr int MSC_RING = 20;          // CIF slices kept per selected sub-channel: 16 (de-interleaver depth) + 4 (one frame)

// per (stream, slot) sub-channel state, device resident
struct MscSlotState {
    int32_t enabled;
    int32_t start_cu, frag;           // frag = length_cu * 64 softbits per CIF
    int32_t bitrate, dabplus;
    int32_t profile;                  // index into the context's protection-profile table
    int64_t cif_count;                // CIFs collected since selection (DabAudio::countforInterleaver, dab-audio.cpp:146)
    // superframe filter (SuperframeFilter, dabplus_decoder.cpp:49-142)
    int32_t sf_frame_count;           // logical frames currently in the window (0..5)
    int32_t pad;
};

struct MscCollectParams {
    const int8_t* soft; int64_t soft_stride; const int32_t* active;
    const MscSlotState* slots; int n_slots; int slot;
    int8_t* ring; int ring_pitch;
};

struct MscPrepParams {
    const int32_t* active; const MscSlotState* slots; int n_slots; int slot;
    const int8_t* ring; int ring_pitch;
    int8_t* frag_out; int frag_pitch; // [n_streams*4][frag_pitch] time-de-interleaved punctured fragments (pitch: multiple of 16)
    int32_t* valid;                   // [n_streams*4] set to 1 for every codeword produced
};

// one entry of a context's protection-profile table on the device: what a grouped launch (ViterbiParams::groups) takes per CTA
struct VitProfile {
    const uint2* steptab; const uint32_t* stage_off; const uint32_t* prbs_words;
    int32_t nsteps, nbits;
};

struct ViterbiParams {
    // punctured softbits of codeword cw at frag + (cw / cw_div) * outer_stride + (cw % cw_div) * inner_stride (16-byte aligned, readable
    // up to 160 bytes past the codeword's last softbit); values >= -127
    const int8_t* frag; int cw_div; int64_t outer_stride, inner_stride;
    const uint2* steptab;             // [nsteps] per-step expansion entries (build_vit_tables)
    const uint32_t* stage_off;        // [nstages + 1]
    int n_cw, nsteps, nbits;
    uint2* dec;                       // [(n_cw+127)/128][nsteps][128]; grouped: each CTA at its descriptor's dec_off
    // optional grouped schedule (vit_groups.cuh): CTA b decodes codewords cw_list[groups[b].first ..] with profiles[groups[b].profile];
    // steptab, stage_off, nsteps, nbits, prbs_words and n_cw are then unused
    const VitGroup* groups; const int32_t* cw_list; const VitProfile* profiles; int n_groups;
    uint8_t* out; int64_t out_stride; // packed bytes, multiple of 4
    const uint32_t* prbs_words;       // energy-dispersal sequence packed like the output (or nullptr)
    const int32_t* valid;             // optional per-codeword flag
    TraceBuf trace; uint32_t trace_kind;    // optional CTA timeline (common.cuh)
};


size_t vit_dec_bytes(int n_cw, int nsteps);
constexpr int VIT_FRAG_SLACK = 160;   // bytes the decoder kernel may read past a codeword's last softbit
void build_vit_tables_u2(const int16_t* map, int nsteps, std::vector<uint2>& steps, std::vector<uint32_t>& stage_off);
void launch_clamp_copy(const int8_t* src, int8_t* dst, int64_t n, cudaStream_t st);
void launch_msc_collect(const MscCollectParams& p, int n_streams, cudaStream_t st);
void launch_msc_gather(const MscPrepParams& p, int n_streams, cudaStream_t st);
void launch_viterbi(const ViterbiParams& p, cudaStream_t st);
void launch_fic_crc(const uint8_t* fibs, const int32_t* active, int n_frames, int32_t* mask_out, cudaStream_t st);
void launch_unpack_bits(const uint8_t* bytes, int64_t stride, int n_cw, int nbits, uint8_t* bits, cudaStream_t st);

// ---- rs.cu ----
struct SuperframeParams {
    const int32_t* active; MscSlotState* slots; int n_slots; int slot; int n_streams;
    const uint8_t* logical; int64_t logical_stride;    // [n_streams*4][stride] logical frames of this step
    const int32_t* valid;                              // [n_streams*4]
    uint8_t* window; int window_pitch;                 // [n_streams][5*frame_len] raw 5-frame window (per slot buffer)
    uint8_t* sf_out; int sf_pitch;                     // [n_streams][5*frame_len] post-RS superframe when synced
    int32_t* info;                                     // [n_streams][16]: n_logical, n_events, uncorr_mask, corr[4], sf_ready, au_count, au_mask
    const uint8_t* gf_exp; const uint8_t* gf_log;
};
void launch_superframe(const SuperframeParams& p, cudaStream_t st);
// stateless: RS + sync check + AU CRCs on n superframes in place; info[n][4]
void launch_rs_superframes(uint8_t* sf, int n, int sf_len, int32_t* info, const uint8_t* gf_exp, const uint8_t* gf_log, cudaStream_t st);

// ---- ber.cu ----
// one sub-channel slot as the bit-error count reads it; frag == nullptr: the slot is not configured
struct BerSlot {
    const int8_t* frag; int64_t frag_pitch;            // [n_streams*4][frag_pitch] the step's fragments (MscPrepParams::frag_out)
    const int32_t* valid;                              // [n_streams*4] codewords the step decoded
    const uint8_t* logical; int64_t logical_stride;    // [n_streams*4][stride] their logical frames
};
struct BerParams {
    const int8_t* soft; int64_t soft_stride;           // FIC codeword (s, b) = softbits [2304 b, 2304 b + 2304) of frame s
    const uint8_t* fibs;                               // [n_streams*4][96] decoded FIC blocks
    const int32_t* active;                             // [n_streams] 1 = the frame was decoded
    const MscSlotState* slots; int n_slots;
    BerSlot slot[4];                                   // DABB_MAX_SUBCH
    const dabb_ber::Profile* profiles;                 // [DABB_MAX_PROFILES + 1]: the context's protection profiles, then the FIC
    int fic_profile;                                   // index of the FIC's entry
    void* res;                                         // [n_streams] dabb_ber_result
    int n_streams;
};
void launch_ber(const BerParams& p, cudaStream_t st);

} // namespace dabb
