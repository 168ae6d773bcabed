/*
 * dab_b200.h — C ABI of the GPU-native (H100, sm_90a) DAB/DAB+ physical-layer decode path (libdab_b200.so).
 *
 * This is the drop-in boundary: plain pointers and sizes, no C++ / torch types.  It is what the host glue
 * (welle.io_b200/host/radio-receiver.{h,cpp}, which mirrors the reference's RadioReceiver surface) and any other
 * FFI (ctypes in welle.io_b200/dabb200.py, or a cgo/JNI stub) binds.  Every entry point names the reference
 * interface it replaces (paths relative to src/ of the welle.io sources).
 *
 * Conventions: every function returns 0 on success or a negative DABB_E_* code; dabb_last_error() gives the text.
 * No CPU fallback exists: without a CUDA device dabb_create fails with DABB_E_NODEVICE.
 * One submitting thread per context.  All device work of a context runs on the context's own CUDA stream.
 *
 * Streams: a context decodes `n_streams` independent ensembles ("streams") in lock-step, one transmission
 * frame (96 ms, 196 608 samples) per stream per dabb_process() call.  Per-stream receiver state (sample position,
 * NCO phase, fine/coarse frequency correctors, FIC success counter, 16-CIF time de-interleaver history,
 * 5-frame superframe window) lives on the device between calls.
 */
#ifndef DAB_B200_H
#define DAB_B200_H
#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DABB_ABI_VERSION 3

enum {
    DABB_OK = 0,
    DABB_E_NODEVICE = -1,   /* no CUDA device / driver */
    DABB_E_CUDA = -2,       /* CUDA runtime error (see dabb_last_error) */
    DABB_E_ARG = -3,        /* invalid argument */
    DABB_E_STATE = -4,      /* call not valid in this state */
    DABB_E_NOMEM = -5,
    DABB_E_UNSUPPORTED = -6 /* e.g. transmission mode other than I */
};

/* Mode I constants (backend/dab-constants.cpp:351-361) */
enum { DABB_L = 76, DABB_K = 1536, DABB_TU = 2048, DABB_TS = 2552, DABB_TG = 504, DABB_TNULL = 2656, DABB_TF = 196608,
       DABB_SOFT_PER_FRAME = 75 * 3072, DABB_FIB_BYTES = 32, DABB_FIBS_PER_FRAME = 12, DABB_MAX_SUBCH = 4 };

typedef struct dabb_ctx dabb_ctx;

/* FFT arithmetic: DABB_FFT_EXACT reproduces the reference's KISS-FFT build bit for bit (same radix-4/2
 * factorisation, separate multiply/add roundings); DABB_FFT_FMA lets the compiler contract to FMA
 * (<= 1e-6 relative difference, faster). */
enum { DABB_FFT_EXACT = 0, DABB_FFT_FMA = 1 };
/* Oscillator arithmetic: DABB_NCO_EXACT reproduces every entry of the reference's 2 048 000-entry table bit for bit (verified
 * exhaustively at dabb_create); DABB_NCO_FAST evaluates the same phase with fp32 sincospi (each oscillator sample within ~1e-6 of
 * the table value: soft-decision intermediates within 1e-4 relative, decoded FIC/MSC bytes unchanged in the tests). */
enum { DABB_NCO_EXACT = 0, DABB_NCO_FAST = 1 };

/* RadioReceiverOptions::fftPlacementMethod / freqsyncMethod (backend/radio-receiver-options.h:35-64).  0 is the reference's
 * default in both enums (the reference's own enumerator values differ: see INTEGRATION.md for the mapping). */
enum { DABB_PLACEMENT_THRESHOLD_BEFORE_PEAK = 0, DABB_PLACEMENT_STRONGEST_PEAK = 1, DABB_PLACEMENT_EARLIEST_PEAK_WITH_BINNING = 2 };
enum { DABB_FREQSYNC_PATTERN_OF_ZEROS = 0, DABB_FREQSYNC_GET_MIDDLE = 1, DABB_FREQSYNC_CORRELATE_PRS = 2 };

typedef struct {
    int32_t abi_version;        /* DABB_ABI_VERSION */
    int32_t device;             /* CUDA device ordinal */
    int32_t n_streams;          /* streams decoded per dabb_process call */
    int32_t transmission_mode;  /* only 1 (RadioReceiver ctor arg, backend/radio-receiver.cpp:66-80) */
    int32_t fft_mode;           /* DABB_FFT_* */
    int32_t disable_coarse;     /* RadioReceiverOptions::disableCoarseCorrector (radio-receiver-options.h:66-85) */
    int32_t keep_taps;          /* 1: keep CIR / softbits / constellation / null symbol of the last frame readable via dabb_read_tap */
    int32_t n_subch_slots;      /* sub-channels decodable per stream at once (1..DABB_MAX_SUBCH), 0 -> 1 */
    int32_t max_subch_cu;       /* largest selectable sub-channel in capacity units, 0 -> 144; values above 864 (the whole MSC) are taken as 864 */
    int32_t ofdm_groups;        /* CTAs per frame in the OFDM kernel (divisor of 75), 0 -> chosen from n_streams */
    int32_t fft_placement;      /* DABB_PLACEMENT_* (PhaseReference::findIndex variant) */
    int32_t freqsync_method;    /* DABB_FREQSYNC_* (OFDMProcessor::processPRS variant) */
    int32_t nco_mode;           /* DABB_NCO_*: arithmetic of the frequency-correcting oscillator (ofdm-processor.cpp:92-94,211-214) */
    int32_t ofdm_tail_split;    /* 0: automatic (large batches cut their last frames into short CTAs), -1: off */
    int32_t reserved[2];
} dabb_config;

/* replaces: RadioReceiver::setReceiverOptions (backend/radio-receiver.cpp:119-124): takes effect from the next frame */
typedef struct {
    int32_t disable_coarse;
    int32_t fft_placement;      /* DABB_PLACEMENT_* */
    int32_t freqsync_method;    /* DABB_FREQSYNC_* */
    int32_t decode_tii;         /* RadioReceiverOptions::decodeTII: analyse the transmitter identification of every decoded frame on the device
                                   (tap 9); with keep_taps, also produce tap 4 (the two spectra TIIDecoder starts from) */
    int32_t count_bit_errors;   /* count the channel bit errors of the FIC and of every decoded sub-channel codeword on the device (tap 10) */
    int32_t soft_demap;         /* DABB_DEMAP_*: how the OFDM demodulator turns each carrier into softbits (see below); a value outside the
                                   enum is refused with DABB_E_ARG and the call changes nothing */
    int32_t sample_clock;       /* DABB_CLOCK_*: track each stream's sample-clock error and remove the phase ramp it puts on the softbits
                                   (see below); a value outside the enum is refused with DABB_E_ARG and the call changes nothing */
    int32_t acquisition;        /* DABB_ACQ_*: how a stream that is not synchronised finds the null symbol (see below); a value outside the enum
                                   is refused with DABB_E_ARG and the call changes nothing */
} dabb_options;

/* Soft-decision demap of the OFDM demodulator, dabb_options.soft_demap; takes effect from the next step, and dabb_ofdm_demod uses the
 * context's current value.
 * DABB_DEMAP_REFERENCE (0, the default) is OfdmDecoder::decodeDataSymbol (ofdm-decoder.cpp:198-219): for data symbol l and carrier k,
 *   r1 = X_l[k] conj(X_{l-1}[k]), l1 = |Re r1| + |Im r1|, softbit = trunc(-Re/Im(r1) * 127 / l1)
 * It divides away every carrier's amplitude, so a carrier in a deep multipath notch is as confident as the strongest one.
 * DABB_DEMAP_WEIGHTED (replaces: none; it deviates from ofdm-decoder.cpp:208-214) scales weak carriers down:
 *   G_l = 2^(mean over the symbol's 1536 carriers of log2(max(l1, 2^-126))), the geometric mean of the carrier levels
 *   softbit = trunc(-Re/Im(r1) * 127 / max(l1, G_l))
 * A carrier with l1 >= G_l gets exactly the reference softbits; a weaker one gets them scaled by l1 / G_l, never more confidence than
 * the reference gives it; |softbit| <= 127.  The geometric mean is barely moved by a few very strong carriers (a narrowband interferer),
 * unlike the arithmetic mean.  G_l = 0 (the reference demap for the whole symbol) when any l1 of the symbol is inf or NaN.  G_l is
 * within 1e-5 relative of its float64 value and is computed inside the CTA that transforms the symbol in a fixed order, so the softbits
 * do not depend on the batch size or the launch configuration.  r1_out (tap 2's constellation, dabb_ofdm_demod's r1_out) is the same in
 * both modes.  The FIC, MSC, BER and TII paths read the softbits unchanged; more softbits truncate to 0, so tap 10 counts more
 * erasures. */
enum { DABB_DEMAP_REFERENCE = 0, DABB_DEMAP_WEIGHTED = 1 };

/* Sample-clock tracking, dabb_options.sample_clock; takes effect from the next step.
 * A recording whose sample clock is off by eps holds 2.048 M (1 + eps) samples per second of air time (ppm > 0: more samples).  Each
 * symbol's FFT window then slips eps T_s samples against its symbol, which rotates the differential product r1 of carrier k by
 * -2 pi k eps T_s / T_u (17 degrees at the band edge at 50 ppm; the DQPSK decision margin is 45).  Every frame is re-synchronised
 * from its own phase reference symbol, so nothing fails visibly: the edge carriers just feed the Viterbi decoder partly wrong softbits.
 * DABB_CLOCK_OFF (0, the default): nothing is estimated or derotated.
 * DABB_CLOCK_TRACK (1) (replaces: none; the reference has no sample-clock correction) estimates eps per stream from its frame timing:
 * a frame placed by the time synchronisation ends T_F eps samples later than the one before it, so over frames start_index - 504
 * averages to T_F eps.  Per stream the estimate e (ppm, double), a count n of frames counted, and a flag "the previous active step
 * decoded a frame" are kept.  In a step that decodes a frame (DABB_FRAME_DECODED) with TRACK:
 *   d = start_index - 504; the frame counts when the flag is set and |d| <= 64 (325 ppm; larger values are placement jumps);
 *   a counting frame does n = n + 1 (saturating), e = e + (1e6 d / 196608 - e) / min(n, 32)  (a running mean over the first 32 counted
 *   frames, then an exponential average of 32 frames); the flag is set after every decoded frame.
 * A step with DABB_FRAME_NO_SYNC or DABB_FRAME_ACQUIRING, or run with the option OFF, clears the flag; DABB_FRAME_NEED_SAMPLES changes
 * nothing; a sync loss keeps e and n (the clock belongs to the recording), dabb_stream_reset clears all three, switching to OFF keeps
 * e and n.  A frame is derotated with applied = (n >= 8 ? e : 0) from before the frame: for data symbol l >= 1 and carrier k
 * (FFT bin k for k > 0, 2048 + k for k < 0) the demap reads
 *   r1' = r1 exp(+2 pi i k applied 1e-6 T_s / T_u)
 * with a phasor within 2^-22 of the exact value in each component, computed the same way whatever the launch configuration; the
 * reference or weighted demap then runs on r1' (the weighted mode's G comes from the derotated levels).  applied == 0 leaves r1
 * untouched, so the softbits are bit-identical to OFF.  r1_out (tap 2's constellation) holds the derotated products, the values the
 * demap read.  Taps 0 and 11 and the FIC, MSC, BER and TII paths read the step's own values. */
enum { DABB_CLOCK_OFF = 0, DABB_CLOCK_TRACK = 1 };
/* one stream in one step: tap 11 (all zero when the step ran with sample_clock OFF) */
typedef struct {
    float ppm;                  /* (float)e after the step */
    float applied_ppm;          /* the value this step's frame was derotated with (0 when no frame was decoded) */
    int32_t frames;             /* n */
    int32_t reserved;
} dabb_clock_result;

/* Acquisition, dabb_options.acquisition; takes effect from the next step.  A stream in the middle of a search continues from its position
 * under whichever method is set; dabb_stream_reset starts a new search.
 * DABB_ACQ_REFERENCE (0, the default) is OFDMProcessor::run's notSynced state (ofdm-processor.cpp:253-323): a 50-sample mean of |Re|+|Im|
 * below 0.5 sLevel.  During the null symbol that ratio is about sqrt(N / (S + N)), 0.71 at 0 dB SNR, so below about 2 dB the dip rarely
 * crosses the threshold, and a narrowband interferer fills the null.
 * DABB_ACQ_ROBUST (1) (replaces: none; it deviates from ofdm-processor.cpp:253-323 and phasereference.cpp:73-97) searches the spectrum:
 *   span: from the stream's position p (logical), nb = min(floor((buf_len - (p - buf_start)) / 256), 784) consecutive blocks of 256
 *     samples aligned to p; nb < 32 (or p outside the buffer): no search in this step, nothing changes.  Sample i of the span is
 *     mixed with the oscillator as OFDMProcessor::getSamples mixes it, osc[(localPhase - (i + 1)(coarse + fine)) mod 2 048 000] (not at
 *     all while both are 0);
 *   block level: with w[n] = 0.5 - 0.5 c[n], c[n] = (float)cos(2 pi n / 256) from double, X = the 256-point DFT of w[n] y[n] (radix-2
 *     decimation in time, every product and sum rounded) and P_k = Re^2 + Im^2 of bin k, |k| <= 87 (|f| <= 700 kHz), the level is
 *     mean over k of log2(min(max(P_k, 2^-126), FLT_MAX)) (NaN reads as 2^-126): lane t of 32 sums k = t - 87, t - 55, ... in ascending
 *     order, the 32 partials are added in lane order, then divided by 175.  log2 is a fixed series within 3e-7 of the exact value, and a level
 *     depends neither on the batch size nor on the stream index;
 *   decision: W_b = the sum of the levels of blocks b .. b + 8 in ascending order (nine blocks lie wholly inside the 2656-sample null at
 *     any alignment); b* = the last b with the smallest W_b (in digital silence, where all are equal, its end); M = the ((nb - 1) / 2)-th smallest level; depth = (M - W_b* / 9) * 3.0103
 *     dB.  A null is found when depth >= 1.2 dB (D) and b* + 11 <= nb;
 *   found: the null ends at about p + 256 b* + 2480 (between 2304 and 2656 samples after the window's first sample when the window lies
 *     in the null); the stream skips 256 b* + 2224 samples (tracking starts 256 samples before that estimate), localPhase advances by
 *     the samples skipped times (coarse + fine) as getSamples would, and it is acquired: time synchronisation places the frame from
 *     there as it does after the reference's search, with any placement.  When the step's buffer does not hold that frame the step
 *     reports DABB_FRAME_NEED_SAMPLES with next_pos at the hand-off (the only case in which that status comes with a changed state);
 *   not found: the stream skips 256 (nb - 11) samples, so that a null the buffer's end cut through is searched whole in the next step,
 *     counts one acq_failed and reports DABB_FRAME_ACQUIRING;
 *   either way sLevel becomes the span's mean |Re| + |Im| (block sums in lane order, then summed in double).
 * Under DABB_ACQ_ROBUST the phase reference correlation (find_index) also excises narrowband interferers: between the forward transform
 * of the window and the multiply by conj(PRS), with G the geometric mean of the 1536 in-band bin powers (same log2 and clamp; thread t of
 * 128 sums its bins t + 128 c in ascending c, the 128 partials in thread order), every in-band bin with log2 P > log2 G + log2 20 (T = 20)
 * and its two neighbours on each side (circularly) are set to 0.  A window with no such bin gives bit for bit the CIR and index of the
 * reference correlation.  Against the float64 restatement (tests/acqref.py) a level is within 2e-5 (2e-5 times the amplitude ratio of a tone to
 * the ensemble beside a tone: the float32 transform's error in the weak bins), a depth within 3.1 times that in dB. */
enum { DABB_ACQ_REFERENCE = 0, DABB_ACQ_ROBUST = 1 };
/* one stream in one step: tap 13 (all zero when the step ran with DABB_ACQ_REFERENCE) */
typedef struct {
    int32_t searched;           /* 1: the stream searched in this step */
    int32_t blocks;             /* nb, the blocks analysed */
    float depth_db;             /* depth of the best window */
    int32_t excised;            /* bins zeroed in this step's phase reference window */
    int64_t null_end;           /* logical position of the found null's estimated end (p + 256 b* + 2480), -1 when none was found */
} dabb_acq_result;

/* Diversity reception (replaces: none; the reference is one receiver with one input).  Coherent multi-channel receivers record one file
 * per antenna on a shared sample clock; decoded as neighbouring streams of one context, the antennas of one capture can be combined.
 * dabb_set_combining groups streams: leader is a HOST array of n == n_streams entries; leader[s] == s means stream s is alone or leads a
 * group, any other value is the stream whose group s joins.  Every entry must satisfy leader[leader[s]] == leader[s], and a group has at
 * most DABB_MAX_BRANCHES members, its leader included; NULL dissolves every group.  A malformed table (an index out of range, a chain, an
 * oversized group, a wrong n) returns DABB_E_ARG and changes nothing.  Like a select call, the function waits for outstanding work and
 * takes effect from the next step (tap 0 of the last step keeps that step's combination); dabb_stream_reset does not change the grouping.  The members of a group must share one logical sample
 * axis (buf_start), as the files of one coherent capture do.
 * In a step where leader L decodes a frame (DABB_FRAME_DECODED):
 *   A_x = buf_start[x] + the start of x's phase reference symbol in its buffer, the symbol's absolute position;
 *   N_x = the mean of |y|^2 over the 2656 samples of the null symbol that ends x's frame window, NCO applied (tap 3's samples): for i in
 *         ascending order the partial sums t = i mod 256 of Re^2 + Im^2, then the 256 partial sums in order, divided by 2656 (fp32);
 *   member b contributes when it also decoded a frame in this step, |A_b - A_L| <= 504 and N_b is finite and > 0; L always contributes
 *   (alone, when N_L itself is 0 or not finite);
 *   for every data symbol l the leader's decoders read and every carrier k, R = sum over the contributors in ascending stream index of
 *   r1_b[l][k] / N_b in fp32 (each division and addition rounded), r1_b the product b's own demap reads (derotated under
 *   DABB_CLOCK_TRACK); the leader's softbits are the context's demap of R: DABB_DEMAP_REFERENCE trunc(-Re/Im(R) 127 / l1(R)),
 *   DABB_DEMAP_WEIGHTED with G taken over the combined levels (per thread of 128 in ascending carrier order, the 128 sums in order).
 * The result depends neither on the batch size, ofdm_groups nor the tail split.  When no other member contributes the leader's softbits
 * are its own, bit for bit.  Every member other than the leader decodes exactly as it would ungrouped (its FIBs, logical frames, BER,
 * TII and clock outputs are unchanged), so each antenna's own result stays available.  The leader's FIC, sub-channels and tap 10 read the
 * combined softbits, and so does tap 0 of a leader (for every symbol); taps 2 and 3 keep every stream's own values.  A context that never
 * forms a group of two or more allocates nothing for it and runs exactly what it runs without this call. */
enum { DABB_MAX_BRANCHES = 8 };
int dabb_set_combining(dabb_ctx* ctx, const int32_t* leader, int32_t n);
/* one stream in one step: tap 12 */
typedef struct {
    int32_t members;            /* contributors of this step (the leader included); 0 for a non-leader or a step without a frame */
    uint32_t mask;              /* bit i: the i-th member of the group in ascending stream order contributed */
    float noise;                /* this stream's N, or 0 when it was not computed (not grouped, or no frame) */
    int32_t reserved;
} dabb_combine_result;

/* Channel bit errors of one stream in one step: tap 10, while dabb_options.count_bit_errors is set.  Per codeword (a FIC block of 768
 * bits, or a logical frame of 24 * bitrate bits) the decoded bits before energy dispersal (the output bytes MSB first, XOR the PRBS; 6
 * zero tail bits) are re-encoded with the K=7 rate-1/4 mother code and punctured like the codeword's protection (FIC: 21 x PI_16,
 * 3 x PI_15; EEP / UEP: the profile's blocks; both with the tail).  The k-th transmitted bit is the k-th softbit the decoder read
 * (softbits past the profile's own length are not counted).  A softbit 0 is an erasure; otherwise s > 0 decides 1 and s < 0 decides 0,
 * and an error is a decision that differs from the re-encoded bit.  bits counts the transmitted positions, erasures included:
 * channel BER = errors / (bits - erasures).  The FIC counts cover the 4 codewords of a frame with status DABB_FRAME_DECODED; subch[k]
 * covers the logical frames the step delivered in slot k (codewords == n_logical[k]).  Everything else is zero. */
typedef struct {
    int32_t fic_bits, fic_errors, fic_erasures, reserved;
    struct { int32_t codewords, bits, errors, erasures; } subch[DABB_MAX_SUBCH];
} dabb_ber_result;

/* Modulation error ratio (MER) of one stream in one step: tap 14, while dabb_set_mer is on (replaces: none; the reference's only signal
 * figure is OfdmDecoder::get_snr, dabb_frame_result.snr_raw, measured on bins outside the ensemble's 1536 carriers).
 * MER is measured on the softbits the FIC decoder reads, so it shows what the decoder is given.  Under DABB_DEMAP_REFERENCE the softbits
 * of a carrier are trunc(-Re r1 127 / l1) and trunc(-Im r1 127 / l1), l1 = |Re r1| + |Im r1|, which fixes the phase of r1 to within
 * the 8-bit quantization.  For one carrier with softbits a (Re) and b (Im):
 *   u = |a| + |b|,  v = |a| - |b|        (int32; a, b the int8 softbits, -128 read as -128)
 * v / u = tan(pi/4 - theta), theta the angle of r1 folded into its quadrant, so v^2 / u^2 is the squared error of the unit-normalised
 * product against its nearest DQPSK point and u^2 that point's power.  For a stream whose step has status DABB_FRAME_DECODED, with the
 * measurement on:
 *   points: data symbols l = 1, 2, 3 (the FIC's: softbits [l - 1][0 .. 3071] of tap 0, in every decoded frame whatever the symbol mask,
 *     keep_taps or sub-channel selection), logical carriers i = 0 .. 1535, a = soft[i], b = soft[1536 + i];
 *   group: logical carrier i is physical carrier k = perm[i] (the frequency interleaver, freq-interleaver.cpp:35-59), k in [-768, 768]
 *     without 0; its group is g = (k + 768 - (k > 0)) / 24, 0 .. 63 with 24 carriers each, lowest frequency first;
 *   sig = sum of u^2 and err = sum of v^2 over the 4608 points, exact int64; group[g].sig / .err the same sums over the group's 72
 *     points, int32 (at most 72 * 256^2 < 2^31); points = the number of the 4608 points with u > 0;
 *   mer_db = 10 log10(sig / err) in double, rounded to float; +INFINITY when err == 0 < sig, 0 when sig == 0.
 * Every other stream, and every stream of a step run with the measurement off, gets an all-zero record.  The sums are integers, so a
 * record depends neither on the batch size, ofdm_groups, the tail split, keep_taps nor the stream index.
 * The softbits are those the FIC decoder reads: a diversity leader's are the combined ones (the record shows the combination's gain),
 * its members keep their own antenna's; under DABB_CLOCK_TRACK they are the derotated ones.  Under DABB_DEMAP_WEIGHTED a carrier below
 * the symbol's geometric-mean level has smaller softbits, so it weighs less in sig / err and its phase is resolved more coarsely:
 * compare MER only between streams under the same demap.
 * Meaning (a model of one carrier pair, reference demap, AWGN on both symbols): from 12 to 40 dB per-carrier SNR the MER follows the SNR
 * within 0.9 dB; below about 10 dB it saturates towards 5.6 dB (the decision-directed floor, where tap 10's bit errors take over); above
 * about 40 dB the 8-bit softbits cannot resolve the phase.  Valid range: 10 to 40 dB of per-carrier SNR, which is the SNR over 2.048 MHz
 * plus 1.25 dB (10 log10(2048 / 1536)).  The 64-group profile shows multipath notches, narrowband interferers and band-edge roll-off.
 * dabb_set_mer(ctx, 1) switches the measurement on, dabb_set_mer(ctx, 0) off, from the next dabb_process / dabb_submit (steps already
 * enqueued keep what they were enqueued with).  The first enable allocates the group table and the records and waits for outstanding
 * work; a context that never enables it allocates and launches nothing for it. */
enum { DABB_MER_GROUPS = 64 };
typedef struct {
    int32_t points;             /* points with u > 0 (at most 4608) */
    float mer_db;               /* 10 log10(sig / err) */
    int64_t sig, err;           /* sum of u^2, sum of v^2 over the 4608 points */
    struct { int32_t sig, err; } group[DABB_MER_GROUPS];
} dabb_mer_result;
int dabb_set_mer(dabb_ctx* ctx, int32_t enable);

/* Transmitter identification (TIIDecoder, backend/tii-decoder.cpp:236-383) of one stream in one step: tap 9.  Every decoded frame is
 * analysed while dabb_options.decode_tii is set; each (comb, pattern) combination found in a frame accumulates its phase-error table over
 * five analyses and is then reported once, like onTIIMeasurement.  A frame reports at most DABB_TII_MAX combinations (the reference
 * skips frames with 10 or more); within a record they are in ascending (comb, pattern) order (the reference's order within a frame is
 * that of an unordered_map).  A stream keeps at most 32 combinations open: a new one beyond that replaces the least recently analysed
 * one, which then starts over (`evicted`).  dabb_stream_reset clears a stream's combinations; switching decode_tii off keeps them. */
enum { DABB_TII_MAX = 9 };
typedef struct {
    int32_t count;              /* measurements reported in this step (0..DABB_TII_MAX) */
    int32_t evicted;            /* open combinations replaced in this step */
    int32_t skipped;            /* 1: the frame was decoded but not analysed (10 or more likely combinations) */
    int32_t reserved;
    struct {
        int32_t comb, pattern;  /* tii_measurement_t::comb, pattern */
        int32_t delay_samples;  /* delay hypothesis -4 .. 499 with the smallest accumulated phase error */
        float error;            /* that accumulated error (integer valued) */
    } m[DABB_TII_MAX];
} dabb_tii_result;

/* replaces: RadioReceiver::RadioReceiver / ~RadioReceiver (backend/radio-receiver.h:52-116) */
int dabb_create(const dabb_config* cfg, dabb_ctx** out);
void dabb_destroy(dabb_ctx* ctx);
const char* dabb_last_error(const dabb_ctx* ctx);   /* ctx may be NULL for create failures */
int dabb_abi_version(void);

/* replaces: OFDMProcessor::restart (backend/ofdm-processor.cpp:115-132): stream goes back to acquisition at
 * logical sample position `pos` with zeroed correctors, cleared FIC counter, de-interleaver and superframe window */
int dabb_stream_reset(dabb_ctx* ctx, int32_t first_stream, int32_t count, int64_t pos);
int dabb_set_options(dabb_ctx* ctx, const dabb_options* opt);
/* introspection.  DABB_INFO_OSC_MODE: 1 = the oscillator of OFDMProcessor::getSamples (ofdm-processor.cpp:92-94,211-214) is
 * evaluated on the fly, which dabb_create allows only after comparing it on the device with the 2 048 000-entry table for every
 * index (DABB_INFO_OSC_MISMATCHES must be 0), 0 = table lookups; DABB_INFO_OSC_PATCHED: how many of the 2000 double-precision
 * factors had to be replaced by the table's own value for that (3: the quarter turns) */
enum { DABB_INFO_OSC_MODE = 0, DABB_INFO_OSC_MISMATCHES = 1, DABB_INFO_OSC_PATCHED = 2 };
int dabb_get_info(dabb_ctx* ctx, int32_t what, int64_t* out);

/* replaces: MscHandler::addSubchannel / removeSubchannel (backend/msc-handler.cpp:61-127) + DabAudio ctor
 * (backend/dab-audio.cpp:46-85).  slot in [0, DABB_MAX_SUBCH).  Protection exactly as ProtectionSettings
 * (backend/dab-constants.h:152-166): short_form -> UEP (bitrate + uep_level), else EEP profile/level. */
typedef struct {
    int32_t subch_id;     /* informational */
    int32_t start_cu;     /* Subchannel::startAddr */
    int32_t length_cu;    /* Subchannel::length */
    int32_t bitrate;      /* kbit/s = Subchannel::bitrate() */
    int32_t short_form;   /* 1 = UEP */
    int32_t uep_level;    /* ProtectionSettings::uepLevel (1..5) */
    int32_t eep_profile_a;/* 1 = EEP-A, 0 = EEP-B */
    int32_t eep_level;    /* 1..4 */
    int32_t dabplus;      /* 1 = DAB+ (RS + Fire code + AU CRC), 0 = DAB MP2 (logical frames only) */
} dabb_subchannel;
/* Streams in one slot are independent: each may use its own sub-channel, bitrate, protection profile and DAB/DAB+, and a call that
 * selects or removes some streams leaves the decoding of every other stream of the slot byte for byte as it was (the named streams
 * restart their time de-interleaver and superframe search).  A context holds up to DABB_MAX_PROFILES distinct protection profiles
 * (bitrate + UEP level or EEP profile/level), counted over all slots from its creation on; a select call that would add one more
 * returns DABB_E_UNSUPPORTED and changes nothing.  Step outputs: a stream's logical frames are 3*bitrate bytes and its superframes
 * 15*bitrate bytes of its own bitrate, so msc_stride / sf_stride must cover the largest of them among the streams enabled in any
 * slot; bytes behind a stream's own length, and the rows of streams not enabled in a slot, are left as the caller had them. */
enum { DABB_MAX_PROFILES = 64 };
int dabb_select_subchannel(dabb_ctx* ctx, int32_t first_stream, int32_t count, int32_t slot, const dabb_subchannel* sc);
int dabb_remove_subchannel(dabb_ctx* ctx, int32_t first_stream, int32_t count, int32_t slot);

/* Per-stream, per-call result record (POD). */
typedef struct {
    int32_t status;         /* DABB_FRAME_* */
    int32_t start_index;    /* PhaseReference::findIndex result (phasereference.cpp:73) */
    int32_t fine_corr;      /* OFDMProcessor::fineCorrector after the frame (ofdm-processor.cpp:450) */
    int32_t coarse_corr;    /* OFDMProcessor::coarseCorrector */
    int32_t snr_raw;        /* OfdmDecoder::get_snr value for this PRS (ofdm-decoder.cpp:240) */
    int32_t fib_crc_mask;   /* bit f set = FIB f CRC ok (fic-handler.cpp:214-229) */
    int32_t fic_ratio;      /* FicHandler::getFicDecodeRatioPercent()/10 */
    int32_t n_logical[DABB_MAX_SUBCH];     /* logical frames produced this call per slot (0..4) */
    int32_t n_rs_events[DABB_MAX_SUBCH];   /* RS decode attempts this call per slot (0..4) */
    int32_t rs_uncorr_mask[DABB_MAX_SUBCH];/* bit e = attempt e had uncorrectable codewords */
    int32_t rs_corr[DABB_MAX_SUBCH][4];    /* corrected symbols per attempt (RSDecoder::DecodeSuperframe) */
    int32_t sf_ready[DABB_MAX_SUBCH];      /* 1 = a superframe passed the Fire-code sync check this call */
    int32_t sf_au_count[DABB_MAX_SUBCH];
    int32_t sf_au_crc_mask[DABB_MAX_SUBCH];/* bit i = AU i CRC ok (dabplus_decoder.cpp:122-131) */
    int64_t next_pos;       /* logical sample position where the next frame's T_u read starts */
    float   freq_corr_re, freq_corr_im;    /* FreqCorr accumulator (ofdm-processor.cpp:435-442) */
    float   slevel;
    int32_t acq_failed;     /* null searches that failed inside this call (each one re-enters OFDMProcessor::run's notSynced state,
                               ofdm-processor.cpp:253-323: what RadioReceiver::restart(doScan) counts for onSignalPresence) */
    int32_t reserved[2];
} dabb_frame_result;

enum { DABB_FRAME_DECODED = 0, DABB_FRAME_NEED_SAMPLES = 1, DABB_FRAME_NO_SYNC = 2, DABB_FRAME_ACQUIRING = 3 };

/* One decode step for all streams.
 *   iq            interleaved (re,im) samples in `iq_format` (default cf32), stream s at iq + s*stride_samples complex samples
 *   iq_is_host    0: device pointer; 1: host pointer (pinned or pageable) -> copied H2D inside the call
 *   buf_start[s]  logical sample index of the first sample in stream s's buffer (host array, n_streams entries)
 *   buf_len       complex samples available per stream buffer
 * The stream consumes [pos, pos + T_u + startIndex + 75*T_s + T_null) of its logical sample axis; if the buffer
 * does not cover what is needed the stream reports DABB_FRAME_NEED_SAMPLES and its state is unchanged.
 * Outputs are written to host memory (any of them may be NULL):
 *   results [n_streams]
 *   fibs    [n_streams][12][32]   FIB bytes, MSB first (RadioControllerInterface::onFIBDecodeSuccess payload packed)
 *   msc     [n_streams][DABB_MAX_SUBCH][4][msc_stride] logical frames (3*bitrate bytes each; DecoderAdapter::addtoFrame data)
 *   sf      [n_streams][DABB_MAX_SUBCH][sf_stride]     post-RS superframe (15*bitrate bytes) when sf_ready
 * replaces: one iteration of OFDMProcessor::run (ofdm-processor.cpp:324-490) + OfdmDecoder::workerthread
 * (ofdm-decoder.cpp:93-130) + FicHandler::processFicBlock + MscHandler::processMscBlock + DabAudio::run +
 * DecoderAdapter::addtoFrame + SuperframeFilter::Feed, for n_streams receivers at once.
 */
typedef struct {
    const float* iq; int32_t iq_is_host; int64_t stride_samples; const int64_t* buf_start; int64_t buf_len;
    dabb_frame_result* results; uint8_t* fibs; uint8_t* msc; int32_t msc_stride; uint8_t* sf; int32_t sf_stride;
    int32_t iq_format;   /* DABB_IQ_*: raw sample format of `iq` (strides and lengths stay in complex samples); converted on the
                            device exactly like CRAWFile::convertSamples (input/raw_file.cpp:324-366) */
    int32_t carry_samples;   /* dabb_submit only: the first `carry_samples` complex samples of every stream's window are the LAST
                                `carry_samples` of the window given to the previous dabb_submit (a receiver reads its input once; the overlap
                                a frame needs is kept on the device): they are taken from the previous staging slot instead of being copied
                                host->device again.  0 = copy the whole window.  Ignored by dabb_process / dabb_process_async. */
} dabb_io;
enum { DABB_IQ_CF32 = 0, DABB_IQ_U8 = 1, DABB_IQ_S8 = 2, DABB_IQ_S16LE = 3, DABB_IQ_S16BE = 4 };
/* dabb_process and dabb_submit check their arguments before anything is enqueued: a call refused with DABB_E_ARG or DABB_E_STATE
 * (for example an msc_stride below 3*bitrate or an sf_stride below 15*bitrate of a selected sub-channel) runs no step and leaves
 * every stream's state as it was. */
int dabb_process(dabb_ctx* ctx, const dabb_io* io);
/* asynchronous form for benchmarking with device-resident inputs: enqueue only, no host copies */
int dabb_process_async(dabb_ctx* ctx, const dabb_io* io);
int dabb_sync(dabb_ctx* ctx);
/* Pipelined form of dabb_process for HOST buffers (io->iq_is_host must be 1; pinned memory for full overlap): dabb_submit enqueues the
 * host->device copy of the step's samples on a copy stream (two device staging slots), the kernels, and the device->host copy of the
 * results into pinned staging, and returns without waiting; at most two steps may be outstanding (DABB_E_STATE otherwise).
 * dabb_collect waits for the OLDEST outstanding step and writes its results to the output pointers given at that dabb_submit (they
 * must stay valid until then; io->iq must stay valid until the step has been collected).  Results come back in submit order; the
 * copy of step n+1 overlaps the kernels of step n and the read-back of step n-1. */
int dabb_submit(dabb_ctx* ctx, const dabb_io* io);
int dabb_collect(dabb_ctx* ctx);
/* makes the context's main stream (dabb_cuda_stream) wait for everything enqueued so far on the library's other streams, so that an
 * event recorded on it afterwards marks the completion of all work of the preceding dabb_process_async calls (timing) */
int dabb_join_lanes(dabb_ctx* ctx);
void* dabb_cuda_stream(dabb_ctx* ctx);              /* cudaStream_t of the context */
int64_t dabb_kernel_launches(const dabb_ctx* ctx);  /* number of CUDA kernels this context has launched */

/* per-kernel device timing: while enabled, one CUDA event is recorded on the context's stream after every kernel launch;
 * dabb_profile_read returns {"kernel": {"ms": total, "n": launches}, ...} as JSON text */
int dabb_profile(dabb_ctx* ctx, int32_t enable);
int dabb_profile_read(dabb_ctx* ctx, char* json_out, size_t cap);

/* taps (valid after a dabb_process when keep_taps=1):
 *   0 = softbits int8 [n_streams][75*3072]               also without keep_taps.  Such a context demaps only the symbols its decoders
 *                                                        read (the FIC's and each selected sub-channel's); reading tap 0 repeats the
 *                                                        last step's OFDM launch over every symbol first, so the last step's input
 *                                                        samples must still be in place
 *   1 = CIR float [n_streams][2048]                     RadioControllerInterface::onNewImpulseResponse (phasereference.cpp:93)
 *   2 = constellation cf32 [n_streams][75][16]          onConstellationPoints: r1 of every 96th carrier (ofdm-decoder.cpp:216-218)
 *   3 = null symbol cf32 [n_streams][2656], NCO applied  onNewNullSymbol (ofdm-processor.cpp:462-469)
 *   4 = TII spectra cf32 [n_streams][2][2048] (only while dabb_options.decode_tii is set): fft::Forward of the frame's phase
 *       reference symbol and of the last T_u samples of the null symbol that follows it, what TIIDecoder::run computes first
 *       (tii-decoder.cpp:197-214); tap 9 is the analysis of these spectra
 * and, with any keep_taps, what the last step of dabb_process_async left on the device, the outputs dabb_process would have returned:
 *   5 = dabb_frame_result [n_streams]
 *   6 = FIBs uint8 [n_streams][12][32]
 *   7 = logical frames uint8 [n_streams][DABB_MAX_SUBCH][4][stride], the layout of dabb_io.msc; stride = bytes / (n_streams * DABB_MAX_SUBCH * 4)
 *   8 = DAB+ superframes uint8 [n_streams][DABB_MAX_SUBCH][stride], the layout of dabb_io.sf; stride = bytes / (n_streams * DABB_MAX_SUBCH)
 *   9 = dabb_tii_result [n_streams] of the last step (all zero when that step ran with decode_tii off); DABB_E_STATE until
 *       dabb_options.decode_tii has been set once
 *  10 = dabb_ber_result [n_streams] of the last step (all zero when that step ran with count_bit_errors off); DABB_E_STATE until
 *       dabb_options.count_bit_errors has been set once
 *  11 = dabb_clock_result [n_streams] of the last step (all zero when that step ran with sample_clock OFF); DABB_E_STATE until
 *       dabb_options.sample_clock has been set to DABB_CLOCK_TRACK once
 *  12 = dabb_combine_result [n_streams] of the last step (all zero when that step ran without a group); DABB_E_STATE until
 *       dabb_set_combining has formed a group of two or more streams once
 *  13 = dabb_acq_result [n_streams] of the last step; DABB_E_STATE until dabb_options.acquisition has been set to DABB_ACQ_ROBUST once
 *  14 = dabb_mer_result [n_streams] of the last step (all zero when that step ran with the measurement off); DABB_E_STATE until
 *       dabb_set_mer(ctx, 1) has been called once */
int dabb_read_tap(dabb_ctx* ctx, int32_t what, void* host_out, size_t bytes);

/* ---------------------------------------------------------------------------------------------------------
 * Wideband channelizer: turns recordings at other sample rates, tuned between ensembles or holding several of them, into the
 * 2 048 000 samples/s streams dabb_process decodes.
 * replaces: none.  The reference's only rate conversion is the Airspy driver's 2:1 average of neighbouring samples
 * (input/airspy_sdr.cpp:188-209); its input layer hands the backend 2.048 Msps only.
 *
 * A channelizer belongs to a context.  It reads n_inputs wideband inputs at a common rate R Hz (an integer) in one DABB_IQ_* format
 * (converted exactly like convert_iq_kernel / CRAWFile::convertSamples) and produces n_channels channels; channel c reads input
 * input_of_channel[c] and is centred at offset_hz[c].  Accepted: 2 048 000 <= R <= 64 000 000 with 2 048 000 / R = L / M in lowest
 * terms and L <= 1024 (2.048, 2.4, 2.5, 3, 4.096, 6, 8, 8.192, 10, 20, 61.44 Msps and more), |offset_hz| + 768 000 <= R / 2,
 * 1 <= n_channels <= 4096; a rate outside this is DABB_E_UNSUPPORTED, anything else malformed DABB_E_ARG.
 *
 * Filter: one Kaiser-windowed-sinc prototype h of L*T taps at rate L*R, cutoff 856 000 Hz (midway between the 768 kHz edge of the
 * 1536 carriers and the 944 kHz edge of the neighbouring ensemble), beta = 0.1102 * (72 - 8.7), T = ceil((72 - 7.95) /
 * (14.36 * 176 000 / R)) + 1 taps per branch; designed in double, scaled so that the taps sum to L, rounded to float.  At the rates
 * listed above it has at most 0.005 dB ripple for |f| <= 768 kHz and at least 71 dB attenuation for |f| >= 944 kHz.
 *
 * Output m of channel c is the absolute sample index m on that channel's 2.048 Msps axis.  With n_m = floor(m M / L),
 * p_m = (m M) mod L and x the channel's input:
 *     y[m] = sum_{j=0}^{T-1} h[p_m + j L] x[n_m - j] exp(-2 pi i k(n_m - j) / R),   k(n) = (offset_hz * n) mod R in exact integers
 * so an output depends on m and the input samples [n_m - T + 1, n_m] only.  The channelizer keeps no state between calls: cutting a
 * run into calls of any size gives the same samples bit for bit, and a stream that re-acquires simply asks for another range.
 * Every output is within 1e-5 of rms(y) (rms error) and 1e-4 (largest error) of the same sum in exact arithmetic. */
typedef struct dabb_chan dabb_chan;
typedef struct {
    int64_t rate_hz;                    /* R */
    int32_t iq_format;                  /* DABB_IQ_* of the inputs */
    int32_t n_inputs;
    int32_t n_channels;
    int32_t reserved;
    const int32_t* input_of_channel;    /* [n_channels] host array, 0 .. n_inputs - 1 */
    const int64_t* offset_hz;           /* [n_channels] host array */
} dabb_chan_config;
/* creates a channelizer of ctx (designs its filter and uploads it).  A context that never creates one allocates nothing for it.
 * Destroy every channelizer of a context before the context. */
int dabb_chan_create(dabb_ctx* ctx, const dabb_chan_config* cfg, dabb_chan** out);
void dabb_chan_destroy(dabb_chan* ch);   /* NULL is a no-op; waits for the context's work */
/* the input span [*in_first, *in_end) (absolute input indices) that outputs [out_start, out_start + out_len) of any channel read:
 * in_first = n_{out_start} - T + 1, in_end = n_{out_start + out_len - 1} + 1.  out_start >= 0, out_len >= 1 */
int dabb_chan_input_range(const dabb_chan* ch, int64_t out_start, int64_t out_len, int64_t* in_first, int64_t* in_end);
/* One channelizer call.
 *   in            input i at in + i * in_stride samples of the configured format; host (in_is_host = 1, copied inside the call) or device
 *   in_start[i]   absolute index of input i's first sample (host array, n_inputs entries); every buffer holds in_len samples
 *   out           device float2 [n_channels][out_stride]: row c receives outputs [out_start[c], out_start[c] + out_len) of channel c
 *   out_start[c]  host array, n_channels entries, >= 0; out_start[c] + out_len <= 2^45
 * The work is enqueued on the context's main stream, so a following dabb_process / dabb_process_async on the same context reads `out`
 * as a device iq (iq_is_host = 0, stride_samples = out_stride, buf_start[s] = out_start[s]).  Arguments are checked before anything is
 * enqueued: a NULL pointer, out_len < 1, a stride below its length, or a channel whose input span (dabb_chan_input_range) does not
 * lie inside its buffer returns DABB_E_ARG and writes nothing. */
typedef struct {
    const void* in; int32_t in_is_host; int64_t in_stride; const int64_t* in_start; int64_t in_len;
    float* out; int64_t out_stride; const int64_t* out_start; int64_t out_len;
} dabb_chan_io;
int dabb_channelize(dabb_chan* ch, const dabb_chan_io* io);

/* ---------------------------------------------------------------------------------------------------------
 * Spectrum survey: where the ensembles of a wideband recording are, before anything is decoded.
 * replaces: the reference's channel scan (CRadioController::startScan / nextChannel, welle-gui/radio_controller.cpp:406,902), which
 * retunes the receiver channel by channel and waits for onSignalPresence; a recording cannot be retuned, so the whole band is looked at
 * at once and each candidate is then confirmed by decoding it (batch_decode --scan).
 *
 * dabb_survey: the averaged power spectrum of each of n_inputs inputs of in_len samples (input i at in + i * in_stride samples, in
 * iq_format, converted exactly like dabb_channelize / CRAWFile::convertSamples; host with in_is_host = 1, else device).  Welch segments
 * of nfft samples (a power of two, 1024 .. 16384) with 50 % overlap: S = floor((in_len - nfft) / (nfft/2)) + 1 segments, segment s
 * starting at sample s * nfft/2 (samples past the last segment are not read).  With the periodic Hann window w[n] = sin^2(pi n / nfft):
 *     P[j] = (1/S) sum_s |sum_n w[n] x[s nfft/2 + n] exp(-2 pi i k n / nfft)|^2 / sum_n w[n]^2,   k = (j + nfft/2) mod nfft
 * so bin j is at frequency (j - nfft/2) R / nfft, from -R/2 up to R/2 (R the input's sample rate; the survey does not need it).
 * psd is HOST float [n_inputs][nfft], written when the call returns.  The transform is fp32 (every P[j] within 1e-4 P[j] + 1e-7 mean(P)
 * of the exact value in the tests); the segments are summed in a fixed order without atomics, so the same call gives the same bits.
 * The work runs on the context's main stream; scratch is allocated on the first call and kept until dabb_destroy (a context that never
 * surveys allocates nothing).  Arguments are checked before anything is enqueued: a NULL pointer, a bad nfft, format or in_is_host,
 * n_inputs outside 1 .. 4096, in_len < nfft or in_stride < in_len returns DABB_E_ARG and writes nothing. */
typedef struct {
    const void* in; int32_t in_is_host; int32_t iq_format;
    int64_t in_stride; int32_t n_inputs; int32_t nfft;
    int64_t in_len;
    float* psd;
} dabb_survey_io;
int dabb_survey(dabb_ctx* ctx, const dabb_survey_io* io);

/* dabb_survey_candidates: the ensemble candidates of one spectrum psd[nfft] of an input at rate_hz (host code, no context).  With
 * f_j = (j - nfft/2) R / nfft and L_j = 10 log10(max(P_j, 1e-12 max P)) (no candidates when max P = 0):
 *   - a centre bin c is considered when |f_c| + 768 000 <= R/2 (the channelizer's rule);
 *   - its in-band set is I = {j : |f_j - f_c| <= 700 000};
 *   - its guard sides are G- = {j : 784 000 <= f_c - f_j <= 896 000} and G+ = {j : 784 000 <= f_j - f_c <= 896 000}, each clipped to
 *     |f_j| <= R/2 - R/nfft; a side is present when it keeps at least ceil(56 000 nfft / R) bins, and c is skipped when neither is
 *     (the guards lie inside the 176 kHz gap to a neighbour on the 1.712 MHz raster, clear of its 944 kHz edge);
 *   - score(c) = mean over I of L - the larger mean over the present guard sides (double sums in ascending j), so a centre at the edge
 *     of a wider signal, with one side inside it, scores about 0 dB;
 *   - every maximal run of consecutive considered bins with score >= min_score_db is one candidate: offset_hz is the run's midpoint
 *     ((c_first + c_last - nfft) R) / (2 nfft) rounded to the nearest Hz (ties away from zero), score_db the run's largest score.
 * Membership is decided by exact integer comparisons.  Candidates are written in ascending offset, at most cap of them; *n_found is
 * the full count.  DABB_E_ARG for a NULL pointer, a bad nfft, a rate outside 1 .. 64 000 000 or cap < 0. */
typedef struct { int64_t offset_hz; float score_db; int32_t reserved; } dabb_survey_candidate;
int dabb_survey_candidates(const float* psd, int32_t nfft, int64_t rate_hz, float min_score_db,
                           dabb_survey_candidate* out, int32_t cap, int32_t* n_found);

/* ---------------------------------------------------------------------------------------------------------
 * Stage-level entry points (stateless).  Pointers are DEVICE pointers unless named host_*.
 * ------------------------------------------------------------------------------------------------------- */

/* OfdmDecoder::processPRS + decodeDataSymbol for n frames (ofdm-decoder.cpp:144-230).
 * Frame f: PRS useful part at iq + f*stride + prs_start[f] (2048 samples) followed by 75 symbols of 2552 samples.
 * soft_out: int8 [n][75][3072]; r1_out (may be NULL): float2 [n][75][1536] pre-quantisation products;
 * freqcorr_out (may be NULL): float2 [n] CP correlation sums (ofdm-processor.cpp:436-442).
 * nco (may be NULL): int32 [n][2] = {localPhase at the first PRS sample, phase increment Hz} (ofdm-processor.cpp:211-214).
 * The softbits follow the context's dabb_options.soft_demap (DABB_DEMAP_*); r1_out does not depend on it. */
int dabb_ofdm_demod(dabb_ctx* ctx, const float* iq, int64_t stride_samples, const int64_t* prs_start, int32_t n_frames,
                    const int32_t* nco, int8_t* soft_out, float* r1_out, float* freqcorr_out);
/* the same, with frame f derotated by clock_ppm[f] (device float [n], or NULL: none) as DABB_CLOCK_TRACK derotates a frame with its
 * applied value; r1_out holds the derotated products.  NULL is exactly dabb_ofdm_demod; zeros give the same bits. */
int dabb_ofdm_demod_ex(dabb_ctx* ctx, const float* iq, int64_t stride_samples, const int64_t* prs_start, int32_t n_frames,
                       const int32_t* nco, const float* clock_ppm, int8_t* soft_out, float* r1_out, float* freqcorr_out);

/* PhaseReference::findIndex, ThresholdBeforePeak (phasereference.cpp:73-97,212-253) for n windows of 2048 samples
 * at iq + f*stride + win_start[f]; index_out int32[n]; cir_out (may be NULL) float [n][2048] */
int dabb_find_index(dabb_ctx* ctx, const float* iq, int64_t stride_samples, const int64_t* win_start, int32_t n,
                    int32_t* index_out, float* cir_out);
/* the same with any of the three placements (phasereference.cpp:93-256); negative index_out = no synchronisation, with the
 * reference's own negative value for StrongestPeak */
int dabb_find_index_ex(dabb_ctx* ctx, const float* iq, int64_t stride_samples, const int64_t* win_start, int32_t n,
                       int32_t placement, int32_t* index_out, float* cir_out);
/* OFDMProcessor::processPRS (ofdm-processor.cpp:537-644): coarse frequency estimate, in carriers, of n aligned phase reference
 * symbols (2048 samples at iq + f*stride + prs_start[f]); offset_out int32[n]; 100 = no estimate */
int dabb_coarse_estimate(dabb_ctx* ctx, const float* iq, int64_t stride_samples, const int64_t* prs_start, int32_t n,
                         int32_t freqsync_method, int32_t* offset_out);

/* Viterbi::deconvolve (viterbi.cpp:227-245) for n codewords: soft int8 [n][(nbits+6)*4] (already de-punctured,
 * 0 = punctured), bits_out uint8 [n][nbits] (one bit per byte) */
int dabb_viterbi(dabb_ctx* ctx, const int8_t* soft, int32_t n_codewords, int32_t nbits, uint8_t* bits_out);

/* FicHandler::processFicBlock x3 (fic-handler.cpp:111-230): soft int8 [n][9216] (symbols 1..3),
 * fib_out uint8 [n][12][32], crc_mask_out int32 [n] */
int dabb_fic_decode(dabb_ctx* ctx, const int8_t* soft, int32_t n_frames, uint8_t* fib_out, int32_t* crc_mask_out);

/* EEPProtection/UEPProtection::deconvolve + EnergyDispersal + byte pack (eep-protection.cpp:115-152,
 * energy_dispersal.h:35-54, decoder_adapter.cpp:57-67): soft int8 [n][length_cu*64] (time-de-interleaved),
 * bytes_out uint8 [n][3*bitrate] */
int dabb_msc_decode(dabb_ctx* ctx, const dabb_subchannel* sc, const int8_t* soft, int32_t n_cifs, uint8_t* bytes_out);

/* RSDecoder::DecodeSuperframe + SuperframeFilter::CheckSync + AU CRCs (dabplus_decoder.cpp:326-359,171-215,122-131)
 * on n superframes in place: sf uint8 [n][sf_len]; info int32 [n][4] = {corr, uncorr, sync_ok, au_crc_mask|num_aus<<8} */
int dabb_rs_superframes(dabb_ctx* ctx, uint8_t* sf, int32_t n, int32_t sf_len, int32_t* info);

/* device memory helpers so that non-CUDA hosts (ctypes) can stage buffers */
int dabb_dev_alloc(dabb_ctx* ctx, size_t bytes, void** out);
int dabb_dev_free(dabb_ctx* ctx, void* p);
int dabb_memcpy_h2d(dabb_ctx* ctx, void* dst_dev, const void* src_host, size_t bytes);
int dabb_memcpy_d2h(dabb_ctx* ctx, void* dst_host, const void* src_dev, size_t bytes);

#ifdef __cplusplus
}
#endif
#endif
