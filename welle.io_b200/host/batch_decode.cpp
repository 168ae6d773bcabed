/*
 * batch_decode.cpp — native batch driver over the C ABI: decodes many RAW IQ recordings at once, one stream per file (or per ensemble of a
 * wideband file, --rate), on one GPU.
 *
 *   batch_decode [--format cf32|u8|s8|s16le|s16be] [--device N] [--coarse] [--tii] [--ber] [--mer] [--soft weighted|reference] [--clock]
 *                [--acq robust|reference] [--diversity N] [--rate HZ --offset HZ[,HZ...]|auto] [--rate HZ --scan] --out DIR file1 [file2 ...]
 *
 * What `welle-cli -f FILE -D` does for one recording (welle-cli.cpp:215-235,612-707: dump the FIC, tune to the first audio
 * service, dump its logical frames) done for all files in lock-step: every iteration hands each stream's next window of samples
 * to one dabb_process() call (host buffers, copied to the device inside the call), then walks the per-stream result records:
 * FIBs (33-byte records: CRC flag + 32 bytes) go to DIR/<name>.fic, the FIGs feed the stream's service database (fig-db.h), the
 * first audio service is selected as soon as its sub-channel is known (every stream's in slot 0 of the library, whatever its bitrate
 * and protection), logical frames go to DIR/<name>.msc, Reed-Solomon statistics to DIR/<name>.rs.  Streams progress independently
 * (per-stream sample position, acquisition state, end of file).  No signal processing happens here.
 *
 * --tii: transmitter identification of every decoded frame, analysed on the device (dabb_options.decode_tii, tap 9); each measurement
 * goes to DIR/<name>.tii as one line "comb pattern delay_samples error", the format of glue_test's .tii (onTIIMeasurement).
 *
 * --ber: channel bit errors counted on the device (dabb_options.count_bit_errors, tap 10); every decoded frame adds one line
 * "fic_bits fic_errors fic_erasures codewords bits errors erasures" to DIR/<name>.ber, the last four for the service's slot (0).
 *
 * --mer: the modulation error ratio of the FIC softbits, measured on the device (dabb_set_mer, tap 14) in the decode context only (not in
 * the --scan / --offset auto survey and confirmation contexts).  Every decoded frame adds one line "points mer_db sig err" to
 * DIR/<name>.mer; at the end DIR/<name>.merprof gets one line "first_carrier last_carrier sig err mer_db" per group of 24 carriers
 * (DABB_MER_GROUPS, lowest frequency first), sig and err summed in int64 over every decoded frame of the run and mer_db = 10 log10(sig /
 * err) of those sums (inf when err == 0 < sig, 0 when sig == 0).
 *
 * --soft weighted|reference: the OFDM demodulator's soft-decision demap (dabb_options.soft_demap) of every context the driver creates,
 * the --scan / --offset auto survey and confirmation contexts included.  reference (the default) is the reference decoder's demap and
 * leaves the options untouched; weighted scales down the softbits of carriers below the symbol's geometric-mean level, which helps the
 * Viterbi decoder in multipath (DABB_DEMAP_WEIGHTED).
 *
 * --clock: sample-clock tracking (dabb_options.sample_clock = DABB_CLOCK_TRACK) in every context the driver creates, the --scan /
 * --offset auto survey and confirmation contexts included: each stream estimates its recording's sample-clock error from its frame
 * timing and the demodulator removes the phase ramp it puts on the softbits.  Every decoded frame adds one line "ppm applied_ppm frames"
 * (tap 11) to DIR/<name>.clk.
 *
 * --acq robust|reference: how a stream that is not synchronised finds the null symbol (dabb_options.acquisition) in every context the
 * driver creates, the --scan / --offset auto survey and confirmation contexts included.  reference (the default) is the reference's
 * envelope-dip search and leaves the options untouched; robust finds the null from the spectral level of 256-sample blocks, down to
 * about 0 dB SNR and beside strong narrowband interferers, and excises such interferers from the phase reference correlation
 * (DABB_ACQ_ROBUST).  Every step in which a stream searched adds one line "blocks depth_db found" (tap 13) to DIR/<name>.acq.
 *
 * --diversity N: consecutive runs of N files are the antennas of one capture (one coherent receiver's files: same rate, same first
 * sample); the first file of each run leads its group (dabb_set_combining) and decodes from the noise-weighted sum of the group's
 * differential products.  Every file keeps its outputs as without the option (the leader's are those of the combination, the others'
 * their own antenna's), and every decoded frame of a leader adds one line "members mask noise" (tap 12) to DIR/<name>.div.  1 <= N <=
 * DABB_MAX_BRANCHES, the file count a multiple of N; not with --rate.
 *
 * --rate HZ --offset HZ[,HZ...]: every file is a wideband recording at HZ samples/s (any rate dabb_chan_create accepts) and every offset
 * (Hz from the tuned frequency, may be negative) is one stream of the batch, decoded by a channelizer of the same context (dabb_chan_*):
 * outputs go to DIR/<name>@<offset>.{fic,msc,rs} (and .tii / .ber / .clk / .mer / .merprof), in the formats above.  The streams of one file progress
 * independently (their own position, acquisition and end of file).  Every step channelizes exactly each stream's [pos, pos + need) of its
 * 2.048 Msps axis into that stream's device window and then runs dabb_process on the windows; the channelizer keeps no state, so nothing
 * is shifted on the device, and the host keeps per file only the input span its live streams still need.
 *
 * --rate HZ --scan: finds the ensembles of every wideband recording and writes them to DIR/<name>.scan, one line per ensemble in ascending
 * offset: "offset_hz candidate_hz score_db frames_ok eid label".  Every file is surveyed over its first R/4 samples (0.25 s), or the
 * whole file if it is shorter (a file shorter than nfft is not surveyed), in one dabb_survey call with nfft the smallest power of two >= 1024 with R / nfft <= 4000 Hz, and
 * dabb_survey_candidates turns each spectrum into candidates (min_score_db = 6).  Every candidate becomes one stream of a context with
 * the coarse corrector on (estimator GetMiddle), channelized at the candidate's offset and decoded over at most the first 8 frames; its
 * located offset is the candidate's plus coarse_corr + fine_corr of a decoded frame (the decoder's oscillator removes that much) plus
 * the 0.9 of that frame's measured residual (atan2(freq_corr_im, freq_corr_re) / pi * 500 Hz) the fine corrector has not yet taken, of
 * the frame whose residual is smallest (the latest of equals).  Then the located offset and the offsets 1 kHz to either side are decoded with the coarse corrector off over at most the first
 * 16 frames (16 x 196 608 samples of the channel); the one with the most frames whose 12 FIB CRCs all pass, if it has at least 2, is an
 * ensemble at its offset + fine_corr + 0.9 of the residual, as above.  Of ensembles within 10 kHz of each other the one with the higher
 * score is kept.  eid is FIG 0/0's EId in four hex digits and label
 * FIG 1/0's ensemble label, "-" where not received.  Each candidate's confirmation (frames decoded, good frames, measured offset) and
 * the survey and confirmation times go to stderr.
 * --rate HZ --offset auto: the same scan (no .scan file), then the --offset decode of each file at its own ensembles' offsets: the outputs
 * are those of --offset with those offsets.
 *
 * Sample formats are the RAW-file formats of CRAWFile (input/raw_file.cpp:324-366); they are shipped as they are and converted on
 * the device.
 */
#include "dab_api.h"
#include "fig-db.h"
#include "../../include/dab_b200.h"

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <memory>
#include <string>
#include <vector>

namespace {

struct Stream {
    std::string path, name; FILE* in = nullptr; FILE* fic = nullptr; FILE* msc = nullptr; FILE* rs = nullptr; FILE* tii = nullptr; FILE* ber = nullptr; FILE* clk = nullptr;
    FILE* div = nullptr;                                          /* --diversity: a group leader's combinations */
    FILE* acq = nullptr;                                          /* --acq robust: the null searches */
    FILE* mer = nullptr;                                          /* --mer: every decoded frame's MER */
    std::vector<int64_t> mer_prof;                                /* --mer: [DABB_MER_GROUPS][2] sig, err summed over the run */
    int64_t buf_start = 0, have = 0, pos = 0, acq_need = 0;      /* logical sample indices; `have` samples are buffered from buf_start */
    bool tracking = false, eof = false, done = false;
    std::unique_ptr<dabb_host::FigDb> db{new dabb_host::FigDb()};
    int slot = -1; int bitrate = 0; uint32_t sid = 0;
    long frames = 0, fibs_ok = 0, fibs = 0, logical = 0;
    int file = -1; int64_t offset = 0;                            /* wideband mode: the recording and the channel's offset in Hz */
    /* --scan confirmation: the detector's candidate and score, frames whose 12 FIB CRCs pass, and the frequency error the decoder
     * found at `offset` in its last decoded frame (confirm_result) */
    int64_t candidate = 0; float score = 0.f; long frames_ok = 0; int64_t corr = 0; double best_residual = 0.0; bool eid_seen = false, label_seen = false;
};

/* wideband mode: one recording, read into a host buffer that holds input samples [first, first + have) (silence past the end of the
 * file up to `len`), and the channelizer of its streams */
struct Wide {
    std::string path; FILE* in = nullptr; std::vector<uint8_t> buf; int64_t first = 0, have = 0; bool eof = false;
    std::vector<int> streams; std::vector<int64_t> offsets; dabb_chan* ch = nullptr;
};

struct Outputs {
    std::vector<dabb_frame_result> res; std::vector<uint8_t> fibs, msc, sf; std::vector<dabb_tii_result> tres; std::vector<dabb_ber_result> bres;
    std::vector<dabb_clock_result> cres;        /* tap 11, read after every step when not empty (--clock) */
    std::vector<dabb_combine_result> dres;      /* tap 12, read after every step when not empty (--diversity) */
    std::vector<dabb_acq_result> ares;          /* tap 13, read after every step when not empty (--acq robust) */
    std::vector<dabb_mer_result> mres;          /* tap 14, read after every step when not empty (--mer) */
};

/* the receiver position after one step's result r of stream s: 0 = the stream ended, 1 = no frame decoded, 2 = a frame was decoded */
int advance(dabb_ctx* ctx, Stream& z, int s, const dabb_frame_result& r, int64_t TF)
{
    if (r.status == DABB_FRAME_NEED_SAMPLES) return 0;          /* cannot happen for a live stream: stop it rather than spin */
    z.pos = r.next_pos;
    if (r.status == DABB_FRAME_NO_SYNC) { z.tracking = false; return 1; }
    if (r.status == DABB_FRAME_ACQUIRING) {
        z.tracking = false;
        if (z.acq_need < 5 * TF) z.acq_need += TF;
        else { z.pos += 2 * TF; z.acq_need = 3 * TF; dabb_stream_reset(ctx, s, 1, z.pos); }
        return z.eof ? 0 : 1;
    }
    z.tracking = true; z.acq_need = 3 * TF; z.frames++;
    return 2;
}

/* what one dabb_process step returned for stream s: files, service database, tuning, the receiver position; false = the stream ended */
bool handle_result(dabb_ctx* ctx, Stream& z, int s, const Outputs& o, bool tii, bool ber, int64_t TF)
{
    const dabb_frame_result& r = o.res[(size_t)s];
    if (z.acq && o.ares[(size_t)s].searched) {
        const dabb_acq_result& q = o.ares[(size_t)s];
        fprintf(z.acq, "%d %.3f %d\n", q.blocks, q.depth_db, q.null_end >= 0 ? 1 : 0);
    }
    if (tii)
        for (int i = 0; i < o.tres[(size_t)s].count; i++) {
            const auto& m = o.tres[(size_t)s].m[i];
            fprintf(z.tii, "%d %d %d %.1f\n", m.comb, m.pattern, m.delay_samples, m.error);
        }
    const int a = advance(ctx, z, s, r, TF);
    if (a != 2) return a != 0;
    if (ber) {
        const dabb_ber_result& b = o.bres[(size_t)s];
        fprintf(z.ber, "%d %d %d %d %d %d %d\n", b.fic_bits, b.fic_errors, b.fic_erasures, b.subch[0].codewords, b.subch[0].bits, b.subch[0].errors, b.subch[0].erasures);
    }
    if (z.clk) {
        const dabb_clock_result& c = o.cres[(size_t)s];
        fprintf(z.clk, "%.4f %.4f %d\n", c.ppm, c.applied_ppm, c.frames);
    }
    if (z.div) {
        const dabb_combine_result& d = o.dres[(size_t)s];
        fprintf(z.div, "%d %u %.6e\n", d.members, d.mask, d.noise);
    }
    if (z.mer) {
        const dabb_mer_result& m = o.mres[(size_t)s];
        fprintf(z.mer, "%d %.3f %lld %lld\n", m.points, m.mer_db, (long long)m.sig, (long long)m.err);
        for (int g = 0; g < DABB_MER_GROUPS; g++) { z.mer_prof[(size_t)g * 2] += m.group[g].sig; z.mer_prof[(size_t)g * 2 + 1] += m.group[g].err; }
    }
    for (int f = 0; f < 12; f++) {
        const uint8_t* fb = o.fibs.data() + ((size_t)s * 12 + (size_t)f) * 32;
        const uint8_t ok = (r.fib_crc_mask >> f) & 1;
        fputc(ok, z.fic); fwrite(fb, 32, 1, z.fic);
        z.fibs++; z.fibs_ok += ok;
        if (ok) { dabb_host::FigEvents ev; z.db->parseFib(fb, ev); }
    }
    if (z.slot >= 0) {
        const int flen = 3 * z.bitrate, k = z.slot;
        for (int c = 4 - r.n_logical[k]; c < 4; c++) { fwrite(o.msc.data() + (((size_t)s * DABB_MAX_SUBCH + (size_t)k) * 4 + (size_t)c) * 1152, (size_t)flen, 1, z.msc); z.logical++; }
        for (int e = 0; e < r.n_rs_events[k]; e++) fprintf(z.rs, "%d %d\n", (r.rs_uncorr_mask[k] >> e) & 1, r.rs_corr[k][e]);
    } else {
        /* tune to the first audio service whose sub-channel organisation is known */
        for (const auto& c : z.db->components) {
            if (c.transportMode() != TransportMode::Audio || c.audioType() == AudioServiceComponentType::Unknown) continue;
            if (c.subchannelId < 0 || c.subchannelId >= 64 || !z.db->subch[(size_t)c.subchannelId].valid()) continue;
            const Subchannel& u = z.db->subch[(size_t)c.subchannelId];
            dabb_subchannel sc; memset(&sc, 0, sizeof sc);
            sc.subch_id = u.subChId; sc.start_cu = u.startAddr; sc.length_cu = u.length; sc.bitrate = u.bitrate();
            sc.short_form = u.protectionSettings.shortForm; sc.uep_level = u.protectionSettings.uepLevel;
            sc.eep_profile_a = u.protectionSettings.eepProfile == EEPProtectionProfile::EEP_A; sc.eep_level = (int)u.protectionSettings.eepLevel;
            sc.dabplus = c.audioType() == AudioServiceComponentType::DABPlus;
            const int k = 0;
            if (dabb_select_subchannel(ctx, s, 1, k, &sc) != DABB_OK) { fprintf(stderr, "batch_decode: %s: %s\n", z.name.c_str(), dabb_last_error(ctx)); z.slot = -2; break; }
            z.slot = k; z.bitrate = sc.bitrate; z.sid = c.SId;
            break;
        }
    }
    return true;
}

/* the result of a --scan confirmation step for stream s: the receiver position, good frames, the correctors, the ensemble's EId and label */
bool confirm_result(dabb_ctx* ctx, Stream& z, int s, const Outputs& o, int64_t TF)
{
    const dabb_frame_result& r = o.res[(size_t)s];
    const int a = advance(ctx, z, s, r, TF);
    if (a != 2) return a != 0;
    if (r.fib_crc_mask == 0xFFF) z.frames_ok++;
    /* the oscillator removes coarse + fine; the frame's residual (the CP correlation's phase, in Hz) is what the fine corrector still
     * lacks, of which it has just taken a tenth (OFDMProcessor::run's fineCorrector update) */
    const double residual = atan2((double)r.freq_corr_im, (double)r.freq_corr_re) / 3.14159265358979323846 * 500.0;
    /* the residual is only known modulo 1 kHz: the frame with the smallest one (the latest of equals) is the least likely to have
     * wrapped, e.g. while the coarse corrector still alternates between two neighbouring kHz */
    if (z.frames == 1 || fabs(residual) <= z.best_residual) {
        z.best_residual = fabs(residual);
        z.corr = (int64_t)r.coarse_corr + r.fine_corr + (int64_t)llround(0.9 * residual);
    }
    for (int f = 0; f < 12; f++) {
        if (!((r.fib_crc_mask >> f) & 1)) continue;
        dabb_host::FigEvents ev;
        z.db->parseFib(o.fibs.data() + ((size_t)s * 12 + (size_t)f) * 32, ev);
        for (const auto& e : ev.list) {
            if (e.kind == dabb_host::FigEvents::NewEnsemble) z.eid_seen = true;
            if (e.kind == dabb_host::FigEvents::EnsembleLabel) z.label_seen = true;
        }
    }
    return true;
}

/* --mer: DIR/<name>.merprof, one line "first_carrier last_carrier sig err mer_db" per carrier group of the run's summed tap-14 records */
bool write_mer_profile(const std::string& path, const std::vector<int64_t>& prof)
{
    FILE* f = fopen(path.c_str(), "w");
    if (!f) return false;
    for (int g = 0; g < DABB_MER_GROUPS; g++) {
        const int first = 24 * g - 768 + (g >= DABB_MER_GROUPS / 2 ? 1 : 0);       /* carrier 0 is not used */
        const long long sig = prof[(size_t)g * 2], err = prof[(size_t)g * 2 + 1];
        const double db = sig == 0 ? 0.0 : err == 0 ? INFINITY : 10.0 * log10((double)sig / (double)err);
        fprintf(f, "%d %d %lld %lld %.3f\n", first, first + 23, sig, err, db);
    }
    return fclose(f) == 0;
}

int bytes_per_sample(int fmt) { return fmt == DABB_IQ_CF32 ? 8 : (fmt == DABB_IQ_U8 || fmt == DABB_IQ_S8) ? 2 : 4; }

/* one dabb_process step of every stream's window, and the taps the options ask for */
bool step(dabb_ctx* ctx, Outputs& o, std::vector<int64_t>& buf_start, const float* iq, int iq_is_host, int64_t stride, int64_t buf_len, int iq_format, bool tii, bool ber)
{
    dabb_io io; memset(&io, 0, sizeof io);
    io.iq = iq; io.iq_is_host = iq_is_host; io.stride_samples = stride; io.buf_start = buf_start.data(); io.buf_len = buf_len;
    io.results = o.res.data(); io.fibs = o.fibs.data(); io.iq_format = iq_format;
    if (!o.msc.empty()) { io.msc = o.msc.data(); io.msc_stride = 1152; io.sf = o.sf.data(); io.sf_stride = 5760; }
    if (dabb_process(ctx, &io) != DABB_OK) { fprintf(stderr, "batch_decode: %s\n", dabb_last_error(ctx)); return false; }
    if (tii && dabb_read_tap(ctx, 9, o.tres.data(), o.tres.size() * sizeof(dabb_tii_result)) != DABB_OK) { fprintf(stderr, "batch_decode: %s\n", dabb_last_error(ctx)); return false; }
    if (ber && dabb_read_tap(ctx, 10, o.bres.data(), o.bres.size() * sizeof(dabb_ber_result)) != DABB_OK) { fprintf(stderr, "batch_decode: %s\n", dabb_last_error(ctx)); return false; }
    if (!o.cres.empty() && dabb_read_tap(ctx, 11, o.cres.data(), o.cres.size() * sizeof(dabb_clock_result)) != DABB_OK) { fprintf(stderr, "batch_decode: %s\n", dabb_last_error(ctx)); return false; }
    if (!o.dres.empty() && dabb_read_tap(ctx, 12, o.dres.data(), o.dres.size() * sizeof(dabb_combine_result)) != DABB_OK) { fprintf(stderr, "batch_decode: %s\n", dabb_last_error(ctx)); return false; }
    if (!o.ares.empty() && dabb_read_tap(ctx, 13, o.ares.data(), o.ares.size() * sizeof(dabb_acq_result)) != DABB_OK) { fprintf(stderr, "batch_decode: %s\n", dabb_last_error(ctx)); return false; }
    if (!o.mres.empty() && dabb_read_tap(ctx, 14, o.mres.data(), o.mres.size() * sizeof(dabb_mer_result)) != DABB_OK) { fprintf(stderr, "batch_decode: %s\n", dabb_last_error(ctx)); return false; }
    return true;
}

/* Decodes the streams of wideband recordings until all have ended: one channelizer per recording (at its streams' offsets, w.offsets;
 * the streams of a recording are consecutive in st), every stream a device window of W samples of its 2.048 Msps axis.  limit > 0 ends a
 * stream whose next step would read outputs at or past `limit`.  handle(s) takes stream s's result of a step; false ends the stream. */
bool run_wide(dabb_ctx* ctx, std::vector<Stream>& st, std::vector<Wide>& wf, int64_t rate, int fmt, int64_t limit, std::vector<int64_t>& buf_start,
              const std::function<bool(const float*, int64_t)>& run_step, const std::function<bool(int)>& handle)
{
    const int S = (int)st.size();
    const int64_t TF = DABB_TF, W = 6 * TF;
    const int64_t need_track = DABB_TU + (DABB_TU - 1) + 75LL * DABB_TS + DABB_TNULL;
    const int bps = bytes_per_sample(fmt);
    int active = S;
    for (Wide& w : wf) {
        if (w.streams.empty()) continue;
        w.in = fopen(w.path.c_str(), "rb");
        if (!w.in) { fprintf(stderr, "batch_decode: cannot open %s\n", w.path.c_str()); return false; }
        const std::vector<int32_t> input_of(w.offsets.size(), 0);
        dabb_chan_config cc; memset(&cc, 0, sizeof cc);
        cc.rate_hz = rate; cc.iq_format = fmt; cc.n_inputs = 1; cc.n_channels = (int32_t)w.offsets.size();
        cc.input_of_channel = input_of.data(); cc.offset_hz = w.offsets.data();
        if (dabb_chan_create(ctx, &cc, &w.ch) != DABB_OK) { fprintf(stderr, "batch_decode: %s\n", dabb_last_error(ctx)); return false; }
        int64_t end0 = 0;                                         /* the recording is input [0, ...); silence before it */
        dabb_chan_input_range(w.ch, 0, 1, &w.first, &end0);
    }
    void* win = nullptr;
    if (dabb_dev_alloc(ctx, (size_t)S * (size_t)W * 8, &win) != DABB_OK) { fprintf(stderr, "batch_decode: %s\n", dabb_last_error(ctx)); return false; }
    const uint8_t silence = fmt == DABB_IQ_U8 ? 0x80 : 0;
    std::vector<int64_t> out_start;
    while (active > 0) {
        /* the ABI takes one window length for all streams: the neediest live stream's */
        int64_t out_len = 0;
        for (const Stream& z : st) if (!z.done) out_len = std::max(out_len, z.tracking ? need_track : z.acq_need);
        for (Wide& w : wf) {
            /* [lo, hi): the input span the file's live streams read for outputs [pos, pos + out_len); live: one of them */
            int live = -1;
            int64_t lo = INT64_MAX, hi = INT64_MIN;
            auto span = [&]() {
                live = -1; lo = INT64_MAX; hi = INT64_MIN;
                for (int s : w.streams) {
                    if (st[(size_t)s].done) continue;
                    int64_t a, b;
                    dabb_chan_input_range(w.ch, st[(size_t)s].pos, out_len, &a, &b);
                    lo = std::min(lo, a); hi = std::max(hi, b); live = s;
                }
            };
            /* keep only [lo, ...) of the buffer */
            auto trim = [&]() {
                if (lo <= w.first) return;
                const int64_t drop = std::min(lo - w.first, w.have);
                memmove(w.buf.data(), w.buf.data() + drop * bps, (size_t)(w.have - drop) * (size_t)bps);
                w.have -= drop; w.first += drop;
                if (w.have == 0 && w.first < lo) {                /* every live stream skipped ahead of everything buffered */
                    if (fseek(w.in, (long)((lo - w.first) * bps), SEEK_CUR) != 0) w.eof = true;
                    w.first = lo;
                }
            };
            span();
            if (live < 0) continue;
            trim();
            const int64_t len = hi - w.first;
            if ((int64_t)w.buf.size() < len * bps) w.buf.resize((size_t)(len * bps));
            if (w.first < 0 && w.have == 0) {                    /* the silence in front of the recording */
                memset(w.buf.data(), silence, (size_t)(-w.first * bps)); w.have = -w.first;
            }
            if (w.have < len && !w.eof) {
                const size_t got = fread(w.buf.data() + w.have * bps, (size_t)bps, (size_t)(len - w.have), w.in);
                if ((int64_t)got < len - w.have) w.eof = true;
                w.have += (int64_t)got;
            }
            if (w.have < len) memset(w.buf.data() + w.have * bps, silence, (size_t)((len - w.have) * bps));   /* silence behind the data */
            /* a stream ends when the recording cannot give the samples its own next step needs, or that step would reach `limit` */
            bool ended = false;
            for (int s : w.streams) {
                Stream& z = st[(size_t)s];
                if (z.done) continue;
                z.eof = w.eof;
                const int64_t need = z.tracking ? need_track : z.acq_need;
                int64_t a, b;
                dabb_chan_input_range(w.ch, z.pos, need, &a, &b);
                if ((w.eof && b > w.first + w.have) || (limit > 0 && z.pos + need > limit)) { z.done = true; active--; ended = true; }
            }
            if (ended) {                                          /* the remaining streams may need less */
                span();
                if (live < 0) continue;
                trim();
                if (w.have < hi - w.first) memset(w.buf.data() + w.have * bps, silence, (size_t)((hi - w.first - w.have) * bps));
            }
            /* every stream's window = its outputs [pos, pos + out_len); a finished stream gets a live one's range (never decoded) */
            out_start.assign(w.streams.size(), 0);
            for (size_t k = 0; k < w.streams.size(); k++) {
                const Stream& z = st[(size_t)w.streams[k]];
                out_start[k] = z.done ? st[(size_t)live].pos : z.pos;
            }
            dabb_chan_io cio; memset(&cio, 0, sizeof cio);
            cio.in = w.buf.data(); cio.in_is_host = 1; cio.in_stride = hi - w.first; cio.in_start = &w.first; cio.in_len = hi - w.first;
            cio.out = static_cast<float*>(win) + (size_t)w.streams[0] * (size_t)W * 2; cio.out_stride = W; cio.out_start = out_start.data(); cio.out_len = out_len;
            if (dabb_channelize(w.ch, &cio) != DABB_OK) { fprintf(stderr, "batch_decode: %s\n", dabb_last_error(ctx)); return false; }
        }
        if (active <= 0) break;
        for (int s = 0; s < S; s++) buf_start[(size_t)s] = st[(size_t)s].done ? -(1LL << 40) : st[(size_t)s].pos;
        if (!run_step(static_cast<const float*>(win), out_len)) return false;
        for (int s = 0; s < S; s++) {
            Stream& z = st[(size_t)s];
            if (z.done) continue;
            if (!handle(s)) { z.done = true; active--; }
        }
    }
    for (Wide& w : wf) { if (w.ch) dabb_chan_destroy(w.ch); if (w.in) fclose(w.in); w.ch = nullptr; w.in = nullptr; }
    dabb_dev_free(ctx, win);
    return true;
}

std::string base_name(const std::string& path) { const size_t slash = path.find_last_of('/'); return slash == std::string::npos ? path : path.substr(slash + 1); }

/* a context of the scan with dabb_options.soft_demap = soft (--soft), sample_clock = clock (--clock) and acquisition = acq (--acq); the
 * other options as cfg gives them; false on an error */
static bool create_scan_ctx(const dabb_config& cfg, int soft, int clock, int acq, dabb_ctx** ctx)
{
    if (dabb_create(&cfg, ctx) != DABB_OK) { fprintf(stderr, "batch_decode: %s\n", dabb_last_error(nullptr)); return false; }
    if (soft == DABB_DEMAP_REFERENCE && clock == DABB_CLOCK_OFF && acq == DABB_ACQ_REFERENCE) return true;
    dabb_options op; memset(&op, 0, sizeof op);
    op.disable_coarse = cfg.disable_coarse; op.fft_placement = cfg.fft_placement; op.freqsync_method = cfg.freqsync_method; op.soft_demap = soft;
    op.sample_clock = clock; op.acquisition = acq;
    if (dabb_set_options(*ctx, &op) == DABB_OK) return true;
    fprintf(stderr, "batch_decode: %s\n", dabb_last_error(*ctx));
    dabb_destroy(*ctx);
    *ctx = nullptr;
    return false;
}

/* --scan: the ensembles of every file (ascending offset, per file), as the streams of their confirmation decode; false on an error */
bool scan(const std::vector<std::string>& files, int64_t rate, int fmt, int device, int soft, int clock, int acq, std::vector<std::vector<Stream>>& found)
{
    const int64_t TF = DABB_TF;
    const int bps = bytes_per_sample(fmt);
    const float min_score_db = 6.0f;                              /* the detector's threshold (DESIGN.md 3.6) */
    const int64_t locate_frames = 8, confirm_frames = 16, min_frames_ok = 2, same_hz = 10000, step_hz = 1000;
    auto t0 = std::chrono::steady_clock::now();
    int32_t nfft = 1024;
    while (rate > 4000LL * nfft) nfft *= 2;
    /* every file's first R/4 samples, or the whole file if it is shorter: the inputs of one call share one length, so a shorter file is
     * padded with silence, which scales its spectrum by a constant the detector (differences of dB means) does not see.  A file shorter
     * than nfft gives no spectrum and no candidates. */
    int64_t in_len = 0;
    std::vector<int64_t> lens(files.size());
    for (size_t i = 0; i < files.size(); i++) {
        FILE* in = fopen(files[i].c_str(), "rb");
        if (!in) { fprintf(stderr, "batch_decode: cannot open %s\n", files[i].c_str()); return false; }
        fseek(in, 0, SEEK_END); lens[i] = std::min<int64_t>(rate / 4, (int64_t)ftell(in) / bps); fclose(in);
        if (lens[i] < nfft) fprintf(stderr, "batch_decode: %s: fewer than %d samples, not surveyed\n", files[i].c_str(), nfft);
        in_len = std::max(in_len, lens[i]);
    }
    in_len = std::max<int64_t>(in_len, nfft);
    std::vector<uint8_t> buf(files.size() * (size_t)in_len * (size_t)bps, fmt == DABB_IQ_U8 ? 0x80 : 0);
    for (size_t i = 0; i < files.size(); i++) {
        FILE* in = fopen(files[i].c_str(), "rb");
        const size_t got = in ? fread(buf.data() + i * (size_t)in_len * (size_t)bps, (size_t)bps, (size_t)lens[i], in) : 0;
        if (in) fclose(in);
        if ((int64_t)got != lens[i]) { fprintf(stderr, "batch_decode: cannot read %s\n", files[i].c_str()); return false; }
    }
    dabb_config cfg; memset(&cfg, 0, sizeof cfg);
    cfg.abi_version = DABB_ABI_VERSION; cfg.device = device; cfg.n_streams = 1; cfg.transmission_mode = 1;
    dabb_ctx* ctx = nullptr;
    if (!create_scan_ctx(cfg, soft, clock, acq, &ctx)) return false;
    std::vector<float> psd(files.size() * (size_t)nfft);
    dabb_survey_io sio; memset(&sio, 0, sizeof sio);
    sio.in = buf.data(); sio.in_is_host = 1; sio.iq_format = fmt; sio.in_stride = in_len; sio.n_inputs = (int32_t)files.size(); sio.nfft = nfft;
    sio.in_len = in_len; sio.psd = psd.data();
    const int rc = dabb_survey(ctx, &sio);
    if (rc != DABB_OK) fprintf(stderr, "batch_decode: %s\n", dabb_last_error(ctx));
    dabb_destroy(ctx);
    if (rc != DABB_OK) return false;
    /* every candidate one stream of the first confirmation context, file by file */
    std::vector<Stream> st;
    std::vector<Wide> wf(files.size());
    std::vector<dabb_survey_candidate> cand((size_t)nfft);
    for (size_t f = 0; f < files.size(); f++) {
        int32_t n = 0;
        wf[f].path = files[f];
        if (lens[f] < nfft) continue;
        if (dabb_survey_candidates(psd.data() + f * (size_t)nfft, nfft, rate, min_score_db, cand.data(), (int32_t)cand.size(), &n) != DABB_OK) return false;
        for (int32_t k = 0; k < std::min<int32_t>(n, (int32_t)cand.size()); k++) {
            st.emplace_back();
            Stream& z = st.back();
            z.path = files[f]; z.name = base_name(files[f]); z.file = (int)f; z.candidate = z.offset = cand[(size_t)k].offset_hz; z.score = cand[(size_t)k].score_db;
            z.acq_need = 3 * TF;
            wf[f].streams.push_back((int)st.size() - 1); wf[f].offsets.push_back(z.offset);
        }
    }
    auto t1 = std::chrono::steady_clock::now();
    found.clear(); found.resize(files.size());
    /* decodes the streams of `cw` from the start of their files over at most `frames` frames */
    auto confirm = [&](std::vector<Stream>& cs, std::vector<Wide>& cw, int disable_coarse, int freqsync, int64_t frames) -> bool {
        const int S = (int)cs.size();
        if (S == 0) return true;
        cfg.n_streams = S; cfg.disable_coarse = disable_coarse; cfg.freqsync_method = freqsync;
        if (!create_scan_ctx(cfg, soft, clock, acq, &ctx)) return false;
        dabb_stream_reset(ctx, 0, S, 0);
        Outputs o; o.res.resize((size_t)S); o.fibs.resize((size_t)S * 12 * 32);
        std::vector<int64_t> buf_start((size_t)S);
        const bool ok = run_wide(ctx, cs, cw, rate, fmt, frames * TF, buf_start,
                                 [&](const float* iq, int64_t len) { return step(ctx, o, buf_start, iq, 0, 6 * TF, len, DABB_IQ_CF32, false, false); },
                                 [&](int s) { return confirm_result(ctx, cs[(size_t)s], s, o, TF); });
        dabb_destroy(ctx);
        return ok;
    };
    /* 1. locate: every candidate with the coarse corrector on.  The reference's default estimator (pattern of zeros) does not lock on
     *    offsets of a few kHz and jumps by tens of kHz between frames; GetMiddle (the centre of the spectrum's energy) settles within
     *    about 1 kHz, and the frame's residual then gives the offset modulo 1 kHz */
    if (!confirm(st, wf, 0, DABB_FREQSYNC_GET_MIDDLE, locate_frames)) return false;
    /* 2. confirm: the coarse corrector off, at the located offset and 1 kHz to either side; the fine corrector has only the last few Hz
     *    left, so the FIC passes from the first frame at the right one */
    std::vector<Stream> again;
    std::vector<Wide> wa(files.size());
    for (size_t f = 0; f < files.size(); f++) {
        wa[f].path = files[f];
        for (int s : wf[f].streams) {
            const Stream& z = st[(size_t)s];
            fprintf(stderr, "batch_decode: %s: candidate %lld (%.2f dB): %ld frames decoded, located at %lld Hz\n", z.name.c_str(), (long long)z.candidate,
                    z.score, z.frames, (long long)(z.offset + z.corr));
            if (z.frames == 0) continue;
            for (const int64_t d : {int64_t(0), -step_hz, step_hz}) {
                const int64_t at = z.offset + z.corr + d, a = at < 0 ? -at : at;
                if (2 * (a + 768000) > rate) continue;
                again.emplace_back();
                Stream& y = again.back();
                y.path = z.path; y.name = z.name; y.file = z.file; y.candidate = z.candidate; y.score = z.score; y.offset = at; y.acq_need = 3 * TF;
                wa[f].streams.push_back((int)again.size() - 1); wa[f].offsets.push_back(at);
            }
        }
    }
    if (!confirm(again, wa, 1, DABB_FREQSYNC_PATTERN_OF_ZEROS, confirm_frames)) return false;
    /* of each candidate's offsets the one with the most good frames (the located one on a tie); confirmed ones at their refined offsets;
     * of those within same_hz of each other the higher score stays */
    for (size_t f = 0; f < files.size(); f++) {
        std::vector<Stream*> c;
        for (size_t k = 0; k < wa[f].streams.size(); k++) {
            Stream& y = again[(size_t)wa[f].streams[k]];
            fprintf(stderr, "batch_decode: %s: candidate %lld at %lld Hz: %ld frames decoded, %ld with every FIB CRC good, at %lld Hz\n", y.name.c_str(),
                    (long long)y.candidate, (long long)y.offset, y.frames, y.frames_ok, (long long)(y.offset + y.corr));
            if (y.frames_ok < min_frames_ok) continue;
            if (!c.empty() && c.back()->candidate == y.candidate) { if (y.frames_ok > c.back()->frames_ok) c.back() = &y; }
            else c.push_back(&y);
        }
        std::stable_sort(c.begin(), c.end(), [](const Stream* a, const Stream* b) { return a->score > b->score; });
        std::vector<Stream*> keep;
        for (Stream* z : c) {
            bool dup = false;
            for (Stream* k : keep) { const int64_t d = (k->offset + k->corr) - (z->offset + z->corr); if (d <= same_hz && d >= -same_hz) dup = true; }
            if (!dup) keep.push_back(z);
        }
        std::sort(keep.begin(), keep.end(), [](const Stream* a, const Stream* b) { return a->offset + a->corr < b->offset + b->corr; });
        for (Stream* z : keep) found[f].push_back(std::move(*z));
    }
    auto t2 = std::chrono::steady_clock::now();
    fprintf(stderr, "batch_decode: scan of %zu file(s): survey %.1f ms (nfft %d, %lld samples), confirmation of %zu candidate(s) at %zu offsets %.1f ms\n", files.size(),
            std::chrono::duration<double, std::milli>(t1 - t0).count(), nfft, (long long)in_len, st.size(), again.size(),
            std::chrono::duration<double, std::milli>(t2 - t1).count());
    return true;
}

} // namespace

int main(int argc, char** argv)
{
    int fmt = DABB_IQ_CF32, device = 0, soft = DABB_DEMAP_REFERENCE, clock = DABB_CLOCK_OFF, acq = DABB_ACQ_REFERENCE; bool coarse = false, tii = false, ber = false, mer = false; std::string out;
    int64_t rate = 0; std::vector<int64_t> offsets; bool scan_only = false, auto_offsets = false; int diversity = 0; bool diversity_set = false;
    std::vector<std::string> files;
    for (int i = 1; i < argc; i++) {
        const std::string a = argv[i];
        if (a == "--format" && i + 1 < argc) {
            const std::string f = argv[++i];
            fmt = f == "cf32" ? DABB_IQ_CF32 : f == "u8" ? DABB_IQ_U8 : f == "s8" ? DABB_IQ_S8 : f == "s16le" ? DABB_IQ_S16LE : f == "s16be" ? DABB_IQ_S16BE : -1;
            if (fmt < 0) { fprintf(stderr, "unknown format %s\n", f.c_str()); return 2; }
        }
        else if (a == "--device" && i + 1 < argc) device = atoi(argv[++i]);
        else if (a == "--out" && i + 1 < argc) out = argv[++i];
        else if (a == "--coarse") coarse = true;
        else if (a == "--tii") tii = true;
        else if (a == "--ber") ber = true;
        else if (a == "--mer") mer = true;
        else if (a == "--clock") clock = DABB_CLOCK_TRACK;
        else if (a == "--diversity" && i + 1 < argc) { diversity = atoi(argv[++i]); diversity_set = true; }
        else if (a == "--soft" && i + 1 < argc) {
            const std::string m = argv[++i];
            soft = m == "reference" ? DABB_DEMAP_REFERENCE : m == "weighted" ? DABB_DEMAP_WEIGHTED : -1;
            if (soft < 0) { fprintf(stderr, "unknown soft demap %s\n", m.c_str()); return 2; }
        }
        else if (a == "--acq" && i + 1 < argc) {
            const std::string m = argv[++i];
            acq = m == "reference" ? DABB_ACQ_REFERENCE : m == "robust" ? DABB_ACQ_ROBUST : -1;
            if (acq < 0) { fprintf(stderr, "unknown acquisition %s\n", m.c_str()); return 2; }
        }
        else if (a == "--rate" && i + 1 < argc) rate = atoll(argv[++i]);
        else if (a == "--scan") scan_only = true;
        else if (a == "--offset" && i + 1 < argc && std::string(argv[i + 1]) == "auto") { auto_offsets = true; i++; }
        else if (a == "--offset" && i + 1 < argc) {
            const std::string l = argv[++i];
            for (size_t p = 0; p <= l.size();) {
                const size_t q = std::min(l.find(',', p), l.size());
                offsets.push_back(atoll(l.substr(p, q - p).c_str()));
                p = q + 1;
            }
        }
        else files.push_back(a);
    }
    if (out.empty() || files.empty() || (rate > 0) != ((int)!offsets.empty() + (int)scan_only + (int)auto_offsets == 1)
        || (rate <= 0 && (scan_only || auto_offsets))) {
        fprintf(stderr, "usage: batch_decode [--format cf32|u8|s8|s16le|s16be] [--device N] [--coarse] [--tii] [--ber] [--mer] [--soft weighted|reference] [--clock] [--acq robust|reference] [--diversity N] [--rate HZ --offset HZ[,HZ...]|auto] [--rate HZ --scan] --out DIR file...\n");
        return 2;
    }
    if (diversity_set && (rate > 0 || diversity < 1 || diversity > DABB_MAX_BRANCHES || files.size() % (size_t)diversity)) {
        fprintf(stderr, "batch_decode: --diversity N needs 1 <= N <= %d, a file count that is a multiple of N, and no --rate\n", DABB_MAX_BRANCHES);
        return 2;
    }
    const bool wide = rate > 0;
    /* wideband mode: the offsets of each file's streams */
    std::vector<std::vector<int64_t>> file_offsets(wide ? files.size() : 0, offsets);
    if (scan_only || auto_offsets) {
        std::vector<std::vector<Stream>> found;
        if (!scan(files, rate, fmt, device, soft, clock, acq, found)) return 1;
        for (size_t f = 0; f < files.size(); f++) {
            file_offsets[f].clear();
            for (const Stream& z : found[f]) file_offsets[f].push_back(z.offset + z.corr);
        }
        if (scan_only) {
            for (size_t f = 0; f < files.size(); f++) {
                FILE* sf = fopen((out + "/" + base_name(files[f]) + ".scan").c_str(), "w");
                if (!sf) { fprintf(stderr, "batch_decode: cannot write into %s\n", out.c_str()); return 1; }
                for (const Stream& z : found[f]) {
                    char eid[8] = "-";
                    if (z.eid_seen) snprintf(eid, sizeof eid, "%04X", z.db->eid);
                    const std::string& label = z.db->ensLabel.fig1_label;
                    fprintf(sf, "%lld %lld %.2f %ld %s %s\n", (long long)(z.offset + z.corr), (long long)z.candidate, z.score, z.frames_ok, eid,
                            z.label_seen && !label.empty() ? label.c_str() : "-");
                }
                fclose(sf);
            }
            return 0;
        }
    }

    int S = (int)files.size();
    if (wide) { S = 0; for (const auto& l : file_offsets) S += (int)l.size(); }
    if (S == 0) { fprintf(stderr, "batch_decode: no ensemble found\n"); return 0; }
    const int64_t TF = DABB_TF, W = 6 * TF;                       /* per-stream window capacity in samples */
    const int64_t need_track = DABB_TU + (DABB_TU - 1) + 75LL * DABB_TS + DABB_TNULL;
    const int bps = bytes_per_sample(fmt);

    dabb_config cfg; memset(&cfg, 0, sizeof cfg);
    cfg.abi_version = DABB_ABI_VERSION; cfg.device = device; cfg.n_streams = S; cfg.transmission_mode = 1; cfg.fft_mode = DABB_FFT_EXACT;
    cfg.disable_coarse = coarse ? 0 : 1; cfg.n_subch_slots = DABB_MAX_SUBCH; cfg.max_subch_cu = 416;
    dabb_ctx* ctx = nullptr;
    if (dabb_create(&cfg, &ctx) != DABB_OK) { fprintf(stderr, "batch_decode: %s\n", dabb_last_error(nullptr)); return 1; }
    if (tii || ber || soft != DABB_DEMAP_REFERENCE || clock != DABB_CLOCK_OFF || acq != DABB_ACQ_REFERENCE) {
        dabb_options op; memset(&op, 0, sizeof op);
        op.disable_coarse = cfg.disable_coarse; op.decode_tii = tii; op.count_bit_errors = ber; op.soft_demap = soft; op.sample_clock = clock;
        op.acquisition = acq;
        if (dabb_set_options(ctx, &op) != DABB_OK) { fprintf(stderr, "batch_decode: %s\n", dabb_last_error(ctx)); return 1; }
    }
    if (diversity > 1) {          /* the antennas of one capture: the first file of each run of `diversity` leads */
        std::vector<int32_t> leader((size_t)S);
        for (int s = 0; s < S; s++) leader[(size_t)s] = s - s % diversity;
        if (dabb_set_combining(ctx, leader.data(), S) != DABB_OK) { fprintf(stderr, "batch_decode: %s\n", dabb_last_error(ctx)); return 1; }
    }
    if (mer && dabb_set_mer(ctx, 1) != DABB_OK) { fprintf(stderr, "batch_decode: %s\n", dabb_last_error(ctx)); return 1; }

    std::vector<Stream> st((size_t)S);
    std::vector<Wide> wf(wide ? files.size() : 0);
    for (int s = 0, f = 0, k = 0; s < S; s++) {
        Stream& z = st[(size_t)s];
        if (wide) while (k >= (int)file_offsets[(size_t)f].size()) { f++; k = 0; }
        else f = s;
        z.path = files[(size_t)f];
        z.name = base_name(z.path);
        if (wide) {
            z.file = f; z.offset = file_offsets[(size_t)f][(size_t)k++];
            z.name += "@" + std::to_string(z.offset);
            wf[(size_t)f].streams.push_back(s); wf[(size_t)f].offsets.push_back(z.offset); wf[(size_t)f].path = files[(size_t)f];
        } else {
            z.in = fopen(z.path.c_str(), "rb");
            if (!z.in) { fprintf(stderr, "batch_decode: cannot open %s\n", z.path.c_str()); return 1; }
        }
        z.fic = fopen((out + "/" + z.name + ".fic").c_str(), "wb"); z.msc = fopen((out + "/" + z.name + ".msc").c_str(), "wb"); z.rs = fopen((out + "/" + z.name + ".rs").c_str(), "w");
        if (tii) z.tii = fopen((out + "/" + z.name + ".tii").c_str(), "w");
        if (ber) z.ber = fopen((out + "/" + z.name + ".ber").c_str(), "w");
        if (clock) z.clk = fopen((out + "/" + z.name + ".clk").c_str(), "w");
        const bool leads = diversity > 1 && s % diversity == 0;
        if (leads) z.div = fopen((out + "/" + z.name + ".div").c_str(), "w");
        if (acq == DABB_ACQ_ROBUST) z.acq = fopen((out + "/" + z.name + ".acq").c_str(), "w");
        if (mer) { z.mer = fopen((out + "/" + z.name + ".mer").c_str(), "w"); z.mer_prof.assign(2 * DABB_MER_GROUPS, 0); }
        if (!z.fic || !z.msc || !z.rs || (tii && !z.tii) || (ber && !z.ber) || (clock && !z.clk) || (leads && !z.div) || (acq == DABB_ACQ_ROBUST && !z.acq) || (mer && !z.mer)) { fprintf(stderr, "batch_decode: cannot write into %s\n", out.c_str()); return 1; }
        z.acq_need = 3 * TF;
    }
    dabb_stream_reset(ctx, 0, S, 0);

    Outputs o;
    o.res.resize((size_t)S); o.fibs.resize((size_t)S * 12 * 32); o.msc.resize((size_t)S * DABB_MAX_SUBCH * 4 * 1152); o.sf.resize((size_t)S * DABB_MAX_SUBCH * 5760);
    o.tres.resize(tii ? (size_t)S : 0); o.bres.resize(ber ? (size_t)S : 0); o.cres.resize(clock ? (size_t)S : 0); o.dres.resize(diversity > 1 ? (size_t)S : 0);
    o.ares.resize(acq == DABB_ACQ_ROBUST ? (size_t)S : 0); o.mres.resize(mer ? (size_t)S : 0);
    std::vector<int64_t> buf_start((size_t)S);

    int active = S;
    if (!wide) {
        std::vector<uint8_t> iq((size_t)S * (size_t)W * (size_t)bps);
        while (active > 0) {
            /* 1. every live stream gets the samples its next step needs: [pos, pos + need) inside its window */
            for (int s = 0; s < S; s++) {
                Stream& z = st[(size_t)s];
                uint8_t* w = iq.data() + (size_t)s * (size_t)W * (size_t)bps;
                if (z.done) { buf_start[(size_t)s] = z.buf_start; continue; }
                if (z.pos > z.buf_start) {                            /* drop consumed samples: the window always starts at the receiver position */
                    const int64_t drop = std::min(z.pos - z.buf_start, z.have);
                    memmove(w, w + drop * bps, (size_t)(z.have - drop) * (size_t)bps);
                    z.buf_start += drop; z.have -= drop;
                    if (z.buf_start < z.pos && z.have == 0) {         /* the receiver skipped ahead of everything buffered */
                        if (fseek(z.in, (long)((z.pos - z.buf_start) * bps), SEEK_CUR) != 0) z.eof = true;
                        z.buf_start = z.pos;
                    }
                }
                const int64_t need_end = z.pos + (z.tracking ? need_track : z.acq_need);
                int64_t missing = std::min(need_end - (z.buf_start + z.have), W - z.have);
                if (missing > 0 && !z.eof) {
                    const size_t got = fread(w + z.have * bps, (size_t)bps, (size_t)missing, z.in);
                    z.have += (int64_t)got;
                    if ((int64_t)got < missing) z.eof = true;
                }
                if (z.buf_start + z.have < need_end && z.eof) { z.done = true; active--; }       /* not enough samples left for another frame */
                if (z.have < W) memset(w + z.have * bps, fmt == DABB_IQ_U8 ? 0x80 : 0, (size_t)(W - z.have) * (size_t)bps);   /* silence behind the data */
                buf_start[(size_t)s] = z.buf_start;
            }
            if (active <= 0) break;
            /* the ABI takes one window length for all streams.  Whether a stream really holds the samples its next step needs was decided
             * above from its own fill level (the rest of its window is silence); a finished stream is given a window far behind its position,
             * so the library reports DABB_FRAME_NEED_SAMPLES for it and touches nothing */
            int64_t buf_len = 0;                                      /* = what is copied to the device per stream: no more than the neediest stream asks for */
            for (int s = 0; s < S; s++) {
                const Stream& z = st[(size_t)s];
                if (z.done) buf_start[(size_t)s] = -(1LL << 40);
                else buf_len = std::max(buf_len, std::min<int64_t>(W, (z.pos - z.buf_start) + (z.tracking ? need_track : z.acq_need)));
            }
            if (!step(ctx, o, buf_start, reinterpret_cast<const float*>(iq.data()), 1, W, buf_len, fmt, tii, ber)) return 1;
            /* 2. per-stream results */
            for (int s = 0; s < S; s++) {
                Stream& z = st[(size_t)s];
                if (z.done) continue;
                if (!handle_result(ctx, z, s, o, tii, ber, TF)) { z.done = true; active--; }
            }
        }
    } else if (!run_wide(ctx, st, wf, rate, fmt, 0, buf_start,
                         [&](const float* win, int64_t out_len) { return step(ctx, o, buf_start, win, 0, W, out_len, DABB_IQ_CF32, tii, ber); },
                         [&](int s) { return handle_result(ctx, st[(size_t)s], s, o, tii, ber, TF); })) {
        return 1;
    }
    for (auto& z : st) {
        printf("%s frames=%ld fibs=%ld fib_crc_ok=%ld service=0x%X bitrate=%d logical_frames=%ld\n", z.name.c_str(), z.frames, z.fibs, z.fibs_ok, z.sid, z.bitrate, z.logical);
        if (z.in) fclose(z.in);
        fclose(z.fic); fclose(z.msc); fclose(z.rs); if (z.tii) fclose(z.tii); if (z.ber) fclose(z.ber); if (z.clk) fclose(z.clk); if (z.div) fclose(z.div); if (z.acq) fclose(z.acq);
        if (z.mer) {
            fclose(z.mer);
            if (!write_mer_profile(out + "/" + z.name + ".merprof", z.mer_prof)) { fprintf(stderr, "batch_decode: cannot write into %s\n", out.c_str()); return 1; }
        }
    }
    dabb_destroy(ctx);
    return 0;
}
