/*
 * batch_decode.cpp — native batch driver over the C ABI: decodes many RAW IQ recordings at once, one stream per file (or per ensemble of a
 * wideband file, --rate), on one GPU.
 *
 *   batch_decode [--format cf32|u8|s8|s16le|s16be] [--device N] [--coarse] [--tii] [--ber] [--rate HZ --offset HZ[,HZ...]] --out DIR file1 [file2 ...]
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
 * --rate HZ --offset HZ[,HZ...]: every file is a wideband recording at HZ samples/s (any rate dabb_chan_create accepts) and every offset
 * (Hz from the tuned frequency, may be negative) is one stream of the batch, decoded by a channelizer of the same context (dabb_chan_*):
 * outputs go to DIR/<name>@<offset>.{fic,msc,rs} (and .tii / .ber), in the formats above.  The streams of one file progress
 * independently (their own position, acquisition and end of file).  Every step channelizes exactly each stream's [pos, pos + need) of its
 * 2.048 Msps axis into that stream's device window and then runs dabb_process on the windows; the channelizer keeps no state, so nothing
 * is shifted on the device, and the host keeps per file only the input span its live streams still need.
 *
 * Sample formats are the RAW-file formats of CRAWFile (input/raw_file.cpp:324-366); they are shipped as they are and converted on
 * the device.
 */
#include "dab_api.h"
#include "fig-db.h"
#include "../../include/dab_b200.h"

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

namespace {

struct Stream {
    std::string path, name; FILE* in = nullptr; FILE* fic = nullptr; FILE* msc = nullptr; FILE* rs = nullptr; FILE* tii = nullptr; FILE* ber = nullptr;
    int64_t buf_start = 0, have = 0, pos = 0, acq_need = 0;      /* logical sample indices; `have` samples are buffered from buf_start */
    bool tracking = false, eof = false, done = false;
    std::unique_ptr<dabb_host::FigDb> db{new dabb_host::FigDb()};
    int slot = -1; int bitrate = 0; uint32_t sid = 0;
    long frames = 0, fibs_ok = 0, fibs = 0, logical = 0;
    int file = -1; int64_t offset = 0;                            /* wideband mode: the recording and the channel's offset in Hz */
};

/* wideband mode: one recording, read into a host buffer that holds input samples [first, first + have) (silence past the end of the
 * file up to `len`), and the channelizer of its streams */
struct Wide {
    std::string path; FILE* in = nullptr; std::vector<uint8_t> buf; int64_t first = 0, have = 0; bool eof = false;
    std::vector<int> streams; dabb_chan* ch = nullptr;
};

struct Outputs {
    std::vector<dabb_frame_result> res; std::vector<uint8_t> fibs, msc, sf; std::vector<dabb_tii_result> tres; std::vector<dabb_ber_result> bres;
};

/* what one dabb_process step returned for stream s: files, service database, tuning, the receiver position; false = the stream ended */
bool handle_result(dabb_ctx* ctx, Stream& z, int s, const Outputs& o, bool tii, bool ber, int64_t TF)
{
    const dabb_frame_result& r = o.res[(size_t)s];
    if (tii)
        for (int i = 0; i < o.tres[(size_t)s].count; i++) {
            const auto& m = o.tres[(size_t)s].m[i];
            fprintf(z.tii, "%d %d %d %.1f\n", m.comb, m.pattern, m.delay_samples, m.error);
        }
    if (r.status == DABB_FRAME_NEED_SAMPLES) return false;      /* cannot happen for a live stream: stop it rather than spin */
    z.pos = r.next_pos;
    if (r.status == DABB_FRAME_NO_SYNC) { z.tracking = false; return true; }
    if (r.status == DABB_FRAME_ACQUIRING) {
        z.tracking = false;
        if (z.acq_need < 5 * TF) z.acq_need += TF;
        else { z.pos += 2 * TF; z.acq_need = 3 * TF; dabb_stream_reset(ctx, s, 1, z.pos); }
        return !z.eof;
    }
    z.tracking = true; z.acq_need = 3 * TF; z.frames++;
    if (ber) {
        const dabb_ber_result& b = o.bres[(size_t)s];
        fprintf(z.ber, "%d %d %d %d %d %d %d\n", b.fic_bits, b.fic_errors, b.fic_erasures, b.subch[0].codewords, b.subch[0].bits, b.subch[0].errors, b.subch[0].erasures);
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

int bytes_per_sample(int fmt) { return fmt == DABB_IQ_CF32 ? 8 : (fmt == DABB_IQ_U8 || fmt == DABB_IQ_S8) ? 2 : 4; }

} // namespace

int main(int argc, char** argv)
{
    int fmt = DABB_IQ_CF32, device = 0; bool coarse = false, tii = false, ber = false; std::string out;
    int64_t rate = 0; std::vector<int64_t> offsets;
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
        else if (a == "--rate" && i + 1 < argc) rate = atoll(argv[++i]);
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
    if (out.empty() || files.empty() || (rate > 0) != !offsets.empty()) {
        fprintf(stderr, "usage: batch_decode [--format cf32|u8|s8|s16le|s16be] [--device N] [--coarse] [--tii] [--ber] [--rate HZ --offset HZ[,HZ...]] --out DIR file...\n");
        return 2;
    }
    const bool wide = rate > 0;

    const int S = (int)(wide ? files.size() * offsets.size() : files.size());
    const int64_t TF = DABB_TF, W = 6 * TF;                       /* per-stream window capacity in samples */
    const int64_t need_track = DABB_TU + (DABB_TU - 1) + 75LL * DABB_TS + DABB_TNULL;
    const int bps = bytes_per_sample(fmt);

    dabb_config cfg; memset(&cfg, 0, sizeof cfg);
    cfg.abi_version = DABB_ABI_VERSION; cfg.device = device; cfg.n_streams = S; cfg.transmission_mode = 1; cfg.fft_mode = DABB_FFT_EXACT;
    cfg.disable_coarse = coarse ? 0 : 1; cfg.n_subch_slots = DABB_MAX_SUBCH; cfg.max_subch_cu = 416;
    dabb_ctx* ctx = nullptr;
    if (dabb_create(&cfg, &ctx) != DABB_OK) { fprintf(stderr, "batch_decode: %s\n", dabb_last_error(nullptr)); return 1; }
    if (tii || ber) {
        dabb_options op; memset(&op, 0, sizeof op);
        op.disable_coarse = cfg.disable_coarse; op.decode_tii = tii; op.count_bit_errors = ber;
        if (dabb_set_options(ctx, &op) != DABB_OK) { fprintf(stderr, "batch_decode: %s\n", dabb_last_error(ctx)); return 1; }
    }

    std::vector<Stream> st((size_t)S);
    std::vector<Wide> wf(wide ? files.size() : 0);
    for (int s = 0; s < S; s++) {
        Stream& z = st[(size_t)s];
        const int f = wide ? s / (int)offsets.size() : s;
        z.path = files[(size_t)f];
        const size_t slash = z.path.find_last_of('/');
        z.name = slash == std::string::npos ? z.path : z.path.substr(slash + 1);
        if (wide) {
            z.file = f; z.offset = offsets[(size_t)(s % (int)offsets.size())];
            z.name += "@" + std::to_string(z.offset);
            wf[(size_t)f].streams.push_back(s);
        } else {
            z.in = fopen(z.path.c_str(), "rb");
            if (!z.in) { fprintf(stderr, "batch_decode: cannot open %s\n", z.path.c_str()); return 1; }
        }
        z.fic = fopen((out + "/" + z.name + ".fic").c_str(), "wb"); z.msc = fopen((out + "/" + z.name + ".msc").c_str(), "wb"); z.rs = fopen((out + "/" + z.name + ".rs").c_str(), "w");
        if (tii) z.tii = fopen((out + "/" + z.name + ".tii").c_str(), "w");
        if (ber) z.ber = fopen((out + "/" + z.name + ".ber").c_str(), "w");
        if (!z.fic || !z.msc || !z.rs || (tii && !z.tii) || (ber && !z.ber)) { fprintf(stderr, "batch_decode: cannot write into %s\n", out.c_str()); return 1; }
        z.acq_need = 3 * TF;
    }
    dabb_stream_reset(ctx, 0, S, 0);

    Outputs o;
    o.res.resize((size_t)S); o.fibs.resize((size_t)S * 12 * 32); o.msc.resize((size_t)S * DABB_MAX_SUBCH * 4 * 1152); o.sf.resize((size_t)S * DABB_MAX_SUBCH * 5760);
    o.tres.resize(tii ? (size_t)S : 0); o.bres.resize(ber ? (size_t)S : 0);
    std::vector<int64_t> buf_start((size_t)S);
    auto step = [&](const float* iq, int iq_is_host, int64_t stride, int64_t buf_len, int iq_format) -> bool {
        dabb_io io; memset(&io, 0, sizeof io);
        io.iq = iq; io.iq_is_host = iq_is_host; io.stride_samples = stride; io.buf_start = buf_start.data(); io.buf_len = buf_len;
        io.results = o.res.data(); io.fibs = o.fibs.data(); io.msc = o.msc.data(); io.msc_stride = 1152; io.sf = o.sf.data(); io.sf_stride = 5760; io.iq_format = iq_format;
        if (dabb_process(ctx, &io) != DABB_OK) { fprintf(stderr, "batch_decode: %s\n", dabb_last_error(ctx)); return false; }
        if (tii && dabb_read_tap(ctx, 9, o.tres.data(), o.tres.size() * sizeof(dabb_tii_result)) != DABB_OK) { fprintf(stderr, "batch_decode: %s\n", dabb_last_error(ctx)); return false; }
        if (ber && dabb_read_tap(ctx, 10, o.bres.data(), o.bres.size() * sizeof(dabb_ber_result)) != DABB_OK) { fprintf(stderr, "batch_decode: %s\n", dabb_last_error(ctx)); return false; }
        return true;
    };

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
            if (!step(reinterpret_cast<const float*>(iq.data()), 1, W, buf_len, fmt)) return 1;
            /* 2. per-stream results */
            for (int s = 0; s < S; s++) {
                Stream& z = st[(size_t)s];
                if (z.done) continue;
                if (!handle_result(ctx, z, s, o, tii, ber, TF)) { z.done = true; active--; }
            }
        }
    } else {
        /* one channelizer per recording; every stream has a device window of W samples of its 2.048 Msps axis */
        for (size_t f = 0; f < wf.size(); f++) {
            Wide& w = wf[f];
            w.path = files[f];
            w.in = fopen(w.path.c_str(), "rb");
            if (!w.in) { fprintf(stderr, "batch_decode: cannot open %s\n", w.path.c_str()); return 1; }
            const std::vector<int32_t> input_of(offsets.size(), 0);
            dabb_chan_config cc; memset(&cc, 0, sizeof cc);
            cc.rate_hz = rate; cc.iq_format = fmt; cc.n_inputs = 1; cc.n_channels = (int32_t)offsets.size();
            cc.input_of_channel = input_of.data(); cc.offset_hz = offsets.data();
            if (dabb_chan_create(ctx, &cc, &w.ch) != DABB_OK) { fprintf(stderr, "batch_decode: %s\n", dabb_last_error(ctx)); return 1; }
            int64_t end0 = 0;                                         /* the recording is input [0, ...); silence before it */
            dabb_chan_input_range(w.ch, 0, 1, &w.first, &end0);
        }
        void* win = nullptr;
        if (dabb_dev_alloc(ctx, (size_t)S * (size_t)W * 8, &win) != DABB_OK) { fprintf(stderr, "batch_decode: %s\n", dabb_last_error(ctx)); return 1; }
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
                /* a stream ends when the recording cannot give the samples its own next step needs */
                bool ended = false;
                for (int s : w.streams) {
                    Stream& z = st[(size_t)s];
                    if (z.done) continue;
                    z.eof = w.eof;
                    int64_t a, b;
                    dabb_chan_input_range(w.ch, z.pos, z.tracking ? need_track : z.acq_need, &a, &b);
                    if (w.eof && b > w.first + w.have) { z.done = true; active--; ended = true; }
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
                if (dabb_channelize(w.ch, &cio) != DABB_OK) { fprintf(stderr, "batch_decode: %s\n", dabb_last_error(ctx)); return 1; }
            }
            if (active <= 0) break;
            for (int s = 0; s < S; s++) buf_start[(size_t)s] = st[(size_t)s].done ? -(1LL << 40) : st[(size_t)s].pos;
            if (!step(static_cast<const float*>(win), 0, W, out_len, DABB_IQ_CF32)) return 1;
            for (int s = 0; s < S; s++) {
                Stream& z = st[(size_t)s];
                if (z.done) continue;
                if (!handle_result(ctx, z, s, o, tii, ber, TF)) { z.done = true; active--; }
            }
        }
        for (Wide& w : wf) { dabb_chan_destroy(w.ch); fclose(w.in); }
        dabb_dev_free(ctx, win);
    }
    for (auto& z : st) {
        printf("%s frames=%ld fibs=%ld fib_crc_ok=%ld service=0x%X bitrate=%d logical_frames=%ld\n", z.name.c_str(), z.frames, z.fibs, z.fibs_ok, z.sid, z.bitrate, z.logical);
        if (z.in) fclose(z.in);
        fclose(z.fic); fclose(z.msc); fclose(z.rs); if (z.tii) fclose(z.tii); if (z.ber) fclose(z.ber);
    }
    dabb_destroy(ctx);
    return 0;
}
