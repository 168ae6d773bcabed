/*
 * radio-receiver.cpp — host glue: the reference's RadioReceiver surface (backend/radio-receiver.h:52-116) implemented over
 * the C ABI of libdab_b200.so (include/dab_b200.h).  One worker thread replaces the reference's OFDMProcessor, OfdmDecoder
 * and DabAudio threads: it pulls samples from the InputInterface exactly like OFDMProcessor::getSamples
 * (backend/ofdm-processor.cpp:186-224), hands one frame's worth to dabb_process() (n_streams = 1) and turns the POD
 * results back into the reference's callbacks.  No signal processing happens here.
 *
 * The service database behind getServiceList / getComponents / getSubchannel lives in fig-db.h (FIG 0/0-0/3, 0/5, 0/9, 0/10, 0/14,
 * 0/17, FIG 1, FIG 2 with the reference FIBProcessor's acceptance rule); tests/test_figdb.py compares it with the compiled reference.
 */
#include "dab_api.h"
#include "fig-db.h"
#include "tii.h"
#include "../../include/dab_b200.h"

#include <atomic>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <stdexcept>
#include <thread>

/* ---------------------------------------------------------------------------------------------------------------- */
DABParams::DABParams(int mode) { setMode(mode); }
void DABParams::setMode(int mode)
{
    /* backend/dab-constants.cpp:347-402 */
    switch (mode) {
        case 1: dabMode = 1; L = 76; K = 1536; T_F = 196608; T_null = 2656; T_s = 2552; T_u = 2048; guardLength = 504; carrierDiff = 1000; break;
        case 2: dabMode = 2; L = 76; K = 384; T_null = 664; T_F = 49152; T_s = 638; T_u = 512; guardLength = 126; carrierDiff = 4000; break;
        case 3: dabMode = 3; L = 153; K = 192; T_F = 49152; T_null = 345; T_s = 319; T_u = 256; guardLength = 63; carrierDiff = 2000; break;
        case 4: dabMode = 4; L = 76; K = 768; T_F = 98304; T_null = 1328; T_s = 1276; T_u = 1024; guardLength = 252; carrierDiff = 2000; break;
        default: throw std::out_of_range("Unknown mode " + std::to_string(mode));
    }
}

using dabb_host::FigDb; using dabb_host::FigEvents;
static const int16_t* const kUepSize = dabb_host::kUepSizeCu;
static const int16_t kUepRate[64] = {32,32,32,32,32, 48,48,48,48,48, 56,56,56,56, 64,64,64,64,64, 80,80,80,80,80, 96,96,96,96,96, 112,112,112,112,
                                     128,128,128,128,128, 160,160,160,160,160, 192,192,192,192,192, 224,224,224,224,224, 256,256,256,256,256, 320,320,320, 384,384,384};

int Subchannel::bitrate() const
{
    const auto& ps = protectionSettings;
    if (ps.shortForm) return kUepRate[ps.uepTableIndex & 63];
    static const int da[5] = {0, 12, 8, 6, 4}, db[5] = {0, 27, 21, 18, 15};
    const int lv = (int)ps.eepLevel;
    if (lv < 1 || lv > 4) throw std::runtime_error("Unsupported protection");
    return ps.eepProfile == EEPProtectionProfile::EEP_A ? length / da[lv] * 8 : length / db[lv] * 32;   /* dab-constants.cpp:404-440 */
}
int Subchannel::numCU() const
{
    const auto& ps = protectionSettings;
    if (ps.shortForm) return kUepSize[ps.uepTableIndex & 63];
    const int b = bitrate();
    switch ((int)ps.eepLevel) {       /* dab-constants.cpp:442-477 */
        case 1: return ps.eepProfile == EEPProtectionProfile::EEP_A ? (b * 12) >> 3 : (b * 27) >> 5;
        case 2: return ps.eepProfile == EEPProtectionProfile::EEP_A ? b : (b * 21) >> 5;
        case 3: return ps.eepProfile == EEPProtectionProfile::EEP_A ? (b * 6) >> 3 : (b * 18) >> 5;
        case 4: return ps.eepProfile == EEPProtectionProfile::EEP_A ? b >> 1 : (b * 15) >> 5;
    }
    return -1;
}

const char* fftPlacementMethodToString(FFTPlacementMethod m)
{
    switch (m) { case FFTPlacementMethod::StrongestPeak: return "StrongestPeak"; case FFTPlacementMethod::EarliestPeakWithBinning: return "EarliestPeakWithBinning"; default: return "ThresholdBeforePeak"; }
}
const char* freqSyncMethodToString(FreqsyncMethod m)
{
    switch (m) { case FreqsyncMethod::GetMiddle: return "GetMiddle"; case FreqsyncMethod::CorrelatePRS: return "CorrelatePRS"; default: return "PatternOfZeros"; }
}

/* ---------------------------------------------------------------------------------------------------------------- */
struct RadioReceiver::Impl {
    RadioControllerInterface& rci; InputInterface& input; RadioReceiverOptions rro; DABParams params;
    dabb_ctx* ctx = nullptr;
    std::thread worker; std::atomic<bool> running{false};
    FigDb db;
    struct Slot { bool used = false; uint32_t sid = 0; ProgrammeHandlerInterface* handler = nullptr; FILE* dump = nullptr; int bitrate = 0; bool dabplus = false; };
    Slot slots[DABB_MAX_SUBCH];
    std::mutex slotMutex;
    /* The library context is not thread safe (one submitting thread per handle): EVERY dabb_* call on ctx is made under ctxMutex -
     * the worker's dabb_process / dabb_read_tap as well as the application thread's select / remove / reset / set_options.  Lock order
     * where both are needed: slotMutex, then ctxMutex. */
    std::mutex ctxMutex;
    bool synced = false; float snr = 0; int snrCount = 0; long sampleCnt = 0;
    /* OFDMProcessor::scanMode / attempts (ofdm-processor.cpp:258-262,351-355): set by restart(doScan) */
    std::atomic<bool> scanMode{false}; int failedSearches = 0;
    dabb_host::TiiAnalyzer tii;            /* RadioReceiverOptions::decodeTII (ofdm-processor.cpp:383-386,464-466) */

    /* the reference's enumerators (radio-receiver-options.h:35-64) -> DABB_PLACEMENT_* / DABB_FREQSYNC_* (0 = the reference's default) */
    static int placementOf(FFTPlacementMethod m) { return m == FFTPlacementMethod::StrongestPeak ? DABB_PLACEMENT_STRONGEST_PEAK : m == FFTPlacementMethod::EarliestPeakWithBinning ? DABB_PLACEMENT_EARLIEST_PEAK_WITH_BINNING : DABB_PLACEMENT_THRESHOLD_BEFORE_PEAK; }
    static int freqsyncOf(FreqsyncMethod m) { return m == FreqsyncMethod::GetMiddle ? DABB_FREQSYNC_GET_MIDDLE : m == FreqsyncMethod::CorrelatePRS ? DABB_FREQSYNC_CORRELATE_PRS : DABB_FREQSYNC_PATTERN_OF_ZEROS; }
    void applyOptions(const RadioReceiverOptions& o)
    {
        dabb_options op; memset(&op, 0, sizeof op);
        op.disable_coarse = o.disableCoarseCorrector ? 1 : 0; op.fft_placement = placementOf(o.fftPlacementMethod); op.freqsync_method = freqsyncOf(o.freqsyncMethod);
        op.decode_tii = o.decodeTII ? 1 : 0;
        std::lock_guard<std::mutex> l(ctxMutex);
        dabb_set_options(ctx, &op);
    }

    Impl(RadioControllerInterface& r, InputInterface& i, RadioReceiverOptions o, int mode) : rci(r), input(i), rro(o), params(mode)
    {
        if (mode != 1) throw std::runtime_error("B200 backend: only transmission mode I is implemented");
        dabb_config cfg; memset(&cfg, 0, sizeof cfg);
        cfg.abi_version = DABB_ABI_VERSION; cfg.device = 0; cfg.n_streams = 1; cfg.transmission_mode = 1; cfg.fft_mode = DABB_FFT_EXACT;
        cfg.disable_coarse = o.disableCoarseCorrector ? 1 : 0; cfg.fft_placement = placementOf(o.fftPlacementMethod); cfg.freqsync_method = freqsyncOf(o.freqsyncMethod);
        cfg.keep_taps = 1; cfg.n_subch_slots = DABB_MAX_SUBCH; cfg.max_subch_cu = 416; cfg.ofdm_groups = 25;
        if (dabb_create(&cfg, &ctx) != DABB_OK) throw std::runtime_error(std::string("B200 backend: ") + dabb_last_error(nullptr));
        applyOptions(o);
    }
    ~Impl() { stopWorker(); closeSlots(); if (ctx) dabb_destroy(ctx); }

    void closeSlots() { std::lock_guard<std::mutex> l(slotMutex); for (auto& s : slots) { if (s.dump) fclose(s.dump); s = Slot(); } }
    void stopWorker() { running = false; if (worker.joinable()) worker.join(); }

    /* pull exactly n samples like OFDMProcessor::getSamples (ofdm-processor.cpp:186-210); false = input failure / stop */
    bool pull(DSPCOMPLEX* dst, int64_t n)
    {
        while (n > 0 && running) {
            int32_t avail = input.getSamplesToRead();
            while (avail == 0 && running) {
                if (!input.is_ok()) return false;
                std::this_thread::sleep_for(std::chrono::microseconds(10));
                avail = input.getSamplesToRead();
            }
            if (!running) return false;
            /* never more than one symbol per call, like the reference (its n is an int16_t: T_u, T_s or T_null samples): CRAWFile
             * over-reports cf32 availability four times (raw_file.cpp:239-242) and its getSamples waits until the ring really holds
             * the request, which a large request can never be (256 KiB ring = 32 768 cf32 samples) */
            const int32_t want = (int32_t)std::min<int64_t>(n, std::min<int64_t>(avail, DABB_TS));
            const int32_t got = input.getSamples(dst, want);
            if (got <= 0) { if (!input.is_ok()) return false; continue; }
            dst += got; n -= got; sampleCnt += got;
        }
        return n == 0;
    }

    void run()
    {
        const int64_t TF = DABB_TF;
        const int64_t need_track = DABB_TU + (DABB_TU - 1) + 75LL * DABB_TS + DABB_TNULL;
        std::vector<DSPCOMPLEX> buf((size_t)(8 * TF));
        int64_t acq_need = 3 * TF;
        int64_t buf_start = 0, have = 0, pos = 0;     /* logical index of buf[0], samples held, receiver position */
        bool tracking = false;
        dabb_frame_result res; uint8_t fibs[12 * 32];
        std::vector<uint8_t> msc((size_t)DABB_MAX_SUBCH * 4 * 1152), sf((size_t)DABB_MAX_SUBCH * 5760);
        { std::lock_guard<std::mutex> l(ctxMutex); dabb_stream_reset(ctx, 0, 1, 0); }
        bool failed = false; failedSearches = 0;
        while (running) {
            /* acquisition needs the sLevel warm-up, the null search and a whole frame: 3 frames; tracking one frame */
            const int64_t need_end = pos + (tracking ? need_track : acq_need);
            if (pos > buf_start + TF) {            /* drop consumed samples */
                const int64_t drop = pos - buf_start;
                memmove(buf.data(), buf.data() + drop, (size_t)(have - drop) * sizeof(DSPCOMPLEX));
                buf_start += drop; have -= drop;
            }
            const int64_t missing = need_end - (buf_start + have);
            if (missing > 0) { if (!pull(buf.data() + have, missing)) { failed = running.load(); break; } have += missing; }
            dabb_io io; memset(&io, 0, sizeof io);
            io.iq = reinterpret_cast<const float*>(buf.data()); io.iq_is_host = 1; io.stride_samples = (int64_t)buf.size(); io.buf_start = &buf_start; io.buf_len = have;
            io.results = &res; io.fibs = fibs; io.msc = msc.data(); io.msc_stride = 1152; io.sf = sf.data(); io.sf_stride = 5760;
            int prc; { std::lock_guard<std::mutex> l(ctxMutex); prc = dabb_process(ctx, &io); }
            if (prc != DABB_OK) { rci.onMessage(message_level_t::Error, "B200 backend", dabb_last_error(ctx)); failed = true; break; }
            pos = res.next_pos;
            /* every entry into the reference's notSynced state but the first follows a failed null search or a failed SyncOnPhase:
             * with doScan the sixth entry reports "no signal", the first successful SyncOnPhase "signal" (ofdm-processor.cpp:258-262,351-355) */
            failedSearches += res.acq_failed + (res.status == DABB_FRAME_NO_SYNC ? 1 : 0);
            if (scanMode.load() && res.status != DABB_FRAME_DECODED && failedSearches >= 5) { rci.onSignalPresence(false); scanMode = false; failedSearches = 0; }
            if (res.status == DABB_FRAME_DECODED) {
                if (scanMode.load()) { rci.onSignalPresence(true); scanMode = false; failedSearches = 0; }
                if (!synced) { synced = true; rci.onSyncChange(true); }
                tracking = true; acq_need = 3 * TF;
                dispatch(res, fibs, msc.data(), sf.data());
            } else if (res.status == DABB_FRAME_NO_SYNC) {
                if (synced) { synced = false; rci.onSyncChange(false); }
                tracking = false;
                {   /* the impulse response is handed over after every findIndex, found or not (ofdm-processor.cpp:341-345) */
                    std::vector<float> cir(DABB_TU);
                    int trc; { std::lock_guard<std::mutex> l(ctxMutex); trc = dabb_read_tap(ctx, 1, cir.data(), cir.size() * sizeof(float)); }
                    if (trc == DABB_OK) rci.onNewImpulseResponse(std::move(cir));
                }
            } else if (res.status == DABB_FRAME_ACQUIRING) {
                if (synced) { synced = false; rci.onSyncChange(false); }
                tracking = false;
                /* the null search did not finish inside the samples at hand: give it one more frame, and after five frames
                 * without a null start over two frames further on */
                /* the search keeps its progress (position, level, oscillator phase) between calls: just keep feeding it */
                acq_need = 3 * TF;
            } else {
                /* DABB_FRAME_NEED_SAMPLES cannot happen (the loop above always supplies the samples a frame needs); if the library and the
                 * glue ever disagree about that number, stop instead of spinning */
                rci.onMessage(message_level_t::Error, "B200 backend", "frame needs more samples than the glue supplied");
                failed = true; break;
            }
        }
        if (failed) { running = false; rci.onInputFailure(); }
    }

    void dispatch(const dabb_frame_result& r, const uint8_t* fibs, const uint8_t* msc, const uint8_t* sf)
    {
        /* OfdmDecoder::processPRS: snr = 0.7 snr + 0.3 get_snr, reported every 10th frame (ofdm-decoder.cpp:156-160) */
        snr = 0.7f * snr + 0.3f * (float)r.snr_raw;
        if (++snrCount > 10) { rci.onSNR(snr); snrCount = 0; }
        if (sampleCnt > INPUT_RATE / 5) { rci.onFrequencyCorrectorChange(r.fine_corr, r.coarse_corr); sampleCnt = 0; }   /* ofdm-processor.cpp:218-223 */
        {
            std::vector<float> cir(DABB_TU);
            int trc; { std::lock_guard<std::mutex> l(ctxMutex); trc = dabb_read_tap(ctx, 1, cir.data(), cir.size() * sizeof(float)); }
            if (trc == DABB_OK) rci.onNewImpulseResponse(std::move(cir));
        }
        {   /* OfdmDecoder hands over r1 of every 96th carrier once per frame (ofdm-decoder.cpp:119-125,216-218) */
            std::vector<DSPCOMPLEX> pts((size_t)(DABB_L - 1) * DABB_K / 96);
            int trc; { std::lock_guard<std::mutex> l(ctxMutex); trc = dabb_read_tap(ctx, 2, pts.data(), pts.size() * sizeof(DSPCOMPLEX)); }
            if (trc == DABB_OK) rci.onConstellationPoints(std::move(pts));
        }
        {   /* the null symbol that follows the frame, as read with the corrected oscillator (ofdm-processor.cpp:462-469) */
            std::vector<DSPCOMPLEX> nul(DABB_TNULL);
            int trc; { std::lock_guard<std::mutex> l(ctxMutex); trc = dabb_read_tap(ctx, 3, nul.data(), nul.size() * sizeof(DSPCOMPLEX)); }
            if (trc == DABB_OK) rci.onNewNullSymbol(std::move(nul));
        }
        if (rro.decodeTII) {
            /* TIIDecoder::pushSymbols(nullSymbol, prs): the two transforms come from the GPU (tap 4), the pattern analysis runs here */
            std::vector<complexf> spec(2 * DABB_TU);
            int trc; { std::lock_guard<std::mutex> l(ctxMutex); trc = dabb_read_tap(ctx, 4, spec.data(), spec.size() * sizeof(complexf)); }
            if (trc == DABB_OK) tii.process(spec.data() + DABB_TU, spec.data(), [this](tii_measurement_t&& m) { rci.onTIIMeasurement(std::move(m)); });
        }
        for (int f = 0; f < 12; f++) {
            uint8_t bits[256];
            for (int i = 0; i < 256; i++) bits[i] = (fibs[32 * f + (i >> 3)] >> (7 - (i & 7))) & 1;
            const bool ok = (r.fib_crc_mask >> f) & 1;
            rci.onFIBDecodeSuccess(ok, bits);
            if (ok) {
                FigEvents ev;
                db.parseFib(fibs + 32 * f, ev);
                for (const auto& e : ev.list) {          /* the FIG-derived callbacks, in the order the FIGs appear (fib-processor.cpp) */
                    switch (e.kind) {
                        case FigEvents::NewEnsemble: rci.onNewEnsemble((uint16_t)e.id); break;
                        case FigEvents::ServiceDetected: rci.onServiceDetected(e.id); break;
                        case FigEvents::EnsembleLabel: { DabLabel l; { std::lock_guard<std::mutex> g(db.m); l = db.ensLabel; } rci.onSetEnsembleLabel(l); break; }
                        case FigEvents::RestartService: rci.onRestartService(); break;
                        case FigEvents::DateTime: { dab_date_time_t t; { std::lock_guard<std::mutex> g(db.m); t = db.dateTime; } rci.onDateTimeUpdate(t); break; }
                    }
                }
            }
        }
        std::lock_guard<std::mutex> l(slotMutex);
        for (int k = 0; k < DABB_MAX_SUBCH; k++) {
            Slot& s = slots[k];
            if (!s.used) continue;
            const int flen = 3 * s.bitrate;
            for (int c = 4 - r.n_logical[k]; c < 4; c++) {
                const uint8_t* fr = msc + ((size_t)k * 4 + c) * 1152;
                if (s.dump) fwrite(fr, flen, 1, s.dump);                 /* DecoderAdapter::addtoFrame dump (decoder_adapter.cpp:71-73) */
                if (s.handler) s.handler->onFrameErrors(0);
            }
            for (int e = 0; e < r.n_rs_events[k]; e++)
                if (s.handler) s.handler->onRsErrors((r.rs_uncorr_mask[k] >> e) & 1, r.rs_corr[k][e]);   /* DecoderAdapter::FECInfo */
            if (r.sf_ready[k] && s.handler) s.handler->onSuperframe(sf + (size_t)k * 5760, 5 * flen, r.sf_au_count[k], r.sf_au_crc_mask[k]);
        }
    }

    bool play(ProgrammeHandlerInterface& handler, const std::string& dumpFileName, const Service& srv, bool unique)
    {
        Subchannel sub; AudioServiceComponentType at = AudioServiceComponentType::Unknown;
        {
            std::lock_guard<std::mutex> l(db.m);
            for (const auto& sc : db.components) {
                if (sc.SId != srv.serviceId || sc.transportMode() != TransportMode::Audio) continue;
                if (sc.subchannelId < 0 || sc.subchannelId >= 64 || !db.subch[sc.subchannelId].valid()) continue;
                if (sc.audioType() == AudioServiceComponentType::Unknown) continue;
                sub = db.subch[sc.subchannelId]; at = sc.audioType();
                break;
            }
        }
        if (!sub.valid()) return false;
        std::lock_guard<std::mutex> l(slotMutex);
        std::lock_guard<std::mutex> lc(ctxMutex);          /* the worker may be inside dabb_process: wait for the frame to finish */
        if (unique) for (int k = 0; k < DABB_MAX_SUBCH; k++) if (slots[k].used) { dabb_remove_subchannel(ctx, 0, 1, k); if (slots[k].dump) fclose(slots[k].dump); slots[k] = Slot(); }
        for (int k = 0; k < DABB_MAX_SUBCH; k++) if (slots[k].used && slots[k].sid == srv.serviceId) return true;   /* already decoding (msc-handler.cpp:69-74) */
        int k = 0;
        while (k < DABB_MAX_SUBCH && slots[k].used) k++;
        if (k == DABB_MAX_SUBCH) return false;
        dabb_subchannel sc; memset(&sc, 0, sizeof sc);
        sc.subch_id = sub.subChId; sc.start_cu = sub.startAddr; sc.length_cu = sub.length; sc.bitrate = sub.bitrate();
        sc.short_form = sub.protectionSettings.shortForm; sc.uep_level = sub.protectionSettings.uepLevel;
        sc.eep_profile_a = sub.protectionSettings.eepProfile == EEPProtectionProfile::EEP_A; sc.eep_level = (int)sub.protectionSettings.eepLevel;
        sc.dabplus = at == AudioServiceComponentType::DABPlus;
        if (dabb_select_subchannel(ctx, 0, 1, k, &sc) != DABB_OK) { rci.onMessage(message_level_t::Error, "B200 backend", dabb_last_error(ctx)); return false; }
        Slot& s = slots[k]; s.used = true; s.sid = srv.serviceId; s.handler = &handler; s.bitrate = sc.bitrate; s.dabplus = sc.dabplus;
        if (!dumpFileName.empty()) s.dump = fopen(dumpFileName.c_str(), "wb");
        return true;
    }
};

RadioReceiver::RadioReceiver(RadioControllerInterface& rci, InputInterface& input, RadioReceiverOptions rro, int transmission_mode)
{
    DABParams check(transmission_mode);   /* throws std::out_of_range like the reference for a bad mode */
    (void)check;
    d.reset(new Impl(rci, input, rro, transmission_mode));
}
RadioReceiver::~RadioReceiver() {}

void RadioReceiver::restart(bool doScan)
{
    d->stopWorker(); d->closeSlots(); d->db.clear(); d->tii.clear();
    d->scanMode = doScan;                                    /* OFDMProcessor::set_scanMode (radio-receiver.cpp:84) */
    { std::lock_guard<std::mutex> l(d->ctxMutex); for (int k = 0; k < DABB_MAX_SUBCH; k++) dabb_remove_subchannel(d->ctx, 0, 1, k); }
    d->input.restart();
    d->synced = false; d->running = true;
    d->worker = std::thread(&Impl::run, d.get());
}
void RadioReceiver::restart_decoder()
{
    d->closeSlots(); d->db.clear();
    std::lock_guard<std::mutex> l(d->ctxMutex);
    for (int k = 0; k < DABB_MAX_SUBCH; k++) dabb_remove_subchannel(d->ctx, 0, 1, k);
}
void RadioReceiver::stop()
{
    d->stopWorker(); d->closeSlots(); d->db.clear();
}
void RadioReceiver::setReceiverOptions(const RadioReceiverOptions rro) { d->rro = rro; d->applyOptions(rro); }
bool RadioReceiver::playSingleProgramme(ProgrammeHandlerInterface& h, const std::string& dump, const Service& s) { return d->play(h, dump, s, true); }
bool RadioReceiver::addServiceToDecode(ProgrammeHandlerInterface& h, const std::string& dump, const Service& s) { return d->play(h, dump, s, false); }
bool RadioReceiver::removeServiceToDecode(const Service& s)
{
    std::lock_guard<std::mutex> l(d->slotMutex);
    for (int k = 0; k < DABB_MAX_SUBCH; k++)
        if (d->slots[k].used && d->slots[k].sid == s.serviceId) {
            { std::lock_guard<std::mutex> lc(d->ctxMutex); dabb_remove_subchannel(d->ctx, 0, 1, k); }
            if (d->slots[k].dump) fclose(d->slots[k].dump);
            d->slots[k] = Impl::Slot();
            return true;
        }
    return false;
}
uint16_t RadioReceiver::getEnsembleId(void) const { std::lock_guard<std::mutex> l(d->db.m); return d->db.eid; }
uint8_t RadioReceiver::getEnsembleEcc(void) const { std::lock_guard<std::mutex> l(d->db.m); return d->db.ecc; }
DabLabel RadioReceiver::getEnsembleLabel(void) const { std::lock_guard<std::mutex> l(d->db.m); return d->db.ensLabel; }
std::vector<Service> RadioReceiver::getServiceList(void) const
{
    std::lock_guard<std::mutex> l(d->db.m);
    return d->db.services;
}
Service RadioReceiver::getService(uint32_t sId) const
{
    std::lock_guard<std::mutex> l(d->db.m);
    for (const auto& s : d->db.services) if (s.serviceId == sId) return s;
    return Service(0);
}
std::list<ServiceComponent> RadioReceiver::getComponents(const Service& s) const
{
    std::lock_guard<std::mutex> l(d->db.m);
    std::list<ServiceComponent> out;
    for (const auto& c : d->db.components) if (c.SId == s.serviceId) out.push_back(c);
    return out;
}
bool RadioReceiver::serviceHasAudioComponent(const Service& s) const
{
    for (const auto& sc : getComponents(s))
        if (sc.transportMode() == TransportMode::Audio && sc.audioType() != AudioServiceComponentType::Unknown) return true;
    return false;
}
Subchannel RadioReceiver::getSubchannel(const ServiceComponent& sc) const
{
    std::lock_guard<std::mutex> l(d->db.m);
    return d->db.subch.at(sc.subchannelId);          /* throws std::out_of_range like the reference's vector::at (fib-processor.cpp:1313) */
}
DABParams& RadioReceiver::getParams() { return d->params; }
RadioReceiverStats RadioReceiver::getReceiverStats() const
{
    RadioReceiverStats s;
    std::lock_guard<std::mutex> l(d->db.m);
    s.timeLastFCT0Frame = d->db.timeLastFCT0Frame;          /* radio-receiver.cpp:225-230 */
    return s;
}

/* test hook: the TII analysis of n frames of spectra (natural bin order, 2048 complex floats each); out: 4 floats per measurement
 * (comb, pattern, delay_samples, error) in the order of the onTIIMeasurement callbacks; returns their number */
extern "C" int welle_b200_tii_run(const float* null_specs, const float* prs_specs, int n, float* out, int cap)
{
    dabb_host::TiiAnalyzer an; int k = 0;
    for (int f = 0; f < n; f++)
        an.process(reinterpret_cast<const complexf*>(null_specs) + (size_t)f * 2048, reinterpret_cast<const complexf*>(prs_specs) + (size_t)f * 2048,
                   [&](tii_measurement_t&& m) { if (k < cap) { out[4 * k] = (float)m.comb; out[4 * k + 1] = (float)m.pattern; out[4 * k + 2] = (float)m.delay_samples; out[4 * k + 3] = m.error; } k++; });
    return k;
}

/* test hook: the same analysis with the frame of every measurement; out: 5 floats per measurement (frame index 0 .. n-1, comb, pattern,
 * delay_samples, error) in the order of the onTIIMeasurement callbacks; returns their number */
extern "C" int welle_b200_tii_run_framed(const float* null_specs, const float* prs_specs, int n, float* out, int cap)
{
    dabb_host::TiiAnalyzer an; int k = 0;
    for (int f = 0; f < n; f++)
        an.process(reinterpret_cast<const complexf*>(null_specs) + (size_t)f * 2048, reinterpret_cast<const complexf*>(prs_specs) + (size_t)f * 2048,
                   [&](tii_measurement_t&& m) {
                       if (k < cap) { float* o = out + 5 * k; o[0] = (float)f; o[1] = (float)m.comb; o[2] = (float)m.pattern; o[3] = (float)m.delay_samples; o[4] = m.error; }
                       k++; });
    return k;
}

/* test hook: the phase-error table's container as TIIDecoder::analyse_phase uses it (tii-decoder.cpp:344-381): a
 * std::unordered_map<float, uint64_t> filled for err = -4 .. 499 in that order, after `clears` earlier fill + clear() cycles, with
 * value sums[err + 4]; keys_out[504]: the keys in iteration order; returns the key std::min_element picks */
extern "C" int welle_b200_tii_map_argmin(const uint32_t* sums, int clears, int32_t* keys_out)
{
    std::unordered_map<float, uint64_t> m;
    for (int c = 0; c <= clears; c++) {
        if (c) m.clear();
        for (int err = -4; err < 500; err++) m[(float)err] += c == clears ? sums[err + 4] : 0;
    }
    int i = 0;
    for (const auto& kv : m) keys_out[i++] = (int32_t)kv.first;
    const auto best = std::min_element(m.begin(), m.end(), [](const std::pair<const float, uint64_t>& a, const std::pair<const float, uint64_t>& b) { return a.second < b.second; });
    return (int)best->first;
}

/* test hook: feeds n FIBs (32 bytes each) to a fresh service database and writes its text dump (callbacks first) */
extern "C" int welle_b200_figdb_dump(const uint8_t* fibs, int n, char* out, int cap)
{
    FigDb db; std::string cb;
    for (int i = 0; i < n; i++) {
        FigEvents ev; db.parseFib(fibs + 32 * i, ev);
        for (const auto& e : ev.list) {
            char t[64];
            static const char* const names[] = {"newEnsemble", "serviceDetected", "ensembleLabel", "restartService", "dateTime"};
            snprintf(t, sizeof t, "cb %s %u\n", names[e.kind], e.kind == FigEvents::DateTime || e.kind == FigEvents::RestartService ? 0u : e.id); cb += t;
        }
    }
    const std::string s = cb + db.dump();
    if ((int)s.size() + 1 > cap) return -(int)s.size() - 1;
    memcpy(out, s.c_str(), s.size() + 1);
    return (int)s.size();
}
