/*
 * mock_dab_b200_chan.cpp — TEST DOUBLE of the C ABI with the wideband channelizer (dabb_chan_*, dabb_channelize) and the device memory
 * helpers, for running batch_decode --rate / --offset on a machine without a GPU (tests/test_chan_batch_mock.py).  NOT part of the
 * product.
 *
 * It is the test double of tests/mock_backend/mock_dab_b200.c, included unchanged: dabb_process hands out the oracle's frame records of
 * the 2.048 Msps files named by $DABB_MOCK_IQ, one per stream.  The channelizer entry points are real: they check their arguments like
 * the library and compute every output with the host build of welle.io_b200/csrc/chan_core.cuh, into "device" memory that is host memory
 * here (dabb_dev_alloc = malloc).  Every call is logged to $DABB_MOCK_CHAN_LOG (if set): one line "out_start... out_len in_start in_len"
 * per dabb_channelize, so that a test can check which ranges the driver asked for.
 */
extern "C" {
#include "mock_dab_b200.c"
}
#include "../../welle.io_b200/csrc/chan_core.cuh"

#include <algorithm>
#include <cmath>
#include <vector>

using namespace dabb_channel;

struct dabb_chan {
    dabb_ctx* ctx;
    Geometry g;
    int fmt, n_in, n_ch;
    std::vector<int32_t> input_of;
    std::vector<int64_t> fmod;
    std::vector<float> packed;
};

static int chan_range(const dabb_chan* ch, int64_t out_start, int64_t out_len, int64_t& first, int64_t& end)
{
    if (out_start < 0 || out_len < 1 || out_len > MAX_OUT_INDEX || out_start > MAX_OUT_INDEX - out_len) return DABB_E_ARG;
    first = last_input(out_start, ch->g.L, ch->g.M) - ch->g.T + 1;
    end = last_input(out_start + out_len - 1, ch->g.L, ch->g.M) + 1;
    return DABB_OK;
}

extern "C" {

int dabb_dev_alloc(dabb_ctx* c, size_t bytes, void** out) { if (!c || !out) return DABB_E_ARG; *out = malloc(bytes ? bytes : 16); return *out ? DABB_OK : DABB_E_NOMEM; }
int dabb_dev_free(dabb_ctx* c, void* p) { if (!c) return DABB_E_ARG; free(p); return DABB_OK; }

int dabb_chan_create(dabb_ctx* ctx, const dabb_chan_config* cfg, dabb_chan** out)
{
    if (!ctx || !cfg || !out) return DABB_E_ARG;
    *out = nullptr;
    Geometry g{};
    if (geometry(cfg->rate_hz, g) != DABB_OK) return DABB_E_UNSUPPORTED;
    if (cfg->iq_format < DABB_IQ_CF32 || cfg->iq_format > DABB_IQ_S16BE || cfg->n_inputs < 1 || cfg->n_inputs > MAX_CHANNELS || cfg->n_channels < 1
        || cfg->n_channels > MAX_CHANNELS || !cfg->input_of_channel || !cfg->offset_hz) return DABB_E_ARG;
    for (int c = 0; c < cfg->n_channels; c++)
        if (cfg->input_of_channel[c] < 0 || cfg->input_of_channel[c] >= cfg->n_inputs || !offset_ok(g.R, cfg->offset_hz[c])) return DABB_E_ARG;
    dabb_chan* ch = new dabb_chan{ctx, g, cfg->iq_format, cfg->n_inputs, cfg->n_channels, {}, {}, {}};
    ch->input_of.assign(cfg->input_of_channel, cfg->input_of_channel + cfg->n_channels);
    for (int c = 0; c < cfg->n_channels; c++) ch->fmod.push_back(floor_mod(cfg->offset_hz[c], g.R));
    std::vector<float> h((size_t)g.L * g.T);
    design_taps(g, h.data());
    ch->packed.resize((size_t)g.L * g.TP);
    pack_taps(g, h.data(), ch->packed.data());
    *out = ch;
    return DABB_OK;
}

void dabb_chan_destroy(dabb_chan* ch) { delete ch; }

int dabb_chan_input_range(const dabb_chan* ch, int64_t out_start, int64_t out_len, int64_t* in_first, int64_t* in_end)
{
    if (!ch || !in_first || !in_end) return DABB_E_ARG;
    int64_t f, e;
    if (chan_range(ch, out_start, out_len, f, e)) return DABB_E_ARG;
    *in_first = f; *in_end = e;
    return DABB_OK;
}

int dabb_channelize(dabb_chan* ch, const dabb_chan_io* io)
{
    if (!ch || !io || !io->in || !io->in_start || !io->out || !io->out_start) return DABB_E_ARG;
    if ((io->in_is_host != 0 && io->in_is_host != 1) || io->in_len < 1 || io->in_stride < io->in_len || io->out_len < 1 || io->out_stride < io->out_len) return DABB_E_ARG;
    for (int c = 0; c < ch->n_ch; c++) {
        int64_t f, e;
        const int i = ch->input_of[(size_t)c];
        if (chan_range(ch, io->out_start[c], io->out_len, f, e) || f < io->in_start[i] || e > io->in_start[i] + io->in_len) return DABB_E_ARG;
    }
    if (const char* log = getenv("DABB_MOCK_CHAN_LOG")) {
        if (FILE* lf = fopen(log, "a")) {
            for (int c = 0; c < ch->n_ch; c++) fprintf(lf, "%lld ", (long long)io->out_start[c]);
            fprintf(lf, "%lld %lld %lld\n", (long long)io->out_len, (long long)io->in_start[0], (long long)io->in_len);
            fclose(lf);
        }
    }
    const Geometry& g = ch->g;
    const int bps = bytes_per_sample(ch->fmt);
    const float inv_r = (float)(1.0 / (double)g.R);
    const f4* taps = reinterpret_cast<const f4*>(ch->packed.data());
    std::vector<cf> xs;
    for (int c = 0; c < ch->n_ch; c++) {
        const int i = ch->input_of[(size_t)c];
        const uint8_t* in = static_cast<const uint8_t*>(io->in) + (size_t)i * (size_t)io->in_stride * (size_t)bps;
        const int64_t m0 = io->out_start[c], first = io->in_start[i];
        const int64_t n_lo = last_input(m0, g.L, g.M) - (g.TP - 1), n_hi = last_input(m0 + io->out_len - 1, g.L, g.M);
        const int64_t n_def = n_lo + (g.TP - g.T);               // the first sample of the defined span; the padding taps read zeros
        xs.assign((size_t)(n_hi - n_lo + 1), cf{0.f, 0.f});
        for (int64_t n = n_def; n <= n_hi; n++) {
            const double a = (double)mixer_arg(phase_index(ch->fmod[(size_t)c], n, g.R), g.R, inv_r);
            xs[(size_t)(n - n_lo)] = mix(in_sample(in, n - first, ch->fmt), (float)sin(M_PI * a), (float)cos(M_PI * a));
        }
        float* out = io->out + (size_t)c * (size_t)io->out_stride * 2;
        for (int64_t o = 0; o < io->out_len; o++) {
            const int64_t m = m0 + o;
            const cf y = dot(xs.data() + (last_input(m, g.L, g.M) - n_lo), taps + floor_mod(m, g.L), g.L, g.T);
            out[2 * o] = y.x; out[2 * o + 1] = y.y;
        }
    }
    return DABB_OK;
}

} // extern "C"
