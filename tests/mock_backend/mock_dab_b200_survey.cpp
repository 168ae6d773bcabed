/*
 * mock_dab_b200_survey.cpp — TEST DOUBLE of the C ABI with the spectrum survey (dabb_survey, dabb_survey_candidates), for running
 * batch_decode --scan / --offset auto on a machine without a GPU (tests/test_survey_batch_mock.py).  NOT part of the product.
 *
 * It is the channelizer double tests/mock_backend/mock_dab_b200_chan.cpp, included unchanged, with three entry points wrapped: dabb_create
 * takes the stream files of the n-th context created from $DABB_MOCK_IQ_<n> (if set; ':'-separated, one per stream, as $DABB_MOCK_IQ)
 * so that the survey, confirmation and decode contexts of one run each get their own; dabb_chan_create logs its channels; and
 * dabb_process moves a stream that is still acquiring one frame past its window's start, as the library's null search does (the base
 * double reports position 0 for it: its streams of the oracle either decode or have ended).  The survey
 * entry points are real: dabb_survey checks its arguments like the library and computes the spectra with the host build of
 * welle.io_b200/csrc/survey_core.cuh (tests/host_emul/survey_host.h), and dabb_survey_candidates is the library's detector.  $DABB_MOCK_SURVEY_LOG (if set) gets one line
 * "survey n_inputs nfft in_len" per dabb_survey and "chan offset..." per dabb_chan_create.
 */
#define dabb_create mock_chan_base_create
#define dabb_chan_create mock_chan_base_chan_create
#define dabb_process mock_chan_base_process
#include "mock_dab_b200_chan.cpp"
#undef dabb_create
#undef dabb_chan_create
#undef dabb_process
#include "../host_emul/survey_host.h"

#include <string>

using namespace dabb_spectrum;

static int g_contexts = 0;

static void survey_log(const std::string& line)
{
    if (const char* log = getenv("DABB_MOCK_SURVEY_LOG"))
        if (FILE* lf = fopen(log, "a")) { fprintf(lf, "%s\n", line.c_str()); fclose(lf); }
}

extern "C" {

int dabb_create(const dabb_config* cfg, dabb_ctx** out)
{
    const std::string key = "DABB_MOCK_IQ_" + std::to_string(g_contexts++);
    if (const char* list = getenv(key.c_str())) setenv("DABB_MOCK_IQ", list, 1);
    return mock_chan_base_create(cfg, out);
}

int dabb_process(dabb_ctx* c, const dabb_io* io)
{
    const int rc = mock_chan_base_process(c, io);
    if (rc == DABB_OK && io->buf_start)
        for (int s = 0; s < c->S; s++)
            if (io->results[s].status == DABB_FRAME_ACQUIRING) io->results[s].next_pos = io->buf_start[s] + DABB_TF;
    return rc;
}

int dabb_chan_create(dabb_ctx* ctx, const dabb_chan_config* cfg, dabb_chan** out)
{
    const int rc = mock_chan_base_chan_create(ctx, cfg, out);
    if (rc == DABB_OK) {
        std::string l = "chan";
        for (int c = 0; c < cfg->n_channels; c++) l += " " + std::to_string((long long)cfg->offset_hz[c]);
        survey_log(l);
    }
    return rc;
}

int dabb_survey(dabb_ctx* ctx, const dabb_survey_io* io)
{
    if (!ctx || !io || !io->in || !io->psd) return DABB_E_ARG;
    const int log2n = log2_nfft(io->nfft);
    if (log2n < 0 || (io->in_is_host != 0 && io->in_is_host != 1) || io->iq_format < DABB_IQ_CF32 || io->iq_format > DABB_IQ_S16BE || io->n_inputs < 1
        || io->n_inputs > MAX_INPUTS || io->in_len < io->nfft || io->in_len > MAX_LEN || io->in_stride < io->in_len) return DABB_E_ARG;
    survey_log("survey " + std::to_string(io->n_inputs) + " " + std::to_string(io->nfft) + " " + std::to_string((long long)io->in_len));
    host_survey(static_cast<const uint8_t*>(io->in), io->iq_format, io->in_stride, io->n_inputs, io->nfft, io->in_len, io->psd);
    return DABB_OK;
}

int dabb_survey_candidates(const float* psd, int32_t nfft, int64_t rate_hz, float min_score_db, dabb_survey_candidate* out, int32_t cap, int32_t* n_found)
{
    return candidates(psd, nfft, rate_hz, min_score_db, out, cap, n_found);
}

} // extern "C"
