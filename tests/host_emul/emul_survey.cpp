// CPU build of the spectrum survey and the candidate detector (welle.io_b200/csrc/survey_core.cuh): the spectrum evaluated chunk by chunk
// in survey_kernel's order (tests/test_survey_emul.py).  Compile with -ffp-contract=off.
#include "survey_host.h"
#include <stdint.h>

using namespace dabb_spectrum;

extern "C" {

// psd [n_inputs][nfft] of n_inputs raw buffers of in_len samples at in + i * in_stride samples; DABB_OK or DABB_E_ARG
int emul_survey(const uint8_t* in, int fmt, int64_t in_stride, int n_inputs, int nfft, int64_t in_len, float* psd)
{
    const int log2n = log2_nfft(nfft);
    if (log2n < 0 || fmt < DABB_IQ_CF32 || fmt > DABB_IQ_S16BE || n_inputs < 1 || n_inputs > MAX_INPUTS || in_len < nfft || in_stride < in_len) return DABB_E_ARG;
    host_survey(in, fmt, in_stride, n_inputs, nfft, in_len, psd);
    return DABB_OK;
}

int emul_survey_candidates(const float* psd, int32_t nfft, int64_t rate_hz, float min_score_db, dabb_survey_candidate* out, int32_t cap, int32_t* n_found)
{
    return candidates(psd, nfft, rate_hz, min_score_db, out, cap, n_found);
}

} // extern "C"
