// survey_host.h — the spectrum survey evaluated on the CPU in survey_kernel's order with survey_core.cuh's arithmetic (one chunk of
// segments after the other, float sums per chunk, double sums over the chunks in ascending order); shared by the host build
// (emul_survey.cpp) and the CPU test double of the ABI (mock_dab_b200_survey.cpp).  The caller checks the arguments.
#pragma once
#include "../../welle.io_b200/csrc/survey_core.cuh"
#include <algorithm>
#include <vector>

// psd [n_inputs][nfft] of n_inputs buffers of in_len samples in format fmt at in + i * in_stride samples
inline void host_survey(const uint8_t* in, int fmt, int64_t in_stride, int n_inputs, int nfft, int64_t in_len, float* psd)
{
    using namespace dabb_spectrum;
    const int log2n = log2_nfft(nfft);
    std::vector<cf> tw(MAX_NFFT / 2), a((size_t)nfft);
    std::vector<float> win(MAX_NFFT), acc((size_t)nfft);
    make_tables(tw.data(), win.data());
    const int64_t S = n_segments(in_len, nfft), chunk = chunk_segments(S, n_inputs);
    const int bps = dabb_channel::bytes_per_sample(fmt);
    for (int i = 0; i < n_inputs; i++) {
        std::vector<double> sum((size_t)nfft, 0.0);
        for (int64_t s0 = 0; s0 < S; s0 += chunk) {
            std::fill(acc.begin(), acc.end(), 0.f);
            for (int64_t s = s0; s < s0 + chunk && s < S; s++) {
                const uint8_t* seg = in + ((size_t)i * (size_t)in_stride + (size_t)(s * (nfft / 2))) * (size_t)bps;
                for (int n = 0; n < nfft; n++) a[(size_t)n] = windowed(seg, n, fmt, win.data(), log2n);
                for (int lh = log2n - 1; lh >= 0; lh--)
                    for (int b = 0; b < nfft / 2; b++) butterfly(a.data(), lh, b, tw.data(), log2n);
                for (int n = 0; n < nfft; n++) acc[(size_t)n] += a[(size_t)n].x * a[(size_t)n].x + a[(size_t)n].y * a[(size_t)n].y;
            }
            for (int n = 0; n < nfft; n++) sum[(size_t)n] += (double)acc[(size_t)n];
        }
        const double scale = 1.0 / ((double)S * (3.0 * nfft / 8.0));
        for (int pos = 0; pos < nfft; pos++) psd[(size_t)i * nfft + (bin_position(pos, log2n) ^ (nfft / 2))] = (float)(sum[(size_t)pos] * scale);
    }
}
