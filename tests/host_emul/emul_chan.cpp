// CPU build of the wideband channelizer (welle.io_b200/csrc/chan_core.cuh): the geometry, the filter design the library uploads, and
// one channel's outputs evaluated in chan_kernel's order (tests/test_chan_emul.py).  Compile with -ffp-contract=off.
#include "../../welle.io_b200/csrc/chan_core.cuh"
#include <math.h>
#include <stdint.h>
#include <vector>

using namespace dabb_channel;

extern "C" {

// {L, M, T, TP}; returns DABB_OK or DABB_E_UNSUPPORTED
int emul_chan_geometry(int64_t R, int32_t* out)
{
    Geometry g{};
    const int rc = geometry(R, g);
    if (rc == DABB_OK) { out[0] = g.L; out[1] = g.M; out[2] = g.T; out[3] = g.TP; }
    return rc;
}

int emul_chan_offset_ok(int64_t R, int64_t f) { return offset_ok(R, f) ? 1 : 0; }

// the prototype h[0 .. L T)
void emul_chan_taps(int64_t R, float* h)
{
    Geometry g{};
    geometry(R, g);
    design_taps(g, h);
}

// outputs [out_start, out_start + out_len) of the channel at offset f from a raw buffer whose first sample is absolute index in_start
// (in_len samples, format fmt); the mixer's sin / cos are the double functions rounded to float (the device uses sincospif)
int emul_chan_run(int64_t R, int fmt, int64_t f, const uint8_t* in, int64_t in_start, int64_t in_len, int64_t out_start, int64_t out_len, float* out)
{
    Geometry g{};
    if (geometry(R, g) != DABB_OK) return -1;
    std::vector<float> h((size_t)g.L * g.T), packed((size_t)g.L * g.TP);
    design_taps(g, h.data());
    pack_taps(g, h.data(), packed.data());
    const f4* taps = reinterpret_cast<const f4*>(packed.data());
    const int64_t n_lo = last_input(out_start, g.L, g.M) - (g.TP - 1), n_hi = last_input(out_start + out_len - 1, g.L, g.M);
    if (n_lo + (g.TP - g.T) < in_start || n_hi >= in_start + in_len) return -2;
    const int64_t fm = floor_mod(f, R);
    const float inv_r = (float)(1.0 / (double)R);
    std::vector<cf> xs((size_t)(n_hi - n_lo + 1));
    for (int64_t n = n_lo; n <= n_hi; n++) {
        cf v{0.f, 0.f};
        if (n >= in_start) {
            const double a = (double)mixer_arg(phase_index(fm, n, R), R, inv_r);
            v = mix(in_sample(in, n - in_start, fmt), (float)sin(M_PI * a), (float)cos(M_PI * a));
        }
        xs[(size_t)(n - n_lo)] = v;
    }
    for (int64_t o = 0; o < out_len; o++) {
        const int64_t m = out_start + o;
        const cf y = dot(xs.data() + (last_input(m, g.L, g.M) - n_lo), taps + floor_mod(m, g.L), g.L, g.T);
        out[2 * o] = y.x; out[2 * o + 1] = y.y;
    }
    return 0;
}

} // extern "C"
