// CPU build of the weighted soft-decision demap (DABB_DEMAP_WEIGHTED) of welle.io_b200/csrc/ofdm_core.cuh: level_acc, level_gmean,
// demap_weighted and the reference demap's q127 / soft_q, symbol by symbol (tests/test_soft_demap_emul.py).  The device sums the
// per-carrier terms per thread and then in a CTA tree; here they are summed in carrier order.  Compile with -ffp-contract=off.
#include "../../welle.io_b200/csrc/ofdm_core.cuh"
#include <stdint.h>

using namespace dabb;

extern "C" {

// n symbols of r1, KC complex floats each: softbits of both modes in the reference layout (KC Re bits, then KC Im bits) and G per symbol
void emul_softdemap(const float* r1, int n, int8_t* soft_w, int8_t* soft_r, float* g)
{
    for (int l = 0; l < n; l++) {
        const float* x = r1 + (int64_t)l * 2 * KC;
        LevelSum a{0, 0.f};
        for (int k = 0; k < KC; k++) level_acc(a, level_l1(make_float2(x[2 * k], x[2 * k + 1])));
        const float G = level_gmean(a), rG = q127(G);
        g[l] = G;
        int8_t* w = soft_w + (int64_t)l * 2 * KC;
        int8_t* r = soft_r + (int64_t)l * 2 * KC;
        for (int k = 0; k < KC; k++) {
            const float2 v = make_float2(x[2 * k], x[2 * k + 1]);
            demap_weighted(v, G, rG, w[k], w[KC + k]);
            const float ab1 = q127(level_l1(v));
            r[k] = soft_q(v.x, ab1);
            r[KC + k] = soft_q(v.y, ab1);
        }
    }
}

} // extern "C"
