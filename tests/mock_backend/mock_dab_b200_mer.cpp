/*
 * mock_dab_b200_mer.cpp — TEST DOUBLE of the C ABI with tap 14 (dabb_set_mer), for running batch_decode --mer on a machine without a
 * GPU (tests/test_mer_batch_mock.py).  NOT part of the product.
 *
 * It is the test double of tests/mock_backend/mock_dab_b200.c, included unchanged, with four entry points wrapped and dabb_set_mer
 * added: dabb_create and dabb_destroy keep a record table per context, dabb_set_mer switches the measurement (and appends "mer <ctx>
 * <enable>" to $DABB_MOCK_MER_LOG if set), and dabb_process fills the step's records from the frame records it hands out.  The double
 * never sees softbits, so the record of stream s's n-th decoded frame (n from 0) is made up, deterministically (mock_record; the test
 * restates it): group g has sig = 50000 + 1000 s + 37 g + n and err = 0 for g mod 7 == 3, else 100 + 3 g + s + n; points = 4608 - s - n.
 */
#define dabb_create mock_base_create
#define dabb_destroy mock_base_destroy
#define dabb_process mock_base_process
#define dabb_read_tap mock_base_read_tap
#include "mock_dab_b200.c"
#undef dabb_create
#undef dabb_destroy
#undef dabb_process
#undef dabb_read_tap
#include <cmath>
#include <map>
#include <vector>

namespace {

struct MerState {
    bool on = false, enabled_once = false;
    std::vector<dabb_mer_result> rec;        // tap 14 of the last step
    std::vector<int> frames;                 // decoded frames so far, per stream
};
std::map<const dabb_ctx*, MerState> g_mer;

void mer_log(const dabb_ctx* c, int enable)
{
    if (const char* log = getenv("DABB_MOCK_MER_LOG"))
        if (FILE* lf = fopen(log, "a")) { fprintf(lf, "mer %p %d\n", (const void*)c, enable); fclose(lf); }
}

dabb_mer_result mock_record(int s, int n)
{
    dabb_mer_result r;
    memset(&r, 0, sizeof r);
    r.points = 4608 - s - n;
    for (int g = 0; g < DABB_MER_GROUPS; g++) {
        r.group[g].sig = 50000 + 1000 * s + 37 * g + n;
        r.group[g].err = g % 7 == 3 ? 0 : 100 + 3 * g + s + n;
        r.sig += r.group[g].sig; r.err += r.group[g].err;
    }
    r.mer_db = (float)(10.0 * log10((double)r.sig / (double)r.err));
    return r;
}

} // namespace

extern "C" {

int dabb_create(const dabb_config* cfg, dabb_ctx** out)
{
    const int rc = mock_base_create(cfg, out);
    if (rc == DABB_OK) g_mer[*out] = MerState{};
    return rc;
}

void dabb_destroy(dabb_ctx* c)
{
    g_mer.erase(c);
    mock_base_destroy(c);
}

int dabb_set_mer(dabb_ctx* c, int32_t enable)
{
    if (!c || !g_mer.count(c)) return DABB_E_ARG;
    MerState& m = g_mer[c];
    if (enable && !m.enabled_once) { m.enabled_once = true; m.rec.assign((size_t)c->S, dabb_mer_result{}); m.frames.assign((size_t)c->S, 0); }
    m.on = enable != 0;
    mer_log(c, enable);
    return DABB_OK;
}

int dabb_process(dabb_ctx* c, const dabb_io* io)
{
    const int rc = mock_base_process(c, io);
    auto it = g_mer.find(c);
    if (rc != DABB_OK || it == g_mer.end() || !it->second.enabled_once) return rc;
    MerState& m = it->second;
    for (int s = 0; s < c->S; s++) {
        memset(&m.rec[(size_t)s], 0, sizeof(dabb_mer_result));
        if (m.on && io->results[s].status == DABB_FRAME_DECODED) m.rec[(size_t)s] = mock_record(s, m.frames[(size_t)s]++);
    }
    return DABB_OK;
}

int dabb_read_tap(dabb_ctx* c, int32_t what, void* out, size_t bytes)
{
    if (what != 14) return mock_base_read_tap(c, what, out, bytes);
    if (!c || !out) return DABB_E_ARG;
    auto it = g_mer.find(c);
    if (it == g_mer.end() || !it->second.enabled_once) return DABB_E_STATE;
    const size_t n = sizeof(dabb_mer_result) * (size_t)c->S;
    memcpy(out, it->second.rec.data(), bytes < n ? bytes : n);
    return DABB_OK;
}

} // extern "C"
