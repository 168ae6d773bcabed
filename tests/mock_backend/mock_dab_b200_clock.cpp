/*
 * mock_dab_b200_clock.cpp — TEST DOUBLE of the C ABI that records dabb_options.sample_clock, for running batch_decode --clock on a machine
 * without a GPU (tests/test_clock_batch_mock.py).  NOT part of the product.
 *
 * It is the survey double tests/mock_backend/mock_dab_b200_survey.cpp, included unchanged, with three entry points wrapped:
 * dabb_set_options refuses a sample_clock outside DABB_CLOCK_* like the library and appends "options <ctx> <sample_clock>
 * <disable_coarse> <freqsync_method>" to $DABB_MOCK_CLOCK_LOG (if set); dabb_read_tap serves tap 11 once TRACK has been set (every
 * stream: ppm 1.25, applied_ppm 0.5, frames 9), DABB_E_STATE before; dabb_destroy appends "destroy <ctx>".
 */
#define dabb_set_options mock_clock_base_set_options
#define dabb_destroy mock_clock_base_destroy
#define dabb_read_tap mock_clock_base_read_tap
#include "mock_dab_b200_survey.cpp"
#undef dabb_set_options
#undef dabb_destroy
#undef dabb_read_tap
#include <set>

static std::set<const void*> g_tracking;

static void clock_log(const char* fmt, const void* ctx, int a = 0, int b = 0, int c = 0)
{
    if (const char* log = getenv("DABB_MOCK_CLOCK_LOG"))
        if (FILE* lf = fopen(log, "a")) { fprintf(lf, fmt, ctx, a, b, c); fputc('\n', lf); fclose(lf); }
}

extern "C" {

int dabb_set_options(dabb_ctx* c, const dabb_options* o)
{
    if (o && o->sample_clock != DABB_CLOCK_OFF && o->sample_clock != DABB_CLOCK_TRACK) return DABB_E_ARG;
    const int rc = mock_clock_base_set_options(c, o);
    if (rc == DABB_OK) {
        clock_log("options %p %d %d %d", c, o->sample_clock, o->disable_coarse, o->freqsync_method);
        if (o->sample_clock == DABB_CLOCK_TRACK) g_tracking.insert(c);
    }
    return rc;
}

int dabb_read_tap(dabb_ctx* c, int32_t what, void* out, size_t bytes)
{
    if (what != 11) return mock_clock_base_read_tap(c, what, out, bytes);
    if (!c || !out) return DABB_E_ARG;
    if (!g_tracking.count(c)) return DABB_E_STATE;
    std::vector<dabb_clock_result> rec((size_t)c->S);
    for (auto& r : rec) { r.ppm = 1.25f; r.applied_ppm = 0.5f; r.frames = 9; r.reserved = 0; }
    const size_t n = sizeof(dabb_clock_result) * rec.size();
    memcpy(out, rec.data(), bytes < n ? bytes : n);
    return DABB_OK;
}

void dabb_destroy(dabb_ctx* c)
{
    clock_log("destroy %p", c);
    g_tracking.erase(c);
    mock_clock_base_destroy(c);
}

} // extern "C"
