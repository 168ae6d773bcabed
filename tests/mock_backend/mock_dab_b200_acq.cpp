/*
 * mock_dab_b200_acq.cpp — TEST DOUBLE of the C ABI that records dabb_options.acquisition, for running batch_decode --acq on a machine
 * without a GPU (tests/test_acq_batch_mock.py).  NOT part of the product.
 *
 * It is the survey double tests/mock_backend/mock_dab_b200_survey.cpp, included unchanged, with three entry points wrapped:
 * dabb_set_options refuses an acquisition outside DABB_ACQ_* like the library and appends "options <ctx> <acquisition>
 * <disable_coarse> <freqsync_method>" to $DABB_MOCK_ACQ_LOG (if set); dabb_read_tap serves tap 13 once ROBUST has been set (every
 * stream: searched, 774 blocks, depth 2.5 dB, a null found at 1000), DABB_E_STATE before; dabb_destroy appends "destroy <ctx>".
 */
#define dabb_set_options mock_acq_base_set_options
#define dabb_destroy mock_acq_base_destroy
#define dabb_read_tap mock_acq_base_read_tap
#include "mock_dab_b200_survey.cpp"
#undef dabb_set_options
#undef dabb_destroy
#undef dabb_read_tap
#include <set>

static std::set<const void*> g_robust;

static void acq_log(const char* fmt, const void* ctx, int a = 0, int b = 0, int c = 0)
{
    if (const char* log = getenv("DABB_MOCK_ACQ_LOG"))
        if (FILE* lf = fopen(log, "a")) { fprintf(lf, fmt, ctx, a, b, c); fputc('\n', lf); fclose(lf); }
}

extern "C" {

int dabb_set_options(dabb_ctx* c, const dabb_options* o)
{
    if (o && o->acquisition != DABB_ACQ_REFERENCE && o->acquisition != DABB_ACQ_ROBUST) return DABB_E_ARG;
    const int rc = mock_acq_base_set_options(c, o);
    if (rc == DABB_OK) {
        acq_log("options %p %d %d %d", c, o->acquisition, o->disable_coarse, o->freqsync_method);
        if (o->acquisition == DABB_ACQ_ROBUST) g_robust.insert(c);
    }
    return rc;
}

int dabb_read_tap(dabb_ctx* c, int32_t what, void* out, size_t bytes)
{
    if (what != 13) return mock_acq_base_read_tap(c, what, out, bytes);
    if (!c || !out) return DABB_E_ARG;
    if (!g_robust.count(c)) return DABB_E_STATE;
    std::vector<dabb_acq_result> rec((size_t)c->S);
    for (auto& r : rec) { r.searched = 1; r.blocks = 774; r.depth_db = 2.5f; r.excised = 0; r.null_end = 1000; }
    const size_t n = sizeof(dabb_acq_result) * rec.size();
    memcpy(out, rec.data(), bytes < n ? bytes : n);
    return DABB_OK;
}

void dabb_destroy(dabb_ctx* c)
{
    acq_log("destroy %p", c);
    g_robust.erase(c);
    mock_acq_base_destroy(c);
}

} // extern "C"
