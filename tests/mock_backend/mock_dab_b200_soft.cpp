/*
 * mock_dab_b200_soft.cpp — TEST DOUBLE of the C ABI that records dabb_options.soft_demap, for running batch_decode --soft on a machine
 * without a GPU (tests/test_soft_batch_mock.py).  NOT part of the product.
 *
 * It is the survey double tests/mock_backend/mock_dab_b200_survey.cpp, included unchanged, with two entry points wrapped: dabb_set_options
 * refuses a soft_demap outside DABB_DEMAP_* like the library and appends "options <ctx> <soft_demap> <disable_coarse> <freqsync_method>"
 * to $DABB_MOCK_SOFT_LOG (if set), and dabb_destroy appends "destroy <ctx>".
 */
#define dabb_set_options mock_soft_base_set_options
#define dabb_destroy mock_soft_base_destroy
#include "mock_dab_b200_survey.cpp"
#undef dabb_set_options
#undef dabb_destroy

static void soft_log(const char* fmt, const void* ctx, int a = 0, int b = 0, int c = 0)
{
    if (const char* log = getenv("DABB_MOCK_SOFT_LOG"))
        if (FILE* lf = fopen(log, "a")) { fprintf(lf, fmt, ctx, a, b, c); fputc('\n', lf); fclose(lf); }
}

extern "C" {

int dabb_set_options(dabb_ctx* c, const dabb_options* o)
{
    if (o && o->soft_demap != DABB_DEMAP_REFERENCE && o->soft_demap != DABB_DEMAP_WEIGHTED) return DABB_E_ARG;
    const int rc = mock_soft_base_set_options(c, o);
    if (rc == DABB_OK) soft_log("options %p %d %d %d", c, o->soft_demap, o->disable_coarse, o->freqsync_method);
    return rc;
}

void dabb_destroy(dabb_ctx* c)
{
    soft_log("destroy %p", c);
    mock_soft_base_destroy(c);
}

} // extern "C"
