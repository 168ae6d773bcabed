/*
 * mock_dab_b200_ber.c — TEST DOUBLE of the C ABI with tap 10 (dabb_options.count_bit_errors), for running batch_decode --ber on a
 * machine without a GPU (tests/test_ber_emul.py).  NOT part of the product.
 *
 * It is the test double of tests/mock_backend/mock_dab_b200.c, included unchanged, with five entry points wrapped: dabb_create and
 * dabb_destroy keep a record table per context, dabb_set_options notes the option, dabb_select_subchannel notes each stream's profile,
 * and dabb_process fills the step's records from the frame records it hands out.  The double never sees softbits, so a record carries
 * the transmitted bit counts of the step's decoded codewords (4 x 2304 FIC bits for a decoded frame, n_logical x the profile's bits per
 * slot) and no errors or erasures; tests/test_gpu_ber.py checks the real counts.
 */
#define dabb_create mock_base_create
#define dabb_destroy mock_base_destroy
#define dabb_set_options mock_base_set_options
#define dabb_select_subchannel mock_base_select_subchannel
#define dabb_process mock_base_process
#define dabb_read_tap mock_base_read_tap
#include "mock_dab_b200.c"
#undef dabb_create
#undef dabb_destroy
#undef dabb_set_options
#undef dabb_select_subchannel
#undef dabb_process
#undef dabb_read_tap

enum { MAX_CTX = 8 };
typedef struct {
    const dabb_ctx* ctx;
    int count;                               /* count_bit_errors of the next step */
    dabb_ber_result* rec;                    /* tap 10: allocated when the option is first set */
    int* in_bits;                            /* [S][DABB_MAX_SUBCH] transmitted bits per logical frame of the selected profile */
} ber_state;
static ber_state g_ber[MAX_CTX];

static ber_state* ber_of(const dabb_ctx* c)
{
    for (int i = 0; i < MAX_CTX; i++) if (c && g_ber[i].ctx == c) return &g_ber[i];
    return NULL;
}

int dabb_create(const dabb_config* cfg, dabb_ctx** out)
{
    const int rc = mock_base_create(cfg, out);
    if (rc != DABB_OK) return rc;
    for (int i = 0; i < MAX_CTX; i++)
        if (!g_ber[i].ctx) {
            g_ber[i].ctx = *out; g_ber[i].count = 0; g_ber[i].rec = NULL;
            g_ber[i].in_bits = (int*)calloc((size_t)(*out)->S * DABB_MAX_SUBCH, sizeof(int));
            return DABB_OK;
        }
    mock_base_destroy(*out); *out = NULL;
    return DABB_E_NOMEM;
}

void dabb_destroy(dabb_ctx* c)
{
    ber_state* b = ber_of(c);
    if (b) { free(b->rec); free(b->in_bits); memset(b, 0, sizeof *b); }
    mock_base_destroy(c);
}

int dabb_set_options(dabb_ctx* c, const dabb_options* o)
{
    const int rc = mock_base_set_options(c, o);
    ber_state* b = ber_of(c);
    if (rc != DABB_OK || !b) return rc;
    if (o->count_bit_errors && !b->rec) b->rec = (dabb_ber_result*)calloc((size_t)c->S, sizeof(dabb_ber_result));
    b->count = o->count_bit_errors != 0;
    return DABB_OK;
}

int dabb_select_subchannel(dabb_ctx* c, int32_t first, int32_t count, int32_t slot, const dabb_subchannel* sc)
{
    const int rc = mock_base_select_subchannel(c, first, count, slot, sc);
    ber_state* b = ber_of(c);
    if (rc != DABB_OK || !b) return rc;
    orc_prot_t p;
    if (sc->short_form ? orc_prot_uep(sc->bitrate, sc->uep_level, &p) : orc_prot_eep(sc->bitrate, sc->eep_profile_a, sc->eep_level, &p)) return DABB_E_UNSUPPORTED;
    for (int s = first; s < first + count; s++) b->in_bits[(size_t)s * DABB_MAX_SUBCH + slot] = p.in_bits;
    return DABB_OK;
}

int dabb_process(dabb_ctx* c, const dabb_io* io)
{
    const int rc = mock_base_process(c, io);
    ber_state* b = ber_of(c);
    if (rc != DABB_OK || !b || !b->rec) return rc;
    memset(b->rec, 0, sizeof(dabb_ber_result) * (size_t)c->S);
    if (!b->count) return DABB_OK;
    for (int s = 0; s < c->S; s++) {
        const dabb_frame_result* r = &io->results[s];
        if (r->status != DABB_FRAME_DECODED) continue;
        b->rec[s].fic_bits = 4 * 2304;
        for (int k = 0; k < DABB_MAX_SUBCH; k++) {
            b->rec[s].subch[k].codewords = r->n_logical[k];
            b->rec[s].subch[k].bits = r->n_logical[k] * b->in_bits[(size_t)s * DABB_MAX_SUBCH + k];
        }
    }
    return DABB_OK;
}

int dabb_read_tap(dabb_ctx* c, int32_t what, void* out, size_t bytes)
{
    ber_state* b = ber_of(c);
    if (what != 10) return mock_base_read_tap(c, what, out, bytes);
    if (!c || !out) return DABB_E_ARG;
    if (!b || !b->rec) return DABB_E_STATE;
    const size_t n = sizeof(dabb_ber_result) * (size_t)c->S;
    memcpy(out, b->rec, bytes < n ? bytes : n);
    return DABB_OK;
}
