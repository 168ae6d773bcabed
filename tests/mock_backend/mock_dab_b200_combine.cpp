/*
 * mock_dab_b200_combine.cpp — TEST DOUBLE of the C ABI with diversity combining (dabb_set_combining, tap 12), for running
 * batch_decode --diversity on a machine without a GPU (tests/test_combine_batch_mock.py).  NOT part of the product.
 *
 * It is the clock double tests/mock_backend/mock_dab_b200_clock.cpp, included unchanged, with three entry points wrapped and one added.
 * The inner doubles #undef the names they wrap themselves, so the wrappers here are combine_wrap_{process,read_tap,destroy} and call the
 * inner entry points by their own names; the build swaps the names in the object (tests/test_combine_batch_mock.py):
 *   objcopy --redefine-sym dabb_process=mock_combine_base_process --redefine-sym combine_wrap_process=dabb_process  (and the same for
 *   read_tap and destroy).
 * The entry points:
 * dabb_set_combining checks the table like the library (DABB_E_ARG, nothing changed) and appends "combining <ctx> <leader...>" (or
 * "combining <ctx> none" for NULL) to $DABB_MOCK_COMBINE_LOG (if set); dabb_process records every stream's status, the position of its
 * phase reference symbol (next_pos - T_u - 75 T_s - T_null of the oracle's frame record) and N, the mean |x|^2 of the null symbol that
 * ends its frame window in the stream's file (combine_core.cuh's sums; the oscillator only rotates the samples), and applies the
 * library's contributor rule (dabb_comb::contributors) to every group; dabb_read_tap serves tap 12 from that once a group of two or
 * more has formed, DABB_E_STATE before; dabb_destroy forgets the context.  The softbits are the oracle's: the FIBs do not change.
 */
#include "mock_dab_b200_clock.cpp"
#include "../../welle.io_b200/csrc/combine_core.cuh"
#include <map>

namespace {
struct CombineState { std::vector<int32_t> leader; bool formed = false; std::vector<dabb_combine_result> res; };
std::map<const void*, CombineState> g_comb;

void combine_log(const dabb_ctx* c, const int32_t* leader)
{
    const char* log = getenv("DABB_MOCK_COMBINE_LOG");
    if (!log) return;
    if (FILE* lf = fopen(log, "a")) {
        fprintf(lf, "combining %p", (const void*)c);
        if (!leader) fprintf(lf, " none");
        else for (int s = 0; s < c->S; s++) fprintf(lf, " %d", leader[s]);
        fputc('\n', lf); fclose(lf);
    }
}
} // namespace

extern "C" {

int dabb_set_combining(dabb_ctx* c, const int32_t* leader, int32_t n)
{
    if (!c) return DABB_E_ARG;
    std::vector<int32_t> L((size_t)c->S);
    if (leader) {
        if (n != c->S) return DABB_E_ARG;
        std::vector<int> size((size_t)c->S, 0);
        for (int s = 0; s < c->S; s++) {
            const int32_t v = leader[s];
            if (v < 0 || v >= c->S || leader[v] != v || ++size[(size_t)v] > DABB_MAX_BRANCHES) return DABB_E_ARG;
            L[(size_t)s] = v;
        }
    } else
        for (int s = 0; s < c->S; s++) L[(size_t)s] = s;
    CombineState& g = g_comb[c];
    g.leader = L;
    for (int s = 0; s < c->S; s++) if (L[(size_t)s] != s) g.formed = true;
    if (g.res.empty()) g.res.assign((size_t)c->S, dabb_combine_result{0, 0u, 0.f, 0});
    combine_log(c, leader);
    return DABB_OK;
}

int combine_wrap_process(dabb_ctx* c, const dabb_io* io)
{
    const int rc = dabb_process(c, io);
    auto it = g_comb.find(c);
    if (rc != DABB_OK || it == g_comb.end()) return rc;
    CombineState& g = it->second;
    const int S = c->S;
    std::vector<int32_t> dec((size_t)S); std::vector<int64_t> a((size_t)S); std::vector<float> nz((size_t)S);
    for (int s = 0; s < S; s++) {
        const dabb_frame_result& r = io->results[s];
        const mock_stream* z = &c->st[s];
        dec[(size_t)s] = r.status == DABB_FRAME_DECODED;
        a[(size_t)s] = r.next_pos - DABB_TU - 75LL * DABB_TS - DABB_TNULL;
        nz[(size_t)s] = 0.f;
        const bool grouped = g.leader[(size_t)s] != s || std::count(g.leader.begin(), g.leader.end(), s) > 1;
        if (dec[(size_t)s] && grouped) {
            std::vector<float2> y((size_t)DABB_TNULL, make_float2(0.f, 0.f));
            for (int i = 0; i < DABB_TNULL; i++) {
                const int64_t p = r.next_pos - DABB_TNULL + i;
                if (p >= 0 && p < z->n) y[(size_t)i] = make_float2(z->iq[2 * p], z->iq[2 * p + 1]);
            }
            float part[dabb_comb::NULL_THREADS];
            for (int t = 0; t < dabb_comb::NULL_THREADS; t++) part[t] = dabb_comb::null_partial(y.data(), t);
            nz[(size_t)s] = dabb_comb::null_noise(part);
        }
        g.res[(size_t)s] = dabb_combine_result{0, 0u, nz[(size_t)s], 0};
    }
    for (int L = 0; L < S; L++) {
        std::vector<int> mb;
        for (int s = 0; s < S; s++) if (g.leader[(size_t)s] == L) mb.push_back(s);
        if (mb.size() < 2) continue;
        int32_t d8[dabb_comb::MAX_BRANCHES]; int64_t a8[dabb_comb::MAX_BRANCHES]; float n8[dabb_comb::MAX_BRANCHES]; int lpos = 0;
        for (size_t i = 0; i < mb.size(); i++) { d8[i] = dec[(size_t)mb[i]]; a8[i] = a[(size_t)mb[i]]; n8[i] = nz[(size_t)mb[i]]; if (mb[i] == L) lpos = (int)i; }
        const uint32_t m = dabb_comb::contributors((int)mb.size(), lpos, d8, a8, n8);
        g.res[(size_t)L].members = dabb_comb::popcount(m); g.res[(size_t)L].mask = m;
    }
    return rc;
}

int combine_wrap_read_tap(dabb_ctx* c, int32_t what, void* out, size_t bytes)
{
    if (what != 12) return dabb_read_tap(c, what, out, bytes);
    if (!c || !out) return DABB_E_ARG;
    auto it = g_comb.find(c);
    if (it == g_comb.end() || !it->second.formed) return DABB_E_STATE;
    const size_t n = sizeof(dabb_combine_result) * it->second.res.size();
    memcpy(out, it->second.res.data(), bytes < n ? bytes : n);
    return DABB_OK;
}

void combine_wrap_destroy(dabb_ctx* c)
{
    g_comb.erase(c);
    dabb_destroy(c);
}

} // extern "C"
