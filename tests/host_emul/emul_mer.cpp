// CPU build of the modulation error ratio (welle.io_b200/csrc/mer_core.cuh) with the library's frequency-interleaver table (tables.cpp is
// host code in a CUDA translation unit: compile with nvcc -x cu; no device is involved).  tests/test_mer_emul.py, tests/test_gpu_mer.py
#include "../../welle.io_b200/csrc/tables.cpp"
#include "../../welle.io_b200/csrc/mer_core.cuh"
#include "../../include/dab_b200.h"
#include <stddef.h>
using namespace dabb;

static const HostTables& tables()
{
    static HostTables* t = nullptr;
    if (!t) { t = new HostTables; build_host_tables(*t); }
    return *t;
}

// [1536] each logical carrier's group, as api.cu uploads it
extern "C" void emul_mer_groups(uint8_t* out)
{
    for (int i = 0; i < KC; i++) out[i] = (uint8_t)dabb_mer::group_of(tables().perm[i]);
}

// the tap-14 records of n frames: frame i's softbits start at soft + i * stride (its first 9216 bytes are read); active[i] == 0 (or a null
// active) gives the all-zero record of a stream that decoded no frame
extern "C" void emul_mer(const int8_t* soft, int64_t stride, const int32_t* active, int n, dabb_mer_result* out)
{
    uint8_t grp[KC];
    emul_mer_groups(grp);
    for (int f = 0; f < n; f++) {
        dabb_mer_result r;
        memset(&r, 0, sizeof r);
        if (!active || active[f]) {
            const int8_t* x = soft + (int64_t)f * stride;
            for (int l = 0; l < dabb_mer::SYMBOLS; l++)
                for (int i = 0; i < dabb_mer::CARRIERS; i++) {
                    int32_t u2, v2;
                    dabb_mer::point(x[l * 3072 + i], x[l * 3072 + 1536 + i], u2, v2);
                    r.group[grp[i]].sig += u2; r.group[grp[i]].err += v2; r.points += u2 > 0;
                }
            for (int g = 0; g < DABB_MER_GROUPS; g++) { r.sig += r.group[g].sig; r.err += r.group[g].err; }
            r.mer_db = dabb_mer::mer_db(r.sig, r.err);
        }
        out[f] = r;
    }
}

extern "C" float emul_mer_db(int64_t sig, int64_t err) { return dabb_mer::mer_db(sig, err); }

// sizeof(dabb_mer_result), then the offsets of points, mer_db, sig, err, group, group[1].err
extern "C" void emul_mer_layout(int32_t* out)
{
    out[0] = (int32_t)sizeof(dabb_mer_result); out[1] = (int32_t)offsetof(dabb_mer_result, points); out[2] = (int32_t)offsetof(dabb_mer_result, mer_db);
    out[3] = (int32_t)offsetof(dabb_mer_result, sig); out[4] = (int32_t)offsetof(dabb_mer_result, err); out[5] = (int32_t)offsetof(dabb_mer_result, group);
    out[6] = (int32_t)offsetof(dabb_mer_result, group[1].err);
}
