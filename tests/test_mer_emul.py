"""The modulation error ratio of the device (welle.io_b200/csrc/mer_core.cuh, with the library's frequency-interleaver table from
tables.cpp) compiled as host code (tests/host_emul/emul_mer.cpp), against the restatement of the definition in include/dab_b200.h
(tests/merref.py), which shares nothing with it: random softbits, all zeros, the +-127 / -128 extremes, a symbol of erasures, u == v,
err == 0 and sig == 0.  Every carrier's group, the layout of dabb_mer_result, and what the measurement means, on the CPU through the
oracle's demodulator (whose softbits equal the device's bit for bit in the exact FFT mode): MER against AWGN SNR, and the 64-group
profile beside a tone and in a two-path channel."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import dabtx
import merref as M
from conftest import load_pkg

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_mer") / "libemul_mer.so")
    subprocess.check_call([os.environ.get("NVCC", "nvcc"), "-O2", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-x", "cu", "-shared", "-Xcompiler", "-fPIC",
                           "-o", so, os.path.join(HERE, "host_emul", "emul_mer.cpp")])
    lib = C.CDLL(so)
    lib.emul_mer_db.restype = C.c_float
    lib.emul_mer_db.argtypes = [C.c_int64, C.c_int64]
    return lib


def host_records(emul, soft, active=None):
    """tap-14 records of the host build for frames soft [n][>= 9216] (int8)"""
    pkg = load_pkg()
    soft = np.ascontiguousarray(soft, np.int8)
    n = soft.shape[0]
    out = np.zeros(n, pkg.MER_DTYPE)
    act = None if active is None else np.ascontiguousarray(active, np.int32)
    emul.emul_mer(soft.ctypes.data_as(C.c_void_p), C.c_int64(soft.shape[1]), None if act is None else act.ctypes.data_as(C.c_void_p), n,
                  out.ctypes.data_as(C.c_void_p))
    return out


def same(rec, want):
    got = M.from_tap(rec)
    assert (got["points"], got["sig"], got["err"], got["gsig"], got["gerr"]) == (want["points"], want["sig"], want["err"], want["gsig"], want["gerr"])
    w = want["mer_db"]
    if math.isinf(w) or w == 0.0:
        assert got["mer_db"] == w, (got["mer_db"], w)
    else:
        assert abs(got["mer_db"] - w) <= 2e-6 * abs(w), (got["mer_db"], w)


def frames_of(rng):
    f = []
    f.append(rng.integers(-128, 128, 9216))                                 # random
    f.append(np.zeros(9216))                                                # sig == 0
    f.append(rng.choice([-128, -127, 127], 9216))                           # saturation: u == |v| on +-127 / -128 pairs
    x = rng.integers(-128, 128, 9216); x[3072:6144] = 0; f.append(x)        # symbol 2 all erasures
    x = rng.integers(-128, 128, 9216); x[::7] = 0; f.append(x)              # a softbit of 0: u == |v|
    x = rng.choice([-60, 60], 9216); f.append(x)                            # |a| == |b| everywhere: err == 0
    x = rng.integers(-128, 128, 9216); x[rng.random(9216) < 0.5] = 0; f.append(x)
    x = np.zeros(9216); x[1536:3072] = -128; f.append(x)                    # only Im softbits: sig == err
    x = np.zeros(9216); x[5] = 1; f.append(x)                               # one point
    return np.stack(f).astype(np.int8)


def test_host_build_matches_restatement(emul):
    rng = np.random.default_rng(0x3E1)
    soft = np.concatenate([frames_of(rng), rng.integers(-128, 128, (23, 9216)).astype(np.int8)])
    got = host_records(emul, soft)
    for i in range(len(soft)):
        same(got[i], M.record(soft[i]))
    assert got[1]["sig"] == 0 and got[1]["mer_db"] == 0.0 and got[1]["points"] == 0
    assert got[5]["err"] == 0 < got[5]["sig"] and got[5]["mer_db"] == np.inf and got[5]["points"] == 4608
    assert got[7]["sig"] == got[7]["err"] and got[7]["mer_db"] == 0.0
    assert got[8]["points"] == 1 and got[8]["sig"] == got[8]["err"] == 1


def test_inactive_and_stride(emul):
    """a frame that was not decoded gives the all-zero record; only the first 9216 softbits of a row are read"""
    rng = np.random.default_rng(0x3E2)
    soft = rng.integers(-128, 128, (4, 75 * 3072)).astype(np.int8)
    got = host_records(emul, soft, active=[1, 0, 1, 0])
    assert not got[1].tobytes().strip(b"\0") and not got[3].tobytes().strip(b"\0")
    same(got[0], M.record(soft[0])); same(got[2], M.record(soft[2]))
    soft[0, 9216:] = 0
    assert host_records(emul, soft[:1])[0].tobytes() == got[0].tobytes()


def test_mer_db_edges(emul):
    assert emul.emul_mer_db(0, 0) == 0.0 and emul.emul_mer_db(0, 5) == 0.0 and emul.emul_mer_db(7, 0) == math.inf
    rng = np.random.default_rng(0x3E3)
    for _ in range(2000):
        sig, err = int(rng.integers(1, 4608 * 65536)), int(rng.integers(1, 4608 * 65536))
        want = float(np.float32(10 * math.log10(sig / err)))
        got = emul.emul_mer_db(sig, err)
        assert abs(got - want) <= 1.2e-7 * max(1.0, abs(want)), (sig, err, got, want)


def test_groups(emul):
    """every logical carrier's group against the restatement; each group holds 24 carriers per symbol, lowest frequency first"""
    g = np.zeros(1536, np.uint8)
    emul.emul_mer_groups(g.ctypes.data_as(C.c_void_p))
    assert np.array_equal(g.astype(np.int64), M.groups())
    assert np.array_equal(np.bincount(g, minlength=64), np.full(64, 24))
    k = M.physical_carriers()
    for grp in range(64):
        c = np.sort(k[g == grp])
        first = 24 * grp - 768 + (grp >= 32)
        assert np.array_equal(c, np.arange(first, first + 24)), grp
    assert g[np.argmax(k == 301)] == 44


def test_layout(emul):
    pkg = load_pkg()
    lay = np.zeros(7, np.int32)
    emul.emul_mer_layout(lay.ctypes.data_as(C.c_void_p))
    d = pkg.MER_DTYPE
    assert lay[0] == d.itemsize == 536 and pkg.MER_GROUPS == 64
    assert [lay[1], lay[2], lay[3], lay[4], lay[5]] == [d.fields[f][1] for f in ("points", "mer_db", "sig", "err", "group")]
    assert lay[6] == d.fields["group"][1] + 8 + 4


# ---- what the number means: the oracle's demodulator on tests/dabtx.py recordings
FRAMES = 4


def run_sum(recs):
    r = M.zero_record()
    for q in recs:
        r["sig"] += q["sig"]; r["err"] += q["err"]
        r["gsig"] = [a + b for a, b in zip(r["gsig"], q["gsig"])]
        r["gerr"] = [a + b for a, b in zip(r["gerr"], q["gerr"])]
    return r


def measured(oracle, y):
    return run_sum([M.record(s) for s in M.oracle_softbits(oracle, y, FRAMES)])


@pytest.fixture(scope="module")
def clean():
    return dabtx.DabTx(seed=0x3E0).frames(FRAMES)


def test_awgn_sweep(oracle, clean):
    """MER rises monotonically with the SNR from 0 to 40 dB, saturating towards 5.6 dB at the bottom; from 12 to 30 dB it lies within
    1 dB of SNR + 1.25 dB (the per-carrier SNR).  Measured on this recording: -0.61 dB at 12 dB, -0.09 to -0.22 dB from 15 to 30 dB, 5.64 dB at 0 dB."""
    snrs = [0, 4, 8, 10, 12, 15, 20, 25, 30, 35, 40]
    mer = []
    for snr in snrs:
        r = measured(oracle, dabtx.add_awgn(clean, snr, seed=0x3E00 + snr))
        mer.append(M.mer_db(r["sig"], r["err"]))
    assert all(b > a for a, b in zip(mer, mer[1:])), mer
    assert 5.0 < mer[0] < 6.5, mer
    for snr, m in zip(snrs, mer):
        if 12 <= snr <= 30:
            assert abs(m - (snr + 1.25)) < 1.0, (snr, m)


def test_tone_profile(oracle, clean):
    """a tone on carrier 301 (301 kHz), 10 dB above the ensemble at 20 dB SNR: group 44 (carriers 289 .. 312) is the lowest of the
    profile.  Measured: 1.1 dB below the next lowest group and 2.1 dB below the median."""
    y = M.tone(dabtx.add_awgn(clean, 20, seed=0x3E10), 301000, 10, seed=1)
    g = M.group_mer(measured(oracle, y))
    order = np.argsort(g)
    assert order[0] == 44, (order[:4], g[order[:4]])
    assert g[order[1]] - g[44] > 0.4 and np.median(g) - g[44] > 1.5, g


def test_two_path_profile(oracle, clean):
    """the two-path channel [(0, 1), (20, 0.95j)] at 20 dB SNR notches the band every 102 carriers: the 64 group MERs spread far more
    than with AWGN alone.  Measured: standard deviation 0.5 dB (AWGN) against 5.9 dB, range 2.5 against 16.5 dB."""
    a = M.group_mer(measured(oracle, dabtx.add_awgn(clean, 20, seed=0x3E20)))
    b = M.group_mer(measured(oracle, dabtx.add_awgn(M.two_path(clean, [(0, 1), (20, 0.95j)]), 20, seed=0x3E20)))
    assert np.std(a) < 1.0 and np.ptp(a) < 4.0, a
    assert np.std(b) > 4 * np.std(a) and np.ptp(b) > 10.0, b
