"""The weighted soft-decision demap (DABB_DEMAP_WEIGHTED) of welle.io_b200/csrc/ofdm_core.cuh compiled as host C++
(tests/host_emul/emul_softdemap.cpp) against the numpy restatement (tests/softref.py): random and faded r1, all-zero symbols, subnormal
levels, an inf or NaN carrier, power-of-two scales.  Then the gain it is for, on the CPU: the float64 demodulator (tests/ofdmref.py) at
the direct-path window, both demaps, and the oracle's FIC decoder, in AWGN, two- and three-path channels and beside a strong tone."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import dabtx
import ofdmref
import softref
from conftest import ROOT

K = 1536
HERE = os.path.join(ROOT, "tests", "host_emul")


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_soft") / "libemul_softdemap.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "emul_softdemap.cpp")])
    return C.CDLL(so)


def run(lib, r1):
    r1 = np.ascontiguousarray(np.asarray(r1).astype(np.complex64).reshape(-1, K))
    n = len(r1)
    w = np.zeros((n, 2 * K), np.int8); r = np.zeros((n, 2 * K), np.int8); g = np.zeros(n, np.float32)
    lib.emul_softdemap(r1.ctypes.data_as(C.c_void_p), n, w.ctypes.data_as(C.c_void_p), r.ctypes.data_as(C.c_void_p), g.ctypes.data_as(C.c_void_p))
    return w, r, g


def faded(seed, n=16):
    """QPSK-like r1 through a random frequency-selective channel: levels spread over several decades"""
    rng = np.random.default_rng(seed)
    k = np.arange(K)
    out = []
    for _ in range(n):
        taps = rng.standard_normal(4) + 1j * rng.standard_normal(4)
        h = np.exp(-2j * np.pi * np.outer(k, rng.integers(0, 200, 4)) / 2048) @ taps
        x = (rng.integers(0, 4, K) * 2 + 1) * np.pi / 4
        out.append(np.abs(h) ** 2 * 38.6 * np.exp(1j * x) + (rng.standard_normal(K) + 1j * rng.standard_normal(K)) * 2.0)
    return np.array(out)


@pytest.mark.parametrize("case", ["random", "faded"])
def test_emulation_matches_restatement(emul, case):
    rng = np.random.default_rng(0x50F7)
    r1 = (rng.standard_normal((16, K)) + 1j * rng.standard_normal((16, K))) * 20 if case == "random" else faded(0x50F8)
    w, r, g = run(emul, r1)
    assert np.array_equal(r, softref.soft_reference_f32(r1))
    weak = softref.check(r1, w, g)
    assert weak > 16 * K // 8          # a good share of the carriers is below G
    assert np.all(np.abs(w.astype(int)) <= np.abs(r.astype(int)))     # never more confident than the reference demap


def test_zero_subnormal_and_nonfinite(emul):
    base = faded(0x50F9, 6)
    r1 = base.copy()
    r1[0] = 0                                            # all-zero symbol: softbits 0
    r1[1, ::3] *= 1e-40                                  # subnormal levels: clamped to 2^-126 in G
    r1[2, 77] = np.inf                                   # one inf carrier: G = 0, the reference demap
    r1[3, 900] = complex(np.nan, 1.0)                    # one NaN carrier: the same
    r1[4, :] = base[4] * 1e-41                           # a whole symbol of subnormal levels
    w, r, g = run(emul, r1)
    assert not w[0].any() and not r[0].any()
    assert g[2] == 0 and g[3] == 0 and g[0] > 0 and g[1] > 0
    assert np.array_equal(w[2], r[2]) and np.array_equal(w[3], r[3])
    softref.check(r1, w, g)


def test_power_of_two_scales(emul):
    r1 = faded(0x50FA, 4)
    w0, _, g0 = run(emul, r1)
    for e in range(-60, 61, 5):
        w, _, g = run(emul, r1 * 2.0 ** e)
        # the exponents are summed exactly: G moves by exactly 2^e, and so does every quotient
        assert np.array_equal(g, (g0.astype(np.float64) * 2.0 ** e).astype(np.float32)), e
        assert np.array_equal(w, w0), e


# ---- the gain on the CPU: float64 demodulator, oracle FIC decoder
TF, TNULL = 196608, 2656
SEEDS = (0x100, 0x101, 0x102)
CHANNELS = {"awgn": None, "2path": [(0, 1.0), (20, 0.95j)], "3path": [(0, 1.0), (37, 0.7 - 0.3j), (211, 0.5j)], "tone": "tone"}
POINTS = [("awgn", 3.0), ("2path", 3.0), ("2path", 5.0), ("3path", 3.0), ("3path", 5.0), ("tone", 4.0)]


def channel(x, name, snr_db, seed):
    """the SNR is that of the received ensemble (after the echoes, without the tone)"""
    ch = CHANNELS[name]
    if ch not in (None, "tone"):
        x = ofdmref.multipath(x, ch)
    p = float(np.mean(np.abs(x) ** 2))
    if ch == "tone":
        x = x + np.sqrt(100.0 * p) * np.exp(2j * np.pi * 301000.0 * np.arange(len(x)) / 2048000.0)
    return dabtx.add_awgn(x, snr_db, seed=seed, signal_power=p)


def fib_passes(oracle, name, snr_db):
    ok = {False: 0, True: 0}
    for seed in SEEDS:
        clean = dabtx.DabTx(seed=seed).frames(4, noise_floor=0)
        x = channel(clean, name, snr_db, seed + 0x7000)
        for f in range(4):
            fr = ofdmref.frame(x, f * TF + TNULL + 305)
            for weighted in (False, True):
                s = softref.soft(fr["r1"][:3], weighted) if weighted else fr["soft"][:3]
                _, crc = oracle.fic_decode(np.ascontiguousarray(s).reshape(-1))
                ok[weighted] += int(crc.sum())
    return ok[False], ok[True]


@pytest.fixture(scope="module")
def gains(oracle):
    return {pt: fib_passes(oracle, *pt) for pt in POINTS}


def test_weighted_gain_cpu(gains):
    print({f"{n}@{s}dB": v for (n, s), v in gains.items()})
    for pt, (ref, wt) in gains.items():
        assert wt >= ref, (pt, ref, wt)
    # 144 FIBs per point; at these seeds: AWGN 141 / 141, two paths 1 / 73 and 57 / 143, three paths 9 / 78 and 86 / 143, tone 144 / 144
    for pt in (("2path", 5.0), ("3path", 5.0)):
        ref, wt = gains[pt]
        assert wt >= 137 and ref <= 90 and wt - ref >= 50, (pt, ref, wt)
    ref, wt = gains[("2path", 5.0)]
    assert wt - ref >= 80, (ref, wt)
    assert gains[("tone", 4.0)][1] >= 140
