"""Robust acquisition of welle.io_b200/csrc/acq_core.cuh compiled as host C++ (tests/host_emul/emul_acq.cpp) against the float64 numpy
restatement (tests/acqref.py): block levels within 2e-5, times the tone's amplitude over the ensemble's beside a tone (the float32
transform's error in the weak bins), depths within 3.1 times that in dB, the chosen window equal wherever the best two candidates are
further apart than that, and the excised bins equal.  Inputs: clean frames, AWGN from -4 to 10 dB, two and three paths, +-35 kHz,
a 150 ppm clock, tones on and off the bin grid at 10 to 40 dB above the ensemble, noise only, all-zero and NaN samples.  Also checks
the rule itself: the null is found with the window inside it at 0 dB and beside a 40 dB tone, and not on noise only."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import acqref
import dabtx
from conftest import ROOT

HERE = os.path.join(ROOT, "tests", "host_emul")
SPAN = 198151          # what a caller's step buffer holds at least (plan_kernel's `need`)
LV_TOL = 2e-5


def tol(kind):
    """level tolerance: the float32 transform's error grows with a tone's amplitude"""
    return LV_TOL * (10 ** (float(kind[4:].split("_")[0]) / 20) if kind.startswith("tone") else 1.0)


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_acq") / "libemul_acq.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "emul_acq.cpp")])
    lib = C.CDLL(so)
    lib.emul_acq_levels.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    lib.emul_acq_decide.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    lib.emul_acq_excise.argtypes = [C.c_void_p, C.c_void_p]
    lib.emul_acq_excise.restype = C.c_int
    lib.emul_acq_log2.argtypes = [C.c_float]
    lib.emul_acq_log2.restype = C.c_float
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def host(lib, y):
    """levels, envelope sums and decision (found, best, depth, median) of the host build over the span y"""
    y = np.ascontiguousarray(y, np.complex64)
    nb = min(len(y) // acqref.BLK, acqref.NB_MAX)
    lv, l1 = np.zeros(nb, np.float32), np.zeros(nb, np.float32)
    lib.emul_acq_levels(_p(y), nb, _p(lv), _p(l1))
    o, f = np.zeros(2, np.int32), np.zeros(2, np.float32)
    lib.emul_acq_decide(_p(lv), nb, _p(o), _p(f))
    return lv, l1, bool(o[0]), int(o[1]), float(f[0]), float(f[1])


@pytest.fixture(scope="module")
def clean():
    return dabtx.DabTx(seed=0xACC0).frames(3, noise_floor=0)


def signal(clean, kind):
    p = float(np.mean(np.abs(clean) ** 2))
    if kind == "clean":
        return clean
    if kind.startswith("awgn"):
        return dabtx.add_awgn(clean, float(kind[4:]), seed=11, signal_power=p)
    if kind == "two_paths":
        return dabtx.add_awgn(acqref.paths(clean, [(0, 1.0), (37, 0.7 - 0.3j)]), 3.0, seed=12, signal_power=p)
    if kind == "three_paths":
        return dabtx.add_awgn(acqref.paths(clean, [(0, 1.0), (37, 0.7 - 0.3j), (211, 0.5j)]), 3.0, seed=13, signal_power=p)
    if kind in ("plus35k", "minus35k"):
        return dabtx.add_awgn(dabtx.freq_shift(clean, 35000.0 if kind == "plus35k" else -35000.0), 3.0, seed=14, signal_power=p)
    if kind == "ppm150":
        return dabtx.add_awgn(acqref.resample_ppm(clean, 150.0), 3.0, seed=15, signal_power=p)
    if kind.startswith("tone"):            # tone<dB>_<on|off>
        db, grid = kind[4:].split("_")
        return acqref.tone(dabtx.add_awgn(clean, 0.0, seed=16, signal_power=p), 301000.0 if grid == "on" else 301500.0, float(db))
    raise ValueError(kind)


KINDS = ["clean"] + ["awgn%d" % s for s in (-4, -2, 0, 3, 6, 10)] + ["two_paths", "three_paths", "plus35k", "minus35k", "ppm150"] + \
        ["tone%d_%s" % (d, g) for d in (10, 20, 30, 40) for g in ("on", "off")]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("offset", [1000, 60001, 150000])
def test_levels_and_decision(emul, clean, kind, offset):
    y = signal(clean, kind)[offset:offset + SPAN]
    lv, l1, found, best, depth, med = host(emul, y)
    ref = acqref.levels(y)[:len(lv)]
    t = tol(kind)
    assert np.abs(lv - ref).max() < t, kind
    assert np.allclose(l1, acqref.l1sums(y)[:len(lv)], rtol=1e-5)
    rfound, rbest, rdepth, rmed, W = acqref.decide(ref)
    assert abs(depth - rdepth) < 3.1 * t and abs(med - rmed) < t
    second = np.sort(np.delete(W, rbest))[0]
    if second - W[rbest] > 2 * 9 * t:
        assert best == rbest
    if abs(rdepth - acqref.DEPTH_DB) > 3.1 * t:
        assert found == rfound
    # the rule: down to -4 dB, and beside every tone, the window lies inside the null that the span holds whole
    null_start = (-offset) % acqref.TF
    if null_start + acqref.TNULL + acqref.EDGE * acqref.BLK <= len(lv) * acqref.BLK:
        assert found, (kind, depth)
        assert null_start <= best * acqref.BLK + 256 and best * acqref.BLK + 2304 <= null_start + acqref.TNULL + 256, (kind, best, null_start)


def test_noise_only(emul):
    rng = np.random.default_rng(0xACC1)
    depths = []
    for i in range(12):
        y = ((rng.standard_normal(SPAN) + 1j * rng.standard_normal(SPAN)) * (0.01 * (i + 1))).astype(np.complex64)
        lv, _, found, _, depth, _ = host(emul, y)
        assert np.abs(lv - acqref.levels(y)[:len(lv)]).max() < LV_TOL
        assert not found
        depths.append(depth)
    assert max(depths) < 0.9


def test_zero_and_nan(emul):
    z = np.zeros(SPAN, np.complex64)
    lv, l1, found, best, depth, _ = host(emul, z)
    assert not found and depth == 0.0 and best == len(lv) - acqref.WIN and np.all(lv == -126.0) and np.all(l1 == 0)
    rng = np.random.default_rng(5)
    y = ((rng.standard_normal(SPAN) + 1j * rng.standard_normal(SPAN)) * 0.1).astype(np.complex64)
    y[5000:5300] = np.nan
    y[90000] = np.inf
    lv, _, found, _, depth, _ = host(emul, y)
    assert np.all(np.isfinite(lv)) and np.isfinite(depth)
    assert np.abs(lv - acqref.levels(y)[:len(lv)]).max() < LV_TOL


def test_log2(emul):
    x = np.concatenate([2.0 ** np.arange(-126, 128, 0.37), np.random.default_rng(1).uniform(1e-30, 1e30, 2000)]).astype(np.float32)
    got = np.array([emul.emul_acq_log2(float(v)) for v in x])
    assert np.abs(got - np.log2(x.astype(np.float64))).max() < 3e-5      # 3e-7 relative to |log2 x| <= 128


def prs_window_spectrum(clean, extra):
    """the 2048-point spectrum of a phase reference window (504 samples late) with an optional interferer"""
    w = clean[acqref.TNULL:acqref.TNULL + 2048].astype(np.complex128)
    n = np.arange(2048)
    for hz, db in extra:
        w = w + np.sqrt(np.mean(np.abs(w) ** 2) * 10 ** (db / 10)) * np.exp(2j * np.pi * hz * n / 2048000.0)
    return np.fft.fft(w).astype(np.complex64)


@pytest.mark.parametrize("extra", [[], [(301000.0, 20)], [(301500.0, 20)], [(301500.0, 40)], [(-500250.0, 30), (120000.0, 25)],
                                   [(760000.0, 30)]])
def test_excision(emul, clean, extra):
    X = prs_window_spectrum(dabtx.add_awgn(clean, 0.0, seed=3), extra)
    z = np.zeros(2048, np.uint8)
    n = emul.emul_acq_excise(_p(np.ascontiguousarray(X)), _p(z))
    ref = acqref.excise(X)
    assert np.array_equal(z.astype(bool), ref) and n == int(ref.sum())
    if not extra:
        assert n == 0
    else:
        for hz, _ in extra:
            assert z[int(round(hz / 1000.0)) % 2048]
