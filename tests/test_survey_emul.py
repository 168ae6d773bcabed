"""The spectrum survey and the candidate detector without a GPU: the host build of welle.io_b200/csrc/survey_core.cuh
(tests/host_emul/emul_survey.cpp: the kernel's transform, chunking and summation order; the library's detector) against the numpy
restatement of the definitions (tests/surveyref.py).

Spectrum bound (the GPU test uses the same): |P_j - P_ref_j| <= 1e-4 P_ref_j + 1e-7 mean(P_ref).  Each bin is an fp32 radix-2 transform:
its error is about sqrt(log2 nfft) 2^-24 of the segment's rms bin amplitude, which the second term covers where P_j is small, and a
relative 1e-6 or so where it is not.  The detector must give exactly the numpy lists; every synthetic case keeps its scores at least
0.5 dB away from the 6 dB threshold."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import chanref
import surveyref
from conftest import ROOT

HERE = os.path.join(ROOT, "tests", "host_emul")
THR = 6.0


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_survey") / "libemul_survey.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "emul_survey.cpp")])
    lib = C.CDLL(so)
    lib.emul_survey.argtypes = [C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_int64, C.c_void_p]
    lib.emul_survey_candidates.argtypes = [C.c_void_p, C.c_int32, C.c_int64, C.c_float, C.c_void_p, C.c_int32, C.c_void_p]
    return lib


def emul_psd(lib, raw, fmt, n_inputs, nfft, in_len):
    raw = np.ascontiguousarray(raw)
    stride = raw.nbytes // chanref.BYTES[fmt] // n_inputs
    psd = np.zeros((n_inputs, nfft), np.float32)
    assert lib.emul_survey(raw.ctypes.data, fmt, stride, n_inputs, nfft, in_len, psd.ctypes.data) == 0
    return psd


def emul_candidates(lib, psd, R, cap=4096, min_db=THR):
    psd = np.ascontiguousarray(psd, np.float32)
    out = np.zeros(max(cap, 1), surveyref.CAND_DTYPE)
    n = C.c_int32()
    assert lib.emul_survey_candidates(psd.ctypes.data, len(psd), R, min_db, out.ctypes.data, cap, C.byref(n)) == 0
    return out[:min(cap, n.value)], n.value


def within_bound(p, ref):
    return np.all(np.abs(p.astype(np.float64) - ref) <= 1e-4 * ref + 1e-7 * ref.mean())


def raw_input(rng, fmt, n):
    if fmt == chanref.IQ_CF32:
        t = np.arange(n)
        x = (rng.standard_normal(n) + 1j * rng.standard_normal(n)) * 0.1 + np.exp(2j * np.pi * 0.123457 * t)   # a tone over noise
        return x.astype(np.complex64).view(np.uint8)
    return rng.integers(0, 256, n * chanref.BYTES[fmt], dtype=np.uint8)


@pytest.mark.parametrize("nfft", [1024, 2048, 4096, 8192, 16384])
@pytest.mark.parametrize("fmt", [0, 1, 2, 3, 4])
def test_transform_matches_definition(emul, nfft, fmt):
    """every FFT size and format, two inputs, an odd in_len whose tail past the last segment is not read"""
    rng = np.random.default_rng(nfft + fmt)
    in_len = 5 * nfft // 2 + 777
    raw = np.stack([raw_input(rng, fmt, in_len) for _ in range(2)])
    psd = emul_psd(emul, raw, fmt, 2, nfft, in_len)
    for i in range(2):
        ref = surveyref.spectrum_raw(raw[i], fmt, nfft)
        assert within_bound(psd[i], ref), (i, np.max(np.abs(psd[i] - ref) / (ref + 1e-3 * ref.mean())))


def test_many_segments_and_chunks(emul):
    """enough segments for several chunks (the float chunk sums and the double total)"""
    rng = np.random.default_rng(5)
    nfft, in_len = 1024, 1024 * 300 + 5
    raw = raw_input(rng, 0, in_len)
    psd = emul_psd(emul, raw, 0, 1, nfft, in_len)
    assert within_bound(psd[0], surveyref.spectrum_raw(raw, 0, nfft))


def test_refusals(emul):
    psd = np.full(1024, 7.0, np.float32)
    raw = np.zeros(4096 * 8, np.uint8)
    for nfft, in_len, stride in ((512, 2048, 2048), (1536, 2048, 2048), (32768, 40000, 40000), (1024, 1023, 2048), (1024, 2048, 2047)):
        assert emul.emul_survey(raw.ctypes.data, 0, stride, 1, nfft, in_len, psd.ctypes.data) == -3
    assert np.all(psd == 7.0)
    n = C.c_int32()
    out = np.zeros(4, surveyref.CAND_DTYPE)
    assert emul.emul_survey_candidates(psd.ctypes.data, 1000, 2048000, THR, out.ctypes.data, 4, C.byref(n)) == -3
    assert emul.emul_survey_candidates(psd.ctypes.data, 1024, 0, THR, out.ctypes.data, 4, C.byref(n)) == -3
    assert emul.emul_survey_candidates(psd.ctypes.data, 1024, 2048000, THR, None, 4, C.byref(n)) == -3
    assert emul.emul_survey_candidates(psd.ctypes.data, 1024, 2048000, THR, out.ctypes.data, -1, C.byref(n)) == -3


# ---------------------------------------------------------------------------------------------------------------- detector

def floor_spectrum(rng, R, nfft, level=1.0):
    return level * np.exp(rng.normal(0.0, 0.25, nfft))                # +-1 dB or so of ripple, no ties


def add_plateau(P, R, f0, width, gain_db):
    f = (np.arange(len(P)) - len(P) // 2) * R / len(P)
    P[np.abs(f - f0) <= width / 2] *= 10 ** (gain_db / 10)
    return P


def case(name):
    rng = np.random.default_rng(abs(hash(name)) % 2 ** 32)
    if name == "one plateau":
        R, nfft = 10000000, 4096
        return R, add_plateau(floor_spectrum(rng, R, nfft), R, 1234000, 1536000, 20), 1
    if name == "raster neighbours, one 20 dB stronger":
        R, nfft = 10000000, 4096
        P = floor_spectrum(rng, R, nfft)
        for f, g in ((-1712000, 15), (0, 35), (1712000, 15)):
            add_plateau(P, R, f, 1536000, g)
        return R, P, 3
    if name == "mistuned 2.048 Msps":
        R, nfft = 2048000, 1024
        return R, add_plateau(floor_spectrum(rng, R, nfft), R, 200000, 1536000, 20), 1
    if name == "plateau cut by the band edge":
        R, nfft = 4096000, 1024
        return R, add_plateau(floor_spectrum(rng, R, nfft), R, -1700000, 1536000, 20), None
    if name == "7 MHz plateau":
        R, nfft = 20000000, 8192
        return R, add_plateau(floor_spectrum(rng, R, nfft), R, 500000, 7000000, 20), 0
    if name == "DC spike in a guard":
        R, nfft = 4096000, 1024
        P = add_plateau(floor_spectrum(rng, R, nfft), R, 856000, 1536000, 20)
        P[nfft // 2] *= 1e4
        return R, P, 1
    if name == "flat noise":
        R, nfft = 8192000, 2048
        return R, floor_spectrum(rng, R, nfft), 0
    if name == "zeros":
        return 2048000, np.zeros(1024), 0
    raise KeyError(name)


CASES = ["one plateau", "raster neighbours, one 20 dB stronger", "mistuned 2.048 Msps", "plateau cut by the band edge", "7 MHz plateau",
         "DC spike in a guard", "flat noise", "zeros"]


@pytest.mark.parametrize("name", CASES)
def test_detector_matches_definition(emul, name):
    R, P, expect = case(name)
    P = P.astype(np.float32)
    want = surveyref.candidates(P, R, THR)
    got, n = emul_candidates(emul, P, R)
    print(name, [(int(o), float(s)) for o, s, _ in got])
    assert n == len(want) and got.tobytes() == want.tobytes(), (got, want)
    if expect is not None:
        assert n == expect, (name, got)
    s = surveyref.scores(P, R)
    for o, sc, _ in got:                                      # away from the threshold: the lists cannot hinge on a last-bit difference
        assert sc >= THR + 0.5, (name, o, sc)
    if n == 0 and np.isfinite(s).any():
        assert np.nanmax(s) <= THR - 0.5, (name, np.nanmax(s))


def test_candidate_offsets():
    """the plateau cases find their centres within two bins.  The mistuned 2.048 Msps plateau lies partly beyond the centres the
    detector considers (|f_c| <= 256 kHz), so its run is cut there and the midpoint falls short; it stays within the +-35 kHz the
    decoder's coarse corrector pulls in"""
    for name, centres, tol in (("one plateau", [1234000], None), ("raster neighbours, one 20 dB stronger", [-1712000, 0, 1712000], None),
                               ("mistuned 2.048 Msps", [200000], 35000), ("DC spike in a guard", [856000], None)):
        R, P, _ = case(name)
        tol = 2 * R / len(P) if tol is None else tol
        got = surveyref.candidates(P.astype(np.float32), R, THR)
        assert len(got) == len(centres) and all(abs(int(o) - c) <= tol for o, c in zip(got["offset_hz"], centres)), (name, got)


def test_cap_smaller_than_count(emul):
    R, P, _ = case("raster neighbours, one 20 dB stronger")
    P = np.ascontiguousarray(P, np.float32)
    out = np.zeros(3, surveyref.CAND_DTYPE)
    out["offset_hz"] = 12345
    n = C.c_int32()
    assert emul.emul_survey_candidates(P.ctypes.data, len(P), R, THR, out.ctypes.data, 1, C.byref(n)) == 0
    want = surveyref.candidates(P, R, THR)
    assert n.value == 3 and out[:1].tobytes() == want[:1].tobytes() and list(out["offset_hz"][1:]) == [12345, 12345]
    assert emul.emul_survey_candidates(P.ctypes.data, len(P), R, THR, None, 0, C.byref(n)) == 0 and n.value == 3


@pytest.mark.parametrize("R", [2048000, 2400000, 10000000, 20000000, 61440000])
def test_fft_size_rule(R):
    n = surveyref.nfft_for_rate(R)
    assert R / n <= 4000 and (n == 1024 or R / (n // 2) > 4000)
    assert {2048000: 1024, 20000000: 8192, 61440000: 16384}.get(R, n) == n
