"""The wideband channelizer without a GPU: the filter meets its specification at every listed rate, and the host build of
welle.io_b200/csrc/chan_core.cuh (tests/host_emul/emul_chan.cpp, the kernel's own arithmetic and summation order) matches the float64
restatement of the definition (tests/chanref.py).

Bound (the GPU test uses the same): rms error <= 1e-5 x rms(y_ref) and largest error <= 1e-4 x rms(y_ref).  It holds because every
term of an output's sum is one float product of a tap (rounded once from double, relative error 2^-24) and a mixed sample (the phase
-2 k / R rounded to float, |error| < 2^-23 half turns, about 4e-7 rad; sincospi within an ulp), and the T terms are added in fp32
into two accumulators, so rounding errors grow like sqrt(T) 2^-24 |partial sum| (T <= 1559 here: about 3e-6 of the output's scale)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import chanref
from conftest import ROOT

HERE = os.path.join(ROOT, "tests", "host_emul")
RMS_BOUND, MAX_BOUND = 1e-5, 1e-4


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_chan") / "libemul_chan.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "emul_chan.cpp")])
    lib = C.CDLL(so)
    lib.emul_chan_geometry.argtypes = [C.c_int64, C.c_void_p]
    lib.emul_chan_offset_ok.argtypes = [C.c_int64, C.c_int64]
    lib.emul_chan_taps.argtypes = [C.c_int64, C.c_void_p]
    lib.emul_chan_run.argtypes = [C.c_int64, C.c_int, C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.c_void_p]
    return lib


def emul_taps(lib, R):
    L, M, T = chanref.geometry(R)
    h = np.zeros(L * T, np.float32)
    lib.emul_chan_taps(R, h.ctypes.data)
    return h


def emul_run(lib, R, fmt, f, raw, in_start, out_start, out_len):
    raw = np.ascontiguousarray(raw)
    in_len = raw.nbytes // chanref.BYTES[fmt]
    out = np.zeros(2 * out_len, np.float32)
    rc = lib.emul_chan_run(R, fmt, f, raw.ctypes.data, in_start, in_len, out_start, out_len, out.ctypes.data)
    assert rc == 0, rc
    return out.view(np.complex64)


def raw_signal(rng, fmt, n):
    """n random samples in format fmt (raw bytes / complex64)"""
    if fmt == chanref.IQ_CF32:
        return (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(np.complex64)
    return rng.integers(0, 256, n * chanref.BYTES[fmt], dtype=np.uint8)


@pytest.mark.parametrize("R", chanref.RATES)
def test_geometry_and_taps(emul, R):
    g = np.zeros(4, np.int32)
    assert emul.emul_chan_geometry(R, g.ctypes.data) == 0
    L, M, T = chanref.geometry(R)
    assert g.tolist() == [L, M, T, (T + 3) // 4 * 4]
    h = emul_taps(emul, R)
    want = chanref.taps(R)
    assert np.max(np.abs(h - want)) <= 2 * np.finfo(np.float32).eps * np.max(np.abs(want))
    assert abs(float(h.astype(np.float64).sum()) - L) < 1e-5 * L


@pytest.mark.parametrize("R", chanref.RATES)
def test_filter_specification(emul, R):
    """at most 0.01 dB ripple for |f| <= 768 kHz and at least 70 dB attenuation from 944 kHz to half the prototype's rate, on a grid of
    500 Hz or finer"""
    h = emul_taps(emul, R)
    f, db = chanref.response_db(h, R)
    pb, sb = db[f <= 768000], db[f >= 944000]
    print(f"R {R}: ripple {pb.max() - pb.min():.4f} dB, attenuation {-sb.max():.2f} dB")
    assert pb.max() - pb.min() <= 0.01 and np.abs(pb).max() <= 0.01
    assert sb.max() <= -70


def test_refusals(emul):
    g = np.zeros(4, np.int32)
    for R in (2047999, 64000001, 2048001, 9999999):          # out of range, or L > 1024
        assert emul.emul_chan_geometry(R, g.ctypes.data) == -6, R
    for R in (64000000, 2050000, 2000 * 1023 * 3):
        assert emul.emul_chan_geometry(R, g.ctypes.data) == 0, R
    assert emul.emul_chan_offset_ok(10000000, 5000000 - 768000) == 1
    assert emul.emul_chan_offset_ok(10000000, -(5000000 - 768000)) == 1
    assert emul.emul_chan_offset_ok(10000000, 5000000 - 767999) == 0
    assert emul.emul_chan_offset_ok(2048000, 256001) == 0 and emul.emul_chan_offset_ok(2048000, -256000) == 1


def offsets(R):
    edge = R // 2 - 768000
    return sorted({0, edge, -edge} | ({1712000, -1712000} if 1712000 <= edge else set()))


@pytest.mark.parametrize("R", chanref.RATES)
def test_matches_definition(emul, R):
    rng = np.random.default_rng(R % 9973)
    L, M, T = chanref.geometry(R)
    for f in offsets(R):
        for out_start in (0, 5, (1 << 40) * L // M + 3):
            out_len = 300
            first, end = chanref.input_range(R, out_start, out_len)
            in_start = first - 7
            x = raw_signal(rng, chanref.IQ_CF32, end - in_start + 5)
            y = emul_run(emul, R, chanref.IQ_CF32, f, x, in_start, out_start, out_len)
            want = chanref.channelize(chanref.convert(x, 0), in_start, R, f, out_start, out_len)
            rms, mx = chanref.error_ratio(y, want)
            assert rms <= RMS_BOUND and mx <= MAX_BOUND, (f, out_start, rms, mx)


@pytest.mark.parametrize("fmt", [chanref.IQ_CF32, chanref.IQ_U8, chanref.IQ_S8, chanref.IQ_S16LE, chanref.IQ_S16BE])
def test_every_format(emul, fmt):
    R, f = 2400000, 100000
    rng = np.random.default_rng(fmt)
    first, end = chanref.input_range(R, 1000, 500)
    raw = raw_signal(rng, fmt, end - first)
    y = emul_run(emul, R, fmt, f, raw, first, 1000, 500)
    want = chanref.channelize(chanref.convert(raw, fmt), first, R, f, 1000, 500)
    rms, mx = chanref.error_ratio(y, want)
    assert rms <= RMS_BOUND and mx <= MAX_BOUND, (rms, mx)


@pytest.mark.parametrize("R", [2400000, 10000000, 61440000])
def test_calls_of_any_size_give_the_same_bits(emul, R):
    rng = np.random.default_rng(3)
    f = 1712000 if R > 4 * 1712000 else 0
    start, total = 12345, 4000
    first, end = chanref.input_range(R, start, total)
    x = raw_signal(rng, chanref.IQ_S16LE, end - first)
    whole = emul_run(emul, R, chanref.IQ_S16LE, f, x, first, start, total)
    parts, m = [], start
    for n in (1, 7, 256, 1000, 999, total - 2263):
        parts.append(emul_run(emul, R, chanref.IQ_S16LE, f, x, first, m, n))
        m += n
    assert m == start + total
    assert np.concatenate(parts).view(np.uint32).tolist() == whole.view(np.uint32).tolist()


@pytest.mark.parametrize("R", chanref.RATES)
def test_input_range_is_the_definition(emul, R):
    """the span outputs need is what the sum reads: exactly that span is accepted, without its first or its last sample it is refused"""
    L, M, T = chanref.geometry(R)
    for out_start, out_len in ((0, 1), (17, 64), (L * 3 + 1, 2 * L + 5)):
        first, end = chanref.input_range(R, out_start, out_len)
        assert first == (out_start * M) // L - T + 1 and end == ((out_start + out_len - 1) * M) // L + 1
        x = raw_signal(np.random.default_rng(1), chanref.IQ_CF32, end - first)
        emul_run(emul, R, chanref.IQ_CF32, 0, x, first, out_start, out_len)
        out = np.zeros(2 * out_len, np.float32)
        assert emul.emul_chan_run(R, 0, 0, x[1:].ctypes.data, first + 1, end - first - 1, out_start, out_len, out.ctypes.data) == -2
        assert emul.emul_chan_run(R, 0, 0, x.ctypes.data, first, end - first - 1, out_start, out_len, out.ctypes.data) == -2
