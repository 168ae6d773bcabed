"""Diversity combining of welle.io_b200/csrc/combine_core.cuh compiled as host C++ (tests/host_emul/emul_combine.cpp) against the float64
numpy restatement (tests/combineref.py): the null-symbol noise power, the contributor rule (offsets at the 504-sample edge, a leader or
member without a frame, zero / inf / NaN noise), and the combined softbits of 1 to 8 members under both demaps, with faded members and a
member whose r1 is all zero.  Softbits differ from the float64 value only at rounding boundaries: by at most 1, for at most 0.5 % of
them.  The sum is taken in ascending stream order: the reference demap of it is bit for bit that of the float32 sum in that order."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import combineref
import softref
from conftest import ROOT

HERE = os.path.join(ROOT, "tests", "host_emul")
K = 1536
RATE = 0.005


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_combine") / "libemul_combine.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "emul_combine.cpp")])
    lib = C.CDLL(so)
    lib.emul_combine_select.restype = C.c_uint32
    lib.emul_combine_select.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.emul_combine_symbol.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_uint32, C.c_int, C.c_void_p]
    lib.emul_combine_noise.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def host_noise(lib, y):
    y = np.ascontiguousarray(y, np.complex64).reshape(-1, combineref.TNULL)
    out = np.zeros(len(y), np.float32)
    lib.emul_combine_noise(_p(y), len(y), _p(out))
    return out


def host_symbol(lib, r1, nz, mask, weighted):
    r1 = np.ascontiguousarray(r1, np.complex64)
    nz = np.ascontiguousarray(nz, np.float32)
    out = np.zeros(2 * K, np.int8)
    lib.emul_combine_symbol(_p(r1), len(r1), _p(nz), int(mask), int(weighted), _p(out))
    return out


def test_noise(emul):
    rng = np.random.default_rng(0xC0B1)
    y = (rng.normal(0, 1, (6, combineref.TNULL)) + 1j * rng.normal(0, 1, (6, combineref.TNULL))) * np.array([1e-3, 0.1, 1, 30, 1e4, 1e-17])[:, None]
    got = host_noise(emul, y)
    want = combineref.noise(y.astype(np.complex64))
    assert np.all(np.abs(got - want) <= 1e-5 * want), (got, want)
    # the fixed order: partial sums of i = t mod 256 in ascending i, then the partials in order (float32, each operation rounded)
    assert np.array_equal(got, combineref.noise_f32(y))
    z = np.zeros((3, combineref.TNULL), np.complex64)
    z[1, 7] = np.inf; z[2, 100] = np.nan
    g = host_noise(emul, z)
    assert g[0] == 0 and np.isinf(g[1]) and np.isnan(g[2])


def test_select(emul):
    rng = np.random.default_rng(0xC0B2)
    specials = [0.0, np.inf, -np.inf, np.nan, -1.0, 1e-30, 3e38]
    for case in range(4000):
        n = int(rng.integers(1, 9)); lpos = int(rng.integers(0, n))
        dec = (rng.random(n) < 0.8).astype(np.int32)
        a = (1_000_000 + rng.integers(-520, 521, n)).astype(np.int64)
        if rng.random() < 0.3:
            a[int(rng.integers(0, n))] = a[lpos] + int(rng.choice([-505, -504, 504, 505]))
        nz = rng.uniform(1e-4, 10, n).astype(np.float32)
        for i in range(n):
            if rng.random() < 0.1:
                nz[i] = specials[int(rng.integers(0, len(specials)))]
        got = emul.emul_combine_select(n, lpos, _p(dec), _p(a), _p(nz))
        want = combineref.select(dec, a, nz, lpos)
        assert got == want, (case, n, lpos, dec, a, nz, got, want)


def members(rng, n, fade=True):
    """r1 of n antennas seeing one DQPSK symbol through independent channels and noise: [n, K] complex64"""
    sym = np.exp(1j * (np.pi / 4 + np.pi / 2 * rng.integers(0, 4, K)))
    out = []
    for i in range(n):
        h = rng.normal(0, 1, K) + 1j * rng.normal(0, 1, K) if fade else np.ones(K)
        nse = (rng.normal(0, 1, K) + 1j * rng.normal(0, 1, K)) * rng.uniform(0.05, 1.0)
        out.append(np.abs(h) ** 2 * sym * rng.uniform(0.1, 50) + nse)
    return np.asarray(out, np.complex64)


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("n", range(1, 9))
def test_combined_softbits(emul, n, weighted):
    rng = np.random.default_rng(0xC0B3 + 16 * n + int(weighted))
    diff = []
    for trial in range(12):
        r1 = members(rng, n, fade=trial % 3 != 0)
        nz = rng.uniform(1e-3, 5, n).astype(np.float32)
        if n > 1 and trial % 4 == 1:
            r1[int(rng.integers(0, n))] = 0                   # a member of zero r1
        mask = int(rng.integers(1, 1 << n))
        got = host_symbol(emul, r1, nz, mask, weighted)
        diff.append(combineref.compare(got, combineref.combined(r1, nz, mask), weighted, RATE))
        if not weighted:                                      # the order: exactly the float32 sum in ascending stream order
            assert np.array_equal(got, softref.soft_reference_f32(combineref.combined_f32(r1, nz, mask)))
    print(n, weighted, max(diff))


def test_order_matters(emul):
    """the float32 sum depends on the order; the library's is ascending stream order"""
    rng = np.random.default_rng(0xC0B4)
    r1 = members(rng, 8)
    nz = rng.uniform(1e-3, 5, 8).astype(np.float32)
    asc, rev = combineref.combined_f32(r1, nz, 0xFF), combineref.combined_f32(r1, nz, 0xFF, order=range(7, -1, -1))
    assert not np.array_equal(asc.view(np.uint64), rev.view(np.uint64))
    assert np.array_equal(host_symbol(emul, r1, nz, 0xFF, False), softref.soft_reference_f32(asc))


@pytest.mark.parametrize("weighted", [False, True])
def test_unusable_noise(emul, weighted):
    """a member whose N is 0, inf or NaN is not selected; selected anyway (host function), it would poison the sum: the rule keeps it
    out, and the remaining members combine as if it were absent"""
    rng = np.random.default_rng(0xC0B5 + int(weighted))
    r1 = members(rng, 4)
    for bad in (0.0, np.inf, np.nan):
        nz = np.array([0.5, bad, 2.0, 1.0], np.float32)
        dec = np.ones(4, np.int32); a = np.full(4, 5000, np.int64)
        m = emul.emul_combine_select(4, 0, _p(dec), _p(a), _p(nz))
        assert m == 0b1101
        got = host_symbol(emul, r1, nz, m, weighted)
        assert np.array_equal(got, host_symbol(emul, r1[[0, 2, 3]], nz[[0, 2, 3]], 0b111, weighted))
        combineref.compare(got, combineref.combined(r1, nz, m), weighted, RATE)
    # the leader's own noise unusable: it decodes alone
    nz = np.array([np.nan, 1.0, 1.0, 1.0], np.float32)
    assert emul.emul_combine_select(4, 0, _p(np.ones(4, np.int32)), _p(np.zeros(4, np.int64)), _p(nz)) == 1


FLT_MIN, SUBNORMAL = np.float32(2.0 ** -126), np.float32(2.0 ** -140)


def _edge_cases(rng):
    """(name, r1 [3, K], N [3], contributor mask) at the scale edges of the combination"""
    r1 = members(rng, 3)
    out = []
    for tiny in (FLT_MIN, SUBNORMAL):                         # r1 / N overflows to +-inf on most carriers, stays finite on the rest
        out.append((f"N {tiny:g}", r1, np.array([0.5, tiny, 2.0], np.float32), 0b111))
    r = r1.copy(); r[2] = -r[0]                               # +inf and -inf terms of two members: NaN in R
    out.append(("opposite infinities", r, np.array([SUBNORMAL, 1.0, SUBNORMAL], np.float32), 0b111))
    r = r1.copy(); r[1] = -r[0]; r[1, 1::2] *= 0.5            # R exactly 0 on every other carrier (and -0 in a component)
    r[0, ::5] = r[0, ::5].real                                # some components 0 in both members
    r[1, ::5] = -r[0, ::5]
    out.append(("R = 0", r, np.array([0.75, 0.75, 1.0], np.float32), 0b011))
    r = r1.copy()                                             # inf and NaN in one member's r1
    r[1, ::7] = np.inf; r[1, 3::7] = complex(np.nan, 1.0); r[1, 5::11] = complex(-np.inf, np.inf); r[1, 6::13] = complex(2.0, np.nan)
    out.append(("inf / NaN in r1", r, np.array([0.5, 1.5, 2.0], np.float32), 0b111))
    return out


@pytest.mark.parametrize("weighted", [False, True])
def test_scale_edges(emul, weighted):
    """the combined softbits where R leaves the finite range: a valid but tiny N (FLT_MIN, subnormal) whose quotients overflow to
    +-inf, infinite terms of opposite signs (NaN), R exactly 0, inf and NaN in one member's r1.  The reference demap is bit for bit
    softref.soft_reference_f32 of the float32 sum in ascending stream order; a carrier whose R is not finite, or 0, gets softbit 0 (DESIGN
    5: NaN gives 0); a symbol with a level that is not finite has G = 0, so the weighted demap is the reference demap there, and elsewhere
    it is the restatement of tests/softref.py.  (The host build's reciprocal is the IEEE quotient; for a combined level l1 >= 2^126 the
    device's flushes to 0, the demap's documented range, DESIGN 5.)"""
    rng = np.random.default_rng(0xC0B6 + int(weighted))
    for name, r1, nz, mask in _edge_cases(rng):
        assert emul.emul_combine_select(3, 0, _p(np.ones(3, np.int32)), _p(np.zeros(3, np.int64)), _p(nz)) == 0b111, name   # tiny N is valid
        got = host_symbol(emul, r1, nz, mask, weighted)
        R = combineref.combined_f32(r1, nz, mask)
        ref = softref.soft_reference_f32(R)
        re_bad = ~np.isfinite(R.real) | ~np.isfinite(R.imag) | (R == 0)
        assert not got[:K][re_bad].any() and not got[K:][re_bad].any(), name
        if name != "R = 0":
            assert re_bad.sum() > K // 8, (name, int(re_bad.sum()))
        else:
            assert (R == 0).sum() >= K // 2 and got[:K].any(), name
        if not weighted:
            assert np.array_equal(got, ref), (name, int((got != ref).sum()))
        elif not np.isfinite(softref.levels(R)[2]).all():
            assert np.array_equal(got, host_symbol(emul, r1, nz, mask, False)) and np.array_equal(got, ref), name
        else:
            softref.check(R, got)
