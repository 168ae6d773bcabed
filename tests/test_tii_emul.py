"""The device TII analysis (welle.io_b200/csrc/tii_core.cuh) compiled as host C++ (tests/host_emul/emul_tii.cpp) against the glue's host
analyser (welle.io_b200/host/tii.h, pinned to the unmodified TIIDecoder by test_figdb.py), frame by frame.  Comb, pattern, delay and
the number of measurements must be equal; within a frame the device reports in ascending (comb, pattern) order, so both sides are
compared in that order.  The error sums may differ where glibc's float atan2f / sinf / cosf round differently from the correctly
rounded values the device code uses; such differences are counted and printed."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import tiiref
from conftest import ROOT

HERE = os.path.join(ROOT, "tests", "host_emul")


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_tii") / "libemul_tii.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "emul_tii.cpp")])
    lib = C.CDLL(so)
    lib.emul_tii_run.restype = C.c_int
    lib.emul_tii_argmin.restype = C.c_int
    return lib


@pytest.fixture(scope="module")
def host():
    return tiiref.host_lib()


def emul_run(lib, nspec, pspec):
    nspec = np.ascontiguousarray(nspec, np.complex64); pspec = np.ascontiguousarray(pspec, np.complex64)
    n = len(nspec); cap = 9 * n + 16
    out = np.zeros(5 * cap, np.float32); info = np.zeros((n, 4), np.int32)
    k = lib.emul_tii_run(nspec.ctypes.data_as(C.c_void_p), pspec.ctypes.data_as(C.c_void_p), n, out.ctypes.data_as(C.c_void_p), cap, info.ctypes.data_as(C.c_void_p))
    meas = [(int(r[0]), int(r[1]), int(r[2]), int(r[3]), float(r[4])) for r in out[:5 * k].reshape(-1, 5)]
    return meas, info


def test_rank_tables_are_the_unordered_map_order(emul, host):
    """the two tie-order tables = the iteration order of a std::unordered_map<float, uint64_t> filled like analyse_phase: fresh, and
    after clear(); a second clear() gives the same order again, so two tables cover every report"""
    rank = np.zeros((2, 504), np.uint16)
    emul.emul_tii_rank(rank.ctypes.data_as(C.c_void_p))
    zeros = np.zeros(504, np.uint32)
    orders = []
    for clears in range(3):
        keys = np.zeros(504, np.int32)
        host.welle_b200_tii_map_argmin(zeros.ctypes.data_as(C.c_void_p), clears, keys.ctypes.data_as(C.c_void_p))
        assert sorted(keys.tolist()) == list(range(-4, 500))
        orders.append(keys)
    assert not np.array_equal(orders[0], orders[1])           # the two forms really differ
    assert np.array_equal(orders[1], orders[2])
    for t in range(2):
        assert np.array_equal(np.argsort(rank[t]) - 4, orders[t]), t


def test_argmin_ties_follow_the_map_order(emul, host):
    """smallest sum first; among equal sums the entry std::min_element meets first"""
    rng = np.random.default_rng(11)
    cases = [np.full(504, 7, np.uint32)]
    for _ in range(40):
        s = rng.integers(3, 40, 504).astype(np.uint32)
        tied = rng.choice(504, int(rng.integers(2, 30)), replace=False)
        s[tied] = 1                                           # several delays share the smallest sum
        cases.append(s)
    for s in cases:
        for t in range(2):
            keys = np.zeros(504, np.int32)
            want = host.welle_b200_tii_map_argmin(s.ctypes.data_as(C.c_void_p), t, keys.ctypes.data_as(C.c_void_p))
            assert emul.emul_tii_argmin(s.ctypes.data_as(C.c_void_p), t) == want


@pytest.mark.parametrize("tx_set", [
    [],
    [(4, 17, 23, 0.5)],
    [(4, 17, 23, 0.5), (11, 52, 140, 0.35)],
    [(2, 5, -3, 0.5), (13, 69, 311, 0.4), (21, 40, 77, 0.3)],
], ids=["none", "one", "two", "three"])
@pytest.mark.parametrize("snr_db", [15.0, 25.0, None], ids=["15dB", "25dB", "clean"])
def test_recordings_match_host_analyser(oracle, emul, host, tx_set, snr_db):
    nspec, pspec = tiiref.recording_spectra(oracle, tx_set, snr_db, 13, seed=0x711 + len(tx_set))
    want = tiiref.host_run_framed(host, nspec, pspec)
    got, info = emul_run(emul, nspec, pspec)
    assert len(got) == len(want)
    n, ndiff, worst = tiiref.compare(tiiref.by_frame(want), tiiref.by_frame(got))
    print(f"{len(tx_set)} transmitters, snr {snr_db}: {n} measurements, {ndiff} error values differ (largest {worst})")
    if tx_set:              # the strongest transmitter is found with its delay (weaker ones are not always, by either analyser)
        assert tuple(tx_set[0][:3]) in {(c, p, d) for _, c, p, d, _ in got}, got
    assert info[:, 3].sum() == 0


def test_nine_likely_combinations_are_analysed_and_ten_skipped(emul, host):
    """comb 2 with five active groups (C(5,4) = 5 patterns) + four combs with exactly four (1 each) = 9: every frame is analysed and the
    fifth frame reports all nine; one more comb with five (10) skips the frame"""
    rng = np.random.default_rng(9)
    nine = tiiref.pairs_of(2, 0b11111000) + sum((tiiref.pairs_of(c, 0b01010101) for c in (5, 9, 13, 17)), [])
    ten = tiiref.pairs_of(2, 0b11111000) + tiiref.pairs_of(7, 0b10111010)
    nspec, pspec = tiiref.active_pairs_spectra(rng, [nine] * 6 + [ten] * 6 + [nine] * 4)
    want = tiiref.host_run_framed(host, nspec, pspec)
    got, info = emul_run(emul, nspec, pspec)
    assert info[:6, 0].tolist() == [9] * 6 and info[6:12, 2].tolist() == [1] * 6 and info[6:12, 0].tolist() == [0] * 6
    assert info[4, 1] == 9 and info[15, 1] == 9                # 5 analyses: frames 0-4 and 5, 12-15
    assert len(got) == len(want) == 18
    n, ndiff, worst = tiiref.compare(tiiref.by_frame(want), tiiref.by_frame(got))
    print(f"9 / 10 likely combinations: {n} measurements, {ndiff} error values differ (largest {worst})")


def test_eviction_beyond_32_open_combinations(emul, host):
    """(1) random combinations beside a steady transmitter open more than 32 accumulators: until the first eviction the measurements are
    the host analyser's.  (2) the policy: the least recently analysed combination is replaced and starts over (the reference would keep
    it: DESIGN.md 5)"""
    rng = np.random.default_rng(32)
    frames = []
    for f in range(40):
        combs = rng.choice([c for c in range(24) if c != 6], int(rng.integers(1, 4)), replace=False)
        pairs = tiiref.pairs_of(6, tiiref.PATTERN_WORDS[33])
        for c in combs:
            pairs += tiiref.pairs_of(int(c), tiiref.PATTERN_WORDS[int(rng.integers(0, 70))])
        frames.append(pairs)
    nspec, pspec = tiiref.active_pairs_spectra(rng, frames)
    want = tiiref.host_run_framed(host, nspec, pspec)
    got, info = emul_run(emul, nspec, pspec)
    first = int(np.nonzero(info[:, 3])[0][0])
    assert 10 < first < 40
    n, ndiff, _ = tiiref.compare(tiiref.by_frame(want), tiiref.by_frame(got), frames=range(first))
    assert n >= 2
    print(f"noise run: first eviction in frame {first}, {n} measurements before it equal ({ndiff} error values differ)")
    # (2) X_i = (i % 24, i // 24): frames 0..31 open X_0..X_31; frame 32 analyses X_0 again and opens X_32, which replaces X_1;
    # frames 33..36 analyse X_0 and X_1
    X = [(i % 24, i // 24) for i in range(33)]
    sched = [[X[i]] for i in range(32)] + [[X[0], X[32]]] + [[X[0], X[1]]] * 5
    frames = [sum((tiiref.pairs_of(c, tiiref.PATTERN_WORDS[p]) for c, p in s), []) for s in sched]
    nspec, pspec = tiiref.active_pairs_spectra(rng, frames)
    got, info = emul_run(emul, nspec, pspec)
    want = tiiref.host_run_framed(host, nspec, pspec)
    assert info[:, 3].tolist() == [0] * 32 + [1, 1] + [0] * 4      # X_1 comes back in frame 33 and replaces X_2
    assert [(f, c, p) for f, c, p, _, _ in got] == [(35, 0, 0), (37, 1, 0)]
    assert [(f, c, p) for f, c, p, _, _ in want] == [(35, 0, 0), (36, 1, 0)]         # the reference kept X_1's first analysis
