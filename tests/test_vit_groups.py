"""The grouped codeword schedule of a sub-channel slot's Viterbi launch (welle.io_b200/csrc/vit_groups.cuh), built as host C++
(tests/host_emul/emul_vit_groups.cpp) on random memberships: every enabled codeword is decoded exactly once, a CTA holds codewords of
one profile and at most 128 of them, CTAs come in descending trellis length, and decision ranges are disjoint and inside the
allocation.  A fully selected slot with one profile gets the identity schedule of the ungrouped launch."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT

HERE = os.path.join(ROOT, "tests", "host_emul")
CW = 128


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_vit_groups") / "libemul_vit_groups.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "emul_vit_groups.cpp")])
    lib = C.CDLL(so)
    lib.emul_vit_schedule.restype = C.c_int
    return lib


def schedule(lib, prof_of, nsteps):
    prof_of = np.ascontiguousarray(prof_of, np.int32); nsteps = np.ascontiguousarray(nsteps, np.int32)
    S = len(prof_of); cap = 4 * S // CW + len(nsteps) + 2
    groups = np.zeros((cap, 5), np.int32); lst = np.zeros(max(4 * S, 1), np.int32)
    n_list = C.c_int32(0); dec = C.c_int64(0)
    n = lib.emul_vit_schedule(prof_of.ctypes.data_as(C.c_void_p), S, nsteps.ctypes.data_as(C.c_void_p), len(nsteps),
                              groups.ctypes.data_as(C.c_void_p), cap, lst.ctypes.data_as(C.c_void_p), C.byref(n_list), C.byref(dec))
    assert n > 0
    g = groups[:n]
    dec_off = g[:, 3].astype(np.int64) & 0xFFFFFFFF | (g[:, 4].astype(np.int64) << 32)
    return g[:, 0], g[:, 1], g[:, 2], dec_off, lst[:n_list.value], dec.value


def check(lib, prof_of, nsteps):
    prof_of = np.asarray(prof_of, np.int32); nsteps = np.asarray(nsteps, np.int32)
    prof, first, count, dec_off, lst, dec_words = schedule(lib, prof_of, nsteps)
    enabled = np.flatnonzero(prof_of >= 0)
    want = np.sort(np.concatenate([4 * enabled + c for c in range(4)])) if len(enabled) else np.zeros(0, np.int64)
    if not len(enabled):            # one empty CTA keeps the launch a valid grid
        assert len(prof) == 1 and count[0] == 0 and dec_words == 0 and len(lst) == 0
        return prof, first, count, dec_off, lst
    assert np.all((count >= 1) & (count <= CW))
    # the CTAs cover the list exactly once, in order
    assert first[0] == 0 and np.array_equal(first[1:], (first + count)[:-1]) and first[-1] + count[-1] == len(lst)
    assert np.array_equal(np.sort(lst), want)                                   # every enabled codeword exactly once
    for b in range(len(prof)):                                                  # one profile per CTA, the codewords' own
        cws = lst[first[b]:first[b] + count[b]]
        assert np.all(prof_of[cws // 4] == prof[b])
    steps = nsteps[prof]
    assert np.all(np.diff(steps) <= 0)                                          # longest codewords first
    size = steps.astype(np.int64) * CW
    assert dec_off[0] == 0 and np.array_equal(dec_off[1:], np.cumsum(size)[:-1]) and dec_off[-1] + size[-1] == dec_words
    # per profile at most one partial CTA
    for p in np.unique(prof):
        assert np.sum((prof == p) & (count < CW)) <= 1
    return prof, first, count, dec_off, lst


def test_single_stream(lib):
    prof, first, count, dec_off, lst = check(lib, [3], [2310, 1158, 774, 9222])
    assert list(prof) == [3] and list(count) == [4] and list(lst) == [0, 1, 2, 3]


def test_uniform_full_slot_is_the_identity(lib):
    S = 4096
    prof, first, count, dec_off, lst = check(lib, np.zeros(S, np.int32), [2310])
    assert np.array_equal(lst, np.arange(4 * S)) and np.all(count == CW)
    assert np.array_equal(dec_off, np.arange(len(prof), dtype=np.int64) * 2310 * CW)


def test_empty_slot(lib):
    check(lib, np.full(100, -1, np.int32), [2310, 774])


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_4096_streams_over_40_profiles(lib, seed):
    rng = np.random.default_rng(seed)
    nsteps = 24 * rng.choice(np.arange(1, 49) * 8, 40, replace=False) + 6       # distinct bitrates 8..384 kbit/s
    prof_of = rng.integers(-1, 40, 4096).astype(np.int32)                       # about 1 in 41 streams not enabled
    check(lib, prof_of, nsteps)


@pytest.mark.parametrize("n", [1, 31, 32, 33, 127, 128, 129])
def test_group_sizes(lib, n):
    """groups of n streams (4 n codewords) beside other profiles, with unselected streams interleaved"""
    rng = np.random.default_rng(n)
    S = 3 * n + 200
    prof_of = np.full(S, -1, np.int32)
    idx = rng.permutation(S)
    prof_of[idx[:n]] = 0; prof_of[idx[n:2 * n]] = 1; prof_of[idx[2 * n:2 * n + 100]] = 2
    prof, first, count, dec_off, lst = check(lib, prof_of, [774, 2310, 2310])    # equal lengths: profile order by index
    for p in range(3):
        k = n if p < 2 else 100
        assert count[prof == p].sum() == 4 * k and (prof == p).sum() == -(-4 * k // CW)
    assert list(dict.fromkeys(prof.tolist())) == [1, 2, 0]


def test_streams_removed_in_between(lib):
    """a membership changed step by step like select / remove calls do: the schedule is rebuilt from scratch every time"""
    rng = np.random.default_rng(7)
    S = 1000
    nsteps = np.array([1158, 2310, 9222, 774, 3462], np.int32)
    prof_of = np.full(S, -1, np.int32)
    for it in range(40):
        a = int(rng.integers(0, S)); b = int(rng.integers(a, min(S, a + 300)) + 1)
        prof_of[a:b] = -1 if rng.random() < 0.3 else int(rng.integers(0, len(nsteps)))
        check(lib, prof_of, nsteps)
