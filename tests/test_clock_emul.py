"""Sample-clock tracking (DABB_CLOCK_TRACK) of welle.io_b200/csrc/clock_core.cuh compiled as host C++ (tests/host_emul/emul_clock.cpp)
against the numpy restatement (tests/clockref.py): the estimator over random status and start_index sequences with every kind of step,
the |d| bound, the n = 8 and n = 32 thresholds and resets; every carrier's phasor; and resample_clock."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import clockref
from conftest import ROOT

HERE = os.path.join(ROOT, "tests", "host_emul")


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_clock") / "libemul_clock.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "emul_clock.cpp")])
    lib = C.CDLL(so)
    lib.emul_clock_phasors.argtypes = [C.c_float, C.c_void_p]
    assert lib.emul_clock_state_size() == 16
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def run(lib, steps, S):
    st = np.zeros(16 * S, np.uint8)
    out = []
    for ev in steps:
        if ev[0] == "reset":
            lib.emul_clock_reset(_p(st), ev[1], ev[2])
            continue
        rec = np.zeros(S, clockref.CLOCK_DTYPE)
        ppm = np.zeros(S, np.float32); ap = np.zeros(S, np.float32); fr = np.zeros(S, np.int32)
        status = np.ascontiguousarray(ev[2], np.int32); idx = np.ascontiguousarray(ev[3], np.int32)
        lib.emul_clock_step(_p(st), S, ev[1], _p(status), _p(idx), _p(ppm), _p(ap), _p(fr))
        rec["ppm"], rec["applied_ppm"], rec["frames"] = ppm, ap, fr
        out.append(rec)
    return out


def random_steps(seed, S, n, p_dec=0.85, spread=70, ppm=60.0):
    rng = np.random.default_rng(seed)
    base = 504 + ppm * 196608e-6
    steps = []
    for i in range(n):
        if rng.random() < 0.03:
            f = int(rng.integers(0, S)); steps.append(("reset", f, int(rng.integers(1, S - f + 1)))); continue
        mode = clockref.CLOCK_OFF if rng.random() < 0.06 else clockref.CLOCK_TRACK
        status = np.where(rng.random(S) < p_dec, 0, rng.integers(1, 4, S)).astype(np.int32)
        idx = np.round(base + rng.normal(0, 2, S) + np.where(rng.random(S) < 0.05, rng.integers(-spread, spread + 1, S), 0)).astype(np.int32)
        steps.append(("step", mode, status, idx))
    return steps


def assert_same(got, want):
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        assert g.tobytes() == w.tobytes(), (i, g, w)


@pytest.mark.parametrize("seed", range(6))
def test_estimator_random_sequences(emul, seed):
    S = 16
    steps = random_steps(0xC10C + seed, S, 300, ppm=[-120, -50, 0, 50, 120, 300][seed])
    assert_same(run(emul, steps, S), clockref.records(steps, S))


def test_bound_and_thresholds(emul):
    """|d| = 64 counts and 65 does not; applied stays 0 until 8 frames are counted; the running mean turns into an average of 32"""
    S = 2
    steps = [("step", 1, [0, 0], [504 + 64, 504 + 65])]
    for i in range(60):
        steps.append(("step", 1, [0, 0], [504 + 64, 504 + 65 if i % 2 else 504 - 64 - (i % 3)]))
    steps += [("step", 1, [0, 0], [504 + (i % 7) - 3, 504 + 10]) for i in range(40)]
    got = run(emul, steps, S)
    assert_same(got, clockref.records(steps, S))
    fr = np.array([g["frames"] for g in got])
    ap = np.array([g["applied_ppm"] for g in got])
    assert fr[0, 0] == 0 and fr[1, 0] == 1 and fr[-1, 0] == 100
    first_applied = int(np.argmax(ap[:, 0] != 0))
    assert fr[first_applied - 1, 0] == 8            # the step after the 8th counted frame is the first derotated one
    assert np.all(ap[:first_applied, 0] == 0)
    assert clockref.records([("step", 1, [0], [504 + 65])] * 3, 1)[-1]["frames"][0] == 0


def test_flag_rules(emul):
    """NO_SYNC, ACQUIRING and OFF steps break the chain, NEED_SAMPLES does not; a reset clears everything; OFF keeps e and n"""
    S = 5
    idx = [520] * S
    steps = [("step", 1, [0] * S, idx)] * 12
    steps += [("step", 1, [1, 2, 3, 0, 0], idx), ("step", 0, [0] * S, idx), ("step", 1, [0] * S, idx)]
    steps += [("reset", 3, 1), ("step", 1, [0] * S, idx), ("step", 1, [0] * S, idx)]
    got = run(emul, steps, S)
    want = clockref.records(steps, S)
    assert_same(got, want)
    assert np.all(got[13]["ppm"] == 0) and np.all(got[13]["frames"] == 0)      # OFF writes zeros
    assert got[14]["frames"][0] == 11 and got[14]["frames"][4] == got[12]["frames"][4] == 12      # after OFF the first frame does not count
    assert got[-1]["frames"][3] == 1 and got[-2]["frames"][3] == 0            # reset: starts over


@pytest.mark.parametrize("ppm", [0.1, -0.1, 50.0, -50.0, 325.0, -325.0, 37.61234])
def test_phasors(emul, ppm):
    out = np.zeros(2 * 1537, np.float32)
    emul.emul_clock_phasors(ppm, _p(out))
    got = out[0::2].astype(np.float64) + 1j * out[1::2].astype(np.float64)
    want = clockref.phasor(np.arange(-768, 769), ppm)
    assert np.max(np.abs(got.real - want.real)) <= 2.0 ** -22
    assert np.max(np.abs(got.imag - want.imag)) <= 2.0 ** -22
    assert got[768] == 1.0


def test_derotate_and_resample():
    r1 = np.ones(clockref.K, np.complex64)
    d = clockref.derotate(r1, 100.0)
    k = clockref.CARRIER
    assert np.allclose(np.angle(d), 2 * np.pi * k * np.float64(np.float32(100.0)) * 1e-6 * 2552 / 2048)
    x = np.exp(2j * np.pi * 0.01 * np.arange(4096)).astype(np.complex64)
    y, eff = clockref.resample_clock(x, 50.0)
    assert len(y) == round(4096 * (1 + 50e-6)) and eff == 1e6 * (len(y) / 4096 - 1)
