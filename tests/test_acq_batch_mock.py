"""batch_decode --acq on the test double of the ABI that records dabb_options.acquisition (tests/mock_backend/mock_dab_b200_acq.cpp):
--acq robust sets DABB_ACQ_ROBUST on every context the driver creates - the plain decode, the wideband decode, and the survey, locate
and confirmation contexts of --scan / --offset auto, each with the disable_coarse and freqsync_method it was created with - and writes
one .acq line "blocks depth_db found" per step in which a stream searched (tap 13); --acq reference, like no option, sets nothing and
writes no .acq file.  The .fic, .msc and .rs outputs do not change: the double's frame records come from the oracle."""
import os
import subprocess

import pytest

import dabtx
from conftest import ROOT

EXE = os.path.join(ROOT, "welle.io_b200", "batch_decode")


@pytest.fixture(scope="module")
def setup(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("acq_mock")
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "welle.io_b200", "host")])
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", str(tmp / "libdab_b200.so"),
                           os.path.join(ROOT, "tests", "mock_backend", "mock_dab_b200_acq.cpp"),
                           "-L" + os.path.join(ROOT, "oracle"), "-loracle", "-Wl,-rpath," + os.path.join(ROOT, "oracle")])
    iq = tmp / "ens.iq"
    dabtx.DabTx(seed=0xAC0).frames(10).tofile(iq)
    return tmp, str(iq)


def run(tmp, name, args, iq, contexts):
    out = tmp / name
    out.mkdir()
    log = tmp / f"{name}.log"
    env = dict(os.environ, LD_LIBRARY_PATH=str(tmp), DABB_MOCK_ACQ_LOG=str(log), DABB_MOCK_IQ=iq)
    for k, n in enumerate(contexts):
        env[f"DABB_MOCK_IQ_{k}"] = ":".join([iq] * n)
    r = subprocess.run([EXE] + args + ["--out", str(out), iq], capture_output=True, text=True, timeout=900, env=env)
    assert r.returncode == 0, r.stderr
    lines = [l.split() for l in log.read_text().splitlines()] if log.exists() else []
    return out, lines, r.stdout


def contexts_with(lines):
    opts, done = {}, []
    for l in lines:
        if l[0] == "options":
            opts.setdefault(l[1], []).append(tuple(int(v) for v in l[2:]))
        else:
            done.append(opts.pop(l[1], []))
    return done


MODES = {"plain": ([], [1]), "wide": (["--rate", "2048000", "--offset", "0"], [1]), "scan": (["--rate", "2048000", "--scan"], [1, 1, 3]),
         "auto": (["--rate", "2048000", "--offset", "auto"], [1, 1, 3, 1])}


@pytest.mark.parametrize("mode", list(MODES))
def test_acq_reaches_every_context(setup, mode):
    tmp, iq = setup
    args, ctxs = MODES[mode]
    out_r, lr, so_r = run(tmp, f"{mode}_r", args + ["--acq", "robust"], iq, ctxs)
    out_d, ld, so_d = run(tmp, f"{mode}_d", args + ["--acq", "reference"], iq, ctxs)
    done = contexts_with(lr)
    assert len(done) == len(ctxs), lr
    for opts in done:
        assert len(opts) == 1 and opts[0][0] == 1, done
    if mode in ("scan", "auto"):
        assert [o[0][1:] for o in done[1:3]] == [(0, 1), (1, 0)], done
    assert not [l for l in ld if l[0] == "options"], ld
    assert so_r == so_d
    files_d, files_r = sorted(os.listdir(out_d)), sorted(os.listdir(out_r))
    assert not [f for f in files_d if f.endswith(".acq")]
    assert [f for f in files_r if not f.endswith(".acq")] == files_d
    for f in files_d:
        assert (out_r / f).read_bytes() == (out_d / f).read_bytes(), f
    acq = [f for f in files_r if f.endswith(".acq")]
    if mode == "scan":
        assert not acq
        return
    assert acq == [f[:-4] + ".acq" for f in files_d if f.endswith(".fic")]
    for f in acq:
        lines = (out_r / f).read_text().splitlines()
        assert lines and all(l == "774 2.500 1" for l in lines)


def test_acq_arguments(setup):
    tmp, iq = setup
    for args in (["--acq"], ["--acq", "fast", "--out", str(tmp), iq]):
        r = subprocess.run([EXE] + args, capture_output=True, text=True, timeout=60)
        assert r.returncode == 2, args
