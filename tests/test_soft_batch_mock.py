"""batch_decode --soft on the test double of the ABI that records dabb_options.soft_demap (tests/mock_backend/mock_dab_b200_soft.cpp):
--soft weighted sets DABB_DEMAP_WEIGHTED on every context the driver creates - the plain decode, the wideband decode, and the survey
and confirmation contexts of --scan / --offset auto, each with the disable_coarse and freqsync_method it was created with - and the
default (or --soft reference) never sets it.  The outputs do not change: the double's frame records come from the oracle."""
import os
import subprocess

import pytest

import dabtx
from conftest import ROOT

EXE = os.path.join(ROOT, "welle.io_b200", "batch_decode")


@pytest.fixture(scope="module")
def setup(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("soft_mock")
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "welle.io_b200", "host")])
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", str(tmp / "libdab_b200.so"),
                           os.path.join(ROOT, "tests", "mock_backend", "mock_dab_b200_soft.cpp"),
                           "-L" + os.path.join(ROOT, "oracle"), "-loracle", "-Wl,-rpath," + os.path.join(ROOT, "oracle")])
    iq = tmp / "ens.iq"
    dabtx.DabTx(seed=0x50B0).frames(10).tofile(iq)
    return tmp, str(iq)


def run(tmp, name, args, iq, contexts):
    out = tmp / name
    out.mkdir()
    log = tmp / f"{name}.log"
    env = dict(os.environ, LD_LIBRARY_PATH=str(tmp), DABB_MOCK_SOFT_LOG=str(log), DABB_MOCK_IQ=iq)
    for k, n in enumerate(contexts):
        env[f"DABB_MOCK_IQ_{k}"] = ":".join([iq] * n)
    r = subprocess.run([EXE] + args + ["--out", str(out), iq], capture_output=True, text=True, timeout=900, env=env)
    assert r.returncode == 0, r.stderr
    lines = [l.split() for l in log.read_text().splitlines()] if log.exists() else []
    return out, lines


def contexts_with(lines):
    """[(options of the context before it was destroyed, ...)] per destroyed context, in order"""
    opts, done = {}, []
    for l in lines:
        if l[0] == "options":
            opts.setdefault(l[1], []).append(tuple(int(v) for v in l[2:]))
        else:
            done.append(opts.pop(l[1], []))
    return done


# (arguments, streams of each context the run creates: the plain and the wideband decode one; --scan the survey, locate and confirm
# contexts; --offset auto those and the decode)
MODES = {"plain": ([], [1]), "wide": (["--rate", "2048000", "--offset", "0"], [1]), "scan": (["--rate", "2048000", "--scan"], [1, 1, 3]),
         "auto": (["--rate", "2048000", "--offset", "auto"], [1, 1, 3, 1])}


@pytest.mark.parametrize("mode", list(MODES))
def test_soft_reaches_every_context(setup, mode):
    tmp, iq = setup
    args, ctxs = MODES[mode]
    out_w, lw = run(tmp, f"{mode}_w", args + ["--soft", "weighted"], iq, ctxs)
    out_d, ld = run(tmp, f"{mode}_d", args, iq, ctxs)
    out_r, lr = run(tmp, f"{mode}_r", args + ["--soft", "reference"], iq, ctxs)
    done = contexts_with(lw)
    assert len(done) == len(ctxs), lw
    for opts in done:
        assert len(opts) == 1 and opts[0][0] == 1, done
    if mode in ("scan", "auto"):
        # locate: coarse corrector on with GetMiddle; confirm: off
        assert [o[0][1:] for o in done[1:3]] == [(0, 1), (1, 0)], done
    for lines in (ld, lr):
        assert all(int(l[2]) == 0 for l in lines if l[0] == "options"), lines
        assert len(contexts_with(lines)) == len(ctxs)
    for f in sorted(os.listdir(out_d)):
        assert (out_w / f).read_bytes() == (out_d / f).read_bytes() == (out_r / f).read_bytes(), f


def test_soft_arguments(setup):
    tmp, iq = setup
    for args in (["--soft"], ["--soft", "median"]):
        r = subprocess.run([EXE] + args + ["--out", str(tmp), iq], capture_output=True, text=True, timeout=60)
        assert r.returncode == 2, args
