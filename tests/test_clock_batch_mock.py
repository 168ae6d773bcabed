"""batch_decode --clock on the test double of the ABI that records dabb_options.sample_clock (tests/mock_backend/mock_dab_b200_clock.cpp):
--clock sets DABB_CLOCK_TRACK on every context the driver creates - the plain decode, the wideband decode, and the survey, locate and
confirmation contexts of --scan / --offset auto, each with the disable_coarse and freqsync_method it was created with - and writes one
.clk line per decoded frame from tap 11; without it nothing is set and no .clk file appears.  The .fic, .msc and .rs outputs do not
change: the double's frame records come from the oracle."""
import os
import subprocess

import pytest

import dabtx
from conftest import ROOT

EXE = os.path.join(ROOT, "welle.io_b200", "batch_decode")


@pytest.fixture(scope="module")
def setup(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("clock_mock")
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "welle.io_b200", "host")])
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", str(tmp / "libdab_b200.so"),
                           os.path.join(ROOT, "tests", "mock_backend", "mock_dab_b200_clock.cpp"),
                           "-L" + os.path.join(ROOT, "oracle"), "-loracle", "-Wl,-rpath," + os.path.join(ROOT, "oracle")])
    iq = tmp / "ens.iq"
    dabtx.DabTx(seed=0xC10C).frames(10).tofile(iq)
    return tmp, str(iq)


def run(tmp, name, args, iq, contexts):
    out = tmp / name
    out.mkdir()
    log = tmp / f"{name}.log"
    env = dict(os.environ, LD_LIBRARY_PATH=str(tmp), DABB_MOCK_CLOCK_LOG=str(log), DABB_MOCK_IQ=iq)
    for k, n in enumerate(contexts):
        env[f"DABB_MOCK_IQ_{k}"] = ":".join([iq] * n)
    r = subprocess.run([EXE] + args + ["--out", str(out), iq], capture_output=True, text=True, timeout=900, env=env)
    assert r.returncode == 0, r.stderr
    lines = [l.split() for l in log.read_text().splitlines()] if log.exists() else []
    return out, lines, r.stdout


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
def test_clock_reaches_every_context(setup, mode):
    tmp, iq = setup
    args, ctxs = MODES[mode]
    out_c, lc, so_c = run(tmp, f"{mode}_c", args + ["--clock"], iq, ctxs)
    out_d, ld, so_d = run(tmp, f"{mode}_d", args, iq, ctxs)
    done = contexts_with(lc)
    assert len(done) == len(ctxs), lc
    for opts in done:
        assert len(opts) == 1 and opts[0][0] == 1, done
    if mode in ("scan", "auto"):
        # locate: coarse corrector on with GetMiddle; confirm: off
        assert [o[0][1:] for o in done[1:3]] == [(0, 1), (1, 0)], done
    assert not [l for l in ld if l[0] == "options"], ld
    assert so_c == so_d
    files_d, files_c = sorted(os.listdir(out_d)), sorted(os.listdir(out_c))
    assert not [f for f in files_d if f.endswith(".clk")]
    assert [f for f in files_c if not f.endswith(".clk")] == files_d
    for f in files_d:
        assert (out_c / f).read_bytes() == (out_d / f).read_bytes(), f
    clk = [f for f in files_c if f.endswith(".clk")]
    if mode == "scan":
        assert not clk                  # --scan writes no decode outputs
        return
    assert clk == [f[:-4] + ".clk" for f in files_d if f.endswith(".fic")]
    for f in clk:
        lines = (out_c / f).read_text().splitlines()
        frames = os.path.getsize(out_c / (f[:-4] + ".fic")) // (12 * 33)
        assert len(lines) == frames > 0
        assert all(l == "1.2500 0.5000 9" for l in lines)


def test_clock_arguments(setup):
    tmp, iq = setup
    for args in (["--clock"], ["--clock", "--scan", "--out", str(tmp), iq], ["--clock", "--rate", "2048000", "--out", str(tmp), iq]):
        r = subprocess.run([EXE] + args, capture_output=True, text=True, timeout=60)
        assert r.returncode == 2, args
