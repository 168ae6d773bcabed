"""batch_decode --mer on the test double of the ABI with tap 14 (tests/mock_backend/mock_dab_b200_mer.cpp): dabb_set_mer is called once,
on the decode context; every decoded frame adds one .mer line "points mer_db sig err" equal to the double's record of that frame, and
the .merprof holds the int64 sums of the records' groups with their MER.  Without --mer no .mer or .merprof file exists and every other
output, stdout included, is byte-identical.  The double's frame records come from the oracle."""
import math
import os
import subprocess

import numpy as np
import pytest

import dabtx
from conftest import ROOT

EXE = os.path.join(ROOT, "welle.io_b200", "batch_decode")


def mock_record(s, n):
    """the double's record of stream s's n-th decoded frame (mock_dab_b200_mer.cpp::mock_record)"""
    gsig = [50000 + 1000 * s + 37 * g + n for g in range(64)]
    gerr = [0 if g % 7 == 3 else 100 + 3 * g + s + n for g in range(64)]
    sig, err = sum(gsig), sum(gerr)
    return dict(points=4608 - s - n, sig=sig, err=err, mer_db=float(np.float32(10 * math.log10(sig / err))), gsig=gsig, gerr=gerr)


@pytest.fixture(scope="module")
def setup(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("mer_mock")
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "welle.io_b200", "host")])
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-o", str(tmp / "libdab_b200.so"),
                           os.path.join(ROOT, "tests", "mock_backend", "mock_dab_b200_mer.cpp"),
                           "-L" + os.path.join(ROOT, "oracle"), "-loracle", "-Wl,-rpath," + os.path.join(ROOT, "oracle")])
    files = []
    for k in range(2):
        f = tmp / f"rec{k}.iq"
        np.concatenate([np.zeros(211 * k, np.complex64), dabtx.DabTx(seed=0x3E5 + k).frames(9)]).tofile(f)
        files.append(str(f))
    return tmp, files


def run(tmp, name, args, files):
    out = tmp / name
    out.mkdir()
    log = tmp / f"{name}.log"
    env = dict(os.environ, LD_LIBRARY_PATH=str(tmp), DABB_MOCK_MER_LOG=str(log), DABB_MOCK_IQ=":".join(files))
    r = subprocess.run([EXE] + args + ["--out", str(out)] + files, capture_output=True, text=True, timeout=900, env=env)
    assert r.returncode == 0, r.stderr
    return out, (log.read_text().split("\n")[:-1] if log.exists() else []), r.stdout


def test_mer_files(setup):
    tmp, files = setup
    out_m, log_m, so_m = run(tmp, "mer", ["--mer"], files)
    out_d, log_d, so_d = run(tmp, "plain", [], files)
    assert len(log_m) == 1 and log_m[0].split()[2] == "1", log_m
    assert not log_d
    assert so_m == so_d
    names_d, names_m = sorted(os.listdir(out_d)), sorted(os.listdir(out_m))
    assert not [f for f in names_d if f.endswith((".mer", ".merprof"))]
    assert [f for f in names_m if not f.endswith((".mer", ".merprof"))] == names_d
    for f in names_d:
        assert (out_m / f).read_bytes() == (out_d / f).read_bytes(), f
    for s, line in enumerate(so_m.splitlines()):
        name = os.path.basename(files[s])
        frames = int(line.split("frames=")[1].split()[0])
        lines = (out_m / f"{name}.mer").read_text().splitlines()
        assert len(lines) == frames >= 7
        recs = [mock_record(s, n) for n in range(frames)]
        assert lines == [f"{r['points']} {r['mer_db']:.3f} {r['sig']} {r['err']}" for r in recs]
        prof = (out_m / f"{name}.merprof").read_text().splitlines()
        assert len(prof) == 64
        for g, pl in enumerate(prof):
            first = 24 * g - 768 + (g >= 32)
            sig, err = sum(r["gsig"][g] for r in recs), sum(r["gerr"][g] for r in recs)
            db = math.inf if err == 0 else 10 * math.log10(sig / err)
            assert pl == f"{first} {first + 23} {sig} {err} {db:.3f}", (g, pl)
