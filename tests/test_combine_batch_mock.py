"""batch_decode --diversity on the test double of the ABI with diversity combining (tests/mock_backend/mock_dab_b200_combine.cpp):
consecutive runs of N files are grouped with the first of each run as leader (one dabb_set_combining call), every file keeps the
outputs it has without the option, and each leader gets DIR/<name>.div with one "members mask noise" line per decoded frame (tap 12,
computed by the double with the library's contributor rule on the oracle's frame records and the files' null symbols): a capture whose
second antenna holds the same ensemble combines two members, one whose second antenna holds only noise keeps its leader alone.
--diversity with --rate, with a file count that is not a multiple of N, or with N outside 1 .. 8 is refused."""
import os
import subprocess

import numpy as np
import pytest

import dabtx
from conftest import ROOT

EXE = os.path.join(ROOT, "welle.io_b200", "batch_decode")


@pytest.fixture(scope="module")
def setup(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("combine_mock")
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "welle.io_b200", "host")])
    obj = str(tmp / "mock_combine.o")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-fno-inline", "-c", "-o", obj,
                           os.path.join(ROOT, "tests", "mock_backend", "mock_dab_b200_combine.cpp")])
    swap = []
    for f in ("process", "read_tap", "destroy"):          # the wrappers take the entry points' names (see the double's header)
        swap += ["--redefine-sym", f"dabb_{f}=mock_combine_base_{f}", "--redefine-sym", f"combine_wrap_{f}=dabb_{f}"]
    subprocess.check_call(["objcopy"] + swap + [obj])
    subprocess.check_call(["g++", "-shared", "-o", str(tmp / "libdab_b200.so"), obj,
                           "-L" + os.path.join(ROOT, "oracle"), "-loracle", "-Wl,-rpath," + os.path.join(ROOT, "oracle")])
    x = dabtx.DabTx(seed=0xC0D1).frames(8)
    p = float(np.mean(np.abs(x) ** 2))
    files = {"a0.iq": x, "a1.iq": dabtx.add_awgn(x, 20.0, seed=1, signal_power=p),
             "b0.iq": dabtx.DabTx(seed=0xC0D2).frames(8), "b1.iq": dabtx.add_awgn(np.zeros_like(x), 0.0, seed=2, signal_power=p)}
    for name, sig in files.items():
        np.asarray(sig, np.complex64).tofile(tmp / name)
    return tmp, [str(tmp / n) for n in files]


def run(tmp, name, args, files):
    out = tmp / name
    out.mkdir()
    log = tmp / f"{name}.log"
    env = dict(os.environ, LD_LIBRARY_PATH=str(tmp), DABB_MOCK_COMBINE_LOG=str(log), DABB_MOCK_IQ=":".join(files), DABB_MOCK_IQ_0=":".join(files))
    r = subprocess.run([EXE] + args + ["--out", str(out)] + files, capture_output=True, text=True, timeout=900, env=env)
    assert r.returncode == 0, r.stderr
    return out, (log.read_text().splitlines() if log.exists() else []), r.stdout


def test_diversity_layout(setup):
    tmp, files = setup
    out_d, log_d, so_d = run(tmp, "div", ["--diversity", "2"], files)
    out_p, log_p, so_p = run(tmp, "plain", [], files)
    assert len(log_d) == 1 and log_d[0].split()[2:] == ["0", "0", "2", "2"], log_d
    assert not log_p
    assert so_d == so_p
    plain, div = sorted(os.listdir(out_p)), sorted(os.listdir(out_d))
    assert [f for f in div if not f.endswith(".div")] == plain
    for f in plain:
        assert (out_d / f).read_bytes() == (out_p / f).read_bytes(), f
    assert [f for f in div if f.endswith(".div")] == ["a0.iq.div", "b0.iq.div"]
    for name, members, mask in (("a0.iq", 2, 3), ("b0.iq", 1, 1)):
        lines = [l.split() for l in (out_d / f"{name}.div").read_text().splitlines()]
        frames = os.path.getsize(out_d / f"{name}.fic") // (12 * 33)
        assert len(lines) == frames > 0
        assert all(len(l) == 3 and int(l[0]) == members and int(l[1]) == mask and float(l[2]) > 0 for l in lines), lines


def test_diversity_arguments(setup):
    tmp, files = setup
    for args in (["--diversity", "2", "--rate", "2048000", "--offset", "0"] + files[:2], ["--diversity", "3"] + files[:2],
                 ["--diversity", "9"] + files[:2], ["--diversity", "0"] + files[:2]):
        r = subprocess.run([EXE] + args + ["--out", str(tmp)], capture_output=True, text=True, timeout=60)
        assert r.returncode == 2, args
