"""welle.io_b200/batch_decode with more distinct protection profiles than the library has sub-channel slots: six recordings, each with
its own EEP-A / EEP-B profile, all decoded in slot 0.  Runs on the CPU against the test double of the C ABI
(tests/mock_backend/mock_dab_b200.c, which decodes every stream on its own); every .msc dump must equal the oracle's for its recording."""
import os
import subprocess

import numpy as np

import dabtx
from conftest import ROOT

SPECS = [dict(seed=0x41, bitrate=96, profile_a=True, level=3), dict(seed=0x42, bitrate=64, profile_a=True, level=2),
         dict(seed=0x43, bitrate=48, profile_a=True, level=1), dict(seed=0x44, bitrate=32, profile_a=True, level=4),
         dict(seed=0x45, bitrate=64, profile_a=False, level=2), dict(seed=0x46, bitrate=96, profile_a=False, level=4)]


def test_batch_decode_six_profiles_with_mock_backend(oracle, tmp_path):
    exe = os.path.join(ROOT, "welle.io_b200", "batch_decode")
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "welle.io_b200", "host")])
    mock = tmp_path / "libdab_b200.so"
    subprocess.check_call(["gcc", "-O1", "-shared", "-fPIC", "-o", str(mock), os.path.join(ROOT, "tests", "mock_backend", "mock_dab_b200.c"),
                           "-L" + os.path.join(ROOT, "oracle"), "-loracle", "-Wl,-rpath," + os.path.join(ROOT, "oracle")])
    files, sigs = [], []
    for k, sp in enumerate(SPECS):
        tx = dabtx.DabTx(**sp)
        iq = np.concatenate([np.zeros(311 * k, np.complex64), tx.frames(10)])
        f = tmp_path / f"rec{k}.iq"
        iq.tofile(f); files.append(str(f)); sigs.append(iq)
    outdir = tmp_path / "out"; outdir.mkdir()
    env = dict(os.environ, LD_LIBRARY_PATH=str(tmp_path), DABB_MOCK_IQ=":".join(files))
    run = subprocess.run([exe, "--out", str(outdir)] + files, capture_output=True, text=True, timeout=600, env=env)
    assert run.returncode == 0, run.stderr
    assert "protection profiles" not in run.stderr, run.stderr
    lines = run.stdout.strip().splitlines()
    assert len(lines) == len(SPECS)
    for k, sp in enumerate(SPECS):
        br, pa, lv = sp["bitrate"], sp["profile_a"], sp["level"]
        msc = np.fromfile(outdir / f"rec{k}.iq.msc", np.uint8)
        o = oracle.rx_run(sigs[k], prot=oracle.prot_eep(br, int(pa), lv), start_cu=0, len_cu=dabtx.eep_cu(br, pa, lv), select_after_frames=1,
                          disable_coarse=True)
        m = min(len(msc), len(o["msc"]))
        assert m >= 3 * br * 8 and np.array_equal(msc[:m], o["msc"][:m]), k
        assert f"bitrate={br}" in lines[k] and f"logical_frames={len(msc) // (3 * br)}" in lines[k]
