"""batch_decode --rate / --offset on the test double of the ABI with the channelizer (tests/mock_backend/mock_dab_b200_chan.cpp): two
wideband recordings at 4.096 Msps with two ensembles each become four streams.  The double decodes each stream from the ensemble's own
2.048 Msps signal ($DABB_MOCK_IQ, through the oracle) and runs the channelizer calls for real on the host build of chan_core.cuh, logging
them.  Checked: the output files DIR/<name>@<offset>.{fic,msc,rs} and their record formats, every FIB dump against the oracle's decode of
the ensemble, and that every step channelizes exactly each stream's [pos, pos + need) out of a host buffer that holds only the span the
streams of the file still need."""
import os
import subprocess

import numpy as np

import chanref
import dabtx
from conftest import ROOT

R = 4096000
OFFSETS = [-856000, 856000]
TF = 196608


def test_batch_decode_wideband_on_mock_backend(oracle, tmp_path):
    from scipy.signal import resample_poly
    exe = os.path.join(ROOT, "welle.io_b200", "batch_decode")
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "welle.io_b200", "host")])
    mock = tmp_path / "libdab_b200.so"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", str(mock),
                           os.path.join(ROOT, "tests", "mock_backend", "mock_dab_b200_chan.cpp"),
                           "-L" + os.path.join(ROOT, "oracle"), "-loracle", "-Wl,-rpath," + os.path.join(ROOT, "oracle")])
    files, own_files, owns = [], [], []
    for k in range(2):
        x = None
        for j, f in enumerate(OFFSETS):
            s = np.concatenate([np.zeros(311 * (2 * k + j), np.complex64), dabtx.DabTx(seed=0x5A0 + 2 * k + j).frames(12)])
            of = tmp_path / f"own{k}{j}.iq"
            s.tofile(of); own_files.append(str(of)); owns.append(s)
            y = resample_poly(s.astype(np.complex128), 2, 1)
            y = y * np.exp(2j * np.pi * (((f % R) * np.arange(len(y), dtype=np.int64)) % R) / R)
            x = y if x is None else x[:min(len(x), len(y))] + y[:min(len(x), len(y))]
        fw = tmp_path / f"wide{k}.iq"
        x.astype(np.complex64).tofile(fw); files.append(str(fw))
    outdir = tmp_path / "out"; outdir.mkdir()
    log = tmp_path / "chan.log"
    env = dict(os.environ, LD_LIBRARY_PATH=str(tmp_path), DABB_MOCK_IQ=":".join(own_files), DABB_MOCK_CHAN_LOG=str(log))
    run = subprocess.run([exe, "--rate", str(R), "--offset", ",".join(map(str, OFFSETS)), "--out", str(outdir)] + files,
                         capture_output=True, text=True, timeout=900, env=env)
    assert run.returncode == 0, run.stderr
    lines = run.stdout.strip().splitlines()
    names = [f"wide{k}.iq@{f}" for k in range(2) for f in OFFSETS]
    assert [ln.split()[0] for ln in lines] == names
    for s, name in enumerate(names):
        fibs = np.fromfile(outdir / f"{name}.fic", np.uint8).reshape(-1, 33)
        o = oracle.rx_run(owns[s], disable_coarse=True)
        n = min(len(fibs), len(o["fibs"]))
        assert n >= 12 * 8 and np.array_equal(fibs[:n], o["fibs"][:n]), name
        msc = np.fromfile(outdir / f"{name}.msc", np.uint8)
        assert len(msc) > 0 and len(msc) % 288 == 0
        o = oracle.rx_run(owns[s], prot=oracle.prot_eep(96, 1, 3), start_cu=0, len_cu=dabtx.eep_cu(96, True, 3), select_after_frames=1, disable_coarse=True)
        m = min(len(msc), len(o["msc"]))
        assert m >= 288 * 16 and np.array_equal(msc[:m], o["msc"][:m]), name
        for ln in (outdir / f"{name}.rs").read_text().splitlines():
            a, b = ln.split()
            assert a in ("0", "1") and int(b) >= 0
        assert f"frames={len(fibs) // 12}" in lines[s]
    # the channelizer calls: one per recording and step, each channel's window [pos, pos + out_len), the input buffer exactly the span
    # its channels read
    calls = [list(map(int, ln.split())) for ln in log.read_text().splitlines()]
    assert len(calls) >= 2 * 10
    need_track = 2048 + 2047 + 75 * 2552 + 2656
    for c in calls:
        starts, out_len, in_start, in_len = c[:2], c[2], c[3], c[4]
        assert need_track <= out_len <= 5 * TF
        spans = [chanref.input_range(R, p, out_len) for p in starts]
        assert in_start == min(a for a, _ in spans) and in_start + in_len == max(b for _, b in spans)
    assert calls[0][:2] == [0, 0] and calls[1][:2] == [0, 0]
