"""batch_decode --rate / --offset on the GPU against the Python path (Channelizer + Context) on the same wideband recording: two DabTx
ensembles in a 4.096 Msps cf32 file (the recordings of tests/test_gpu_chan.py's closed loop).  The driver channelizes each stream's
[pos, pos + need) every step; the Python path channelizes the whole recording once.  The channelizer is stateless, so both decode the
same samples: the .fic records of every frame once both are tracking, the logical frames once the time de-interleaver has settled, and
the Reed-Solomon records of those frames must be equal."""
import os
import subprocess

import numpy as np
import pytest

import chanref
import test_gpu_chan as tg
from conftest import ROOT, load_pkg

pytestmark = pytest.mark.gpu
R = 4096000
OFFSETS = [-856000, 856000]


def python_path(pkg, xb, T, n_in, out_len, txs):
    """per stream: [(33-byte FIB records of a frame, CRC mask)], [(frame, logical frame)], [(frame, 'uncorr corr')]"""
    S = len(OFFSETS)
    c = pkg.Context(n_streams=S)
    try:
        ch = pkg.Channelizer(c, R, OFFSETS)
        d = ch.run(xb, [-T], n_in + T, 0, out_len)
        for s, tx in enumerate(txs):
            c.select_subchannel(tx.start_cu, tx.size_cu, tx.bitrate, eep_profile_a=tx.profile_a, eep_level=tx.level, dabplus=tx.dabplus, first=s, count=1)
        fic, msc, rs = [[] for _ in range(S)], [[] for _ in range(S)], [[] for _ in range(S)]
        for _ in range(tg.FRAMES + 3):
            out = c.process(d, out_len, np.zeros(S, np.int64), out_len, msc_stride=1152)
            r = out["results"]
            for s in range(S):
                if r["status"][s] != pkg.FRAME_DECODED or r["next_pos"][s] > out_len:
                    continue
                mask = int(r["fib_crc_mask"][s])
                rec = b"".join(bytes([(mask >> f) & 1]) + out["fibs"][s, f].tobytes() for f in range(12))
                fic[s].append((rec, mask))
                k = len(fic[s]) - 1
                for j in range(4 - int(r["n_logical"][s][0]), 4):
                    msc[s].append((k, out["msc"][s, 0, j, :3 * txs[s].bitrate].tobytes()))
                for e in range(int(r["n_rs_events"][s][0])):
                    rs[s].append((k, f"{(int(r['rs_uncorr_mask'][s][0]) >> e) & 1} {int(r['rs_corr'][s][0][e])}"))
        ch.destroy()
        d.free()
        return fic, msc, rs
    finally:
        c.close()


def test_batch_decode_wideband_equals_python_path(tmp_path):
    pkg = load_pkg()
    exe = os.path.join(ROOT, "welle.io_b200", "batch_decode")
    assert os.path.exists(exe), "build() makes welle.io_b200/batch_decode"
    sigs = tg.ensembles(3, seed=0x4096)[0::2]          # two DAB+ ensembles (96 and 128 kbit/s): DabTx signals every service as DAB+
    txs = [tx for tx, _ in sigs]
    x = tg.quantize(tg.wideband(sigs, R, OFFSETS, [0.0, 0.0], snr_db=24.0, seed=7), 0)
    L, M, T = chanref.geometry(R)
    n_in = x.shape[1]
    f = tmp_path / "wide.iq"
    x.tofile(f)
    outdir = tmp_path / "out"; outdir.mkdir()
    run = subprocess.run([exe, "--rate", str(R), "--offset", ",".join(map(str, OFFSETS)), "--out", str(outdir), str(f)],
                         capture_output=True, text=True, timeout=900)
    assert run.returncode == 0, run.stderr
    print(run.stdout)
    xb = np.concatenate([np.zeros((1, T), np.complex64), x], axis=1)
    out_len = (n_in - 1) * L // M + 1
    fic, msc, rs = python_path(pkg, xb, T, n_in, out_len, txs)
    for s, off in enumerate(OFFSETS):
        name = f"wide.iq@{off}"
        recs = np.fromfile(outdir / f"{name}.fic", np.uint8).reshape(-1, 12 * 33)
        d_fic = [(r.tobytes(), sum(int(r[33 * k]) << k for k in range(12))) for r in recs]
        # frame for frame once both are tracking: the driver's frames are the Python path's, shifted by the frames it decoded before
        a, b = tg.tracking(d_fic), tg.tracking(fic[s])
        assert len(a) >= tg.FRAMES - 10 and all(m == 0xFFF for _, m in a), (s, [hex(m) for _, m in d_fic])
        shift = tg.aligned([r for r, _ in a], [r for r, _ in b], tg.FRAMES - 10)
        assert shift is not None, f"{name}: .fic differs from the Python path"
        flen = 3 * txs[s].bitrate
        raw = np.fromfile(outdir / f"{name}.msc", np.uint8)
        drv = [raw[i:i + flen].tobytes() for i in range(0, len(raw), flen)]
        settled = tg.settled_logical(fic[s], msc[s])
        # the driver tunes after its first decoded frame and decodes to the end of the file: the Python path's settled logical frames are
        # a contiguous run of the driver's
        assert len(settled) >= 16 and tg.aligned(settled, drv, len(settled)) is not None, f"{name}: .msc differs from the Python path"
        k0 = tg.first_tracking(fic[s]) + 6
        py_rs = [line for k, line in rs[s] if k >= k0]
        drv_rs = (outdir / f"{name}.rs").read_text().splitlines()
        assert len(py_rs) >= 2 and tg.aligned(py_rs, drv_rs, len(py_rs)) is not None, f"{name}: .rs differs from the Python path"
