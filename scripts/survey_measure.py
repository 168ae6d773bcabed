"""Measures the spectrum survey on the GPU (writes nothing into the tree unless --out is given).

1. survey_kernel + survey_sum_kernel alone, device-resident input of 0.25 s: 10, 20 and 61.44 Msps, each in cf32 and s16le, with
   batch_decode's nfft (1024 / 4096 / 8192 / 16384: the smallest power of two >= 1024 with R / nfft <= 4000 Hz).  Kernel time from the
   library's per-launch CUDA events (dabb_profile), per second of input; against the HBM bound (the input bytes read once at the data
   sheet's 3.35 TB/s) and the FP32 bound (5 nfft log2 nfft flops per segment at 67 TFLOP/s).
2. batch_decode --scan on the 61.44 Msps capture of 32 ensembles that scripts/chan_measure.py synthesises (one DabTx ensemble at 32
   offsets 1.712 MHz apart, each with its own delay): wall time, split into survey and confirmation as the driver reports them.

usage: python scripts/survey_measure.py [--repeat 8] [--frames 8] [--out DIR]
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))

FP32_PEAK = 67e12          # H100 SXM data sheet, dense FP32, at up to 700 W
HBM_PEAK = 3.35e12         # H100 SXM data sheet, HBM3


def kernel_only(pkg, surveyref, R, fmt, repeat):
    import ctypes as C
    nfft = surveyref.nfft_for_rate(R)
    n = R // 4
    bps = (8, 2, 2, 4, 4)[fmt]
    rng = np.random.default_rng(1)
    x = rng.integers(0, 256, n * bps, dtype=np.uint8) if fmt else ((rng.standard_normal(n) + 1j * rng.standard_normal(n)) * 0.1).astype(np.complex64)
    c = pkg.Context(n_streams=1)
    try:
        d = c.dev(x)
        psd = np.zeros(nfft, np.float32)
        io = pkg.dabb200.SurveyIO(d.ptr, 0, fmt, n, 1, nfft, n, psd.ctypes.data)
        c._ck(c.lib.dabb_survey(c.h, C.byref(io)))            # warm-up: tables, scratch, modules
        c.profile(True)
        t0 = time.perf_counter()
        for _ in range(repeat):
            c._ck(c.lib.dabb_survey(c.h, C.byref(io)))
        wall = (time.perf_counter() - t0) / repeat
        prof = c.profile_read()
        c.profile(False)
        d.free()
    finally:
        c.close()
    k = prof["survey_kernel"]["ms"] / repeat
    s = prof["survey_sum_kernel"]["ms"] / repeat
    S = (n - nfft) // (nfft // 2) + 1
    hbm = n * bps / HBM_PEAK * 1e3
    fp32 = S * 5 * nfft * np.log2(nfft) / FP32_PEAK * 1e3
    per_s = 4.0                                                 # calls of 0.25 s per second of input
    return {"rate": R, "format": ["cf32", "u8", "s8", "s16le", "s16be"][fmt], "nfft": nfft, "segments": S,
            "survey_kernel_ms_per_s": round(k * per_s, 4), "survey_sum_kernel_ms_per_s": round(s * per_s, 4),
            "call_wall_ms_per_s": round(wall * 1e3 * per_s, 3),
            "hbm_bound_ms_per_s": round(hbm * per_s, 4), "fp32_bound_ms_per_s": round(fp32 * per_s, 4),
            "share_of_hbm_bound": round(hbm / k, 3), "share_of_fp32_bound": round(fp32 / k, 3)}


def capture_61(dabtx, chanref, frames, path):
    """scripts/chan_measure.py's 61.44 Msps, 32-ensemble capture, written as cf32; returns its offsets"""
    from scipy.signal import resample_poly
    from chan_measure import band_offsets
    R, S = 61440000, 32
    L, M, T = chanref.geometry(R)
    tx = dabtx.DabTx(seed=0x6144)
    base = tx.frames(frames + 2)
    Sp = np.fft.fft(base)
    Sp[np.abs(np.fft.fftfreq(len(base), 1 / 2048000)) > 800000] = 0
    y = resample_poly(np.fft.ifft(Sp), M, L).astype(np.complex64)
    n = len(y)
    offs = band_offsets(R, S)
    rng = np.random.default_rng(2)
    x = np.zeros(n, np.complex64)
    idx = np.arange(n, dtype=np.int64)
    for f in offs:
        ph = (2 * np.pi * (((f % R) * idx) % R) / R).astype(np.float32)
        x += np.roll(y, int(rng.integers(0, 30 * 196608))) * np.exp(1j * ph).astype(np.complex64)
    x += ((rng.standard_normal(n) + 1j * rng.standard_normal(n)) * 0.002).astype(np.complex64)
    x.tofile(path)
    return offs, n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeat", type=int, default=8)
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import chanref
    import dabtx
    import surveyref
    from chan_measure import gpu_name
    from conftest import load_pkg
    pkg = load_pkg()
    res = {"gpu": gpu_name(), "kernel": []}
    print("gpu:", res["gpu"], flush=True)
    for R in (10000000, 20000000, 61440000):
        for fmt in (0, 3):
            r = kernel_only(pkg, surveyref, R, fmt, a.repeat)
            res["kernel"].append(r)
            print(json.dumps(r), flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        f = os.path.join(tmp, "band.iq")
        offs, n = capture_61(dabtx, chanref, a.frames, f)
        out = os.path.join(tmp, "out"); os.mkdir(out)
        t0 = time.perf_counter()
        r = subprocess.run([os.path.join(ROOT, "welle.io_b200", "batch_decode"), "--rate", "61440000", "--scan", "--out", out, f],
                           capture_output=True, text=True, timeout=1800)
        wall = time.perf_counter() - t0
        assert r.returncode == 0, r.stderr
        lines = open(os.path.join(out, "band.iq.scan")).read().splitlines()
        m = re.search(r"survey ([0-9.]+) ms.*confirmation of (\d+) candidate\(s\) at \d+ offsets ([0-9.]+) ms", r.stderr)
        found = [int(ln.split()[0]) for ln in lines]
        res["scan_61440000"] = {"seconds_of_input": n / 61440000, "wall_s": round(wall, 3), "survey_ms": float(m.group(1)),
                                "candidates": int(m.group(2)), "confirmation_ms": float(m.group(3)), "ensembles": len(lines),
                                "all_found_within_30_hz": len(found) == len(offs) and all(abs(a_ - b) <= 30 for a_, b in zip(found, offs)),
                                "largest_offset_error_hz": max((abs(a_ - b) for a_, b in zip(found, offs)), default=None) if len(found) == len(offs) else None}
        print(json.dumps(res["scan_61440000"]), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "survey_measure.json"), "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
