"""Measures the wideband channelizer on the GPU (writes nothing into the tree unless --out is given).

1. chan_kernel alone, device-resident input: (10 Msps, 5 channels), (20 Msps, 11), (61.44 Msps, 32), each in cf32 and s16le.  Kernel
   time from the library's per-launch CUDA events (dabb_profile), per second of input; algorithmic FLOPs and bytes from T, L, M and
   the channel count; share of the H100 SXM data-sheet FP32 peak and HBM bandwidth, and an estimated share of the shared-memory / L1
   bandwidth from the inner loop's loads (samples and tap groups); which of the three is largest; real-time factor.
2. End to end, device-resident input: a 61.44 Msps capture of 32 ensembles (one DabTx ensemble at 32 offsets 1.712 MHz apart, each
   with its own delay) is channelized and decoded by one context; frames/s and the split between channelizer and decode.

usage: python scripts/chan_measure.py [--seconds 0.25] [--repeat 8] [--frames 8] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

FP32_PEAK = 67e12          # H100 SXM data sheet, dense FP32, at up to 700 W
HBM_PEAK = 3.35e12         # H100 SXM data sheet, HBM3
# shared memory / L1: 128 B per clock and SM (the Hopper tuning guide), 132 SMs at the 1980 MHz maximum SM clock
L1_PEAK = 128 * 132 * 1.98e9
CONFIGS = [(10000000, 5), (20000000, 11), (61440000, 32)]


def gpu_name():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], text=True).strip()
    except Exception as e:      # the measurement itself needs the device; this is only the label
        return f"unknown ({e})"


def band_offsets(R, n):
    """n offsets 1.712 MHz apart, centred on 0, inside the accepted band"""
    offs = [int(round((k - (n - 1) / 2) * 1712000)) for k in range(n)]
    edge = R // 2 - 768000
    assert all(abs(o) <= edge for o in offs), (R, n)
    return offs


def kernel_only(pkg, chanref, R, n_ch, fmt, seconds, repeat):
    L, M, T = chanref.geometry(R)
    c = pkg.Context(n_streams=1)
    try:
        ch = pkg.Channelizer(c, R, band_offsets(R, n_ch), iq_format=fmt)
        out_len = int(seconds * 2048000)
        first, end = ch.input_range(0, out_len)
        n_in = end - first
        bps = chanref.BYTES[fmt]
        rng = np.random.default_rng(1)
        x = rng.integers(0, 256, n_in * bps, dtype=np.uint8) if fmt else (rng.standard_normal(n_in) + 1j * rng.standard_normal(n_in)).astype(np.complex64)
        if fmt == 0:
            x = x * 0.1
        d_in = c.dev(x.astype(np.complex64) if fmt == 0 else x)
        d_out = c.dev(n_ch * out_len * 8)
        for _ in range(2):                      # warm-up
            ch.run(d_in.ptr, [first], n_in, 0, out_len, in_stride=n_in, in_is_host=False, out=d_out)
        c.sync()
        c.profile(True)
        t0 = time.perf_counter()
        for _ in range(repeat):
            ch.run(d_in.ptr, [first], n_in, 0, out_len, in_stride=n_in, in_is_host=False, out=d_out)
        c.sync()
        wall = time.perf_counter() - t0
        prof = c.profile_read()["chan_kernel"]
        c.profile(False)
        ms = prof["ms"] / prof["n"]
        in_seconds = n_in / R
        TP = (T + 3) // 4 * 4
        flops = n_ch * out_len * 4 * T + n_ch * n_in * 6          # taps (2 FMA per tap and output) + the mixer's complex product
        nbytes = n_in * bps + n_ch * out_len * 8                  # input read once, outputs written once
        # the bytes the inner loop moves through the shared-memory / L1 datapath, an estimate from the algorithm's loads (not a profiler
        # count): per tap and output one 8-byte sample from shared memory, and per 4 taps one 16-byte tap group (a broadcast when L = 1)
        l1_bytes = n_ch * out_len * T * 8 + n_ch * out_len * (TP // 4) * (16 if L > 1 else 16 / 32)
        t = ms / 1e3
        f_share, b_share, l_share = flops / t / FP32_PEAK, nbytes / t / HBM_PEAK, l1_bytes / t / L1_PEAK
        d_in.free(); d_out.free(); ch.destroy()
        return {"rate": R, "channels": n_ch, "format": ["cf32", "u8", "s8", "s16le", "s16be"][fmt], "L": L, "M": M, "T": T,
                "input_seconds": in_seconds, "kernel_ms": ms, "kernel_ms_per_input_second": ms / in_seconds,
                "wall_ms_per_call": wall / repeat * 1e3, "tflop": flops / 1e12, "gbyte": nbytes / 1e9,
                "tflops_achieved": flops / t / 1e12, "fp32_peak_share": f_share, "hbm_peak_share": b_share,
                "l1_gbyte_estimate": l1_bytes / 1e9, "l1_peak_share_estimate": l_share,
                "bound": max((f_share, "FP32"), (b_share, "HBM"), (l_share, "shared memory / L1 (estimate)"))[1], "realtime_factor": in_seconds / t}
    finally:
        c.close()


def end_to_end(pkg, chanref, dabtx, frames):
    from scipy.signal import resample_poly
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
    c = pkg.Context(n_streams=S)
    try:
        ch = pkg.Channelizer(c, R, offs)
        out_len = (n - 1) * L // M + 1 - T
        first, end = ch.input_range(0, out_len)
        d_in = c.dev(np.concatenate([np.zeros(T, np.complex64), x]))
        d_out = c.dev(S * out_len * 8)
        ch.run(d_in.ptr, [-T], n + T, 0, out_len, in_stride=n + T, in_is_host=False, out=d_out)      # warm-up
        for s in range(S):
            c.select_subchannel(tx.start_cu, tx.size_cu, tx.bitrate, eep_profile_a=tx.profile_a, eep_level=tx.level, first=s, count=1)
        c.sync()
        t0 = time.perf_counter()
        ch.run(d_in.ptr, [-T], n + T, 0, out_len, in_stride=n + T, in_is_host=False, out=d_out)
        c.sync()
        t_chan = time.perf_counter() - t0
        decoded = 0
        t0 = time.perf_counter()
        for _ in range(frames + 2):
            out = c.process(d_out, out_len, np.zeros(S, np.int64), out_len, msc_stride=3 * tx.bitrate)
            decoded += int((out["results"]["status"] == pkg.FRAME_DECODED).sum())
        t_dec = time.perf_counter() - t0
        d_in.free(); d_out.free(); ch.destroy()
        return {"rate": R, "ensembles": S, "input_seconds": n / R, "channelize_s": t_chan, "decode_s": t_dec, "decoded_frames": decoded,
                "frames_per_s": decoded / (t_chan + t_dec), "channelizer_share": t_chan / (t_chan + t_dec)}
    finally:
        c.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=0.25)
    ap.add_argument("--repeat", type=int, default=8)
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import __graft_entry__ as ge
    import chanref
    import dabtx
    pkg = ge._pkg()
    res = {"gpu": gpu_name(), "fp32_peak": FP32_PEAK, "hbm_peak": HBM_PEAK, "kernel": [], "end_to_end": None}
    for R, n_ch in CONFIGS:
        for fmt in (0, 3):
            r = kernel_only(pkg, chanref, R, n_ch, fmt, a.seconds, a.repeat)
            print(json.dumps(r), flush=True)
            res["kernel"].append(r)
    res["end_to_end"] = end_to_end(pkg, chanref, dabtx, a.frames)
    print(json.dumps(res["end_to_end"]), flush=True)
    print("gpu:", res["gpu"])
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        json.dump(res, open(os.path.join(a.out, "chan_measure.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
