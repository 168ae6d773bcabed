"""Robust acquisition (dabb_options.acquisition): acquisition and FIB CRC passes against SNR and tone level in both methods, false
acquisitions on noise only, and the cost of a step in which 4096 streams acquire and of a steady step with the option on.

    python scripts/acq_measure.py [--streams 8] [--steps 8] [--out FILE.json]

Every recording starts at a random position inside a frame; a stream counts as acquired when it decodes a frame within the steps, and
"steps to first frame" is the first step that decodes one.  Each step's buffer is the least a step needs plus a frame, from the
stream's next_pos.  Prints one JSON document with the card's name and power limit, and writes it to FILE.json with --out."""
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
import acqref  # noqa: E402
import dabtx  # noqa: E402
import ofdmref  # noqa: E402
from conftest import load_pkg  # noqa: E402

TF = 196608
NEED = 198151


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        return "unknown"


def recordings(n, frames, snr, chan=None, tone=None, seed=0):
    rng = np.random.default_rng(seed)
    out, starts = [], []
    for i in range(n):
        clean = dabtx.DabTx(seed=0xB000 + seed * 100 + i).frames(frames, noise_floor=0)
        p = float(np.mean(np.abs(clean) ** 2))
        x = ofdmref.multipath(clean, chan) if chan else clean
        if snr is not None:
            x = dabtx.add_awgn(x, snr, seed=seed * 1000 + i, signal_power=p)
        else:
            x = dabtx.add_awgn(np.zeros_like(clean), 0.0, seed=seed * 1000 + i, signal_power=p)
        if tone is not None:
            x = acqref.tone(x, *tone)
        out.append(np.asarray(x, np.complex64))
        starts.append(int(rng.integers(0, TF)))
    return np.stack(out), np.array(starts, np.int64)


def run(pkg, rec, starts, steps, acq):
    S, N = rec.shape
    L = NEED + TF
    ctx = pkg.Context(n_streams=S)
    ctx.set_options(acquisition=acq)
    for s in range(S):
        ctx.reset(s, 1, int(starts[s]))
    pos = starts.copy()
    first = [None] * S
    crc = 0
    false_acq = 0
    for k in range(steps):
        win = np.zeros((S, L), np.complex64)
        for s in range(S):
            a = rec[s, pos[s]:pos[s] + L]
            win[s, :len(a)] = a
        out = ctx.process(win, L, pos, L, iq_is_host=True)
        r = out["results"]
        for s in range(S):
            if r["status"][s] == 0:
                crc += bin(int(r["fib_crc_mask"][s])).count("1")
                if first[s] is None:
                    first[s] = k
            if r["status"][s] == 2:
                false_acq += 1
        pos = r["next_pos"].copy()
    ctx.close()
    got = [f for f in first if f is not None]
    return {"acquired": len(got), "of": S, "mean_steps_to_first_frame": float(np.mean(got)) + 1 if got else None,
            "fib_crc_pass": crc, "no_sync_steps": false_acq}


def timing(pkg, S, acq, steady):
    """ms of the first step of S acquiring streams (steady: the mean of steps 2 .. 7, every stream tracking), host clock around a
    synchronised step"""
    x = dabtx.add_awgn(dabtx.DabTx(seed=0xB900).frames(12, noise_floor=0), 10.0, seed=1)
    ctx = pkg.Context(n_streams=S)
    ctx.set_options(acquisition=acq)
    d = ctx.dev(x)
    ts = []
    for k in range(8 if steady else 1):
        ctx.sync()
        t0 = time.perf_counter()
        ctx.process(d, 0, np.zeros(S, np.int64), len(x))
        ctx.sync()
        ts.append((time.perf_counter() - t0) * 1e3)
    d.free()
    ctx.close()
    return float(np.mean(ts[2:])) if steady else ts[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=8)
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--out", help="also write the JSON document to this file")
    a = ap.parse_args()
    pkg = load_pkg()
    res = {"card": card(), "streams": a.streams, "steps": a.steps, "snr": {}, "tone": {}, "noise_only": {}, "timing_ms": {}}
    modes = {"reference": pkg.ACQ_REFERENCE, "robust": pkg.ACQ_ROBUST}
    for chan_name, chan in (("awgn", None), ("multipath", [(0, 1.0), (37, 0.7 - 0.3j), (211, 0.5j)])):
        for snr in (-4, -2, 0, 2, 4, 6):
            rec, st = recordings(a.streams, a.steps + 2, snr, chan, seed=snr + 10)
            res["snr"]["%s %+d dB" % (chan_name, snr)] = {m: run(pkg, rec, st, a.steps, v) for m, v in modes.items()}
            print(chan_name, snr, res["snr"]["%s %+d dB" % (chan_name, snr)], flush=True)
    for db in (10, 20, 30, 40):
        for hz in (301000.0, 301500.0):
            rec, st = recordings(a.streams, a.steps + 2, 10.0, tone=(hz, float(db)), seed=db + 50)
            key = "%d dB at %.1f kHz (SNR 10 dB)" % (db, hz / 1000)
            res["tone"][key] = {m: run(pkg, rec, st, a.steps, v) for m, v in modes.items()}
            print(key, res["tone"][key], flush=True)
    rec, st = recordings(a.streams * 4, a.steps + 2, None, seed=99)
    res["noise_only"] = {m: run(pkg, rec, st, a.steps, v) for m, v in modes.items()}
    print("noise only", res["noise_only"], flush=True)
    for m, v in modes.items():
        res["timing_ms"]["first step, 4096 acquiring, " + m] = timing(pkg, 4096, v, False)
        res["timing_ms"]["steady step, 4096 tracking, " + m] = timing(pkg, 4096, v, True)
    print(json.dumps(res["timing_ms"]), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
