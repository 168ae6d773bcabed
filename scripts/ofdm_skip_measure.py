"""What the OFDM demodulator's symbol mask (welle.io_b200/csrc/ofdm_mask.cuh) saves.

  python scripts/ofdm_skip_measure.py [--batch 4096] [--steps 20] [--cases bench,fic_only,whole_msc,keep_taps] [--out FILE.json]

For four configurations of a --batch-stream context on the benchmark's input (periodic rings at 20 dB, keep_taps off unless named):
  bench      FIC + one 96 kbit/s EEP 3-A DAB+ sub-channel at CU 0..71 (the benchmark's configuration)
  fic_only   no sub-channel
  whole_msc  one 384 kbit/s EEP 3-A DAB sub-channel over CU 0..863: every symbol is transformed, so the mask skips nothing
  keep_taps  the bench configuration with keep_taps on: no mask at all
it prints ofdm_demod_kernel's device time per step (dabb_profile, serial per-kernel timing after --steps warm-up steps), the step time
without profiling, the bytes the kernel moves per frame under the mask (input samples staged, softbits written), and those bytes over the
kernel time as a share of the data-sheet 3.35 TB/s of H100 SXM HBM3, with the card's name and power limit.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "scripts")); sys.path.insert(0, os.path.join(ROOT, "tests"))

from ber_measure import BUF_LEN, RING_FRAMES, TF, card, fill, rings  # noqa: E402

TU, TS, TG, THREADS = 2048, 2552, 504, 128
HBM_BPS = 3.35e12
CASES = {
    "bench": dict(keep_taps=False, sub=(0, 72, 96, True)),
    "fic_only": dict(keep_taps=False, sub=None),
    "whole_msc": dict(keep_taps=False, sub=(0, 864, 384, False)),
    "keep_taps": dict(keep_taps=True, sub=(0, 72, 96, True)),
}


def frame_bytes(sub, masked):
    """bytes ofdm_demod_kernel reads and writes per frame (one CTA per frame): staged samples and softbits"""
    demap = np.zeros(77, bool)
    demap[1:4] = True
    if sub is not None:
        st, ln = sub[0], sub[1]
        a, b = 64 * st // 3072, (64 * (st + ln) - 1) // 3072
        for c in range(4):
            demap[4 + 18 * c + a: 4 + 18 * c + b + 1] = True
    if not masked:
        demap[1:76] = True
    fft = [l for l in range(1, 76) if demap[l] or demap[l + 1]]
    light = 75 - len(fft)
    samples = TU + len(fft) * TS + light * (TG + THREADS + TG)
    return {"transformed": 1 + len(fft), "demapped": int(demap[1:76].sum()), "light": light,
            "bytes": 8 * samples + 3072 * int(demap[1:76].sum())}


def run_case(pkg, buf, S, steps, keep_taps, sub):
    ctx = pkg.Context(n_streams=S, disable_coarse=True, keep_taps=keep_taps, n_subch_slots=1, max_subch_cu=864 if sub and sub[1] > 72 else 72)
    if sub is not None:
        st, ln, br, dabplus = sub
        ctx.select_subchannel(st, ln, br, eep_profile_a=True, eep_level=3, dabplus=dabplus)
    call = [0]

    def step():
        n = call[0] + 1
        bs = np.full(S, RING_FRAMES * TF * (n // RING_FRAMES), np.int64) if call[0] > 0 else np.zeros(S, np.int64)
        ctx.process_async(buf.data_ptr(), BUF_LEN, bs, BUF_LEN); call[0] += 1

    for _ in range(steps):
        step()
    ctx.sync()
    t0 = time.perf_counter()
    for _ in range(steps):
        step()
    ctx.sync()
    step_ms = (time.perf_counter() - t0) * 1e3 / steps
    ctx.profile(True)
    for _ in range(steps):
        step()
    ctx.sync()
    prof = ctx.profile_read()
    ctx.profile(False)
    ctx.close()
    k = prof.get("ofdm_demod_kernel", {"ms": float("nan"), "n": 1})
    return step_ms, k["ms"] / max(k["n"], 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--cases", default=",".join(CASES), help="comma-separated subset of " + ", ".join(CASES))
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch
    from conftest import load_pkg
    pkg = load_pkg()
    torch.cuda.set_device(0)
    dev = torch.device("cuda:0")
    S = a.batch
    buf = fill(torch, dev, S, rings(8), lambda s: 20.0, 0x0FD0)
    out = {"card": card(), "batch": S, "steps": a.steps, "cases": {}}
    for name in a.cases.split(","):
        c = CASES[name]
        step_ms, ofdm_ms = run_case(pkg, buf, S, a.steps, c["keep_taps"], c["sub"])
        fb = frame_bytes(c["sub"], not c["keep_taps"])
        out["cases"][name] = dict(step_ms=round(step_ms, 3), ofdm_demod_ms=round(ofdm_ms, 3), **fb,
                                  hbm_share=round(fb["bytes"] * S / (ofdm_ms * 1e-3) / HBM_BPS, 3))
        print(name, out["cases"][name], flush=True)
    print(json.dumps(out))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
