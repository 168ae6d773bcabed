"""Cost and gain of the weighted soft-decision demap (dabb_options.soft_demap = DABB_DEMAP_WEIGHTED).

  python scripts/soft_measure.py [--batch 4096] [--steps 10] [--reps 4] [--streams 256] [--out FILE.json]

Prints one JSON object:
  - step time with the reference and the weighted demap, in alternating runs of --steps steps at the benchmark's configuration (4096
    streams, one 96 kbit/s EEP 3-A DAB+ sub-channel, keep_taps off, AWGN at --snr dB), each timed with CUDA events on the context's
    stream (dabb_join_lanes before the closing event);
  - ofdm_demod_kernel's device time per step in each mode from dabb_profile (serial per-kernel timing);
  - a sensitivity table on the closed loop: FIB CRC pass rate, RS-uncorrectable superframe rate and AU CRC failure rate of the DAB+
    sub-channel against SNR, for AWGN, two paths [(0, 1), (20, 0.95j)], three paths [(0, 1), (37, 0.7-0.3j), (211, 0.5j)] and a CW
    tone at +301 kHz 20 dB above the ensemble, both modes on the same recordings, --streams streams per point.  The SNR is that of the
    received ensemble (after the echoes, without the tone).  With the tone no stream acquires (the null-symbol search sees it), so its
    rows count no FIBs; the tests check the tone at stage level;
  - the card's name and power limit, which belong to every number.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "scripts")); sys.path.insert(0, os.path.join(ROOT, "tests"))

from ber_measure import BUF_LEN, RING_FRAMES, TF, card, fill, make_stepper, rings  # noqa: E402

CHANNELS = {"awgn": None, "2path": [(0, 1.0), (20, 0.95j)], "3path": [(0, 1.0), (37, 0.7 - 0.3j), (211, 0.5j)], "tone": "tone"}
SNRS = (3.0, 4.0, 5.0, 6.0, 8.0)


def received(torch, dev, rings_np, name):
    """the rings through the channel (complex64 numpy, periodic, so the echoes wrap) and the ensemble's received power"""
    out = []
    for r in rings_np:
        x = r.astype(np.complex128)
        ch = CHANNELS[name]
        if ch not in (None, "tone"):
            x = sum(g * np.roll(x, d) for d, g in ch)
        p = float(np.mean(np.abs(x) ** 2))
        if ch == "tone":
            x = x + np.sqrt(100 * p) * np.exp(2j * np.pi * 301000.0 * np.arange(len(x)) / 2048000.0)
        out.append((x.astype(np.complex64), p))
    return out


def sensitivity(pkg, torch, dev, rings_np, n, weighted):
    rows = []
    for name in CHANNELS:
        rx = received(torch, dev, rings_np, name)
        p_ens = np.mean([p for _, p in rx])
        p_all = np.mean([float(np.mean(np.abs(x) ** 2)) for x, _ in rx])
        S = n * len(SNRS)
        # fill() sets the noise from the power of what it is given: refer the SNR to the ensemble's power instead
        buf = fill(torch, dev, S, [x for x, _ in rx], lambda s: SNRS[s // n] + 10 * np.log10(p_all / p_ens), 0x50F0)
        ctx, step = make_stepper(pkg, S, buf)
        ctx.set_options(disable_coarse=True, soft_demap=pkg.DEMAP_WEIGHTED if weighted else pkg.DEMAP_REFERENCE)
        acc = np.zeros((len(SNRS), 6), np.int64)    # fibs, fibs ok, rs events, rs uncorrectable, AUs, AU CRC failures
        for i in range(14):
            step(); ctx.sync()
            if i < 6:                                  # acquisition and the de-interleaver's warm-up
                continue
            r = ctx.read_tap(5)
            dec = r["status"] == pkg.FRAME_DECODED
            ok = np.array([bin(int(m)).count("1") for m in r["fib_crc_mask"]])
            nev = r["n_rs_events"][:, 0].astype(np.int64)
            bad = np.array([bin(int(m) & ((1 << int(k)) - 1)).count("1") for m, k in zip(r["rs_uncorr_mask"][:, 0], nev)])
            nau = np.where(r["sf_ready"][:, 0] != 0, r["sf_au_count"][:, 0], 0).astype(np.int64)
            aub = np.array([int(k) - bin(int(m) & ((1 << int(k)) - 1)).count("1") for m, k in zip(r["sf_au_crc_mask"][:, 0], nau)])   # bit i: AU i CRC ok
            for j in range(len(SNRS)):
                sl = slice(j * n, (j + 1) * n)
                acc[j] += [12 * dec[sl].sum(), ok[sl][dec[sl]].sum(), nev[sl].sum(), bad[sl].sum(), nau[sl].sum(), aub[sl].sum()]
        ctx.close(); del buf; torch.cuda.empty_cache()
        for j, snr in enumerate(SNRS):
            nf, nok, ne, nb, na, nab = (int(x) for x in acc[j])
            rows.append({"channel": name, "snr_db": snr, "fib_crc_pass": nok / max(nf, 1), "rs_uncorrectable": nb / max(ne, 1),
                         "au_crc_fail": nab / max(na, 1), "fibs": nf, "rs_events": ne, "aus": na})
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--reps", type=int, default=4)
    ap.add_argument("--snr", type=float, default=20.0, help="AWGN SNR of the timed batch")
    ap.add_argument("--streams", type=int, default=256, help="streams per point of the sensitivity table")
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch
    from conftest import load_pkg
    pkg = load_pkg()
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    res = {"batch": a.batch, "card": card()}
    rings_np = rings(4)
    S = a.batch
    # ---- cost at the headline batch
    buf = fill(torch, dev, S, rings_np, lambda s: a.snr, 0x50F1)
    ctx, step = make_stepper(pkg, S, buf)
    ext = torch.cuda.ExternalStream(ctx.cuda_stream(), device=dev)
    for _ in range(8):
        step()
    ctx.sync()
    modes = {"reference": pkg.DEMAP_REFERENCE, "weighted": pkg.DEMAP_WEIGHTED}
    times = {m: [] for m in modes}
    for rep in range(a.reps):
        for m, v in modes.items():
            ctx.set_options(disable_coarse=True, soft_demap=v)
            step(); ctx.sync()                    # one untimed step in the new mode
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(ext)
            for _ in range(a.steps):
                step()
            ctx.join_lanes(); e1.record(ext); torch.cuda.synchronize()
            times[m].append(e0.elapsed_time(e1) / a.steps)
    res["step_ms"] = {m: {"runs": v, "median": float(np.median(v))} for m, v in times.items()}
    res["step_ms"]["weighted_cost_median"] = res["step_ms"]["weighted"]["median"] - res["step_ms"]["reference"]["median"]
    res["ofdm_demod_kernel_ms_per_step"] = {}
    for rep in range(2):
        for m, v in modes.items():
            ctx.set_options(disable_coarse=True, soft_demap=v)
            step(); ctx.sync()
            ctx.profile(True)
            for _ in range(a.steps):
                step()
            ctx.sync()
            prof = ctx.profile_read(); ctx.profile(False)
            k = prof["ofdm_demod_kernel"]
            res["ofdm_demod_kernel_ms_per_step"].setdefault(m, []).append(k["ms"] / k["n"])
    ctx.close(); del buf; torch.cuda.empty_cache()
    # ---- sensitivity
    table = {m: sensitivity(pkg, torch, dev, rings_np, a.streams, m == "weighted") for m in modes}
    res["sensitivity"] = table
    res["note"] = ("step times: decode step of the whole batch with the benchmark's configuration; kernel time: serial per-kernel profile; "
                   f"sensitivity: {a.streams} streams per point, 8 steps each after 6 warm-up steps, the same recordings and noise in both modes")
    txt = json.dumps(res, indent=1)
    print(txt)
    print("\n  channel SNR dB | FIB CRC pass ref / weighted | RS uncorrectable ref / weighted | AU CRC fail ref / weighted")
    for r0, r1 in zip(table["reference"], table["weighted"]):
        print(f"  {r0['channel']:6s} {r0['snr_db']:5.1f} | {r0['fib_crc_pass']:.4f} / {r1['fib_crc_pass']:.4f} | "
              f"{r0['rs_uncorrectable']:.4f} / {r1['rs_uncorrectable']:.4f} | {r0['au_crc_fail']:.4f} / {r1['au_crc_fail']:.4f}")
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write(txt + "\n")


if __name__ == "__main__":
    main()
