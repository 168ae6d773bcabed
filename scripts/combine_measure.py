"""Cost and gain of diversity reception (dabb_set_combining).

  python scripts/combine_measure.py [--batch 4096] [--steps 10] [--reps 4] [--pairs 32] [--out FILE.json]

Prints one JSON object:
  - step time of the benchmark's configuration (--batch streams, one 96 kbit/s EEP 3-A DAB+ sub-channel, keep_taps off) grouped in
    pairs (--batch / 2 groups of 2: streams 2g and 2g + 1 receive the same ring of ber_measure.rings with their own AWGN at --snr dB)
    against the same batch ungrouped, in alternating runs of --steps steps on one context (dabb_set_combining(None) / the pairs between
    runs), each timed with CUDA events on the context's stream (dabb_join_lanes before the closing event); the launches per step of both;
  - the device time per step of ofdm_demod_kernel, null_power_kernel and combine_kernel in both from dabb_profile (serial timing);
  - gain tables: --pairs transmitters per point, each received by two antennas with their own channel (AWGN, or the two- and three-path
    channels of tests/test_gpu_combine.py with different echo phases per antenna) and their own noise, at 3 and 5 dB, under both demaps:
    FIB CRC passes, RS-uncorrectable superframe codewords and FIC channel BER (tap 10) of antenna A alone, antenna B alone and the
    combined leader, over steps 2 .. 9 of 10;
  - the card's name and power limit, which belong to every number.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "scripts")); sys.path.insert(0, os.path.join(ROOT, "tests"))

from ber_measure import BITRATE, SUBCH_CU, card, fill, make_stepper, rings  # noqa: E402

POINTS = [("awgn", 3.0), ("awgn", 5.0), ("2path", 3.0), ("2path", 5.0), ("3path", 3.0), ("3path", 5.0)]
CHANNELS = {"awgn": (None, None), "2path": ([(0, 1.0), (20, 0.95j)], [(0, 1.0), (20, -0.95)]),
            "3path": ([(0, 1.0), (37, 0.7 - 0.3j), (211, 0.5j)], [(0, 1.0), (37, -0.3 + 0.7j), (211, -0.5)])}
GAIN_STEPS, GAIN_FROM = 10, 2


def gain_point(pkg, name, snr, pairs, weighted, seed):
    import dabtx
    import ofdmref
    ca, cb = CHANNELS[name]
    sig = []
    for t in range(pairs):
        clean = dabtx.DabTx(seed=seed + t).frames(GAIN_STEPS + 1)
        for i, ch in enumerate((ca, cb)):
            x = ofdmref.multipath(clean, ch) if ch else clean
            sig.append(dabtx.add_awgn(x, snr, seed=seed + 1000 + 2 * t + i, signal_power=float(np.mean(np.abs(x) ** 2))))
    sig = np.stack(sig).astype(np.complex64)
    S = len(sig)
    out = {}
    for mode in ("alone", "combined"):
        ctx = pkg.Context(n_streams=S)
        ctx.select_subchannel(0, dabtx.eep_cu(BITRATE), BITRATE, eep_profile_a=True, eep_level=3, dabplus=True)
        ctx.set_options(count_bit_errors=True, soft_demap=pkg.DEMAP_WEIGHTED if weighted else pkg.DEMAP_REFERENCE)
        if mode == "combined":
            ctx.set_combining(np.arange(S) & ~1)
        d = ctx.dev(sig)
        acc = np.zeros((S, 4), np.int64)          # FIBs passed, RS uncorrectable, FIC errors, FIC bits
        for k in range(GAIN_STEPS):
            o = ctx.process(d, sig.shape[1], np.zeros(S, np.int64), sig.shape[1], msc_stride=3 * BITRATE, sf_stride=15 * BITRATE)
            b = ctx.read_tap(10)
            if k < GAIN_FROM:
                continue
            r = o["results"]
            for s in range(S):
                if r["status"][s] != pkg.FRAME_DECODED:
                    continue
                n = int(r["n_rs_events"][s][0])
                acc[s] += (bin(int(r["fib_crc_mask"][s])).count("1"), bin(int(r["rs_uncorr_mask"][s][0]) & ((1 << n) - 1)).count("1"),
                           int(b["fic_errors"][s]), int(b["fic_bits"][s] - b["fic_erasures"][s]))
        d.free(); ctx.close()
        out[mode] = acc

    def row(a):
        return {"fib_pass": int(a[:, 0].sum()), "rs_uncorrectable": int(a[:, 1].sum()), "fic_ber": float(a[:, 2].sum() / max(a[:, 3].sum(), 1))}
    return {"channel": name, "snr_db": snr, "demap": "weighted" if weighted else "reference", "fibs": 12 * pairs * (GAIN_STEPS - GAIN_FROM),
            "antenna_a": row(out["alone"][0::2]), "antenna_b": row(out["alone"][1::2]), "combined": row(out["combined"][0::2])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--reps", type=int, default=4)
    ap.add_argument("--snr", type=float, default=20.0, help="AWGN SNR of the timed batch")
    ap.add_argument("--pairs", type=int, default=32, help="transmitters (antenna pairs) per point of the gain tables")
    ap.add_argument("--no-gain", action="store_true")
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch
    from conftest import load_pkg
    pkg = load_pkg()
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    res = {"batch": a.batch, "card": card()}
    S = a.batch
    r4 = rings(4)
    buf = fill(torch, dev, S, [r for r in r4 for _ in range(2)], lambda s: a.snr, 0xC0B0)     # streams 2g, 2g + 1: one ring, own noise
    ctx, step = make_stepper(pkg, S, buf)
    ext = torch.cuda.ExternalStream(ctx.cuda_stream(), device=dev)
    pairs = np.arange(S) & ~1
    for _ in range(6):
        step()
    ctx.sync()
    modes = {"ungrouped": None, "pairs": pairs}
    times = {m: [] for m in modes}
    launches = {}
    for rep in range(a.reps):
        for m, tab in modes.items():
            ctx.set_combining(tab)
            step(); ctx.sync()
            n0 = ctx.kernel_launches()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(ext)
            for _ in range(a.steps):
                step()
            ctx.join_lanes(); e1.record(ext); torch.cuda.synchronize()
            times[m].append(e0.elapsed_time(e1) / a.steps)
            launches[m] = (ctx.kernel_launches() - n0) / a.steps
            if tab is not None:
                res["members"] = float(ctx.read_tap(12)["members"][::2].mean())
    res["step_ms"] = {m: {"runs": v, "median": float(np.median(v))} for m, v in times.items()}
    res["step_ms"]["pairs_cost_median"] = res["step_ms"]["pairs"]["median"] - res["step_ms"]["ungrouped"]["median"]
    res["launches_per_step"] = launches
    res["kernel_ms_per_step"] = {}
    for m, tab in modes.items():
        ctx.set_combining(tab)
        step(); ctx.sync()
        ctx.profile(True)
        for _ in range(a.steps):
            step()
        ctx.sync()
        prof = ctx.profile_read(); ctx.profile(False)
        res["kernel_ms_per_step"][m] = {k: v["ms"] / a.steps for k, v in prof.items() if k in ("ofdm_demod_kernel", "null_power_kernel", "combine_kernel")}
    ctx.close(); del buf; torch.cuda.empty_cache()
    if not a.no_gain:
        res["gain"] = [gain_point(pkg, n, snr, a.pairs, w, 0xC100 + 97 * i) for w in (False, True) for i, (n, snr) in enumerate(POINTS)]
    res["note"] = (f"step times: the whole batch ({S} streams, {SUBCH_CU} CU sub-channel at {BITRATE} kbit/s), ungrouped against "
                   f"{S // 2} groups of 2, alternating runs on one context; gain: {a.pairs} antenna pairs per point, steps {GAIN_FROM}.."
                   f"{GAIN_STEPS - 1}")
    txt = json.dumps(res, indent=1)
    print(txt)
    for g in res.get("gain", []):
        A, B, Cb = g["antenna_a"], g["antenna_b"], g["combined"]
        print(f"  {g['demap']:9s} {g['channel']:5s} {g['snr_db']:3.0f} dB | FIBs {A['fib_pass']}/{B['fib_pass']} -> {Cb['fib_pass']} of {g['fibs']} | "
              f"RS uncorr {A['rs_uncorrectable']}/{B['rs_uncorrectable']} -> {Cb['rs_uncorrectable']} | FIC BER {A['fic_ber']:.2e}/{B['fic_ber']:.2e} -> {Cb['fic_ber']:.2e}")
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write(txt + "\n")


if __name__ == "__main__":
    main()
