"""Cost of the device MER measurement (dabb_set_mer, tap 14) at the headline batch, and what it reports: 4096 streams in the benchmark's
configuration (one 96 kbit/s EEP 3-A DAB+ sub-channel, keep_taps off), the same rings and helpers as scripts/ber_measure.py.

  python scripts/mer_measure.py [--batch 4096] [--steps 10] [--reps 4] [--snr-streams 256] [--out FILE.json]

Prints one JSON object:
  - step time with the measurement off and on, in alternating runs of --steps steps, each timed with CUDA events on the context's
    stream (dabb_join_lanes before the closing event);
  - mer_kernel's device time per step from dabb_profile (serial per-kernel timing), the softbits it reads (9216 per stream) and the
    time those bytes take at the data sheet's 3.35 TB/s (the memory bound, which is the one that applies: the kernel does a few integer
    operations per byte);
  - a table: AWGN SNR -> MER of the band (summed over the streams and steps) and the FIC channel BER of tap 10 from the same run, over
    --snr-streams streams per SNR;
  - 64-group MER profiles at 25 dB SNR for two-path and three-path channels and for a tone 10 dB above the ensemble on carrier 301 and
    half a carrier off it;
  - the card's name and power limit, which belong to every number.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, os.path.join(ROOT, "scripts"))

from ber_measure import BUF_LEN, RING_FRAMES, TF, card, fill, make_stepper, rings  # noqa: E402

SNRS = (2.0, 4.0, 6.0, 8.0, 10.0, 12.0, 15.0, 20.0, 25.0, 30.0, 35.0, 40.0)
HBM_BYTES_PER_S = 3.35e12


def profiles(pkg):
    """64-group MER (dB) over 8 steps of each channel at 25 dB SNR, one stream each"""
    import dabtx
    import merref as M
    base = dabtx.DabTx(seed=0x3F00).frames(10)
    cases = {"awgn": dabtx.add_awgn(base, 25, seed=1),
             "two_path_0_20": dabtx.add_awgn(M.two_path(base, [(0, 1), (20, 0.95j)]), 25, seed=2),
             "three_path_0_13_37": dabtx.add_awgn(M.two_path(base, [(0, 1), (13, 0.6j), (37, -0.5)]), 25, seed=3),
             "tone_301000_hz_10_db": M.tone(dabtx.add_awgn(base, 25, seed=4), 301000, 10, seed=1),
             "tone_301500_hz_10_db": M.tone(dabtx.add_awgn(base, 25, seed=5), 301500, 10, seed=1)}
    buf = np.stack(list(cases.values()))
    S = len(cases)
    ctx = pkg.Context(n_streams=S)
    ctx.set_options(disable_coarse=True, acquisition=pkg.ACQ_ROBUST)
    ctx.set_mer(True)
    d = ctx.dev(buf)
    gs, ge = np.zeros((S, 64), np.int64), np.zeros((S, 64), np.int64)
    for _ in range(9):
        ctx.process(d, buf.shape[1], np.zeros(S, np.int64), buf.shape[1])
        t = ctx.read_tap(14)
        gs += t["group"]["sig"]; ge += t["group"]["err"]
    ctx.close()
    out = {}
    for i, name in enumerate(cases):
        g = [round(M.mer_db(int(a), int(b)), 2) for a, b in zip(gs[i], ge[i])]
        out[name] = {"band_db": round(M.mer_db(int(gs[i].sum()), int(ge[i].sum())), 2), "min_group": int(np.argmin(g)), "groups_db": g}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--reps", type=int, default=4)
    ap.add_argument("--snr", type=float, default=20.0, help="AWGN SNR of the timed batch")
    ap.add_argument("--snr-streams", type=int, default=256, help="streams per SNR of the MER table")
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch
    import merref as M
    from conftest import load_pkg
    pkg = load_pkg()
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    res = {"batch": a.batch, "card": card()}
    rings_np = rings(4)
    S = a.batch
    # ---- cost at the headline batch
    buf = fill(torch, dev, S, rings_np, lambda s: a.snr, 0x3F1)
    ctx, step = make_stepper(pkg, S, buf)
    ext = torch.cuda.ExternalStream(ctx.cuda_stream(), device=dev)
    for _ in range(8):
        step()
    ctx.sync()
    times = {"off": [], "on": []}
    for rep in range(a.reps):
        for mode in ("off", "on"):
            ctx.set_mer(mode == "on")
            step(); ctx.sync()                    # one untimed step in the new mode
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(ext)
            for _ in range(a.steps):
                step()
            ctx.join_lanes(); e1.record(ext); torch.cuda.synchronize()
            times[mode].append(e0.elapsed_time(e1) / a.steps)
    res["step_ms"] = {m: {"runs": v, "median": float(np.median(v))} for m, v in times.items()}
    res["step_ms"]["mer_cost_median"] = res["step_ms"]["on"]["median"] - res["step_ms"]["off"]["median"]
    ctx.set_mer(True)
    ctx.profile(True)
    for _ in range(a.steps):
        step()
    ctx.sync()
    prof = ctx.profile_read(); ctx.profile(False)
    k = prof.get("mer_kernel")
    step(); ctx.sync()
    dec = int((ctx.read_tap(5)["status"] == pkg.FRAME_DECODED).sum())
    soft_bytes = 9216 * S
    ms = k["ms"] / k["n"] if k else None
    res["mer_kernel"] = {"ms_per_step": ms, "streams_decoded_last_step": dec, "softbits_read_per_step": soft_bytes,
                         "hbm_bound_ms": soft_bytes / HBM_BYTES_PER_S * 1e3,
                         "achieved_GB_per_s": (soft_bytes / ms / 1e6) if ms else None}
    ctx.close(); del buf; torch.cuda.empty_cache()
    # ---- MER and FIC BER against SNR
    n = a.snr_streams
    S2 = n * len(SNRS)
    buf = fill(torch, dev, S2, rings_np, lambda s: SNRS[s // n], 0x3F2)
    ctx, step = make_stepper(pkg, S2, buf)
    ctx.set_options(disable_coarse=True, count_bit_errors=True)
    ctx.set_mer(True)
    acc = np.zeros((len(SNRS), 5), np.int64)       # mer sig, err, fic bits, errors, erasures
    for i in range(14):
        step(); ctx.sync()
        if i < 6:
            continue
        t, b = ctx.read_tap(14), ctx.read_tap(10)
        for j in range(len(SNRS)):
            sl = slice(j * n, (j + 1) * n)
            acc[j] += [t["sig"][sl].sum(), t["err"][sl].sum(), b["fic_bits"][sl].sum(), b["fic_errors"][sl].sum(), b["fic_erasures"][sl].sum()]
    ctx.close(); del buf; torch.cuda.empty_cache()
    table = []
    for j, snr in enumerate(SNRS):
        sig, err, fb, fe, fz = (int(x) for x in acc[j])
        table.append({"snr_db": snr, "per_carrier_snr_db": snr + 1.25, "mer_db": round(M.mer_db(sig, err), 3), "fic_ber": fe / max(fb - fz, 1),
                      "fic_bits": fb})
    res["mer_vs_snr"] = table
    res["profiles_25db"] = profiles(pkg)
    res["note"] = ("step times: decode step of the whole batch with the benchmark's configuration; kernel time: serial per-kernel profile; "
                   f"MER table: {n} streams per SNR, 8 steps each after 6 warm-up steps; SNR over 2.048 MHz (tests/dabtx.add_awgn)")
    txt = json.dumps(res, indent=1)
    print(txt)
    print("\n  SNR dB | MER dB  | FIC BER")
    for row in table:
        print(f"  {row['snr_db']:6.1f} | {row['mer_db']:7.2f} | {row['fic_ber']:.3e}")
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write(txt + "\n")


if __name__ == "__main__":
    main()
