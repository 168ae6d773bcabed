"""Cost and gain of sample-clock tracking (dabb_options.sample_clock = DABB_CLOCK_TRACK).

  python scripts/clock_measure.py [--batch 4096] [--steps 10] [--reps 4] [--streams 256] [--out FILE.json]

Every stream decodes a periodic ring of 5 frames (ber_measure.rings) resampled as a receiver whose sample clock is off by the point's ppm
records it (tests/clockref.py: an FFT resample of the ring to round(5 T_F (1 + eps)) samples, periodic like the ring), plus AWGN.
Prints one JSON object:
  - step time with the option OFF and TRACK, in alternating runs of --steps steps at the benchmark's configuration (4096 streams, one
    96 kbit/s EEP 3-A DAB+ sub-channel, keep_taps off, AWGN at --snr dB) on rings at 100 ppm, after enough steps that TRACK derotates
    every frame; each run timed with CUDA events on the context's stream (dabb_join_lanes before the closing event);
  - ofdm_demod_kernel's device time per step in each mode from dabb_profile (serial per-kernel timing);
  - a gain table: FIC and sub-channel channel BER (tap 10), FIB CRC pass rate and RS-uncorrectable superframes for ppm {0, 25, 50,
    100, 150} x SNR {6, 8, 10, 14} dB, OFF against TRACK on the same recordings, --streams streams per point, counted over steps 12 ..
    43 of 44; and TRACK's estimate error (tap 11's ppm minus the injected ppm) at the last step;
  - the card's name and power limit, which belong to every number.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "scripts")); sys.path.insert(0, os.path.join(ROOT, "tests"))

from ber_measure import BITRATE, RING_FRAMES, SUBCH_CU, TF, card, rings  # noqa: E402
import clockref  # noqa: E402

PPMS = (0.0, 25.0, 50.0, 100.0, 150.0)
SNRS = (6.0, 8.0, 10.0, 14.0)
GAIN_STEPS, GAIN_FROM = 44, 12


def resampled_rings(rings_np, ppm):
    out = [clockref.resample_clock(r, ppm) for r in rings_np]
    return [y for y, _ in out], out[0][1]


def fill(torch, dev, S, rings_np, snr_of, seed):
    """[S, buf_len, 2] float32 on the device: stream s = ring s % len(rings) plus AWGN at snr_of(s) dB, wrapped by one frame; the ring length"""
    M = len(rings_np[0])
    buf_len = M + TF + 4096
    r = torch.from_numpy(np.stack(rings_np).view(np.float32).reshape(len(rings_np), M, 2)).to(dev)
    p = float((r[:, 3000:190000] ** 2).sum(-1).mean())
    buf = torch.empty((S, buf_len, 2), dtype=torch.float32, device=dev)
    gen = torch.Generator(device=dev); gen.manual_seed(seed)
    for s0 in range(0, S, 256):
        n = min(256, S - s0)
        sig = torch.tensor([(p / (10 ** (snr_of(s) / 10)) / 2) ** 0.5 for s in range(s0, s0 + n)], device=dev).view(n, 1, 1)
        blk = r[torch.arange(s0, s0 + n, device=dev) % len(rings_np)] + torch.randn((n, M, 2), device=dev, generator=gen) * sig
        buf[s0:s0 + n, :M] = blk
        buf[s0:s0 + n, M:] = blk[:, :buf_len - M]
        del blk
    torch.cuda.synchronize()
    return buf, M


def make_stepper(pkg, S, buf, M):
    """ber_measure.make_stepper for a ring of M samples (RING_FRAMES frames of the recording's clock)"""
    ctx = pkg.Context(n_streams=S, disable_coarse=True, n_subch_slots=1, max_subch_cu=SUBCH_CU)
    ctx.select_subchannel(0, SUBCH_CU, BITRATE, eep_profile_a=True, eep_level=3, dabplus=True)
    call = [0]
    buf_len = buf.shape[1]

    def step():
        n = call[0] + 1
        bs = np.full(S, M * (n // RING_FRAMES), np.int64) if call[0] > 0 else np.zeros(S, np.int64)
        ctx.process_async(buf.data_ptr(), buf_len, bs, buf_len); call[0] += 1
    return ctx, step


def gain(pkg, torch, dev, rings_np, n, ppm, mode):
    rr, eff = resampled_rings(rings_np, ppm)
    S = n * len(SNRS)
    buf, M = fill(torch, dev, S, rr, lambda s: SNRS[s // n], 0xC1A0)
    ctx, step = make_stepper(pkg, S, buf, M)
    ctx.set_options(disable_coarse=True, count_bit_errors=True, sample_clock=mode)
    acc = np.zeros((len(SNRS), 8), np.int64)      # fic errors, fic bits, subch errors, subch bits, fibs, fibs ok, rs events, rs uncorrectable
    for i in range(GAIN_STEPS):
        step(); ctx.sync()
        if i < GAIN_FROM:
            continue
        r = ctx.read_tap(5); b = ctx.read_tap(10)
        dec = r["status"] == pkg.FRAME_DECODED
        ok = np.array([bin(int(m)).count("1") for m in r["fib_crc_mask"]])
        nev = r["n_rs_events"][:, 0].astype(np.int64)
        bad = np.array([bin(int(m) & ((1 << int(k)) - 1)).count("1") for m, k in zip(r["rs_uncorr_mask"][:, 0], nev)])
        row = np.stack([b["fic_errors"], b["fic_bits"] - b["fic_erasures"], b["subch"]["errors"][:, 0],
                        b["subch"]["bits"][:, 0] - b["subch"]["erasures"][:, 0], 12 * dec, np.where(dec, ok, 0), nev, bad], 1).astype(np.int64)
        for j in range(len(SNRS)):
            acc[j] += row[j * n:(j + 1) * n].sum(0)
    est = ctx.read_tap(11) if mode else None
    ctx.close(); del buf; torch.cuda.empty_cache()
    rows = []
    for j, snr in enumerate(SNRS):
        fe, fb, se, sb, nf, nok, ne, nb = (int(x) for x in acc[j])
        row = {"ppm": ppm, "snr_db": snr, "fic_ber": fe / max(fb, 1), "msc_ber": se / max(sb, 1), "fib_crc_pass": nok / max(nf, 1),
               "rs_uncorrectable": nb, "rs_events": ne, "fibs": nf}
        if est is not None:
            e = est["ppm"][j * n:(j + 1) * n].astype(np.float64) - eff
            row["estimate_error_ppm"] = {"mean": float(e.mean()), "max_abs": float(np.abs(e).max()), "frames_min": int(est["frames"][j * n:(j + 1) * n].min())}
        rows.append(row)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--reps", type=int, default=4)
    ap.add_argument("--snr", type=float, default=20.0, help="AWGN SNR of the timed batch")
    ap.add_argument("--streams", type=int, default=256, help="streams per point of the gain table")
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
    # ---- cost at the headline batch, on rings at 100 ppm
    rr, _ = resampled_rings(rings_np, 100.0)
    buf, M = fill(torch, dev, S, rr, lambda s: a.snr, 0xC1A1)
    ctx, step = make_stepper(pkg, S, buf, M)
    ext = torch.cuda.ExternalStream(ctx.cuda_stream(), device=dev)
    ctx.set_options(disable_coarse=True, sample_clock=pkg.CLOCK_TRACK)
    for _ in range(14):                            # acquisition and 8 counted frames: every frame is derotated from here on
        step()
    ctx.sync()
    modes = {"off": pkg.CLOCK_OFF, "track": pkg.CLOCK_TRACK}
    times = {m: [] for m in modes}
    applied = []
    for rep in range(a.reps):
        for m, v in modes.items():
            ctx.set_options(disable_coarse=True, sample_clock=v)
            step(); ctx.sync()                    # one untimed step in the new mode (TRACK: the first frame after OFF does not count)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(ext)
            for _ in range(a.steps):
                step()
            ctx.join_lanes(); e1.record(ext); torch.cuda.synchronize()
            times[m].append(e0.elapsed_time(e1) / a.steps)
            if v:
                applied.append(float((ctx.read_tap(11)["applied_ppm"] != 0).mean()))
    res["step_ms"] = {m: {"runs": v, "median": float(np.median(v))} for m, v in times.items()}
    res["step_ms"]["track_cost_median"] = res["step_ms"]["track"]["median"] - res["step_ms"]["off"]["median"]
    res["track_frames_derotated"] = applied
    res["ofdm_demod_kernel_ms_per_step"] = {}
    for rep in range(2):
        for m, v in modes.items():
            ctx.set_options(disable_coarse=True, sample_clock=v)
            step(); ctx.sync()
            ctx.profile(True)
            for _ in range(a.steps):
                step()
            ctx.sync()
            prof = ctx.profile_read(); ctx.profile(False)
            k = prof["ofdm_demod_kernel"]
            res["ofdm_demod_kernel_ms_per_step"].setdefault(m, []).append(k["ms"] / k["n"])
    ctx.close(); del buf; torch.cuda.empty_cache()
    # ---- gain
    table = {m: [row for p in PPMS for row in gain(pkg, torch, dev, rings_np, a.streams, p, v)] for m, v in modes.items()}
    res["gain"] = table
    res["note"] = ("step times: decode step of the whole batch with the benchmark's configuration on rings at 100 ppm; kernel time: serial "
                   f"per-kernel profile; gain: {a.streams} streams per point, steps {GAIN_FROM}..{GAIN_STEPS - 1}, the same recordings and noise in both modes")
    txt = json.dumps(res, indent=1)
    print(txt)
    print("\n  ppm  SNR dB | FIC BER off / track | MSC BER off / track | FIB CRC pass off / track | RS uncorr off / track | estimate error max")
    for r0, r1 in zip(table["off"], table["track"]):
        print(f"  {r0['ppm']:5.0f} {r0['snr_db']:5.1f} | {r0['fic_ber']:.2e} / {r1['fic_ber']:.2e} | {r0['msc_ber']:.2e} / {r1['msc_ber']:.2e} | "
              f"{r0['fib_crc_pass']:.4f} / {r1['fib_crc_pass']:.4f} | {r0['rs_uncorrectable']} / {r1['rs_uncorrectable']} | "
              f"{r1['estimate_error_ppm']['max_abs']:.3f}")
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write(txt + "\n")


if __name__ == "__main__":
    main()
