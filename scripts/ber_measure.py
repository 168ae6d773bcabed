"""Cost of the device channel bit-error count (dabb_options.count_bit_errors, tap 10) at the headline batch, and the channel BER it
reports against AWGN SNR: 4096 streams in the benchmark's configuration (one 96 kbit/s EEP 3-A DAB+ sub-channel, keep_taps off).

  python scripts/ber_measure.py [--batch 4096] [--steps 10] [--reps 4] [--out FILE.json]

Prints one JSON object:
  - step time with count_bit_errors off and on, in alternating runs of --steps steps, each timed with CUDA events on the context's
    stream (dabb_join_lanes before the closing event);
  - ber_kernel's device time per step from dabb_profile (serial per-kernel timing), and the bytes it reads;
  - a table: AWGN SNR -> FIC and sub-channel channel BER (errors / (bits - erasures)) and the FIB CRC pass rate, over --snr-streams
    streams per SNR;
  - the card's name and power limit, which belong to every number.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))

TF = 196608
RING_FRAMES = 5
BUF_LEN = (RING_FRAMES + 1) * TF + 4096
BITRATE, SUBCH_CU = 96, 72
SNRS = (2.0, 3.0, 4.0, 5.0, 6.0, 8.0, 10.0, 14.0)


def card():
    import torch
    out = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        import pynvml as nv
        nv.nvmlInit()
        out["power_limit_w"] = nv.nvmlDeviceGetPowerManagementLimit(nv.nvmlDeviceGetHandleByIndex(0)) / 1000.0
    except Exception as e:  # noqa
        out["power_limit_w"] = f"not read ({type(e).__name__})"
    return out


def rings(n):
    import dabtx
    return [dabtx.periodic_ring(0xBE00 + i, n_frames=RING_FRAMES)[1] for i in range(n)]


def fill(torch, dev, S, rings_np, snr_of, seed):
    """[S, BUF_LEN, 2] float32 on the device: stream s = ring s % len(rings) plus AWGN at snr_of(s) dB, wrapped to BUF_LEN"""
    r = torch.from_numpy(np.stack(rings_np).view(np.float32).reshape(len(rings_np), RING_FRAMES * TF, 2)).to(dev)
    p = float((r[:, 3000:190000] ** 2).sum(-1).mean())
    buf = torch.empty((S, BUF_LEN, 2), dtype=torch.float32, device=dev)
    gen = torch.Generator(device=dev); gen.manual_seed(seed)
    for s0 in range(0, S, 256):
        n = min(256, S - s0)
        sig = torch.tensor([(p / (10 ** (snr_of(s) / 10)) / 2) ** 0.5 for s in range(s0, s0 + n)], device=dev).view(n, 1, 1)
        blk = r[torch.arange(s0, s0 + n, device=dev) % len(rings_np)] + torch.randn((n, RING_FRAMES * TF, 2), device=dev, generator=gen) * sig
        buf[s0:s0 + n, :RING_FRAMES * TF] = blk
        buf[s0:s0 + n, RING_FRAMES * TF:] = blk[:, :BUF_LEN - RING_FRAMES * TF]
        del blk
    torch.cuda.synchronize()
    return buf


def make_stepper(pkg, S, buf):
    ctx = pkg.Context(n_streams=S, disable_coarse=True, n_subch_slots=1, max_subch_cu=SUBCH_CU)
    ctx.select_subchannel(0, SUBCH_CU, BITRATE, eep_profile_a=True, eep_level=3, dabplus=True)
    call = [0]

    def step():
        n = call[0] + 1
        bs = np.full(S, RING_FRAMES * TF * (n // RING_FRAMES), np.int64) if call[0] > 0 else np.zeros(S, np.int64)
        ctx.process_async(buf.data_ptr(), BUF_LEN, bs, BUF_LEN); call[0] += 1
    return ctx, step


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--reps", type=int, default=4)
    ap.add_argument("--snr", type=float, default=20.0, help="AWGN SNR of the timed batch")
    ap.add_argument("--snr-streams", type=int, default=256, help="streams per SNR of the BER table")
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
    buf = fill(torch, dev, S, rings_np, lambda s: a.snr, 0xBE1)
    ctx, step = make_stepper(pkg, S, buf)
    ext = torch.cuda.ExternalStream(ctx.cuda_stream(), device=dev)
    for _ in range(8):
        step()
    ctx.sync()
    times = {"off": [], "on": []}
    for rep in range(a.reps):
        for mode in ("off", "on"):
            ctx.set_options(disable_coarse=True, count_bit_errors=mode == "on")
            step(); ctx.sync()                    # one untimed step in the new mode
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(ext)
            for _ in range(a.steps):
                step()
            ctx.join_lanes(); e1.record(ext); torch.cuda.synchronize()
            times[mode].append(e0.elapsed_time(e1) / a.steps)
    res["step_ms"] = {m: {"runs": v, "median": float(np.median(v))} for m, v in times.items()}
    res["step_ms"]["ber_cost_median"] = res["step_ms"]["on"]["median"] - res["step_ms"]["off"]["median"]
    ctx.set_options(disable_coarse=True, count_bit_errors=True)
    ctx.profile(True)
    for _ in range(a.steps):
        step()
    ctx.sync()
    prof = ctx.profile_read(); ctx.profile(False)
    k = prof.get("ber_kernel")
    step(); ctx.sync()
    t10 = ctx.read_tap(10)
    soft_bytes = int(t10["fic_bits"].sum()) + int(t10["subch"]["bits"][:, 0].sum())
    res["ber_kernel"] = {"ms_per_step": k["ms"] / k["n"] if k else None, "softbits_read_per_step": soft_bytes,
                         "GB_per_s_softbits": (soft_bytes / (k["ms"] / k["n"]) / 1e6) if k else None,
                         "viterbi_kernel_MSC_ms_per_step": prof["viterbi_kernel(MSC)"]["ms"] / prof["viterbi_kernel(MSC)"]["n"] if "viterbi_kernel(MSC)" in prof else None}
    ctx.close(); del buf; torch.cuda.empty_cache()
    # ---- channel BER against SNR
    n = a.snr_streams
    S2 = n * len(SNRS)
    buf = fill(torch, dev, S2, rings_np, lambda s: SNRS[s // n], 0xBE2)
    ctx, step = make_stepper(pkg, S2, buf)
    ctx.set_options(disable_coarse=True, count_bit_errors=True)
    acc = np.zeros((len(SNRS), 8), np.int64)       # fic bits, errors, erasures, msc bits, errors, erasures, fibs, fibs ok
    for i in range(14):
        ctx.process_async(buf.data_ptr(), BUF_LEN, np.full(S2, RING_FRAMES * TF * ((i + 1) // RING_FRAMES) if i else 0, np.int64), BUF_LEN)
        ctx.sync()
        if i < 6:                                  # acquisition and the de-interleaver's warm-up
            continue
        r, t = ctx.read_tap(5), ctx.read_tap(10)
        dec = r["status"] == pkg.FRAME_DECODED
        mask = r["fib_crc_mask"].astype(np.int64)
        ok = np.array([bin(int(m)).count("1") for m in mask])
        for j in range(len(SNRS)):
            sl = slice(j * n, (j + 1) * n)
            acc[j] += [t["fic_bits"][sl].sum(), t["fic_errors"][sl].sum(), t["fic_erasures"][sl].sum(), t["subch"]["bits"][sl, 0].sum(),
                       t["subch"]["errors"][sl, 0].sum(), t["subch"]["erasures"][sl, 0].sum(), 12 * dec[sl].sum(), ok[sl][dec[sl]].sum()]
    ctx.close()
    table = []
    for j, snr in enumerate(SNRS):
        fb, fe, fz, mb, me, mz, nf, nok = (int(x) for x in acc[j])
        table.append({"snr_db": snr, "fic_ber": fe / max(fb - fz, 1), "msc_ber": me / max(mb - mz, 1), "fib_crc_pass": nok / max(nf, 1),
                      "fic_bits": fb, "msc_bits": mb})
    res["ber_vs_snr"] = table
    res["note"] = ("step times: decode step of the whole batch with the benchmark's configuration; kernel time: serial per-kernel profile; "
                   f"BER table: {n} streams per SNR, 8 steps each after 6 warm-up steps")
    txt = json.dumps(res, indent=1)
    print(txt)
    print("\n  SNR dB | FIC BER   | MSC BER   | FIB CRC pass")
    for row in table:
        print(f"  {row['snr_db']:6.1f} | {row['fic_ber']:.3e} | {row['msc_ber']:.3e} | {row['fib_crc_pass']:.4f}")
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write(txt + "\n")


if __name__ == "__main__":
    main()
