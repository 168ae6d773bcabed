"""Cost of decoding streams with different bitrates and protection profiles in one sub-channel slot (one grouped Viterbi launch), at
the headline batch: 4096 streams reading the benchmark's kind of resident periodic IQ ring.

  python scripts/mixed_subch_measure.py [--batch 4096] [--steps 10] [--reps 4] [--out FILE.json]

Two arms, each a context of its own, timed in alternating runs in one process:
  A  every stream decodes 96 kbit/s EEP 3-A DAB+ (the benchmark's sub-channel);
  B  stream s decodes MIX[s % 8] (DAB+; mean bitrate 78 kbit/s).
Every stream's ring carries the sub-channel it decodes (so that the superframe search syncs in both arms); the one IQ buffer is
refilled with the arm's rings before each of its runs.  Both arms use max_subch_cu = 96, so that they differ only in the profiles.
Prints one JSON object:
  - step time per arm, each run timed with CUDA events on the context's stream over --steps steps (dabb_join_lanes before the
    closing event);
  - every kernel's device time per step from dabb_profile (serial per-kernel timing), in a run of its own;
  - trellis steps per step (4 codewords per stream, 24 x bitrate + 6 steps each) and the add-compare-select rate they give
    (64 states per trellis step) over the MSC kernel time;
  - the card's name and power limit, which belong to every number.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))

TF = 196608
RING_FRAMES = 5
BUF_LEN = (RING_FRAMES + 1) * TF + 4096
MAX_CU = 96
# (bitrate kbit/s, EEP-A?, level, capacity units)
ARM_A = [(96, True, 3, 72)]
MIX = [(32, True, 3, 24), (48, True, 3, 36), (64, True, 3, 48), (80, True, 3, 60), (96, True, 3, 72), (112, True, 3, 84), (128, True, 3, 96),
       (64, False, 3, 36)]


def periodic_ring(seed, bitrate=96, profile_a=True, level=3):
    """a seamless 5-frame ring (the benchmark's resident input): content repeats every 4 superframes = 5 frames"""
    import dabtx
    tx = dabtx.DabTx(seed=seed, bitrate=bitrate, profile_a=profile_a, level=level, period_sf=4 * RING_FRAMES // 5)
    sig = np.concatenate([tx.modulate(tx.frame_bits()) for _ in range(2 * RING_FRAMES)])
    return sig[RING_FRAMES * TF:].astype(np.complex64)


def card():
    import torch
    out = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=60)
        lim, clk = [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")]
        out["power_limit_w"] = float(lim); out["max_sm_clock_mhz"] = float(clk)
    except Exception as e:  # noqa
        out["power_limit_w"] = f"not read ({type(e).__name__})"
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--reps", type=int, default=4)
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch
    from conftest import load_pkg
    pkg = load_pkg()
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    S = a.batch
    res = {"batch": S, "card": card(), "max_subch_cu": MAX_CU,
           "arms": {"A": {"profiles": ["96 kbit/s EEP 3-A"]},
                    "B": {"profiles": [f"{br} kbit/s EEP {lv}-{'A' if pa else 'B'}" for br, pa, lv, _ in MIX],
                          "mean_bitrate_kbps": float(np.mean([MIX[s % len(MIX)][0] for s in range(S)]))}}}
    def upload(rs):
        return torch.from_numpy(np.stack(rs).view(np.float32).reshape(len(rs), RING_FRAMES * TF, 2)).to(dev)
    ring_sets = {"A": upload([periodic_ring(0xB200 + i) for i in range(len(MIX))]),                  # stream s: ring s % 8
                 "B": upload([periodic_ring(0xB200 + i, br, pa, lv) for i, (br, pa, lv, _) in enumerate(MIX)])}
    buf = torch.empty((S, BUF_LEN, 2), dtype=torch.float32, device=dev)

    def fill(name):
        rings = ring_sets[name]
        for s0 in range(0, S, 256):
            n = min(256, S - s0)
            blk = rings[torch.arange(s0, s0 + n, device=dev) % rings.shape[0]]
            buf[s0:s0 + n, :RING_FRAMES * TF] = blk
            buf[s0:s0 + n, RING_FRAMES * TF:] = blk[:, :BUF_LEN - RING_FRAMES * TF]
        torch.cuda.synchronize()

    arms = {}
    for name, profs in (("A", ARM_A), ("B", MIX)):
        ctx = pkg.Context(n_streams=S, disable_coarse=True, n_subch_slots=1, max_subch_cu=MAX_CU)
        if len(profs) == 1:
            br, pa, lv, cu = profs[0]
            ctx.select_subchannel(0, cu, br, eep_profile_a=pa, eep_level=lv, dabplus=True)
        else:
            for s in range(S):
                br, pa, lv, cu = profs[s % len(profs)]
                ctx.select_subchannel(0, cu, br, eep_profile_a=pa, eep_level=lv, dabplus=True, first=s, count=1)
        steps_per_step = sum(4 * (24 * profs[s % len(profs)][0] + 6) for s in range(S))
        arms[name] = dict(ctx=ctx, ext=torch.cuda.ExternalStream(ctx.cuda_stream(), device=dev), call=0, trellis=steps_per_step)

    def step(arm):
        n = arm["call"] + 1
        bs = np.full(S, RING_FRAMES * TF * (n // RING_FRAMES), np.int64) if arm["call"] > 0 else np.zeros(S, np.int64)
        arm["ctx"].process_async(buf.data_ptr(), BUF_LEN, bs, BUF_LEN); arm["call"] += 1

    for name, arm in arms.items():     # acquisition, de-interleaver fill, warm kernels
        fill(name)
        for _ in range(8):
            step(arm)
        arm["ctx"].sync()
    times = {k: [] for k in arms}
    for rep in range(a.reps):
        for name, arm in arms.items():
            fill(name)
            step(arm); arm["ctx"].sync()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(arm["ext"])
            for _ in range(a.steps):
                step(arm)
            arm["ctx"].join_lanes(); e1.record(arm["ext"]); torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / a.steps)
    for name, arm in arms.items():
        ctx = arm["ctx"]
        fill(name)
        r = ctx.read_tap(5)
        decoded = int((r["status"] == pkg.FRAME_DECODED).sum())
        ctx.profile(True)
        for _ in range(a.steps):
            step(arm)
        ctx.sync()
        prof = ctx.profile_read(); ctx.profile(False)
        vit_ms = prof["viterbi_kernel(MSC)"]["ms"] / prof["viterbi_kernel(MSC)"]["n"]
        out = res["arms"][name]
        out["step_ms"] = {"runs": times[name], "median": float(np.median(times[name]))}
        out["viterbi_msc_ms_per_step"] = vit_ms
        out["streams_decoding"] = decoded
        out["kernels_ms_per_step"] = {k: v["ms"] / v["n"] for k, v in prof.items()}
        out["trellis_steps_per_step"] = arm["trellis"]
        out["acs_per_s"] = arm["trellis"] * 64 / (vit_ms * 1e-3)
        out["frames_per_s"] = S / (out["step_ms"]["median"] * 1e-3)
        ctx.close()
    res["note"] = ("step times: whole decode step of the batch, alternating arms; viterbi_kernel(MSC): serial per-kernel profile in a "
                   "separate run; ACS/s = trellis steps x 64 states / MSC kernel time")
    txt = json.dumps(res, indent=1)
    print(txt)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write(txt + "\n")


if __name__ == "__main__":
    main()
