"""Cost of the device TII analysis at the headline batch: 4096 streams, every one carrying two TII transmitters, the benchmark's
configuration (one 96 kbit/s DAB+ sub-channel, keep_taps off).

  python scripts/tii_measure.py [--batch 4096] [--steps 10] [--reps 4] [--out FILE.json]

Prints one JSON object:
  - step time with dabb_options.decode_tii off and on, in alternating runs of --steps steps, each timed with CUDA events on the
    context's stream (dabb_join_lanes before the closing event);
  - the TII kernels' device time per step from dabb_profile (serial per-kernel timing: null mix, spectra, plan, phase table);
  - the glue's host analyser (welle.io_b200/host/tii.h) on the same kind of spectra: CPU time per frame, times the batch;
  - the card's name and power limit, which belong to every number.
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))

TF, TU, TNULL = 196608, 2048, 2656
RING_FRAMES = 5
BUF_LEN = (RING_FRAMES + 1) * TF + 4096
BITRATE, SUBCH_CU = 96, 72
TII_SETS = [[(4, 17, 23, 0.5), (11, 52, 140, 0.35)], [(1, 3, 7, 0.5), (20, 66, 250, 0.4)], [(7, 40, 60, 0.45), (15, 9, 333, 0.4)],
            [(2, 69, 0, 0.5), (22, 1, 480, 0.35)]]


def ring_with_tii(seed, tii):
    """a seamless 5-frame ring (dabtx.periodic_ring) whose null symbols carry the transmitters `tii`"""
    import dabtx
    tx = dabtx.DabTx(seed=seed, period_sf=4 * RING_FRAMES // 5)
    tx.tii = tii
    sig = np.concatenate([tx.modulate(tx.frame_bits()) for _ in range(2 * RING_FRAMES)])
    return sig[RING_FRAMES * TF:].astype(np.complex64)


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


def host_analyser_ms_per_frame(rings, n_frames=40):
    """welle_b200_tii_run (the glue's analyser) on the rings' spectra (oracle FFT = the reference's), ms per frame"""
    from oracle.bind import Oracle
    orc = Oracle()
    lib = C.CDLL(os.path.join(ROOT, "welle.io_b200", "libwelle_b200_host.so"))
    lib.welle_b200_tii_run.restype = C.c_int
    nspec, pspec = [], []
    for f in range(n_frames):
        r = rings[f % len(rings)]; k = f % (RING_FRAMES - 1)
        null = r[(k + 1) * TF: (k + 1) * TF + TNULL]; prs = r[k * TF + TNULL + 504: k * TF + TNULL + 504 + TU]
        nspec.append(orc.fft(null[TNULL - TU:])); pspec.append(orc.fft(prs))
    nspec, pspec = np.ascontiguousarray(np.stack(nspec)), np.ascontiguousarray(np.stack(pspec))
    out = np.zeros(4 * 9 * n_frames, np.float32)
    best = None
    for _ in range(3):
        t0 = time.perf_counter()
        k = lib.welle_b200_tii_run(nspec.ctypes.data_as(C.c_void_p), pspec.ctypes.data_as(C.c_void_p), n_frames, out.ctypes.data_as(C.c_void_p), 9 * n_frames)
        dt = (time.perf_counter() - t0) * 1e3 / n_frames
        best = dt if best is None else min(best, dt)
    return best, k


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--reps", type=int, default=4)
    ap.add_argument("--snr", type=float, default=20.0)
    ap.add_argument("--out")
    a = ap.parse_args()
    res = {"batch": a.batch, "transmitters_per_stream": 2}
    rings_np = [ring_with_tii(0xB200 + i, TII_SETS[i]) for i in range(len(TII_SETS))]
    hms, hk = host_analyser_ms_per_frame(rings_np)
    res["host_analyser"] = {"ms_per_frame": hms, "measurements": hk, "ms_per_step_at_batch": hms * a.batch,
                            "cpu": "one core of the machine this ran on"}
    import torch
    from conftest import load_pkg
    pkg = load_pkg()
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    res["card"] = card()
    S = a.batch
    rings = torch.from_numpy(np.stack(rings_np).view(np.float32).reshape(len(rings_np), RING_FRAMES * TF, 2)).to(dev)
    sigma = (float((rings[:, 3000:190000] ** 2).sum(-1).mean()) / (10 ** (a.snr / 10)) / 2) ** 0.5
    buf = torch.empty((S, BUF_LEN, 2), dtype=torch.float32, device=dev)
    gen = torch.Generator(device=dev); gen.manual_seed(0x711)
    for s0 in range(0, S, 256):
        n = min(256, S - s0)
        blk = rings[torch.arange(s0, s0 + n, device=dev) % len(rings_np)] + torch.randn((n, RING_FRAMES * TF, 2), device=dev, generator=gen) * sigma
        buf[s0:s0 + n, :RING_FRAMES * TF] = blk
        buf[s0:s0 + n, RING_FRAMES * TF:] = blk[:, :BUF_LEN - RING_FRAMES * TF]
        del blk
    torch.cuda.synchronize()
    ctx = pkg.Context(n_streams=S, disable_coarse=True, n_subch_slots=1, max_subch_cu=SUBCH_CU)
    ctx.select_subchannel(0, SUBCH_CU, BITRATE, eep_profile_a=True, eep_level=3, dabplus=True)
    ext = torch.cuda.ExternalStream(ctx.cuda_stream(), device=dev)
    call = [0]

    def step():
        n = call[0] + 1
        bs = np.full(S, RING_FRAMES * TF * (n // RING_FRAMES), np.int64) if call[0] > 0 else np.zeros(S, np.int64)
        ctx.process_async(buf.data_ptr(), BUF_LEN, bs, BUF_LEN); call[0] += 1

    for _ in range(8):
        step()
    ctx.sync()
    times = {"off": [], "on": []}
    for rep in range(a.reps):
        for mode in ("off", "on"):
            ctx.set_options(disable_coarse=True, decode_tii=mode == "on")
            step(); ctx.sync()                    # one untimed step in the new mode
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(ext)
            for _ in range(a.steps):
                step()
            ctx.join_lanes(); e1.record(ext); torch.cuda.synchronize()
            times[mode].append(e0.elapsed_time(e1) / a.steps)
    res["step_ms"] = {m: {"runs": v, "median": float(np.median(v))} for m, v in times.items()}
    res["step_ms"]["tii_cost_median"] = res["step_ms"]["on"]["median"] - res["step_ms"]["off"]["median"]
    ctx.set_options(disable_coarse=True, decode_tii=True)
    n_meas = 0
    for _ in range(5):
        step(); n_meas += int(ctx.read_tap(9)["count"].sum())
    res["measurements_per_step"] = n_meas / 5
    ctx.profile(True)
    for _ in range(a.steps):
        step()
    ctx.sync()
    prof = ctx.profile_read(); ctx.profile(False)
    tii = {k: v["ms"] / v["n"] for k, v in prof.items() if k in ("null_tap_kernel", "tii_spectra_kernel", "tii_plan_kernel", "tii_phase_kernel")}
    res["tii_kernels_ms_per_step"] = dict(tii, total=sum(tii.values()))
    res["note"] = "step times: decode step of the whole batch with the benchmark's configuration; kernel times: serial per-kernel profile"
    ctx.close()
    txt = json.dumps(res, indent=1)
    print(txt)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write(txt + "\n")


if __name__ == "__main__":
    main()
