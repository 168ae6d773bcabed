"""Transmitter identification analysed on the device for every stream of a batch (dabb_options.decode_tii, tap 9) against the glue's host
analyser (welle.io_b200/host/tii.h) fed the same spectra (tap 4); the same analysis without keep_taps; a context that had TII on and
switched it off launches what a context that never had it launches; dabb_stream_reset; batch_decode --tii against glue_test."""
import os
import subprocess
from collections import Counter

import numpy as np
import pytest

import dabtx
import tiiref
from conftest import ROOT

pytestmark = pytest.mark.gpu

TF, TNULL = tiiref.TF, tiiref.TNULL


def with_tii(base, tx_set, snr_db, seed):
    """base (a dabtx recording without TII) with the null symbol of every frame replaced by the one of tx_set, plus noise"""
    sig = base.copy()
    if tx_set:
        tx = dabtx.DabTx(seed=0)
        tx.amp = 0.1
        tx.tii = list(tx_set)
        null = tx.tii_null().astype(np.complex64)
        for f in range(len(sig) // TF):
            sig[f * TF: f * TF + TNULL] = null
    return dabtx.add_awgn(sig, snr_db, seed=seed) if snr_db is not None else sig


def tii_sets(rng, n):
    out = []
    for s in range(n):
        k = s % 4
        combs = rng.choice(24, k, replace=False)
        out.append([(int(c), int(rng.integers(0, 70)), int(rng.integers(-4, 400)), float(rng.uniform(0.3, 0.6))) for c in combs])
    return out


def records(tap9, s):
    r = tap9[s]
    return [(int(m["comb"]), int(m["pattern"]), int(m["delay_samples"]), float(m["error"])) for m in r["m"][:int(r["count"])]]


def test_device_matches_host_analyser(pkg):
    """64 streams (0-3 transmitters, 15-30 dB, one stream of noise only), 16 steps, keep_taps=1: every step's tap 9 = the host analyser
    fed that stream's tap-4 spectra of its decoded frames so far; error within 1 per accumulated frame"""
    S, steps = 64, 16
    rng = np.random.default_rng(64)
    base = dabtx.DabTx(seed=0x64).frames(steps + 1)
    sets = tii_sets(rng, S)
    snrs = rng.uniform(15, 30, S)
    buf = np.stack([with_tii(base, sets[s], float(snrs[s]), 100 + s) for s in range(S)])
    rng_n = np.random.default_rng(1)
    buf[S - 1] = ((rng_n.standard_normal(buf.shape[1]) + 1j * rng_n.standard_normal(buf.shape[1])) * 0.05).astype(np.complex64)
    ctx = pkg.Context(n_streams=S, keep_taps=True)
    ctx.set_options(disable_coarse=True, decode_tii=True)
    d = ctx.dev(buf)
    spectra = [[] for _ in range(S)]          # per stream: (step, tap-4 spectra) of its decoded frames
    dev = {}                                  # (stream, step) -> tap-9 measurements
    for step in range(steps):
        r = ctx.process(d, buf.shape[1], np.zeros(S, np.int64), buf.shape[1])["results"]
        t4, t9 = ctx.read_tap(4), ctx.read_tap(9)
        for s in range(S):
            if r["status"][s] == pkg.FRAME_DECODED:
                spectra[s].append((step, t4[s].copy()))
            else:
                assert t9[s]["count"] == 0 and t9[s]["skipped"] == 0
            if t9[s]["count"]:
                dev[(s, step)] = records(t9, s)
    host = tiiref.host_lib()
    want = {}
    for s in range(S):
        if not spectra[s]:
            continue
        steps_s = [st for st, _ in spectra[s]]
        sp = np.stack([x for _, x in spectra[s]])
        for f, c, p, dl, e in tiiref.host_run_framed(host, sp[:, 1], sp[:, 0]):
            want.setdefault((s, steps_s[f]), []).append((c, p, dl, e))
    want = {k: sorted(v) for k, v in want.items()}
    ctx.close()
    assert sorted(want) == sorted(dev), (sorted(set(want) ^ set(dev)))
    n = ndiff = 0
    for k in want:
        assert [x[:3] for x in want[k]] == [x[:3] for x in dev[k]], (k, want[k], dev[k])
        for a, b in zip(want[k], dev[k]):
            n += 1
            assert abs(a[3] - b[3]) <= 5, (k, a, b)
            ndiff += a[3] != b[3]
    found = sum(1 for s in range(S) for c, p, dl, _ in sets[s] if any((c, p, dl) == x[:3] for (t, _), v in dev.items() if t == s for x in v))
    print(f"{S} streams x {steps} steps: {n} measurements equal, {ndiff} error values differ; {found} of {sum(map(len, sets))} transmitters found with their delay")
    assert n >= 40
    assert not any(k[0] == S - 1 for k in dev)         # noise: nothing decoded, nothing reported


def overlapping_batch(S, stride, frames, seed):
    """one recording with two transmitters; stream s reads it from sample s * stride on (every stream meets other frames and noise)"""
    rec_frames = (S * stride) // TF + frames + 2
    base = dabtx.DabTx(seed=seed).frames(rec_frames)
    return with_tii(base, [(4, 17, 23, 0.5), (11, 52, 140, 0.35)], 22.0, seed)


def run_tap9(pkg, sig, S, stride, buf_len, steps, keep_taps):
    ctx = pkg.Context(n_streams=S, keep_taps=keep_taps)
    ctx.set_options(disable_coarse=True, decode_tii=True)
    d = ctx.dev(sig)
    out = []
    for _ in range(steps):
        ctx.process(d, stride, np.zeros(S, np.int64), buf_len, want=("results",))
        out.append(ctx.read_tap(9))
    ctx.close()
    return np.stack(out)


def test_without_keep_taps(pkg):
    """1024 streams, keep_taps=0 (the null symbol goes to an internal buffer, no tap 3 / 4): tap 9 equals the keep_taps=1 run"""
    S, stride, frames = 1024, 7919, 9
    sig = overlapping_batch(S, stride, frames, seed=0x1024)
    buf_len = frames * TF
    a = run_tap9(pkg, sig, S, stride, buf_len, frames - 1, keep_taps=False)
    b = run_tap9(pkg, sig, S, stride, buf_len, frames - 1, keep_taps=True)
    assert a.tobytes() == b.tobytes()
    n = int(a["count"].sum())
    assert n >= S, n                                  # every stream reports at least its first measurements
    rng = np.random.default_rng(3)
    for s in rng.choice(S, 16, replace=False):
        assert any((4, 17) == (int(m["comb"]), int(m["pattern"])) for st in range(frames - 1) for m in a[st, s]["m"][:a[st, s]["count"]])
    print(f"keep_taps=0 vs 1 at {S} streams: {n} measurements, identical records")


def test_decode_tii_off_launches_like_never_on(pkg):
    """a context that ran TII and switched it off launches the same kernels per step as one that never had it (count and names), and
    taps 5-8 of every step are byte-identical between the two"""
    S, steps, on_steps = 8, 10, 4
    base = dabtx.DabTx(seed=0x0FF).frames(steps + 1)
    buf = np.stack([with_tii(base, [(4, 17, 23, 0.5)], 25.0, s) for s in range(S)])
    ctxs = [pkg.Context(n_streams=S), pkg.Context(n_streams=S)]
    ds = []
    for c in ctxs:
        c.select_subchannel(0, 72, 96, eep_profile_a=True, eep_level=3)
        ds.append(c.dev(buf))
    ctxs[1].set_options(disable_coarse=True, decode_tii=True)
    per_step = [[], []]
    for step in range(steps):
        if step == on_steps:
            ctxs[1].set_options(disable_coarse=True, decode_tii=False)
            for c in ctxs:
                c.profile(True)
        taps = []
        for i, c in enumerate(ctxs):
            n0 = c.kernel_launches()
            c.process_async(ds[i].ptr, buf.shape[1], np.zeros(S, np.int64), buf.shape[1])
            c.sync()
            per_step[i].append(c.kernel_launches() - n0)
            taps.append([c.read_tap(5).tobytes(), c.read_tap(6).tobytes(), c.read_tap(7, stride=288).tobytes(), c.read_tap(8, stride=1440).tobytes()])
        assert taps[0] == taps[1], step
        if step >= on_steps:
            t9 = ctxs[1].read_tap(9)
            assert int(t9["count"].sum()) == 0
    names = [sorted(c.profile_read()) for c in ctxs]
    assert per_step[0][on_steps:] == per_step[1][on_steps:]
    assert names[0] == names[1] and not any("tii" in n for n in names[1])
    assert per_step[1][:on_steps] != per_step[0][:on_steps]       # while on, the TII kernels did run
    for c in ctxs:
        c.close()
    print(f"launches per step never on {per_step[0]}, on then off {per_step[1]}")


def test_reset_restarts_the_accumulation(pkg):
    """after dabb_stream_reset a stream's first measurement comes with its fifth newly analysed frame; the other stream is untouched"""
    S, steps = 2, 22
    base = dabtx.DabTx(seed=0x5E7).frames(steps + 2)
    buf = np.stack([with_tii(base, [(4, 17, 23, 0.5)], 25.0, 7 + s) for s in range(S)])
    ctx = pkg.Context(n_streams=S, keep_taps=False)
    ctx.set_options(disable_coarse=True, decode_tii=True)
    d = ctx.dev(buf)
    analysed = [0, 0]; reports = [[], []]; reset_done = False
    for step in range(steps):
        r = ctx.process(d, buf.shape[1], np.zeros(S, np.int64), buf.shape[1])["results"]
        t9 = ctx.read_tap(9)
        for s in range(S):
            if r["status"][s] == pkg.FRAME_DECODED and not t9[s]["skipped"]:
                analysed[s] += 1
            if t9[s]["count"]:
                reports[s].append(analysed[s])
        if not reset_done and analysed[0] == 7:      # two analyses into the second accumulation
            ctx.reset(first=0, count=1, pos=int(r["next_pos"][0]))
            analysed[0] = 0; reports[0].append("reset"); reset_done = True
    ctx.close()
    assert reset_done
    i = reports[0].index("reset")
    assert reports[0][:i] == [5] and reports[0][i + 1] == 5, reports[0]
    assert reports[1][:3] == [5, 10, 15], reports[1]


def test_batch_decode_tii_matches_glue(tmp_path):
    """batch_decode --tii on three recordings: each DIR/<name>.tii holds glue_test's measurements of that file (comb, pattern, delay as
    multisets; error within 1 per accumulated frame)"""
    exe_b = os.path.join(ROOT, "welle.io_b200", "batch_decode")
    exe_g = os.path.join(ROOT, "welle.io_b200", "glue_test")
    if not (os.path.exists(exe_b) and os.path.exists(exe_g)):
        subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "welle.io_b200", "host")])
    specs = [dict(seed=0x11, n=14, pad=0, tii=[(4, 17, 23, 0.5), (11, 52, 140, 0.35)]),
             dict(seed=0x22, n=12, pad=5000, tii=[(7, 3, 60, 0.5)]),
             dict(seed=0x33, n=16, pad=777, tii=[(1, 40, 5, 0.45), (20, 66, 250, 0.4)])]
    files = []
    for k, sp in enumerate(specs):
        sig = with_tii(dabtx.DabTx(seed=sp["seed"]).frames(sp["n"]), sp["tii"], 25.0, sp["seed"])
        iq = np.concatenate([np.zeros(sp["pad"], np.complex64), sig])
        f = tmp_path / f"rec{k}.iq"
        iq.tofile(f); files.append(f)
    outdir = tmp_path / "out"; outdir.mkdir()
    run = subprocess.run([exe_b, "--tii", "--out", str(outdir)] + [str(f) for f in files], capture_output=True, text=True, timeout=600)
    assert run.returncode == 0, run.stderr
    total = 0
    for k, f in enumerate(files):
        g = subprocess.run([exe_g, str(f), str(tmp_path / f"g{k}"), "12", "1", "1"], capture_output=True, text=True, timeout=600)
        assert g.returncode == 0, g.stderr
        parse = lambda p: [tuple(float(x) for x in ln.split()) for ln in open(p).read().splitlines()]
        got, want = parse(outdir / f"rec{k}.iq.tii"), parse(tmp_path / f"g{k}.tii")
        assert Counter(x[:3] for x in got) == Counter(x[:3] for x in want), (k, got, want)
        errs = {}
        for x in want:
            errs.setdefault(x[:3], []).append(x[3])
        for x in got:
            assert min(abs(x[3] - e) for e in errs[x[:3]]) <= 5, (k, x, errs[x[:3]])
        assert len(got) >= 2, (k, got)
        total += len(got)
    print(f"batch_decode --tii: {total} measurements equal to glue_test's")
