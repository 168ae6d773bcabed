"""The weighted soft-decision demap (dabb_options.soft_demap = DABB_DEMAP_WEIGHTED) on the device.

Stage level (dabb_ofdm_demod), in every kernel instance (DABB_FFT_EXACT / FMA; no oscillator, DABB_NCO_EXACT, DABB_NCO_FAST; with and
without r1_out) and with 1, 64 and 1024 frames (25, 5 and 1 CTAs per frame), on clean, noisy, multipath, 150 Hz offset, tone and NaN
frames: the weighted and the reference call give the same r1_out, the reference softbits are the float32 reference demap of that r1,
and the weighted ones pass tests/softref.py's check (strong carriers exactly the reference's, weak ones the restatement).
Pipeline: tap 0 is bit-identical for every ofdm_groups and the tail split; switching the option on and back off decodes like a context
that never set it from the next step on (logical frames once the de-interleaver history has refilled); out-of-range values are refused
and change nothing.  Closed loop: with the same recordings, weighted passes at least as many FIB CRCs as the reference demap at every
point, far more in multipath, and its DAB+ RS-uncorrectable count is no higher."""
import ctypes as C

import numpy as np
import pytest

import dabtx
import ofdmref
import softref
from conftest import load_pkg

pytestmark = pytest.mark.gpu
TF, TNULL, K = 196608, 2656, 1536
KINDS = ("clean", "noisy", "multipath", "offset", "tone", "nan")


@pytest.fixture(scope="module")
def pkg():
    return load_pkg()


@pytest.fixture(scope="module")
def recording():
    """one frame of each kind, TF samples apart; frame k's first useful PRS sample at k TF + TNULL + 305"""
    parts = []
    for k, kind in enumerate(KINDS):
        x = dabtx.DabTx(seed=0x50D0 + k).frames(1, noise_floor=0)
        if kind == "noisy":
            x = dabtx.add_awgn(x, 6.0, seed=k)
        elif kind == "multipath":
            x = dabtx.add_awgn(ofdmref.multipath(x, [(0, 1.0), (37, 0.7 - 0.3j), (211, 0.5j)]), 9.0, seed=k)
        elif kind == "offset":
            x = dabtx.add_awgn(dabtx.freq_shift(x, 150.0), 12.0, seed=k)
        elif kind == "tone":
            p = float(np.mean(np.abs(x) ** 2))
            x = dabtx.add_awgn(x + np.sqrt(100 * p) * np.exp(2j * np.pi * 301000.0 * np.arange(len(x)) / 2048000.0), 8.0, seed=k, signal_power=p)
        elif kind == "nan":
            x = dabtx.add_awgn(ofdmref.multipath(x, [(0, 1.0), (20, 0.95j)]), 9.0, seed=k)
            x[TNULL + 305 + 2048 + 20 * 2552 + 1000] = np.nan            # inside data symbol 21: symbols 21 and 22 are all NaN
        parts.append(np.asarray(x[:TF], np.complex64))
    return np.concatenate(parts)


def stage(ctx, d_iq, n, nco, r1, kinds=KINDS):
    """dabb_ofdm_demod of n frames cycling through the kinds (stride 0)"""
    prs = np.array([(f % len(kinds)) * TF + TNULL + 305 for f in range(n)], np.int64)
    d_ps = ctx.dev(prs)
    d_soft = ctx.dev(n * 75 * 3072)
    d_r1 = ctx.dev(n * 75 * K * 8) if r1 else None
    d_nco = None
    if nco:
        h = np.zeros((n, 2), np.int32)
        h[[f for f in range(n) if KINDS[f % len(KINDS)] == "offset"]] = (12345, 150)
        d_nco = ctx.dev(h)
    ctx._ck(ctx.lib.dabb_ofdm_demod(ctx.h, C.c_void_p(d_iq.ptr), C.c_int64(0), C.c_void_p(d_ps.ptr), n, C.c_void_p(d_nco.ptr) if d_nco else None,
                                    C.c_void_p(d_soft.ptr), C.c_void_p(d_r1.ptr) if d_r1 else None, None))
    ctx.sync()
    soft = d_soft.download(np.int8).reshape(n, 75, 3072)
    out = (soft, d_r1.download(np.complex64).reshape(n, 75, K) if r1 else None)
    for b in (d_ps, d_soft, d_r1, d_nco):
        if b:
            b.free()
    return out


@pytest.mark.parametrize("n", [1, 64, 1024])
@pytest.mark.parametrize("nco_mode", ["none", "exact", "fast"])
@pytest.mark.parametrize("fft_mode", ["exact", "fma"])
def test_stage_every_instance(pkg, recording, fft_mode, nco_mode, n):
    ctx = pkg.Context(n_streams=1, fft_mode=pkg.FFT_EXACT if fft_mode == "exact" else pkg.FFT_FMA,
                      nco_mode=pkg.NCO_FAST if nco_mode == "fast" else pkg.NCO_EXACT)
    d_iq = ctx.dev(recording)
    nco = nco_mode != "none"
    ctx.set_options(soft_demap=pkg.DEMAP_WEIGHTED)
    sw, rw = stage(ctx, d_iq, n, nco, True)
    sw0, _ = stage(ctx, d_iq, n, nco, False)
    ctx.set_options(soft_demap=pkg.DEMAP_REFERENCE)
    sr, rr = stage(ctx, d_iq, n, nco, True)
    d_iq.free(); ctx.close()
    assert np.array_equal(rw.view(np.uint64), rr.view(np.uint64))                 # r1_out does not depend on the mode
    assert np.array_equal(sw, sw0)                                                 # nor do the softbits on r1_out
    m = min(n, len(KINDS))
    for f in range(m, n):                                                          # every frame of a kind decodes alike, whatever CTA it ran in
        assert np.array_equal(sw[f], sw[f % len(KINDS)]), f
    assert np.array_equal(sr[:m].reshape(-1, 3072), softref.soft_reference_f32(rr[:m].reshape(-1, K)))
    weak = softref.check(rr[:m].reshape(-1, K), sw[:m].reshape(-1, 3072))
    assert weak > 0
    if m > KINDS.index("nan"):
        f = KINDS.index("nan")
        assert np.isnan(rr[f, 20:22]).all() and np.array_equal(sw[f, 20:22], sr[f, 20:22])
        assert not np.array_equal(sw[f, 22:], sr[f, 22:])                          # the symbols after them are weighted again


S_PIPE = 2048


def _pipe_soft(pkg, sig, **kw):
    ctx = pkg.Context(n_streams=S_PIPE, keep_taps=True, **kw)
    ctx.set_options(soft_demap=pkg.DEMAP_WEIGHTED)
    d = ctx.dev(sig)
    soft = []
    for _ in range(5):
        out = ctx.process(d, 0, np.zeros(S_PIPE, np.int64), len(sig))
        if out["results"]["status"][0] == pkg.FRAME_DECODED:
            assert (out["results"]["status"] == pkg.FRAME_DECODED).all()
            soft.append(ctx.read_tap(0).reshape(S_PIPE, -1))
    d.free(); ctx.close()
    assert len(soft) >= 2
    return soft


def test_pipeline_every_launch_configuration(pkg):
    sig = dabtx.add_awgn(ofdmref.multipath(dabtx.DabTx(seed=0x50E0).frames(6), [(0, 1.0), (20, 0.95j)]), 8.0, seed=0x50E1)
    want = None
    for kw in ({"ofdm_groups": 1, "ofdm_tail_split": -1}, {"ofdm_groups": 3}, {"ofdm_groups": 5}, {"ofdm_groups": 15}, {"ofdm_groups": 25},
               {"ofdm_groups": 75}, {}, {"ofdm_tail_split": -1}):
        soft = _pipe_soft(pkg, sig, **kw)
        for s in soft:
            assert (s == s[:1]).all(), kw
        if want is None:
            want = soft
        assert len(soft) == len(want) and all(np.array_equal(a, b) for a, b in zip(soft, want)), kw
    # against one stream in the reference mode: never more confident, and weaker on some carriers
    ctx = pkg.Context(n_streams=1, keep_taps=True)
    d = ctx.dev(sig)
    ref = []
    for _ in range(5):
        if ctx.process(d, 0, np.zeros(1, np.int64), len(sig))["results"]["status"][0] == pkg.FRAME_DECODED:
            ref.append(ctx.read_tap(0).reshape(-1))
    d.free(); ctx.close()
    assert len(ref) == len(want)
    for w, r in zip(want, ref):
        w, r = w[0].astype(int), r.astype(int)
        assert np.all(np.abs(w) <= np.abs(r)) and (np.abs(w) < np.abs(r)).mean() > 0.1


BITRATE = 96


def _decode(pkg, sig, S, steps, switch=None, **kw):
    ctx = pkg.Context(n_streams=S, **kw)
    ctx.select_subchannel(0, dabtx.eep_cu(BITRATE), BITRATE, eep_profile_a=True, eep_level=3, dabplus=True)
    d = ctx.dev(sig)
    outs = []
    for k in range(steps):
        if switch:
            switch(ctx, k)
        outs.append(ctx.process(d, sig.shape[1] if sig.ndim == 2 else 0, np.zeros(S, np.int64), sig.shape[-1], msc_stride=3 * BITRATE,
                                sf_stride=15 * BITRATE))
    d.free(); ctx.close()
    return outs


def test_switching_and_refusals(pkg):
    sig = dabtx.add_awgn(ofdmref.multipath(dabtx.DabTx(seed=0x50F0).frames(14), [(0, 1.0), (37, 0.7 - 0.3j), (211, 0.5j)]), 6.0, seed=0x50F1)
    S, STEPS, ON, OFF = 4, 13, 3, 6

    def switch(ctx, k):
        if k == 1:
            for bad in (2, -1, 0x100):
                with pytest.raises(pkg.DabbError):
                    ctx.set_options(soft_demap=bad, decode_tii=True, count_bit_errors=True)
            with pytest.raises(pkg.DabbError):
                ctx.read_tap(9)                    # the refused call allocated nothing
        if k == ON:
            ctx.set_options(soft_demap=pkg.DEMAP_WEIGHTED)
        if k == OFF:
            ctx.set_options(soft_demap=pkg.DEMAP_REFERENCE)

    a = _decode(pkg, sig, S, STEPS)
    b = _decode(pkg, sig, S, STEPS, switch)
    differed = False
    for k in range(STEPS):
        ra, rb = a[k]["results"], b[k]["results"]
        assert np.array_equal(ra["status"], rb["status"]) and np.array_equal(ra["next_pos"], rb["next_pos"]), k
        if ON <= k < OFF:
            differed |= not np.array_equal(a[k]["fibs"], b[k]["fibs"]) or not np.array_equal(ra["fib_crc_mask"], rb["fib_crc_mask"])
            continue
        assert np.array_equal(a[k]["fibs"], b[k]["fibs"]) and np.array_equal(ra["fib_crc_mask"], rb["fib_crc_mask"]), k
        if k < ON or k >= OFF + 4:                 # 16 CIFs of de-interleaver history = 4 frames
            assert np.array_equal(a[k]["msc"], b[k]["msc"]) and np.array_equal(ra["n_logical"], rb["n_logical"]), k
    assert differed
    assert sum(int((a[k]["results"]["status"] == pkg.FRAME_DECODED).sum()) for k in range(STEPS)) >= S * (STEPS - 4)


# ---- closed loop: FIB CRC passes and RS-uncorrectable superframes, same recordings in both modes
# the tone is checked at stage level (test_tone_stage_level): with a tone 20 dB above the ensemble the null-symbol search acquires no
# stream in either mode
POINTS = [("awgn", 3.0), ("awgn", 5.0), ("2path", 3.0), ("2path", 5.0), ("3path", 3.0), ("3path", 5.0)]
CHANNELS = {"2path": [(0, 1.0), (20, 0.95j)], "3path": [(0, 1.0), (37, 0.7 - 0.3j), (211, 0.5j)]}
N_TX, N_NOISE, FRAMES, STEPS_CL = 4, 4, 8, 8


def received(clean, name, snr_db, seed):
    """the SNR is that of the received ensemble (after the echoes, without the tone)"""
    x = ofdmref.multipath(clean, CHANNELS[name]) if name in CHANNELS else clean
    p = float(np.mean(np.abs(x) ** 2))
    if name == "tone":
        x = x + np.sqrt(100 * p) * np.exp(2j * np.pi * 301000.0 * np.arange(len(x)) / 2048000.0)
    return dabtx.add_awgn(x, snr_db, seed=seed, signal_power=p)


def closed_loop(pkg, sig, weighted):
    S = len(sig)

    def switch(ctx, k):
        if k == 0 and weighted:
            ctx.set_options(soft_demap=pkg.DEMAP_WEIGHTED)

    fib = fib_n = rs_bad = rs_n = 0
    for out in _decode(pkg, sig, S, STEPS_CL, switch):
        r = out["results"]
        dec = r["status"] == pkg.FRAME_DECODED
        fib += sum(bin(int(m)).count("1") for m in r["fib_crc_mask"][dec]); fib_n += 12 * int(dec.sum())
        for s in range(S):
            n = int(r["n_rs_events"][s][0])
            rs_n += n
            rs_bad += bin(int(r["rs_uncorr_mask"][s][0]) & ((1 << n) - 1)).count("1")
    return fib, fib_n, rs_bad, rs_n


def test_closed_loop_gain(pkg):
    clean = [dabtx.DabTx(seed=0x5100 + t).frames(FRAMES) for t in range(N_TX)]
    res = {}
    for i, (name, snr) in enumerate(POINTS):
        sig = np.stack([received(clean[s % N_TX], name, snr, 0x5200 + 16 * i + s) for s in range(N_TX * N_NOISE)])
        res[(name, snr)] = (closed_loop(pkg, sig, False), closed_loop(pkg, sig, True))
    print({f"{n}@{s}dB": v for (n, s), v in res.items()})
    for pt, ((fr, nr, rr, _), (fw, nw, rw, _)) in res.items():       # (FIBs passed, FIBs, RS uncorrectable, RS events)
        assert nr == nw and nr > 0, pt
        assert fw >= fr and rw <= rr, (pt, fr, fw, rr, rw)
    for pt, limit in ((("2path", 5.0), 0.6), (("3path", 5.0), 0.75)):
        (fr, n, _, _), (fw, _, _, _) = res[pt]
        assert fw >= 0.95 * n and fr <= limit * n, (pt, fr, fw, n)


def test_tone_stage_level(pkg, oracle):
    """a CW tone at +301 kHz 20 dB above the ensemble, 4 dB SNR: the FIC of the device's weighted softbits decodes as well as the
    reference demap's (the tone barely moves the geometric mean)"""
    n = 6
    x = np.concatenate([np.asarray(received(dabtx.DabTx(seed=0x5400 + k).frames(1, noise_floor=0), "tone", 4.0, 0x5410 + k)[:TF], np.complex64)
                        for k in range(n)])
    ctx = pkg.Context(n_streams=1)
    d = ctx.dev(x)
    passed = {}
    for mode in (pkg.DEMAP_REFERENCE, pkg.DEMAP_WEIGHTED):
        ctx.set_options(soft_demap=mode)
        soft, _ = stage(ctx, d, n, False, False, kinds=range(n))
        passed[mode] = sum(int(oracle.fic_decode(soft[f, :3].reshape(-1))[1].sum()) for f in range(n))
    d.free(); ctx.close()
    assert passed[pkg.DEMAP_WEIGHTED] >= passed[pkg.DEMAP_REFERENCE] and passed[pkg.DEMAP_WEIGHTED] >= 12 * n - 2, passed


def test_batch_decode_soft_weighted(tmp_path):
    """batch_decode --soft weighted on a two-path recording, end to end on the library: more FIBs pass than with the reference demap"""
    import os
    import subprocess
    from conftest import ROOT
    exe = os.path.join(ROOT, "welle.io_b200", "batch_decode")
    sig = received(dabtx.DabTx(seed=0x5300).frames(12), "2path", 5.0, 0x5301)
    f = tmp_path / "echo.iq"
    sig.tofile(f)
    passed = {}
    for mode in ("reference", "weighted"):
        out = tmp_path / mode
        out.mkdir()
        r = subprocess.run([exe, "--soft", mode, "--out", str(out), str(f)], capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr
        rec = np.frombuffer((out / "echo.iq.fic").read_bytes(), np.uint8).reshape(-1, 33)
        assert len(rec) >= 12 * 8 and (out / "echo.iq.msc").exists()
        passed[mode] = int((rec[:, 0] != 0).sum())
    assert passed["weighted"] > passed["reference"] and passed["weighted"] >= 0.9 * len(rec), passed
