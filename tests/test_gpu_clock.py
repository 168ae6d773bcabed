"""Sample-clock tracking (dabb_options.sample_clock = DABB_CLOCK_TRACK) on the device.

Stage level (dabb_ofdm_demod_ex), in every kernel instance (DABB_FFT_EXACT / FMA; no oscillator, DABB_NCO_EXACT, DABB_NCO_FAST; with
and without r1_out; reference and weighted demap) with 1, 64 and 1024 frames, on clean, noisy, multipath and offset frames with per-frame
ppm including 0 and both signs: ppm 0 gives dabb_ofdm_demod's bits, r1_out is the ppm-0 r1_out times the float64 phasor, the softbits
are the demap of that r1_out, and every frame of a kind decodes alike whatever CTA ran it.
Pipeline, on recordings resampled by +-50 and +-120 ppm (tests/clockref.py): tap 11 equals the numpy estimator run over the step's own
result records bit for bit, through OFF steps, a reset, a sync loss and refused options; tap 0 is the same for every launch
configuration and with keep_taps; a TRACK context keeps the timing of its OFF twin and its constellation is the twin's times the phasor
of the applied value; dabb_submit / dabb_collect give dabb_process's records.  Closed loop over 40 frames: the estimate converges to the
injected error, the clean 0 ppm recording decodes bit-identically to OFF, and at +-120 ppm and 10 dB the channel BER drops to at
most half of OFF's."""
import ctypes as C

import numpy as np
import pytest

import clockref
import dabtx
import ofdmref
import softref
from conftest import load_pkg

pytestmark = pytest.mark.gpu
TF, TNULL, K = 196608, 2656, 1536
KINDS = ("clean", "noisy", "multipath", "offset")
PPMS = (0.0, 55.5, -120.25)          # per frame, cycling: frame f has kind f % 4 and ppm f % 3


@pytest.fixture(scope="module")
def pkg():
    return load_pkg()


@pytest.fixture(scope="module")
def recording():
    """one frame of each kind, TF samples apart; frame k's first useful PRS sample at k TF + TNULL + 305"""
    parts = []
    for k, kind in enumerate(KINDS):
        x = dabtx.DabTx(seed=0xC1D0 + k).frames(1, noise_floor=0)
        if kind == "noisy":
            x = dabtx.add_awgn(x, 6.0, seed=k)
        elif kind == "multipath":
            x = dabtx.add_awgn(ofdmref.multipath(x, [(0, 1.0), (37, 0.7 - 0.3j), (211, 0.5j)]), 9.0, seed=k)
        elif kind == "offset":
            x = dabtx.add_awgn(dabtx.freq_shift(x, 150.0), 12.0, seed=k)
        parts.append(np.asarray(x[:TF], np.complex64))
    return np.concatenate(parts)


def stage(ctx, d_iq, n, nco, r1, ppm):
    """dabb_ofdm_demod_ex (ppm: None -> dabb_ofdm_demod) of n frames cycling through the kinds (stride 0)"""
    prs = np.array([(f % len(KINDS)) * TF + TNULL + 305 for f in range(n)], np.int64)
    d_ps = ctx.dev(prs)
    d_soft = ctx.dev(n * 75 * 3072)
    d_r1 = ctx.dev(n * 75 * K * 8) if r1 else None
    d_nco = d_clk = None
    if nco:
        h = np.zeros((n, 2), np.int32)
        h[[f for f in range(n) if KINDS[f % len(KINDS)] == "offset"]] = (12345, 150)
        d_nco = ctx.dev(h)
    args = (ctx.h, C.c_void_p(d_iq.ptr), C.c_int64(0), C.c_void_p(d_ps.ptr), n, C.c_void_p(d_nco.ptr) if d_nco else None)
    tail = (C.c_void_p(d_soft.ptr), C.c_void_p(d_r1.ptr) if d_r1 else None, None)
    if ppm is None:
        ctx._ck(ctx.lib.dabb_ofdm_demod(*args, *tail))
    else:
        d_clk = ctx.dev(np.ascontiguousarray(ppm, np.float32))
        ctx._ck(ctx.lib.dabb_ofdm_demod_ex(*args, C.c_void_p(d_clk.ptr), *tail))
    ctx.sync()
    soft = d_soft.download(np.int8).reshape(n, 75, 3072)
    out = (soft, d_r1.download(np.complex64).reshape(n, 75, K) if r1 else None)
    for b in (d_ps, d_soft, d_r1, d_nco, d_clk):
        if b:
            b.free()
    return out


def frame_ppm(n):
    return np.array([PPMS[f % len(PPMS)] for f in range(n)], np.float32)


@pytest.mark.parametrize("demap", ["reference", "weighted"])
@pytest.mark.parametrize("n", [1, 64, 1024])
@pytest.mark.parametrize("nco_mode", ["none", "exact", "fast"])
@pytest.mark.parametrize("fft_mode", ["exact", "fma"])
def test_stage_every_instance(pkg, recording, fft_mode, nco_mode, n, demap):
    ctx = pkg.Context(n_streams=1, fft_mode=pkg.FFT_EXACT if fft_mode == "exact" else pkg.FFT_FMA,
                      nco_mode=pkg.NCO_FAST if nco_mode == "fast" else pkg.NCO_EXACT)
    ctx.set_options(soft_demap=pkg.DEMAP_WEIGHTED if demap == "weighted" else pkg.DEMAP_REFERENCE)
    d_iq = ctx.dev(recording)
    nco = nco_mode != "none"
    ppm = frame_ppm(n)
    s_null, r_null = stage(ctx, d_iq, n, nco, True, None)
    s_zero, r_zero = stage(ctx, d_iq, n, nco, True, np.zeros(n, np.float32))
    s_clk, r_clk = stage(ctx, d_iq, n, nco, True, ppm)
    s_clk0, _ = stage(ctx, d_iq, n, nco, False, ppm)
    d_iq.free(); ctx.close()
    assert np.array_equal(s_null, s_zero) and np.array_equal(r_null.view(np.uint64), r_zero.view(np.uint64))
    assert np.array_equal(s_clk, s_clk0)                                           # the softbits do not depend on r1_out
    m = min(n, 12)                                                                 # every (kind, ppm) pair once
    for f in range(m):
        want = clockref.derotate(r_null[f], ppm[f])
        err = np.abs(r_clk[f].astype(np.complex128) - want)
        assert np.all(err <= 1e-5 * np.abs(want) + 1e-30), (f, float(np.max(err / (np.abs(want) + 1e-30))))
        if ppm[f] == 0:
            assert np.array_equal(s_clk[f], s_null[f]) and np.array_equal(r_clk[f].view(np.uint64), r_null[f].view(np.uint64))
    if demap == "reference":
        assert np.array_equal(s_clk[:m].reshape(-1, 3072), softref.soft_reference_f32(r_clk[:m].reshape(-1, K)))
    else:
        softref.check(r_clk[:m].reshape(-1, K), s_clk[:m].reshape(-1, 3072))
    for f in range(m, n):                                                          # whatever CTA decoded it
        assert np.array_equal(s_clk[f], s_clk[f % 12]), f


# ---- pipeline on resampled recordings
PIPE_PPM = (50.0, -50.0, 120.0, -120.0)


@pytest.fixture(scope="module")
def resampled():
    """16 frames of one transmitter, resampled by each of PIPE_PPM at 14 dB; rows padded with noise to a common length"""
    clean = dabtx.DabTx(seed=0xC1E0).frames(16)
    rows, eff = [], []
    for i, p in enumerate(PIPE_PPM):
        y, e = clockref.resample_clock(clean, p)
        rows.append(dabtx.add_awgn(y, 14.0, seed=0xC1E1 + i)); eff.append(e)
    n = max(len(r) for r in rows)
    buf = np.full((len(rows), n), 1e-6, np.complex64)
    for i, r in enumerate(rows):
        buf[i, :len(r)] = r
    return buf, eff


def test_tap11_follows_the_estimator(pkg, resampled):
    """every step's tap 11 equals clockref over the step's own records: TRACK, a refused option, OFF steps, a reset, a sync loss"""
    buf, _ = resampled
    buf = buf.copy()
    gap0 = 9 * TF
    buf[1, gap0:gap0 + 2 * TF] = 0                    # stream 1 loses sync for two frames
    S, n = buf.shape
    ctx = pkg.Context(n_streams=S)
    with pytest.raises(pkg.DabbError):
        ctx.read_tap(11)
    for bad in (2, -1, 0x100):
        with pytest.raises(pkg.DabbError):
            ctx.set_options(sample_clock=bad)
    with pytest.raises(pkg.DabbError):
        ctx.read_tap(11)                             # the refused calls allocated nothing
    d = ctx.dev(buf)
    est = clockref.Estimator(S)
    modes = {k: pkg.CLOCK_TRACK for k in range(18)}
    modes.update({10: pkg.CLOCK_OFF, 11: pkg.CLOCK_OFF})
    lost, n_at_loss, status1 = False, 0, []
    for k in range(18):
        if k == 4:
            with pytest.raises(pkg.DabbError):
                ctx.set_options(sample_clock=3)      # refused: stays TRACK
        elif modes[k] != modes.get(k - 1):
            ctx.set_options(sample_clock=modes[k])
        if k == 13:
            ctx.reset(3, 1, 0)
            est.reset(3, 1)
        r = ctx.process(d, n, np.zeros(S, np.int64), n)["results"]
        got = ctx.read_tap(11)
        want = est.step(modes[k], r["status"], r["start_index"])
        assert got.tobytes() == want.tobytes(), (k, got, want, r["status"], r["start_index"])
        if modes[k] == pkg.CLOCK_OFF:
            assert not got.tobytes().strip(b"\0")
        status1.append(int(r["status"][1]))
        if r["status"][1] in (pkg.FRAME_NO_SYNC, pkg.FRAME_ACQUIRING) and k > 3 and not lost:
            lost, n_at_loss = True, int(got["frames"][1])
    counted_after = int(got["frames"][1])
    d.free(); ctx.close()
    assert lost and n_at_loss > 0 and counted_after >= n_at_loss, (status1, n_at_loss, counted_after)    # the sync loss kept the count
    assert est.n[3] < est.n[2]                                # the reset started stream 3 over


def _pipe_tap0(pkg, sig, steps, **kw):
    S = 2048
    ctx = pkg.Context(n_streams=S, **kw)
    ctx.set_options(sample_clock=pkg.CLOCK_TRACK)
    d = ctx.dev(sig)
    for _ in range(steps):
        r = ctx.process(d, 0, np.zeros(S, np.int64), len(sig))["results"]
    clk = ctx.read_tap(11)
    soft = ctx.read_tap(0).reshape(S, -1)
    d.free(); ctx.close()
    assert (r["status"] == pkg.FRAME_DECODED).all() and (clk["applied_ppm"] != 0).all()
    return soft


def test_tap0_every_launch_configuration(pkg, resampled):
    buf, _ = resampled
    sig = np.ascontiguousarray(buf[2])                      # +120 ppm
    want = None
    for kw in ({"ofdm_groups": 1, "ofdm_tail_split": -1}, {"ofdm_groups": 5}, {"ofdm_groups": 25}, {}, {"keep_taps": True}):
        soft = _pipe_tap0(pkg, sig, 14, **kw)
        assert (soft == soft[:1]).all(), kw
        if want is None:
            want = soft[0]
        assert np.array_equal(soft[0], want), kw


def test_twin_timing_and_constellation(pkg, resampled):
    buf, _ = resampled
    S, n = buf.shape
    ctx = {m: pkg.Context(n_streams=S, keep_taps=True) for m in (pkg.CLOCK_OFF, pkg.CLOCK_TRACK)}
    ctx[pkg.CLOCK_TRACK].set_options(sample_clock=pkg.CLOCK_TRACK)
    d = {m: c.dev(buf) for m, c in ctx.items()}
    applied_seen = 0
    for k in range(14):
        r = {m: c.process(d[m], n, np.zeros(S, np.int64), n)["results"] for m, c in ctx.items()}
        for f in ("status", "start_index", "fine_corr", "coarse_corr", "next_pos"):
            assert np.array_equal(r[0][f], r[1][f]), (k, f)
        clk = ctx[pkg.CLOCK_TRACK].read_tap(11)
        t_off, t_on = ctx[pkg.CLOCK_OFF].read_tap(2), ctx[pkg.CLOCK_TRACK].read_tap(2)
        for s in range(S):
            if r[0]["status"][s] != pkg.FRAME_DECODED:
                continue
            want = t_off[s].astype(np.complex128) * clockref.phasor(clockref.CARRIER[::96], clk["applied_ppm"][s])
            assert np.all(np.abs(t_on[s] - want) <= 1e-5 * np.abs(want) + 1e-30), (k, s)
            applied_seen += int(clk["applied_ppm"][s] != 0)
    for m in ctx:
        d[m].free(); ctx[m].close()
    assert applied_seen >= S * 3


def test_submit_collect_matches_process(pkg, resampled):
    buf, _ = resampled
    S, n = buf.shape
    recs = {}
    for how in ("process", "submit"):
        ctx = pkg.Context(n_streams=S)
        ctx.set_options(sample_clock=pkg.CLOCK_TRACK)
        d = ctx.dev(buf) if how == "process" else None
        recs[how] = []
        for k in range(12):
            if how == "process":
                ctx.process(d, n, np.zeros(S, np.int64), n)
            else:
                ctx.submit(buf, n, np.zeros(S, np.int64), n)
                ctx.collect()
            recs[how].append(ctx.read_tap(11).tobytes())
        if d:
            d.free()
        ctx.close()
    assert recs["process"] == recs["submit"]


# ---- closed loop: 40 frames per stream
EPS = (-120.0, -50.0, 0.0, 50.0, 120.0)
SEEDS = 3
BITRATE = 96


def closed_loop_inputs(frames=42):
    """rows: (eps, condition, seed); condition clean, 10 dB AWGN, or multipath (three paths, 14 dB, eps +-50 only)"""
    clean = [dabtx.DabTx(seed=0xC200 + t).frames(frames) for t in range(SEEDS)]
    meta = [(e, c, t) for e in EPS for t in range(SEEDS) for c in (("clean", "10dB", "multipath") if abs(e) == 50.0 else ("clean", "10dB"))]
    buf = np.full((len(meta), int(round(frames * TF * (1 + max(EPS) * 1e-6)))), 1e-6, np.complex64)
    out = []
    for i, (e, c, t) in enumerate(meta):
        y, eff = clockref.resample_clock(clean[t], e)
        if c == "10dB":
            y = dabtx.add_awgn(y, 10.0, seed=0xC300 + 7 * t + int(e))
        elif c == "multipath":
            y = dabtx.add_awgn(ofdmref.multipath(y, [(0, 1.0), (37, 0.7 - 0.3j), (211, 0.5j)]), 14.0, seed=0xC400 + t)
        buf[i, :len(y)] = y
        out.append((e, eff, c, t))
    return buf, out


def run_loop(pkg, buf, mode, steps=42):
    S, n = buf.shape
    ctx = pkg.Context(n_streams=S)
    ctx.select_subchannel(0, dabtx.eep_cu(BITRATE), BITRATE, eep_profile_a=True, eep_level=3, dabplus=True)
    ctx.set_options(count_bit_errors=True, sample_clock=mode)
    d = ctx.dev(buf)
    outs = []
    for _ in range(steps):
        o = ctx.process(d, n, np.zeros(S, np.int64), n, msc_stride=3 * BITRATE, sf_stride=15 * BITRATE)
        o["ber"] = ctx.read_tap(10)
        if mode == pkg.CLOCK_TRACK:
            o["clk"] = ctx.read_tap(11)
        outs.append(o)
    d.free(); ctx.close()
    return outs


def test_closed_loop(pkg):
    buf, meta = closed_loop_inputs()
    off = run_loop(pkg, buf, pkg.CLOCK_OFF)
    on = run_loop(pkg, buf, pkg.CLOCK_TRACK)
    S = len(meta)
    conv = np.zeros((len(on), S), bool)                        # steps whose frame was decoded after 32 counted frames
    for k, o in enumerate(on):
        conv[k] = (o["results"]["status"] == pkg.FRAME_DECODED) & (o["clk"]["frames"] >= 32)
    stats = {}
    for s, (e, eff, cond, t) in enumerate(meta):
        ks = np.nonzero(conv[:, s])[0]
        assert len(ks) >= 3, (e, cond, t)
        err = max(abs(float(on[k]["clk"]["ppm"][s]) - eff) for k in ks)
        assert err <= (0.5 if cond == "clean" else 1.5), (e, cond, t, err)
        fib_on = sum(bin(int(o["results"]["fib_crc_mask"][s])).count("1") for o in on if o["results"]["status"][s] == pkg.FRAME_DECODED)
        fib_off = sum(bin(int(o["results"]["fib_crc_mask"][s])).count("1") for o in off if o["results"]["status"][s] == pkg.FRAME_DECODED)
        assert fib_on >= fib_off, (e, cond, t, fib_on, fib_off)
        if e == 0.0 and cond == "clean":
            for a, b in zip(off, on):
                for key in ("results", "fibs", "msc", "sf", "ber"):
                    assert np.array_equal(a[key][s], b[key][s]), key
        acc = stats.setdefault((e, cond), np.zeros((2, 4)))
        for i, outs in enumerate((off, on)):
            for k in ks:
                b = outs[k]["ber"][s]
                acc[i] += (b["fic_errors"], b["fic_bits"] - b["fic_erasures"], b["subch"]["errors"][0], b["subch"]["bits"][0] - b["subch"]["erasures"][0])
    print({f"{e}@{c}": (v[:, 0] / v[:, 1], v[:, 2] / v[:, 3]) for (e, c), v in stats.items()})
    # the ramp is removed, the clock error's inter-carrier interference is not (about -17 dB on the edge carriers at 100 ppm): at
    # +-120 ppm and 10 dB TRACK's channel BER stays about twice the 0 ppm recording's
    base = stats[(0.0, "10dB")][1]
    for e in (-120.0, 120.0):
        v_off, v_on = stats[(e, "10dB")]
        for num, den in ((0, 1), (2, 3)):
            ber_off, ber_on, ber_0 = v_off[num] / v_off[den], v_on[num] / v_on[den], base[num] / base[den]
            assert ber_on <= 0.5 * ber_off and ber_on <= 3.0 * ber_0, (e, num, ber_off, ber_on, ber_0)
