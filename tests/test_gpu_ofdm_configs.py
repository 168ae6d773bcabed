"""The OFDM demodulator (ofdm_demod_kernel) in every launch configuration, sample alignment, oscillator mode and input scale.

Stage level (dabb_ofdm_demod): in DABB_FFT_EXACT + DABB_NCO_EXACT the softbits and r1 must equal the oracle's bit for bit (r1 as
uint32, NaN against NaN); the tolerance modes are held to the float64 reference of tests/ofdmref.py (r1 within 1e-4 of
|X_l| |X_{l-1}|, softbits within 1, the guard-interval correlation within 1e-5 relative).  Every frame reads its own window of a
buffer at an odd stride, so that both 16-byte alignments of the symbol copy occur and a CTA that read another frame's window,
start or oscillator would be seen.  Pipeline level (dabb_process): every CTAs-per-frame setting and the tail split decode exactly
what one CTA per frame decodes, and what the oracle's closed-loop receiver decodes."""
import ctypes as C

import numpy as np
import pytest

import dabtx
import ofdmref
from conftest import load_pkg

pytestmark = pytest.mark.gpu
TU, TS, TG, K, TF, TNULL = 2048, 2552, 504, 1536, 196608, 2656
SPAN = ofdmref.SPAN
SOFT = 75 * 3072
FLOATS = ("freq_corr_re", "freq_corr_im", "slevel")
FLT_MAX = float(np.finfo(np.float32).max)


# ------------------------------------------------------------------------------------------------ helpers
@pytest.fixture(scope="module")
def pkg():
    return load_pkg()


@pytest.fixture(scope="module")
def recordings():
    """four distinct recordings of three frames: clean, noisy, multipath, and a 150 Hz carrier offset"""
    clean = dabtx.DabTx(seed=0x0C1).frames(3)
    noisy = dabtx.add_awgn(dabtx.DabTx(seed=0x0C2).frames(3), 15.0, seed=0x0C3)
    echo = ofdmref.multipath(dabtx.DabTx(seed=0x0C4).frames(3), [(0, 1.0), (29, 0.3 + 0.2j), (230, -0.12j)])
    shifted = dabtx.freq_shift(dabtx.DabTx(seed=0x0C5).frames(3), 150.0)
    return [clean, noisy, echo, shifted], [0, 0, 0, 150]


def aligned_starts(rec_len):
    """first useful PRS samples of the frames of a recording that lie inside the guard interval (every symbol window then holds one
    whole transmitted symbol), with both parities"""
    return [k * TF + TNULL + o for k in range(rec_len // TF - 1) for o in (250, 331, 400, 504)]


def stage(ctx, buf, stride, prs, nco=None, r1=False, fc=False, offset=0):
    """dabb_ofdm_demod on the device copy of the flat sample buffer `buf`; frame f reads from buf[offset + f * stride + prs[f]]"""
    n = len(prs)
    d_iq = ctx.dev(np.ascontiguousarray(buf, np.complex64))
    d_ps = ctx.dev(np.ascontiguousarray(prs, np.int64))
    d_soft = ctx.dev(n * SOFT)
    d_r1 = ctx.dev(n * 75 * K * 8) if r1 else None
    d_fc = ctx.dev(n * 8) if fc else None
    d_nco = ctx.dev(np.ascontiguousarray(nco, np.int32)) if nco is not None else None
    ctx._ck(ctx.lib.dabb_ofdm_demod(ctx.h, C.c_void_p(d_iq.ptr + 8 * offset), C.c_int64(stride), C.c_void_p(d_ps.ptr), n,
                                    C.c_void_p(d_nco.ptr) if d_nco else None, C.c_void_p(d_soft.ptr),
                                    C.c_void_p(d_r1.ptr) if d_r1 else None, C.c_void_p(d_fc.ptr) if d_fc else None))
    ctx.sync()
    out = dict(soft=d_soft.download(np.int8).reshape(n, 75, 3072))
    if r1:
        out["r1"] = d_r1.download(np.complex64).reshape(n, 75, K)
    if fc:
        out["fc"] = d_fc.download(np.complex64)
    for b in (d_iq, d_ps, d_soft, d_r1, d_fc, d_nco):
        if b:
            b.free()
    return out


def oracle_frame(oracle, seg, nco=None):
    """the oracle's softbits and r1 of the frame seg[0 : SPAN] (mixed like the exact oscillator first when nco = (lp0, ph))"""
    seg = np.asarray(seg[:SPAN], np.complex64)
    if nco is not None:
        seg = ofdmref.oracle_input(seg, *nco)
    return oracle.demod_frame(seg[:TU], seg[TU:], True)


def same_bits(a, b):
    """float32 arrays equal bit for bit, any NaN equal to any NaN and +0 equal to -0 (the kernel leaves out the products with the
    unit twiddle (1, -0), which only decide the sign of a zero: DESIGN.md 5)"""
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    fa, fb = a.view(np.float32), b.view(np.float32)
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(fa) & np.isnan(fb)) | ((fa == 0) & (fb == 0))


def assert_exact(got, oracle, windows, buf, ncos=None, r1=True):
    for f, w in enumerate(windows):
        s_o, r_o = oracle_frame(oracle, buf[w: w + SPAN], None if ncos is None else ncos[f])
        assert np.array_equal(got["soft"][f], s_o), (f, w, int((got["soft"][f] != s_o).sum()))
        if r1 and "r1" in got:
            ok = same_bits(got["r1"][f], r_o)
            assert ok.all(), (f, w, int((~ok).sum()))


def assert_tolerance(got, buf, windows, ncos=None, what=""):
    for f, w in enumerate(windows):
        nco = None if ncos is None else tuple(int(v) for v in ncos[f])
        ref = ofdmref.frame(buf, w, nco)
        d = np.abs(got["soft"][f].astype(int) - ref["soft"].astype(int))
        assert d.max() <= 1, (what, f, int(d.max()), int((d > 1).sum()))
        if "r1" in got:
            err = np.abs(got["r1"][f].astype(np.complex128) - ref["r1"]) / ref["mag"]
            assert err.max() <= 1e-4, (what, f, float(err.max()))
        if "fc" in got:
            assert abs(complex(got["fc"][f]) - ref["corr"]) <= 1e-5 * abs(ref["corr"]), (what, f, got["fc"][f], ref["corr"])


def distinct_windows(sig, n, tail=8):
    """n windows of `sig` at an odd stride D with per-frame starts p_f: frame 0 at p = 0, the last frame ending on the last sample
    of the signal, both address parities.  Returns (buf = sig + `tail` NaN sentinels, D, prs, windows)."""
    L = len(sig)
    D = (L - SPAN - 1000) // max(n - 1, 1)
    D -= 1 - D % 2
    prs = np.array([(f * 7919) % 997 for f in range(n)], np.int64)
    prs[0] = 0
    if n > 1:
        prs[-1] = L - SPAN - (n - 1) * D
    windows = np.arange(n, dtype=np.int64) * D + prs
    assert windows[-1] + SPAN == L and (windows >= 0).all() and prs.min() == 0
    assert n < 2 or len(set((windows % 2).tolist())) == 2
    buf = np.concatenate([sig, np.full(tail, np.nan, np.complex64)]).astype(np.complex64)
    return buf, D, prs, windows


# ------------------------------------------------------------------------------------------------ stage level, exact mode
@pytest.mark.parametrize("n", [7, 64, 1024])
def test_stage_every_group_count_reads_its_own_window(pkg, oracle, recordings, n):
    """n = 7, 64, 1024 frames: 25, 5 and 1 CTAs per frame (dabb_ofdm_demod picks the count from n).  Every frame reads another
    window of four concatenated recordings; softbits and r1 bit-exact against the oracle."""
    sig = np.concatenate(recordings[0])
    buf, D, prs, windows = distinct_windows(sig, n)
    ctx = pkg.Context(n_streams=1)
    got = stage(ctx, buf, D, prs, r1=n <= 64)
    assert_exact(got, oracle, windows, buf)
    if n == 7:
        # one CTA per frame (forced by the correlation output): the same bytes, and the correlation of the float64 reference
        one = stage(ctx, buf, D, prs, r1=True, fc=True)
        assert np.array_equal(one["soft"], got["soft"]) and np.array_equal(one["r1"].view(np.uint32), got["r1"].view(np.uint32))
        for f, w in enumerate(windows):
            # unaligned windows: the terms need not add up coherently, so the float32 sum is held to 1e-5 of sum |x[i]| |x[i - T_u]|
            sym = buf[w + TU: w + SPAN].astype(np.complex128).reshape(75, TS)
            scale = np.sum(np.abs(sym[:, TU:]) * np.abs(sym[:, :TG]))
            assert abs(complex(one["fc"][f]) - ofdmref.frame(buf, w)["corr"]) <= 1e-5 * scale, f
    ctx.close()


@pytest.mark.parametrize("n", [7, 64])
def test_stage_never_uses_a_sample_outside_its_frame(pkg, oracle, recordings, n):
    """Rows of an odd width with NaN in every sample a frame must not use (padding before and after each frame, NaN rows edges, NaN
    before the first and after the last row, all inside the allocation).  Frames start at their row's first sample and end on its
    last; the symbol copy reads one aligned sample before or after the symbol, which must never reach a result."""
    sig = np.concatenate(recordings[0])
    offs = np.cumsum([0] + [len(r) for r in recordings[0]])[:-1]
    src = [offs[r] + s for r in range(4) for s in aligned_starts(len(recordings[0][r]))]
    W = SPAN + 301                                   # odd
    lead = 8
    buf = np.full(lead + n * W + 8, np.nan, np.complex64)
    prs = np.array([(f * 100) % (W - SPAN + 1) for f in range(n)], np.int64)
    prs[0], prs[1] = 0, W - SPAN                     # the first frame starts at its row's first sample, the second ends on its row's last
    windows = []
    for f in range(n):
        w = lead + f * W + int(prs[f])
        s = src[f % len(src)]
        buf[w: w + SPAN] = sig[s: s + SPAN]
        windows.append(w)
    assert len(set(w % 2 for w in windows)) == 2
    ctx = pkg.Context(n_streams=1)
    got = stage(ctx, buf, W, prs, r1=True, offset=lead)
    assert_exact(got, oracle, windows, buf)
    if n == 7:
        one = stage(ctx, buf, W, prs, r1=True, fc=True, offset=lead)
        assert np.array_equal(one["soft"], got["soft"])
        for f, w in enumerate(windows):
            ref = ofdmref.frame(buf, w)
            assert np.isfinite(one["fc"][f]).all() and abs(complex(one["fc"][f]) - ref["corr"]) <= 1e-5 * abs(ref["corr"]), f
    ctx.close()


# ------------------------------------------------------------------------------------------------ all eight kernel instances
@pytest.mark.parametrize("fft_mode", ["exact", "fma"])
@pytest.mark.parametrize("nco_mode", ["exact", "fast"])
def test_stage_every_kernel_instance(pkg, oracle, recordings, fft_mode, nco_mode):
    """{FFT_EXACT, FFT_FMA} x {NCO_EXACT, NCO_FAST} x {r1 on, off}, each with and without an oscillator, on 7 aligned frames of the
    four recordings (25 CTAs per frame), plus the one-CTA form with the correlation.  The r1-on and r1-off instances write the same
    softbits; exact + exact equals the oracle bit for bit, every mode is within tolerance of the float64 reference."""
    recs, hz = recordings
    sig = np.concatenate(recs)
    offs = np.cumsum([0] + [len(r) for r in recs])[:-1]
    picks = [(0, 0), (1, 1), (2, 2), (3, 3), (0, 5), (3, 6), (2, 7)]          # (recording, aligned start)
    windows = np.array([offs[r] + aligned_starts(len(recs[r]))[i] for r, i in picks], np.int64)
    n = len(windows)
    prs = windows - np.arange(n)                     # stride 1
    assert len(set((windows % 2).tolist())) == 2
    extra = [0, 37, -100, 0, 55, -20, 0]
    ncos = np.array([[(f * 290011 + 1) % 2048000, hz[r] + extra[f]] for f, (r, _) in enumerate(picks)], np.int32)
    ctx = pkg.Context(n_streams=1, fft_mode=pkg.FFT_EXACT if fft_mode == "exact" else pkg.FFT_FMA,
                      nco_mode=pkg.NCO_EXACT if nco_mode == "exact" else pkg.NCO_FAST)
    for nco in (None, ncos):
        off = stage(ctx, sig, 1, prs, nco=nco)
        on = stage(ctx, sig, 1, prs, nco=nco, r1=True)
        one = stage(ctx, sig, 1, prs, nco=nco, r1=True, fc=True)
        assert np.array_equal(off["soft"], on["soft"]), (fft_mode, nco_mode, nco is not None)
        if fft_mode == "exact":
            assert np.array_equal(one["soft"], on["soft"]) and same_bits(one["r1"], on["r1"]).all()
        what = f"{fft_mode}/{nco_mode}/nco={nco is not None}"
        assert_tolerance(on, sig, windows, nco, what)
        assert_tolerance(one, sig, windows, nco, what)
        if fft_mode == "exact" and (nco is None or nco_mode == "exact"):
            assert_exact(on, oracle, windows, sig, nco)
    ctx.close()


# ------------------------------------------------------------------------------------------------ oscillator edges
LP0 = [0, 1, 1023999, 2047999]
PH = [0, 1, -1, 35500, -35500, 1023999, -1023999]


@pytest.mark.parametrize("mode", ["exact", "fast_fma"])
def test_stage_oscillator_edges(pkg, oracle, recordings, mode):
    """lp0 in {0, 1, 1 023 999, 2 047 999} x ph in {0, +-1, +-35 500, +-1 023 999} (lp0 = ph = 0 is no oscillator at all), each on a
    frame shifted by +ph Hz so that the mixed frame is the transmitted one: its FIC decodes.  Exact mode bit for bit against the
    oracle fed with the frame mixed through the float32 table; NCO_FAST + FFT_FMA within tolerance of the float64 reference."""
    clean = recordings[0][0]
    combos = [(lp0, ph) for lp0 in LP0 for ph in PH if lp0 or ph]
    st = TF + TNULL + 400
    W = SPAN + 501
    buf = np.zeros(len(combos) * W, np.complex64)
    windows = []
    for f, (lp0, ph) in enumerate(combos):
        x = dabtx.freq_shift(clean[:2 * TF + TNULL], float(ph)) if ph else clean[:2 * TF + TNULL]
        p = 1 + (f * 131) % 500
        buf[f * W + p: f * W + p + SPAN] = x[st: st + SPAN]
        windows.append(f * W + p)
    prs = np.array(windows, np.int64) - np.arange(len(combos)) * W
    ncos = np.array(combos, np.int32)
    if mode == "exact":
        ctx = pkg.Context(n_streams=1)
    else:
        ctx = pkg.Context(n_streams=1, fft_mode=pkg.FFT_FMA, nco_mode=pkg.NCO_FAST)
    got = stage(ctx, buf, W, prs, nco=ncos, r1=True)
    fc = stage(ctx, buf, W, prs, nco=ncos, fc=True)
    ctx.close()
    assert np.array_equal(fc["soft"], got["soft"])
    got["fc"] = fc["fc"]
    if mode == "exact":
        assert_exact(got, oracle, windows, buf, ncos)
    assert_tolerance(got, buf, windows, ncos, mode)
    for f in range(len(combos)):
        _, crc = oracle.fic_decode(got["soft"][f, :3].reshape(-1))
        assert crc.all(), (mode, combos[f])


# ------------------------------------------------------------------------------------------------ input scale
def in_range(r1_scaled):
    """carriers whose l1 = |re| + |im| (float32) is a normal float below 2^126 and whose 127 / l1 is finite in float32: there the
    demap's reciprocal equals the IEEE quotient (DESIGN.md 5)"""
    l1 = (np.abs(r1_scaled.real) + np.abs(r1_scaled.imag)).astype(np.float32).astype(np.float64)
    with np.errstate(divide="ignore", over="ignore"):
        q = np.float32(127.0) / l1.astype(np.float32)
    return (l1 >= 2.0 ** -126) & (l1 < 2.0 ** 126) & np.isfinite(q)


def test_stage_input_scale_over_the_whole_float_range(pkg, oracle, recordings):
    """One clean and one noisy frame times 2^k for every k from all-zero to all-infinite samples.  Where l1 is in range the softbits
    equal the unscaled ones and the oracle's, and r1 is the unscaled r1 times 2^2k exactly (for l1 >= 2^-100, where no product inside
    r1 is subnormal); everywhere r1 equals the oracle's bit for
    bit and every softbit is the oracle's or 0.  Plus an all-zero PRS and an all-zero data symbol (r1 = 0 on two symbols)."""
    st = TF + TNULL + 350
    base = [recordings[0][0][st: st + SPAN], recordings[0][1][st: st + SPAN]]
    ks = list(range(-152, 132))
    jobs = [(b, k) for k in ks for b in range(2)]
    ctx = pkg.Context(n_streams=1)
    unscaled = [stage(ctx, base[b], 0, np.zeros(1, np.int64), r1=True) for b in range(2)]
    for b in range(2):
        s_o, r_o = oracle_frame(oracle, base[b])
        assert np.array_equal(unscaled[b]["soft"][0], s_o) and same_bits(unscaled[b]["r1"][0], r_o).all()
    counts = dict(in_range=0, zero_outside=0, equal_outside=0)
    for c0 in range(0, len(jobs), 64):
        chunk = jobs[c0: c0 + 64]
        with np.errstate(over="ignore", under="ignore", invalid="ignore"):
            frames = np.stack([(base[b].astype(np.complex128) * 2.0 ** k).astype(np.complex64) for b, k in chunk])
        got = stage(ctx, frames.reshape(-1), SPAN, np.zeros(len(chunk), np.int64), r1=True)
        for f, (b, k) in enumerate(chunk):
            s_o, r_o = oracle_frame(oracle, frames[f])
            assert same_bits(got["r1"][f], r_o).all(), (b, k)
            g, u = got["soft"][f], unscaled[b]["soft"][0]
            with np.errstate(over="ignore", under="ignore", invalid="ignore"):
                m = in_range(unscaled[b]["r1"][0].astype(np.complex128) * 2.0 ** (2 * k))
            mm = np.concatenate([m, m], axis=1)
            assert np.array_equal(g[mm], s_o[mm]) and np.array_equal(g[mm], u[mm]), (b, k, int((g[mm] != u[mm]).sum()))
            # r1 scales exactly where none of its four products can be subnormal: l1 >= 2^-100 leaves a margin of 2^26
            with np.errstate(over="ignore", under="ignore", invalid="ignore"):
                scaled = unscaled[b]["r1"][0].astype(np.complex128) * 2.0 ** (2 * k)
                m &= np.abs(scaled.real) + np.abs(scaled.imag) >= 2.0 ** -100
            assert np.array_equal(got["r1"][f][m].astype(np.complex128), scaled[m]), (b, k)
            out = ~mm
            bad = out & (g != s_o) & (g != 0)
            assert not bad.any(), (b, k, int(bad.sum()), g[bad][:8], s_o[bad][:8])
            counts["in_range"] += int(mm.sum())
            counts["zero_outside"] += int((out & (g == 0) & (s_o != 0)).sum())
            counts["equal_outside"] += int((out & (g == s_o)).sum())
    print("input scale:", counts)
    # the range holds for most carriers of the scales in between, and the upper end (l1 >= 2^126) returns 0 where the oracle does not
    assert counts["in_range"] > 100 * 75 * 3072 and counts["zero_outside"] > 0
    # zero PRS (r1 = 0 on symbol 1) and a zero data symbol 20 (r1 = 0 on symbols 20 and 21)
    z = np.stack([base[0].copy(), base[1].copy()])
    z[0, :TU] = 0
    z[1, TU + 19 * TS: TU + 20 * TS] = 0
    got = stage(ctx, z.reshape(-1), SPAN, np.zeros(2, np.int64), r1=True)
    ctx.close()
    assert_exact(got, oracle, [0, SPAN], z.reshape(-1))
    assert not got["soft"][0, 0].any() and got["soft"][0, 1].any()
    assert not got["soft"][1, 19:21].any() and not got["r1"][1, 19:21].any() and got["soft"][1, 21].any()


@pytest.mark.parametrize("fmt", ["s16_full_scale", "u8_one_lsb"])
def test_pipeline_extreme_raw_sample_levels(pkg, oracle, fmt):
    """a full-scale s16 signal and a u8 signal of +-1 LSB, converted on the device (convert_iq_kernel) and decoded by dabb_process:
    softbits, FIBs and start index of every frame equal the oracle's receiver fed with the CPU-converted samples"""
    sig = dabtx.DabTx(seed=0x5CA).frames(8)
    inter = np.stack([sig.real, sig.imag], axis=-1).astype(np.float64)
    peak = np.abs(inter).max()
    if fmt == "s16_full_scale":
        s16 = np.clip(np.round(inter / peak * 32767.0 * 1.5), -32768, 32767).astype(np.int16)     # clipped at full scale
        ref = s16.astype(np.float32).view(np.complex64).reshape(-1)
        raw, f = s16.astype(">i2").view(np.uint8).reshape(len(sig), 4), pkg.IQ_S16LE
    else:
        u8 = (np.clip(np.round(inter / np.std(inter)), -1, 1) + 128).astype(np.uint8)
        ref = ((u8.astype(np.float32) - 128.0) / 128.0).view(np.complex64).reshape(-1)
        raw, f = u8, pkg.IQ_U8
    raw = np.ascontiguousarray(raw)
    ctx = pkg.Context(n_streams=1, keep_taps=True)
    frames = []
    for step in range(9):
        out = ctx.process(raw, len(sig), np.zeros(1, np.int64), len(sig), iq_is_host=True, iq_format=f)
        r = out["results"]
        if r["status"][0] == pkg.FRAME_DECODED and r["next_pos"][0] <= len(sig):
            frames.append((int(r["start_index"][0]), out["fibs"][0].copy(), ctx.read_tap(0)[0].copy()))
    ctx.close()
    o = oracle.rx_run(ref, disable_coarse=True, want_soft=8)
    n = min(len(frames), o["frames"])
    assert n >= 4, (fmt, len(frames), o["frames"])
    for k in range(n):
        assert frames[k][0] == o["info"][k]["start_index"], (fmt, k)
        assert np.array_equal(frames[k][2], o["soft"][k]), (fmt, k, int((frames[k][2] != o["soft"][k]).sum()))
        assert np.array_equal(frames[k][1], o["fibs"][12 * k: 12 * k + 12, 1:]), (fmt, k)


# ------------------------------------------------------------------------------------------------ pipeline: CTAs per frame
S_PIPE, BITRATE, STEPS = 48, 96, 9
LOCK = [(0x51, 2000.0), (4, 1000.0), (8, -1000.0)]          # offsets on which the coarse corrector locks (test_gpu_pipeline.py)


def _pipe_streams():
    """48 streams: 8 transmitters, each stream with its own time offset, carrier offset and noise; streams 0-2 need the coarse
    corrector (whole-carrier offsets)"""
    rng = np.random.default_rng(0x48)
    txs = [dabtx.DabTx(seed=0x4800 + i, bitrate=BITRATE).frames(STEPS + 2) for i in range(8)]
    n = len(txs[0]) - TF
    sigs = []
    for s in range(S_PIPE):
        if s < 3:
            x = dabtx.DabTx(seed=LOCK[s][0], bitrate=BITRATE).frames(STEPS + 2)
            sigs.append(dabtx.freq_shift(x, LOCK[s][1])[:n])
            continue
        off = int(rng.integers(0, TF - 1))
        x = txs[s % 8][off: off + n]
        x = dabtx.freq_shift(x, float(rng.integers(-300, 301)))
        if s % 3:
            x = dabtx.add_awgn(x, float(rng.uniform(9.0, 25.0)), seed=s)
        sigs.append(x)
    return np.stack(sigs).astype(np.complex64)


def _run_pipe(pkg, buf, d, **kw):
    ctx = pkg.Context(n_streams=S_PIPE, keep_taps=True, disable_coarse=False, **kw)
    ctx.select_subchannel(0, dabtx.eep_cu(BITRATE), BITRATE, eep_profile_a=True, eep_level=3, dabplus=True)
    steps = []
    for k in range(STEPS):
        out = ctx.process(d, buf.shape[1], np.zeros(S_PIPE, np.int64), buf.shape[1], msc_stride=3 * BITRATE, sf_stride=15 * BITRATE)
        out["soft"] = ctx.read_tap(0)
        out["const"] = ctx.read_tap(2)
        steps.append(out)
    ctx.close()
    return steps


def _without_floats(res):
    r = res.copy()
    for f in FLOATS:
        r[f] = 0
    return r


def _close(a, b):
    za = a["freq_corr_re"].astype(np.float64) + 1j * a["freq_corr_im"]
    zb = b["freq_corr_re"].astype(np.float64) + 1j * b["freq_corr_im"]
    la, lb = a["slevel"].astype(np.float64), b["slevel"].astype(np.float64)
    return (np.abs(za - zb) <= 1e-5 * np.abs(za)) & (np.abs(la - lb) <= 1e-5 * np.abs(la))


def _per_stream(pkg, steps, s, n):
    """stream s's decoded frames: (start index, fine, coarse, crc mask, FIBs, softbits) and its logical frames"""
    frames, msc = [], []
    for out in steps:
        r = out["results"]
        if r["status"][s] != pkg.FRAME_DECODED or r["next_pos"][s] > n:
            continue
        frames.append((int(r["start_index"][s]), int(r["fine_corr"][s]), int(r["coarse_corr"][s]), int(r["fib_crc_mask"][s]),
                       out["fibs"][s], out["soft"][s]))
        for c in range(4 - int(r["n_logical"][s][0]), 4):
            msc.append(out["msc"][s, 0, c])
    return frames, (np.concatenate(msc) if msc else np.zeros(0, np.uint8))


def _crc_mask(orc, f):
    return int(sum(int(o) << k for k, o in enumerate(orc["fibs"][12 * f: 12 * f + 12, 0])))


def test_pipeline_every_group_count_decodes_the_same(pkg, oracle):
    """ofdm_groups 1, 3, 5, 15, 25, 75 and the default on 48 distinct streams (coarse corrector on): softbits, constellation, FIBs,
    logical frames, superframes and every result field identical across the settings (the fine-AFC correlation and the level within
    1e-5: partial sums added in another order).  One CTA per frame against the oracle's receiver for 8 streams; DABB_NCO_FAST
    against it for the streams whose coarse corrector moves between the phase reference and the data symbols."""
    buf = _pipe_streams()
    n = buf.shape[1]
    holder = pkg.Context(n_streams=1)
    d = holder.dev(buf)
    runs = {g: _run_pipe(pkg, buf, d, ofdm_groups=g) for g in (1, 3, 5, 15, 25, 75, 0)}
    fast = _run_pipe(pkg, buf, d, nco_mode=pkg.NCO_FAST)
    d.free(); holder.close()
    base = runs[1]
    decoded = 0
    for g, steps in runs.items():
        for k in range(STEPS):
            x, y = steps[k], base[k]
            assert (_without_floats(x["results"]) == _without_floats(y["results"])).all(), (g, k)
            ok = _close(y["results"], x["results"])
            assert ok.all(), (g, k, np.flatnonzero(~ok)[:8])
            dec = x["results"]["status"] == pkg.FRAME_DECODED
            for name in ("fibs", "msc", "sf"):
                assert np.array_equal(x[name], y[name]), (g, k, name)
            for name in ("soft", "const"):         # the taps of a stream that decoded nothing in this step are stale
                assert np.array_equal(x[name][dec], y[name][dec]), (g, k, name)
            decoded += int(dec.sum())
    assert decoded >= 7 * S_PIPE * (STEPS - 3), decoded
    prot = oracle.prot_eep(BITRATE, 1, 3)
    coarse_moved = 0
    for s in (0, 1, 2, 3, 4, 9, 20, 47):
        orc = oracle.rx_run(buf[s], prot=prot, start_cu=0, len_cu=dabtx.eep_cu(BITRATE), select_after_frames=0, disable_coarse=False,
                            want_soft=STEPS)
        got, msc = _per_stream(pkg, base, s, n)
        m = min(len(got), orc["frames"])
        assert m >= STEPS - 3, (s, len(got), orc["frames"])
        for f in range(m):
            info = orc["info"][f]
            assert (got[f][0], got[f][2], got[f][3]) == (info["start_index"], info["coarse"], _crc_mask(orc, f)), (s, f)
            if s >= 3:
                assert got[f][1] == info["fine"], (s, f)
                assert np.array_equal(got[f][4], orc["fibs"][12 * f: 12 * f + 12, 1:]), (s, f)
                assert np.array_equal(got[f][5], orc["soft"][f]), (s, f, int((got[f][5] != orc["soft"][f]).sum()))
            else:
                assert abs(got[f][1] - info["fine"]) <= 1, (s, f)
        if s >= 3:
            k = min(len(msc), len(orc["msc"]))
            assert k >= 3 * BITRATE * 4 and np.array_equal(msc[:k], orc["msc"][:k]), s
        else:
            coarse_moved += sum(1 for f in range(1, m) if orc["info"][f]["coarse"] != orc["info"][f - 1]["coarse"]) + (orc["info"][0]["coarse"] != 0)
            # the fast oscillator: same coarse corrector and FIB CRCs as the oracle's receiver
            fgot, _ = _per_stream(pkg, fast, s, n)
            mf = min(len(fgot), orc["frames"])
            assert mf >= STEPS - 3
            assert [(a[0], a[2], a[3]) for a in fgot[:mf]] == [(orc["info"][f]["start_index"], orc["info"][f]["coarse"], _crc_mask(orc, f)) for f in range(mf)], s
            assert _crc_mask(orc, mf - 1) == 0xFFF
    assert coarse_moved >= 3


# ------------------------------------------------------------------------------------------------ pipeline: tail split
S_TAIL, D_TAIL, TAIL_STEPS = 2048, 95, 9


def test_tail_split_with_distinct_streams(pkg, oracle):
    """2048 streams read one recording at an odd stride D = 95: stream s starts 95 s samples later, so it has its own start index,
    sample alignment and oscillator phase.  The tail split against one CTA per frame, stream by stream: identical but for the partial
    sums of the tail streams (a suffix of the batch).  Four tail and two head streams against the oracle's receiver on their slice."""
    sig = dabtx.add_awgn(dabtx.freq_shift(dabtx.DabTx(seed=0x7A12, bitrate=BITRATE).frames(11), 30.0), 18.0, seed=11)
    n = len(sig) - D_TAIL * (S_TAIL - 1)
    split, whole = (pkg.Context(n_streams=S_TAIL, ofdm_tail_split=t) for t in (0, -1))
    for c in (split, whole):
        c.select_subchannel(0, dabtx.eep_cu(BITRATE), BITRATE, eep_profile_a=True, eep_level=3, dabplus=True)
    ds, dw = split.dev(sig), whole.dev(sig)
    watch = [0, 1, S_TAIL - 200, S_TAIL - 101, S_TAIL - 2, S_TAIL - 1]
    kept = {s: [] for s in watch}
    tail = np.zeros(S_TAIL, bool)
    starts = set()
    for k in range(TAIL_STEPS):
        outs = []
        for c, d in ((split, ds), (whole, dw)):
            out = c.process(d, D_TAIL, np.zeros(S_TAIL, np.int64), n, msc_stride=3 * BITRATE, sf_stride=15 * BITRATE)
            out["soft"] = c.read_tap(0)
            outs.append(out)
        x, y = outs
        rx, ry = x["results"], y["results"]
        assert (_without_floats(rx) == _without_floats(ry)).all(), k
        ok = _close(ry, rx)
        assert ok.all(), (k, np.flatnonzero(~ok)[:8])
        for f in FLOATS:
            tail |= rx[f] != ry[f]
        dec = rx["status"] == pkg.FRAME_DECODED
        for name in ("fibs", "msc", "sf"):
            assert np.array_equal(x[name], y[name]), (name, k)
        assert np.array_equal(x["soft"][dec], y["soft"][dec]), k
        starts |= set(rx["start_index"][dec].tolist())
        for s in watch:
            if dec[s] and rx["next_pos"][s] <= n:
                kept[s].append((int(rx["start_index"][s]), int(rx["fine_corr"][s]), x["fibs"][s].copy(), x["soft"][s].copy(),
                                [x["msc"][s, 0, c].copy() for c in range(4 - int(rx["n_logical"][s][0]), 4)]))
        del outs, x, y
    ds.free(); dw.free(); split.close(); whole.close()
    n_tail = int(tail.sum())
    assert 0 < n_tail <= S_TAIL // 4 and tail[S_TAIL - n_tail:].all(), np.flatnonzero(tail)[:8]
    assert all(s >= S_TAIL - n_tail for s in watch[2:]), n_tail
    assert len(starts) >= 2, starts
    prot = oracle.prot_eep(BITRATE, 1, 3)
    for s in watch:
        orc = oracle.rx_run(sig[D_TAIL * s: D_TAIL * s + n], prot=prot, start_cu=0, len_cu=dabtx.eep_cu(BITRATE), select_after_frames=0,
                            want_soft=TAIL_STEPS)
        got = kept[s]
        m = min(len(got), orc["frames"])
        assert m >= TAIL_STEPS - 3, (s, len(got), orc["frames"])
        for f in range(m):
            assert (got[f][0], got[f][1]) == (orc["info"][f]["start_index"], orc["info"][f]["fine"]), (s, f)
            assert np.array_equal(got[f][2], orc["fibs"][12 * f: 12 * f + 12, 1:]), (s, f)
            assert np.array_equal(got[f][3], orc["soft"][f]), (s, f, int((got[f][3] != orc["soft"][f]).sum()))
        msc = np.concatenate([c for g in got for c in g[4]])
        k = min(len(msc), len(orc["msc"]))
        assert k >= 3 * BITRATE * 4 and np.array_equal(msc[:k], orc["msc"][:k]), s
