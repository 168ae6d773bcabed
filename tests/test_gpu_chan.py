"""The wideband channelizer on the device (dabb_channelize, chan_kernel).

Stage level: against the float64 definition (tests/chanref.py) with the bound of tests/test_chan_emul.py, rms error <= 1e-5 x rms(y_ref)
and largest error <= 1e-4 x rms(y_ref) per channel.  Each term of an output's sum is a float tap (relative error 2^-24) times a mixed
sample whose phase -2 k / R is rounded to float (under 4e-7 rad); T terms are summed in fp32 into two accumulators, so the rounding
error grows like sqrt(T) 2^-24 of the output's scale, about 3e-6 at T = 1559.  Calls cut anywhere give the same bits as one call.

Closed loop: wideband recordings of several DabTx ensembles (own seed, bitrate, protection, DAB / DAB+, frame timing, a few hundred Hz of
carrier offset; each band-limited to +-800 kHz at 2.048 Msps and then resampled with scipy.signal.resample_poly, one 20 dB above its
neighbours, AWGN at 24 dB in-band SNR) are channelized and decoded by one context.  Every stream's FIBs and logical frames must be the same bytes as those
of the ensemble's own 2.048 Msps signal decoded by a second context, frame for frame once both are tracking, with every FIB CRC good."""
import numpy as np
import pytest

import chanref
import dabtx
from conftest import load_pkg

pytestmark = pytest.mark.gpu
RMS_BOUND, MAX_BOUND = 1e-5, 1e-4
TF = 196608


@pytest.fixture(scope="module")
def ctx():
    pkg = load_pkg()
    c = pkg.Context(n_streams=1)
    yield c
    c.close()


def noise(rng, shape):
    return (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).astype(np.complex64)


def run_device(pkg, ctx, R, offsets, inputs_of, x, in_start, out_start, out_len, fmt=0, host=True):
    ch = pkg.Channelizer(ctx, R, offsets, inputs_of, iq_format=fmt)
    try:
        if host:
            d = ch.run(x, in_start, x.shape[1] if fmt == 0 else x.shape[1] // chanref.BYTES[fmt], out_start, out_len)
        else:
            dx = ctx.dev(x)
            n = x.shape[1] if fmt == 0 else x.shape[1] // chanref.BYTES[fmt]
            d = ch.run(dx, in_start, n, out_start, out_len, in_stride=n, in_is_host=False)
            ctx.sync()
            dx.free()
        ctx.sync()
        y = d.download(np.complex64).reshape(len(offsets), out_len)
        d.free()
        return y
    finally:
        ch.destroy()


CASES = [(R, o) for R in chanref.RATES for o in sorted({0, R // 2 - 768000, -(R // 2 - 768000)} | ({1712000, -1712000} if R // 2 - 768000 >= 1712000 else set()))]


@pytest.mark.parametrize("R", chanref.RATES)
def test_stage_against_definition(ctx, R):
    """every listed rate, offsets 0, +-1 712 000 and the band edges, indices near 0 and near 2^40, an odd input alignment, host and device
    input, several inputs and channels"""
    pkg = load_pkg()
    rng = np.random.default_rng(R % 10007)
    L, M, T = chanref.geometry(R)
    offs = [o for (r, o) in CASES if r == R]
    n_ch = len(offs)
    for out_start, host in ((0, True), ((1 << 40) * L // M + 3, False)):
        out_len = 700
        first, end = chanref.input_range(R, out_start, out_len)
        in_start = first - 3                                    # the buffers start 3 samples early: an odd alignment of the span
        n = end - in_start + 1
        x = noise(rng, (2, n))
        inputs_of = np.arange(n_ch, dtype=np.int32) % 2
        y = run_device(pkg, ctx, R, offs, inputs_of, x, [in_start, in_start], out_start, out_len, host=host)
        for c, f in enumerate(offs):
            want = chanref.channelize(x[inputs_of[c]].astype(np.complex128), in_start, R, f, out_start, out_len)
            rms, mx = chanref.error_ratio(y[c], want)
            assert rms <= RMS_BOUND and mx <= MAX_BOUND, (R, f, out_start, rms, mx)


@pytest.mark.parametrize("fmt", [1, 2, 3, 4])
def test_raw_formats(ctx, fmt):
    pkg = load_pkg()
    R, offs = 8192000, [-3000000, 0, 1712000]
    rng = np.random.default_rng(fmt)
    first, end = chanref.input_range(R, 5000, 2000)
    raw = rng.integers(0, 256, (1, (end - first) * chanref.BYTES[fmt]), dtype=np.uint8)
    y = run_device(pkg, ctx, R, offs, None, raw, [first], 5000, 2000, fmt=fmt)
    for c, f in enumerate(offs):
        want = chanref.channelize(chanref.convert(raw[0], fmt), first, R, f, 5000, 2000)
        rms, mx = chanref.error_ratio(y[c], want)
        assert rms <= RMS_BOUND and mx <= MAX_BOUND, (fmt, f, rms, mx)


@pytest.mark.parametrize("n_ch", [1, 7, 64])
def test_many_channels_and_calls_cut_anywhere(ctx, n_ch):
    """n_channels 1..64 over 3 inputs with their own buffer starts; the run cut into calls of 1, 255, 256, 257, 3000 and the rest
    outputs (each channel at its own output position) gives the same bits as one call"""
    pkg = load_pkg()
    R = 20000000
    rng = np.random.default_rng(n_ch)
    offs = list(rng.integers(-(R // 2 - 768000), R // 2 - 768000, n_ch))
    inputs_of = rng.integers(0, 3, n_ch).astype(np.int32)
    out_start = rng.integers(0, 50000, n_ch)
    total = 6000
    spans = [chanref.input_range(R, int(s), total) for s in out_start]
    in_start = np.array([min(spans[c][0] for c in range(n_ch) if inputs_of[c] == i) if (inputs_of == i).any() else 0 for i in range(3)]) - 1
    n = max(spans[c][1] - in_start[inputs_of[c]] for c in range(n_ch)) + 2
    x = noise(rng, (3, n))
    ch = pkg.Channelizer(ctx, R, offs, inputs_of, n_inputs=3)
    try:
        whole = ch.run(x, in_start, n, out_start, total)
        ctx.sync()
        w = whole.download(np.complex64).reshape(n_ch, total)
        parts, done = [], 0
        for k in (1, 255, 256, 257, 3000, total - 3769):
            d = ch.run(x, in_start, n, out_start + done, k)
            ctx.sync()
            parts.append(d.download(np.complex64).reshape(n_ch, k)); d.free()
            done += k
        assert done == total
        assert np.array_equal(np.concatenate(parts, axis=1).view(np.uint64), w.view(np.uint64))
        for c in range(0, n_ch, max(1, n_ch // 4)):
            i = inputs_of[c]
            want = chanref.channelize(x[i].astype(np.complex128), int(in_start[i]), R, int(offs[c]), int(out_start[c]), 1500)
            rms, mx = chanref.error_ratio(w[c, :1500], want)
            assert rms <= RMS_BOUND and mx <= MAX_BOUND, (c, rms, mx)
        whole.free()
    finally:
        ch.destroy()


def test_refusals_write_nothing(ctx):
    import ctypes as C
    pkg = load_pkg()
    lib = ctx.lib
    E_ARG, E_UNSUPPORTED = -3, -6
    R = 10000000
    off = np.array([0, 1712000], np.int64); inp = np.array([0, 0], np.int32)

    def create(rate=R, fmt=0, n_in=1, n_ch=2, inputs=inp, offsets=off):
        cfg = pkg.dabb200.ChanConfig(rate, fmt, n_in, n_ch, 0, None if inputs is None else inputs.ctypes.data, None if offsets is None else offsets.ctypes.data)
        h = C.c_void_p()
        rc = lib.dabb_chan_create(ctx.h, C.byref(cfg), C.byref(h))
        if rc == 0:
            lib.dabb_chan_destroy(h)
        return rc

    assert create() == 0
    assert create(rate=2047999) == E_UNSUPPORTED and create(rate=64000001) == E_UNSUPPORTED and create(rate=9999999) == E_UNSUPPORTED
    assert create(fmt=5) == E_ARG and create(n_in=0) == E_ARG and create(n_ch=0) == E_ARG and create(n_ch=4097) == E_ARG
    assert create(inputs=None) == E_ARG and create(offsets=None) == E_ARG
    assert create(inputs=np.array([0, 1], np.int32)) == E_ARG and create(inputs=np.array([0, -1], np.int32)) == E_ARG
    assert create(offsets=np.array([0, R // 2 - 767999], np.int64)) == E_ARG and create(offsets=np.array([-(R // 2 - 767999), 0], np.int64)) == E_ARG
    h = C.c_void_p()
    assert lib.dabb_chan_create(None, None, C.byref(h)) == E_ARG
    lib.dabb_chan_destroy(None)

    ch = pkg.Channelizer(ctx, R, off)
    try:
        out_len, stride = 512, 600
        first, end = ch.input_range(1000, out_len)
        assert (first, end) == chanref.input_range(R, 1000, out_len)
        x = noise(np.random.default_rng(0), (1, end - first))
        canary = np.full(2 * 2 * stride, 12345.0, np.float32)
        d = ctx.dev(canary)

        def call(**kw):
            a = dict(in_=x.ctypes.data, in_is_host=1, in_stride=x.shape[1], in_start=np.array([first], np.int64), in_len=x.shape[1],
                     out=d.ptr, out_stride=stride, out_start=np.array([1000, 1000], np.int64), out_len=out_len)
            a.update(kw)
            keep = [a["in_start"], a["out_start"]]
            io = pkg.dabb200.ChanIO(a["in_"], a["in_is_host"], a["in_stride"], None if a["in_start"] is None else a["in_start"].ctypes.data, a["in_len"],
                                    a["out"], a["out_stride"], None if a["out_start"] is None else a["out_start"].ctypes.data, a["out_len"])
            rc = lib.dabb_channelize(ch.h, C.byref(io))
            del keep
            return rc

        refusals = {
            "in NULL": dict(in_=None), "out NULL": dict(out=None), "in_start NULL": dict(in_start=None), "out_start NULL": dict(out_start=None),
            "out_len 0": dict(out_len=0), "out_stride short": dict(out_stride=out_len - 1), "in_stride short": dict(in_stride=x.shape[1] - 1),
            "in_is_host 2": dict(in_is_host=2), "span starts early": dict(in_start=np.array([first + 1], np.int64)),
            "span ends late": dict(in_len=x.shape[1] - 1), "one channel outside": dict(out_start=np.array([1000, 1001], np.int64)),
            "negative out_start": dict(out_start=np.array([-1, 1000], np.int64)), "out index past 2^45": dict(out_start=np.array([1000, (1 << 45) - 100], np.int64)),
        }
        for name, kw in refusals.items():
            assert call(**kw) == E_ARG, name
            ctx.sync()
            assert np.array_equal(d.download(np.float32), canary), name
        assert lib.dabb_channelize(None, None) == E_ARG
        io = pkg.dabb200.ChanIO()
        assert lib.dabb_channelize(ch.h, None) == E_ARG and lib.dabb_channelize(ch.h, C.byref(io)) == E_ARG
        f, e = C.c_int64(), C.c_int64()
        assert lib.dabb_chan_input_range(ch.h, C.c_int64(-1), C.c_int64(1), C.byref(f), C.byref(e)) == E_ARG
        assert lib.dabb_chan_input_range(ch.h, C.c_int64(0), C.c_int64(0), C.byref(f), C.byref(e)) == E_ARG
        assert lib.dabb_chan_input_range(None, C.c_int64(0), C.c_int64(1), C.byref(f), C.byref(e)) == E_ARG
        assert call() == 0                                       # the same call with good arguments does write
        ctx.sync()
        assert not np.array_equal(d.download(np.float32), canary)
        d.free()
    finally:
        ch.destroy()


# ---------------------------------------------------------------------------------------------------------------- closed loop

ENSEMBLES = [  # seed, bitrate, EEP-A, level, DAB+
    (0xC1, 96, True, 3, True), (0xC2, 64, False, 2, False), (0xC3, 128, True, 2, True), (0xC4, 48, True, 3, False), (0xC5, 80, False, 3, True)]
FRAMES = 20


def ensembles(n, seed):
    """n ensembles at 2.048 Msps: own timing (a delay of up to one frame) and a carrier offset of 100 to 200 Hz, band-limited to
    +-800 kHz"""
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n):
        sd, br, a, lv, dp = ENSEMBLES[k % len(ENSEMBLES)]
        tx = dabtx.DabTx(seed=sd, bitrate=br, profile_a=a, level=lv, dabplus=dp)
        s = tx.frames(FRAMES)
        s = np.concatenate([np.zeros(int(rng.integers(0, TF)), np.complex64), s])
        s = dabtx.freq_shift(s, float(rng.integers(100, 200) * (1 if k % 2 else -1)))
        S = np.fft.fft(s)
        fr = np.fft.fftfreq(len(s), 1 / 2048000)
        S[np.abs(fr) > 800000] = 0
        out.append((tx, np.fft.ifft(S).astype(np.complex64)))
    return out


def wideband(sigs, R, offsets, gains_db, snr_db, seed):
    """the sum of the ensembles resampled to R and moved to their offsets (exact integer phase), with AWGN: snr_db is the in-band SNR of
    a 0 dB ensemble"""
    from math import gcd
    from scipy.signal import resample_poly
    g = gcd(2048000, R)
    up, down = R // g, 2048000 // g
    n = min(len(s) for _, s in sigs) * up // down
    x = np.zeros(n, np.complex128)
    idx = np.arange(n, dtype=np.int64)
    for (tx, s), f, gdb in zip(sigs, offsets, gains_db):
        y = resample_poly(s.astype(np.complex128), up, down)[:n]
        x += y * 10 ** (gdb / 20) * np.exp(2j * np.pi * (((f % R) * idx) % R) / R)
    p = float(np.mean(np.abs(sigs[0][1]) ** 2)) * 2048000 / R                 # a 0 dB ensemble's power per sample at R
    rng = np.random.default_rng(seed)
    sigma = np.sqrt(p * (R / 1536000) / 10 ** (snr_db / 10) / 2)
    x += (rng.standard_normal(n) + 1j * rng.standard_normal(n)) * sigma
    return x


def quantize(x, fmt):
    if fmt == 0:
        return x.astype(np.complex64)[None, :]
    v = np.empty(2 * len(x)); v[0::2], v[1::2] = x.real, x.imag
    v = v / (4 * np.sqrt(np.mean(v ** 2)))                                     # rms a quarter of full scale
    q = np.clip(np.round(v * 128), -128, 127)
    return (q + 128).astype(np.uint8)[None, :] if fmt == 1 else q.astype(np.int8).view(np.uint8)[None, :]


def decode(pkg, c, txs, iq_dev, stride, buf_len, steps=FRAMES + 3):
    """decode with context c (one stream per transmitter, each its own sub-channel): per stream the (FIB bytes, CRC mask) of every
    decoded frame, its logical frames and the status of every step"""
    S = len(txs)
    flen = max(3 * tx.bitrate for tx in txs)
    for s, tx in enumerate(txs):
        c.select_subchannel(tx.start_cu, tx.size_cu, tx.bitrate, eep_profile_a=tx.profile_a, eep_level=tx.level, dabplus=tx.dabplus, first=s, count=1)
    fibs, msc, status = [[] for _ in range(S)], [[] for _ in range(S)], [[] for _ in range(S)]
    for _ in range(steps):
        out = c.process(iq_dev, stride, np.zeros(S, np.int64), buf_len, msc_stride=flen)
        r = out["results"]
        for s in range(S):
            status[s].append(int(r["status"][s]))
            if r["status"][s] == pkg.FRAME_DECODED and r["next_pos"][s] <= buf_len:
                fibs[s].append((out["fibs"][s].tobytes(), int(r["fib_crc_mask"][s])))
                for k in range(4 - int(r["n_logical"][s][0]), 4):
                    msc[s].append((len(fibs[s]) - 1, out["msc"][s, 0, k, :3 * txs[s].bitrate].tobytes()))
    return fibs, msc, status


def aligned(a, b, least):
    """the shift d such that a[i] == b[i + d] over their whole overlap, which holds at least `least` entries; None if there is none"""
    for d in range(-len(a) + least, len(b) - least + 1):
        lo, hi = max(0, -d), min(len(a), len(b) - d)
        if hi - lo >= least and all(a[i] == b[i + d] for i in range(lo, hi)):
            return d
    return None


def first_tracking(fibs):
    """the first decoded frame whose 12 FIB CRCs all pass (the frequency correctors have converged)"""
    return next((i for i, (_, crc) in enumerate(fibs) if crc == 0xFFF), len(fibs))


def tracking(fibs):
    return fibs[first_tracking(fibs):]


def settled_logical(fibs, msc):
    """the logical frames of the frames from 6 after the first tracking one on: the time de-interleaver's 16 CIFs of history hold only
    tracked frames, and the fine frequency corrector has settled"""
    k = first_tracking(fibs) + 6
    return [b for f, b in msc if f >= k]


@pytest.mark.parametrize("R,fmt,offsets", [
    (10000000, 0, [-3424000, -1712000, 0, 1712000, 3424000]),
    (2400000, 1, [100000]),
    (8192000, 2, [-1712000, 0, 1712000]),
], ids=["10Msps-cf32-5", "2.4Msps-u8-mistuned", "8.192Msps-s8-3"])
def test_closed_loop(R, fmt, offsets):
    pkg = load_pkg()
    S = len(offsets)
    sigs = ensembles(S, seed=R % 977)
    txs = [tx for tx, _ in sigs]
    gains = [0.0] * S
    if S > 1:
        gains[S // 2] = 20.0
    x = quantize(wideband(sigs, R, offsets, gains, snr_db=24.0, seed=R % 31), fmt)
    L, M, T = chanref.geometry(R)
    n_in = x.shape[1] if fmt == 0 else x.shape[1] // chanref.BYTES[fmt]
    # the recording is input [0, n_in), behind T samples of silence at [-T, 0) so that output 0 has its whole span
    silence = np.full((1, T * chanref.BYTES[fmt]), 128 if fmt == 1 else 0, np.uint8)
    xb = np.concatenate([silence.view(x.dtype), x], axis=1)
    out_len = (n_in - 1) * L // M + 1
    c = pkg.Context(n_streams=S)
    try:
        ch = pkg.Channelizer(c, R, offsets, iq_format=fmt)
        d = ch.run(xb, [-T], n_in + T, 0, out_len)
        c.sync()
        # the device output on this recording, two stretches of 3000 outputs per channel, against the definition
        y = d.download(np.complex64).reshape(S, out_len)
        xc = chanref.convert(xb[0], fmt)
        for m0 in (0, out_len // 2):
            for s in range(S):
                want = chanref.channelize(xc, -T, R, offsets[s], m0, 3000)
                rms, mx = chanref.error_ratio(y[s, m0:m0 + 3000], want)
                assert rms <= RMS_BOUND and mx <= MAX_BOUND, (s, m0, rms, mx)
        wide = decode(pkg, c, txs, d, out_len, out_len)
        ch.destroy()
        d.free()
    finally:
        c.close()
    n = max(len(s_) for _, s_ in sigs)
    c = pkg.Context(n_streams=S)
    try:
        d = c.dev(np.stack([np.pad(s_, (0, n - len(s_))) for _, s_ in sigs]).astype(np.complex64))
        own = decode(pkg, c, txs, d, n, n)
        d.free()
    finally:
        c.close()
    for s in range(S):
        print(f"stream {s} at {offsets[s]} Hz: status {wide[2][s]} crc {[hex(c_) for _, c_ in wide[0][s]]}, {len(wide[1][s])} logical frames; "
              f"own signal: status {own[2][s]} crc {[hex(c_) for _, c_ in own[0][s]]}, {len(own[1][s])}")
    for s in range(S):
        fw, fo = tracking(wide[0][s]), tracking(own[0][s])
        assert len(fw) >= FRAMES - 10 and all(crc == 0xFFF for _, crc in fw), (s, [hex(c_) for _, c_ in wide[0][s]])
        assert aligned([f for f, _ in fw], [f for f, _ in fo], FRAMES - 10) is not None, f"stream {s}: FIBs differ from the ensemble's own decode"
        assert aligned(settled_logical(wide[0][s], wide[1][s]), settled_logical(own[0][s], own[1][s]), 16) is not None, \
            f"stream {s}: logical frames differ from the ensemble's own decode"


def test_channelizer_leaves_the_context_as_it_was():
    """a context that created, ran and destroyed a channelizer decodes a 2.048 Msps batch with the same launches, kernels and bytes as
    a context that never did"""
    pkg = load_pkg()
    txs = [dabtx.DabTx(seed=0xE0 + i) for i in range(2)]
    iq = np.stack([dabtx.add_awgn(tx.frames(8), 20.0, seed=i) for i, tx in enumerate(txs)])
    runs = []
    for with_chan in (False, True):
        c = pkg.Context(n_streams=2)
        try:
            if with_chan:
                ch = pkg.Channelizer(c, 10000000, [0, 1712000])
                first, end = ch.input_range(0, 50000)
                o = ch.run(noise(np.random.default_rng(0), (1, end - first)), [first], end - first, 0, 50000)
                c.sync()
                o.free()
                ch.destroy()
            d = c.dev(iq)
            c.profile(True)
            l0 = c.kernel_launches()
            outs = [c.process(d, iq.shape[1], np.zeros(2, np.int64), iq.shape[1], msc_stride=288) for _ in range(8)]
            launches = c.kernel_launches() - l0
            kernels = sorted(c.profile_read().keys())
            d.free()
            runs.append((launches, kernels, [(o_["results"].tobytes(), o_["fibs"].tobytes(), o_["msc"].tobytes()) for o_ in outs]))
        finally:
            c.close()
    assert runs[0][0] == runs[1][0] and runs[0][1] == runs[1][1]
    assert "chan_kernel" not in runs[1][1]
    assert runs[0][2] == runs[1][2]
