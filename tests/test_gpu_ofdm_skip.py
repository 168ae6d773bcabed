"""The OFDM demodulator's symbol skipping (ofdm_mask.cuh): a context without keep_taps transforms and demaps only the symbols its FIC and
sub-channels read and takes the fine-AFC terms and the level sample of every other symbol from its guard interval and window edges.
Twin contexts - keep_taps (every symbol transformed) against none (skipping) - on the same input decode byte for byte alike: every
result field (fine_corr, freq_corr_re/im, slevel, snr_raw, start_index, ...), FIBs, logical frames, superframes and tap 10.  The samples
a skipped symbol does not stage, [632, 2048) of it, are poisoned with NaN and the decode does not change."""
import numpy as np
import pytest

import dabtx
from conftest import load_pkg

pytestmark = pytest.mark.gpu
TF, TU, TS, TG, TNULL = 196608, 2048, 2552, 504, 2656
FRAMES, STEPS = 14, 12
MSC, SF = 3 * 384, 15 * 384


@pytest.fixture(scope="module")
def pkg():
    return load_pkg()


def _recording(S, stride, seed, hz=50.0, snr=14.0):
    """one noisy recording with a carrier offset; stream s reads it from sample s * stride on"""
    rec = dabtx.DabTx(seed=seed).frames((S * stride) // TF + FRAMES + 2)
    return dabtx.add_awgn(dabtx.freq_shift(rec, hz), snr, seed=seed).astype(np.complex64)


def _geometries(S):
    """per stream a list of (slot, start_cu, length_cu, bitrate): odd starts, a sub-channel ending at CU 863, slices crossing a symbol
    boundary (48 CUs per symbol), the whole MSC, two slots over the same CUs, and streams with no slot"""
    base = [[(0, 0, 72, 96)], [(0, 45, 5, 8)], [(0, 791, 72, 96), (1, 101, 12, 16)], [(0, 860, 4, 8)], [],
            [(0, 0, 864, 384)], [(0, 94, 4, 8), (2, 94, 4, 8)], [(1, 301, 35, 48), (3, 17, 48, 64)], [(0, 48, 48, 64)], [(2, 431, 96, 128)]]
    return [base[s % len(base)] for s in range(S)]


def _select(ctx, geoms):
    for s, g in enumerate(geoms):
        for slot, st, ln, br in g:
            ctx.select_subchannel(st, ln, br, eep_profile_a=True, eep_level=4, dabplus=False, slot=slot, first=s, count=1)


def _run(pkg, sig, S, stride, n, keep_taps, geoms, ctx_kw=None, opts=None, events=None, steps=STEPS):
    ctx = pkg.Context(n_streams=S, keep_taps=keep_taps, n_subch_slots=4, max_subch_cu=864, **(ctx_kw or {}))
    ctx.set_options(disable_coarse=True, **(opts or {}))
    _select(ctx, geoms)
    d = ctx.dev(sig)
    outs = []
    for k in range(steps):
        if events and k in events:
            events[k](ctx)
        o = ctx.process(d, stride, np.zeros(S, np.int64), n, msc_stride=MSC, sf_stride=SF)
        if opts and opts.get("count_bit_errors"):
            o["t10"] = ctx.read_tap(10)
        outs.append(o)
    d.free(); ctx.close()
    return outs


def _assert_same(a, b, what):
    assert len(a) == len(b)
    for k, (x, y) in enumerate(zip(a, b)):
        assert x.keys() == y.keys()
        for name in x:
            assert x[name].tobytes() == y[name].tobytes(), (what, k, name)


def _twins(pkg, S, stride, seed, ctx_kw=None, opts=None, events=None, geoms=None):
    sig = _recording(S, stride, seed)
    n = len(sig) - stride * (S - 1)
    geoms = geoms if geoms is not None else _geometries(S)
    full = _run(pkg, sig, S, stride, n, True, geoms, ctx_kw, opts, events)
    skip = _run(pkg, sig, S, stride, n, False, geoms, ctx_kw, opts, events)
    _assert_same(full, skip, (ctx_kw, opts))
    dec = sum(int((o["results"]["status"] == pkg.FRAME_DECODED).sum()) for o in skip)
    lf = sum(int(o["results"]["n_logical"].sum()) for o in skip)
    assert dec >= S * (STEPS - 3) and lf > 0, (dec, lf)
    return skip


@pytest.mark.parametrize("fft_mode", ["exact", "fma"])
@pytest.mark.parametrize("nco_mode", ["exact", "fast"])
@pytest.mark.parametrize("demap", ["reference", "weighted"])
def test_twins_every_arithmetic(pkg, fft_mode, nco_mode, demap):
    """64 streams at an odd stride (both sample alignments, their own oscillator phases), a 50 Hz carrier offset, mixed geometries"""
    kw = dict(fft_mode=pkg.FFT_EXACT if fft_mode == "exact" else pkg.FFT_FMA, nco_mode=pkg.NCO_EXACT if nco_mode == "exact" else pkg.NCO_FAST)
    opts = dict(soft_demap=pkg.DEMAP_REFERENCE if demap == "reference" else pkg.DEMAP_WEIGHTED)
    _twins(pkg, 64, 7919, 0x5C1, kw, opts)


@pytest.mark.parametrize("groups", [1, 5, 25])
def test_twins_ofdm_groups(pkg, groups):
    _twins(pkg, 64, 4001, 0x5C2, dict(ofdm_groups=groups))


def test_twins_tail_split(pkg):
    """2048 streams: one CTA per frame for most frames, five per frame for the tail"""
    _twins(pkg, 2048, 2003, 0x5C3)


def test_twins_select_and_remove_between_steps(pkg):
    """sub-channels selected, moved and removed between steps, with the bit-error count on (tap 10)"""
    S = 40

    def move(ctx):
        ctx.select_subchannel(600, 24, 32, eep_profile_a=True, eep_level=4, dabplus=False, slot=0, first=0, count=20)

    def drop(ctx):
        ctx.remove_subchannel(slot=0, first=10, count=20)
        ctx.select_subchannel(0, 864, 384, eep_profile_a=True, eep_level=4, dabplus=False, slot=3, first=30, count=5)

    _twins(pkg, S, 7919, 0x5C4, opts=dict(count_bit_errors=True), events={3: move, 7: drop})


def test_skipped_samples_are_never_read(pkg):
    """8 streams on rows of their own (both sample alignments): every sample of [632, 2048) of every symbol the stream's mask leaves
    light, in every decoded frame, set to NaN - the decode is the clean one byte for byte"""
    S = 8
    rec = dabtx.add_awgn(dabtx.DabTx(seed=0x5C5).frames(FRAMES + 1), 16.0, seed=5).astype(np.complex64)
    offs = [0, 1, 1000, 4097, 20001, 333, 65536, 99]
    n = len(rec) - max(offs)
    rows = np.stack([rec[o:o + n] for o in offs])
    geoms = _geometries(S)
    clean = _run(pkg, rows, S, n, n, False, geoms)
    full = _run(pkg, rows, S, n, n, True, geoms)
    _assert_same(full, clean, "clean")
    poisoned = rows.copy()
    nan = np.complex64(complex(np.nan, np.nan))
    n_poison = 0
    for s, g in enumerate(geoms):
        demap = np.zeros(77, bool)
        demap[1:4] = True
        for _, st, ln, _ in g:
            a, b = 64 * st // 3072, (64 * (st + ln) - 1) // 3072
            for c in range(4):
                demap[4 + 18 * c + a: 4 + 18 * c + b + 1] = True
        light = [l for l in range(1, 76) if not demap[l] and not demap[l + 1]]
        for o in clean:
            r = o["results"][s]
            if r["status"] != pkg.FRAME_DECODED:
                continue
            prs = int(r["next_pos"]) - (TU + 75 * TS + TNULL)                 # first useful sample of the phase reference symbol
            for l in light:
                s0 = prs + TU + (l - 1) * TS
                poisoned[s, s0 + TG + 128: s0 + TU] = nan
                n_poison += TU - TG - 128
    assert n_poison > 0
    got = _run(pkg, poisoned, S, n, n, False, geoms)
    _assert_same(clean, got, "poisoned")
    dec = sum(int((o["results"]["status"] == pkg.FRAME_DECODED).sum()) for o in got)
    assert dec >= S * (STEPS - 3), dec
