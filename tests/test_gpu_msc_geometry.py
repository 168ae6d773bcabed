"""The sub-channel chain (msc_collect_kernel -> msc_gather_kernel -> grouped viterbi_kernel -> superframe_kernel) across the whole MSC:
sub-channels at CU 0, ending at CU 863 and at odd starts, from 4 to 864 CUs, EEP-A and EEP-B up to 1728 / 1824 kbit/s, DAB+ at every
RS width from 1 to 64 columns, UEP, all four slots, and noise that makes the RS decoder both correct and fail.

Every logical frame is compared with the oracle's time de-interleaver, de-puncturing, Viterbi and dispersal applied to the softbits
the GPU produced for the stream (tap 0) - exact, whatever the fine corrector did (DESIGN.md 5(i)).  A clean stream's frames must also
be a run of what its transmitter sent; a DAB+ stream's RS events and superframes must equal the oracle's superframe filter fed the same
logical frames.  The stage entry point dabb_msc_decode is checked on the profiles of tests/test_msc_profiles_wide.py, and the
Viterbi kernel on the adversarial input families at the longest trellis the MSC has (43 776 bits, EEP 4-B 1824 kbit/s)."""
import time

import numpy as np
import pytest

import dabtx
import plainref as P
from conftest import load_pkg
from test_gpu_decoder_limits import _place

pytestmark = pytest.mark.gpu
E_ARG = -3
FRAMES = 9
MSC = 3 * 1824            # the longest logical frame
SF = 5 * MSC


@pytest.fixture(scope="module", autouse=True)
def _timer():
    t0 = time.time()
    yield
    print(f"\n{__name__}: {time.time() - t0:.1f} s")


@pytest.fixture(scope="module")
def ctx():
    c = load_pkg().Context(n_streams=1)
    yield c
    c.close()


def _prot(oracle, sel):
    if sel.get("short_form"):
        return oracle.prot_uep(sel["bitrate"], sel["uep_level"])
    return oracle.prot_eep(sel["bitrate"], int(sel["eep_profile_a"]), sel["eep_level"])


# ------------------------------------------------------------------------------------------------ stage level
def test_msc_decode_wide_profiles(ctx, oracle):
    """dabb_msc_decode on two codewords of every profile of plainref.eep_wide_profiles() (200 kbit/s up to EEP 4-A 1728 and EEP 4-B
    1824, both sides of 682 kbit/s): == oracle de-puncturing + Viterbi + dispersal"""
    t0 = time.time()
    rng = np.random.default_rng(682)
    for pa, br, lv in P.eep_wide_profiles():
        cu = dabtx.eep_cu(br, bool(pa), lv)
        sel = dict(bitrate=br, eep_profile_a=bool(pa), eep_level=lv)
        prot = _prot(oracle, sel)
        soft = rng.integers(-128, 128, (2, cu * 64)).astype(np.int8)
        out = ctx.msc_decode(soft, cu, br, eep_profile_a=bool(pa), eep_level=lv)
        for r in range(2):
            exp = oracle.pack_bits(oracle.msc_deconvolve(prot, np.maximum(soft[r, :prot.in_bits], -127), True))
            bad = np.flatnonzero(out[r] != exp)
            assert bad.size == 0, f"EEP {lv}-{'A' if pa else 'B'} {br} kbit/s, codeword {r}: {bad.size} bytes differ, the first at {bad[0]}"
    print(f"\n{len(P.eep_wide_profiles())} profiles: {time.time() - t0:.1f} s")


def test_viterbi_families_longest_trellis(ctx, oracle):
    """the adversarial families of plainref.viterbi_families at 43 776 bits, punctured with the EEP 4-B 1824 kbit/s map, in threads 0, 31,
    32, 127 of a CTA and in the partial last CTA, random codewords around them: == plain 64-bit Viterbi (the 16-bit metric margin of
    DESIGN 3.2 does not depend on the length) == oracle"""
    t0 = time.time()
    br, pa, lv = 1824, 0, 4
    nbits, cu = 24 * br, dabtx.eep_cu(br, False, lv)
    blocks = P.eep_blocks(br, pa, lv)
    mask = P.puncture_mask(blocks); n_in = int(mask.sum())
    fam = P.viterbi_families(nbits); names = list(fam)
    frags = np.stack([fam[k][mask] for k in names])
    plain, _ = P.viterbi_plain(P.depuncture(frags, blocks), nbits)
    exp = P.pack(P.dedisperse(plain))
    prot = oracle.prot_eep(br, pa, lv)
    n_cw = 130
    soft = np.random.default_rng(43776).integers(-128, 128, (n_cw, cu * 64)).astype(np.int8)
    where = _place(n_cw, len(names), 0)
    for r, k in where.items():
        soft[r, :n_in] = frags[k]
    out = ctx.msc_decode(soft, cu, br, eep_profile_a=False, eep_level=lv)
    for r, k in where.items():
        assert np.array_equal(out[r], exp[k]), f"{names[k]} in row {r}: {int((out[r] != exp[k]).sum())} bytes differ from the plain decoder"
    for r in range(n_cw):
        assert np.array_equal(out[r], oracle.pack_bits(oracle.msc_deconvolve(prot, np.maximum(soft[r, :n_in], -127), True))), r
    print(f"\nfamilies at {nbits} bits: {time.time() - t0:.1f} s")


# ------------------------------------------------------------------------------------------------ decode step
def _eep(br, pa, lv, start, dp=True):
    return dict(start_cu=start, length_cu=dabtx.eep_cu(br, bool(pa), lv), bitrate=br, eep_profile_a=bool(pa), eep_level=lv, dabplus=bool(dp))


UEP_384_1 = dict(start_cu=864 - 416, length_cu=416, bitrate=384, short_form=True, uep_level=1, dabplus=False)


def _stream_list():
    """[(transmitter kwargs, {slot: select kwargs}, SNR in dB or None)]: the transmitted sub-channel is the selection whose geometry
    equals the transmitter's; any other selection reads capacity units the transmitter fills with random bits"""
    out = []

    def own(br, pa, lv, start, dp=True, slot=0, snr=None):
        out.append((dict(bitrate=br, profile_a=bool(pa), level=lv, start_cu=start, dabplus=dp), {slot: _eep(br, pa, lv, start, dp)}, snr))
    # position: CU 0, ending at CU 863, odd starts; the smallest sub-channels (4 CUs at CU 860, the 8 kbit/s EEP 2-A special case)
    own(96, 1, 3, 0); own(96, 1, 3, 864 - 72); own(64, 0, 2, 1); own(256, 1, 3, 333); own(160, 0, 4, 511)
    own(8, 1, 4, 860); own(8, 1, 2, 511); own(224, 0, 3, 511); own(40, 1, 1, 803); own(56, 1, 2, 807)
    # the whole MSC and other large sub-channels (DAB content)
    own(1152, 1, 3, 0, False); own(1728, 1, 4, 0, False); own(1824, 0, 4, 864 - 855, False); own(1024, 0, 1, 0, False)
    own(576, 1, 1, 0, False); own(1312, 0, 2, 3, False); own(1344, 0, 3, 108, False); own(880, 1, 3, 1, False); own(1016, 1, 4, 355, False)
    # either side of 682 kbit/s
    own(680, 1, 2, 184, False); own(688, 1, 2, 0, False); own(680, 1, 4, 1, False); own(688, 1, 4, 864 - 344, False)
    own(672, 0, 2, 333, False); own(704, 0, 3, 1, False); own(672, 0, 4, 511, False); own(704, 0, 4, 864 - 330, False)
    # DAB+ at 1, 3, 4, 6, 12, 24, 37, 40, 48 and 64 RS columns
    own(8, 1, 1, 333); own(24, 1, 3, 864 - 18); own(32, 0, 4, 1); own(48, 1, 2, 700); own(96, 0, 1, 864 - 81); own(192, 1, 4, 511)
    own(296, 1, 3, 1); own(320, 0, 2, 333); own(384, 1, 2, 864 - 384); own(384, 0, 1, 1); own(512, 1, 3, 333)
    # UEP 384 kbit/s level 1 ending at CU 863, on random fill
    out.append((dict(start_cu=0), {0: UEP_384_1}, None))
    # a stream's only sub-channel in slot 1, 2 or 3
    own(128, 1, 3, 200, slot=1); own(64, 1, 1, 600, slot=2); own(320, 1, 4, 700, slot=3)
    # one stream in all four slots; slots 0 and 1 cover the same capacity units with different profiles
    out.append((dict(bitrate=96, profile_a=True, level=3, start_cu=300, dabplus=True),
                {0: _eep(96, 1, 3, 300), 1: dict(_eep(128, 1, 4, 300, False), length_cu=72),
                 2: dict(start_cu=0, length_cu=48, bitrate=64, short_form=True, uep_level=3, dabplus=False), 3: _eep(1152, 1, 3, 0, False)}, None))
    # noise: the RS decoder corrects columns and fails on some
    for k, snr in enumerate((6.0, 6.5, 7.0, 7.5)):
        own(192, 1, 4, 100 + 37 * k, snr=snr)
    return out


@pytest.fixture(scope="module")
def signals():
    """the transmitters and their FRAMES frames, built once"""
    t0 = time.time()
    txs, sigs = [], []
    for i, (kw, _, snr) in enumerate(_stream_list()):
        tx = dabtx.DabTx(seed=0x6E0 + i, **kw)
        s = tx.frames(FRAMES)
        if snr is not None:
            s = dabtx.add_awgn(s, snr, seed=0x6F0 + i, signal_power=float(np.mean(np.abs(s[3000:190000]) ** 2)))
        txs.append(tx); sigs.append(s)
    print(f"\n{len(sigs)} transmitters: {time.time() - t0:.1f} s")
    return txs, np.stack(sigs)


def _run(pkg, sigs, selections, max_cu=864, n_slots=4, taps=False):
    """one context, every (stream, slot, select kwargs) selected before the first step -> per-step outputs (and MSC softbits)"""
    S, n = sigs.shape
    c = pkg.Context(n_streams=S, max_subch_cu=max_cu, n_subch_slots=n_slots)
    d = c.dev(sigs)
    for s, slot, sel in selections:
        c.select_subchannel(first=s, count=1, slot=slot, **sel)
    outs, soft = [], []
    for _ in range(FRAMES):
        outs.append(c.process(d, n, np.zeros(S, np.int64), n, msc_stride=MSC, sf_stride=SF))
        if taps:
            soft.append(c.read_tap(0)[:, 3:75].copy())          # the 72 MSC symbols: 4 CIFs of 18
    d.free(); c.close()
    return outs, soft


def _frames_of(pkg, outs, soft, s, slot, sel):
    """(the stream's logical frames of the slot, its MSC softbits of the sub-channel per CIF since selection, RS events, superframes)"""
    flen = 3 * sel["bitrate"]
    a, b = 64 * sel["start_cu"], 64 * (sel["start_cu"] + sel["length_cu"])
    got, cifs, rs, sfs = [], [], [], []
    for o, sb in zip(outs, soft):
        r = o["results"][s]
        if r["status"] != pkg.FRAME_DECODED:
            continue
        cifs += [sb[s, 18 * c:18 * c + 18].reshape(-1)[a:b] for c in range(4)]
        got += [o["msc"][s, slot, c, :flen].copy() for c in range(4 - int(r["n_logical"][slot]), 4)]
        rs += [((int(r["rs_uncorr_mask"][slot]) >> e) & 1, int(r["rs_corr"][slot][e])) for e in range(int(r["n_rs_events"][slot]))]
        if r["sf_ready"][slot]:
            sfs.append((o["sf"][s, slot, :5 * flen].copy(), int(r["sf_au_count"][slot]), int(r["sf_au_crc_mask"][slot])))
    return got, cifs, rs, sfs


def test_decode_step_across_the_msc(oracle, signals):
    """one context (max_subch_cu = 864, four slots), one stream per geometry of _stream_list; every stream and slot against the oracle's
    chain on the GPU's own softbits, clean transmitted sub-channels against their transmitter, DAB+ against the oracle's superframe
    filter and RS decoder"""
    t0 = time.time()
    pkg = load_pkg()
    txs, sigs = signals
    streams = _stream_list()
    sel = [(s, slot, kw) for s, (_, sl, _) in enumerate(streams) for slot, kw in sl.items()]
    outs, soft = _run(pkg, sigs, sel, taps=True)
    t_gpu = time.time() - t0
    noisy_corr = noisy_fail = 0
    n_sf = 0
    for s, slot, kw in sel:
        txkw, _, snr = streams[s]
        what = f"stream {s} slot {slot}: {kw}"
        got, cifs, rs, sfs = _frames_of(pkg, outs, soft, s, slot, kw)
        prot = _prot(oracle, kw)
        de = oracle.deinterleave(np.stack(cifs))
        exp = [oracle.pack_bits(oracle.msc_deconvolve(prot, x[:prot.in_bits], True)) for x in de]
        assert len(got) == len(exp) >= 8, (what, len(got), len(exp))
        for k, (x, y) in enumerate(zip(got, exp)):
            bad = np.flatnonzero(x != y)
            assert bad.size == 0, f"{what}: logical frame {k}, {bad.size} bytes differ from the oracle, the first at {bad[0]}"
        own = "bitrate" in txkw and _eep(txkw["bitrate"], txkw["profile_a"], txkw["level"], txkw["start_cu"], txkw["dabplus"]) == kw
        if own and snr is None:        # a run of what was transmitted
            flen = 3 * kw["bitrate"]
            lf = np.concatenate(txs[s].logical); g = np.concatenate(got)
            hits = [k for k in range(len(txs[s].logical)) if np.array_equal(g[:flen], lf[k * flen:(k + 1) * flen])]
            assert hits and np.array_equal(g, lf[hits[0] * flen:hits[0] * flen + len(g)]), what
        if kw["dabplus"]:
            ev, osfs = oracle.superframe_filter(np.stack(got))
            assert rs == [(e["uncorr"], e["corr"]) for e in ev], (what, rs, ev)
            synced = [e for e in ev if e["sync"]]
            assert len(sfs) == len(synced) == len(osfs), what
            for (x, na, m), e, y in zip(sfs, synced, osfs):
                assert np.array_equal(x, y) and (na, m) == (e["num_aus"], e["au_ok"]), what
            if own and snr is None:
                assert sfs and all(m == 0x3F and na == 6 for _, na, m in sfs), what
                assert all(any(np.array_equal(x, t) for t in txs[s].superframes) for x, _, _ in sfs), what
            n_sf += len(sfs)
            if snr is not None:
                noisy_corr += sum(c for _, c in rs); noisy_fail += sum(u for u, _ in rs)
    assert noisy_corr > 0 and noisy_fail > 0, (noisy_corr, noisy_fail)
    print(f"\n{len(streams)} streams, {len(sel)} sub-channels, {n_sf} superframes, noisy streams: {noisy_corr} bytes corrected, {noisy_fail} "
          f"superframes uncorrectable; GPU {t_gpu:.1f} s, checks {time.time() - t0 - t_gpu:.1f} s")


def _same(x, y, what):
    assert x["results"].tobytes() == y["results"].tobytes(), what
    assert np.array_equal(x["msc"], y["msc"]) and np.array_equal(x["sf"], y["sf"]), what


def test_refused_geometries_leave_the_context_unchanged(signals):
    """a sub-channel ending at CU 865, one of length 0, one longer than max_subch_cu, and a profile that needs more bits than its
    sub-channel holds: DABB_E_ARG, no launch, and every later step byte-identical to a twin context that never saw the calls"""
    pkg = load_pkg()
    _, sigs = signals
    sig = sigs[:2]                          # 96 kbit/s EEP 3-A at CU 0 and at CU 792
    S, n = sig.shape
    keeper = pkg.Context(n_streams=1)
    d = keeper.dev(sig)

    def make():
        c = pkg.Context(n_streams=S, max_subch_cu=144, n_subch_slots=2)
        c.select_subchannel(first=0, count=1, **_eep(96, 1, 3, 0))
        c.select_subchannel(first=1, count=1, **_eep(96, 1, 3, 864 - 72))
        return c
    a, b = make(), make()
    run = lambda c: c.process(d, n, np.zeros(S, np.int64), n, msc_stride=MSC, sf_stride=SF)
    for _ in range(3):
        _same(run(a), run(b), "before")
    refused = [dict(_eep(64, 1, 3, 864 - 64), length_cu=65),            # start_cu + length_cu = 865
               dict(_eep(96, 1, 3, 0), length_cu=0),
               dict(_eep(96, 1, 3, 0), length_cu=145),                  # > max_subch_cu
               dict(_eep(96, 1, 3, 10), length_cu=71)]                  # 72 CUs of punctured bits
    for kw in refused:
        for slot in (0, 1):
            launches = a.kernel_launches()
            with pytest.raises(Exception) as e:
                a.select_subchannel(first=slot, count=1, slot=slot, **kw)
            assert f"error {E_ARG}:" in str(e.value), (kw, str(e.value))
            assert a.kernel_launches() == launches, kw
    logical = 0
    for k in range(3, FRAMES):
        x, y = run(a), run(b)
        _same(x, y, f"step {k}")
        logical += int(x["results"]["n_logical"][:, 0].sum())
    assert logical > 0
    a.close(); b.close(); keeper.close()


def test_max_subch_cu_above_the_msc_is_864(signals):
    """a context created with max_subch_cu = 4000 decodes the 864-CU EEP 4-A 1728 kbit/s sub-channel exactly like one created with 864"""
    pkg = load_pkg()
    txs, sigs = signals
    s = next(i for i, (kw, _, _) in enumerate(_stream_list()) if kw.get("bitrate") == 1728)
    sig = sigs[s:s + 1]
    sel = [(0, 0, _eep(1728, 1, 4, 0, False))]
    a, _ = _run(pkg, sig, sel, max_cu=4000, n_slots=1)
    b, _ = _run(pkg, sig, sel, max_cu=864, n_slots=1)
    for k, (x, y) in enumerate(zip(a, b)):
        _same(x, y, f"step {k}")
    assert sum(int(o["results"]["n_logical"][0, 0]) for o in a) >= 8
