"""GPU parity tests, stage level: every CUDA stage through the C ABI against the CPU oracle on the same seeded inputs.
Bar: bit-exact for integer/byte work; the float OFDM stage is bit-exact too in DABB_FFT_EXACT mode (and within 1e-4
relative in DABB_FFT_FMA mode)."""
import numpy as np
import pytest

import dabtx
from conftest import load_pkg

pytestmark = pytest.mark.gpu
TU, TS, TF, TNULL, TG, K = 2048, 2552, 196608, 2656, 504, 1536


@pytest.fixture(scope="module")
def ctx():
    pkg = load_pkg()
    c = pkg.Context(n_streams=4, keep_taps=True)
    yield c
    c.close()


@pytest.fixture(scope="module")
def iq12():
    tx = dabtx.DabTx(seed=0xDAB)
    return tx, tx.frames(6)


def test_ofdm_demod_bit_exact(ctx, oracle, iq12):
    tx, iq = iq12
    frames = np.stack([iq[f * TF: (f + 1) * TF + 4096] for f in range(1, 5)])
    prs = np.full(4, TNULL + 305, np.int64)          # the reference's steady-state window (SURVEY §9)
    soft, r1, fc = ctx.ofdm_demod(frames, prs, want_r1=True, want_fc=True)
    for f in range(4):
        st = TNULL + 305
        s_o, r_o = oracle.demod_frame(frames[f, st: st + TU], frames[f, st + TU: st + TU + 75 * TS], True)
        assert np.array_equal(soft[f], s_o), f"softbits differ in frame {f}: {(soft[f] != s_o).sum()}"
        assert np.array_equal(r1[f].view(np.uint32), r_o.view(np.uint32)), "pre-quantisation products not bit-equal"
        # CP correlation: float sum in a different order -> relative tolerance
        x = frames[f, st + TU: st + TU + 75 * TS].reshape(75, TS).astype(np.complex128)
        ref = (x[:, TU:] * np.conj(x[:, :TG])).sum()
        assert abs(fc[f] - ref) <= 1e-4 * abs(ref)


def test_ofdm_demod_fma_mode_within_tolerance(oracle, iq12):
    pkg = load_pkg()
    c = pkg.Context(n_streams=1, fft_mode=pkg.FFT_FMA)
    tx, iq = iq12
    frames = np.stack([iq[TF: 2 * TF + 4096]])
    soft, r1 = c.ofdm_demod(frames, np.array([TNULL + 305], np.int64), want_r1=True)
    st = TNULL + 305
    s_o, r_o = oracle.demod_frame(frames[0, st: st + TU], frames[0, st + TU: st + TU + 75 * TS], True)
    rel = np.abs(r1[0] - r_o) / np.abs(r_o)
    assert rel.max() <= 1e-4          # north_star tolerance for soft-decision intermediates
    assert np.array_equal(np.sign(soft[0]), np.sign(s_o)) or (np.sign(soft[0]) != np.sign(s_o)).mean() < 1e-4
    assert np.abs(soft[0].astype(int) - s_o.astype(int)).max() <= 1
    c.close()


def test_ofdm_demod_with_nco(ctx, oracle, iq12):
    tx, iq = iq12
    shifted = dabtx.freq_shift(iq, 1234.0)
    frames = np.stack([shifted[TF: 2 * TF + 4096]])
    st = TNULL + 305
    lp0, ph = 777, 1234
    nco = np.array([[lp0, ph]], np.int32)
    soft = ctx.ofdm_demod(frames, np.array([st], np.int64), nco=nco)
    # oracle: mix on the CPU exactly like OFDMProcessor::getSamples, then demod
    n = np.arange(TU + 75 * TS, dtype=np.int64)
    lp = (lp0 - n * ph) % 2048000
    osc = (np.cos(2.0 * np.pi * lp / 2048000).astype(np.float32) + 1j * np.sin(2.0 * np.pi * lp / 2048000).astype(np.float32)).astype(np.complex64)
    x = frames[0, st: st + TU + 75 * TS]
    re = (x.real * osc.real).astype(np.float32) - (x.imag * osc.imag).astype(np.float32)
    im = (x.real * osc.imag).astype(np.float32) + (x.imag * osc.real).astype(np.float32)
    mixed = (re + 1j * im).astype(np.complex64)
    s_o = oracle.demod_frame(mixed[:TU], mixed[TU:])
    assert np.array_equal(soft[0], s_o)
    fibs, crc = oracle.fic_decode(s_o[:3].reshape(-1))
    assert crc.all()


def test_find_index(ctx, oracle, iq12):
    tx, iq = iq12
    starts = np.array([TNULL - 199, TNULL - 100, TNULL - 400, TNULL + 3000], np.int64)   # last one: no PRS inside -> -1 or garbage-consistent
    frames = np.stack([iq[2 * TF: 3 * TF]] * 4)
    idx, cir = ctx.find_index(frames, starts, want_cir=True)
    for i, s in enumerate(starts):
        i_o, c_o = oracle.find_index(frames[i, s: s + TU])
        assert idx[i] == i_o, (i, idx[i], i_o)
        assert np.array_equal(cir[i].view(np.uint32), c_o.view(np.uint32)), f"CIR not bit-equal ({np.abs(cir[i]-c_o).max()})"
    assert idx[0] == 504


def test_find_index_threshold_search_many_windows(oracle, iq12):
    """ThresholdBeforePeak over the whole range of peak positions (window starts swept over more than a symbol, so the correlation peak
    lands everywhere incl. the first 200 and the last samples, and outside: no synchronisation), on clean, noisy, pre-echo and
    noise-only input.  The library's warp-per-window search (no sliding maximum: DESIGN.md 3) must equal the oracle's index for every
    window."""
    from conftest import load_pkg
    pkg = load_pkg()
    tx, iq = iq12
    rng = np.random.default_rng(77)
    base = iq[2 * TF: 3 * TF]
    variants = [base, dabtx.add_awgn(iq, 3.0, seed=5)[2 * TF: 3 * TF], (base + 0.8 * np.roll(base, -150)).astype(np.complex64),
                (base * 0.02 + (rng.standard_normal(TF) + 1j * rng.standard_normal(TF)) * 0.05).astype(np.complex64)]
    frames = []
    for v, sig in enumerate(variants):
        for d in range(-260, 2300, 17 + v):
            st = TNULL + 504 - d
            frames.append(sig[st: st + TU])
    frames = np.stack(frames); starts = np.zeros(len(frames), np.int64)
    exp = np.array([oracle.find_index(frames[i])[0] for i in range(len(frames))])
    assert len(set(exp.tolist())) > 100 and (exp < 0).any() and (exp < 200).any() and (exp > 1800).any()
    c = pkg.Context(n_streams=len(starts))
    idx = c.find_index(frames, starts)
    c.close()
    bad = np.nonzero(idx != exp)[0]
    assert bad.size == 0, (bad[:10], idx[bad[:10]], exp[bad[:10]])


@pytest.mark.parametrize("placement", [1, 2])
def test_find_index_other_placements(ctx, oracle, iq12, placement):
    """StrongestPeak / EarliestPeakWithBinning (phasereference.cpp:93-211): index (incl. the negative scores) and CIR bit-equal"""
    tx, iq = iq12
    rng = np.random.default_rng(placement)
    noisy = dabtx.add_awgn(iq, 3.0, seed=3)
    echo = (iq[2 * TF: 3 * TF] + 0.7 * np.roll(iq[2 * TF: 3 * TF], -180)).astype(np.complex64)       # pre-echo 180 samples early
    noise = ((rng.standard_normal(TF) + 1j * rng.standard_normal(TF)) * 0.05).astype(np.complex64)
    frames = np.stack([iq[2 * TF: 3 * TF]] * 4 + [noisy[2 * TF: 3 * TF], echo, noise, np.zeros(TF, np.complex64)])
    starts = np.array([TNULL - 199, TNULL - 100, TNULL - 700, TNULL + 3000, TNULL - 250, TNULL - 300, 1000, 0], np.int64)
    idx, cir = ctx.find_index(frames, starts, want_cir=True, placement=placement)
    for i, s in enumerate(starts):
        i_o, c_o = oracle.find_index(frames[i, s: s + TU], placement)
        assert idx[i] == i_o, (i, idx[i], i_o)
        assert np.array_equal(cir[i].view(np.uint32), c_o.view(np.uint32)), i


@pytest.mark.parametrize("method", [0, 1, 2])
def test_coarse_estimate(ctx, oracle, iq12, method):
    """OFDMProcessor::processPRS: PatternOfZeros / GetMiddle / CorrelatePRS on aligned, misaligned and noisy phase reference symbols
    at several carrier offsets.  GetMiddle is bit-exact arithmetic; the two arg()-based methods truncate atan2f results to integers
    (see oracle/dab_oracle.c), so a CUDA/glibc atan2f difference can only matter within an ulp of an integer: none may show here."""
    tx, iq = iq12
    frames, starts = [], []
    for hz in (0, 1000, 2000, -3000, 7000, -12000, 333):
        sh = dabtx.freq_shift(iq[2 * TF: 3 * TF], hz)
        for k, src in enumerate((sh, dabtx.add_awgn(sh, 6.0, seed=hz & 0xFF))):
            for d in (0, 100, 327, -200):
                frames.append(src); starts.append(TNULL + 504 - d)
    frames = np.stack(frames); starts = np.array(starts, np.int64)
    got = ctx.coarse_estimate(frames, starts, method)
    exp = np.array([oracle.coarse(frames[i, s: s + TU], method) for i, s in enumerate(starts)])
    assert np.array_equal(got, exp), np.nonzero(got != exp)


@pytest.mark.parametrize("nbits", [768, 2304, 192])
def test_viterbi_bit_exact(ctx, oracle, nbits):
    rng = np.random.default_rng(nbits)
    n = 200
    soft = rng.integers(-128, 128, (n, (nbits + 6) * 4)).astype(np.int8)
    for i in range(0, n, 2):   # half of them: real codewords with noise and punctures
        bits = rng.integers(0, 2, nbits).astype(np.uint8)
        enc = oracle.conv_encode(bits).astype(np.float32) * 2 - 1
        s = np.clip(enc * 35 + rng.standard_normal(enc.size) * 50, -127, 127).astype(np.int8)
        s[rng.random(s.size) < 0.25] = 0
        soft[i] = s
    out = ctx.viterbi(soft, nbits)
    for i in range(n):
        assert np.array_equal(out[i], oracle.viterbi(soft[i], nbits)), f"codeword {i}"


def test_fic_decode(ctx, oracle, iq12):
    tx, iq = iq12
    rng = np.random.default_rng(5)
    frames = np.stack([iq[f * TF: (f + 1) * TF + 4096] for f in range(1, 4)])
    soft = ctx.ofdm_demod(frames, np.full(3, TNULL + 305, np.int64))
    fic_soft = soft[:, :3].reshape(3, 9216).copy()
    noisy = np.clip(fic_soft.astype(int) + rng.integers(-90, 91, fic_soft.shape), -127, 127).astype(np.int8)
    allsoft = np.concatenate([fic_soft, noisy, rng.integers(-127, 128, (2, 9216)).astype(np.int8)])
    fibs, crc = ctx.fic_decode(allsoft)
    for i in range(len(allsoft)):
        fb, ok = oracle.fic_decode(allsoft[i])
        assert np.array_equal(fibs[i], np.packbits(fb, axis=1)), i
        assert crc[i] == int(sum(int(o) << k for k, o in enumerate(ok))), i
    assert crc[0] == 0xFFF and np.array_equal(fibs[0, 0], dabtx.fib_bytes(tx))


@pytest.mark.parametrize("cfg", [(96, True, 3), (64, True, 1), (8, True, 2), (32, True, 2), (128, True, 4), (32, False, 1), (96, False, 3), (128, False, 4)])
def test_msc_decode_eep(ctx, oracle, cfg):
    br, pa, lv = cfg
    rng = np.random.default_rng(br + lv)
    prot = oracle.prot_eep(br, pa, lv)
    cu = dabtx.eep_cu(br, pa, lv)
    n = 20
    soft = rng.integers(-127, 128, (n, cu * 64)).astype(np.int8)
    out = ctx.msc_decode(soft, cu, br, eep_profile_a=pa, eep_level=lv)
    for i in range(n):
        bits = oracle.msc_deconvolve(prot, soft[i, :prot.in_bits], True)
        assert np.array_equal(out[i], oracle.pack_bits(bits)), i


@pytest.mark.parametrize("cfg", [(32, 5), (48, 3), (128, 1), (192, 2), (80, 1)])
def test_msc_decode_uep(ctx, oracle, cfg):
    br, lv = cfg
    rng = np.random.default_rng(br * 7 + lv)
    prot = oracle.prot_uep(br, lv)
    cu = (prot.in_bits + 63) // 64
    soft = rng.integers(-127, 128, (8, cu * 64)).astype(np.int8)
    out = ctx.msc_decode(soft, cu, br, short_form=True, uep_level=lv)
    for i in range(8):
        bits = oracle.msc_deconvolve(prot, soft[i, :prot.in_bits], True)
        assert np.array_equal(out[i], oracle.pack_bits(bits)), i


def test_rs_superframes(ctx, oracle):
    rng = np.random.default_rng(9)
    tx = dabtx.DabTx(seed=4)
    sfs = []
    for i in range(40):
        sf = tx.superframe(bad_au=(i % 6 if i % 5 == 0 else None))
        ne = [0, 3, 20, 60, 200, 1440][i % 6]
        if ne:
            pos = rng.choice(len(sf), ne, replace=False)
            sf = sf.copy(); sf[pos] ^= rng.integers(1, 256, ne).astype(np.uint8)
        sfs.append(sf)
    sfs.append(np.zeros(1440, np.uint8))
    sfs = np.stack(sfs)
    out, info = ctx.rs_superframes(sfs)
    for i in range(len(sfs)):
        o_sf, corr, unc = oracle.rs_decode_superframe(sfs[i])
        assert np.array_equal(out[i], o_sf), i
        assert (info[i, 0], info[i, 1]) == (corr, unc), (i, info[i], corr, unc)
        ev, _ = oracle.superframe_filter(np.concatenate([sfs[i].reshape(5, -1)]))
        assert info[i, 2] == ev[0]["sync"]
        if ev[0]["sync"]:
            assert (info[i, 3] & 0xFF) == ev[0]["au_ok"] and (info[i, 3] >> 8) == ev[0]["num_aus"]


@pytest.mark.parametrize("bitrate", [32, 96, 192])
def test_rs_superframes_au_layouts(ctx, oracle, bitrate):
    """AU CRCs over odd layouts (AUs of 2, 3, 4, 17, 18, 33 bytes, AUs that are not multiples of the CRC chunk) and with single
    corrupted AUs; compared with the oracle's SuperframeFilter restatement (dabplus_decoder.cpp:122-131,171-215)"""
    rng = np.random.default_rng(bitrate)
    tx = dabtx.DabTx(seed=11, bitrate=bitrate)
    n_data = 110 * bitrate // 8
    sfs = []
    small = [2, 3, 4, 17, 18, 33, 16, 32, 19]
    for i in range(48):
        if i % 3 == 0:
            lens = [small[(i + k) % len(small)] for k in range(5)]
        else:
            room = n_data - 11 - 12
            cuts = np.sort(rng.choice(np.arange(1, room // 2), 5, replace=False)) * 2 + (i & 1)
            lens = np.diff(np.concatenate([[0], cuts])).tolist()
            lens = [max(2, int(x)) for x in lens]
        starts = 11 + np.cumsum(lens)
        if starts[-1] >= n_data - 1:
            continue
        sf = tx.superframe(bad_au=(i % 6 if i % 4 == 0 else None), au_starts=starts)
        sfs.append(sf)
    assert len(sfs) > 20
    sfs = np.stack(sfs)
    out, info = ctx.rs_superframes(sfs)
    for i in range(len(sfs)):
        ev, _ = oracle.superframe_filter(sfs[i].reshape(5, -1))
        assert info[i, 2] == ev[0]["sync"] == 1, i
        assert (info[i, 3] & 0xFF) == ev[0]["au_ok"] and (info[i, 3] >> 8) == ev[0]["num_aus"], (i, info[i], ev[0])
        assert np.array_equal(out[i], sfs[i])


def test_oscillator_on_the_fly_is_verified(ctx):
    """dabb_create compares the on-the-fly oscillator (three double-precision factors) with the reference's 2 048 000-entry float table
    for EVERY index and only then switches the table lookups off; exactly the three quarter-turn factors take the table's own value"""
    assert ctx.get_info(0) == 1 and ctx.get_info(1) == 0 and ctx.get_info(2) == 3


def test_msc_decode_every_protection_profile(ctx, oracle):
    """every UEP table entry and every EEP-A / EEP-B profile up to 192 kbit/s through dabb_msc_decode: de-puncturing maps, Viterbi,
    energy de-dispersal and byte packing bit-identical to the oracle (which matches the reference for all of them,
    tests/test_oracle_vs_ref.py::test_all_uep_profiles / test_all_eep_profiles)"""
    import ctypes as C
    from oracle.bind import ProtT
    cases = []
    for br in (32, 48, 56, 64, 80, 96, 112, 128, 160, 192, 224, 256, 320, 384):
        for lv in range(1, 6):
            p = ProtT()
            # pairs that are not in the table (56/1, 112/1, 320/1, 320/3, 384/2, 384/4) make the reference fall back to another row
            # whose block lengths do not cover the frame (uep-protection.cpp:152-155); the ABI rejects them instead
            if oracle.lib.orc_prot_uep(br, lv, C.byref(p)) == 0 and sum(p.L) * 32 == 24 * br:
                cases.append((p, br, dict(short_form=True, uep_level=lv)))
    for pa, step in ((True, 8), (False, 32)):
        for br in range(step, 193, step):
            for lv in (1, 2, 3, 4):
                cases.append((oracle.prot_eep(br, int(pa), lv), br, dict(eep_profile_a=pa, eep_level=lv)))
    assert len(cases) == 64 + 96 + 24
    for k, (prot, br, kw) in enumerate(cases):
        rng = np.random.default_rng(k)
        cu = (prot.in_bits + 63) // 64
        soft = rng.integers(-127, 128, (2, cu * 64)).astype(np.int8)
        out = ctx.msc_decode(soft, cu, br, **kw)
        for i in range(2):
            bits = oracle.msc_deconvolve(prot, soft[i, :prot.in_bits], True)
            assert np.array_equal(out[i], oracle.pack_bits(bits)), (br, kw, i)
