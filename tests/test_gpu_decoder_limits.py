"""The Viterbi and Reed-Solomon kernels at their arithmetic limits, through the stateless stage entry points of the C ABI: the
adversarial input families and superframe case lists of tests/plainref.py (the ones tests/test_decoder_limits.py runs through the CPU
emulation) against the plain wide-integer references, the builder's truth and the oracle.  What the emulation cannot see is what
this file adds: the cp.async staging, the decision words' round trip through memory, clamp_copy_kernel (-128 goes in unclamped),
the traceback prefetch, partial CTAs, and all of rs.cu."""
import ctypes as C

import numpy as np
import pytest

import dabtx
import plainref as P
from conftest import load_pkg
from test_decoder_limits import _profiles

pytestmark = pytest.mark.gpu
E_ARG, E_UNSUPPORTED = -3, -6


@pytest.fixture(scope="module")
def ctx():
    c = load_pkg().Context(n_streams=1)
    yield c
    c.close()


def _place(n_rows, n_fam, shift):
    """rows of a batch that get an adversarial input: threads 0, 31, 32, 127 of every CTA of 128 codewords and the last row (the
    partial CTA), then the rows behind them, `shift` rotating which family lands where"""
    first = [r for r in range(n_rows) if r % 128 in (0, 31, 32, 127) or r == n_rows - 1]
    rest = [r for r in range(n_rows) if r not in first]
    rows = (first + rest)[:n_fam]
    return {r: (k + shift) % n_fam for k, r in enumerate(rows)}


@pytest.mark.parametrize("nbits", [192, 768, 2304, 9216])
def test_viterbi_families(ctx, oracle, nbits):
    fams = P.viterbi_families(nbits); names = list(fams)
    fam = np.stack([fams[k] for k in names])
    plain, _ = P.viterbi_plain(fam, nbits)
    rng = np.random.default_rng(nbits)
    for shift, n_cw in enumerate((1, 127, 128, 129, 300)):
        soft = rng.integers(-128, 128, (n_cw, (nbits + 6) * 4)).astype(np.int8)
        where = _place(n_cw, len(names), 5 * shift)
        for r, k in where.items():
            soft[r] = fam[k]
        out = ctx.viterbi(soft, nbits)
        for r, k in where.items():
            assert np.array_equal(out[r], plain[k]), f"{names[k]} in row {r} of {n_cw}, {nbits} bits: {int((out[r] != plain[k]).sum())} bits differ from the plain decoder"
        for r in range(n_cw):
            assert np.array_equal(out[r], oracle.viterbi(soft[r], nbits)), f"row {r} of {n_cw}, {nbits} bits"


def test_fic_decode_families(ctx, oracle):
    """the 768-bit families as punctured FIC codewords (four per 9216-softbit block), -128 included, and one valid FIC block: FIBs and CRC
    mask == plain de-puncturing + plain Viterbi + de-dispersal + packing + CRC"""
    mask = P.puncture_mask(P.FIC_BLOCKS)
    fam = P.viterbi_families(768); names = list(fam)
    frags = np.stack([fam[k][mask] for k in names] + [fam["zeros"][mask]] * (-len(names) % 4))
    tx = dabtx.DabTx(seed=3)
    valid = np.tile((tx.ficblk.astype(np.int16) * 254 - 127).astype(np.int8), 4)
    soft = np.concatenate([frags.reshape(-1, 9216), valid[None]])
    fibs, crc = ctx.fic_decode(soft)
    bits, _ = P.viterbi_plain(P.depuncture(soft.reshape(-1, 2304), P.FIC_BLOCKS), 768)
    exp = P.pack(P.dedisperse(bits)).reshape(-1, 12, 32)
    for f in range(len(soft)):
        assert np.array_equal(fibs[f], exp[f]), f"FIC block {f}"
        assert crc[f] == sum(int(P.fib_crc_ok(exp[f, k])) << k for k in range(12)), f
        fb, ok = oracle.fic_decode(soft[f])
        assert np.array_equal(fibs[f], np.packbits(fb, axis=1)) and crc[f] == sum(int(o) << k for k, o in enumerate(ok)), f
    assert crc[-1] == 0xFFF and np.array_equal(fibs[-1, 0], dabtx.fib_bytes(tx))


@pytest.mark.parametrize("n_cifs", [1, 130])
def test_msc_decode_families(ctx, oracle, n_cifs):
    """the families as punctured fragments of EEP-A / EEP-B / UEP sub-channels from 8 to 384 kbit/s (EEP 1-A at 384 kbit/s: 36 864
    softbits per codeword), one CIF and a batch that ends in a partial CTA"""
    from oracle.bind import ProtT
    for pi, (pname, blocks, nbits, args) in enumerate(_profiles(oracle)[1:]):
        _, br, short_form, uep_level, eep_a, eep_level = args
        mask = P.puncture_mask(blocks); n_in = int(mask.sum()); cu = (n_in + 63) // 64
        fam = P.viterbi_families(nbits); names = list(fam)
        rng = np.random.default_rng(100 * n_cifs + pi)
        soft = rng.integers(-128, 128, (n_cifs, cu * 64)).astype(np.int8)
        where = _place(n_cifs, len(names), pi) if n_cifs > 1 else {0: (7 * pi) % len(names)}
        for r, k in where.items():
            soft[r, :n_in] = fam[names[k]][mask]
        out = ctx.msc_decode(soft, cu, br, eep_profile_a=bool(eep_a), eep_level=eep_level, short_form=bool(short_form), uep_level=uep_level)
        rows = sorted(where)
        bits, _ = P.viterbi_plain(P.depuncture(soft[rows, :n_in], blocks), nbits)
        exp = P.pack(P.dedisperse(bits))
        for j, r in enumerate(rows):
            assert np.array_equal(out[r], exp[j]), f"{pname}: {names[where[r]]} in row {r} of {n_cifs} differs from the plain decoder"
        prot = ProtT()
        assert (oracle.lib.orc_prot_uep(br, uep_level, C.byref(prot)) if short_form else oracle.lib.orc_prot_eep(br, eep_a, eep_level, C.byref(prot))) == 0
        for r in range(n_cifs):
            clamped = np.maximum(soft[r, :n_in], -127)       # both are symbol 0; the oracle's de-puncturing is not asked about -128
            assert np.array_equal(out[r], oracle.pack_bits(oracle.msc_deconvolve(prot, clamped, True))), (pname, r)


def _oracle_sf(oracle, sf):
    ev, _ = oracle.superframe_filter(sf.reshape(5, -1))
    return ev[0]


def _run_by_width(ctx, cases):
    """one dabb_rs_superframes call per superframe length -> {name: (corrected superframe, info row)}"""
    res = {}
    for n in sorted({len(c[1]) for c in cases}):
        group = [c for c in cases if len(c[1]) == n]
        out, info = ctx.rs_superframes(np.stack([c[1] for c in group]))
        for k, c in enumerate(group):
            res[c[0]] = (out[k], info[k])
    return res


def test_rs_superframe_formats(ctx, oracle):
    """2, 3, 4 and 6 AUs at S = 1, 2, 3, 5, 12, 17, 24 and 64 columns, clean and with one AU's CRC broken: sync, AU count and AU mask ==
    the builder's truth == oracle, superframe untouched, nothing corrected"""
    cases = P.sf_format_cases()
    res = _run_by_width(ctx, cases)
    for name, sf, truth in cases:
        out, info = res[name]
        assert np.array_equal(out, sf), name
        assert tuple(info) == (0, 0, 1, truth["au_mask"] | truth["num_aus"] << 8), (name, info, truth)
        e = _oracle_sf(oracle, sf)
        assert (e["sync"], e["num_aus"], e["au_ok"]) == (1, info[3] >> 8, info[3] & 0xFF), name


def test_rs_superframe_controlled_errors(ctx, oracle):
    """exactly 1 .. 5 byte errors in one column, 5 in every column, 5 in the parity rows, 5 in the header bytes (the Fire code passes only
    after correction): every column with <= 5 errors comes back as it was built and `corr` counts the bytes changed - no decoder
    needed to know that.  6 and 10 errors in a column: output, corr and uncorr == oracle (what an uncorrectable word does to the
    bytes is defined by the reference's step sequence)."""
    cases = P.sf_error_cases()
    res = _run_by_width(ctx, cases)
    for name, rx, sent, truth, per_col in cases:
        out, info = res[name]
        S = len(rx) // 120
        good = [c for c in range(S) if per_col[c] <= 5]
        assert np.array_equal(P.columns(out)[good], P.columns(sent)[good]), name
        if len(good) == S:
            assert tuple(info) == (sum(per_col), 0, 1, truth["au_mask"] | truth["num_aus"] << 8), (name, info)
        o_sf, corr, unc = oracle.rs_decode_superframe(rx)
        e = _oracle_sf(oracle, rx)
        assert np.array_equal(out, o_sf) and (info[0], info[1], info[2]) == (corr, unc, e["sync"]), (name, info, corr, unc, e)
        if e["sync"]:
            assert (info[3] >> 8, info[3] & 0xFF) == (e["num_aus"], e["au_ok"]), name


def test_rs_superframe_rejections(ctx, oracle):
    """valid RS columns, but a zero first AU address, any one bit of the Fire code flipped, AU addresses equal / decreasing / at or beyond
    the end of the data: no synchronisation, nothing corrected"""
    cases = P.sf_reject_cases()
    res = _run_by_width(ctx, cases)
    for name, sf in cases:
        out, info = res[name]
        assert np.array_equal(out, sf) and (info[0], info[1], info[2]) == (0, 0, 0), (name, info)
        assert _oracle_sf(oracle, sf)["sync"] == 0, name


def test_argument_checks_return_before_any_launch(ctx):
    """lengths the host-side checks refuse: only return codes are looked at"""
    lib, h = ctx.lib, ctx.h
    buf = ctx.dev(120 * 65); info = ctx.dev(64)
    for sf_len in (0, 119, 121):
        assert lib.dabb_rs_superframes(h, C.c_void_p(buf.ptr), 1, sf_len, C.c_void_p(info.ptr)) == E_ARG, sf_len
    assert lib.dabb_rs_superframes(h, C.c_void_p(buf.ptr), 1, 120 * 65, C.c_void_p(info.ptr)) == E_UNSUPPORTED
    for nbits in (0, 100, 64):
        assert lib.dabb_viterbi(h, C.c_void_p(buf.ptr), 1, nbits, C.c_void_p(info.ptr)) == E_ARG, nbits
    buf.free(); info.free()
