"""EEP sub-channels above 192 kbit/s, up to the largest the 864 CUs of the MSC hold (EEP 4-A 1728 kbit/s, EEP 4-B 1824 kbit/s), on the
CPU: the energy-dispersal words the library builds for every profile (tables.cpp, compiled for the host) against the plain PRBS and
the oracle's, and the oracle's de-puncturing + Viterbi + dispersal against the unmodified reference (live where oracle/_ref is built,
else its answers stored in tests/golden/eep_wide_v1.npz) and against the plain wide-integer Viterbi.  The reference keeps a frame's
length in 16 bits and cannot decode above 1365 kbit/s; there the plain Viterbi is the second answer.
tests/test_gpu_msc_geometry.py runs the same profiles through the kernels."""
import ctypes as C
import hashlib
import importlib.util
import os
import subprocess

import numpy as np
import pytest

import dabtx
import plainref as P

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def tables(tmp_path_factory):
    # the library's table builders are host code in a CUDA translation unit: nvcc compiles them, no device is involved
    so = str(tmp_path_factory.mktemp("emul") / "libemul_tables.so")
    subprocess.check_call([os.environ.get("NVCC", "nvcc"), "-O2", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-x", "cu", "-shared", "-Xcompiler", "-fPIC",
                           "-o", so, os.path.join(HERE, "host_emul", "emul_tables.cpp")])
    return C.CDLL(so)


def _eep_bitrates():
    """every bitrate of an EEP-A (multiple of 8 kbit/s) or EEP-B (multiple of 32) profile whose sub-channel fits in the MSC"""
    return sorted({b for pa in (1, 0) for lv in (1, 2, 3, 4) for b in range(8, 2048, 8) if P.eep_fits(b, pa, lv)})


def test_dispersal_words_every_eep_bitrate(tables, oracle):
    """the words add_profile and dabb_msc_decode hand to the decoder, for every EEP bitrate up to 1824 kbit/s (43 776 bits) ==
    the plain PRBS x^9 + x^5 + 1 packed the same way == the oracle's orc_dedisperse"""
    brs = _eep_bitrates()
    assert brs[-1] == 1824 and 1728 in brs and len(brs) == 216 + 3       # multiples of 8 up to 1728, then 1760, 1792, 1824
    plain = P.pack(P.dedisperse(np.zeros(24 * brs[-1], np.uint8)))
    orc = np.zeros(24 * brs[-1], np.uint8)
    oracle.lib.orc_dedisperse(orc.ctypes.data_as(C.c_void_p), len(orc))
    assert np.array_equal(plain, oracle.pack_bits(orc))
    for br in brs:
        nbits = 24 * br
        w = np.full((nbits + 31) // 32 + 4, 0xA5A5A5A5, np.uint32)
        assert tables.emul_prot_prbs_words(br, w.ctypes.data_as(C.c_void_p)) == nbits // 32, br
        got = w[:nbits // 32].view(np.uint8)
        bad = np.flatnonzero(got != plain[:nbits // 8])
        assert bad.size == 0, f"{br} kbit/s: {bad.size} dispersal bytes wrong, the first at byte {bad[0]}"
        assert (w[nbits // 32:] == 0xA5A5A5A5).all(), br


def _prot(oracle, pa, br, lv):
    p = oracle.prot_eep(br, pa, lv)
    assert p.in_bits == int(P.puncture_mask(P.eep_blocks(br, pa, lv)).sum()), (pa, br, lv)
    return p


def test_wide_profile_list():
    prof = P.eep_wide_profiles()
    for pa, lv, top in ((1, 1, 576), (1, 2, 864), (1, 3, 1152), (1, 4, 1728), (0, 1, 1024), (0, 2, 1312), (0, 3, 1536), (0, 4, 1824)):
        assert P.eep_largest(pa, lv) == top and (pa, top, lv) in prof
    assert all((pa, br, 4) in prof for pa, br in P.EEP_BOUNDARY)
    assert len(prof) == len(set(prof)) and min(br for _, br, _ in prof) == 200


def _stored():
    spec = importlib.util.spec_from_file_location("make_eep_wide", os.path.join(HERE, "golden", "make_eep_wide.py"))
    mod = importlib.util.module_from_spec(spec); spec.loader.exec_module(mod)
    return mod


def test_oracle_equals_reference_above_192(oracle):
    """oracle de-puncturing + Viterbi + dispersal == the reference's EEPProtection::deconvolve + EnergyDispersal on seeded random
    softbits, EEP-A and EEP-B from 200 kbit/s to 1365 kbit/s: live where the reference is built, else its stored answers"""
    from oracle.bind import Ref
    g = _stored()
    with np.load(g.PATH, allow_pickle=False) as z:
        stored = {k: z[k] for k in z.files}
    live = Ref() if Ref.available() else None
    cases = [p for p in P.eep_wide_profiles() if P.ref_decodes(p[1])]
    assert [tuple(int(x) for x in r) for r in stored["profile"]] == cases
    for i, (pa, br, lv) in enumerate(cases):
        soft = P.eep_wide_soft(pa, br, lv)
        assert hashlib.sha256(soft.tobytes()).digest() == stored["input_sha256"][i].tobytes(), f"{(pa, br, lv)}: the case generator changed"
        mine = oracle.msc_deconvolve(_prot(oracle, pa, br, lv), soft, True)
        if live is not None:
            assert np.array_equal(mine, live.eep_deconvolve(br, pa, lv, soft, True)), (pa, br, lv)
        assert hashlib.sha256(np.packbits(mine).tobytes()).digest() == stored["output_sha256"][i].tobytes(), (pa, br, lv)


def test_eep_wide_reference_answers_are_current():
    """where the reference build exists, its live answers equal the stored ones"""
    from oracle.bind import Ref
    if not Ref.available():
        pytest.skip("live reference not built")
    g = _stored()
    with np.load(g.PATH, allow_pickle=False) as z:
        stored = {k: z[k] for k in z.files}
    live = g.record(Ref())
    assert sorted(live) == sorted(stored)
    for k in stored:
        assert np.array_equal(live[k], stored[k]), k


def test_oracle_equals_plain_viterbi_largest_profiles(oracle):
    """the largest profile of every (A/B, level), and every profile the reference cannot decode: oracle == plain de-puncturing + 64-bit
    never-renormalised Viterbi + dispersal, on the seeded softbits and on a clean codeword with every seventh step inverted"""
    largest = {(pa, P.eep_largest(pa, lv), lv) for pa in (1, 0) for lv in (1, 2, 3, 4)}
    cases = sorted(largest | {p for p in P.eep_wide_profiles() if not P.ref_decodes(p[1])})
    assert len(cases) == 8 + 5
    rng = np.random.default_rng(17)
    for pa, br, lv in cases:
        nbits = 24 * br
        blocks = P.eep_blocks(br, pa, lv)
        mask = P.puncture_mask(blocks)
        cw = ((2 * dabtx.conv_encode(rng.integers(0, 2, nbits).astype(np.uint8)).astype(np.int16) - 1) * 127).astype(np.int8).reshape(-1, 4)
        cw[::7] = -cw[::7]
        frags = np.stack([P.eep_wide_soft(pa, br, lv), cw.reshape(-1)[mask]])
        bits, _ = P.viterbi_plain(P.depuncture(frags, blocks), nbits)
        prot = _prot(oracle, pa, br, lv)
        for k in range(2):
            assert np.array_equal(oracle.msc_deconvolve(prot, frags[k], True), P.dedisperse(bits[k])), (pa, br, lv, k)


@pytest.mark.parametrize("br, pa, lv, start, dabplus", [(1728, 1, 4, 0, False), (1824, 0, 4, 9, False), (512, 1, 3, 480, True)])
def test_closed_loop_large_subchannels(oracle, br, pa, lv, start, dabplus):
    """the oracle's closed-loop receiver on the transmitter's largest sub-channels - the whole MSC with DAB content, DAB+ at 64 RS
    columns ending at CU 863 - gives back a run of the transmitted logical frames, and the DAB+ superframes synchronise with nothing to
    correct and every AU CRC good"""
    tx = dabtx.DabTx(seed=br, bitrate=br, profile_a=bool(pa), level=lv, start_cu=start, dabplus=dabplus)
    o = oracle.rx_run(tx.frames(7), prot=oracle.prot_eep(br, pa, lv), start_cu=start, len_cu=dabtx.eep_cu(br, bool(pa), lv), dabplus=dabplus,
                      select_after_frames=0)
    flen = 3 * br
    g = o["msc"]; lf = np.concatenate(tx.logical)
    assert len(g) >= 8 * flen
    hits = [k for k in range(len(tx.logical)) if np.array_equal(g[:flen], lf[k * flen:(k + 1) * flen])]
    assert hits and np.array_equal(g, lf[hits[0] * flen:hits[0] * flen + len(g)])
    if dabplus:
        ev, sfs = oracle.superframe_filter(g.reshape(-1, flen))
        assert sfs and all(e["num_aus"] == 6 and e["au_ok"] == 0x3F for e in ev if e["sync"])
        assert all((e["corr"], e["uncorr"]) == (0, 0) for e in ev if e["sync"])
        assert all(any(np.array_equal(x, t) for t in tx.superframes) for x in sfs)
