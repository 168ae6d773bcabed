"""The Viterbi and Reed-Solomon decoders at their arithmetic limits, on the CPU: the per-thread code of the kernels (viterbi_core.cuh
compiled as plain C++, tests/host_emul) and the oracle against the plain wide-integer references of
tests/plainref.py, on inputs chosen to break a packed 16-bit decoder (ties, pinned symbols, the largest metric spread, patterns aligned
with the register layouts and the 24-step stage) instead of random ones; and the superframe builder, the RS syndrome check and the
oracle's superframe handling for all four DAB+ audio formats, with the unmodified reference's stored answers
(tests/golden/sf_formats_v1.npz).  tests/test_gpu_decoder_limits.py runs the same inputs through the kernels."""
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
NBITS = (192, 768, 2304, 9216)           # 9216 = 24 x 384, the longest MSC codeword


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    d = tmp_path_factory.mktemp("emul")
    libs = {}
    for name in ("emul_viterbi", "emul_vitdec"):
        so = str(d / f"lib{name}.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "host_emul", name + ".cpp")])
        libs[name] = C.CDLL(so)
    # the library's table builders are host code in a CUDA translation unit: nvcc compiles them, no device is involved
    so = str(d / "libemul_tables.so")
    subprocess.check_call([os.environ.get("NVCC", "nvcc"), "-O2", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-x", "cu", "-shared", "-Xcompiler", "-fPIC",
                           "-o", so, os.path.join(HERE, "host_emul", "emul_tables.cpp")])
    libs["emul_tables"] = C.CDLL(so)
    return libs


def _stack(fam):
    names = list(fam)
    return names, np.stack([fam[k] for k in names])


def test_viterbi_families_packed_equals_plain_equals_oracle(emul, oracle):
    """packed 16-bit add-compare-select (emul_viterbi) == 64-bit never-renormalised Viterbi == oracle on every family and length.
    No input ties every decision: an erased softbit is symbol 127, which costs 127 for a 0 and 128 for a 1 (the reference's symbol
    scale has no midpoint), so even the all-zero codeword prefers a branch in most butterflies; the `ties` family reaches the most ties
    a constant input gives, a quarter of all decisions."""
    worst = (0, None); most_tied = 0.0
    for nbits in NBITS:
        names, soft = _stack(P.viterbi_families(nbits))
        bits, st = P.viterbi_plain(soft, nbits)
        for i, name in enumerate(names):
            out = np.zeros(nbits, np.uint8)
            emul["emul_viterbi"].emul_viterbi(nbits, soft[i].ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p))
            assert np.array_equal(out, bits[i]), f"packed != plain: {name} at {nbits} bits, {int((out != bits[i]).sum())} bits differ"
            assert np.array_equal(oracle.viterbi(soft[i], nbits), bits[i]), f"oracle != plain: {name} at {nbits} bits"
        k = int(st["peak24"].argmax())
        worst = max(worst, (int(st["peak24"][k]), f"{names[k]} at {nbits} bits: spread {int(st['spread'][k])}, 24-step growth {int(st['growth24'][k])}"))
        most_tied = max(most_tied, float(st["tied"].max()))
        assert int((st["spread"] + st["growth24"]).max()) < 32767
    assert most_tied > 0.2, most_tied
    # the largest candidate metric a decoder that subtracts the minimum every 24 steps has to hold, of the 32767 a signed half offers
    assert 12000 < worst[0] < 32767, worst


def _profiles(oracle):
    """(name, [(L, PI)], nbits, arguments of emul_prot_map): FIC, EEP-A / EEP-B and UEP profiles from 8 to 384 kbit/s, where the profile exists"""
    from oracle.bind import ProtT
    out = [("fic", P.FIC_BLOCKS, 768, (1, 0, 0, 0, 0, 0))]
    for kind, br, lvl in (("a", 8, 1), ("a", 96, 3), ("a", 192, 4), ("a", 384, 1), ("b", 32, 1), ("b", 192, 4), ("u", 32, 5), ("u", 192, 2), ("u", 384, 5)):
        p = ProtT()
        rc = oracle.lib.orc_prot_uep(br, lvl, C.byref(p)) if kind == "u" else oracle.lib.orc_prot_eep(br, int(kind == "a"), lvl, C.byref(p))
        blocks = [(p.L[k], p.PI[k]) for k in range(p.nblk) if p.L[k]]
        if rc == 0 and sum(L for L, _ in blocks) * 32 == 24 * br:
            out.append((f"{kind}{br}/{lvl}", blocks, 24 * br, (0, br, 1, lvl, 0, 0) if kind == "u" else (0, br, 0, 0, int(kind == "a"), lvl)))
    return out


def test_profiles_exist(oracle):
    assert [p[0] for p in _profiles(oracle)] == ["fic", "a8/1", "a96/3", "a192/4", "a384/1", "b32/1", "b192/4", "u32/5", "u192/2", "u384/5"]


@pytest.mark.parametrize("variant", ["one_thread"])
def test_decoder_emulation_families_as_fragments(emul, oracle, variant):
    """one thread of the decoder kernel - expansion tables, 8-byte window, packed ACS, 24-step traceback, de-dispersal,
    packing - on the families as PUNCTURED fragments: output bytes == pack(dedisperse(viterbi_plain(depuncture(fragment)))).  The
    fragment starts on a 16-byte boundary, ends on one, or ends one byte behind one; random bytes follow it.  (-128 is not an input of
    this code: the stage entry points map it to -127 first, which tests/test_gpu_decoder_limits.py covers.)  The de-puncturing map is the
    one the library builds for the profile (tables.cpp), and must mark exactly the softbits the puncturing vectors transmit - also for
    EEP 1-A at 384 kbit/s, whose 36 864 softbits per codeword do not fit a 16-bit index."""
    fn = emul["emul_vitdec"].emul_vitdec
    rng = np.random.default_rng(31)
    for pname, blocks, nbits, args in _profiles(oracle):
        mask = P.puncture_mask(blocks); n_in = int(mask.sum())
        m16 = np.zeros(mask.size, np.int16)
        assert emul["emul_tables"].emul_prot_map(*args, m16.ctypes.data_as(C.c_void_p)) == n_in, pname
        assert np.array_equal(m16 >= 0, mask), (pname, int((m16 >= 0).sum()), n_in)
        fam = P.viterbi_families(nbits); del fam["m128"]
        names, full = _stack(fam)
        frags = full[:, mask]
        bits, _ = P.viterbi_plain(P.depuncture(frags, blocks), nbits)
        exp = P.pack(P.dedisperse(bits))
        prbs_words = np.ascontiguousarray(P.pack(dabtx.prbs(nbits))).view(np.uint32)
        for i, name in enumerate(names):
            for place in ("start_aligned", "end_aligned", "end_plus_1"):
                raw = rng.integers(-127, 128, n_in + 32 + 192).astype(np.int8)
                want = {"start_aligned": 0, "end_aligned": -n_in, "end_plus_1": 1 - n_in}[place]
                off = (want - raw.ctypes.data) % 16
                raw[off:off + n_in] = frags[i]
                out = np.zeros(nbits // 8, np.uint8)
                rc = fn(C.c_void_p(raw.ctypes.data + off), m16.ctypes.data_as(C.c_void_p), nbits, prbs_words.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p))
                assert rc == 0 and np.array_equal(out, exp[i]), (pname, name, place, rc, int((out != exp[i]).sum()))


# ------------------------------------------------------------------------------------------------ superframes
def test_superframe_builder_equals_transmitter():
    """for dac_rate = 1, sbr_flag = 0 (6 AUs) the builder is byte-identical to dabtx.DabTx.superframe on the same payload"""
    for br in (8, 32, 96, 192):
        for bad in (None, 0, 5):
            sf, truth = P.build_superframe(np.random.default_rng(br), br, 1, 0, bad_au=bad)
            assert np.array_equal(sf, dabtx.DabTx(seed=br, bitrate=br).superframe(bad_au=bad))
            assert truth["num_aus"] == 6 and P.rs_check(P.columns(sf))
    sf, _ = P.build_superframe(np.random.default_rng(1), 96, 1, 0, au_lens=[17, 300, 2, 33, 500])
    assert np.array_equal(sf, dabtx.DabTx(seed=1).superframe(au_starts=11 + np.cumsum([17, 300, 2, 33, 500])))


def test_rs_check_against_encoder_and_oracle(oracle):
    rng = np.random.default_rng(2)
    for _ in range(20):
        d = rng.integers(0, 256, 110).astype(np.uint8)
        cw = P.rs_encode_column(d)
        assert np.array_equal(cw[110:], oracle.rs_encode(d)) and P.rs_check(cw)
        for pos in (0, 57, 109, 110, 119):
            bad = cw.copy(); bad[pos] ^= 1 + int(rng.integers(255))
            assert not P.rs_check(bad)


def _oracle_sf(oracle, sf):
    ev, _ = oracle.superframe_filter(sf.reshape(5, -1))
    assert len(ev) == 1
    return ev[0]


def test_superframe_formats_oracle_equals_builder(oracle):
    """2, 3, 4 and 6 AUs per superframe at 1 .. 64 RS columns, clean and with one AU's CRC broken: the oracle's header parse and AU
    CRCs equal the builder's truth"""
    seen = set()
    for name, sf, truth in P.sf_format_cases():
        assert P.rs_check(P.columns(sf)), name
        e = _oracle_sf(oracle, sf)
        assert (e["sync"], e["num_aus"], e["au_ok"], e["corr"], e["uncorr"]) == (1, truth["num_aus"], truth["au_mask"], 0, 0), (name, e, truth)
        seen.add((len(sf) // 120, truth["num_aus"]))
    assert len(seen) == 32


def test_superframe_controlled_errors_oracle(oracle):
    """<= 5 byte errors in a column: the oracle restores the superframe that was built and counts the bytes changed; 6 and 10: the
    column is reported uncorrectable and no column that still checks differs from what was sent"""
    for name, rx, sent, truth, per_col in P.sf_error_cases():
        S = len(rx) // 120
        assert [int(x) for x in (P.columns(rx) != P.columns(sent)).sum(1)] == per_col, name
        out, corr, unc = oracle.rs_decode_superframe(rx)
        e = _oracle_sf(oracle, rx)
        assert (e["corr"], e["uncorr"]) == (corr, unc)
        good = [c for c in range(S) if per_col[c] <= 5]
        assert np.array_equal(P.columns(out)[good], P.columns(sent)[good]), name
        if len(good) == S:
            assert (corr, unc) == (sum(per_col), 0), (name, corr, unc)
            assert (e["sync"], e["num_aus"], e["au_ok"]) == (1, truth["num_aus"], truth["au_mask"]), (name, e)
        else:
            assert unc == 1, name


def test_superframe_rejections_oracle(oracle):
    for name, sf in P.sf_reject_cases():
        assert P.rs_check(P.columns(sf)), name
        e = _oracle_sf(oracle, sf)
        assert (e["sync"], e["corr"], e["uncorr"]) == (0, 0, 0), (name, e)


def _golden():
    spec = importlib.util.spec_from_file_location("make_sf_formats", os.path.join(HERE, "golden", "make_sf_formats.py"))
    mod = importlib.util.module_from_spec(spec); spec.loader.exec_module(mod)
    return mod


def test_superframe_cases_oracle_equals_reference_answers(oracle):
    """what the unmodified reference (RSDecoder::DecodeSuperframe, SuperframeFilter) answered for every superframe of the three case lists,
    stored in tests/golden/sf_formats_v1.npz: the oracle gives the same corrected bytes, counts and number of failed AU CRCs"""
    g = _golden()
    with np.load(g.PATH, allow_pickle=False) as z:
        stored = {k: z[k] for k in z.files}
    cases = P.sf_all_inputs()
    assert [n.decode() for n in stored["name"]] == [c[0] for c in cases]
    for i, (name, sf) in enumerate(cases):
        assert hashlib.sha256(sf.tobytes()).digest() == stored["input_sha256"][i].tobytes(), f"{name}: the case generator changed"
        out, corr, unc = oracle.rs_decode_superframe(sf)
        e = _oracle_sf(oracle, sf)
        au_err = e["num_aus"] - bin(e["au_ok"]).count("1") if e["sync"] else 0
        mine = (hashlib.sha256(out.tobytes()).digest(), corr, unc, e["uncorr"], e["corr"], au_err)
        theirs = (stored["output_sha256"][i].tobytes(), stored["rs_corr"][i], stored["rs_uncorr"][i], stored["fec_uncorr"][i], stored["fec_corr"][i], stored["au_errors"][i])
        assert mine == theirs, (name, mine[1:], theirs[1:])


def test_superframe_reference_answers_are_current():
    """where the reference build exists, its live answers equal the stored ones"""
    from oracle.bind import Ref
    if not Ref.available():
        pytest.skip("live reference not built")
    g = _golden()
    with np.load(g.PATH, allow_pickle=False) as z:
        stored = {k: z[k] for k in z.files}
    live = g.record(Ref())
    assert sorted(live) == sorted(stored)
    for k in stored:
        assert np.array_equal(live[k], stored[k]), k
