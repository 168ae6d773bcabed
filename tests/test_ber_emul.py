"""The channel bit-error count of the device (welle.io_b200/csrc/ber_core.cuh, with the library's profile tables from tables.cpp) compiled
as host code (tests/host_emul/emul_ber.cpp), against a numpy restatement of the definition in include/dab_b200.h that shares nothing with
it: the decoded bits are the output bytes unpacked MSB first XOR the PRBS (dabtx.prbs), re-encoded with dabtx.conv_encode, punctured
with plainref.puncture_mask; softbit k is compared with transmitted position k, 0 is an erasure, s > 0 decides 1.  Every count is an
exact integer.  Also: the struct sizes of the ABI, and the `.ber` file batch_decode --ber writes, on the test double of the ABI with
tap 10 (tests/mock_backend/mock_dab_b200_ber.c)."""
import ctypes as C
import functools
import os
import subprocess

import numpy as np
import pytest

import dabtx
import plainref as P
from conftest import ROOT

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_ber") / "libemul_ber.so")
    subprocess.check_call([os.environ.get("NVCC", "nvcc"), "-O2", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-x", "cu", "-shared", "-Xcompiler", "-fPIC",
                           "-o", so, os.path.join(HERE, "host_emul", "emul_ber.cpp")])
    return C.CDLL(so)


@functools.lru_cache(maxsize=None)
def _prbs(n):
    return dabtx.prbs(n)


def ref_counts(soft, out, blocks, nbits):
    """the definition: (bits, errors, erasures) of one codeword"""
    mask = P.puncture_mask(blocks)
    n = int(mask.sum())
    u = np.unpackbits(np.asarray(out, np.uint8)[:nbits // 8]) ^ _prbs(nbits)
    code = dabtx.conv_encode(u)[mask]
    s = np.asarray(soft, np.int8)[:n].astype(np.int16)
    era = s == 0
    err = ((s > 0).astype(np.uint8) != code) & ~era
    return n, int(err.sum()), int(era.sum())


def profiles(oracle):
    """(name, blocks, nbits, emul arguments): the FIC, every EEP-A / EEP-B level (8 kbit/s 2-A and the largest profile of each level
    included, up to EEP 4-B 1824 kbit/s), and every UEP table entry"""
    from oracle.bind import ProtT
    out = [("fic", P.FIC_BLOCKS, 768, (1, 0, 0, 0, 0, 0))]
    for pa in (1, 0):
        for lv in (1, 2, 3, 4):
            brs = {b for b in (8, 16, 32, 48, 64, 96, 128, 192, 256, 384, 512, 1024) if P.eep_fits(b, pa, lv)} | {P.eep_largest(pa, lv)}
            out += [(f"{'ab'[1 - pa]}{b}/{lv}", P.eep_blocks(b, pa, lv), 24 * b, (0, b, 0, 0, pa, lv)) for b in sorted(brs)]
    for br in (32, 48, 56, 64, 80, 96, 112, 128, 160, 192, 224, 256, 320, 384):
        for lv in (1, 2, 3, 4, 5):
            p = ProtT()
            if oracle.lib.orc_prot_uep(br, lv, C.byref(p)) != 0:
                continue
            blocks = [(p.L[k], p.PI[k]) for k in range(p.nblk) if p.L[k]]
            if sum(L for L, _ in blocks) * 32 == 24 * br:
                out.append((f"u{br}/{lv}", blocks, 24 * br, (0, br, 1, lv, 0, 0)))
    return out


def test_profile_list(oracle):
    names = [p[0] for p in profiles(oracle)]
    assert "a8/2" in names and "b1824/4" in names and "a1728/4" in names
    assert sum(n.startswith("u") for n in names) == 64           # every row of the UEP table


def _cases(rng, blocks, nbits, pitch):
    """rows of (soft [pitch], out [nbits / 8], expected (errors, erasures) or None = compare with the definition only)"""
    mask = P.puncture_mask(blocks)
    n = int(mask.sum())
    rows = []

    def coded(u):
        return dabtx.conv_encode(u)[mask]

    def frame(code, tail_fill):
        s = np.empty(pitch, np.int8)
        s[:n] = np.where(code == 1, 127, -127)
        s[n:] = tail_fill                                        # past the profile's length: never counted
        return s

    def out_of(u):
        return np.packbits(u ^ _prbs(nbits))

    u = rng.integers(0, 2, nbits).astype(np.uint8)
    c = coded(u)
    junk = rng.integers(-128, 128, pitch - n).astype(np.int8)
    rows.append((frame(c, junk), out_of(u), (0, 0)))                                     # clean
    k = int(rng.integers(1, max(2, n // 50)))
    s = frame(c, junk); pos = rng.choice(n, k, replace=False); s[pos] = -s[pos]
    rows.append((s, out_of(u), (k, 0)))                                                  # k flips
    s = frame(c, junk); z = rng.choice(n, k, replace=False); s[z] = 0
    rows.append((s, out_of(u), (0, k)))                                                  # k erasures
    s = frame(c, junk); s[:n][c == 0] = -128; ones = np.flatnonzero(c == 1); m = min(len(ones), k); s[rng.choice(ones, m, replace=False)] = -128
    rows.append((s, out_of(u), (m, 0)))                                                  # -128 decides 0
    s = frame(c, junk); s[pos] = -s[pos]; s[z] = 0
    rows.append((s, out_of(u), (int(len(np.setdiff1d(pos, z))), k)))                    # flips and erasures, overlapping
    rows.append((frame(c, junk), out_of(rng.integers(0, 2, nbits).astype(np.uint8)), None))      # decoded bits that were not sent
    rows.append((rng.integers(-128, 128, pitch).astype(np.int8), out_of(u), None))      # random softbits
    s = rng.choice(np.array([-3, -1, 0, 1, 2], np.int8), pitch)
    rows.append((s, rng.integers(0, 256, nbits // 8).astype(np.uint8), None))          # small values, erasures everywhere
    return rows


def test_counts_equal_the_definition(emul, oracle):
    rng = np.random.default_rng(20261017)
    checked = 0
    for name, blocks, nbits, args in profiles(oracle):
        n = int(P.puncture_mask(blocks).sum())
        pitch = (n + 64 + 15) // 16 * 16
        rows = _cases(rng, blocks, nbits, pitch)
        soft = np.ascontiguousarray(np.stack([r[0] for r in rows]))
        out = np.ascontiguousarray(np.stack([r[1] for r in rows]))
        counts = np.zeros((len(rows), 3), np.int32)
        got = emul.emul_ber_count(*args, soft.ctypes.data_as(C.c_void_p), pitch, out.ctypes.data_as(C.c_void_p), out.shape[1], len(rows),
                                  counts.ctypes.data_as(C.c_void_p))
        assert got == n, (name, got, n)
        for i, (s, o, want) in enumerate(rows):
            ref = ref_counts(s, o, blocks, nbits)
            assert tuple(counts[i]) == ref, (name, i, tuple(counts[i]), ref)
            if want is not None:
                assert ref == (n,) + want, (name, i, ref, want)
            checked += 1
    assert checked >= 8 * 100


def test_struct_sizes(emul, pkg):
    """dabb_ber_result is 80 bytes; the option takes a reserved word, so no other struct of the ABI changes size"""
    sz = np.zeros(5, np.int32)
    emul.emul_ber_sizes(sz.ctypes.data_as(C.c_void_p))
    assert sz.tolist() == [32, 80, 64, 36, 224]
    d = pkg.dabb200
    assert C.sizeof(d.Options) == 32 and d.BER_DTYPE.itemsize == 80
    assert [f[0] for f in d.Options._fields_] == ["disable_coarse", "fft_placement", "freqsync_method", "decode_tii", "count_bit_errors", "reserved"]
    assert d.Options.count_bit_errors.offset == 16 and d.Options.reserved.offset == 20


def test_batch_decode_ber_file_on_mock_backend(oracle, tmp_path):
    """batch_decode --ber writes one line of seven integers per decoded frame; the test double serves the transmitted bit counts (4 x 2304
    FIC bits, n_logical x the profile's bits in slot 0) and no errors"""
    exe = os.path.join(ROOT, "welle.io_b200", "batch_decode")
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "welle.io_b200", "host")])
    mock = tmp_path / "libdab_b200.so"
    subprocess.check_call(["gcc", "-O1", "-shared", "-fPIC", "-o", str(mock), os.path.join(ROOT, "tests", "mock_backend", "mock_dab_b200_ber.c"),
                           "-L" + os.path.join(ROOT, "oracle"), "-loracle", "-Wl,-rpath," + os.path.join(ROOT, "oracle")])
    specs = [dict(seed=0x51, bitrate=96, profile_a=True, level=3), dict(seed=0x52, bitrate=64, profile_a=False, level=2)]
    files = []
    for k, sp in enumerate(specs):
        f = tmp_path / f"rec{k}.iq"
        np.concatenate([np.zeros(173 * k, np.complex64), dabtx.DabTx(**sp).frames(10)]).tofile(f)
        files.append(str(f))
    outdir = tmp_path / "out"; outdir.mkdir()
    env = dict(os.environ, LD_LIBRARY_PATH=str(tmp_path), DABB_MOCK_IQ=":".join(files))
    run = subprocess.run([exe, "--ber", "--out", str(outdir)] + files, capture_output=True, text=True, timeout=600, env=env)
    assert run.returncode == 0, run.stderr
    for k, sp in enumerate(specs):
        lines = (outdir / f"rec{k}.iq.ber").read_text().splitlines()
        frames = int(run.stdout.splitlines()[k].split("frames=")[1].split()[0])
        assert len(lines) == frames >= 8
        rec = np.array([[int(x) for x in ln.split()] for ln in lines])
        assert rec.shape[1] == 7
        assert (rec[:, 0] == 4 * 2304).all() and (rec[:, 1:3] == 0).all()
        in_bits = dabtx.eep_cu(sp["bitrate"], sp["profile_a"], sp["level"]) * 64
        assert rec[:, 3].sum() == len(np.fromfile(outdir / f"rec{k}.iq.msc", np.uint8)) // (3 * sp["bitrate"]) > 0
        assert (rec[:, 4] == rec[:, 3] * in_bits).all() and (rec[:, 5:] == 0).all()
