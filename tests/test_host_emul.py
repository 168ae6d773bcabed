"""CPU emulation of the CUDA per-thread code (the same .cuh headers compiled as plain C++): the FFT pass structure with its
shared-memory swizzle, and the packed-16-bit Viterbi with its rotating register layout, against the oracle."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "host_emul")


@pytest.fixture(scope="module")
def libs():
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-o", os.path.join(HERE, "libemul.so"), os.path.join(HERE, "emul_fft.cpp")])
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", os.path.join(HERE, "libemulv.so"), os.path.join(HERE, "emul_viterbi.cpp")])
    return C.CDLL(os.path.join(HERE, "libemul.so")), C.CDLL(os.path.join(HERE, "libemulv.so"))


def test_fft_passes_bit_exact_and_conflict_free(libs, oracle):
    rng = np.random.default_rng(3)
    for inv in (0, 1):
        x = (rng.standard_normal(2048) + 1j * rng.standard_normal(2048)).astype(np.complex64); y = np.zeros_like(x)
        worst = libs[0].emul_fft2048(x.ctypes.data_as(C.c_void_p), y.ctypes.data_as(C.c_void_p), inv)
        assert np.array_equal(y.view(np.uint32), oracle.fft(x, bool(inv)).view(np.uint32))
        assert worst == 1, "shared-memory exchange pattern has bank conflicts"


def test_packed_viterbi(libs, oracle):
    rng = np.random.default_rng(11)
    for trial in range(16):
        nb = [768, 2304, 192, 24 * 384][trial % 4]
        soft = rng.integers(-128, 128, (nb + 6) * 4).astype(np.int8)
        if trial % 2:
            bits = rng.integers(0, 2, nb).astype(np.uint8)
            soft = np.clip((oracle.conv_encode(bits).astype(np.float32) * 2 - 1) * 30 + rng.standard_normal((nb + 6) * 4) * 60, -127, 127).astype(np.int8)
            soft[rng.random(soft.size) < 0.3] = 0
        out = np.zeros(nb, np.uint8)
        libs[1].emul_viterbi(nb, soft.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p))
        assert np.array_equal(out, oracle.viterbi(soft, nb))


def test_oscillator_on_the_fly_equals_table_for_every_index():
    """the formula the device evaluates instead of reading the reference's 2 048 000-entry oscillator table (osc_factors.h), run with
    IEEE double arithmetic on the CPU: identical to the table for every index; three factors (the quarter turns) carry the table's value"""
    so = os.path.join(HERE, "libemulo.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "emul_osc.cpp")])
    lib = C.CDLL(so)
    patched = C.c_int()
    assert lib.emul_osc_mismatches(C.byref(patched)) == 0
    assert patched.value == 3


import pytest as _pytest


@_pytest.mark.parametrize("variant", ["one_thread"])
def test_decoder_kernel_emulation_depuncture_and_traceback(oracle, variant):
    """one thread of the decoder kernel (expansion tables from a de-puncturing map, 8-byte window expansion, packed ACS, 24-step
    traceback, MSB-first packing) on the CPU from the shared header code: FIC puncturing, EEP-A/B and UEP profiles, no puncturing -
    output bytes equal to oracle de-puncture + Viterbi + pack"""
    so = os.path.join(HERE, f"libemuld_{variant}.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "emul_vitdec.cpp")])
    lib = C.CDLL(so)
    rng = np.random.default_rng(21)
    pc = oracle.pcodes()

    def mapping(blocks, nbits):
        m = []
        for L, PI in blocks:
            m += [1 if pc[PI - 1][i & 31] else -1 for i in range(L * 128)]
        m += [1 if (i & 3) < 2 else -1 for i in range(24)]
        assert len(m) == 4 * (nbits + 6), (len(m), nbits)
        return np.array(m, np.int16)

    cases = [("fic", mapping([(21, 16), (3, 15)], 768), 768)]
    for (br, prof_a, lvl) in ((96, 1, 3), (64, 1, 2), (32, 0, 4), (128, 1, 1), (8, 1, 2)):
        p = oracle.prot_eep(br, prof_a, lvl)
        cases.append((f"eep{br}/{prof_a}/{lvl}", mapping([(p.L[k], p.PI[k]) for k in range(p.nblk) if p.L[k]], 24 * br), 24 * br))
    for (br, lvl) in ((64, 3), (32, 1), (192, 5)):
        p = oracle.prot_uep(br, lvl)
        cases.append((f"uep{br}/{lvl}", mapping([(p.L[k], p.PI[k]) for k in range(p.nblk) if p.L[k]], 24 * br), 24 * br))
    cases.append(("plain", np.zeros(4 * (192 + 6), np.int16), 192))
    for name, m, nbits in cases:
        n_in = int((m >= 0).sum())
        for trial in range(3):
            bits = rng.integers(0, 2, nbits).astype(np.uint8)
            enc = oracle.conv_encode(bits).astype(np.float32) * 2 - 1
            full = np.clip(enc * 40 + rng.standard_normal(len(enc)) * (20 + 30 * trial), -127, 127).astype(np.int8)
            frag = full[m >= 0]
            assert len(frag) == n_in
            depunct = np.zeros(len(m), np.int8); depunct[m >= 0] = frag
            exp = oracle.pack_bits(oracle.viterbi(depunct, nbits))
            # place the fragment at a 16-byte aligned address with slack behind it
            raw = np.zeros(n_in + 16 + 192, np.int8)
            off = (-raw.ctypes.data) % 16
            raw[off:off + n_in] = frag
            raw[off + n_in:off + n_in + 160] = rng.integers(-127, 128, 160)          # whatever follows must not matter
            out = np.zeros(nbits // 8, np.uint8)
            rc = lib.emul_vitdec(C.c_void_p(raw.ctypes.data + off), m.ctypes.data_as(C.c_void_p), nbits, None, out.ctypes.data_as(C.c_void_p))
            assert rc == 0 and np.array_equal(out, exp), (name, trial, int((out != exp).sum()))
