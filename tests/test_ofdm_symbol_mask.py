"""The per-stream OFDM symbol mask (welle.io_b200/csrc/ofdm_mask.cuh), built as host C++ (tests/host_emul/emul_ofdm_mask.cpp), against a
restatement from the byte ranges the decoders read in a frame's softbits (75 symbols of 3072 bytes; data symbol l at (l - 1) * 3072):
- the FIC decoder (run_fic) and the bit-error count of the FIC (ber_kernel, part 0): four codewords of 2304 bytes, [0, 9216);
- msc_collect_kernel, per enabled slot and CIF c = 0..3: [(3 + 18 c) 3072 + 64 start_cu, + 64 length_cu).  The sub-channel's own
  bit-error count reads the fragments msc_gather_kernel rebuilt from those bytes, not the frame's softbits.
A symbol is demapped exactly when one of those bytes lies in it: every byte a reader touches is in a demapped symbol, and every demapped
symbol holds one (the set is minimal).  A symbol is transformed when it or the next one is demapped, and the phase reference symbol always
is."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT

HERE = os.path.join(ROOT, "tests", "host_emul")
NSYM, SYM_BYTES, MSC_CU = 76, 3072, 864


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_ofdm_mask") / "libemul_ofdm_mask.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "emul_ofdm_mask.cpp")])
    lib = C.CDLL(so)
    lib.emul_ofdm_mask.restype = None
    lib.emul_ofdm_mask_words.restype = C.c_int
    return lib


def build(lib, slots):
    """slots [n_streams][n_slots][3] (enabled, start_cu, length_cu) -> masks [n][words], demap [n][76], transform [n][76]"""
    slots = np.ascontiguousarray(slots, np.int32)
    n, k = slots.shape[0], slots.shape[1]
    w = lib.emul_ofdm_mask_words()
    masks = np.zeros((n, w), np.uint32); flags = np.zeros((n, NSYM), np.uint8)
    lib.emul_ofdm_mask(slots.ctypes.data_as(C.c_void_p), n, k, masks.ctypes.data_as(C.c_void_p), flags.ctypes.data_as(C.c_void_p))
    return masks, (flags & 1).astype(bool), (flags >> 1).astype(bool)


def read_symbols(slots):
    """[n][76]: the symbols holding a byte the FIC, MSC-collect and bit-error readers touch"""
    slots = np.asarray(slots, np.int64)
    n = slots.shape[0]
    used = np.zeros((n, NSYM), bool)
    used[:, 1 + np.arange(4 * 2304) // SYM_BYTES] = True                    # FIC: bytes [0, 9216)
    for k in range(slots.shape[1]):
        en, st, ln = slots[:, k, 0] != 0, slots[:, k, 1], slots[:, k, 2]
        for c in range(4):
            b0 = (3 + 18 * c) * SYM_BYTES + 64 * st                          # first and last byte of the slice
            b1 = b0 + 64 * ln - 1
            l0, l1 = 1 + b0 // SYM_BYTES, 1 + b1 // SYM_BYTES
            for d in range(int((l1 - l0).max(initial=0)) + 1):            # a slice spans at most 18 symbols
                ok = en & (ln >= 1) & (l0 + d <= l1)
                used[np.flatnonzero(ok), (l0 + d)[ok]] = True
    return used


def check(lib, slots):
    masks, demap, transform = build(lib, slots)
    want = read_symbols(slots)
    assert np.array_equal(demap, want), np.flatnonzero((demap != want).any(1))[:8]
    assert not demap[:, 0].any()
    nxt = np.concatenate([demap[:, 1:], np.zeros((len(demap), 1), bool)], 1)
    want_t = demap | nxt
    want_t[:, 0] = True
    assert np.array_equal(transform, want_t)
    # the words hold the demapped symbols as bits 1..75 and nothing else
    bits = np.unpackbits(masks.view(np.uint8), axis=1, bitorder="little")[:, :masks.shape[1] * 32].astype(bool)
    assert np.array_equal(bits[:, :NSYM], demap) and not bits[:, NSYM:].any()
    return demap, transform


def test_every_single_slot_geometry(lib):
    """every (start_cu, length_cu) of one enabled slot over the whole MSC"""
    st, ln = np.meshgrid(np.arange(MSC_CU), np.arange(1, MSC_CU + 1), indexing="ij")
    keep = st + ln <= MSC_CU
    slots = np.stack([np.ones(keep.sum(), np.int32), st[keep], ln[keep]], 1)[:, None, :]
    assert len(slots) == MSC_CU * (MSC_CU + 1) // 2
    check(lib, slots)


def test_benchmark_geometry(lib):
    """CU 0..71 (a 96 kbit/s EEP 3-A sub-channel): 11 demapped symbols, 15 transformed of 76"""
    demap, transform = check(lib, [[[1, 0, 72]]])
    assert np.flatnonzero(demap[0]).tolist() == [1, 2, 3, 4, 5, 22, 23, 40, 41, 58, 59]
    assert np.flatnonzero(transform[0]).tolist() == [0, 1, 2, 3, 4, 5, 21, 22, 23, 39, 40, 41, 57, 58, 59]


def test_fic_only(lib):
    """no slot, and four disabled slots (whatever geometry they held): the FIC's symbols 1-3 and the phase reference"""
    for slots in (np.zeros((1, 0, 3), np.int32), [[[0, 0, 864], [0, 100, 50], [0, 863, 1], [0, 0, 72]]]):
        demap, transform = check(lib, slots)
        assert np.flatnonzero(demap[0]).tolist() == [1, 2, 3] and np.flatnonzero(transform[0]).tolist() == [0, 1, 2, 3]


def test_whole_msc_demaps_everything(lib):
    demap, transform = check(lib, [[[1, 0, 864]]])
    assert demap[0, 1:].all() and transform[0].all()


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_random_slot_combinations(lib, seed):
    """1-4 slots per stream, some disabled, overlapping and identical geometries included"""
    rng = np.random.default_rng(seed)
    n = 20000
    k = int(rng.integers(1, 5))
    st = rng.integers(0, MSC_CU, (n, k))
    ln = 1 + (rng.random((n, k)) * (MSC_CU - st)).astype(np.int64)
    short = rng.random((n, k)) < 0.5                                        # mostly short sub-channels, like real ensembles
    ln = np.where(short, np.minimum(ln, rng.integers(1, 200, (n, k))), ln)
    en = rng.random((n, k)) < 0.8
    slots = np.stack([en, st, ln], 2).astype(np.int32)
    if k > 1:                                                               # every 7th stream: slot 1 repeats slot 0
        slots[::7, 1] = slots[::7, 0]
    check(lib, slots)


def test_slices_at_symbol_boundaries(lib):
    """slices that end on, start on and cross a symbol boundary (48 CUs per symbol), and a sub-channel ending at CU 863"""
    geoms = [(0, 48), (0, 49), (47, 1), (47, 2), (48, 48), (95, 2), (96, 1), (816, 48), (815, 49), (863, 1), (0, 864), (431, 2)]
    slots = np.array([[[1, s, l]] for s, l in geoms], np.int32)
    demap, _ = check(lib, slots)
    assert np.flatnonzero(demap[0]).tolist() == [1, 2, 3, 4, 22, 40, 58]
    assert np.flatnonzero(demap[1]).tolist() == [1, 2, 3, 4, 5, 22, 23, 40, 41, 58, 59]
    assert np.flatnonzero(demap[9]).tolist() == [1, 2, 3, 21, 39, 57, 75]
