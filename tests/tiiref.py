"""Helpers of the TII tests (test_tii_emul.py, test_gpu_tii_batch.py): the glue's host analyser (welle.io_b200/host/tii.h, which
test_figdb.py pins to the unmodified TIIDecoder) driven through its test hooks, TII spectra built from dabtx recordings or directly
with chosen active carrier pairs, and measurements grouped by frame."""
import ctypes as C
import os
from collections import defaultdict

import numpy as np

from conftest import ROOT

TF, TU, TNULL, TS = 196608, 2048, 2656, 2552
PATTERN_WORDS = [w for w in range(256) if bin(w).count("1") == 4]


def host_lib():
    lib = C.CDLL(os.path.join(ROOT, "welle.io_b200", "libwelle_b200_host.so"))
    lib.welle_b200_tii_run_framed.restype = C.c_int
    lib.welle_b200_tii_map_argmin.restype = C.c_int
    return lib


def host_run_framed(lib, nspec, pspec):
    """measurements of the host analyser: [(frame, comb, pattern, delay, error)] in callback order"""
    nspec = np.ascontiguousarray(nspec, np.complex64); pspec = np.ascontiguousarray(pspec, np.complex64)
    cap = 9 * len(nspec) + 16
    out = np.zeros(5 * cap, np.float32)
    k = lib.welle_b200_tii_run_framed(nspec.ctypes.data_as(C.c_void_p), pspec.ctypes.data_as(C.c_void_p), len(nspec), out.ctypes.data_as(C.c_void_p), cap)
    assert k <= cap
    return [(int(r[0]), int(r[1]), int(r[2]), int(r[3]), float(r[4])) for r in out[:5 * k].reshape(-1, 5)]


def by_frame(meas):
    """{frame: [(comb, pattern, delay, error)] in ascending (comb, pattern) order}"""
    d = defaultdict(list)
    for f, c, p, dl, e in meas:
        d[f].append((c, p, dl, e))
    return {f: sorted(v) for f, v in d.items()}


def compare(want, got, frames=None, tol=None):
    """want / got: by_frame dicts.  (comb, pattern, delay) must be equal frame by frame; returns (measurements, differing errors,
    largest error difference).  tol: largest error difference allowed (None: any)"""
    keys = sorted(set(want) | set(got))
    if frames is not None:
        keys = [f for f in keys if f in frames]
    n = ndiff = 0; worst = 0.0
    for f in keys:
        a, b = want.get(f, []), got.get(f, [])
        assert [x[:3] for x in a] == [x[:3] for x in b], (f, a, b)
        for x, y in zip(a, b):
            n += 1
            if x[3] != y[3]:
                ndiff += 1; worst = max(worst, abs(x[3] - y[3]))
    if tol is not None:
        assert worst <= tol, worst
    return n, ndiff, worst


def recording_spectra(oracle, tx_set, snr_db, n_frames, seed):
    """dabtx recording with the transmitters tx_set = [(comb, pattern, delay, gain)]: per frame the spectra of the aligned PRS and of the
    last T_u samples of the null symbol that follows it (the pairing of TIIDecoder), made with the oracle's FFT (= the reference's)"""
    import dabtx
    tx = dabtx.DabTx(seed=seed)
    tx.tii = list(tx_set)
    sig = tx.frames(n_frames + 1)
    if snr_db is not None:
        sig = dabtx.add_awgn(sig, snr_db, seed=seed + 1)
    nulls, prss = [], []
    for f in range(1, n_frames + 1):
        base = f * TF
        nulls.append(sig[base: base + TNULL]); prss.append(sig[base + TNULL + 504: base + TNULL + 504 + TU])
    nulls, prss = nulls[1:], prss[:-1]
    nspec = np.stack([oracle.fft(x[TNULL - TU:]) for x in nulls]); pspec = np.stack([oracle.fft(x) for x in prss])
    return nspec, pspec


def active_pairs_spectra(rng, pairs_per_frame):
    """spectra in which exactly the carrier pairs i (0..191) of each frame's set are active: PRS carriers of unit magnitude and random phase,
    null carriers of a pair equal with magnitude 1 and random phase (|mult| = 4 > 0.4 |p|^2), all other null carriers 0"""
    n = len(pairs_per_frame)
    pspec = np.exp(2j * np.pi * rng.random((n, TU))).astype(np.complex64)
    nspec = np.zeros((n, TU), np.complex64)
    for f, pairs in enumerate(pairs_per_frame):
        for i in pairs:
            for k0 in (TU - 768, TU - 384, 1, 385):
                v = np.exp(2j * np.pi * rng.random())
                nspec[f, k0 + 2 * i] = v; nspec[f, k0 + 2 * i + 1] = v
    return nspec, pspec


def pairs_of(comb, word):
    """carrier pairs of a (comb, pattern word): pair c + 24 b for every group b whose bit (7 - b) is set"""
    return [comb + 24 * b for b in range(8) if (word >> (7 - b)) & 1]
