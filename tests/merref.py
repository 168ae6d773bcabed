"""Restatement of the modulation error ratio of include/dab_b200.h (dabb_set_mer, tap 14) in numpy and Python integers, sharing nothing
with welle.io_b200/csrc/mer_core.cuh: the groups come from dabtx.perm_table(), the sums are Python ints.  Also the channel models the
MER tests and scripts/mer_measure.py apply to tests/dabtx.py recordings."""
import math

import numpy as np

import dabtx

GROUPS = 64
TU, TG, TS, TNULL, TF = dabtx.TU, dabtx.TG, dabtx.TS, dabtx.TNULL, dabtx.TF
SPAN = TU + 75 * TS


def physical_carriers():
    """[1536] the physical carrier k (-768 .. 768 without 0) of each logical carrier"""
    return dabtx.perm_table()


def groups():
    """[1536] the group of each logical carrier: 24 carriers each, lowest frequency first"""
    k = physical_carriers()
    return np.array([(int(c) + 768 - (1 if c > 0 else 0)) // 24 for c in k], np.int64)


def mer_db(sig, err):
    if sig == 0:
        return 0.0
    if err == 0:
        return math.inf
    return float(np.float32(10.0 * math.log10(sig / err)))


def record(soft):
    """the tap-14 record of one decoded frame: soft = the frame's softbits, [75][3072] or its first 9216 bytes"""
    s = np.asarray(soft, np.int8).reshape(-1)[:3 * 3072].reshape(3, 3072).astype(np.int64)
    a, b = np.abs(s[:, :1536]), np.abs(s[:, 1536:])
    u2, v2 = (a + b) ** 2, (a - b) ** 2
    g = groups()
    gsig, gerr = [0] * GROUPS, [0] * GROUPS
    for i in range(1536):
        gsig[g[i]] += int(u2[:, i].sum())
        gerr[g[i]] += int(v2[:, i].sum())
    sig, err = sum(gsig), sum(gerr)
    return dict(points=int(((a + b) > 0).sum()), sig=sig, err=err, mer_db=mer_db(sig, err), gsig=gsig, gerr=gerr)


def zero_record():
    return dict(points=0, sig=0, err=0, mer_db=0.0, gsig=[0] * GROUPS, gerr=[0] * GROUPS)


def from_tap(t):
    """a MER_DTYPE element as the dict record() returns"""
    return dict(points=int(t["points"]), sig=int(t["sig"]), err=int(t["err"]), mer_db=float(t["mer_db"]),
                gsig=[int(x) for x in t["group"]["sig"]], gerr=[int(x) for x in t["group"]["err"]])


def group_mer(rec):
    """[64] the MER of each group of one record (or of summed sums), dB"""
    return np.array([mer_db(s, e) for s, e in zip(rec["gsig"], rec["gerr"])])


# ---- channels
def two_path(x, taps):
    """sum over (delay in samples, complex gain) of the delayed recording"""
    y = np.zeros(len(x), np.complex128)
    for d, g in taps:
        y[d:] += g * x[:len(x) - d] if d else g * x
    return y.astype(np.complex64)


def tone(x, hz, rel_db, seed=0):
    """x plus a tone at hz (from the tuned frequency) rel_db above x's mean power, at a random phase"""
    p = float(np.mean(np.abs(x) ** 2)) * 10 ** (rel_db / 10)
    ph = np.random.default_rng(seed).uniform(0, 2 * np.pi)
    n = np.arange(len(x))
    return (x + np.sqrt(p) * np.exp(1j * (2 * np.pi * hz * n / 2048000.0 + ph))).astype(np.complex64)


def oracle_softbits(oracle, x, frames):
    """the oracle demodulator's softbits of frames 0 .. frames-1 of a dabtx recording (the FFT windows at the ends of the guards)"""
    out = []
    for f in range(frames):
        seg = np.asarray(x[f * TF + TNULL + TG:f * TF + TNULL + TG + SPAN], np.complex64)
        out.append(oracle.demod_frame(seg[:TU], seg[TU:]))
    return out
