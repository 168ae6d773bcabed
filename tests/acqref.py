"""float64 restatement of the robust acquisition rule (dabb_options.acquisition = DABB_ACQ_ROBUST, include/dab_b200.h): block levels,
the window decision and the interferer excision of the phase reference correlation, plus the test signals (tones, paths) that
tests/test_acq_emul.py and tests/test_gpu_acq.py feed it."""
import numpy as np

BLK, HALF, WIN, NB_MAX, MIN_BLOCKS, EDGE, KEEP = 256, 87, 9, 784, 32, 2, 11
NULL_END, LEAD = 2480, 256
DEPTH_DB = 1.2
T_EXC, EXC_NEIGH = 20.0, 2
TINY, HUGE = 2.0 ** -126, float(np.finfo(np.float32).max)
TF, TNULL = 196608, 2656


def clamp_power(p):
    p = np.where(np.isnan(p), TINY, p)
    return np.clip(p, TINY, HUGE)


def levels(y):
    """float64 levels of the nb = len(y) // 256 blocks of (mixed) samples y"""
    nb = len(y) // BLK
    x = np.asarray(y[:nb * BLK], np.complex128).reshape(nb, BLK)
    n = np.arange(BLK)
    w = np.sin(np.pi * n / BLK) ** 2
    with np.errstate(invalid="ignore", over="ignore"):
        X = np.fft.fft(x * w, axis=1)
        P = clamp_power(X.real ** 2 + X.imag ** 2)
    k = np.arange(-HALF, HALF + 1) % BLK
    return np.log2(P[:, k]).mean(axis=1)


def l1sums(y):
    nb = len(y) // BLK
    x = np.asarray(y[:nb * BLK], np.complex128).reshape(nb, BLK)
    return (np.abs(x.real) + np.abs(x.imag)).sum(axis=1)


def window_sums(lv):
    c = np.concatenate([[0.0], np.cumsum(np.asarray(lv, np.float64))])
    return c[WIN:] - c[:-WIN]


def decide(lv):
    """(found, best, depth_db, median, W) of a span's levels"""
    lv = np.asarray(lv, np.float64)
    nb = len(lv)
    W = window_sums(lv)
    best = len(W) - 1 - int(np.argmin(W[::-1]))          # the last of equal minima
    med = float(np.sort(lv)[(nb - 1) // 2])
    depth = (med - W[best] / WIN) * 10 * np.log10(2)
    return bool(depth >= DEPTH_DB and best + WIN + EDGE <= nb), best, float(depth), med, W


def excise(X):
    """bins of a window spectrum X[2048] (natural order) that the excision zeroes (bool[2048])"""
    X = np.asarray(X, np.complex128)
    P = clamp_power(X.real ** 2 + X.imag ** 2)
    k = np.arange(2048)
    inb = (k != 0) & ((k <= 768) | (k >= 2048 - 768))
    lg = np.log2(P[inb]).mean()
    over = inb & (np.log2(P) > lg + np.log2(T_EXC))
    z = np.zeros(2048, bool)
    for d in range(-EXC_NEIGH, EXC_NEIGH + 1):
        z |= np.roll(over, d)
    return z


def tone(iq, hz, db_above, phase=0.3):
    """iq plus a continuous tone at hz whose power is db_above the mean power of iq"""
    p = float(np.mean(np.abs(iq.astype(np.complex128)) ** 2))
    a = np.sqrt(p * 10 ** (db_above / 10))
    n = np.arange(len(iq))
    return (iq + a * np.exp(1j * (2 * np.pi * hz * n / 2048000.0 + phase))).astype(np.complex64)


def paths(iq, taps):
    """multipath: sum of delayed, scaled copies [(delay, gain), ...]"""
    out = np.zeros(len(iq), np.complex128)
    for d, g in taps:
        out[d:] += g * iq[:len(iq) - d]
    return out.astype(np.complex64)


def resample_ppm(iq, ppm):
    """linear-interpolation resampling of a recording whose clock is off by ppm (more samples for ppm > 0)"""
    n_out = int(len(iq) * (1 + ppm * 1e-6)) - 2
    t = np.arange(n_out) / (1 + ppm * 1e-6)
    i = np.floor(t).astype(np.int64)
    f = t - i
    return ((1 - f) * iq[i] + f * iq[i + 1]).astype(np.complex64)
