"""The wideband channelizer's definition (include/dab_b200.h, dabb_chan_*) restated in float64 numpy: geometry, prototype taps, the
exact mixer phase, the polyphase sum and the input span of an output range.  Independent of the library's code; the tests compare the
host build of chan_core.cuh and the device kernel with it."""
import math

import numpy as np

OUT_RATE = 2048000
RATES = [2048000, 2400000, 2500000, 3000000, 4096000, 6000000, 8000000, 8192000, 10000000, 20000000, 61440000]
IQ_CF32, IQ_U8, IQ_S8, IQ_S16LE, IQ_S16BE = 0, 1, 2, 3, 4
BYTES = {IQ_CF32: 8, IQ_U8: 2, IQ_S8: 2, IQ_S16LE: 4, IQ_S16BE: 4}


def geometry(R):
    """(L, M, T): 2 048 000 / R = L / M in lowest terms, T taps per polyphase branch"""
    g = math.gcd(OUT_RATE, R)
    L, M = OUT_RATE // g, R // g
    T = math.ceil((72 - 7.95) / (14.36 * 176000 / R)) + 1
    return L, M, T


def supported(R):
    return 2048000 <= R <= 64000000 and geometry(R)[0] <= 1024


def taps(R, dtype=np.float32):
    """the prototype h[0 .. L T) at rate L R: Kaiser window (beta = 0.1102 (72 - 8.7)) times the 856 kHz sinc, summing to L"""
    L, M, T = geometry(R)
    N = L * T
    n = np.arange(N, dtype=np.float64)
    c = (N - 1) / 2
    beta = 0.1102 * (72 - 8.7)
    w = np.i0(beta * np.sqrt(np.maximum(0.0, 1 - ((n - c) / c) ** 2))) / np.i0(beta)
    fc = 856000 / (L * R)
    h = 2 * fc * np.sinc(2 * fc * (n - c)) * w
    return (h * L / h.sum()).astype(dtype)


def response_db(h, R, resolution_hz=500.0):
    """(f, |H(f)| / L in dB) of the prototype at rate L R on a grid no coarser than resolution_hz, from 0 to L R / 2"""
    L = geometry(R)[0]
    nfft = 1 << int(math.ceil(math.log2(max(L * R / resolution_hz, 16 * len(h)))))
    H = np.abs(np.fft.rfft(np.asarray(h, np.float64), nfft)) / L
    return np.arange(len(H)) * (L * R / nfft), 20 * np.log10(np.maximum(H, 1e-300))


def last_input(m, R):
    L, M, _ = geometry(R)
    return (np.asarray(m, dtype=object) * M) // L


def input_range(R, out_start, out_len):
    """[first, end) of the input samples outputs [out_start, out_start + out_len) read"""
    L, M, T = geometry(R)
    return (out_start * M) // L - T + 1, ((out_start + out_len - 1) * M) // L + 1


def mixer(R, f, n):
    """exp(-2 pi i k(n) / R) with k(n) = (f n) mod R, exact integers (Python ints, any size)"""
    k = np.array([(f * int(v)) % R for v in np.asarray(n).ravel()], dtype=np.float64)
    return np.exp(-2j * np.pi * k / R)


def convert(raw, fmt):
    """raw samples -> complex128, value for value like CRAWFile::convertSamples"""
    raw = np.ascontiguousarray(raw)
    if fmt == IQ_CF32:
        return raw.view(np.complex64).astype(np.complex128)
    b = raw.view(np.uint8)
    if fmt == IQ_U8:
        v = (b.astype(np.float64) - 128) / 128
    elif fmt == IQ_S8:
        v = b.view(np.int8).astype(np.float64) / 128
    elif fmt == IQ_S16LE:          # the reference's "s16le" reads the first byte of each value as the high one
        v = b.reshape(-1, 2).astype(np.int32)
        v = ((v[:, 0] << 8) | v[:, 1]).astype(np.uint16).view(np.int16).astype(np.float64)
    else:
        v = b.reshape(-1, 2).astype(np.int32)
        v = ((v[:, 1] << 8) | v[:, 0]).astype(np.uint16).view(np.int16).astype(np.float64)
    return v[0::2] + 1j * v[1::2]


def channelize(x, x_start, R, f, out_start, out_len, h=None):
    """y[m] for m in [out_start, out_start + out_len) of the channel at f Hz; x: complex samples with absolute indices
    x_start, x_start + 1, ... (must cover input_range)"""
    L, M, T = geometry(R)
    h = taps(R).astype(np.float64) if h is None else np.asarray(h, np.float64)
    first, end = input_range(R, out_start, out_len)
    assert first >= x_start and end <= x_start + len(x), (first, end, x_start, len(x))
    xm = np.asarray(x[first - x_start:end - x_start], np.complex128) * mixer(R, f, np.arange(first, end, dtype=object))
    m = np.arange(out_start, out_start + out_len, dtype=object)
    nm = (m * M) // L
    pm = np.array([(int(v) * M) % L for v in m])
    idx = np.array([int(v) - first for v in nm])
    hj = h[pm[:, None] + np.arange(T)[None, :] * L]                 # [out, T]
    xj = xm[idx[:, None] - np.arange(T)[None, :]]                    # [out, T]
    return (hj * xj).sum(axis=1)


def error_ratio(y, y_ref):
    """(rms error, largest error), both relative to rms(y_ref)"""
    d = np.abs(np.asarray(y, np.complex128) - y_ref)
    r = np.sqrt(np.mean(np.abs(y_ref) ** 2))
    return float(np.sqrt(np.mean(d ** 2)) / r), float(d.max() / r)
