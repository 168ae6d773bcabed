"""The spectrum survey and the candidate detector (include/dab_b200.h, dabb_survey / dabb_survey_candidates) restated in numpy:
the Welch spectrum in float64, and the detector with the library's exact integer bin membership and its double sums in ascending
order (np.cumsum, math.log10), so that its candidate lists can be compared for equality.  Independent of the library's code."""
import math

import numpy as np

import chanref

CAND_DTYPE = np.dtype([("offset_hz", "<i8"), ("score_db", "<f4"), ("reserved", "<i4")])


def nfft_for_rate(R):
    """batch_decode's FFT size: the smallest power of two >= 1024 with R / nfft <= 4000 Hz"""
    n = 1024
    while R > 4000 * n:
        n *= 2
    return n


def spectrum(x, nfft):
    """P[j] of complex samples x (float64): Welch, 50 % overlap, periodic Hann, bin j at (j - nfft/2) R / nfft"""
    x = np.asarray(x, np.complex128)
    S = (len(x) - nfft) // (nfft // 2) + 1
    w = np.sin(np.pi * np.arange(nfft) / nfft) ** 2
    idx = (np.arange(S) * (nfft // 2))[:, None] + np.arange(nfft)[None, :]
    X = np.fft.fft(x[idx] * w, axis=1)
    P = (np.abs(X) ** 2).mean(axis=0) / (w ** 2).sum()
    return np.fft.fftshift(P)


def spectrum_raw(raw, fmt, nfft):
    return spectrum(chanref.convert(raw, fmt), nfft)


def candidates(psd, R, min_score_db=6.0):
    """the detector: a CAND_DTYPE array in ascending offset"""
    P = np.asarray(psd, np.float32).astype(np.float64)
    N = len(P)
    pmax = P.max()
    if not pmax > 0:
        return np.zeros(0, CAND_DTYPE)
    fl = 1e-12 * pmax
    Ld = np.array([10.0 * math.log10(p if p > fl else fl) for p in P])
    min_bins = (56000 * N + R - 1) // R
    j = np.arange(1, N, dtype=np.int64)                      # j = 0 lies outside |f_j| <= R/2 - R/nfft
    out, run = [], None
    for c in range(N):
        ok = 2 * abs(c - N // 2) * R + 2 * 768000 * N <= R * N
        score = None
        if ok:
            d = j - c
            ad = np.abs(d) * R
            Lj = Ld[1:]
            I = Lj[ad <= 700000 * N]
            gm = None
            for side in (d < 0, d > 0):
                g = Lj[side & (ad >= 784000 * N) & (ad <= 896000 * N)]
                if len(g) >= min_bins:
                    m = np.cumsum(g)[-1] / len(g)
                    gm = m if gm is None or m > gm else gm
            if gm is not None and len(I):
                score = np.cumsum(I)[-1] / len(I) - gm
        if score is not None and score >= float(np.float32(min_score_db)):
            run = [c, c, score] if run is None else [run[0], c, max(run[2], score)]
        elif run is not None:
            out.append(run); run = None
    if run is not None:
        out.append(run)
    res = np.zeros(len(out), CAND_DTYPE)
    for k, (a, b, s) in enumerate(out):
        num, den = (a + b - N) * R, 2 * N
        q = (2 * abs(num) + den) // (2 * den)
        res[k] = (q if num >= 0 else -q, np.float32(s), 0)
    return res


def scores(psd, R):
    """score(c) of every considered centre (NaN elsewhere), for choosing test spectra away from the threshold"""
    P = np.asarray(psd, np.float32).astype(np.float64)
    N = len(P)
    out = np.full(N, np.nan)
    if not P.max() > 0:
        return out
    L = 10 * np.log10(np.maximum(P, 1e-12 * P.max()))
    f = (np.arange(N) - N // 2) * R / N
    for c in range(N):
        if abs(f[c]) + 768000 > R / 2:
            continue
        d = f - f[c]
        inside = np.abs(f) <= R / 2 - R / N
        gs = [L[inside & (s * d >= 784000) & (s * d <= 896000)] for s in (-1, 1)]
        gs = [g.mean() for g in gs if len(g) >= math.ceil(56000 * N / R)]
        if gs:
            out[c] = L[np.abs(d) <= 700000].mean() - max(gs)
    return out
