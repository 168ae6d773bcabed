"""Plain float64 reference of the OFDM demodulator (TEST TOOLING, numpy only): NCO mix with the exact phase, numpy's complex128 FFT,
the differential demap in the frequency-interleaver order and the guard-interval correlation.  It shares no code with the kernel
(welle.io_b200/csrc/ofdm_core.cuh, ofdm.cu) or with the oracle (oracle/dab_oracle.c): the transform, the oscillator and the
carrier order are numpy's and dabtx's, so agreement with it says something about both."""
import numpy as np

import dabtx

TU, TS, TG, K, RATE = 2048, 2552, 504, 1536, 2048000
SPAN = TU + 75 * TS                       # samples of one frame from the first useful PRS sample to the end of symbol 75
BINS = dabtx.perm_table() % TU            # FFT bin of logical carrier i (frequency-interleaver order)


def mix(x, lp0, ph, idx0=0):
    """x[i] * e^{j 2 pi lp(i) / 2 048 000} with lp(i) = lp0 - (idx0 + i) ph, in float64 with the exact integer phase"""
    i = np.arange(len(x), dtype=np.int64) + idx0
    lp = (int(lp0) - i * int(ph)) % RATE
    return np.asarray(x, np.complex128) * np.exp(2j * np.pi * lp.astype(np.float64) / RATE)


def demod(prs, syms, nco_prs=None, nco_sym=None):
    """One frame: prs = the T_u useful PRS samples, syms = the 75 data symbols (guard interval first, 75 * T_s samples).
    nco_prs / nco_sym: optional (lp0, ph) applied with the frame-relative sample index (PRS sample 0 = index 0, the data symbols
    continue at index T_u).  Returns a dict:
      soft  int8 [75, 3072]     trunc(-re 127 / (|re| + |im|)) of r1 in carrier order (re bits, then im bits), 0 where r1 = 0
      r1    complex128 [75, K]  X_l conj(X_{l-1}) per logical carrier
      mag   float64 [75, K]     |X_l| |X_{l-1}|
      corr  complex128          sum over the data symbols of x[i] conj(x[i - T_u]) over the last T_G samples of each symbol"""
    prs = np.asarray(prs, np.complex128)
    syms = np.asarray(syms, np.complex128)
    assert prs.shape == (TU,) and syms.shape == (75 * TS,)
    if nco_prs is not None:
        prs = mix(prs, *nco_prs)
    if nco_sym is not None:
        syms = mix(syms, *nco_sym, idx0=TU)
    sym = syms.reshape(75, TS)
    X = np.fft.fft(np.concatenate([prs[None, :], sym[:, TG:]]), axis=1)[:, BINS]      # [76, K]
    r1 = X[1:] * np.conj(X[:-1])
    mag = np.abs(X[1:]) * np.abs(X[:-1])
    re, im = r1.real, r1.imag
    l1 = np.abs(re) + np.abs(im)
    with np.errstate(divide="ignore", invalid="ignore"):
        s_re = np.where(l1 > 0, np.trunc(-re * 127.0 / l1), 0.0)
        s_im = np.where(l1 > 0, np.trunc(-im * 127.0 / l1), 0.0)
    soft = np.concatenate([s_re, s_im], axis=1).astype(np.int8)
    corr = np.sum(sym[:, TU:] * np.conj(sym[:, :TG]))
    return dict(soft=soft, r1=r1, mag=mag, corr=corr)


def frame(x, start, nco=None):
    """demod() of the frame whose first useful PRS sample is x[start]; nco = (lp0, ph) for the whole frame (one increment)"""
    x = np.asarray(x)
    return demod(x[start: start + TU], x[start + TU: start + SPAN], nco, nco)


def oracle_input(x, lp0, ph):
    """x mixed like the library's exact oscillator mode: the float32 table e^{j 2 pi lp / 2 048 000} and a complex product with each
    real product and sum rounded to float32 (the oracle is then fed these samples)"""
    x = np.asarray(x, np.complex64)
    n = np.arange(len(x), dtype=np.int64)
    lp = (int(lp0) - n * int(ph)) % RATE
    oc = np.cos(2.0 * np.pi * lp / RATE).astype(np.float32)
    os_ = np.sin(2.0 * np.pi * lp / RATE).astype(np.float32)
    re = (x.real * oc).astype(np.float32) - (x.imag * os_).astype(np.float32)
    im = (x.real * os_).astype(np.float32) + (x.imag * oc).astype(np.float32)
    return (re + 1j * im).astype(np.complex64)


def multipath(x, taps):
    """x through a static channel: taps = [(delay_samples, complex gain), ...], all delays inside the guard interval"""
    y = np.zeros(len(x), np.complex128)
    for d, g in taps:
        y[d:] += g * np.asarray(x[:len(x) - d], np.complex128)
    return y.astype(np.complex64)
