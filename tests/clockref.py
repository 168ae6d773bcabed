"""Numpy restatement of sample-clock tracking (dabb_options.sample_clock = DABB_CLOCK_TRACK, include/dab_b200.h; the device arithmetic
is welle.io_b200/csrc/clock_core.cuh): the per-stream estimator, step by step, giving the expected tap-11 records exactly; the
per-carrier phasor and the derotated r1 in float64; and resample_clock, which makes a recording with a known sample-clock error."""
import numpy as np

import dabtx

TU, TS, TF = 2048, 2552, 196608
K = 1536
FRAME_DECODED, FRAME_NEED_SAMPLES, FRAME_NO_SYNC, FRAME_ACQUIRING = 0, 1, 2, 3
CLOCK_OFF, CLOCK_TRACK = 0, 1
CLOCK_DTYPE = np.dtype([("ppm", "<f4"), ("applied_ppm", "<f4"), ("frames", "<i4"), ("reserved", "<i4")])
BIN = dabtx.perm_table() % TU                       # FFT bin of logical carrier i
CARRIER = np.where(BIN <= 768, BIN, BIN - TU)       # its carrier index k, -768..768 without 0


class Estimator:
    """the estimators of n streams: e (ppm), n (frames counted), prev (the previous active step decoded a frame)"""

    def __init__(self, n_streams):
        self.e = np.zeros(n_streams, np.float64)
        self.n = np.zeros(n_streams, np.int64)
        self.prev = np.zeros(n_streams, bool)

    def reset(self, first, count):
        """dabb_stream_reset"""
        sl = slice(first, first + count)
        self.e[sl] = 0.0
        self.n[sl] = 0
        self.prev[sl] = False

    def applied(self):
        """the ppm the next decoded frame of every stream is derotated with"""
        return np.where(self.n >= 8, self.e, 0.0)

    def step(self, mode, status, start_index):
        """one step with the option `mode`, given the step's result records' status and start_index: the tap-11 records"""
        S = len(self.e)
        out = np.zeros(S, CLOCK_DTYPE)
        for s in range(S):
            st = int(status[s])
            if mode != CLOCK_TRACK:
                self.prev[s] = False
                continue
            if st == FRAME_DECODED:
                out["applied_ppm"][s] = np.float32(self.e[s] if self.n[s] >= 8 else 0.0)
                d = int(start_index[s]) - 504
                if self.prev[s] and abs(d) <= 64:
                    self.n[s] = min(self.n[s] + 1, 2 ** 31 - 1)
                    self.e[s] = self.e[s] + (1e6 * d / TF - self.e[s]) / min(self.n[s], 32)
                self.prev[s] = True
            elif st in (FRAME_NO_SYNC, FRAME_ACQUIRING):
                self.prev[s] = False
            out["ppm"][s] = np.float32(self.e[s])
            out["frames"][s] = self.n[s]
        return out


def records(steps, n_streams):
    """expected tap-11 records of a sequence of steps: ("step", mode, status[S], start_index[S]) or ("reset", first, count)"""
    est = Estimator(n_streams)
    out = []
    for ev in steps:
        if ev[0] == "reset":
            est.reset(ev[1], ev[2])
        else:
            out.append(est.step(ev[1], ev[2], ev[3]))
    return out


def phasor(k, ppm):
    """exp(+2 pi i k ppm 1e-6 T_s / T_u) in float64, ppm taken as the float32 the device holds"""
    a = np.float64(np.float32(ppm))
    return np.exp(2j * np.pi * np.asarray(k, np.float64) * a * 1e-6 * TS / TU)


def derotate(r1, ppm):
    """r1 [..., 1536] in logical carrier order (r1_out, tap 2 takes every 96th) times the phasor of each carrier, float64"""
    return np.asarray(r1, np.complex128) * phasor(CARRIER, ppm)


def resample_clock(iq, ppm):
    """a recording of iq (made at exactly 2.048 Msps) as a receiver whose clock is off by ppm records it: N samples become
    M = round(N (1 + eps)) by an FFT resample (the periodic band-limited interpolation of iq).  Returns (the samples, the effective
    ppm 1e6 (M / N - 1), exact for the returned length)."""
    x = np.asarray(iq, np.complex128)
    N = len(x)
    M = int(round(N * (1.0 + ppm * 1e-6)))
    X = np.fft.fft(x)
    Y = np.zeros(M, np.complex128)
    h = min(N, M) // 2
    Y[:h] = X[:h]
    Y[M - h:] = X[N - h:]
    y = np.fft.ifft(Y) * (M / N)
    return y.astype(np.complex64), 1e6 * (M / N - 1.0)
