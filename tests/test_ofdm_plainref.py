"""The float64 OFDM reference (tests/ofdmref.py) against the oracle's demodulator on clean, noisy, multipath and carrier-offset
frames, before any GPU test relies on it: softbits within 1, r1 within 1e-5 of |X_l| |X_{l-1}| per carrier.  The guard-interval
correlation is checked where its value is known without either implementation: on a frame without noise the guard interval is an
exact copy, so the sum is e^{j 2 pi f T_u / 2 048 000} times the guard energy (f the carrier offset)."""
import numpy as np
import pytest

import dabtx
import ofdmref

TU, TS, TG, TF, TNULL = 2048, 2552, 504, 196608, 2656
ST = TF + TNULL + 305                     # the first useful PRS sample of the second frame, inside its guard interval like the receiver


@pytest.fixture(scope="module")
def clean():
    return dabtx.DabTx(seed=0x0F0).frames(3, noise_floor=0)


def _frames(clean):
    noisy = dabtx.add_awgn(clean, 12.0, seed=0x0F1)
    echo = ofdmref.multipath(clean, [(0, 1.0), (37, 0.35 - 0.2j), (211, 0.15j)])
    return {"clean": (clean, None), "noisy": (noisy, None), "multipath": (echo, None),
            "offset": (dabtx.freq_shift(clean, 321.0), (123456, 321)), "offset_negative": (dabtx.freq_shift(echo, -4321.0), (2047000, -4321))}


@pytest.mark.parametrize("name", ["clean", "noisy", "multipath", "offset", "offset_negative"])
def test_reference_matches_oracle(oracle, clean, name):
    x, nco = _frames(clean)[name]
    if nco is None:
        o_in = x[ST: ST + ofdmref.SPAN]
    else:
        # the receiver mixes with the frame-relative index: sample ST is index 0
        o_in = ofdmref.oracle_input(x[ST: ST + ofdmref.SPAN], *nco)
    s_o, r_o = oracle.demod_frame(o_in[:TU], o_in[TU:], True)
    ref = ofdmref.frame(x, ST, nco)
    d = np.abs(ref["soft"].astype(int) - s_o.astype(int))
    assert d.max() <= 1, (name, int(d.max()), int((d > 1).sum()))
    err = np.abs(ref["r1"] - r_o.astype(np.complex128)) / ref["mag"]
    assert err.max() <= 1e-5, (name, float(err.max()))
    if nco is not None:
        # the mixed frame is the transmitted one: its FIC decodes
        _, crc = oracle.fic_decode(s_o[:3].reshape(-1))
        assert crc.all(), name


@pytest.mark.parametrize("hz", [0.0, 321.0, -4321.0])
def test_reference_correlation_of_a_noiseless_frame(clean, hz):
    x = dabtx.freq_shift(clean, hz) if hz else clean
    st = TF + TNULL + TG                  # symbol windows on the transmitted symbol boundaries: each guard interval is a whole copy
    ref = ofdmref.frame(x, st)
    sym = x[st + TU: st + ofdmref.SPAN].astype(np.complex128).reshape(75, TS)
    energy = np.sum(np.abs(sym[:, :TG]) ** 2)
    want = np.exp(2j * np.pi * hz * TU / 2048000.0) * energy
    assert abs(ref["corr"] - want) <= 1e-6 * abs(want), (ref["corr"], want)


def test_reference_nco_is_the_carrier_offset(clean):
    """mixing with (lp0, ph) undoes a shift of +ph Hz; a constant phase lp0 changes no softbit (differential demodulation)"""
    x = dabtx.freq_shift(clean, 1000.0)
    a = ofdmref.frame(x, ST, (0, 1000))
    b = ofdmref.frame(x, ST, (777777, 1000))
    c = ofdmref.frame(clean, ST)
    assert np.array_equal(a["soft"], b["soft"])
    assert np.abs(a["soft"].astype(int) - c["soft"].astype(int)).max() <= 1
    assert np.allclose(a["mag"], c["mag"], rtol=1e-5)
    # a symbol of zeros gives r1 = 0 on it and on the next symbol, and softbits 0 there
    z = clean.copy()
    z[ST + TU + 9 * TS: ST + TU + 10 * TS] = 0
    r = ofdmref.frame(z, ST)
    assert not r["soft"][9:11].any() and not r["r1"][9:11].any() and r["soft"][11].any()
