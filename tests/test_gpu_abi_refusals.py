"""A call the C ABI refuses runs no step.  dabb_process and dabb_submit with an msc_stride below 3 x bitrate or an sf_stride below
15 x bitrate of a selected sub-channel return DABB_E_ARG before anything is enqueued: no kernel is launched, no stream advances,
and the following steps give byte for byte what a twin context that never saw the bad call gives.  Taps 7 / 8 refuse a stride
that is too small in the same way."""
import numpy as np
import pytest

import dabtx
from conftest import load_pkg

pytestmark = pytest.mark.gpu
S, BITRATE = 2, 96
MSC, SF = 3 * BITRATE, 15 * BITRATE
E_ARG, E_STATE = -3, -4
BAD = {"msc": dict(msc_stride=MSC - 1, sf_stride=SF), "sf": dict(msc_stride=MSC, sf_stride=SF - 1)}


def _signal():
    return np.stack([dabtx.add_awgn(dabtx.DabTx(seed=0xAB0 + i, bitrate=BITRATE).frames(12), 18.0 + i, seed=i) for i in range(S)])


def _context(pkg):
    c = pkg.Context(n_streams=S, disable_coarse=True)
    c.select_subchannel(0, 72, BITRATE, eep_profile_a=True, eep_level=3, dabplus=True)
    return c


def _refused(code, call, *args, **kw):
    with pytest.raises(Exception) as e:
        call(*args, **kw)
    assert f"error {code}:" in str(e.value), str(e.value)


def _same(x, y, step):
    assert x["results"].tobytes() == y["results"].tobytes(), step
    for k in ("fibs", "msc", "sf"):
        assert np.array_equal(x[k], y[k]), (k, step)


@pytest.mark.parametrize("bad", ["msc", "sf"])
def test_process_refusal_runs_no_step(bad):
    pkg = load_pkg()
    sig = _signal()
    n = sig.shape[1]
    a, b = _context(pkg), _context(pkg)
    da, db = a.dev(sig), b.dev(sig)
    step = lambda c, d, **kw: c.process(d, n, np.zeros(S, np.int64), n, **kw)
    for k in range(2):
        _same(step(a, da, msc_stride=MSC, sf_stride=SF), step(b, db, msc_stride=MSC, sf_stride=SF), k)
    launches = a.kernel_launches()
    _refused(E_ARG, step, a, da, **BAD[bad])
    assert a.kernel_launches() == launches
    superframes = 0
    for k in range(2, 9):
        x, y = step(a, da, msc_stride=MSC, sf_stride=SF), step(b, db, msc_stride=MSC, sf_stride=SF)
        _same(x, y, k)
        superframes += int(x["results"]["sf_ready"][:, 0].sum())
    assert superframes > 0 and (x["results"]["status"] == pkg.FRAME_DECODED).all()
    a.close(); b.close()


@pytest.mark.parametrize("bad", ["msc", "sf"])
def test_submit_refusal_runs_no_step(bad):
    pkg = load_pkg()
    sig = np.ascontiguousarray(_signal())
    n = sig.shape[1]
    a, b = _context(pkg), _context(pkg)

    def step(c, **kw):
        c.submit(sig.ctypes.data, n, np.zeros(S, np.int64), n, **kw)
        return c.collect()
    for k in range(2):
        _same(step(a, msc_stride=MSC, sf_stride=SF), step(b, msc_stride=MSC, sf_stride=SF), k)
    launches = a.kernel_launches()
    _refused(E_ARG, a.submit, sig.ctypes.data, n, np.zeros(S, np.int64), n, **BAD[bad])
    assert a.kernel_launches() == launches
    _refused(E_STATE, a.collect)
    superframes = 0
    for k in range(2, 9):
        x, y = step(a, msc_stride=MSC, sf_stride=SF), step(b, msc_stride=MSC, sf_stride=SF)
        _same(x, y, k)
        superframes += int(x["results"]["sf_ready"][:, 0].sum())
    assert superframes > 0 and (x["results"]["status"] == pkg.FRAME_DECODED).all()
    a.close(); b.close()


def test_output_taps_refuse_short_strides():
    pkg = load_pkg()
    sig = _signal()
    n = sig.shape[1]
    c = _context(pkg)
    d = c.dev(sig)
    for _ in range(3):
        out = c.process(d, n, np.zeros(S, np.int64), n, msc_stride=MSC, sf_stride=SF)
    _refused(E_ARG, c.read_tap, 7, MSC - 1)
    _refused(E_ARG, c.read_tap, 8, SF - 1)
    assert np.array_equal(c.read_tap(7, MSC), out["msc"]) and np.array_equal(c.read_tap(8, SF), out["sf"])
    c.close()
