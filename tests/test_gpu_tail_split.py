"""The tail split of the OFDM launch decodes exactly what the unsplit launch decodes.

A large batch cuts its last frames (half a residency of OFDM CTAs) into OFDM_TAIL_GROUPS short CTAs each; `ofdm_tail_split = -1`
gives every frame one CTA.  Two such contexts run 2048 streams (at least two residencies of 660 CTAs on a 132-SM H100, so that the
default context cuts a tail) that all read one shared recording (stride 0).  Status, FIBs, logical frames, superframes and softbits
must be byte-identical between the contexts and, within each context, to stream 0's.  Only the fine-AFC correlation and the signal
level of a tail stream are partial sums added in another order (DESIGN.md 5 (i)): they are compared to 1e-5 of their magnitude, and
every other field of the result record exactly.  Records are compared field by field: the padding before `next_pos` is no field."""
import numpy as np
import pytest

import dabtx
from conftest import load_pkg

pytestmark = pytest.mark.gpu
S, BITRATE, FRAMES, STEPS = 2048, 96, 12, 9
MSC, SF = 3 * BITRATE, 15 * BITRATE
FLOATS = ("freq_corr_re", "freq_corr_im", "slevel")


def _context(pkg, tail_split):
    ctx = pkg.Context(n_streams=S, ofdm_tail_split=tail_split)
    ctx.select_subchannel(0, dabtx.eep_cu(BITRATE), BITRATE, eep_profile_a=True, eep_level=3, dabplus=True)
    return ctx


def _step(pkg, ctx, d, n):
    out = ctx.process(d, 0, np.zeros(S, np.int64), n, msc_stride=MSC, sf_stride=SF)
    decoded = out["results"]["status"][0] == pkg.FRAME_DECODED
    out["soft"] = ctx.read_tap(0).reshape(S, -1).view(np.uint64) if decoded else None      # the softbit buffer of a skipped frame is stale
    return out


def _without_floats(res):
    r = res.copy()
    for f in FLOATS:
        r[f] = 0
    return r


def _close(a, b):
    """result records a, b: the fine-AFC correlation (as one complex number) and the level within 1e-5 of a's magnitude"""
    za = a["freq_corr_re"].astype(np.float64) + 1j * a["freq_corr_im"]
    zb = b["freq_corr_re"].astype(np.float64) + 1j * b["freq_corr_im"]
    la, lb = a["slevel"].astype(np.float64), b["slevel"].astype(np.float64)
    return (np.abs(za - zb) <= 1e-5 * np.abs(za)) & (np.abs(la - lb) <= 1e-5 * np.abs(la))


def test_tail_split_decodes_like_one_cta_per_frame():
    pkg = load_pkg()
    sig = dabtx.add_awgn(dabtx.freq_shift(dabtx.DabTx(seed=0x7A11, bitrate=BITRATE).frames(FRAMES), 30.0), 18.0, seed=7)
    split, whole = _context(pkg, 0), _context(pkg, -1)
    ds, dw = split.dev(sig), whole.dev(sig)
    tail = np.zeros(S, bool)            # streams whose partial sums the split context added in another order than stream 0's
    decoded = superframes = 0
    for k in range(STEPS):
        x, y = _step(pkg, split, ds, len(sig)), _step(pkg, whole, dw, len(sig))
        rx, ry = x["results"], y["results"]
        # one CTA per frame: every stream exactly as stream 0
        assert (ry == ry[:1]).all(), k
        # the tail split, against that and against its own stream 0: exactly but for the partial sums of the tail
        assert (_without_floats(rx) == _without_floats(ry)).all(), k
        assert (_without_floats(rx) == _without_floats(rx)[:1]).all(), k
        ok = _close(ry, rx)
        assert ok.all(), (k, np.flatnonzero(~ok)[:8])
        for f in FLOATS:
            tail |= rx[f] != ry[f]
        for name in ("fibs", "msc", "sf", "soft"):
            if name == "soft" and x["soft"] is None:
                continue
            assert np.array_equal(x[name], y[name]), (name, k)
            assert (x[name] == x[name][:1]).all(), (name, k)
        decoded += x["soft"] is not None
        superframes += int(rx["sf_ready"][:, 0].sum())
    ds.free(); dw.free()
    split.close(); whole.close()
    assert decoded >= STEPS // 2 and superframes > 0, (decoded, superframes)
    # the default context did cut a tail: a suffix of the batch, at most a quarter of it (half a residency; the batch holds two or more)
    n_tail = int(tail.sum())
    assert 0 < n_tail <= S // 4 and tail[S - n_tail:].all(), np.flatnonzero(tail)[:8]
