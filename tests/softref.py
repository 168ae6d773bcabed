"""numpy restatement of the weighted soft-decision demap (DABB_DEMAP_WEIGHTED, include/dab_b200.h), TEST TOOLING.  Per symbol,
l1 = |Re r1| + |Im r1| in float32 (as the demodulator rounds it), G = 2^(mean log2 max(l1, 2^-126)) in float64 (0 where not finite),
softbit = trunc(-Re/Im(r1) * 127 / max(l1, G)) in float64, 0 where that or the float32 quotient 127 / max(l1, G) is not finite.  check() compares a device or host result with
it: carriers with l1 >= G (1 + 1e-5) must equal the reference demap exactly, the others the restatement, except where the exact value
lies within 1e-4 of an integer (or the carrier is within 1e-5 of G, where either mode's value is accepted)."""
import numpy as np

K = 1536
TINY = 2.0 ** -126


def levels(r1):
    """r1: complex [..., K] (rounded to complex64) -> (re, im, l1) as float32"""
    r = np.asarray(r1).astype(np.complex64)
    re, im = r.real.astype(np.float32), r.imag.astype(np.float32)
    return re, im, (np.abs(re) + np.abs(im)).astype(np.float32)


def gmean(l1):
    """G per symbol (float64) of float32 levels [..., K]"""
    with np.errstate(all="ignore"):
        g = np.exp2(np.mean(np.log2(np.maximum(l1.astype(np.float64), TINY)), axis=-1))
    return np.where(np.isfinite(g), g, 0.0)


def _trunc(v):
    with np.errstate(all="ignore"):
        ok = np.isfinite(v)
        return np.where(ok, np.trunc(np.where(ok, v, 0.0)), 0.0).astype(np.int8)


def exact(r1, weighted=True):
    """float64 values -Re/Im * 127 / max(l1, G) (or / l1): ([..., K], [..., K]) and G"""
    re, im, l1 = levels(r1)
    g = gmean(l1) if weighted else np.zeros(l1.shape[:-1])
    m = np.maximum(l1.astype(np.float64), g[..., None])
    with np.errstate(all="ignore"):
        q = 127.0 / m
        q[q > np.finfo(np.float32).max] = np.inf           # 127 / max(l1, G) is a float32: beyond its range the softbit is 0
        return -re.astype(np.float64) * q, -im.astype(np.float64) * q, g


def soft(r1, weighted=True):
    """softbits [..., 2 K] in the reference layout (K Re bits, then K Im bits)"""
    a, b, _ = exact(r1, weighted)
    return np.concatenate([_trunc(a), _trunc(b)], axis=-1)


def soft_reference_f32(r1):
    """the reference demap in float32 arithmetic: trunc(-Re/Im * fl(127 / l1)) (ofdm_core.cuh demap_one)"""
    re, im, l1 = levels(r1)
    with np.errstate(all="ignore"):
        q = np.float32(127.0) / l1
        return np.concatenate([_trunc((-re * q).astype(np.float64)), _trunc((-im * q).astype(np.float64))], axis=-1)


def check(r1, got, g_got=None, band=1e-4, g_tol=1e-5):
    """asserts that softbits `got` [..., 2 K] are the weighted demap of r1 [..., K]; returns the number of weak carriers checked"""
    re, im, l1 = levels(r1)
    a, b, g = exact(r1)
    if g_got is not None:
        gg = np.asarray(g_got, np.float64)
        assert np.all((gg == 0) == (g == 0)), "G = 0 differs"
        nz = g > 0
        assert np.all(np.abs(gg[nz] - g[nz]) <= g_tol * g[nz]), float(np.max(np.abs(gg[nz] - g[nz]) / g[nz]))
    got = np.asarray(got).astype(np.int8)
    ref = soft_reference_f32(r1)
    gw = g[..., None]
    strong = np.concatenate([l1 >= gw * (1 + g_tol)] * 2, axis=-1) | np.concatenate([np.broadcast_to(gw == 0, l1.shape)] * 2, axis=-1)
    assert np.array_equal(got[strong], ref[strong]), int((got[strong] != ref[strong]).sum())
    v = np.concatenate([a, b], axis=-1)
    want = soft(r1)
    with np.errstate(all="ignore"):
        near = np.abs(v - np.round(v)) <= band
    edge = np.concatenate([(l1 >= gw * (1 - g_tol)) & (l1 < gw * (1 + g_tol))] * 2, axis=-1)
    weak = ~strong & ~near
    ok = (got == want) | (edge & (got == ref))
    bad = weak & ~ok
    assert not bad.any(), (int(bad.sum()), got[bad][:8], want[bad][:8], v[bad][:8])
    return int(weak.sum())
