"""numpy restatement of diversity combining (dabb_set_combining, include/dab_b200.h), TEST TOOLING.

noise(y): N = mean |y|^2 of a null symbol in float64, noise_f32(y) the same in the library's float32 order.  select(): the contributor rule.  combined(): R = sum over the contributors of
r1_b / N_b in float64 (ascending stream order), and soft(): the reference or weighted demap of R in float64 (softbit 0 where the value is
not finite).  combined_f32() is the same sum in float32 with every operation rounded in the library's order, so that the order of the
contributors can be checked bit for bit."""
import numpy as np

K, TNULL, MAX_OFFSET = 1536, 2656, 504
TINY = 2.0 ** -126
COMBINE_DTYPE = np.dtype([("members", "<i4"), ("mask", "<u4"), ("noise", "<f4"), ("reserved", "<i4")])


def noise(y):
    """N of null symbols y [..., TNULL] (complex) in float64"""
    y = np.asarray(y).astype(np.complex128)
    with np.errstate(all="ignore"):
        return np.mean(y.real ** 2 + y.imag ** 2, axis=-1)


def noise_f32(y):
    """N of null symbols y [..., TNULL] in the library's float32 order: the partial sums of Re^2 + Im^2 over i = t mod 256 in ascending
    i, then the 256 partials in order, divided by TNULL (each operation rounded): bit for bit the library's value"""
    y = np.asarray(y).astype(np.complex64)
    lead = y.shape[:-1]
    re, im = y.real.astype(np.float32), y.imag.astype(np.float32)
    with np.errstate(all="ignore"):
        p = ((re * re).astype(np.float32) + (im * im).astype(np.float32)).astype(np.float32)
        pad = np.zeros(lead + (256 * 11,), np.float32)
        pad[..., :TNULL] = p
        part = np.zeros(lead + (256,), np.float32)
        for k in range(11):
            part = (part + pad[..., 256 * k:256 * k + 256]).astype(np.float32)
        tot = np.zeros(lead, np.float32)
        for t in range(256):
            tot = (tot + part[..., t]).astype(np.float32)
        return (tot / np.float32(TNULL)).astype(np.float32)


def noise_ok(n):
    return bool(np.isfinite(n) and n > 0)


def select(decoded, a, nz, lpos):
    """bit i: member i (ascending stream order) contributes"""
    if not decoded[lpos]:
        return 0
    if not noise_ok(nz[lpos]):
        return 1 << lpos
    m = 0
    for i in range(len(decoded)):
        if i == lpos or (decoded[i] and noise_ok(nz[i]) and abs(int(a[i]) - int(a[lpos])) <= MAX_OFFSET):
            m |= 1 << i
    return m


def combined(r1, nz, mask):
    """R [..., K] complex128 from the members' r1 [n, ..., K] and noise [n]"""
    r = np.asarray(r1).astype(np.complex128)
    R = np.zeros(r.shape[1:], np.complex128)
    for i in range(r.shape[0]):
        if (mask >> i) & 1:
            R += r[i] / float(nz[i])
    return R


def combined_f32(r1, nz, mask, order=None):
    """the same sum in float32 with each division and addition rounded, members added in `order` (default ascending)"""
    r = np.asarray(r1).astype(np.complex64)
    re = np.zeros(r.shape[1:], np.float32); im = np.zeros(r.shape[1:], np.float32)
    for i in (range(r.shape[0]) if order is None else order):
        if (mask >> i) & 1:
            n = np.float32(nz[i])
            with np.errstate(all="ignore"):
                re = (re + (r[i].real.astype(np.float32) / n).astype(np.float32)).astype(np.float32)
                im = (im + (r[i].imag.astype(np.float32) / n).astype(np.float32)).astype(np.float32)
    out = np.empty(re.shape, np.complex64)                # (re + 1j * im would turn an infinite im into a NaN re)
    out.real, out.imag = re, im
    return out


def exact(R, weighted):
    """float64 values -Re/Im(R) * 127 / max(l1, G) (G = 0 for the reference demap): [..., 2 K]"""
    R = np.asarray(R).astype(np.complex128)
    re, im = R.real, R.imag
    with np.errstate(all="ignore"):
        l1 = np.abs(re) + np.abs(im)
        g = np.zeros(l1.shape[:-1])
        if weighted:
            g = np.exp2(np.mean(np.log2(np.maximum(l1, TINY)), axis=-1))
            g = np.where(np.isfinite(g), g, 0.0)
        q = 127.0 / np.maximum(l1, g[..., None])
        return np.concatenate([-re * q, -im * q], axis=-1)


def soft(R, weighted):
    v = exact(R, weighted)
    with np.errstate(all="ignore"):
        ok = np.isfinite(v)
        return np.where(ok, np.trunc(np.where(ok, v, 0.0)), 0.0).astype(np.int8)


def compare(got, R, weighted, rate):
    """softbits `got` [..., 2 K] against soft(R): every difference at most 1, and at most `rate` of the softbits differ (they sit at
    rounding boundaries: the float32 and float64 values truncate to neighbouring integers).  Returns the fraction that differ."""
    want = soft(R, weighted).astype(int)
    d = np.abs(np.asarray(got).astype(int) - want)
    assert d.max(initial=0) <= 1, int(d.max())
    frac = float((d != 0).mean()) if d.size else 0.0
    assert frac <= rate, frac
    return frac
