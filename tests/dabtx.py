"""Synthetic DAB Mode-I transmitter (TEST TOOLING — the reference has no modulator/encoder).

Builds ETSI EN 300 401 transmission frames in numpy: FIBs (FIG 0/1 + FIG 0/2) -> energy dispersal -> K=7 rate-1/4
convolutional code -> puncturing -> FIC;  DAB+ superframes (Fire code, AU CRCs, RS(120,110) parity) -> dispersal ->
conv. code -> EEP puncturing -> 16-CIF time interleaving -> CIFs;  frequency interleaving -> pi/4-DQPSK against the
phase reference symbol -> IFFT + cyclic prefix -> null symbol.  All tables are derived here from the ETSI rules,
independently of the oracle and of the product, so encode -> decode round trips are meaningful.
The recipe was validated against the unmodified reference backend (SURVEY.md §7 step 2, tests/test_oracle_vs_ref.py).
"""
import numpy as np

L, K, TU, TG, TS, TNULL, TF = 76, 1536, 2048, 504, 2552, 2656, 196608
POLYS = (0o155, 0o117, 0o123, 0o155)
DEINT_MAP = np.array([0, 8, 4, 12, 2, 10, 6, 14, 1, 9, 5, 13, 3, 11, 7, 15])


# ---------------------------------------------------------------- tables
def perm_table():
    pi, out = 0, []
    for i in range(TU):
        if i:
            pi = (13 * pi + 511) % TU
        if pi == TU // 2 or pi < 256 or pi > 256 + K:
            continue
        out.append(pi - TU // 2)
    return np.array(out, np.int64)


_PRS_I = [0, 1, 2, 3] * 6 + [0, 3, 2, 1] * 6
_PRS_N = [1, 2, 0, 1, 3, 2, 2, 3, 2, 1, 2, 3, 1, 2, 3, 3, 2, 2, 2, 1, 1, 3, 1, 2,
          3, 1, 1, 1, 2, 2, 1, 0, 2, 2, 3, 3, 0, 2, 1, 3, 3, 3, 3, 0, 3, 0, 1, 1]
_PRS_H = [[0, 2, 0, 0, 0, 0, 1, 1, 2, 0, 0, 0, 2, 2, 1, 1], [0, 3, 2, 3, 0, 1, 3, 0, 2, 1, 2, 3, 2, 3, 3, 0],
          [0, 0, 0, 2, 0, 2, 1, 3, 2, 2, 0, 2, 2, 0, 1, 3], [0, 1, 2, 1, 0, 3, 3, 2, 2, 3, 2, 1, 2, 1, 3, 2]]


def prs_spectrum():
    z = np.zeros(TU, np.complex128)
    for k in list(range(-768, 0)) + list(range(1, 769)):
        if k < 0:
            b = (k + 768) // 32; kmin = -768 + 32 * b
        else:
            b = 24 + (k - 1) // 32; kmin = 1 + 32 * (b - 24)
        q = (_PRS_H[_PRS_I[b]][(k - kmin) & 15] + _PRS_N[b]) & 3
        z[k % TU] = 1j ** q
    return z


def pcodes():
    order = [0, 4, 2, 6, 1, 5, 3, 7]
    t = np.zeros((24, 32), np.uint8)
    for p in range(1, 25):
        t[p - 1, 0::4] = 1
        for q in range(1, p + 1):
            t[p - 1, 4 * order[(q - 1) & 7] + 1 + (q - 1) // 8] = 1
    return t


PI_TAIL = np.array([1, 1, 0, 0] * 6, np.uint8)


def prbs(n):
    reg, out = 0x1FF, np.zeros(n, np.uint8)
    for i in range(n):
        b = ((reg >> 8) ^ (reg >> 4)) & 1
        reg = ((reg << 1) | b) & 0x1FF
        out[i] = b
    return out


# ---------------------------------------------------------------- coding
def conv_encode(bits):
    b = np.concatenate([np.zeros(6, np.uint8), np.asarray(bits, np.uint8), np.zeros(6, np.uint8)])
    n = len(bits) + 6
    out = np.zeros((n, 4), np.uint8)
    for k, p in enumerate(POLYS):
        acc = np.zeros(n, np.uint8)
        for j in range(7):
            if (p >> j) & 1:
                acc ^= b[6 - j: 6 - j + n]
        out[:, k] = acc
    return out.reshape(-1)


def crc16(data, poly=0x1021, init=0xFFFF, inv=True):
    crc = init
    for byte in bytes(bytearray(data)):
        crc ^= byte << 8
        for _ in range(8):
            crc = ((crc << 1) ^ poly) & 0xFFFF if crc & 0x8000 else (crc << 1) & 0xFFFF
    return (~crc) & 0xFFFF if inv else crc


_GF_EXP = np.zeros(512, np.int64)
_GF_LOG = np.zeros(256, np.int64)
_x = 1
for _i in range(255):
    _GF_EXP[_i] = _x; _GF_LOG[_x] = _i
    _x <<= 1
    if _x & 0x100:
        _x ^= 0x11D
_GF_EXP[255:510] = _GF_EXP[:255]


def gf_mul(a, b):
    a = np.asarray(a, np.int64); b = np.asarray(b, np.int64)
    r = _GF_EXP[(_GF_LOG[a] + _GF_LOG[b]) % 255]
    return np.where((a == 0) | (b == 0), 0, r)


def rs_genpoly():
    g = np.array([1], np.int64)
    for i in range(10):
        root = _GF_EXP[i]
        g = np.concatenate([[0], g]) ^ np.concatenate([gf_mul(g, root), [0]])   # (x + root) * g, g[0] = const term
    return g   # g[0..10], g[10] = 1


def rs_parity(data):
    """data [..., 110] uint8 -> parity [..., 10]; systematic RS(120,110), roots alpha^0..alpha^9, GF poly 0x11D"""
    data = np.asarray(data, np.int64)
    g = rs_genpoly()
    par = np.zeros(data.shape[:-1] + (10,), np.int64)
    for i in range(110):
        fb = data[..., i] ^ par[..., 0]
        par = np.concatenate([par[..., 1:], np.zeros_like(par[..., :1])], axis=-1)
        par ^= gf_mul(fb[..., None], g[9::-1][None, ...] if par.ndim > 1 else g[9::-1])
    return par.astype(np.uint8)


# ---------------------------------------------------------------- protection profiles (EEP)
def eep_profile(bitrate, profile_a=True, level=3):
    b = bitrate
    if profile_a:
        tab = {1: (6 * b // 8 - 3, 3, 24, 23), 2: ((5, 1, 13, 12) if b == 8 else (2 * b // 8 - 3, 4 * b // 8 + 3, 14, 13)),
               3: (6 * b // 8 - 3, 3, 8, 7), 4: (4 * b // 8 - 3, 2 * b // 8 + 3, 3, 2)}[level]
    else:
        pi = {1: (10, 9), 2: (6, 5), 3: (4, 3), 4: (2, 1)}[level]
        tab = (24 * b // 32 - 3, 3) + pi
    return tab   # L1, L2, PI1, PI2


def eep_cu(bitrate, profile_a=True, level=3):
    if profile_a:
        return {1: bitrate * 12 // 8, 2: bitrate, 3: bitrate * 6 // 8, 4: bitrate // 2}[level]
    return {1: bitrate * 27 // 32, 2: bitrate * 21 // 32, 3: bitrate * 18 // 32, 4: bitrate * 15 // 32}[level]


def puncture_mask(blocks):
    """blocks: list of (L, PI index 1..24)"""
    pc = pcodes()
    parts = [np.tile(pc[pi - 1], 4 * Lk) for Lk, pi in blocks if Lk > 0]
    return np.concatenate(parts + [PI_TAIL]).astype(bool)


FIC_MASK = puncture_mask([(21, 16), (3, 15)])


# ---------------------------------------------------------------- FIC content
def make_fib(payload):
    pl = list(payload) + [0xFF]
    pl += [0] * (30 - len(pl))
    c = crc16(pl)
    return np.unpackbits(np.array(pl + [c >> 8, c & 0xFF], np.uint8))


def fig0_1(subch_id, start_cu, eep_a, level, size_cu):
    # long form: SubChId(6) StartAddr(10) | 1 Option(3) ProtLevel(2) SubChSize(10)
    w = (subch_id << 10) | start_cu
    opt = 0 if eep_a else 1
    w2 = 0x8000 | (opt << 12) | ((level - 1) << 10) | size_cu
    return [0x05, 0x01, w >> 8, w & 0xFF, w2 >> 8, w2 & 0xFF]


def fig0_2(sid, subch_id, ascty=63):
    return [0x06, 0x02, sid >> 8, sid & 0xFF, 0x01, ascty & 0x3F, (subch_id << 2) | 0x02]


class DabTx:
    """One ensemble with one DAB+ sub-channel (EEP) in CUs [start_cu, start_cu + size); dabplus=False: the sub-channel carries random
    logical frames instead of superframes (DAB content, any bitrate)."""

    def __init__(self, seed=0xDAB, bitrate=96, profile_a=True, level=3, start_cu=0, subch_id=0, sid=0x1001, amplitude=0.1, period_sf=0, dabplus=True):
        self.period_sf = period_sf          # >0: content repeats every period_sf superframes (= 5*period_sf CIFs): an endless periodic stream
        self.dabplus = dabplus
        self._sf_cache, self._fill_cache = {}, {}
        self.rng = np.random.default_rng(seed)
        self.bitrate, self.profile_a, self.level = bitrate, profile_a, level
        self.start_cu, self.size_cu = start_cu, eep_cu(bitrate, profile_a, level)
        self.S = bitrate // 8
        self.perm = perm_table()
        self.bins = self.perm % TU
        self.prs = prs_spectrum()
        L1, L2, p1, p2 = eep_profile(bitrate, profile_a, level)
        self.msc_mask = puncture_mask([(L1, p1), (L2, p2)])
        assert self.msc_mask.sum() == self.size_cu * 64, (self.msc_mask.sum(), self.size_cu * 64)
        self.prbs_fic = prbs(768)
        self.prbs_msc = prbs(24 * bitrate)
        self.fib = make_fib(fig0_1(subch_id, start_cu, profile_a, level, self.size_cu) + fig0_2(sid, subch_id))
        self.ficblk = conv_encode(np.tile(self.fib, 3) ^ self.prbs_fic)[FIC_MASK]
        assert self.ficblk.size == 2304
        self.amp = amplitude
        self._coded_hist = []     # coded logical frames for the time interleaver
        self.logical = []         # transmitted logical frames (bytes)
        self.superframes = []
        self._sf_queue = np.zeros(0, np.uint8)
        self.cif_count = 0

    # ---- DAB+ superframe
    def superframe(self, bad_au=None, au_starts=None):
        """one DAB+ superframe (dac_rate=1, sbr=0: 6 AUs); au_starts = the five explicit AU start addresses (else even, as far as the
        header's 12-bit addresses reach: above 44 RS columns the first five AUs share bytes 11 .. 4095 evenly and the sixth takes the rest)"""
        S = self.S; n_data = 110 * S
        sf = np.zeros(120 * S, np.uint8)
        au = [11] + [11 + (n_data - 11) * i // 6 for i in range(1, 6)] + [n_data]
        if au[5] > 4095:
            au = [11] + [11 + (4096 - 11) * i // 6 for i in range(1, 6)] + [n_data]
        if au_starts is not None:
            au = [11] + [int(x) for x in au_starts] + [n_data]
        sf[2] = 0x40
        a = au
        sf[3] = a[1] >> 4; sf[4] = ((a[1] & 0xF) << 4) | (a[2] >> 8); sf[5] = a[2] & 0xFF
        sf[6] = a[3] >> 4; sf[7] = ((a[3] & 0xF) << 4) | (a[4] >> 8); sf[8] = a[4] & 0xFF
        sf[9] = a[5] >> 4; sf[10] = (a[5] & 0xF) << 4
        fc = crc16(sf[2:11], poly=0x782F, init=0, inv=False)
        sf[0], sf[1] = fc >> 8, fc & 0xFF
        for i in range(6):
            ln = a[i + 1] - a[i]
            body = self.rng.integers(0, 256, max(ln - 2, 0), dtype=np.uint8)
            if ln < 2:
                continue
            # first syntactic element = ID_END (111): the reference's AAC decoder (out of scope) rejects the AU cleanly instead of
            # mis-parsing random bytes (which can make it throw, dabplus_decoder.cpp:460), and no PAD is signalled (:148-149)
            if len(body):
                body[0] |= 0xE0
            c = crc16(body)
            if bad_au is not None and i == bad_au:
                c ^= 0xFFFF
            sf[a[i]:a[i + 1] - 2] = body; sf[a[i + 1] - 2] = c >> 8; sf[a[i + 1] - 1] = c & 0xFF
        cols = sf[:n_data].reshape(110, S).T       # column i = sf[i::S]
        sf[n_data:] = rs_parity(cols).T.reshape(-1)
        return sf

    def _next_logical(self):
        flen = 3 * self.bitrate
        if not self.dabplus:
            return self.rng.integers(0, 256, flen, dtype=np.uint8)
        if len(self._sf_queue) < flen:
            k = len(self.superframes)
            if self.period_sf:
                if k % self.period_sf not in self._sf_cache:
                    self._sf_cache[k % self.period_sf] = self.superframe()
                sf = self._sf_cache[k % self.period_sf]
            else:
                sf = self.superframe()
            self.superframes.append(sf)
            self._sf_queue = np.concatenate([self._sf_queue, sf])
        fr, self._sf_queue = self._sf_queue[:flen], self._sf_queue[flen:]
        return fr

    def _next_cif_subch(self):
        fr = self._next_logical()
        self.logical.append(fr)
        coded = conv_encode(np.unpackbits(fr) ^ self.prbs_msc)[self.msc_mask]
        self._coded_hist.append(coded)
        if len(self._coded_hist) > 16:
            self._coded_hist.pop(0)
        n = len(coded); idx = np.arange(n); delay = DEINT_MAP[idx & 15]
        out = np.zeros(n, np.uint8)
        h = self._coded_hist
        for d in range(16):
            if d < len(h):
                sel = delay == d
                out[sel] = h[len(h) - 1 - d][sel]
        self.cif_count += 1
        return out

    def frame_bits(self):
        """75 x 3072 bits for one transmission frame"""
        fic = np.tile(self.ficblk, 4)
        cifs = []
        for _ in range(4):
            if self.period_sf:
                key = self.cif_count % (5 * self.period_sf)
                if key not in self._fill_cache:
                    self._fill_cache[key] = self.rng.integers(0, 2, 864 * 64, dtype=np.uint8)
                cif = self._fill_cache[key].copy()
            else:
                cif = self.rng.integers(0, 2, 864 * 64, dtype=np.uint8)
            sub = self._next_cif_subch()
            cif[self.start_cu * 64: self.start_cu * 64 + len(sub)] = sub
            cifs.append(cif)
        return np.concatenate([fic, np.concatenate(cifs)]).reshape(75, 3072)

    def tii_null(self):
        """the null symbol with the transmitter identification carriers of self.tii = [(comb, pattern, delay_samples, gain), ...]
        (EN 300 401 clause 14.8: pairs of adjacent carriers k, k + 1, both with the phase of the phase reference symbol's carrier k, in four
        blocks of 384 carriers; pattern p = the p-th 8-bit word with four ones picks which of the eight groups of a comb are on)"""
        pats = [w for w in range(256) if bin(w).count("1") == 4]
        Z = np.zeros(TU, np.complex128)
        for comb, pattern, delay, gain in self.tii:
            z = np.zeros(TU, np.complex128)
            for b in range(8):
                if (pats[pattern] >> (7 - b)) & 1:
                    k0 = 1 + 2 * comb + 48 * b
                    for k in (k0 - 769, k0 - 385, k0, k0 + 384):
                        z[k % TU] = self.prs[k % TU]; z[(k + 1) % TU] = self.prs[k % TU]
            kk = np.fft.fftfreq(TU, 1.0 / TU)
            Z += gain * z * np.exp(-2j * np.pi * kk * delay / TU)
        x = np.fft.ifft(Z) * (TU / np.sqrt(K) * self.amp)
        return np.concatenate([x[-(TNULL - TU):], x])

    def modulate(self, bits75):
        out = np.zeros(TF, np.complex128)
        if getattr(self, "tii", None):
            out[:TNULL] = self.tii_null()
        Z = self.prs.copy()
        scale = TU / np.sqrt(K) * self.amp
        pos = TNULL
        for l in range(L):
            if l:
                b = bits75[l - 1]
                y = ((1 - 2.0 * b[:K]) + 1j * (1 - 2.0 * b[K:])) / np.sqrt(2)
                Zn = np.zeros(TU, np.complex128); Zn[self.bins] = Z[self.bins] * y; Z = Zn
            x = np.fft.ifft(Z) * scale
            out[pos:pos + TG] = x[-TG:]; out[pos + TG:pos + TS] = x
            pos += TS
        return out

    def frames(self, n, noise_floor=1e-6):
        sig = np.concatenate([self.modulate(self.frame_bits()) for _ in range(n)])
        if noise_floor:
            sig = sig + (self.rng.standard_normal(len(sig)) + 1j * self.rng.standard_normal(len(sig))) * noise_floor
        return sig.astype(np.complex64)


def add_awgn(iq, snr_db, seed, signal_power=None):
    rng = np.random.default_rng(seed)
    p = signal_power if signal_power is not None else float(np.mean(np.abs(iq) ** 2))
    sigma = np.sqrt(p / (10 ** (snr_db / 10)) / 2)
    n = (rng.standard_normal(len(iq)) + 1j * rng.standard_normal(len(iq))) * sigma
    return (iq + n).astype(np.complex64)


def freq_shift(iq, hz):
    n = np.arange(len(iq))
    return (iq * np.exp(2j * np.pi * hz * n / 2048000.0)).astype(np.complex64)


def periodic_ring(seed, n_frames=5, **kw):
    """n_frames (multiple of 5) frames of a steady-state stream that repeats seamlessly: frames [n, 2n) of a
    transmitter whose content has period n frames (time interleaver and superframes wrap consistently)."""
    assert n_frames % 5 == 0
    tx = DabTx(seed=seed, period_sf=4 * n_frames // 5, **kw)
    sig = np.concatenate([tx.modulate(tx.frame_bits()) for _ in range(2 * n_frames)])
    return tx, sig[n_frames * TF:].astype(np.complex64)


def fib_bytes(tx):
    return np.packbits(tx.fib)
