"""Plain references for the two integer decoders (TEST TOOLING, numpy only, no ctypes): a K=7 rate-1/4 Viterbi with 64-bit path
metrics that are never renormalised, de-puncturing / de-dispersal / packing, the RS(120,110) syndrome check, and a DAB+ superframe
builder for all four audio formats.  They share no structure with the packed 16-bit kernel (viterbi_core.cuh), with rs.cu or with
oracle/dab_oracle.c, so agreement with them says something; for up to five byte errors per RS column the right answer needs no
decoder at all (the corrected superframe is the one that was built).  Also the adversarial input families and the superframe case
lists that tests/test_decoder_limits.py (CPU emulation, oracle) and tests/test_gpu_decoder_limits.py (the kernels) both run."""
import numpy as np

import dabtx

POLYS = (0o155, 0o117, 0o123, 0o155)
# branch pattern of butterfly i: bit k of the code word emitted on the transition old[i] -> new[2i]
_PAT = np.array([[bin((2 * i) & p).count("1") & 1 for p in POLYS] for i in range(32)], np.int64)
FIC_BLOCKS = [(21, 16), (3, 15)]


# ------------------------------------------------------------------------------------------------ Viterbi
def viterbi_plain(soft, nbits):
    """soft: int8 [(nbits + 6) * 4] or a batch [n, (nbits + 6) * 4] -> (bits, stats).  Symbol clip(s + 127, 0, 255), branch metric
    sum(sym or 255 - sym), start metrics 63 / 0 for state 0, new[2i] = min(old[i] + m, old[i+32] + 1020 - m), new[2i+1] =
    min(old[i] + 1020 - m, old[i+32] + m), decision a > b (a tie keeps old[i]), traceback from state 0 skipping the 6 tail steps.
    stats (per row): `spread` largest max - min over the 64 metrics, `growth24` largest growth of the minimum over 24 consecutive
    steps, `peak24` largest candidate metric relative to the minimum at the last multiple of 24 steps (what a form that subtracts the
    minimum every 24 steps has to hold), `tied` share of decisions with a == b."""
    soft = np.asarray(soft, np.int8)
    single = soft.ndim == 1
    soft = np.atleast_2d(soft)
    n, ns = soft.shape[0], nbits + 6
    assert soft.shape[1] == 4 * ns
    sym = np.clip(soft.astype(np.int64) + 127, 0, 255).reshape(n, ns, 4)
    M = np.full((n, 64), 63, np.int64); M[:, 0] = 0
    dec = np.zeros((ns, n, 64), bool)
    mins = np.zeros((ns + 1, n), np.int64)
    spread = np.zeros(n, np.int64); peak = np.zeros(n, np.int64); tied = np.zeros(n, np.int64)
    base = np.zeros(n, np.int64)
    N = np.empty((n, 64), np.int64)
    for t in range(ns):
        if t % 24 == 0:
            base = M.min(1)
        s = sym[:, t, None, :]
        m = np.where(_PAT[None] == 0, s, 255 - s).sum(2)                  # [n, 32]
        a0 = M[:, :32] + m; b0 = M[:, 32:] + 1020 - m
        a1 = M[:, :32] + 1020 - m; b1 = M[:, 32:] + m
        dec[t, :, 0::2] = a0 > b0; dec[t, :, 1::2] = a1 > b1
        tied += (a0 == b0).sum(1) + (a1 == b1).sum(1)
        peak = np.maximum(peak, np.maximum(np.maximum(a0, b0), np.maximum(a1, b1)).max(1) - base)
        N[:, 0::2] = np.minimum(a0, b0); N[:, 1::2] = np.minimum(a1, b1)
        M, N = N, M
        mins[t + 1] = M.min(1)
        spread = np.maximum(spread, M.max(1) - mins[t + 1])
    state = np.zeros(n, np.int64); rows = np.arange(n)
    bits = np.zeros((n, nbits), np.uint8)
    for t in range(nbits - 1, -1, -1):
        k = dec[t + 6, rows, state]
        state = (state >> 1) | (k.astype(np.int64) << 5)
        bits[:, t] = k
    w = min(24, ns)
    stats = dict(spread=spread, growth24=(mins[w:] - mins[:-w]).max(0), peak24=peak, tied=tied / (64.0 * ns))
    if single:
        return bits[0], {k: v[0] for k, v in stats.items()}
    return bits, stats


def viterbi_families(nbits):
    """name -> int8 [(nbits + 6) * 4]: inputs that hold the decoder at its arithmetic limits (fixed seeds).  As many ties as an input can force, symbols
    pinned at 0 / 254 / the clamp, saturated and near-tie noise, a codeword at full scale with every k-th step inverted (one path grows
    slowly while the rest grow at full rate: the largest metric spread), long runs of zeros inside a codeword (all metrics equal at a
    renormalisation, then divergence), and patterns of period 24 and 6 steps at every phase against the six register layouts."""
    ns = nbits + 6; n = 4 * ns
    rng = np.random.default_rng(1000 + nbits)
    fam = {"zeros": np.zeros(n, np.int8), "p127": np.full(n, 127, np.int8), "m127": np.full(n, -127, np.int8), "m128": np.full(n, -128, np.int8)}
    # an erased step still costs 127 for a 0 and 128 for a 1 (the midpoint 127.5 is no symbol), so no input ties every decision; symbols
    # (128, 128, 128, 127) make the branch metric exactly 510 = 1020 - 510 for half of the butterflies: the most ties a constant input gives
    fam["ties"] = np.tile(np.array([1, 1, 1, 0], np.int8), ns)
    fam["rnd_pm127"] = rng.choice(np.array([-127, 127], np.int8), n)
    fam["rnd_pm127_0"] = rng.choice(np.array([-127, 0, 127], np.int8), n)
    fam["rnd_pm1_0"] = rng.choice(np.array([-1, 0, 1], np.int8), n)
    cw = ((2 * dabtx.conv_encode(rng.integers(0, 2, nbits).astype(np.uint8)).astype(np.int16) - 1) * 127).astype(np.int8).reshape(ns, 4)
    fam["cw"] = cw.reshape(-1).copy()
    for k in (2, 3, 7):
        x = cw.copy(); x[::k] = -x[::k]
        fam[f"cw_inv{k}"] = x.reshape(-1)
    for run in (96, 500):
        r = min(run, ns // 3)
        x = cw.copy(); x[(np.arange(ns) // r) % 2 == 1] = 0
        fam[f"cw_zeros{run}"] = x.reshape(-1)
    for period in (24, 6):
        pat = rng.choice(np.array([-127, 0, 127], np.int8), (period, 4))
        for ph in range(6):
            fam[f"p{period}_ph{ph}"] = np.roll(np.tile(pat, (ns // period + 2, 1)), ph, axis=0)[:ns].reshape(-1).copy()
    return fam


# ------------------------------------------------------------------------------------------------ puncturing, dispersal, packing
def puncture_mask(blocks):
    """blocks: [(L, PI)] - L groups of 128 code bits punctured with vector PI (1..24) - then the 24 tail bits -> bool [4 * (nbits + 6)]"""
    pc = dabtx.pcodes()
    return np.concatenate([np.tile(pc[pi - 1], 4 * L) for L, pi in blocks if L > 0] + [dabtx.PI_TAIL]).astype(bool)


def depuncture(frag, blocks):
    """the punctured softbits of one codeword (or a batch, last axis) -> mother-code order, 0 where nothing was transmitted"""
    mask = puncture_mask(blocks)
    frag = np.asarray(frag, np.int8)
    out = np.zeros(frag.shape[:-1] + (mask.size,), np.int8)
    out[..., mask] = frag[..., :int(mask.sum())]
    return out


def dedisperse(bits):
    return np.asarray(bits, np.uint8) ^ dabtx.prbs(np.shape(bits)[-1])


def pack(bits):
    return np.packbits(np.asarray(bits, np.uint8), axis=-1)


def eep_blocks(bitrate, profile_a, level):
    L1, L2, p1, p2 = dabtx.eep_profile(bitrate, profile_a, level)
    return [(L1, p1), (L2, p2)]


def eep_fits(bitrate, profile_a, level):
    """the EEP profile exists (EEP-A: multiples of 8 kbit/s, EEP-B: of 32) and its sub-channel fits in the 864 CUs of the MSC"""
    return bitrate > 0 and bitrate % (8 if profile_a else 32) == 0 and dabtx.eep_cu(bitrate, profile_a, level) <= 864


def eep_largest(profile_a, level):
    step = 8 if profile_a else 32
    return max(b for b in range(step, 2048, step) if eep_fits(b, profile_a, level))


# either side of 682 kbit/s (16 384 dispersal bits), where a fixed-length dispersal table used to run out
EEP_BOUNDARY = [(1, 680), (1, 688), (0, 672), (0, 704)]


def eep_wide_profiles():
    """(profile_a, bitrate, level) from 200 kbit/s up to the largest of every (A/B, level) - EEP 4-A 1728 kbit/s (41 472 bits per logical
    frame), EEP 4-B 1824 (43 776) - in a stride, with the profiles around 682 kbit/s and the largest ones always in"""
    out = []
    for pa, first, stride in ((1, 200, 136), (0, 224, 224)):
        for lv in (1, 2, 3, 4):
            brs = set(range(first, eep_largest(pa, lv), stride)) | {b for a, b in EEP_BOUNDARY if a == pa} | {eep_largest(pa, lv)}
            out += [(pa, b, lv) for b in sorted(brs) if eep_fits(b, pa, lv)]
    return out


def ref_decodes(bitrate):
    """the reference's Viterbi keeps a logical frame's length in bits as a 16-bit signed integer: above 1365 kbit/s it cannot decode"""
    return 24 * bitrate <= 32767


def eep_wide_soft(profile_a, bitrate, level):
    """seeded random punctured softbits (-127 .. 127) of one logical frame of the profile"""
    n_in = int(puncture_mask(eep_blocks(bitrate, profile_a, level)).sum())
    return np.random.default_rng([profile_a, bitrate, level]).integers(-127, 128, n_in).astype(np.int8)


def fib_crc_ok(fib32):
    """32 FIB bytes: CRC-16-CCITT (preset ones, inverted) of the first 30 equals the last two"""
    return dabtx.crc16(fib32[:30]) == (int(fib32[30]) << 8 | int(fib32[31]))


# ------------------------------------------------------------------------------------------------ Reed-Solomon, CRCs
_EXP = np.zeros(510, np.int64); _LOG = np.zeros(256, np.int64)
_x = 1
for _i in range(255):
    _EXP[_i] = _x; _LOG[_x] = _i
    _x = (_x << 1) ^ (0x11D if _x & 0x80 else 0)
_EXP[255:] = _EXP[:255]


def rs_syndromes(cols):
    """cols [..., 120] -> [..., 10]: the received polynomial (first byte = highest power) at alpha^0 .. alpha^9, GF(2^8) poly 0x11D"""
    cols = np.asarray(cols, np.int64)
    v = np.zeros(cols.shape[:-1] + (10,), np.int64)
    r = np.arange(10)
    for j in range(120):
        v = np.where(v == 0, 0, _EXP[(_LOG[v] + r) % 255]) ^ cols[..., j, None]
    return v


def rs_check(column120):
    return not rs_syndromes(column120).any()


def rs_encode_column(data110):
    return np.concatenate([np.asarray(data110, np.uint8), dabtx.rs_parity(data110)])


def fire_crc(hdr9):
    return dabtx.crc16(hdr9, poly=0x782F, init=0, inv=False)


def au_crc(body):
    return dabtx.crc16(body)


def columns(sf):
    """superframe [120 * S] -> the S interleaved codewords [S, 120]"""
    return np.asarray(sf).reshape(120, -1).T


# ------------------------------------------------------------------------------------------------ DAB+ superframes
FIRST_AU = {2: 5, 3: 6, 4: 8, 6: 11}


def num_aus(dac_rate, sbr_flag):
    return (3 if sbr_flag else 6) if dac_rate else (2 if sbr_flag else 4)


def seal_superframe(sf, fire=True):
    """recompute the Fire code over bytes 2..10 (unless fire=False) and the RS parity of every column, in place"""
    S = len(sf) // 120
    if fire:
        fc = fire_crc(sf[2:11]); sf[0], sf[1] = fc >> 8, fc & 0xFF
    sf[110 * S:] = dabtx.rs_parity(sf[:110 * S].reshape(110, S).T).T.reshape(-1)
    return sf


def build_superframe(rng, bitrate, dac_rate, sbr_flag, au_lens=None, bad_au=None):
    """one DAB+ superframe of `bitrate` kbit/s (S = bitrate / 8 interleaved RS columns) -> (sf uint8 [120 S], truth).  Header: Fire
    code, dac_rate / sbr_flag, the 12-bit start addresses of AUs 1 .. na-1 packed from byte 3 on; na = 2, 3, 4, 6 AUs, the first at
    byte 5, 6, 8, 11; every AU ends with its CRC (inverted for AU `bad_au`); ten parity rows.  au_lens: lengths of the first na - 1 AUs
    (default: an even split of what 12-bit addresses can reach).  truth: num_aus, au_start [na + 1], au_mask (bit i: CRC of AU i good)."""
    S = bitrate // 8; n_data = 110 * S
    na = num_aus(dac_rate, sbr_flag); first = FIRST_AU[na]
    if au_lens is None:
        span = min(n_data, 4096) - first
        a = [first + span * i // na for i in range(na)] + [n_data]
    else:
        a = [first] + [int(x) for x in first + np.cumsum(au_lens[:na - 1])] + [n_data]
    assert all(a[i + 1] - a[i] >= 2 for i in range(na)) and a[na - 1] < 4096, a
    sf = np.zeros(120 * S, np.uint8)
    sf[2] = (dac_rate << 6) | (sbr_flag << 5)
    nib = 6                                          # nibble index of the next 12-bit address (byte 3, high nibble)
    for v in a[1:na]:
        for sh in (8, 4, 0):
            sf[nib >> 1] |= ((v >> sh) & 0xF) << (0 if nib & 1 else 4); nib += 1
    for i in range(na):
        body = rng.integers(0, 256, a[i + 1] - a[i] - 2, dtype=np.uint8)
        if len(body):
            body[0] |= 0xE0                          # first syntactic element ID_END: an AAC decoder behind the check drops the AU cleanly
        c = au_crc(body) ^ (0xFFFF if i == bad_au else 0)
        sf[a[i]:a[i + 1] - 2] = body; sf[a[i + 1] - 2], sf[a[i + 1] - 1] = c >> 8, c & 0xFF
    seal_superframe(sf)
    mask = ((1 << na) - 1) & ~(1 << bad_au if bad_au is not None else 0)
    return sf, dict(num_aus=na, au_start=a, au_mask=mask)


FORMATS = [(0, 0), (0, 1), (1, 0), (1, 1)]
BITRATES = [8, 16, 24, 40, 96, 136, 192, 512]        # S = 1, 2, 3, 5, 12, 17, 24, 64 (the last width the kernel accepts)


def sf_format_cases():
    """(name, sf, truth): every audio format at every width, clean and with one AU's CRC broken"""
    out = []
    for k, (br, (dac, sbr)) in enumerate((b, f) for b in BITRATES for f in FORMATS):
        rng = np.random.default_rng(5000 + k)
        na = num_aus(dac, sbr)
        out.append((f"fmt_{br}_{dac}{sbr}_clean",) + build_superframe(rng, br, dac, sbr))
        out.append((f"fmt_{br}_{dac}{sbr}_bad{k % na}",) + build_superframe(rng, br, dac, sbr, bad_au=k % na))
    return out


def _hit(rng, sf, col, rows):
    S = len(sf) // 120
    sf[np.asarray(rows) * S + col] ^= rng.integers(1, 256, len(rows)).astype(np.uint8)


def sf_error_cases():
    """(name, received, sent, truth, errors_per_column): a chosen number of byte errors in chosen columns and rows"""
    out = []
    for k, (br, (dac, sbr)) in enumerate([(8, (1, 0)), (24, (0, 1)), (96, (0, 0)), (136, (1, 1)), (512, (1, 0))]):
        S = br // 8
        rng = np.random.default_rng(7000 + k)
        sent, truth = build_superframe(rng, br, dac, sbr)

        def case(name, per_col, pick=lambda n: rng.choice(120, n, replace=False)):
            rx = sent.copy()
            for c, n in enumerate(per_col):
                if n:
                    _hit(rng, rx, c, pick(n))
            out.append((f"err_{br}_{dac}{sbr}_{name}", rx, sent, truth, list(per_col)))
        one = lambda n, c: [n if i == c else 0 for i in range(S)]
        for n in range(1, 6):
            case(f"{n}_in_col", one(n, (n * 7) % S))
        case("5_everywhere", [5] * S)
        case("5_in_parity", one(5, S - 1), lambda n: 110 + rng.choice(10, n, replace=False))
        case("5_in_header", one(5, 0), lambda n: np.arange(n))           # rows 0..4 of column 0: the Fire code must pass after correction
        case("6_in_col", one(6, S // 2))
        case("10_in_col", one(10, S // 3))
    return out


def sf_reject_cases():
    """(name, sf): superframes whose RS columns are all valid but whose header must not synchronise"""
    out = []
    for k, (br, (dac, sbr)) in enumerate([(96, (1, 0)), (24, (0, 0)), (8, (0, 1)), (192, (1, 1))]):
        rng = np.random.default_rng(9000 + k)
        sf, truth = build_superframe(rng, br, dac, sbr)
        na, a, n_data = truth["num_aus"], truth["au_start"], 110 * (br // 8)
        x = sf.copy(); x[3] = 0; x[4] = 0
        out.append((f"rej_{br}_{dac}{sbr}_zero_start", seal_superframe(x)))
        for bit in range(16):
            x = sf.copy(); x[bit >> 3] ^= 0x80 >> (bit & 7)
            out.append((f"rej_{br}_{dac}{sbr}_fire_bit{bit}", seal_superframe(x, fire=False)))
        # the first address: equal to the first AU's start, below it, at and beyond the end of the data (12 bits allowing)
        for tag, v in (("equal", a[0]), ("decreasing", a[0] - 1), ("at_end", n_data), ("beyond", n_data + 7)):
            if v < 4096:
                x = sf.copy(); x[3] = v >> 4; x[4] = (x[4] & 0x0F) | ((v & 0xF) << 4)
                out.append((f"rej_{br}_{dac}{sbr}_au1_{tag}", seal_superframe(x)))
        if na >= 3:                                  # the second address equal to / below the first
            for tag, v in (("equal", a[1]), ("decreasing", a[1] - 3)):
                x = sf.copy(); x[4] = (x[4] & 0xF0) | (v >> 8); x[5] = v & 0xFF
                out.append((f"rej_{br}_{dac}{sbr}_au2_{tag}", seal_superframe(x)))
    return out


def sf_all_inputs():
    """(name, superframe as received) over the three case lists"""
    return [(c[0], c[1]) for c in sf_format_cases() + sf_error_cases() + sf_reject_cases()]
