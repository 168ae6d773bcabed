"""Robust acquisition (dabb_options.acquisition = DABB_ACQ_ROBUST) on the device.

DABB_ACQ_REFERENCE is what a context that never sets the option runs (same outputs, 14 launches per step).  Tap 13 equals the host build
of acq_core.cuh (tests/host_emul/emul_acq.cpp) bit for bit on the same samples, whatever the batch size or stream index.  On 20 dB
recordings both methods decode the same frames with identical FIBs and tap-0 softbits; at 0 dB, and beside an off-grid tone 10 and 20 dB
above the ensemble, ROBUST acquires and keeps sync where REFERENCE does not.  Noise-only streams keep searching and count acq_failed.
Also: buffers that end inside the null, dabb_stream_reset and method switches in the middle of a search, the three placements,
dabb_submit, and two antennas at 0 dB each that acquire on the same frame and combine."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import acqref
import dabtx
import ofdmref
from conftest import ROOT, load_pkg

pytestmark = pytest.mark.gpu
TF, TNULL = 196608, 2656
NEED = 198151           # plan_kernel's `need`: the least a step's buffer holds


@pytest.fixture(scope="module")
def pkg():
    return load_pkg()


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_acq_gpu") / "libemul_acq.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-o", so,
                           os.path.join(ROOT, "tests", "host_emul", "emul_acq.cpp")])
    lib = C.CDLL(so)
    lib.emul_acq_levels.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    lib.emul_acq_decide.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def recording(seed, frames, snr=None, noise_seed=1, tone=None, chan=None):
    clean = dabtx.DabTx(seed=seed).frames(frames, noise_floor=0)
    p = float(np.mean(np.abs(clean) ** 2))
    x = ofdmref.multipath(clean, chan) if chan else clean
    if snr is not None:
        x = dabtx.add_awgn(x, snr, seed=noise_seed, signal_power=p)
    if tone is not None:
        x = acqref.tone(x, *tone)
    return np.asarray(x, np.complex64)


def run(pkg, rec, steps, robust=True, buf_len=None, start=None, taps=(), submit=False, opts=None, between=None, **kw):
    """steps of a context over rec [S, N]; buf_len None: the whole recording is every step's buffer, else each step's buffer is
    buf_len samples from the stream's next_pos.  Per step: the outputs, the launches and the taps asked for"""
    S, N = rec.shape
    ctx = pkg.Context(n_streams=S, **kw)
    o = dict(opts or {})
    if robust:
        o["acquisition"] = pkg.ACQ_ROBUST
    if o:
        ctx.set_options(**o)
    pos = np.zeros(S, np.int64) if start is None else np.asarray(start, np.int64)
    if start is not None:
        for s in range(S):
            ctx.reset(s, 1, int(pos[s]))
    d = ctx.dev(rec) if buf_len is None and not submit else None
    outs = []
    for k in range(steps):
        if between:
            pos = between(ctx, k, pos)
        n0 = ctx.kernel_launches()
        if buf_len is None and not submit:
            out = ctx.process(d, N, np.zeros(S, np.int64), N)
        else:
            L = buf_len or N
            bs = pos if buf_len else np.zeros(S, np.int64)
            win = np.zeros((S, L), np.complex64)
            for s in range(S):
                a = rec[s, max(bs[s], 0):max(bs[s], 0) + L]
                win[s, :len(a)] = a
            if submit:
                ctx.submit(win, L, bs, L)
                out = ctx.collect()
            else:
                out = ctx.process(win, L, bs, L, iq_is_host=True)
        out["launches"] = ctx.kernel_launches() - n0
        for t in taps:
            out[t] = ctx.read_tap(t)
        pos = out["results"]["next_pos"].copy()
        outs.append(out)
    if d:
        d.free()
    ctx.close()
    return outs


def frames_by_pos(outs, s):
    """stream s's decoded frames keyed by the logical position that follows them"""
    return {int(o["results"]["next_pos"][s]): o for o in outs if o["results"]["status"][s] == 0}


def test_reference_unchanged(pkg):
    rec = np.stack([recording(0xA100, 4, 20.0), recording(0xA101, 4, 3.0, noise_seed=2)])
    a = run(pkg, rec, 5, robust=False)
    b = run(pkg, rec, 5, robust=False, opts={"acquisition": pkg.ACQ_REFERENCE})
    for x, y in zip(a, b):
        assert np.array_equal(x["fibs"], y["fibs"]) and np.array_equal(x["results"].view(np.uint8), y["results"].view(np.uint8))
        assert x["launches"] == y["launches"] == a[0]["launches"]
    c = run(pkg, rec, 3)
    assert [o["launches"] for o in c] == [a[0]["launches"] + 2] * 3      # acq_plan, acq_level, acq_decide in place of acquire_kernel
    ctx = pkg.Context(n_streams=1)
    with pytest.raises(pkg.DabbError):
        ctx.read_tap(13)
    o = pkg.Options(); o.disable_coarse = 1; o.acquisition = 2
    assert ctx.lib.dabb_set_options(ctx.h, C.byref(o)) == -3
    with pytest.raises(pkg.DabbError):
        ctx.read_tap(13)                                  # a refused call allocates nothing
    ctx.close()


def test_tap13_matches_host(pkg, emul):
    """the first step of fresh streams (oscillator at rest) against the host build over the same span; every batch size and index"""
    recs = [recording(0xA200, 3, 0.0, noise_seed=5), recording(0xA201, 3, 10.0, noise_seed=6, tone=(301500.0, 20.0)),
            recording(0xA202, 3, None), np.asarray(np.random.default_rng(7).standard_normal(3 * TF) * 0.05, np.float32).astype(np.complex64)]
    starts = [1000, 77777, 150000, 0]
    rec = np.stack(recs)
    full = run(pkg, rec, 1, start=starts, taps=(13,), buf_len=NEED + 3000)[0]
    rev = run(pkg, rec[::-1], 1, start=starts[::-1], taps=(13,), buf_len=NEED + 3000)[0]
    for s in range(len(recs)):
        one = run(pkg, rec[s:s + 1], 1, start=starts[s:s + 1], taps=(13,), buf_len=NEED + 3000)[0]
        y = np.ascontiguousarray(rec[s, starts[s]:starts[s] + NEED + 3000])
        nb = min(len(y) // 256, 784)
        lv, l1 = np.zeros(nb, np.float32), np.zeros(nb, np.float32)
        emul.emul_acq_levels(_p(y), nb, _p(lv), _p(l1))
        dec, f = np.zeros(2, np.int32), np.zeros(2, np.float32)
        emul.emul_acq_decide(_p(lv), nb, _p(dec), _p(f))
        t = full[13][s]
        assert t["searched"] == 1 and t["blocks"] == nb
        assert np.float32(t["depth_db"]).tobytes() == f[0].tobytes(), (s, t["depth_db"], f[0])
        assert t["null_end"] == (starts[s] + dec[1] * 256 + 2480 if dec[0] else -1)
        assert one[13][0].tobytes() == t.tobytes() and rev[13][len(recs) - 1 - s].tobytes() == t.tobytes()
        assert abs(full["results"]["slevel"][s] - l1.astype(np.float64).sum() / (nb * 256)) <= 1e-5 * abs(full["results"]["slevel"][s]) + 1e-30
    zero = run(pkg, np.zeros((1, NEED + 3000), np.complex64), 1, taps=(13,), buf_len=NEED + 3000)[0][13][0]
    assert zero["searched"] == 1 and zero["depth_db"] == 0.0 and zero["null_end"] == -1        # digital silence is no null by itself
    assert full[13]["searched"][3] == 1 and full[13]["null_end"][3] == -1 and full["results"]["acq_failed"][3] == 1


def test_same_frames_at_20db(pkg):
    rec = np.stack([recording(0xA300 + i, 8, 20.0, noise_seed=10 + i) for i in range(3)])
    a = run(pkg, rec, 9, robust=False, keep_taps=True, taps=(0,))
    b = run(pkg, rec, 9, keep_taps=True, taps=(0, 13))
    common = 0
    for s in range(3):
        fa, fb = frames_by_pos(a, s), frames_by_pos(b, s)
        assert len(fb) >= 6, s
        for p in set(fa) & set(fb):
            assert np.array_equal(fa[p]["fibs"][s], fb[p]["fibs"][s]) and np.array_equal(fa[p][0][s], fb[p][0][s]), (s, p)
            common += 1
        assert all(b[k][13]["excised"][s] == 0 for k in range(9))       # nothing to excise without an interferer
    assert common >= 12


def acquired(outs, s):
    """frames stream s decoded (time sync held)"""
    return sum(1 for o in outs if o["results"]["status"][s] == 0)


def test_0db(pkg):
    rec = np.stack([recording(0xA400 + i, 7, 0.0, noise_seed=20 + i) for i in range(6)])
    a = run(pkg, rec, 7, robust=False)
    b = run(pkg, rec, 7)
    ra = sum(acquired(a, s) > 0 for s in range(6))
    rb = sum(acquired(b, s) > 0 for s in range(6))
    crc = sum(bin(int(o["results"]["fib_crc_mask"][s])).count("1") for o in b for s in range(6))
    print("0 dB: streams that decoded a frame, REFERENCE %d, ROBUST %d of 6; ROBUST FIB CRC passes %d" % (ra, rb, crc))
    assert rb >= 5 and rb > ra
    for s in range(6):
        first = next(k for k, o in enumerate(b) if o["results"]["status"][s] == 0)
        assert first <= 2, s                         # found in the first step, decoded once the buffer holds the frame


@pytest.mark.parametrize("db", [10.0, 20.0])
def test_off_grid_tone(pkg, db):
    rec = np.stack([recording(0xA500 + i, 10, 10.0, noise_seed=30 + i, tone=(301500.0, db)) for i in range(4)])
    a = run(pkg, rec, 10, robust=False)
    b = run(pkg, rec, 10, taps=(13,))
    for s in range(4):
        print("tone %.0f dB stream %d: REFERENCE %s ROBUST %s fine %s excised %s" % (db, s, [int(o["results"]["status"][s]) for o in a],
              [int(o["results"]["status"][s]) for o in b], [int(o["results"]["fine_corr"][s]) for o in b], [int(o[13]["excised"][s]) for o in b]))
    for s in range(4):
        dec = [k for k, o in enumerate(b) if o["results"]["status"][s] == 0]
        assert dec and dec[0] <= 2 and len(dec) >= (10 - dec[0]) // 2, (s, dec)
        assert all(b[k][13]["excised"][s] > 0 for k in dec)
        assert not any(o["results"]["status"][s] == 0 for o in a), s                  # the envelope dip never crosses with the tone
    crc_b = sum(bin(int(o["results"]["fib_crc_mask"][s])).count("1") for o in b for s in range(4))
    crc_a = sum(bin(int(o["results"]["fib_crc_mask"][s])).count("1") for o in a for s in range(4))
    print("tone %.0f dB: FIB CRC passes REFERENCE %d, ROBUST %d of %d" % (db, crc_a, crc_b, 4 * 12 * 10))
    assert crc_b >= crc_a


def test_noise_only(pkg):
    rng = np.random.default_rng(0xA600)
    rec = ((rng.standard_normal((3, 3 * TF)) + 1j * rng.standard_normal((3, 3 * TF))) * 0.05).astype(np.complex64)
    b = run(pkg, rec, 4, buf_len=NEED, taps=(13,))
    for o in b:
        assert set(o["results"]["status"].tolist()) <= {2, 3}
    assert all(o["results"]["acq_failed"].sum() >= 1 for o in b[:2])
    assert all(o[13]["null_end"][s] == -1 for o in b for s in range(3) if o["results"]["status"][s] == 3)


def test_buffer_ends_in_null(pkg):
    """the first span stops 1500 samples into the null: nothing is found, the search keeps its last blocks, the next step finds it"""
    rec = recording(0xA700, 4, 15.0, noise_seed=40)[None]
    L = 120000
    p0 = TF + 1500 - L
    b = run(pkg, rec, 4, buf_len=L, start=[p0], taps=(13,))
    t0 = b[0][13][0]
    assert t0["searched"] == 1 and t0["null_end"] == -1 and b[0]["results"]["acq_failed"][0] == 1
    assert b[0]["results"]["next_pos"][0] == p0 + (t0["blocks"] - 11) * 256
    t1 = b[1][13][0]
    assert t1["null_end"] != -1 and abs(int(t1["null_end"]) - (TF + TNULL)) <= 400


def test_reset_and_switch_mid_search(pkg):
    rng = np.random.default_rng(0xA800)
    noise = ((rng.standard_normal(2 * TF) + 1j * rng.standard_normal(2 * TF)) * 0.01).astype(np.complex64)
    sig = recording(0xA801, 6, 12.0, noise_seed=41)
    rec = np.concatenate([noise, sig])[None]

    def between(ctx, k, pos):
        if k == 1:
            ctx.reset(0, 1, 0)                                  # back to the start: the search starts over
            return np.zeros(1, np.int64)
        if k == 2:
            ctx.set_options(acquisition=load_pkg().ACQ_REFERENCE)     # a search in progress continues under the reference method
        if k == 4:
            ctx.set_options(acquisition=load_pkg().ACQ_ROBUST)
        return pos

    b = run(pkg, rec, 9, buf_len=NEED + 2000, between=between, taps=(13,))
    assert b[0][13]["searched"][0] == 1 and b[1][13]["searched"][0] == 1
    assert b[1]["results"]["next_pos"][0] == b[0]["results"]["next_pos"][0]     # the reset repeated the same search
    assert b[2][13]["searched"][0] == 0 and b[3][13]["searched"][0] == 0       # REFERENCE steps: tap 13 all zero
    assert any(o["results"]["status"][0] == 0 for o in b[4:])


@pytest.mark.parametrize("placement", [0, 1, 2])
def test_placements_and_submit(pkg, placement):
    rec = np.stack([recording(0xA900 + i, 6, 5.0, noise_seed=50 + i) for i in range(2)])
    opts = {"fft_placement": placement}
    a = run(pkg, rec, 6, opts=opts, buf_len=NEED + 5000)
    b = run(pkg, rec, 6, opts=opts, buf_len=NEED + 5000, submit=True)
    for x, y in zip(a, b):
        assert np.array_equal(x["results"].view(np.uint8), y["results"].view(np.uint8)) and np.array_equal(x["fibs"], y["fibs"])
    for s in range(2):
        assert acquired(a, s) >= 3, (placement, s)


def test_diversity_at_0db(pkg):
    """two antennas of one transmitter at 0 dB each, no 20 dB lead frame: both acquire on the same frame and the leader combines"""
    clean = dabtx.DabTx(seed=0xAA00).frames(7, noise_floor=0)
    p = float(np.mean(np.abs(clean) ** 2))
    chans = [[(0, 1.0), (20, 0.95j)], [(0, 1.0), (20, -0.95)]]
    rec = np.stack([dabtx.add_awgn(ofdmref.multipath(clean, ch), 0.0, seed=60 + i, signal_power=p) for i, ch in enumerate(chans)])
    S, N = rec.shape
    ctx = pkg.Context(n_streams=S)
    ctx.set_options(acquisition=pkg.ACQ_ROBUST)
    ctx.set_combining([0, 0])
    d = ctx.dev(rec)
    members = []
    for k in range(6):
        out = ctx.process(d, N, np.zeros(S, np.int64), N)
        r = out["results"]
        if r["status"][0] == 0 and r["status"][1] == 0:
            members.append(int(ctx.read_tap(12)["members"][0]))
            assert r["next_pos"][0] == r["next_pos"][1]
    d.free()
    ctx.close()
    assert members and all(m == 2 for m in members), members
