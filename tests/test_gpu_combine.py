"""Diversity reception (dabb_set_combining) on the device.

No groups: a context that never groups and one whose table is all self-leaders decode byte-identically, with 14 launches per step.
Leader alone: a branch with noise only (NO_SYNC), or with the same recording one frame later (misaligned), never contributes: members = 1
and the leader decodes bit for bit like an ungrouped twin.  A leader grouped with an exact copy of itself decodes the same FIBs and logical
frames, with softbits within the rounding rule of tests/combineref.py.  Device against host: tap 12's noise is the host combine_core's
of tap 3's null symbols, and the leader's combined softbits of the constellation carriers are the host combination of tap 2's products.
The combined softbits do not depend on ofdm_groups, the tail split or dabb_submit, with TRACK and WEIGHTED on.  Malformed tables are
refused and change nothing.  Closed loop: two antennas per transmitter, each with its own multipath channel and noise (the first frame
at 20 dB, so that both antennas acquire on the same frame; antennas a frame apart never combine): the leader passes
at least as many FIB CRCs as the better antenna alone at every point, has no more RS-uncorrectable superframe codewords, and is strictly
better summed over the multipath points; batch_decode --diversity 2 writes the leader's .div file and passes more FIBs than either file."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import combineref
import dabtx
import ofdmref
from conftest import ROOT, load_pkg

pytestmark = pytest.mark.gpu
TF, TNULL, K = 196608, 2656, 1536
BITRATE = 96
RATE = 0.005


@pytest.fixture(scope="module")
def pkg():
    return load_pkg()


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_combine") / "libemul_combine.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-o", so,
                           os.path.join(ROOT, "tests", "host_emul", "emul_combine.cpp")])
    lib = C.CDLL(so)
    lib.emul_combine_symbol.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_uint32, C.c_int, C.c_void_p]
    lib.emul_combine_noise.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    return lib


def antennas(seed, frames, snr, chans, noise_seed, lead_snr=None):
    """one transmitter received through each channel of `chans` with its own noise: [len(chans), N] complex64.  lead_snr: the first
    frame at that SNR instead, so that every antenna acquires on the same frame (antennas that acquire on different frames stay a frame
    apart and never combine)"""
    clean = dabtx.DabTx(seed=seed).frames(frames)
    out = []
    for i, ch in enumerate(chans):
        x = ofdmref.multipath(clean, ch) if ch else clean
        p = float(np.mean(np.abs(x) ** 2))
        y = dabtx.add_awgn(x, snr, seed=noise_seed + i, signal_power=p)
        if lead_snr is not None:
            y[:TF] = dabtx.add_awgn(x[:TF], lead_snr, seed=noise_seed + 100 + i, signal_power=p)
        out.append(y)
    return np.stack(out).astype(np.complex64)


def decode(pkg, sig, steps, leader=None, taps=(), submit=False, opts=None, n_streams=None, **kw):
    """steps of a context over sig [S, N] (buf_start 0) with one DAB+ sub-channel; per step the outputs and the taps asked for.
    n_streams: sig is one recording [N] that every stream reads (stride 0)"""
    S = n_streams or sig.shape[0]
    stride = 0 if n_streams else sig.shape[1]
    ctx = pkg.Context(n_streams=S, **kw)
    ctx.select_subchannel(0, dabtx.eep_cu(BITRATE), BITRATE, eep_profile_a=True, eep_level=3, dabplus=True)
    if opts:
        ctx.set_options(**opts)
    if leader is not None:
        ctx.set_combining(leader)
    outs = []
    d = None if submit else ctx.dev(sig)
    for k in range(steps):
        n0 = ctx.kernel_launches()
        if submit:
            ctx.submit(sig, stride, np.zeros(S, np.int64), sig.shape[-1], msc_stride=3 * BITRATE, sf_stride=15 * BITRATE)
            if k == 0:
                continue
            out = ctx.collect()
        else:
            out = ctx.process(d, stride, np.zeros(S, np.int64), sig.shape[-1], msc_stride=3 * BITRATE, sf_stride=15 * BITRATE)
        out["launches"] = ctx.kernel_launches() - n0
        for t in taps:
            if not submit or k == steps - 1:
                out[t] = ctx.read_tap(t)
        outs.append(out)
    if submit:
        outs.append(ctx.collect())
        for t in taps:
            outs[-1][t] = ctx.read_tap(t)
    if d:
        d.free()
    ctx.close()
    return outs


def same(a, b, keys=("fibs", "msc", "sf")):
    return all(np.array_equal(a[k], b[k]) for k in keys) and np.array_equal(a["results"].view(np.uint8), b["results"].view(np.uint8))


CH_A = [(0, 1.0), (20, 0.95j)]
CH_B = [(0, 1.0), (20, -0.95)]


def test_no_groups(pkg):
    sig = np.concatenate([antennas(0xD100, 7, 6.0, [CH_A, CH_B], 0xD110), antennas(0xD101, 7, 6.0, [CH_A, CH_B], 0xD120)])
    S = len(sig)
    a = decode(pkg, sig, 6, taps=(0,))
    b = decode(pkg, sig, 6, leader=np.arange(S), taps=(0,))
    for k, (x, y) in enumerate(zip(a, b)):
        assert same(x, y) and np.array_equal(x[0], y[0]), k
        assert x["launches"] == y["launches"] == 14, (k, x["launches"], y["launches"])
    ctx = pkg.Context(n_streams=S)
    ctx.set_combining(np.arange(S))
    with pytest.raises(pkg.DabbError):
        ctx.read_tap(12)                              # no group has formed
    ctx.close()


@pytest.mark.parametrize("branch", ["noise", "late"])
def test_leader_alone(pkg, branch):
    x = antennas(0xD200, 8, 7.0, [CH_A], 0xD210)[0]
    if branch == "noise":
        y = dabtx.add_awgn(np.zeros_like(x), 0.0, seed=0xD220, signal_power=float(np.mean(np.abs(x) ** 2)))
    else:
        y = np.concatenate([x[TF // 2:], np.zeros(TF // 2, np.complex64)])     # the same recording, half a frame off on the shared axis
    sig = np.stack([x, y]).astype(np.complex64)
    a = decode(pkg, sig, 7, taps=(0,))
    b = decode(pkg, sig, 7, leader=[0, 0], taps=(0, 12))
    dec = 0
    for k, (u, g) in enumerate(zip(a, b)):
        assert same(u, g) and np.array_equal(u[0], g[0]), k
        r = g["results"]
        if r["status"][0] == pkg.FRAME_DECODED:
            dec += 1
            assert g[12]["members"][0] == 1 and g[12]["mask"][0] == 1, (k, g[12])
        assert g[12]["members"][1] == 0
        assert g["launches"] == 16
    assert dec >= 5


def test_copy_of_itself(pkg):
    x = antennas(0xD300, 8, 6.0, [CH_A], 0xD310)[0]
    sig = np.stack([x, x])
    b = decode(pkg, sig, 7, leader=[0, 0], taps=(0, 12))
    dec = 0
    for k, g in enumerate(b):
        r = g["results"]
        assert np.array_equal(g["fibs"][0], g["fibs"][1]) and np.array_equal(g["msc"][0], g["msc"][1]), k
        assert np.array_equal(r["fib_crc_mask"][0], r["fib_crc_mask"][1]) and np.array_equal(r["n_logical"][0], r["n_logical"][1]), k
        if r["status"][0] == pkg.FRAME_DECODED:
            dec += 1
            assert g[12]["members"][0] == 2 and g[12]["mask"][0] == 3 and g[12]["noise"][0] == g[12]["noise"][1] > 0, g[12]
            d = np.abs(g[0][0].astype(int) - g[0][1].astype(int))          # R = 2 r1 / N: the same softbits up to rounding
            assert d.max() <= 1 and (d != 0).mean() <= RATE, (d.max(), (d != 0).mean())
    assert dec >= 5


def test_device_against_host(pkg, emul):
    sig = np.concatenate([antennas(0xD400 + t, 6, 5.0, [CH_A, CH_B, [(0, 1.0), (37, 0.7 - 0.3j)]], 0xD410 + 8 * t) for t in range(2)])
    leader = [0, 0, 0, 3, 3, 3]
    outs = decode(pkg, sig, 5, leader=leader, taps=(0, 2, 3, 12), keep_taps=True)
    checked = 0
    for g in outs:
        res, tap12 = g["results"], g[12]
        y = np.ascontiguousarray(g[3], np.complex64)
        nz = np.zeros(len(sig), np.float32)
        emul.emul_combine_noise(y.ctypes.data_as(C.c_void_p), len(sig), nz.ctypes.data_as(C.c_void_p))
        for s in range(len(sig)):
            if res["status"][s] == pkg.FRAME_DECODED:
                assert tap12["noise"][s] == nz[s], (s, tap12["noise"][s], nz[s])
        for L in (0, 3):
            mask = int(tap12["mask"][L])
            if res["status"][L] != pkg.FRAME_DECODED or bin(mask).count("1") < 2:
                continue
            # the constellation carriers (every 96th) of every symbol: the reference demap is per carrier
            r1 = np.zeros((3, K), np.complex64)
            soft = np.zeros(2 * K, np.int8)
            for l in range(75):
                for i in range(3):
                    r1[i, ::96] = g[2][L + i, l]
                emul.emul_combine_symbol(r1.ctypes.data_as(C.c_void_p), 3, nz[L:L + 3].ctypes.data_as(C.c_void_p), mask, 0, soft.ctypes.data_as(C.c_void_p))
                got = g[0][L].reshape(75, 3072)[l]
                assert np.array_equal(got[0:K:96], soft[0:K:96]) and np.array_equal(got[K::96], soft[K::96]), (L, l)
            checked += 1
    assert checked >= 4


S_CFG = 2048


@pytest.mark.parametrize("weighted", [False, True])
def test_launch_forms(pkg, weighted):
    """the leaders' combined softbits (tap 0, every symbol) are the same in every launch form, with TRACK on: two antennas in 1 / 5 / 25
    CTAs per frame and under dabb_submit / dabb_collect with two steps in flight; 2048 streams reading one recording (groups of two
    copies) with the tail split on and off"""
    opts = {"soft_demap": pkg.DEMAP_WEIGHTED if weighted else pkg.DEMAP_REFERENCE, "sample_clock": pkg.CLOCK_TRACK}
    sig = np.concatenate([antennas(0xD500, 8, 6.0, [CH_A, CH_B], 0xD510, 20.0), antennas(0xD501, 8, 6.0, [CH_A, CH_B], 0xD520, 20.0)])
    want = None
    for kw in ({"ofdm_groups": 1, "ofdm_tail_split": -1}, {"ofdm_groups": 5}, {"ofdm_groups": 25}, {"submit": True}):
        outs = decode(pkg, sig, 5, leader=[0, 0, 2, 2], taps=(0, 12), opts=opts, **kw)
        last = outs[-1]
        assert (last["results"]["status"] == pkg.FRAME_DECODED).all() and (last[12]["members"][::2] == 2).all(), kw
        if want is None:
            want = last[0].copy()
        assert np.array_equal(last[0], want), kw
    assert not np.array_equal(want[0], want[1])
    one = antennas(0xD502, 8, 6.0, [CH_A], 0xD530)[0]
    want = None
    for kw in ({"ofdm_groups": 1, "ofdm_tail_split": -1}, {"ofdm_groups": 1}):
        last = decode(pkg, one, 5, leader=np.arange(S_CFG) & ~1, taps=(0, 12), opts=opts, n_streams=S_CFG, **kw)[-1]
        assert (last["results"]["status"] == pkg.FRAME_DECODED).all() and (last[12]["members"][::2] == 2).all(), kw
        soft = last[0]
        assert (soft[::2] == soft[:1]).all() and (soft[1::2] == soft[1:2]).all(), kw
        if want is None:
            want = soft[:2].copy()
        assert np.array_equal(soft[:2], want), kw


def test_refusals(pkg):
    sig = np.concatenate([antennas(0xD600, 7, 6.0, [CH_A, CH_B], 0xD610), antennas(0xD601, 7, 6.0, [CH_A, CH_B], 0xD620)])
    S = len(sig)
    bad = [([0, 0, 2, 4], S), ([0, 0, 2, -1], S), ([1, 2, 2, 3], S), ([0, 0, 2, 2], S - 1), ([0, 0, 2, 2, 2], S + 1)]
    for grouped in (None, [0, 0, 2, 2]):
        ref = decode(pkg, sig, 5, leader=grouped)
        ctx = pkg.Context(n_streams=S)
        ctx.select_subchannel(0, dabtx.eep_cu(BITRATE), BITRATE, eep_profile_a=True, eep_level=3, dabplus=True)
        if grouped:
            ctx.set_combining(grouped)
        d = ctx.dev(sig)
        for k in range(5):
            for tab, n in bad:
                t = np.asarray(tab, np.int32)
                rc = ctx.lib.dabb_set_combining(ctx.h, t.ctypes.data_as(C.c_void_p), n)
                assert rc == -3, (tab, n, rc)
            out = ctx.process(d, sig.shape[1], np.zeros(S, np.int64), sig.shape[1], msc_stride=3 * BITRATE, sf_stride=15 * BITRATE)
            assert same(out, ref[k]), (grouped, k)
        if not grouped:
            with pytest.raises(pkg.DabbError):
                ctx.read_tap(12)
        d.free(); ctx.close()
    # an oversized group: nine members
    ctx = pkg.Context(n_streams=10)
    with pytest.raises(pkg.DabbError):
        ctx.set_combining([0] * 9 + [9])
    ctx.set_combining([0] * 8 + [8, 8])
    ctx.close()


# ---- closed loop: two antennas per transmitter, each with its own channel (different echo phases) and noise
POINTS = [("awgn", 3.0), ("awgn", 5.0), ("2path", 3.0), ("2path", 5.0), ("3path", 3.0), ("3path", 5.0)]
CHANNELS = {"awgn": (None, None), "2path": ([(0, 1.0), (20, 0.95j)], [(0, 1.0), (20, -0.95)]),
            "3path": ([(0, 1.0), (37, 0.7 - 0.3j), (211, 0.5j)], [(0, 1.0), (37, -0.3 + 0.7j), (211, -0.5)])}
N_TX, FRAMES, STEPS_CL = 12, 8, 8
_SIGNALS = {}


def closed_loop_signal(i, name, snr):
    if i not in _SIGNALS:
        ca, cb = CHANNELS[name]
        _SIGNALS[i] = np.concatenate([antennas(0xD700 + t, FRAMES, snr, [ca, cb], 0xD800 + 64 * i + 2 * t, 20.0) for t in range(N_TX)])
    return _SIGNALS[i]


def tally(outs, streams):
    fib = rs_bad = 0
    for out in outs:
        r = out["results"]
        for s in streams:
            if r["status"][s] != 0:
                continue
            fib += bin(int(r["fib_crc_mask"][s])).count("1")
            n = int(r["n_rs_events"][s][0])
            rs_bad += bin(int(r["rs_uncorr_mask"][s][0]) & ((1 << n) - 1)).count("1")
    return fib, rs_bad


@pytest.mark.parametrize("weighted", [False, True])
def test_closed_loop_gain(pkg, weighted):
    opts = {"soft_demap": pkg.DEMAP_WEIGHTED} if weighted else None
    gain = 0
    table = {}
    for i, (name, snr) in enumerate(POINTS):
        sig = closed_loop_signal(i, name, snr)
        alone = decode(pkg, sig, STEPS_CL, opts=opts)
        comb = decode(pkg, sig, STEPS_CL, leader=np.arange(2 * N_TX) & ~1, opts=opts)
        a, b, c = tally(alone, range(0, 2 * N_TX, 2)), tally(alone, range(1, 2 * N_TX, 2)), tally(comb, range(0, 2 * N_TX, 2))
        assert tally(comb, range(1, 2 * N_TX, 2)) == b             # the members decode as they would alone
        best = max(a, b, key=lambda v: (v[0], -v[1]))
        table[(name, snr)] = (a, b, c)
    print("weighted" if weighted else "reference", {f"{n}@{s}dB": v for (n, s), v in table.items()})
    for (name, snr), (a, b, c) in table.items():
        best = max(a, b, key=lambda v: (v[0], -v[1]))
        assert c[0] >= best[0] and c[1] <= best[1], (name, snr, a, b, c)
        if name != "awgn":
            gain += (c[0] - best[0]) + (best[1] - c[1])
    assert gain > 0


def test_batch_decode_diversity(tmp_path):
    exe = os.path.join(ROOT, "welle.io_b200", "batch_decode")
    sig = antennas(0xD900, 12, 6.0, list(CHANNELS["2path"]), 0xD910)
    files = []
    for i, x in enumerate(sig):
        f = tmp_path / f"ant{i}.iq"
        x.tofile(f)
        files.append(str(f))
    passed = {}
    for mode, args in (("alone", []), ("div", ["--diversity", "2"])):
        out = tmp_path / mode
        out.mkdir()
        r = subprocess.run([exe] + args + ["--out", str(out)] + files, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr
        for i in range(2):
            rec = np.frombuffer((out / f"ant{i}.iq.fic").read_bytes(), np.uint8).reshape(-1, 33)
            passed[(mode, i)] = int((rec[:, 0] != 0).sum())
        if mode == "div":
            lines = [l.split() for l in (out / "ant0.iq.div").read_text().splitlines()]
            assert len(lines) >= 8 and all(len(l) == 3 for l in lines)
            assert sum(int(l[0]) == 2 and int(l[1]) == 3 and float(l[2]) > 0 for l in lines) >= len(lines) - 2, lines
            assert not (out / "ant1.iq.div").exists()
    print(passed)
    assert passed[("div", 1)] == passed[("alone", 1)]
    assert passed[("div", 0)] > max(passed[("alone", 0)], passed[("alone", 1)]), passed
