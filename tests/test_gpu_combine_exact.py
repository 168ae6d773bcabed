"""Diversity reception (dabb_set_combining) against exact restatements, in the path every decode takes.

A, every carrier of every symbol: keep_taps contexts on recordings without a carrier offset, so that the pipeline applies no oscillator
(asserted: fine_corr and coarse_corr stay 0).  Each decoded stream's phase reference symbol is taken from its frame record
(next_pos - (T_u + 75 T_s + T_null)) and its r1 recomputed by the stage-level demodulator (under TRACK with tap 11's applied_ppm); its
16 constellation carriers equal tap 2 bit for bit.  Tap 12's noise is combineref.noise_f32 of tap 3, its members and mask are
combineref.select of the step's statuses, positions and noises, and the leader's 75 x 3072 softbits are the reference demap of the
float32 sum in ascending stream order bit for bit (and the host build's), or within the rounding rule of combineref.compare for the
weighted demap.  Groups of 2, 3, 5 and 8 with the leader first, in the middle and last; members that must not contribute (noise only,
the leader's antenna 505 samples late, a whole frame late) and one that must (504 samples late); both demaps, TRACK off and on.

B, the masked path is what the decoders read: a context without keep_taps, whose members decode other sub-channels than their leaders
(other CU ranges, slot 1 only; a leader with two slots), against a keep_taps twin (tap 0 and every output bit for bit), the oracle
(the leaders' FIBs and their sub-channel chain over their tap-0 softbits) and an ungrouped context (every member's outputs and taps
10 and 11, with count_bit_errors and TRACK on).

C, tables changing between steps: select and remove calls on leaders and members (the combined r1 buffer grows and shrinks), a regroup,
a dissolve (then every stream's FIBs equal the ungrouped context's at once and its logical frames once the time interleaver has
flushed) and a regroup again, each followed by B's checks; a regroup between dabb_submit calls with two steps in flight takes effect
from the next submitted step.

D, tap 0 of the last step does not change when a control call (set_combining with the same table, another table or None, a select or
remove call, dabb_stream_reset) comes between the step and the read."""
import ctypes as C
import os
import subprocess
import time

import numpy as np
import pytest

import clockref
import combineref
import dabtx
import ofdmref
import softref
from conftest import ROOT, load_pkg
from test_gpu_msc_geometry import _frames_of, _prot

pytestmark = pytest.mark.gpu
TU, TS, TG, TNULL, TF, K = 2048, 2552, 504, 2656, 196608, 1536
PRS_BACK = TU + 75 * TS + TNULL               # next_pos - the start of the frame's phase reference symbol
W = TG + TU + 75 * TS + 64                    # the samples one stage-level frame reads, from TG before its phase reference symbol
STEPS, FRAMES = 12, 14
BR = 96
RATE = 0.005
MSC, SF = 3 * BR, 15 * BR


def sel(cu):
    return dict(start_cu=cu, length_cu=dabtx.eep_cu(BR), bitrate=BR, eep_profile_a=True, eep_level=3, dabplus=True)


# the streams: (transmitter, antenna, delay in samples) or None for noise only.  Groups of 2 (leader first), 3 (leader in the middle),
# 5 (leader last; noise only, the leader's antenna 505 and 504 samples late) and 8 (leader in the middle; a whole frame late, noise
# only), and two streams alone
STREAMS = [(0, 0, 0), (0, 1, 0),
           (1, 1, 0), (1, 0, 0), (1, 2, 0),
           (2, 1, 0), None, (2, 0, 505), (2, 0, 504), (2, 0, 0),
           (3, 1, 0), (3, 2, 0), (3, 3, 0), (3, 0, 0), (3, 0, TF), None, (3, 4, 0), (3, 1, 505),
           (4, 0, 0), (4, 1, 0)]
LEADER = [0, 0, 3, 3, 3, 9, 9, 9, 9, 9, 13, 13, 13, 13, 13, 13, 13, 13, 18, 19]
LEADER2 = [2, 2, 2, 2, 2, 5, 5, 7, 7, 7, 11, 11, 11, 11, 16, 16, 16, 16, 18, 18]        # another grouping: leaders become members
PPM = [45.0, -60.0, 30.0, 75.0, -20.0]        # each transmitter's sample-clock error, the same at all its antennas
CHANNELS = [None, [(0, 1.0), (20, 0.95j)], [(0, 1.0), (20, -0.95)], [(0, 1.0), (37, 0.7 - 0.3j), (211, 0.5j)], [(0, 0.8), (9, 0.6)]]
SNR, LEAD_SNR = 8.0, 20.0
# B: per stream {slot: selection}; members read other symbols than their leader (CU 400 and on, slot 1 only), leader 3 has two slots
SELECT_B = {s: {0: sel(0)} for s in range(len(STREAMS))}
SELECT_B.update({1: {0: sel(400)}, 2: {1: sel(600)}, 3: {0: sel(0), 1: sel(200)}, 9: {0: sel(400)}, 10: {0: sel(300)}, 16: {1: sel(700)}})


@pytest.fixture(scope="module", autouse=True)
def _timer():
    t0 = time.time()
    yield
    print(f"\n{__name__}: {time.time() - t0:.1f} s")


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
    return lib


@pytest.fixture(scope="module")
def sig():
    """[len(STREAMS), n] complex64: every antenna of a transmitter resampled by its PPM, through its own channel and noise (the first
    frame at LEAD_SNR, so that all antennas acquire on the same frame)"""
    t0 = time.time()
    ant = {}
    for t in range(len(PPM)):
        clean, _ = clockref.resample_clock(dabtx.DabTx(seed=0xE000 + t).frames(FRAMES), PPM[t])
        p = float(np.mean(np.abs(clean) ** 2))
        for a, ch in enumerate(CHANNELS):
            x = ofdmref.multipath(clean, ch) if ch else clean
            y = dabtx.add_awgn(x, SNR, seed=0xE100 + 16 * t + a, signal_power=p)
            y[:TF] = dabtx.add_awgn(x[:TF], LEAD_SNR, seed=0xE200 + 16 * t + a, signal_power=p)
            ant[(t, a)] = (y, p)
    n = min(len(y) for y, _ in ant.values())
    out = np.zeros((len(STREAMS), n), np.complex64)
    rng = np.random.default_rng(0xE300)
    for s, src in enumerate(STREAMS):
        if src is None:
            out[s] = dabtx.add_awgn(np.zeros(n, np.complex64), 0.0, seed=0xE400 + s, signal_power=ant[(0, 0)][1])
            continue
        t, a, delay = src
        y = ant[(t, a)][0]
        pre = ((rng.standard_normal(delay) + 1j * rng.standard_normal(delay)) * 1e-6).astype(np.complex64)
        out[s] = np.concatenate([pre, y])[:n]
    print(f"\nrecordings: {time.time() - t0:.1f} s")
    return out


def groups_of(leader):
    """{leader: [its members in ascending stream order]} of the groups of two or more"""
    g = {}
    for s, L in enumerate(leader):
        g.setdefault(int(L), []).append(s)
    return {L: m for L, m in g.items() if len(m) >= 2}


def popcount(m):
    return bin(int(m)).count("1")


def stage_r1(stage, sig, streams, prs, ppm):
    """(softbits, r1) of the frames of `streams` whose phase reference symbols start at prs[s], by the stage-level demodulator"""
    rows = np.zeros((len(streams), W), np.complex64)
    for i, s in enumerate(streams):
        a = int(prs[s]) - TG
        seg = sig[s, max(a, 0):a + W]
        rows[i, max(-a, 0):max(-a, 0) + len(seg)] = seg
    clk = None if ppm is None else np.ascontiguousarray(ppm[streams], np.float32)
    return stage.ofdm_demod(rows, np.full(len(streams), TG, np.int64), want_r1=True, clock_ppm=clk)


# ------------------------------------------------------------------------------------------------------------------- A
@pytest.mark.parametrize("weighted,track", [(False, False), (True, False), (False, True), (True, True)])
def test_every_carrier_exact(pkg, emul, sig, weighted, track):
    S, n = sig.shape
    ctx = pkg.Context(n_streams=S, keep_taps=True)
    ctx.set_options(soft_demap=pkg.DEMAP_WEIGHTED if weighted else pkg.DEMAP_REFERENCE, sample_clock=pkg.CLOCK_TRACK if track else pkg.CLOCK_OFF)
    ctx.select_subchannel(**sel(0))
    ctx.set_combining(LEADER)
    stage = pkg.Context(n_streams=1)
    d = ctx.dev(sig)
    grp = groups_of(LEADER)
    grouped = np.zeros(S, bool); grouped[[s for m in grp.values() for s in m]] = True
    combined = {len(m): 0 for m in grp.values()}
    edge = {504: [0, 0], 505: [0, 0]}                   # steps at that offset from the leader: [seen, contributed]
    n_excluded = applied = 0
    for k in range(STEPS):
        r = ctx.process(d, n, np.zeros(S, np.int64), n, msc_stride=MSC, sf_stride=SF)["results"]
        assert (r["fine_corr"] == 0).all() and (r["coarse_corr"] == 0).all(), (k, r["fine_corr"], r["coarse_corr"])
        soft, t2, t3, t12 = ctx.read_tap(0), ctx.read_tap(2), ctx.read_tap(3), ctx.read_tap(12)
        ppm = ctx.read_tap(11)["applied_ppm"] if track else None
        dec = r["status"] == pkg.FRAME_DECODED
        prs = r["next_pos"] - PRS_BACK
        streams = np.flatnonzero(dec)
        own, r1 = stage_r1(stage, sig, streams, prs, ppm)
        r1 = dict(zip(streams.tolist(), r1)); own = dict(zip(streams.tolist(), own))
        for s in streams:
            assert np.array_equal(r1[s][:, ::96], t2[s]), (k, s)          # the position and the stage-level call are the pipeline's
        for s in np.flatnonzero(grouped):
            want = combineref.noise_f32(t3[s]) if dec[s] else np.float32(0)
            assert t12["noise"][s] == want, (k, s, t12["noise"][s], want)
        for L, mb in grp.items():
            lpos = mb.index(L)
            nz = t12["noise"][mb]
            m = combineref.select(dec[mb], prs[mb], nz, lpos)
            assert int(t12["mask"][L]) == m and t12["members"][L] == popcount(m), (k, L, t12[mb], m)
            assert all(t12["members"][s] == 0 and t12["mask"][s] == 0 for s in mb if s != L), (k, L, t12[mb])
            for i, s in enumerate(mb):
                off = abs(int(prs[s]) - int(prs[L]))
                if dec[L] and dec[s] and off in edge:
                    edge[off][0] += 1; edge[off][1] += (m >> i) & 1
                n_excluded += int(dec[L] and not (m >> i) & 1)
            if not dec[L]:
                continue
            if popcount(m) < 2:                                            # the leader's own softbits
                if not weighted:
                    assert np.array_equal(soft[L], own[L]), (k, L)
                continue
            combined[len(mb)] += 1
            if track:
                applied += int(all(ppm[s] != 0 for i, s in enumerate(mb) if (m >> i) & 1))
            R1 = np.stack([r1[s] if (m >> i) & 1 else np.zeros((75, K), np.complex64) for i, s in enumerate(mb)])
            got = soft[L]
            if not weighted:
                want = softref.soft_reference_f32(combineref.combined_f32(R1, nz, m))
                bad = np.argwhere(got != want)
                assert bad.size == 0, (k, L, len(bad), bad[:4])
                h = np.zeros(3072, np.int8)
                nzc = np.ascontiguousarray(nz, np.float32)
                for l in range(75):
                    x = np.ascontiguousarray(R1[:, l])
                    emul.emul_combine_symbol(x.ctypes.data_as(C.c_void_p), len(mb), nzc.ctypes.data_as(C.c_void_p), m, 0, h.ctypes.data_as(C.c_void_p))
                    assert np.array_equal(got[l], h), (k, L, l)
            else:
                combineref.compare(got, combineref.combined(R1, nz, m), True, RATE)
        for s in range(S):                                                 # a stream outside a group keeps its own softbits
            if dec[s] and not grouped[s] and not weighted:
                assert np.array_equal(soft[s], own[s]), (k, s)
        for s in np.flatnonzero(grouped & dec):
            if s not in grp and not weighted:                              # so does every member other than the leader
                assert np.array_equal(soft[s], own[s]), (k, s)
    d.free(); ctx.close(); stage.close()
    print(f"\nweighted={weighted} track={track}: combined steps per group size {combined}, offsets {edge}, excluded {n_excluded}, "
          f"TRACK steps with a ppm applied {applied}")
    assert all(v >= STEPS - 3 for v in combined.values()), combined
    assert edge[504][0] >= STEPS - 3 and edge[504][1] == edge[504][0], edge
    assert edge[505][0] >= STEPS - 3 and edge[505][1] == 0, edge
    assert n_excluded >= 4 * (STEPS - 3)
    assert not track or applied >= 2, applied


# ------------------------------------------------------------------------------------------------------------------- B, C
def open_ctx(pkg, sig, leader, keep_taps, select=SELECT_B):
    S = sig.shape[0]
    c = pkg.Context(n_streams=S, keep_taps=keep_taps, n_subch_slots=2)
    c.set_options(count_bit_errors=True, sample_clock=pkg.CLOCK_TRACK)
    for s, slots in select.items():
        for slot, kw in slots.items():
            c.select_subchannel(first=s, count=1, slot=slot, **kw)
    if leader is not None:
        c.set_combining(leader)
    return c


def step(c, d, sig, taps):
    S, n = sig.shape
    o = c.process(d, n, np.zeros(S, np.int64), n, msc_stride=MSC, sf_stride=SF)
    for t in taps:
        o[t] = c.read_tap(t)
    return o


def same_stream(a, b, s, keys=("fibs", "msc", "sf", 10, 11)):
    return a["results"][s].tobytes() == b["results"][s].tobytes() and all(np.array_equal(a[k][s], b[k][s]) for k in keys)


def check_step(pkg, oracle, k, leader, m, t, u, never_led):
    """B's checks of one step: the masked context m against its keep_taps twin t, the leaders' FIBs against the oracle, the members
    that never led a group against the ungrouped context u"""
    S = len(m["results"])
    assert np.array_equal(m[0], t[0]), (k, np.argwhere(m[0] != t[0])[:4])
    for s in range(S):
        assert same_stream(m, t, s, ("fibs", "msc", "sf")), (k, s)
    if leader is None:
        return 0
    grp = groups_of(leader)
    n = 0
    for L in grp:
        r = m["results"][L]
        if r["status"] != pkg.FRAME_DECODED:
            continue
        fb, ok = oracle.fic_decode(m[0][L, :3].reshape(-1))
        assert np.array_equal(m["fibs"][L], np.packbits(fb, axis=1)), (k, L)
        assert int(r["fib_crc_mask"]) == sum(int(o) << i for i, o in enumerate(ok)), (k, L)
        n += int(m[12]["members"][L] >= 2)
    for s in range(S):
        if leader[s] != s and never_led[s]:
            assert same_stream(m, u, s), (k, s)
    return n


def leader_msc(pkg, oracle, outs, soft, L, slot, kw):
    """the leader's logical frames, RS events and superframes of one slot against the oracle's chain over its tap-0 softbits"""
    got, cifs, rs, sfs = _frames_of(pkg, outs, soft, L, slot, kw)
    prot = _prot(oracle, kw)
    de = oracle.deinterleave(np.stack(cifs))
    exp = [oracle.pack_bits(oracle.msc_deconvolve(prot, x[:prot.in_bits], True)) for x in de]
    assert len(got) == len(exp) >= 4 * (STEPS - 6), (L, slot, len(got), len(exp))
    for i, (x, y) in enumerate(zip(got, exp)):
        assert np.array_equal(x, y), (L, slot, i)
    ev, osfs = oracle.superframe_filter(np.stack(got))
    assert rs == [(e["uncorr"], e["corr"]) for e in ev], (L, slot, rs, ev)
    synced = [e for e in ev if e["sync"]]
    assert len(sfs) == len(synced) == len(osfs), (L, slot)
    for (x, na, mk), e, y in zip(sfs, synced, osfs):
        assert np.array_equal(x, y) and (na, mk) == (e["num_aus"], e["au_ok"]), (L, slot)
    return len(got), len(sfs)


def test_masked_path(pkg, oracle, sig):
    S, n = sig.shape
    ctx = {"m": open_ctx(pkg, sig, LEADER, False), "t": open_ctx(pkg, sig, LEADER, True), "u": open_ctx(pkg, sig, None, False)}
    taps = {"m": (0, 10, 11, 12), "t": (0,), "u": (10, 11)}
    dev = {name: c.dev(sig) for name, c in ctx.items()}
    outs, soft = [], []
    combined = 0
    for k in range(STEPS):
        o = {name: step(c, dev[name], sig, taps[name]) for name, c in ctx.items()}
        combined += check_step(pkg, oracle, k, LEADER, o["m"], o["t"], o["u"], np.ones(S, bool))
        outs.append(o["m"]); soft.append(o["m"][0][:, 3:75].copy())
    for name, c in ctx.items():
        dev[name].free(); c.close()
    assert combined >= len(groups_of(LEADER)) * (STEPS - 3), combined
    frames = superframes = 0
    for L in groups_of(LEADER):
        for slot, kw in SELECT_B[L].items():
            f, s = leader_msc(pkg, oracle, outs, soft, L, slot, kw)
            frames += f; superframes += s
    print(f"\nleaders: {frames} logical frames, {superframes} superframes against the oracle")
    assert superframes > 0


def test_tables_change_between_steps(pkg, oracle, sig):
    S, n = sig.shape
    grow = [(L, 1, sel(500)) for L in (0, 9, 13)]
    events = {      # step: [(method, kwargs)], the table from that step on
        1: [("select_subchannel", dict(first=L, count=1, slot=slot, **kw)) for L, slot, kw in grow],                   # leaders grow
        2: [("remove_subchannel", dict(first=L, count=1, slot=slot)) for L in (0, 3, 9, 13) for slot in (0, 1)]          # ... then shrink
           + [("select_subchannel", dict(first=5, count=1, slot=1, **sel(650)))],                                          # a member
        3: [("remove_subchannel", dict(first=1, count=1, slot=0)), ("select_subchannel", dict(first=3, count=1, slot=0, **sel(0)))],
        4: [("set_combining", LEADER2)],
        5: [("set_combining", None)],
        10: [("set_combining", LEADER)],
    }
    table = {0: LEADER, 4: LEADER2, 5: None, 10: LEADER}
    ctx = {"m": open_ctx(pkg, sig, LEADER, False), "t": open_ctx(pkg, sig, LEADER, True), "u": open_ctx(pkg, sig, None, False)}
    taps = {"m": (0, 10, 11, 12), "t": (0,), "u": (10, 11)}
    dev = {name: c.dev(sig) for name, c in ctx.items()}
    never_led = np.ones(S, bool)
    leader = LEADER
    for k in range(STEPS):
        for name, c in ctx.items():
            for meth, kw in events.get(k, []):
                if meth == "set_combining":
                    if name != "u":
                        c.set_combining(kw)
                else:
                    getattr(c, meth)(**kw)
        leader = table.get(k, leader)
        if leader is not None:
            for L in groups_of(leader):
                never_led[L] = False
        o = {name: step(c, dev[name], sig, taps[name]) for name, c in ctx.items()}
        check_step(pkg, oracle, k, leader, o["m"], o["t"], o["u"], never_led)
        if leader is None:
            for s in range(S):
                assert np.array_equal(o["m"]["fibs"][s], o["u"]["fibs"][s]), (k, s)
                assert o["m"]["results"]["fib_crc_mask"][s] == o["u"]["results"]["fib_crc_mask"][s], (k, s)
                if k >= 5 + 4:                                             # the 16-CIF time interleaver has flushed
                    assert np.array_equal(o["m"]["msc"][s], o["u"]["msc"][s]), (k, s)
    for name, c in ctx.items():
        dev[name].free(); c.close()


def test_regroup_between_submits(pkg, sig):
    """two steps in flight, then a regroup: the steps already submitted decode with the old table, the next with the new one"""
    x = np.ascontiguousarray(sig[:10, :7 * TF])
    S, n = x.shape
    leader, leader2 = LEADER[:10], LEADER2[:10]
    sel10 = {s: SELECT_B[s] for s in range(S)}
    want = []
    c = open_ctx(pkg, x, leader, False, sel10)
    d = c.dev(x)
    for k in range(6):
        if k == 4:
            c.set_combining(leader2)
        want.append(step(c, d, x, ()))
    want_tap0 = c.read_tap(0)
    d.free(); c.close()
    c = open_ctx(pkg, x, leader, False, sel10)
    got = []
    for k in range(6):
        c.submit(x, n, np.zeros(S, np.int64), n, msc_stride=MSC, sf_stride=SF)
        if k == 3:                                                         # steps 2 and 3 are in flight
            c.set_combining(leader2)
        if k >= 1:
            got.append(c.collect())
    got.append(c.collect())
    got_tap0 = c.read_tap(0)
    c.close()
    for k, (a, b) in enumerate(zip(want, got)):
        for s in range(S):
            assert same_stream(a, b, s, ("fibs", "msc", "sf")), (k, s)
    assert np.array_equal(want_tap0, got_tap0)


# ------------------------------------------------------------------------------------------------------------------- D
CALLS = {
    "same table": lambda c: c.set_combining(LEADER[:10]),
    "new table": lambda c: c.set_combining(LEADER2[:10]),
    "dissolve": lambda c: c.set_combining(None),
    "select": lambda c: c.select_subchannel(first=3, count=1, slot=1, **sel(500)),
    "remove": lambda c: c.remove_subchannel(first=3, count=1, slot=0),
    "reset": lambda c: c.reset(),
}


@pytest.mark.parametrize("call", list(CALLS))
def test_tap0_stable_across_control_calls(pkg, sig, call):
    x = np.ascontiguousarray(sig[:10, :6 * TF])
    S, n = x.shape
    sel10 = {s: SELECT_B[s] for s in range(S)}
    tap0 = []
    for late in (False, True):
        c = open_ctx(pkg, x, LEADER[:10], False, sel10)
        d = c.dev(x)
        for k in range(4):
            o = step(c, d, x, (12,) if k == 3 else ())
        assert (o[12]["members"][[0, 3, 9]] >= 2).all(), o[12]
        if late:
            CALLS[call](c)
        tap0.append(c.read_tap(0))
        d.free(); c.close()
    bad = np.argwhere((tap0[0] != tap0[1]).any(axis=-1))
    assert bad.size == 0, f"{call}: tap 0 differs in {len(bad)} (stream, symbol) rows, the first {bad[:4].tolist()}"
