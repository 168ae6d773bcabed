"""Streams of one sub-channel slot with different bitrates and protection profiles, decoded by one grouped Viterbi launch.

The yardstick is a twin context: the same inputs with only some streams selected (or without a select call).  Every stream compared
must give the same result record, the same logical frames at its own length and the same superframes, byte for byte.  One stream
per transmitted profile is also checked against the transmitter's logical frames.  A UEP sub-channel and EEP 1-A at 384 kbit/s,
both on capacity units the transmitter fills with random data, are checked against the oracle's time de-interleaver, Viterbi and
dispersal applied to the GPU's own softbits."""
import numpy as np
import pytest

import dabtx
from conftest import load_pkg

pytestmark = pytest.mark.gpu
E_ARG, E_UNSUPPORTED = -3, -6
MSC, SF = 3 * 384, 15 * 384
FRAMES = 9

# bitrate, EEP-A?, level, DAB+?; a profile without "tx" is decoded from a 96 kbit/s EEP 3-A signal (its capacity units are random fill)
PROFILES = [dict(br=96, a=True, lv=3, dp=1), dict(br=48, a=True, lv=1, dp=1), dict(br=64, a=True, lv=2, dp=1), dict(br=128, a=True, lv=4, dp=1),
            dict(br=64, a=False, lv=3, dp=1), dict(br=96, a=False, lv=1, dp=1), dict(br=32, a=True, lv=2, dp=1), dict(br=192, a=False, lv=4, dp=1),
            dict(br=128, a=True, lv=3, dp=0),                                  # DAB (MP2): logical frames only
            dict(br=384, a=True, lv=1, dp=1, tx=False),                        # 36 864 softbits per codeword
            dict(br=64, uep=3, start=600, cu=48, dp=0, tx=False)]              # UEP-3 on random-filled capacity units


def _sel(p):
    if "uep" in p:
        return dict(start_cu=p["start"], length_cu=p["cu"], bitrate=p["br"], short_form=True, uep_level=p["uep"], dabplus=bool(p["dp"]))
    return dict(start_cu=0, length_cu=dabtx.eep_cu(p["br"], p["a"], p["lv"]), bitrate=p["br"], eep_profile_a=p["a"], eep_level=p["lv"], dabplus=bool(p["dp"]))


def _flen(p):
    return 3 * p["br"]


def _same_stream(x, y, s, flen, slot=0, what=""):
    assert x["results"][s].tobytes() == y["results"][s].tobytes(), (what, s)
    assert np.array_equal(x["msc"][s, slot, :, :flen], y["msc"][s, slot, :, :flen]), (what, s)
    if "sf" in x:
        assert np.array_equal(x["sf"][s, slot, :5 * flen], y["sf"][s, slot, :5 * flen]), (what, s)


def _run(pkg, S, iq, stride, buf_start, n, selections, steps, max_cu=576, msc=MSC, sf=SF, events=None, taps=None):
    """selections: [(first, count, select kwargs)]; events: {step: fn(ctx)} called before that step; taps: {stream: []} gets the
    stream's softbits of every step"""
    ctx = pkg.Context(n_streams=S, max_subch_cu=max_cu)
    for first, count, kw in selections:
        ctx.select_subchannel(first=first, count=count, **kw)
    outs = []
    for k in range(steps):
        if events and k in events:
            events[k](ctx)
        outs.append(ctx.process(iq, stride, buf_start, n, msc_stride=msc, sf_stride=sf))
        if taps:
            soft = ctx.read_tap(0)
            for s in taps:
                taps[s].append(soft[s].copy())
    ctx.close()
    return outs


def _oracle_check(oracle, pkg, outs, soft, s, p):
    """the stream's logical frames = the oracle's chain applied to the softbits the GPU produced for it"""
    sc = _sel(p)
    prot = oracle.prot_uep(p["br"], p["uep"]) if "uep" in p else oracle.prot_eep(p["br"], int(p["a"]), p["lv"])
    cifs, got = [], []
    for o, sb in zip(outs, soft):
        r = o["results"][s]
        if r["status"] != pkg.FRAME_DECODED:
            continue
        for c in range(4):
            cifs.append(sb[3 + 18 * c: 21 + 18 * c].reshape(-1)[sc["start_cu"] * 64:(sc["start_cu"] + sc["length_cu"]) * 64].copy())
        for c in range(4 - int(r["n_logical"][0]), 4):
            got.append(o["msc"][s, 0, c, :_flen(p)].copy())
    de = oracle.deinterleave(np.stack(cifs))
    exp = [oracle.pack_bits(oracle.msc_deconvolve(prot, x[:prot.in_bits], True)) for x in de]
    assert len(got) == len(exp) >= 4, (s, len(got), len(exp))
    for a, b in zip(got, exp):
        assert np.array_equal(a, b), s


def _tx_check(outs, tx, s, p):
    """the stream's logical frames are a contiguous run of what its transmitter sent"""
    flen = _flen(p)
    got = [o["msc"][s, 0, c, :flen] for o in outs for c in range(4 - int(o["results"][s]["n_logical"][0]), 4)]
    assert len(got) >= 4, (s, len(got))
    lf = np.concatenate(tx.logical); g = np.concatenate(got)
    hits = [k for k in range(len(tx.logical)) if np.array_equal(g[:flen], lf[k * flen:(k + 1) * flen])]
    assert hits and np.array_equal(g, lf[hits[0] * flen: hits[0] * flen + len(g)]), s


def test_twin_equivalence_256_streams(oracle):
    """256 streams with distinct seeds; slot 0 cycles through 11 protection profiles (EEP-A levels 1-4, EEP-B, DAB+, MP2, EEP 1-A
    384 kbit/s, UEP).  For each profile a twin context decodes only that profile's streams: they must match the mixed context."""
    pkg = load_pkg()
    S, P = 256, len(PROFILES)
    txs = [dabtx.DabTx(seed=0x700 + k, bitrate=p["br"], profile_a=p["a"], level=p["lv"]) if p.get("tx", True) else dabtx.DabTx(seed=0x700 + k)
           for k, p in enumerate(PROFILES)]
    base = [tx.frames(FRAMES) for tx in txs]
    n = len(base[0])
    rng = np.random.default_rng(0x256)
    host = np.empty((S, n), np.complex64)
    for s in range(S):
        host[s] = base[s % P]
        if s >= P:           # the first stream of every profile is clean: it is checked against its transmitter
            noise = rng.standard_normal(2 * n, dtype=np.float32).view(np.complex64) * np.float32(0.1 * 10 ** (-22 / 20) / np.sqrt(2))
            host[s] += noise
    keeper = pkg.Context(n_streams=1)
    d = keeper.dev(host)
    bs = np.zeros(S, np.int64)
    sel = [(s, 1, _sel(PROFILES[s % P])) for s in range(S)]
    checked = {9: [], 10: []}                   # softbits of the first 384 kbit/s stream and the first UEP stream
    mixed = _run(pkg, S, d, n, bs, n, sel, FRAMES, taps=checked)
    assert sum(int(o["results"]["sf_ready"][:, 0].sum()) for o in mixed) > 0
    for k, p in enumerate(PROFILES):
        mine = [s for s in range(S) if s % P == k]
        twin = _run(pkg, S, d, n, bs, n, [(s, 1, _sel(p)) for s in mine], FRAMES)
        for x, y in zip(mixed, twin):
            for s in mine:
                _same_stream(x, y, s, _flen(p), what=f"profile {k}")
        if p.get("tx", True):
            _tx_check(mixed, txs[k], k, p)
    _oracle_check(oracle, pkg, mixed, checked[9], 9, PROFILES[9])
    _oracle_check(oracle, pkg, mixed, checked[10], 10, PROFILES[10])
    keeper.close()


def _shared_signal(seed=0x5A):
    """one 96 kbit/s EEP 3-A signal that every stream reads (stride 0), each from its own start: the streams differ in time offset"""
    return dabtx.DabTx(seed=seed).frames(FRAMES)


def _offsets(S):
    return -((np.arange(S, dtype=np.int64) * 7919) % 20000)


@pytest.mark.parametrize("group", [1, 31, 32, 33, 127, 128, 129])
def test_group_boundaries(group):
    """a profile with `group` streams beside two others, unselected streams interleaved: the CTA holding the group's last codewords is
    partial (or exactly full), and every stream must equal its twin"""
    pkg = load_pkg()
    sig = _shared_signal()
    n = len(sig)
    S = group + 100 + 60 + 40
    rng = np.random.default_rng(group)
    member = np.full(S, -1)
    perm = rng.permutation(S)
    member[perm[:group]] = 0; member[perm[group:group + 100]] = 1; member[perm[group + 100:group + 160]] = 2
    profs = [PROFILES[1], PROFILES[7], PROFILES[0]]
    keeper = pkg.Context(n_streams=1)
    d = keeper.dev(sig)
    bs = _offsets(S)
    mixed = _run(pkg, S, d, 0, bs, n, [(s, 1, _sel(profs[member[s]])) for s in range(S) if member[s] >= 0], FRAMES, max_cu=144)
    assert sum(int(o["results"]["n_logical"][:, 0].sum()) for o in mixed) > 0
    for k, p in enumerate(profs):
        mine = [s for s in range(S) if member[s] == k]
        twin = _run(pkg, S, d, 0, bs, n, [(s, 1, _sel(p)) for s in mine], FRAMES, max_cu=144)
        for x, y in zip(mixed, twin):
            for s in mine:
                _same_stream(x, y, s, _flen(p), what=f"group {group} profile {k}")
    for x in mixed:           # streams not selected decode no sub-channel
        assert (x["results"]["n_logical"][member < 0, 0] == 0).all()
    keeper.close()


def test_selection_mid_run():
    """at step 4 some streams move to another profile (one to EEP 1-A 384 kbit/s, which widens the slot's rows) and others are removed:
    every stream the call does not name must equal a twin in which the call did not happen"""
    pkg = load_pkg()
    sig = _shared_signal(0x5B)
    n = len(sig)
    S = 64
    profs = [PROFILES[0], PROFILES[2], PROFILES[1]]
    sel = [(s, 1, _sel(profs[s % 3])) for s in range(S)]

    def call(ctx):
        ctx.select_subchannel(first=0, count=8, **_sel(PROFILES[9]))
        ctx.remove_subchannel(first=8, count=4)
        ctx.select_subchannel(first=12, count=4, **_sel(PROFILES[2]))
    keeper = pkg.Context(n_streams=1)
    d = keeper.dev(sig)
    bs = _offsets(S)
    a = _run(pkg, S, d, 0, bs, n, sel, FRAMES, events={4: call})
    b = _run(pkg, S, d, 0, bs, n, sel, FRAMES)
    for k, (x, y) in enumerate(zip(a, b)):
        for s in range(16, S):
            _same_stream(x, y, s, _flen(profs[s % 3]), what=f"step {k}")
    assert sum(int(o["results"]["n_logical"][16:, 0].sum()) for o in a[4:]) > 0
    assert (a[4]["results"]["n_logical"][:16, 0] == 0).all()       # the named streams restart their de-interleaver
    keeper.close()


def test_pipelined_select_between_submit_and_collect():
    """two dabb_submit steps outstanding, then a select call that widens the slot's rows, then the collects: the collected outputs
    equal a dabb_process twin, each in the geometry its step was submitted with"""
    pkg = load_pkg()
    sig = _shared_signal(0x5C)
    S = 12
    host = np.stack([np.roll(sig, -1500 * s) for s in range(S)]).astype(np.complex64)
    n = host.shape[1]
    bs = np.zeros(S, np.int64)
    profs = [PROFILES[0], PROFILES[4], PROFILES[6]]

    def make():
        c = pkg.Context(n_streams=S, max_subch_cu=576)
        for s in range(S):
            c.select_subchannel(first=s, count=1, **_sel(profs[s % 3]))
        return c

    def change(c):
        c.select_subchannel(first=0, count=3, **_sel(PROFILES[9]))
        c.remove_subchannel(first=3, count=1)
    a, b = make(), make()
    ptr = host.ctypes.data
    outs_a, outs_b = [], []
    for k in range(0, FRAMES, 2):
        a.submit(ptr, n, bs, n, msc_stride=MSC, sf_stride=SF)
        a.submit(ptr, n, bs, n, msc_stride=MSC, sf_stride=SF)
        if k == 4:
            change(a)
        outs_a += [a.collect(), a.collect()]
        outs_b += [b.process(ptr, n, bs, n, iq_is_host=True, msc_stride=MSC, sf_stride=SF) for _ in range(2)]
        if k == 4:
            change(b)
    for k, (x, y) in enumerate(zip(outs_a, outs_b)):
        assert x["results"].tobytes() == y["results"].tobytes(), k
        assert np.array_equal(x["msc"], y["msc"]) and np.array_equal(x["sf"], y["sf"]), k
    assert sum(int(o["results"]["n_logical"][:, 0].sum()) for o in outs_a) > 0
    a.close(); b.close()


def test_mixed_slot_launches_like_a_uniform_one():
    pkg = load_pkg()
    sig = _shared_signal(0x5D)
    n = len(sig)
    S = 48
    keeper = pkg.Context(n_streams=1)
    d = keeper.dev(sig)
    bs = _offsets(S)
    report = []
    for mixed in (False, True):
        c = pkg.Context(n_streams=S, max_subch_cu=144)
        for s in range(S):
            c.select_subchannel(first=s, count=1, **_sel(PROFILES[s % 4] if mixed else PROFILES[0]))
        for _ in range(2):
            c.process(d, 0, bs, n, msc_stride=MSC)
        c.profile(True)
        before = c.kernel_launches()
        c.process(d, 0, bs, n, msc_stride=MSC)
        launches = c.kernel_launches() - before
        names = sorted(c.profile_read())
        c.profile(False)
        c.close()
        report.append((launches, names))
    assert report[0] == report[1], report
    assert report[0][0] == 14 and "viterbi_kernel(MSC)" in report[0][1]
    keeper.close()


def test_refusals():
    """an msc_stride between the shortest and the longest logical frame of a mixed slot is refused before anything runs; a protection
    profile beyond DABB_MAX_PROFILES is refused and every stream decodes on as if the call had not happened"""
    pkg = load_pkg()
    sig = _shared_signal(0x5E)
    n = len(sig)
    S = 4
    keeper = pkg.Context(n_streams=1)
    d = keeper.dev(sig)
    bs = _offsets(S)

    def make():
        c = pkg.Context(n_streams=S, max_subch_cu=864)
        for s in range(S):
            c.select_subchannel(first=s, count=1, **_sel([PROFILES[1], PROFILES[0]][s % 2]))      # 144 and 288 bytes per frame
        return c
    a, b = make(), make()
    a.process(d, 0, bs, n, msc_stride=288); b.process(d, 0, bs, n, msc_stride=288)
    launches = a.kernel_launches()
    with pytest.raises(Exception) as e:
        a.process(d, 0, bs, n, msc_stride=200)
    assert f"error {E_ARG}:" in str(e.value)
    assert a.kernel_launches() == launches
    # fill the profile table from a stream of its own (stream 3 changes profile 62 times; the table then holds 64 entries)
    seen = {(48, True, 1), (96, True, 3)}
    for br in range(8, 136, 8):
        for lv in (1, 2, 3, 4):
            if (br, True, lv) in seen:
                continue
            seen.add((br, True, lv))
            for c in (a, b):
                c.select_subchannel(first=3, count=1, start_cu=0, length_cu=dabtx.eep_cu(br, True, lv), bitrate=br, eep_profile_a=True, eep_level=lv, dabplus=False)
    assert len(seen) == 64
    launches = a.kernel_launches()
    with pytest.raises(Exception) as e:
        a.select_subchannel(first=3, count=1, start_cu=0, length_cu=dabtx.eep_cu(32, False, 1), bitrate=32, eep_profile_a=False, eep_level=1, dabplus=False)
    assert f"error {E_UNSUPPORTED}:" in str(e.value) and "protection profiles" in str(e.value)
    assert a.kernel_launches() == launches
    a.select_subchannel(first=3, count=1, start_cu=0, length_cu=72, bitrate=96, eep_profile_a=True, eep_level=3)     # a known profile is still taken
    b.select_subchannel(first=3, count=1, start_cu=0, length_cu=72, bitrate=96, eep_profile_a=True, eep_level=3)
    logical = 0
    for k in range(1, FRAMES):
        x, y = a.process(d, 0, bs, n, msc_stride=288, sf_stride=1440), b.process(d, 0, bs, n, msc_stride=288, sf_stride=1440)
        assert x["results"].tobytes() == y["results"].tobytes(), k
        assert np.array_equal(x["msc"], y["msc"]) and np.array_equal(x["sf"], y["sf"]), k
        logical += int(x["results"]["n_logical"][:3, 0].sum())
    assert logical > 0
    a.close(); b.close(); keeper.close()


def test_scale_4096_streams_8_profiles():
    """4096 streams over 8 profiles in one slot; for three of the profiles a twin decodes only their streams, and 64 sampled streams of
    each must match"""
    pkg = load_pkg()
    sig = _shared_signal(0x5F)
    n = len(sig)
    S = 4096
    profs = PROFILES[:8]
    keeper = pkg.Context(n_streams=1)
    d = keeper.dev(sig)
    bs = _offsets(S)
    member = np.arange(S) % 8
    sel = [(s, 1, _sel(profs[member[s]])) for s in range(S)]
    steps = FRAMES - 1
    mixed = _run(pkg, S, d, 0, bs, n, sel, steps, max_cu=144, msc=576, sf=2880)
    assert sum(int(o["results"]["n_logical"][:, 0].sum()) for o in mixed) > S
    rng = np.random.default_rng(4096)
    for k in (1, 6, 7):              # 48 kbit/s EEP 1-A, 32 kbit/s EEP 2-A, 192 kbit/s EEP 4-B
        mine = np.flatnonzero(member == k)
        twin = _run(pkg, S, d, 0, bs, n, [(int(s), 1, _sel(profs[k])) for s in mine], steps, max_cu=144, msc=576, sf=2880)
        for s in rng.choice(mine, 64, replace=False):
            for x, y in zip(mixed, twin):
                _same_stream(x, y, int(s), _flen(profs[k]), what=f"profile {k}")
    keeper.close()
