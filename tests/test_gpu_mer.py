"""The modulation error ratio on the device (dabb_set_mer, tap 14): bit for bit the host build of mer_core.cuh applied to the step's own
tap-0 softbits (AWGN 0-40 dB, two-path, a tone; both demaps and DABB_CLOCK_TRACK; diversity leaders and members; with and without
keep_taps), equal to the restatement on the oracle's softbits, the same records whatever the batch size, sample offset, ofdm_groups, tail
split and sub-channel selection, the state rules (refusal before the first enable, zeros for streams without a frame and for steps with
the measurement off, toggles between dabb_submit calls, no launch in a context that never enables it), batch_decode --mer against a
Python context, and the AWGN sweep and tone profile of tests/test_mer_emul.py in the closed loop."""
import os
import subprocess

import numpy as np
import pytest

import dabtx
import merref as M
from conftest import ROOT
from test_mer_emul import emul, host_records  # noqa: F401  (emul is a fixture)

pytestmark = pytest.mark.gpu
TF = dabtx.TF


def signals(n_frames, seed=0x3E70):
    """48 recordings of one ensemble: AWGN 0-40 dB (32), two-path (8), a tone (8)"""
    base = dabtx.DabTx(seed=seed).frames(n_frames)
    out = []
    for i in range(32):
        out.append(dabtx.add_awgn(base, 40.0 * i / 31, seed=seed + i))
    for i in range(8):
        out.append(dabtx.add_awgn(M.two_path(base, [(0, 1), (20 + 9 * i, (0.5 + 0.06 * i) * np.exp(1j * i))]), 12 + 3 * i, seed=seed + 100 + i))
    for i in range(8):
        out.append(M.tone(dabtx.add_awgn(base, 20, seed=seed + 200 + i), 1000 * (-700 + 190 * i) + (500 if i % 2 else 0), 10 + 4 * i, seed=i))
    return np.stack(out)


def records_equal(pkg, emul, ctx, res):
    """tap 14 of the last step equals the host build on that step's tap-0 softbits; returns the decoded streams"""
    t14 = ctx.read_tap(14)
    soft = ctx.read_tap(0).reshape(ctx.n_streams, -1)
    act = (res["status"] == pkg.FRAME_DECODED).astype(np.int32)
    want = host_records(emul, soft, act)
    assert t14.tobytes() == want.tobytes(), np.nonzero(t14.view(np.uint8).reshape(ctx.n_streams, -1) != want.view(np.uint8).reshape(ctx.n_streams, -1))[0][:8]
    return act


@pytest.mark.parametrize("keep_taps", [True, False])
@pytest.mark.parametrize("mode", ["reference", "weighted", "clock"])
def test_device_equals_host_build(pkg, emul, keep_taps, mode):  # noqa: F811
    S, steps = 48, 6
    buf = signals(steps + 1)
    # streams 44 .. 47 also form a group of four antennas (the same ensemble under independent noise), 40 .. 41 one of two
    leader = np.arange(S, dtype=np.int32); leader[45:48] = 44; leader[41] = 40
    buf[45:48] = np.stack([dabtx.add_awgn(dabtx.DabTx(seed=0x3E70).frames(steps + 1), 8, seed=0x3E90 + k) for k in range(3)])
    buf[44] = dabtx.add_awgn(dabtx.DabTx(seed=0x3E70).frames(steps + 1), 8, seed=0x3E8F)
    ctx = pkg.Context(n_streams=S, keep_taps=keep_taps)
    ctx.set_options(disable_coarse=True, soft_demap=pkg.DEMAP_WEIGHTED if mode == "weighted" else pkg.DEMAP_REFERENCE,
                    sample_clock=pkg.CLOCK_TRACK if mode == "clock" else pkg.CLOCK_OFF, acquisition=pkg.ACQ_ROBUST)
    ctx.set_combining(leader)
    ctx.set_mer(True)
    d = ctx.dev(buf)
    decoded, combined = 0, 0
    for _ in range(steps):
        res = ctx.process(d, buf.shape[1], np.zeros(S, np.int64), buf.shape[1])["results"]
        decoded += int(records_equal(pkg, emul, ctx, res).sum())
        combined += int((ctx.read_tap(12)["members"] > 1).sum())
    ctx.close()
    assert decoded >= S * (steps - 3) and combined >= steps - 2, (decoded, combined)


def test_device_equals_oracle(pkg, oracle):
    """the exact path: every decoded frame's record equals the restatement on the oracle receiver's softbits of the same frame"""
    base = dabtx.DabTx(seed=0x3EA0).frames(8)
    sigs = [dabtx.add_awgn(base, 15, seed=1), dabtx.add_awgn(base, 30, seed=2), dabtx.add_awgn(M.two_path(base, [(0, 1), (20, 0.95j)]), 25, seed=3)]
    S = len(sigs)
    buf = np.stack(sigs)
    ctx = pkg.Context(n_streams=S)
    ctx.set_mer(True)
    d = ctx.dev(buf)
    got = [[] for _ in range(S)]
    for _ in range(8):
        res = ctx.process(d, buf.shape[1], np.zeros(S, np.int64), buf.shape[1])["results"]
        t14 = ctx.read_tap(14)
        for s in range(S):
            if res["status"][s] == pkg.FRAME_DECODED:
                got[s].append(M.from_tap(t14[s]))
    ctx.close()
    for s, x in enumerate(sigs):
        o = oracle.rx_run(x, disable_coarse=True, want_soft=8)
        want = [M.record(f) for f in o["soft"]]
        n = min(len(want), len(got[s]))
        assert n >= 5, (s, len(want), len(got[s]))
        for k in range(n):
            g, w = got[s][k], want[k]
            assert (g["points"], g["sig"], g["err"], g["gsig"], g["gerr"]) == (w["points"], w["sig"], w["err"], w["gsig"], w["gerr"]), (s, k)
            assert abs(g["mer_db"] - w["mer_db"]) <= 2e-6 * abs(w["mer_db"]), (s, k)


STRIDE = 97


def run_invariance(pkg, d, n_frames, S, j, **kw):
    """the records of stream j (samples from STRIDE * j on) over the steps of an S-stream batch whose stream s starts STRIDE * s samples into
    the recording; sub: select a sub-channel"""
    sub = kw.pop("sub", False)
    ctx = pkg.Context(n_streams=S, **kw)
    ctx.set_mer(True)
    if sub:
        ctx.select_subchannel(0, 72, 96, eep_profile_a=True, eep_level=3)
    out = []
    for _ in range(n_frames - 1):
        ctx.process(d.ptr + 8 * STRIDE * (j - min(j, S - 1)) if S == 1 else d.ptr, STRIDE if S > 1 else 0, np.zeros(S, np.int64), (n_frames - 1) * TF)
        out.append(ctx.read_tap(14)[min(j, S - 1)].tobytes())
    ctx.close()
    return out


def test_invariance(pkg):
    """the same samples give the same records in batches of 1, 48 and 2048 streams, with ofdm_groups 1 / 5 / 25 / 75, the tail split on
    (automatic at 2048 streams) and off, and with and without a sub-channel selected"""
    n_frames = 4
    x = dabtx.add_awgn(M.two_path(dabtx.DabTx(seed=0x3EB0).frames(n_frames), [(0, 1), (31, 0.7j)]), 18, seed=5)
    x = np.concatenate([x, np.zeros(STRIDE * 2048, np.complex64)])
    probe = pkg.Context(n_streams=1)
    d = probe.dev(x)
    j = 37
    ref = run_invariance(pkg, d, n_frames, 1, j)
    assert any(r.strip(b"\0") for r in ref)
    for kw in (dict(S=48), dict(S=2048), dict(S=48, ofdm_groups=1), dict(S=48, ofdm_groups=5), dict(S=48, ofdm_groups=25),
               dict(S=48, ofdm_groups=75), dict(S=2048, ofdm_tail_split=-1), dict(S=48, sub=True), dict(S=2048, sub=True, ofdm_tail_split=-1)):
        S = kw.pop("S")
        assert run_invariance(pkg, d, n_frames, S, j, **kw) == ref, (S, kw)
    d.free()
    probe.close()


def test_state_rules(pkg, emul):  # noqa: F811
    S = 4
    base = dabtx.DabTx(seed=0x3EC0).frames(10)
    noise = dabtx.add_awgn(np.zeros(len(base), np.complex64), 0, seed=9, signal_power=1e-2)
    buf = np.stack([dabtx.add_awgn(base, 20, seed=1), noise, dabtx.add_awgn(base, 25, seed=2), dabtx.add_awgn(base, 30, seed=3)])
    # a context that never enables the measurement: tap 14 refused, no mer_kernel; enabling it adds exactly that launch
    ctx = pkg.Context(n_streams=S)
    with pytest.raises(pkg.DabbError, match="tap 14"):
        ctx.read_tap(14)
    d = ctx.dev(buf)
    bs = np.zeros(S, np.int64)
    for _ in range(2):
        ctx.process(d, buf.shape[1], bs, buf.shape[1])
    ctx.profile(True)
    n0 = ctx.kernel_launches()
    ctx.process(d, buf.shape[1], bs, buf.shape[1])
    plain = ctx.kernel_launches() - n0
    names_plain = set(ctx.profile_read())
    ctx.set_mer(True)
    n0 = ctx.kernel_launches()
    res = ctx.process(d, buf.shape[1], bs, buf.shape[1])["results"]
    assert ctx.kernel_launches() - n0 == plain + 1 and set(ctx.profile_read()) == names_plain | {"mer_kernel"}
    assert "mer_kernel" not in names_plain and plain > 0
    ctx.profile(False)
    ctx.close()

    # zeros for a stream without a frame (noise: NO_SYNC / ACQUIRING; a tracking stream's window far behind it: NEED_SAMPLES) and for a
    # step with the measurement off
    ctx = pkg.Context(n_streams=S)
    ctx.set_mer(True)
    d = ctx.dev(buf)
    seen = set()
    for i in range(5):
        bs = np.zeros(S, np.int64)
        if i >= 3:
            bs[3] = -(1 << 40)          # a tracking stream parked behind its position
        res = ctx.process(d, buf.shape[1], bs, buf.shape[1])["results"]
        act = records_equal(pkg, emul, ctx, res)
        t14 = ctx.read_tap(14)
        for s in range(S):
            seen.add(int(res["status"][s]))
            if not act[s]:
                assert not t14[s].tobytes().strip(b"\0")
    assert {pkg.FRAME_DECODED, pkg.FRAME_NEED_SAMPLES} <= seen and seen & {pkg.FRAME_NO_SYNC, pkg.FRAME_ACQUIRING}
    ctx.set_mer(False)
    res = ctx.process(d, buf.shape[1], bs, buf.shape[1])["results"]
    assert res["status"][0] == pkg.FRAME_DECODED and not ctx.read_tap(14).tobytes().strip(b"\0")
    ctx.close()

    # dabb_submit: a toggle applies from the next submitted step; the steps already enqueued keep theirs
    ctx = pkg.Context(n_streams=S)
    hbuf = np.ascontiguousarray(buf)
    bs = np.zeros(S, np.int64)
    ctx.set_mer(True)
    for _ in range(2):
        ctx.submit(hbuf, hbuf.shape[1], bs, hbuf.shape[1]); ctx.collect()
    ctx.submit(hbuf, hbuf.shape[1], bs, hbuf.shape[1])          # on
    ctx.set_mer(False)
    ctx.submit(hbuf, hbuf.shape[1], bs, hbuf.shape[1])          # off
    ctx.collect(); r = ctx.collect()["results"]
    assert r["status"][0] == pkg.FRAME_DECODED and not ctx.read_tap(14).tobytes().strip(b"\0")
    ctx.submit(hbuf, hbuf.shape[1], bs, hbuf.shape[1])          # off
    ctx.set_mer(True)
    ctx.submit(hbuf, hbuf.shape[1], bs, hbuf.shape[1])          # on
    ctx.collect(); r = ctx.collect()["results"]
    act = records_equal(pkg, emul, ctx, r)
    assert act[0] and ctx.read_tap(14)["sig"][0] > 0
    ctx.close()


def test_batch_decode_mer_matches_context(pkg, tmp_path):
    """batch_decode --mer on two recordings: the .mer lines equal tap 14 of a Python context decoding the same file (selecting the service
    after the first decoded frame, as batch_decode does), and the .merprof holds their int64 sums"""
    exe = os.path.join(ROOT, "welle.io_b200", "batch_decode")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "welle.io_b200", "host")])
    specs = [dict(seed=0x3ED1, snr=14.0, pad=0), dict(seed=0x3ED2, snr=26.0, pad=3001)]
    files, sigs = [], []
    for k, sp in enumerate(specs):
        iq = np.concatenate([np.zeros(sp["pad"], np.complex64), dabtx.add_awgn(dabtx.DabTx(seed=sp["seed"]).frames(12), sp["snr"], seed=sp["seed"])])
        f = tmp_path / f"rec{k}.iq"
        iq.tofile(f); files.append(str(f)); sigs.append(iq)
    outdir = tmp_path / "out"; outdir.mkdir()
    run = subprocess.run([exe, "--mer", "--out", str(outdir)] + files, capture_output=True, text=True, timeout=600)
    assert run.returncode == 0, run.stderr
    for k, sig in enumerate(sigs):
        lines = (outdir / f"rec{k}.iq.mer").read_text().splitlines()
        ctx = pkg.Context(n_streams=1, n_subch_slots=4, max_subch_cu=416)
        ctx.set_mer(True)
        d = ctx.dev(sig[None])
        recs, selected = [], False
        for _ in range(len(sig) // TF + 2):
            r = ctx.process(d, len(sig), np.zeros(1, np.int64), len(sig))["results"][0]
            if r["status"] == pkg.FRAME_NEED_SAMPLES:
                break
            if r["status"] != pkg.FRAME_DECODED:
                continue
            recs.append(M.from_tap(ctx.read_tap(14)[0]))
            if not selected:
                ctx.select_subchannel(0, dabtx.eep_cu(96, True, 3), 96, eep_profile_a=True, eep_level=3, slot=0)
                selected = True
        ctx.close()
        assert len(lines) == len(recs) >= 10, (k, len(lines), len(recs))
        assert lines == [f"{q['points']} {q['mer_db']:.3f} {q['sig']} {q['err']}" for q in recs], k
        prof = [ln.split() for ln in (outdir / f"rec{k}.iq.merprof").read_text().splitlines()]
        assert len(prof) == 64
        for g, p in enumerate(prof):
            assert (int(p[2]), int(p[3])) == (sum(q["gsig"][g] for q in recs), sum(q["gerr"][g] for q in recs)), (k, g)


def test_closed_loop(pkg):
    """on the device: MER rises with the AWGN SNR and lies within 1 dB of SNR + 1.25 dB from 12 to 30 dB; a tone on carrier 301, 10 dB
    above the ensemble at 20 dB SNR, puts group 44 lowest (robust acquisition, which acquires beside the tone)"""
    snrs = [0, 4, 8, 10, 12, 15, 20, 25, 30, 35, 40]
    base = dabtx.DabTx(seed=0x3EE0).frames(9)
    sigs = [dabtx.add_awgn(base, s, seed=0x3EE0 + s) for s in snrs] + [M.tone(dabtx.add_awgn(base, 20, seed=0x3EF0), 301000, 10, seed=1)]
    S = len(sigs)
    buf = np.stack(sigs)
    ctx = pkg.Context(n_streams=S)
    ctx.set_options(disable_coarse=True, acquisition=pkg.ACQ_ROBUST)
    ctx.set_mer(True)
    d = ctx.dev(buf)
    sig, err = np.zeros(S, np.int64), np.zeros(S, np.int64)
    gs, ge = np.zeros((S, 64), np.int64), np.zeros((S, 64), np.int64)
    for _ in range(8):
        ctx.process(d, buf.shape[1], np.zeros(S, np.int64), buf.shape[1])
        t = ctx.read_tap(14)
        sig += t["sig"]; err += t["err"]; gs += t["group"]["sig"]; ge += t["group"]["err"]
    ctx.close()
    mer = [M.mer_db(int(a), int(b)) for a, b in zip(sig, err)]
    assert all(sig[i] > 0 for i, s in enumerate(snrs) if s >= 8) and sig[-1] > 0, sig
    m = [x for x, q in zip(mer[:len(snrs)], sig) if q > 0]
    assert all(b > a for a, b in zip(m, m[1:])), mer
    for s, m in zip(snrs, mer):
        if 12 <= s <= 30:
            assert abs(m - (s + 1.25)) < 1.0, (s, m)
    g = np.array([M.mer_db(int(a), int(b)) for a, b in zip(gs[-1], ge[-1])])
    assert np.argmin(g) == 44, (np.argsort(g)[:4], np.sort(g)[:4])
    print("\nclosed loop MER (dB):", dict(zip(snrs, np.round(mer[:len(snrs)], 2))), "tone: group 44", round(g[44], 2), "median", round(float(np.median(g)), 2))
