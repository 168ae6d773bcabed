"""Channel bit errors counted on the device (dabb_options.count_bit_errors, tap 10) against the definition of include/dab_b200.h restated
in numpy (tests/test_ber_emul.py::ref_counts), applied to the softbits the GPU produced (tap 0) and the bytes it decoded: the FIC of
clean and noisy streams, sub-channels across the MSC geometries of tests/test_gpu_msc_geometry.py (restated here) with the fragments
rebuilt by the oracle's time de-interleaver, the same counts without keep_taps, a context that switched the count off against one that
never had it, and batch_decode --ber against a Python context on the same recordings."""
import os
import subprocess

import numpy as np
import pytest

import dabtx
import plainref as P
from conftest import ROOT
from test_ber_emul import ref_counts

pytestmark = pytest.mark.gpu
TF = 196608
FRAMES = 9
MSC = 3 * 1824
SF = 5 * MSC


def fic_ref(soft, fibs):
    """(bits, errors, erasures) of a frame's four FIC codewords: soft = the frame's first 9216 softbits, fibs [12][32]"""
    tot = np.zeros(3, np.int64)
    for b in range(4):
        tot += ref_counts(soft[2304 * b:2304 * (b + 1)], fibs[3 * b:3 * b + 3].reshape(-1), P.FIC_BLOCKS, 768)
    return tuple(int(x) for x in tot)


def fic_of(t10):
    return (int(t10["fic_bits"]), int(t10["fic_errors"]), int(t10["fic_erasures"]))


def sub_of(t10, slot):
    x = t10["subch"][slot]
    return (int(x["codewords"]), int(x["bits"]), int(x["errors"]), int(x["erasures"]))


def test_fic_counts(pkg):
    """64 streams, 16 clean and 48 at 5-14 dB AWGN, keep_taps: every step's tap-10 FIC counts equal the definition on that step's tap-0
    softbits and FIBs; frames not decoded count nothing; clean streams have no errors, those at 10 dB or less do"""
    S, steps = 64, FRAMES
    base = dabtx.DabTx(seed=0xB0).frames(steps + 1)
    snrs = [None] * 16 + [5.0 + 9.0 * i / 47 for i in range(48)]
    buf = np.stack([base if snr is None else dabtx.add_awgn(base, snr, seed=0xB00 + s) for s, snr in enumerate(snrs)])
    ctx = pkg.Context(n_streams=S, keep_taps=True)
    ctx.set_options(disable_coarse=True, count_bit_errors=True)
    d = ctx.dev(buf)
    errs = np.zeros(S, np.int64); decoded = 0
    for _ in range(steps):
        out = ctx.process(d, buf.shape[1], np.zeros(S, np.int64), buf.shape[1])
        r = out["results"]
        soft, t10 = ctx.read_tap(0).reshape(S, -1), ctx.read_tap(10)
        for s in range(S):
            if r["status"][s] == pkg.FRAME_DECODED:
                want = fic_ref(soft[s, :9216], out["fibs"][s])
                assert fic_of(t10[s]) == want, (s, fic_of(t10[s]), want)
                errs[s] += want[1]; decoded += 1
            else:
                assert fic_of(t10[s]) == (0, 0, 0), s
            assert t10[s]["reserved"] == 0 and all(sub_of(t10[s], k) == (0, 0, 0, 0) for k in range(4)), s
    ctx.close()
    assert decoded >= S * 4, decoded
    noisy = np.array([snr is not None and snr <= 10.0 for snr in snrs])      # above 10 dB a frame may well have no channel error
    assert (errs[:16] == 0).all() and (errs[noisy] > 0).all(), errs
    print(f"\nFIC: {decoded} decoded frames, channel errors per stream {errs[16]} (5 dB) .. {errs[-1]} (14 dB)")


# ------------------------------------------------------------------------------------------------ sub-channels
def _eep(br, pa, lv, start, dp=True):
    return dict(start_cu=start, length_cu=dabtx.eep_cu(br, bool(pa), lv), bitrate=br, eep_profile_a=bool(pa), eep_level=lv, dabplus=bool(dp))


def _streams():
    """[(transmitter kwargs, {slot: select kwargs}, SNR or None)]: geometries of tests/test_gpu_msc_geometry.py.  EEP-A and EEP-B at every
    level, CU 0, sub-channels ending at CU 863, the longest codeword (EEP 4-B 1824 kbit/s), UEP on random fill, all four slots, slot 0
    with streams of many profiles, and noise"""
    out = []

    def own(br, pa, lv, start, dp=True, slot=0, snr=None):
        out.append((dict(bitrate=br, profile_a=bool(pa), level=lv, start_cu=start, dabplus=dp), {slot: _eep(br, pa, lv, start, dp)}, snr))
    own(96, 1, 3, 0); own(96, 1, 3, 864 - 72); own(40, 1, 1, 803); own(8, 1, 2, 511); own(8, 1, 4, 860); own(192, 1, 4, 511)
    own(96, 0, 1, 864 - 81); own(64, 0, 2, 1); own(224, 0, 3, 511); own(160, 0, 4, 511); own(1824, 0, 4, 864 - 855, False)
    out.append((dict(start_cu=0), {0: dict(start_cu=864 - 416, length_cu=416, bitrate=384, short_form=True, uep_level=1, dabplus=False)}, None))
    own(128, 1, 3, 200, slot=1); own(64, 1, 1, 600, slot=2); own(320, 1, 4, 700, slot=3)
    out.append((dict(bitrate=96, profile_a=True, level=3, start_cu=300, dabplus=True),
                {0: _eep(96, 1, 3, 300), 1: dict(_eep(128, 1, 4, 300, False), length_cu=72),
                 2: dict(start_cu=0, length_cu=48, bitrate=64, short_form=True, uep_level=3, dabplus=False), 3: _eep(1152, 1, 3, 0, False)}, None))
    for k, snr in enumerate((4.0, 6.0, 8.0)):
        own(192, 1, 4, 100 + 37 * k, snr=snr)
    own(96, 0, 2, 400, slot=1, snr=5.0)
    return out


def _prot(oracle, sel):
    if sel.get("short_form"):
        return oracle.prot_uep(sel["bitrate"], sel["uep_level"])
    return oracle.prot_eep(sel["bitrate"], int(sel["eep_profile_a"]), sel["eep_level"])


def _blocks(prot):
    return [(prot.L[k], prot.PI[k]) for k in range(prot.nblk) if prot.L[k]]


def test_subchannel_counts(pkg, oracle):
    """one context (four slots, max_subch_cu 864), every stream selected before the first step: per step and slot, codewords ==
    n_logical and bits / errors / erasures equal the definition on the fragments the oracle's de-interleaver rebuilds from tap 0 (all
    zero while the de-interleaver fills); the FIC counts equal the definition as well"""
    streams = _streams()
    sigs = []
    for i, (kw, _, snr) in enumerate(streams):
        s = dabtx.DabTx(seed=0x7E0 + i, **kw).frames(FRAMES)
        if snr is not None:
            s = dabtx.add_awgn(s, snr, seed=0x7F0 + i, signal_power=float(np.mean(np.abs(s[3000:190000]) ** 2)))
        sigs.append(s)
    sigs = np.stack(sigs)
    S, n = sigs.shape
    ctx = pkg.Context(n_streams=S, max_subch_cu=864, n_subch_slots=4)
    ctx.set_options(disable_coarse=True, count_bit_errors=True)
    d = ctx.dev(sigs)
    sel = [(s, slot, kw) for s, (_, sl, _) in enumerate(streams) for slot, kw in sl.items()]
    for s, slot, kw in sel:
        ctx.select_subchannel(first=s, count=1, slot=slot, **kw)
    steps = []
    for _ in range(FRAMES):
        o = ctx.process(d, n, np.zeros(S, np.int64), n, msc_stride=MSC, sf_stride=SF)
        steps.append((o, ctx.read_tap(0).reshape(S, -1).copy(), ctx.read_tap(10)))
    d.free(); ctx.close()
    selected = {(s, slot) for s, slot, _ in sel}
    for s in range(S):
        for slot in range(4):
            if (s, slot) not in selected:
                assert all(sub_of(t10[s], slot) == (0, 0, 0, 0) for _, _, t10 in steps), (s, slot)
    total = np.zeros(3, np.int64); n_cw = 0; noisy_err = 0
    for s, slot, kw in sel:
        prot = _prot(oracle, kw)
        blocks, nbits, flen = _blocks(prot), 24 * kw["bitrate"], 3 * kw["bitrate"]
        a, b = 64 * kw["start_cu"], 64 * (kw["start_cu"] + kw["length_cu"])
        cifs, per_step = [], []
        for o, soft, t10 in steps:
            r = o["results"][s]
            if r["status"] != pkg.FRAME_DECODED:
                assert sub_of(t10[s], slot) == (0, 0, 0, 0) and fic_of(t10[s]) == (0, 0, 0), (s, slot)
                per_step.append(None)
                continue
            assert fic_of(t10[s]) == fic_ref(soft[s, :9216], o["fibs"][s]), s
            msc = soft[s, 3 * 3072:].reshape(4, 18 * 3072)
            cifs += [msc[c, a:b] for c in range(4)]
            nl = int(r["n_logical"][slot])
            per_step.append((nl, [o["msc"][s, slot, c, :flen] for c in range(4 - nl, 4)], sub_of(t10[s], slot)))
        de = oracle.deinterleave(np.stack(cifs))
        k = 0; own_err = 0
        for st in per_step:
            if st is None:
                continue
            nl, frames, got = st
            want = np.zeros(3, np.int64)
            for fr in frames:
                want += ref_counts(de[k], fr, blocks, nbits); k += 1
            assert got == (nl,) + tuple(int(x) for x in want), (s, slot, kw, got, want)
            total += want; n_cw += nl; own_err += int(want[1])
        assert k == len(de) >= 8, (s, slot, k, len(de))
        if streams[s][2] is not None:
            noisy_err += own_err
    assert noisy_err > 0
    print(f"\n{len(sel)} sub-channels: {n_cw} logical frames, {int(total[0])} bits, {int(total[1])} errors, {int(total[2])} erasures")


# ------------------------------------------------------------------------------------------------ keep_taps, off
def _overlapping(S, stride, frames, seed):
    """one noisy recording; stream s reads it from sample s * stride on"""
    rec = dabtx.DabTx(seed=seed).frames((S * stride) // TF + frames + 2)
    return dabtx.add_awgn(rec, 7.0, seed=seed)


def _run_tap10(pkg, sig, S, stride, buf_len, steps, keep_taps):
    ctx = pkg.Context(n_streams=S, keep_taps=keep_taps)
    ctx.set_options(disable_coarse=True, count_bit_errors=True)
    ctx.select_subchannel(0, 72, 96, eep_profile_a=True, eep_level=3)
    d = ctx.dev(sig)
    out = []
    for _ in range(steps):
        ctx.process(d, stride, np.zeros(S, np.int64), buf_len, want=("results",))
        out.append(ctx.read_tap(10))
    ctx.close()
    return np.stack(out)


def test_without_keep_taps(pkg):
    """1024 streams: tap 10 without keep_taps is byte-identical to a keep_taps twin"""
    S, stride, frames = 1024, 7919, 9
    sig = _overlapping(S, stride, frames, seed=0xBE1)
    buf_len = frames * TF
    a = _run_tap10(pkg, sig, S, stride, buf_len, frames - 1, keep_taps=False)
    b = _run_tap10(pkg, sig, S, stride, buf_len, frames - 1, keep_taps=True)
    assert a.tobytes() == b.tobytes()
    assert int(a["fic_errors"].sum()) > 0 and int(a["subch"]["codewords"][:, :, 0].sum()) > 0
    print(f"\nkeep_taps=0 vs 1 at {S} streams: identical; {int(a['fic_bits'].sum())} FIC bits, {int(a['subch']['codewords'][:, :, 0].sum())} logical frames")


def test_off_launches_like_never_on(pkg):
    """before the first set tap 10 is refused (DABB_E_STATE); a context that counted and switched the count off launches the same kernels
    per step as one that never had it (count and names), its process outputs and taps 5-8 are byte-identical, and tap 10 is all zero"""
    S, steps, on_steps = 8, 10, 4
    base = dabtx.DabTx(seed=0x0FB).frames(steps + 1)
    buf = np.stack([dabtx.add_awgn(base, 8.0, seed=s) for s in range(S)])
    ctxs = [pkg.Context(n_streams=S), pkg.Context(n_streams=S)]
    ds = []
    for c in ctxs:
        c.select_subchannel(0, 72, 96, eep_profile_a=True, eep_level=3)
        ds.append(c.dev(buf))
    with pytest.raises(pkg.DabbError, match="-5|tap 10"):
        ctxs[1].read_tap(10)
    ctxs[1].set_options(disable_coarse=True, count_bit_errors=True)
    per_step = [[], []]; counted = 0
    for step in range(steps):
        if step == on_steps:
            ctxs[1].set_options(disable_coarse=True, count_bit_errors=False)
            for c in ctxs:
                c.profile(True)
        outs, taps = [], []
        for i, c in enumerate(ctxs):
            n0 = c.kernel_launches()
            o = c.process(ds[i], buf.shape[1], np.zeros(S, np.int64), buf.shape[1], msc_stride=288, sf_stride=1440)
            per_step[i].append(c.kernel_launches() - n0)
            outs.append(b"".join(v.tobytes() for v in o.values()))
            taps.append([c.read_tap(5).tobytes(), c.read_tap(6).tobytes(), c.read_tap(7, stride=288).tobytes(), c.read_tap(8, stride=1440).tobytes()])
        assert outs[0] == outs[1] and taps[0] == taps[1], step
        t10 = ctxs[1].read_tap(10)
        if step >= on_steps:
            assert not t10.tobytes().strip(b"\0"), step
        else:
            counted += int(t10["fic_bits"].sum())
    names = [sorted(c.profile_read()) for c in ctxs]
    assert per_step[0][on_steps:] == per_step[1][on_steps:]
    assert names[0] == names[1] and "ber_kernel" not in names[1]
    assert [b - a for a, b in zip(per_step[0][:on_steps], per_step[1][:on_steps])] == [1] * on_steps     # while on: one launch more
    assert counted > 0
    for c in ctxs:
        c.close()
    print(f"\nlaunches per step never on {per_step[0]}, on then off {per_step[1]}")


# ------------------------------------------------------------------------------------------------ batch_decode
def test_batch_decode_ber_matches_context(pkg, tmp_path):
    """batch_decode --ber on two noisy recordings: every line of DIR/<name>.ber equals tap 10 of a Python context that decodes the same
    file and selects the service after the first decoded frame, as batch_decode does with these recordings"""
    exe = os.path.join(ROOT, "welle.io_b200", "batch_decode")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "welle.io_b200", "host")])
    specs = [dict(seed=0x91, bitrate=96, profile_a=True, level=3, snr=9.0, pad=0),
             dict(seed=0x92, bitrate=64, profile_a=False, level=2, snr=7.0, pad=3001)]
    files, sigs = [], []
    for k, sp in enumerate(specs):
        tx = dabtx.DabTx(seed=sp["seed"], bitrate=sp["bitrate"], profile_a=sp["profile_a"], level=sp["level"])
        iq = np.concatenate([np.zeros(sp["pad"], np.complex64), dabtx.add_awgn(tx.frames(12), sp["snr"], seed=sp["seed"])])
        f = tmp_path / f"rec{k}.iq"
        iq.tofile(f); files.append(str(f)); sigs.append(iq)
    outdir = tmp_path / "out"; outdir.mkdir()
    run = subprocess.run([exe, "--ber", "--out", str(outdir)] + files, capture_output=True, text=True, timeout=600)
    assert run.returncode == 0, run.stderr
    for k, sp in enumerate(specs):
        got = [[int(x) for x in ln.split()] for ln in (outdir / f"rec{k}.iq.ber").read_text().splitlines()]
        sig = sigs[k]
        ctx = pkg.Context(n_streams=1, n_subch_slots=4, max_subch_cu=416)
        ctx.set_options(disable_coarse=True, count_bit_errors=True)
        d = ctx.dev(sig[None])
        want, selected = [], False
        for _ in range(len(sig) // TF + 2):
            r = ctx.process(d, len(sig), np.zeros(1, np.int64), len(sig))["results"][0]
            if r["status"] == pkg.FRAME_NEED_SAMPLES:
                break
            if r["status"] != pkg.FRAME_DECODED:
                continue
            t = ctx.read_tap(10)[0]
            want.append(list(fic_of(t)) + list(sub_of(t, 0)))
            if not selected:
                ctx.select_subchannel(0, dabtx.eep_cu(sp["bitrate"], sp["profile_a"], sp["level"]), sp["bitrate"],
                                      eep_profile_a=sp["profile_a"], eep_level=sp["level"], slot=0)
                selected = True
        ctx.close()
        assert len(got) == len(want) >= 10, (k, len(got), len(want))
        assert got == want, k
        arr = np.array(got)
        assert arr[:, 1].sum() > 0 and arr[:, 3].sum() > 0 and arr[:, 5].sum() > 0, arr
    print(f"\nbatch_decode --ber: {sum(len((outdir / f'rec{k}.iq.ber').read_text().splitlines()) for k in range(2))} lines equal to tap 10")
