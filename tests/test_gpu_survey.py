"""The spectrum survey on the device (dabb_survey: survey_kernel, survey_sum_kernel), the candidate detector on its spectra, and
batch_decode --scan / --offset auto on synthetic wideband recordings.

Spectrum: against the float64 definition (tests/surveyref.py) with the bound of tests/test_survey_emul.py,
|P_j - P_ref_j| <= 1e-4 P_ref_j + 1e-7 mean(P_ref), for every format, host and device input, one and five inputs; the same call twice gives
the same bits.  Refusals write nothing, and a context that surveyed decodes like one that never did.

Closed loop: the recordings of tests/test_gpu_chan.py's closed loop (its builders, imported), whose ensembles here also send FIG 0/0 (EId)
and FIG 1/0 (ensemble label), plus a 2.048 Msps recording mistuned by +200 kHz, an ensemble beside a 6.66 MHz block of band-limited noise
10 dB above the floor, and noise alone.  batch_decode --scan must report every ensemble exactly once, within 30 Hz of its true offset
(the channel offset plus its carrier offset), with its EId and label, and nothing else; the library's detector on the device spectra of
the recordings must give exactly the numpy detector's lists."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import chanref
import dabtx
import surveyref
import test_gpu_chan as tg
from conftest import ROOT, load_pkg

pytestmark = pytest.mark.gpu
EXE = os.path.join(ROOT, "welle.io_b200", "batch_decode")


@pytest.fixture(scope="module")
def ctx():
    c = load_pkg().Context(n_streams=1)
    yield c
    c.close()


def within_bound(p, ref):
    return np.all(np.abs(p.astype(np.float64) - ref) <= 1e-4 * ref + 1e-7 * ref.mean())


def raw_inputs(rng, fmt, n_inputs, n):
    if fmt == 0:
        t = np.arange(n)
        x = [(rng.standard_normal(n) + 1j * rng.standard_normal(n)) * 0.05 + np.exp(2j * np.pi * (0.1 + 0.07 * i) * t) for i in range(n_inputs)]
        return np.stack(x).astype(np.complex64).view(np.uint8)
    return rng.integers(0, 256, (n_inputs, n * chanref.BYTES[fmt]), dtype=np.uint8)


def device_survey(ctx, raw, fmt, n_inputs, nfft, in_len, stride):
    pkg = load_pkg()
    d = ctx.dev(raw)
    psd = np.zeros((n_inputs, nfft), np.float32)
    io = pkg.dabb200.SurveyIO(d.ptr, 0, fmt, stride, n_inputs, nfft, in_len, psd.ctypes.data)
    ctx._ck(ctx.lib.dabb_survey(ctx.h, C.byref(io)))
    d.free()
    return psd


@pytest.mark.parametrize("nfft", [1024, 4096, 16384])
@pytest.mark.parametrize("fmt", [0, 1, 2, 3, 4])
def test_spectrum_against_definition(ctx, nfft, fmt):
    rng = np.random.default_rng(nfft * 7 + fmt)
    for n_inputs in (1, 5):
        in_len = 9 * nfft // 2 + 333                            # odd; the tail past the last segment is never read
        stride = in_len + 17
        raw = raw_inputs(rng, fmt, n_inputs, stride)
        host = ctx.survey(raw, nfft, in_len=in_len, iq_format=fmt)
        dev = device_survey(ctx, raw, fmt, n_inputs, nfft, in_len, stride)
        again = ctx.survey(raw, nfft, in_len=in_len, iq_format=fmt)
        assert host.shape == (n_inputs, nfft)
        assert host.tobytes() == again.tobytes() == dev.tobytes()
        for i in range(n_inputs):
            ref = surveyref.spectrum_raw(raw[i, :in_len * chanref.BYTES[fmt]], fmt, nfft)
            assert within_bound(host[i], ref), (n_inputs, i, np.max(np.abs(host[i] - ref) / (ref + 1e-3 * ref.mean())))


def test_long_input_many_chunks(ctx):
    """0.25 s of 20 Msps s16le in one input: hundreds of chunks summed in double"""
    rng = np.random.default_rng(20)
    n = 5000000
    raw = rng.integers(0, 256, n * 4, dtype=np.uint8)
    psd = ctx.survey(raw, 8192, iq_format=3)
    assert within_bound(psd[0], surveyref.spectrum_raw(raw, 3, 8192))


def test_refusals_write_nothing(ctx):
    pkg = load_pkg()
    lib = ctx.lib
    x = np.zeros((2, 8192), np.complex64)
    canary = np.full((2, 4096), 4321.0, np.float32)

    def call(**kw):
        a = dict(in_=x.ctypes.data, in_is_host=1, iq_format=0, in_stride=8192, n_inputs=2, nfft=4096, in_len=8192, psd=canary.ctypes.data)
        a.update(kw)
        io = pkg.dabb200.SurveyIO(a["in_"], a["in_is_host"], a["iq_format"], a["in_stride"], a["n_inputs"], a["nfft"], a["in_len"], a["psd"])
        return lib.dabb_survey(ctx.h, C.byref(io))

    refusals = {"nfft 512": dict(nfft=512), "nfft 3000": dict(nfft=3000), "nfft 32768": dict(nfft=32768), "format 5": dict(iq_format=5),
                "format -1": dict(iq_format=-1), "in NULL": dict(in_=None), "psd NULL": dict(psd=None), "in_is_host 2": dict(in_is_host=2),
                "stride short": dict(in_stride=8191), "in_len < nfft": dict(in_len=4095), "no inputs": dict(n_inputs=0),
                "4097 inputs": dict(n_inputs=4097)}
    for name, kw in refusals.items():
        assert call(**kw) == -3, name
        assert np.all(canary == 4321.0), name
    assert lib.dabb_survey(None, None) == -3 and lib.dabb_survey(ctx.h, None) == -3
    assert call() == 0 and not np.all(canary == 4321.0)


def test_survey_leaves_the_context_as_it_was():
    """a context that surveyed decodes a 2.048 Msps batch with the same launches, kernels and bytes as a context that never did"""
    pkg = load_pkg()
    txs = [dabtx.DabTx(seed=0xE5 + i) for i in range(2)]
    iq = np.stack([dabtx.add_awgn(tx.frames(8), 20.0, seed=i) for i, tx in enumerate(txs)])
    runs = []
    for surveyed in (False, True):
        c = pkg.Context(n_streams=2)
        try:
            if surveyed:
                c.survey(iq, 16384, iq_format=0)
                c.survey(iq[:, :100000].copy(), 1024)
            d = c.dev(iq)
            c.profile(True)
            l0 = c.kernel_launches()
            outs = [c.process(d, iq.shape[1], np.zeros(2, np.int64), iq.shape[1], msc_stride=288) for _ in range(8)]
            launches = c.kernel_launches() - l0
            kernels = sorted(c.profile_read().keys())
            d.free()
            runs.append((launches, kernels, [(o["results"].tobytes(), o["fibs"].tobytes(), o["msc"].tobytes()) for o in outs]))
        finally:
            c.close()
    assert runs[0][0] == runs[1][0] and runs[0][1] == runs[1][1] and "survey_kernel" not in runs[1][1]
    assert runs[0][2] == runs[1][2]


# ---------------------------------------------------------------------------------------------------------------- closed loop

def eid_of(seed):
    return 0xE000 | (seed & 0xFFF)


def label_of(seed):
    return f"Ensemble {seed:02X}"


class LabelledTx(dabtx.DabTx):
    """DabTx whose FIC blocks carry FIBs [A, B, A]: A = FIG 0/1 + 0/2 + 0/0 (EId), B = FIG 1/0 (the ensemble label)"""

    def __init__(self, seed=0xDAB, **kw):
        super().__init__(seed=seed, **kw)
        e = eid_of(seed)
        fig0_0 = [0x05, 0x00, e >> 8, e & 0xFF, 0x00, 0x00]
        label = label_of(seed).ljust(16).encode()
        fig1_0 = [0x20 | 21, 0x00, e >> 8, e & 0xFF] + list(label) + [0xFF, 0x00]
        a = dabtx.make_fib(dabtx.fig0_1(kw.get("subch_id", 0), self.start_cu, self.profile_a, self.level, self.size_cu)
                           + dabtx.fig0_2(kw.get("sid", 0x1001), kw.get("subch_id", 0)) + fig0_0)
        b = dabtx.make_fib(fig1_0)
        self.fib = a
        self.ficblk = dabtx.conv_encode(np.concatenate([a, b, a]) ^ self.prbs_fic)[dabtx.FIC_MASK]


def labelled_ensembles(monkeypatch, n, seed):
    """tests/test_gpu_chan.py's ensembles(n, seed) built from LabelledTx, and each ensemble's carrier offset (Hz), drawn as it draws them"""
    with monkeypatch.context() as m:
        m.setattr(dabtx, "DabTx", LabelledTx)
        sigs = tg.ensembles(n, seed)
    rng = np.random.default_rng(seed)
    carriers = []
    for k in range(n):
        rng.integers(0, tg.TF)
        carriers.append(int(rng.integers(100, 200)) * (1 if k % 2 else -1))
    return sigs, carriers


def seeds_of(n):
    return [tg.ENSEMBLES[k % len(tg.ENSEMBLES)][0] for k in range(n)]


def read_scan(path):
    out = []
    for ln in path.read_text().splitlines():
        f = ln.split(" ", 5)
        out.append((int(f[0]), int(f[1]), float(f[2]), int(f[3]), f[4], f[5]))
    return out


def run_batch(args, timeout=900):
    r = subprocess.run([EXE] + args, capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0, r.stderr
    print(r.stderr.strip())
    return r


def check_detector_on_device_spectrum(x_raw, fmt, R):
    """the library's detector on the device spectrum of the file's first R/4 samples equals the numpy restatement; returns the candidates"""
    pkg = load_pkg()
    nfft = surveyref.nfft_for_rate(R)
    n = min(R // 4, x_raw.shape[1] // (chanref.BYTES[fmt] if fmt else 1))
    c = pkg.Context(n_streams=1)
    try:
        psd = c.survey(x_raw, nfft, in_len=n, iq_format=fmt)[0]
    finally:
        c.close()
    got = pkg.survey_candidates(psd, R)
    want = surveyref.candidates(psd, R)
    assert got.tobytes() == want.tobytes(), (got, want)
    return got


CLOSED = [  # id, R, format, offsets, gains
    ("10Msps-cf32-5", 10000000, 0, [-3424000, -1712000, 0, 1712000, 3424000], [0.0, 0.0, 20.0, 0.0, 0.0]),
    ("2.4Msps-u8-mistuned", 2400000, 1, [100000], [0.0]),
    ("8.192Msps-s8-3", 8192000, 2, [-1712000, 0, 1712000], [0.0, 20.0, 0.0]),
    ("2.048Msps-mistuned-200kHz", 2048000, 0, [200000], [0.0]),
]


@pytest.mark.parametrize("name,R,fmt,offsets,gains", CLOSED, ids=["10Msps-cf32-5", "2.4Msps-u8-mistuned", "8.192Msps-s8-3", "2.048Msps-mistuned-200kHz"])
def test_scan_finds_every_ensemble(monkeypatch, tmp_path, name, R, fmt, offsets, gains):
    S = len(offsets)
    sigs, carriers = labelled_ensembles(monkeypatch, S, seed=R % 977)
    x = tg.quantize(tg.wideband(sigs, R, offsets, gains, snr_db=24.0, seed=R % 31), fmt)
    f = tmp_path / "rec.iq"
    x.tofile(f)
    cands = check_detector_on_device_spectrum(x, fmt, R)
    assert len(cands) >= S, cands
    out = tmp_path / "out"; out.mkdir()
    fmt_name = ["cf32", "u8", "s8", "s16le", "s16be"][fmt]
    run_batch(["--format", fmt_name, "--rate", str(R), "--scan", "--out", str(out), str(f)])
    scan = read_scan(out / "rec.iq.scan")
    print(name, scan)
    truth = [o + c for o, c in zip(offsets, carriers)]
    assert len(scan) == S, (scan, truth)
    for (off, cand, score, ok, eid, label), t, sd in zip(scan, truth, seeds_of(S)):
        assert abs(off - t) <= 30, (off, t, cand)
        assert cand in [int(v) for v in cands["offset_hz"]] and score >= 6.0 and 2 <= ok <= 16
        assert eid == f"{eid_of(sd):04X}" and label.rstrip() == label_of(sd), (eid, label)
    if name.startswith("2.048"):
        check_mistuned(tmp_path, sigs, f, [o for o, *_ in scan])


def check_mistuned(tmp_path, sigs, f, offs):
    """--offset auto decodes the mistuned recording with the FIBs of its centred original; plain batch_decode of the mistuned file, with
    or without --coarse, gets no FIB through its CRC"""
    centred = tmp_path / "centred.iq"
    tg.quantize(tg.wideband(sigs, 2048000, [0], [0.0], snr_db=24.0, seed=2048000 % 31), 0).tofile(centred)
    auto = tmp_path / "auto"; auto.mkdir()
    r = run_batch(["--rate", "2048000", "--offset", "auto", "--out", str(auto), str(f)])
    assert [ln.split()[0] for ln in r.stdout.splitlines()] == [f"rec.iq@{offs[0]}"]
    plain = tmp_path / "plain"; plain.mkdir()
    run_batch(["--out", str(plain), str(centred)])

    def fic(p):
        recs = np.fromfile(p, np.uint8).reshape(-1, 12 * 33)
        return [(r.tobytes(), sum(int(r[33 * k]) << k for k in range(12))) for r in recs]
    a, b = tg.tracking(fic(auto / f"rec.iq@{offs[0]}.fic")), tg.tracking(fic(plain / "centred.iq.fic"))
    assert len(a) >= tg.FRAMES - 10 and all(m == 0xFFF for _, m in a)
    assert tg.aligned([r for r, _ in a], [r for r, _ in b], tg.FRAMES - 10) is not None
    for extra in ([], ["--coarse"]):
        d = tmp_path / f"mistuned{len(extra)}"; d.mkdir()
        run_batch(extra + ["--out", str(d), str(f)])
        recs = np.fromfile(d / "rec.iq.fic", np.uint8).reshape(-1, 33)
        assert not recs[:, 0].any(), extra


@pytest.fixture(scope="module")
def wide_noise_scan(tmp_path_factory):
    """an ensemble at -6 MHz beside a 6.66 MHz block of band-limited noise 10 dB above the floor (20 Msps): (candidates of the device
    spectrum, the .scan lines, the ensemble's true offset)"""
    R = 20000000
    tmp = tmp_path_factory.mktemp("wide_noise")
    with pytest.MonkeyPatch.context() as mp:
        sigs, carriers = labelled_ensembles(mp, 1, seed=0x20)
    x = tg.wideband(sigs, R, [-6000000], [0.0], snr_db=24.0, seed=5)
    p = float(np.mean(np.abs(sigs[0][1]) ** 2)) * 2048000 / R
    floor = p * (R / 1536000) / 10 ** 2.4                        # the AWGN power per sample (tg.wideband)
    rng = np.random.default_rng(6)
    n = len(x)
    X = np.fft.fft(rng.standard_normal(n) + 1j * rng.standard_normal(n))
    fr = np.fft.fftfreq(n, 1 / R)
    X[np.abs(fr - 2000000) > 3330000] = 0
    blk = np.fft.ifft(X)
    x = (x + blk * np.sqrt(10 * floor * (6660000 / R) / np.mean(np.abs(blk) ** 2))).astype(np.complex64)
    f = tmp / "rec.iq"
    x.tofile(f)
    cands = check_detector_on_device_spectrum(x[None, :], 0, R)
    out = tmp / "out"; out.mkdir()
    run_batch(["--rate", str(R), "--scan", "--out", str(out), str(f)])
    return cands, read_scan(out / "rec.iq.scan"), -6000000 + carriers[0]


def test_scan_beside_wide_noise(wide_noise_scan):
    """no candidate and no report anywhere in the noise block, not even at its edges; the ensemble is found once, within 30 Hz"""
    cands, scan, truth = wide_noise_scan
    assert len(cands) == 1 and abs(int(cands["offset_hz"][0]) + 6000000) <= 2 * 20000000 // 8192, cands
    assert len(scan) == 1 and abs(scan[0][0] - truth) <= 30, scan


def test_scan_of_noise_alone(tmp_path):
    """a recording of noise alone (8.192 Msps): no candidate, an empty .scan"""
    Rn = 8192000
    rng = np.random.default_rng(7)
    noise = (rng.standard_normal(Rn // 2) + 1j * rng.standard_normal(Rn // 2)).astype(np.complex64)
    fn = tmp_path / "noise.iq"
    noise.tofile(fn)
    assert len(check_detector_on_device_spectrum(noise[None, :], 0, Rn)) == 0
    out = tmp_path / "out"; out.mkdir()
    run_batch(["--rate", str(Rn), "--scan", "--out", str(out), str(fn)])
    assert (out / "noise.iq.scan").read_text() == ""
