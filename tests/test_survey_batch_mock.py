"""batch_decode --scan and --offset auto on the test double of the ABI with the survey (tests/mock_backend/mock_dab_b200_survey.cpp): a
6.144 Msps recording holds two DabTx ensembles at -1 712 000 and +1 712 000 Hz and, between them at 0 Hz, a 1.536 MHz block of
band-limited noise that looks like an ensemble in the spectrum.  The double computes the spectrum with the host build of survey_core.cuh
and runs the library's detector; its frame records come from the oracle's decode of each stream's own 2.048 Msps signal (the noise block's
own signal never synchronises).  Checked: the arguments, the survey call, that every candidate becomes one confirmation stream and only
the confirmed ones are reported, the .scan format, and that --offset auto decodes exactly the reported offsets with the outputs of
--offset at those offsets."""
import os
import subprocess

import numpy as np
import pytest

import dabtx
import surveyref
from conftest import ROOT

R = 6144000
ENSEMBLES = [-1712000, 1712000]


@pytest.fixture(scope="module")
def setup(tmp_path_factory):
    from scipy.signal import resample_poly
    tmp = tmp_path_factory.mktemp("survey_mock")
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "welle.io_b200", "host")])
    mock = tmp / "libdab_b200.so"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", str(mock),
                           os.path.join(ROOT, "tests", "mock_backend", "mock_dab_b200_survey.cpp"),
                           "-L" + os.path.join(ROOT, "oracle"), "-loracle", "-Wl,-rpath," + os.path.join(ROOT, "oracle")])
    rng = np.random.default_rng(0x5CA)
    own = {}
    for k, f in enumerate(ENSEMBLES):
        own[f] = np.concatenate([np.zeros(517 * (k + 1), np.complex64), dabtx.DabTx(seed=0x5C0 + k).frames(12)])
    n = min(len(s) for s in own.values())
    X = np.fft.fft(rng.standard_normal(n) + 1j * rng.standard_normal(n))
    X[np.abs(np.fft.fftfreq(n, 1 / 2048000)) > 768000] = 0
    noise = np.fft.ifft(X)
    own[0] = (noise * np.sqrt(np.mean(np.abs(own[ENSEMBLES[0]]) ** 2) / np.mean(np.abs(noise) ** 2))).astype(np.complex64)
    files = {}
    for f, s in own.items():
        files[f] = tmp / f"own{f}.iq"
        s.tofile(files[f])
    x = np.zeros(n * 3, np.complex128)
    idx = np.arange(n * 3, dtype=np.int64)
    for f, s in own.items():
        x += resample_poly(s[:n].astype(np.complex128), 3, 1) * np.exp(2j * np.pi * (((f % R) * idx) % R) / R)
    wide = tmp / "band.iq"
    x.astype(np.complex64).tofile(wide)
    return tmp, str(wide), {f: str(p) for f, p in files.items()}


def run(tmp, args, iq_lists, name):
    out = tmp / name
    out.mkdir()
    log = tmp / f"{name}.log"
    env = dict(os.environ, LD_LIBRARY_PATH=str(tmp), DABB_MOCK_SURVEY_LOG=str(log), DABB_MOCK_CHAN_LOG=str(tmp / f"{name}.chan"))
    env.pop("DABB_MOCK_IQ", None)
    for k, lst in enumerate(iq_lists):
        env[f"DABB_MOCK_IQ_{k}"] = ":".join(lst)
    r = subprocess.run([os.path.join(ROOT, "welle.io_b200", "batch_decode")] + args + ["--out", str(out)], capture_output=True, text=True,
                       timeout=900, env=env)
    return r, out, (log.read_text().splitlines() if log.exists() else [])


def test_arguments(setup):
    tmp, wide, _ = setup
    exe = os.path.join(ROOT, "welle.io_b200", "batch_decode")
    for args in (["--scan"], ["--offset", "auto"], ["--rate", str(R), "--scan", "--offset", "0"], ["--rate", str(R), "--scan", "--offset", "auto"],
                 ["--rate", str(R)]):
        r = subprocess.run([exe] + args + ["--out", str(tmp), wide], capture_output=True, text=True, timeout=60)
        assert r.returncode == 2 and "usage" in r.stderr, args


def test_scan_and_auto(setup):
    tmp, wide, own = setup
    locate = [own[-1712000], own[0], own[1712000]]             # the candidates in ascending offset: one stream each
    confirm = [own[-1712000]] * 3 + [own[1712000]] * 3            # the two that decoded frames, each at three offsets
    r, out, log = run(tmp, ["--rate", str(R), "--scan", wide], [[own[-1712000]], locate, confirm], "scan")
    assert r.returncode == 0, r.stderr
    assert "survey" in r.stderr and "confirmation of 3 candidate(s) at 6 offsets" in r.stderr, r.stderr
    # one survey call over the first R/4 samples with nfft 2048 (R / 2048 = 3000 Hz), one channelizer over every candidate, then one over
    # the located offsets of those that decoded frames and 1 kHz to either side
    assert log[0] == f"survey 1 {surveyref.nfft_for_rate(R)} {R // 4}" and surveyref.nfft_for_rate(R) == 2048, log
    cands = [int(v) for v in log[1].split()[1:]]
    assert log[1].startswith("chan") and len(cands) == 3 and len(log) == 3, log
    second = [int(v) for v in log[2].split()[1:]]
    assert len(second) == 6 and all(second[3 * k + 1] == second[3 * k] - 1000 and second[3 * k + 2] == second[3 * k] + 1000 for k in range(2)), log
    assert all(abs(second[3 * k] - cands[2 * k]) < 35000 for k in range(2)), log
    for c, f in zip(cands, [-1712000, 0, 1712000]):
        assert abs(c - f) <= 2 * R // 2048, (cands, f)
    # the detector's own candidates on the same spectrum (the numpy restatement of both definitions)
    x = np.fromfile(wide, np.complex64)[:R // 4]
    want = surveyref.candidates(surveyref.spectrum(x, 2048).astype(np.float32), R)
    assert [int(v) for v in want["offset_hz"]] == cands
    lines = (out / "band.iq.scan").read_text().splitlines()
    assert len(lines) == 2, lines                              # the noise block is not confirmed
    offs = []
    for ln, c in zip(lines, [cands[0], cands[2]]):
        f = ln.split(" ", 5)
        offset, cand, score, frames_ok, eid, label = int(f[0]), int(f[1]), float(f[2]), int(f[3]), f[4], f[5]
        assert cand == c and score >= 6.0 and f[2] == f"{score:.2f}" and 2 <= frames_ok <= 16
        assert offset in second                                # the ensembles' own signals carry no carrier offset
        assert eid == "-" and label == "-"                     # DabTx sends neither FIG 0/0 nor FIG 1/0
        assert abs(offset - cand) < 35000
        offs.append(offset)
    assert offs == sorted(offs)
    # --offset auto: the same scan, then exactly the decode of --offset at the reported offsets
    ra, outa, loga = run(tmp, ["--rate", str(R), "--offset", "auto", wide], [[own[-1712000]], locate, confirm, [own[-1712000], own[1712000]]], "auto")
    assert ra.returncode == 0, ra.stderr
    assert loga[3] == "chan " + " ".join(map(str, offs)), loga
    assert not (outa / "band.iq.scan").exists()
    rb, outb, logb = run(tmp, ["--rate", str(R), "--offset", ",".join(map(str, offs)), wide], [[own[-1712000], own[1712000]]], "fixed")
    assert rb.returncode == 0, rb.stderr
    assert ra.stdout == rb.stdout and [ln.split()[0] for ln in ra.stdout.splitlines()] == [f"band.iq@{o}" for o in offs]
    assert sorted(os.listdir(outa)) == sorted(os.listdir(outb))
    for fn in os.listdir(outb):
        assert (outa / fn).read_bytes() == (outb / fn).read_bytes(), fn
    # the channelizer calls of the decode (after those of the three- and six-channel confirmation) are those of --offset
    fixed = (tmp / "fixed.chan").read_text().splitlines()
    auto = (tmp / "auto.chan").read_text().splitlines()
    assert len(auto) > len(fixed) and auto[-len(fixed):] == fixed and all(len(ln.split()) in (3 + 3, 6 + 3) for ln in auto[:-len(fixed)])


def test_nothing_found(setup):
    """a recording of noise: no candidate, an empty .scan, and --offset auto decodes nothing"""
    tmp, _, own = setup
    f = tmp / "noise.iq"
    rng = np.random.default_rng(1)
    (rng.standard_normal(R // 2) + 1j * rng.standard_normal(R // 2)).astype(np.complex64).tofile(f)
    r, out, log = run(tmp, ["--rate", str(R), "--scan", str(f)], [[own[0]]], "noise_scan")
    assert r.returncode == 0 and (out / "noise.iq.scan").read_text() == "" and len(log) == 1, (r.stderr, log)
    r, out, log = run(tmp, ["--rate", str(R), "--offset", "auto", str(f)], [[own[0]]], "noise_auto")
    assert r.returncode == 0 and r.stdout == "" and os.listdir(out) == [], r.stderr
