"""Generate tests/golden/chroma_goldens.npz (and the two chroma_fft_*.csv files) with the UNMODIFIED reference:

    python scripts/make_golden_chroma.py        # needs `make -C oracle ref` (build container only)

Per case <c>: tone_<c> [T, nNotes] and chroma_<c> [T, octaveSize], the tonespec / chroma levels of tests/configs/chroma_taps.conf
(both CSV sinks with a header) for the signal and options of CASES; names_tone_<c> / names_chroma_<c> are the two headers.
Signals (signals() below, seeded): "rec" = the reference's example-audio/opensmile.wav (44.1 kHz, the samples of
tests/golden/egemaps_recordings.npz), pure tones on and between notes, a chord, a glissando over six octaves, noise, near-silence
(below silThresh), at 8 / 16 / 44.1 / 48 kHz, and one stereo file the reference mixes down.  chroma_fft_16k.csv /
chroma_fft_44k1.csv are the output files of the shipped config/chroma/chroma_fft.conf, unchanged, on "mix16" and "rec".
"""
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import refrun  # noqa: E402


def _tone(sr, n, freqs, amp=8000.0, seed=0):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / sr
    x = sum(amp * np.sin(2 * np.pi * f * t + rng.uniform(0, 2 * np.pi)) for f in freqs)
    return np.clip(np.round(x + rng.normal(0, 2.0, n)), -32768, 32767).astype(np.int16)


def signals():
    """name -> (int16 interleaved pcm, sample rate, channels)"""
    s = {}
    rec = np.load(os.path.join(ROOT, "tests", "golden", "egemaps_recordings.npz"))["pcm_opensmile_44k1"]
    s["rec"] = (rec, 44100, 1)
    s["on16"] = (_tone(16000, 12000, [440.0], seed=1), 16000, 1)                                  # A4
    s["between16"] = (_tone(16000, 12000, [440.0 * 2 ** (0.5 / 12)], seed=2), 16000, 1)         # a quarter tone above A4
    s["chord16"] = (_tone(16000, 12000, [261.63, 329.63, 392.0, 130.81], amp=5000, seed=3), 16000, 1)   # C major
    t = np.arange(24000) / 16000.0
    ph = 2 * np.pi * 55.0 * (2.0 ** (6 * t / t[-1]) - 1) * t[-1] / (6 * np.log(2))              # 55 Hz -> 3520 Hz, exponential
    s["gliss16"] = (np.round(9000 * np.sin(ph)).astype(np.int16), 16000, 1)
    s["noise16"] = (np.round(np.random.default_rng(5).normal(0, 3000, 12000)).clip(-32768, 32767).astype(np.int16), 16000, 1)
    quiet = np.round(np.random.default_rng(6).normal(0, 0.6, 12000)).astype(np.int16)           # +-1 LSB: chroma sums below 0.001
    quiet[6000:] = np.round(np.random.default_rng(7).normal(0, 40.0, 6000)).astype(np.int16)    # then noise: every chroma value above
    s["quiet16"] = (quiet, 16000, 1)
    mix = np.concatenate([_tone(16000, 8000, [196.0, 246.9, 293.7], amp=6000, seed=8), s["gliss16"][0][:8000],
                          s["noise16"][0][:4000]])
    s["mix16"] = (mix, 16000, 1)
    s["mix8"] = (np.concatenate([_tone(8000, 6000, [196.0, 493.9], seed=9), _tone(8000, 4000, [880.0], seed=10)]), 8000, 1)
    s["mix48"] = (np.concatenate([_tone(48000, 24000, [261.63, 523.25, 1046.5], seed=11), _tone(48000, 12000, [3000.0], seed=12)]), 48000, 1)
    s["mix44"] = (_tone(44100, 30000, [110.0, 220.0, 659.3], seed=13), 44100, 1)
    left, right = _tone(16000, 10000, [349.2], seed=14), _tone(16000, 10000, [523.3], seed=15)
    s["stereo16"] = (np.stack([left, right], axis=1).reshape(-1), 16000, 2)
    return s


# case -> (signal, options of tests/configs/chroma_taps.conf)
BASE = dict(nOctaves=6, firstNote=55, filterType="gau", usePower=1, dbA=1, octaveSize=12, silThresh=0.001)
CASES = {k: (k, {}) for k in ("rec", "on16", "between16", "chord16", "gliss16", "noise16", "quiet16", "mix16", "mix8", "mix48", "mix44", "stereo16")}
for ft in ("gau", "tri", "trp", "rec"):
    for up in (0, 1):
        for db in (0, 1):
            CASES["v_%s_p%d_d%d" % (ft, up, db)] = ("mix16", dict(filterType=ft, usePower=up, dbA=db))
CASES["oct1"] = ("mix16", dict(nOctaves=1, firstNote=220))
CASES["oct8"] = ("mix44", dict(nOctaves=8))
CASES["note65"] = ("chord16", dict(firstNote=65.406))
CASES["os24"] = ("mix16", dict(nOctaves=6, octaveSize=24))
CASES["tri_rec"] = ("rec", dict(filterType="tri", usePower=0))


def options(case):
    o = dict(BASE)
    o.update(CASES[case][1])
    return o


def csv_rows(path):
    lines = open(path).read().strip().split("\n")
    names = lines[0].split(";")
    rows = np.array([[float(x) for x in ln.split(";")] for ln in lines[1:]], np.float32).reshape(-1, len(names))
    return names, rows


def main():
    assert refrun.available(), "build the reference first: make -C oracle ref"
    sigs = signals()
    wav = os.path.join("/root/reference", "example-audio", "opensmile.wav")
    if os.path.exists(wav):
        assert np.array_equal(refrun.read_wav(wav)[0], sigs["rec"][0])
    taps = os.path.join(ROOT, "tests", "configs", "chroma_taps.conf")
    out = {}
    for case, (sig, _) in CASES.items():
        pcm, sr, nc = sigs[sig]
        with tempfile.TemporaryDirectory() as d:
            refrun.write_wav(os.path.join(d, "in.wav"), pcm, sr, nc)
            cmd = [refrun.SMILEXTRACT, "-C", taps, "-I", "in.wav", "-l", "0"]
            for k, v in options(case).items():
                cmd += ["-" + k, str(v)]
            subprocess.run(cmd, cwd=d, check=True, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
            nt, tone = csv_rows(os.path.join(d, "tone.csv"))
            nc_, ch = csv_rows(os.path.join(d, "chroma.csv"))
        out["tone_" + case], out["chroma_" + case] = tone, ch
        out["names_tone_" + case], out["names_chroma_" + case] = np.array(nt), np.array(nc_)
        print(case, tone.shape, ch.shape)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "chroma_goldens.npz"), **out)
    conf = os.path.join(refrun.CONFIG_DIR, "chroma", "chroma_fft.conf")
    for sig, fn in (("mix16", "chroma_fft_16k.csv"), ("rec", "chroma_fft_44k1.csv")):
        pcm, sr, nc = sigs[sig]
        with tempfile.TemporaryDirectory() as d:
            refrun.write_wav(os.path.join(d, "in.wav"), pcm, sr, nc)
            subprocess.run([refrun.SMILEXTRACT, "-C", conf, "-I", "in.wav", "-O", os.path.join(ROOT, "tests", "golden", fn), "-l", "0"],
                           cwd=d, check=True, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)


if __name__ == "__main__":
    main()
