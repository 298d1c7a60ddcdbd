"""Generate tests/golden/tonefilt_goldens.npz (and the chroma_filt_*.csv files) with the UNMODIFIED reference:

    python scripts/make_golden_tonefilt.py        # needs `make -C oracle ref` (build container only)

Per case <c>: tf_<c> [T, nNotes], chroma_<c> [T, octaveSize], sma_<c> and de_<c> (cContourSmoother(3) and cDeltaRegression(2)
behind the chroma level): the HTK taps of tests/configs/tonefilt_taps.conf (exact floats); names_tf_<c> / names_chroma_<c> /
names_de_<c> are the CSV headers and ts_<c> [T, 2] the (frameIndex, frameTime) columns of the time-stamped chroma CSV.
Case n1 (one note) has the cTonefilt level only: the reference's cChroma (processArrayFields = 1) finds no array field there and
fails, so it runs TAPS with every level behind cTonefilt removed.
Signals: make_golden_chroma.signals(), length variants of "noise16", and one float WAV ("f32" case, its samples in pcmf_f32).
chroma_filt_16k.csv / chroma_filt_44k1.csv are the output files of the shipped config/chroma/chroma_filt.conf, unchanged, on
"mix16" and "rec".
"""
import os
import struct
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from oracle import refrun  # noqa: E402
import make_golden_chroma as mgc  # noqa: E402

TAPS = os.path.join(ROOT, "tests", "configs", "tonefilt_taps.conf")
BASE = dict(nNotes=72, firstNote=55, decayF0=0.9999, decayFN=0.999, outputPeriod=0.01, octaveSize=12, silThresh=0.001)


def float_signal():
    """a float WAV (format tag 3): the chord of make_golden_chroma at a level int16 cannot hold exactly"""
    pcm, sr, _ = mgc.signals()["chord16"]
    return (pcm.astype(np.float32) * np.float32(0.73 / 32767.0)).astype(np.float32), sr


def signals():
    """name -> (samples (int16, or float32 for a float WAV), sample rate, channels)"""
    s = dict(mgc.signals())
    noise = s["noise16"][0]
    for name, n in (("len0", 160 * 40), ("len1", 160 * 40 + 1), ("lenPm1", 160 * 41 - 1), ("lenShort", 100), ("lenOne", 1)):
        s[name] = (noise[:n].copy(), 16000, 1)
    s["f32"] = float_signal() + (1,)
    return s


# case -> (signal, options of tests/configs/tonefilt_taps.conf)
CASES = {k: (k, {}) for k in ("rec", "on16", "between16", "chord16", "gliss16", "noise16", "quiet16", "mix16", "mix8", "mix48",
                              "mix44", "stereo16", "len0", "len1", "lenPm1", "lenShort", "lenOne", "f32")}
CASES["n1"] = ("mix16", dict(nNotes=1, octaveSize=1))          # cTonefilt level only: cChroma finds no array field on it
CASES["n2"] = ("mix16", dict(nNotes=2, octaveSize=1))
CASES["n12"] = ("mix16", dict(nNotes=12))
CASES["n48"] = ("chord16", dict(nNotes=48))
CASES["n96"] = ("mix44", dict(nNotes=96, octaveSize=24))
CASES["first27"] = ("mix16", dict(firstNote=27.5))
CASES["first100"] = ("chord16", dict(firstNote=100.3))
CASES["decaySwap"] = ("mix16", dict(decayF0=0.99, decayFN=0.9995))          # decayF0 < decayFN: raised to decayFN
CASES["per0125"] = ("rec", dict(outputPeriod=0.0125))                          # 551 samples at 44.1 kHz, period 0.0125
CASES["per0125_16"] = ("mix16", dict(outputPeriod=0.0125, nNotes=48))          # 200 samples
CASES["perBelowT"] = ("lenShort", dict(outputPeriod=0.00001))                  # below 1 / fs: one sample per row
CASES["perOdd"] = ("mix44", dict(outputPeriod=0.0231))                         # 1018.71 samples -> 1019


def options(case):
    o = dict(BASE)
    o.update(CASES[case][1])
    return o


def tf_only_conf():
    """TAPS without the components behind the cTonefilt level"""
    keep, out = True, []
    for ln in open(TAPS).read().split("\n"):
        if ln.startswith("instance[") and not any(x in ln for x in ("dataMemory", "waveSource", "tonefilt]", "tfCsv", "tfHtk")):
            continue
        if ln.startswith("["):
            keep = any(ln.startswith(x) for x in ("[componentInstances", "[waveSource", "[tonefilt:", "[tfCsv", "[tfHtk"))
        if keep:
            out.append(ln)
    return "\n".join(out) + "\n"


def write_float_wav(path, x, sr, nc=1):
    data = np.ascontiguousarray(x, "<f4").tobytes()
    with open(path, "wb") as f:
        f.write(b"RIFF" + struct.pack("<I", 36 + len(data)) + b"WAVE")
        f.write(b"fmt " + struct.pack("<IHHIIHH", 16, 3, nc, sr, sr * 4 * nc, 4 * nc, 32))
        f.write(b"data" + struct.pack("<I", len(data)) + data)


def write_input(path, pcm, sr, nc):
    if pcm.dtype == np.float32:
        write_float_wav(path, pcm, sr, nc)
    else:
        refrun.write_wav(path, pcm, sr, nc)


def csv_table(path):
    lines = open(path).read().strip().split("\n")
    names = lines[0].split(";")
    rows = np.array([[float(x) for x in ln.split(";")] for ln in lines[1:]], np.float64).reshape(-1, len(names))
    return names, rows


def main():
    assert refrun.available(), "build the reference first: make -C oracle ref"
    sigs = signals()
    out = {"pcmf_f32": sigs["f32"][0]}
    for case, (sig, _) in CASES.items():
        pcm, sr, nc = sigs[sig]
        with tempfile.TemporaryDirectory() as d:
            write_input(os.path.join(d, "in.wav"), pcm, sr, nc)
            conf = TAPS
            tfOnly = options(case)["nNotes"] == 1
            if tfOnly:
                conf = os.path.join(d, "tf_only.conf")
                open(conf, "w").write(tf_only_conf())
            cmd = [refrun.SMILEXTRACT, "-C", conf, "-I", "in.wav", "-l", "0"]
            for k, v in options(case).items():
                cmd += ["-" + k, str(v)]
            subprocess.run(cmd, cwd=d, check=True, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
            levels = (("tf", "tonefilt"),) if tfOnly else (("tf", "tonefilt"), ("chroma", "chroma"), ("sma", "sma"), ("de", "de"))
            for key, fn in levels:
                out[key + "_" + case] = refrun.read_htk(os.path.join(d, fn + ".htk"))[0]
                if key != "sma":
                    out["names_%s_%s" % (key, case)] = np.array(csv_table(os.path.join(d, fn + ".csv"))[0])
            if not tfOnly:
                out["ts_" + case] = csv_table(os.path.join(d, "chroma_ts.csv"))[1][:, :2]
        print(case, out["tf_" + case].shape)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "tonefilt_goldens.npz"), **out)
    conf = os.path.join(refrun.CONFIG_DIR, "chroma", "chroma_filt.conf")
    for sig, fn in (("mix16", "chroma_filt_16k.csv"), ("rec", "chroma_filt_44k1.csv")):
        pcm, sr, nc = sigs[sig]
        with tempfile.TemporaryDirectory() as d:
            write_input(os.path.join(d, "in.wav"), pcm, sr, nc)
            subprocess.run([refrun.SMILEXTRACT, "-C", conf, "-I", "in.wav", "-O", os.path.join(ROOT, "tests", "golden", fn), "-l", "0"],
                           cwd=d, check=True, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)


if __name__ == "__main__":
    main()
