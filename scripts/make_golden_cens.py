"""Generate tests/golden/cens_goldens.npz (and cens_fft_ds10.csv / cens_fft_ds10.htk) with the UNMODIFIED reference:

    python scripts/make_golden_cens.py        # needs `make -C oracle ref` (build container only)

tests/configs/cens_taps.conf runs both chroma front ends (cTonespec and cTonefilt) with a cCens behind each.  Per case <c> and
path p in (fft, filt): chroma_<p>_<c> and cens_<p>_<c> are the HTK values [T, 12] of the chroma and CENS levels; period_<p>_<c>
is the HTK header period (100 ns units) of the CENS level, time_<p>_<c> the time column of its CSV and names_<p>_<c> its header.
pcm_<c> / sr_<c> is the input (the example recording's samples are those of egemaps_recordings.npz).
Signals: "rec" = the reference's example-audio/opensmile.wav (44.1 kHz), a chord, a glissando, noise, a silent file, one that
starts silent (zero-norm rows), and two utterances shorter than the default window of 41 rows.
cens_fft_ds10.csv / .htk are the reference's own CENS files of the case ds10 (downsampleRatio = 10).
tests/configs/cens_func.conf puts cFunctionals (Means, Extremes and Times, the latter two in seconds) behind the FFT path's cCens:
func_<f> [1, 228] and names_func are its values and header for the cases of FUNC_CASES (signal, downsampleRatio).
"""
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from oracle import refrun  # noqa: E402
from make_golden_chroma import signals as chroma_signals  # noqa: E402

TAPS = os.path.join(ROOT, "tests", "configs", "cens_taps.conf")
FUNC = os.path.join(ROOT, "tests", "configs", "cens_func.conf")
FUNC_CASES = {"chord16_ds1": ("chord16", 1), "chord16_ds10": ("chord16", 10), "gliss16_ds10": ("gliss16", 10),
              "silence16_ds3": ("silence16", 3)}


def signals():
    """name -> (int16 pcm, sample rate, channels)"""
    c = chroma_signals()
    s = {k: c[k] for k in ("rec", "chord16", "gliss16", "noise16", "mix16", "quiet16")}
    s["silence16"] = (np.zeros(16000, np.int16), 16000, 1)
    s["short16"] = (c["chord16"][0][:2400], 16000, 1)          # 9 FFT rows, 15 filter rows: all before W = 41
    s["short16b"] = (c["gliss16"][0][:6400], 16000, 1)         # 35 / 40 rows
    return s


BASE = dict(window="han", winlength=41, l2norm=1, downsampleRatio=1)
CASES = {k: (k, {}) for k in ("rec", "chord16", "gliss16", "noise16", "mix16", "quiet16", "silence16", "short16", "short16b")}
CASES["ham"] = ("mix16", dict(window="ham"))
CASES["bar"] = ("mix16", dict(window="bar"))
CASES["w1"] = ("mix16", dict(winlength=1))
CASES["w101"] = ("gliss16", dict(winlength=101))
CASES["w512"] = ("mix16", dict(winlength=512))
CASES["nonorm"] = ("mix16", dict(l2norm=0))
CASES["nonorm_bar"] = ("quiet16", dict(l2norm=0, window="bar", winlength=7))
CASES["ds10"] = ("mix16", dict(downsampleRatio=10))
CASES["ds10_rec"] = ("rec", dict(downsampleRatio=10, window="ham"))
CASES["ds0"] = ("chord16", dict(downsampleRatio=0))
CASES["wfall"] = ("chord16", dict(window="xyz"))          # unknown: Hanning


def options(case):
    o = dict(BASE)
    o.update(CASES[case][1])
    return o


def csv_table(path):
    lines = open(path).read().strip().split("\n")
    names = lines[0].split(";")
    rows = np.array([[float(x) for x in ln.split(";")] for ln in lines[1:]], np.float64).reshape(-1, len(names))
    return names, rows


def main():
    assert refrun.available(), "build the reference first: make -C oracle ref"
    sigs = signals()
    out = {}
    for case, (sig, _) in CASES.items():
        pcm, sr, nc = sigs[sig]
        with tempfile.TemporaryDirectory() as d:
            refrun.write_wav(os.path.join(d, "in.wav"), pcm, sr, nc)
            cmd = [refrun.SMILEXTRACT, "-C", TAPS, "-I", "in.wav", "-l", "0"]
            for k, v in options(case).items():
                cmd += ["-" + k, str(v)]
            subprocess.run(cmd, cwd=d, check=True, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
            for p in ("fft", "filt"):
                out["chroma_%s_%s" % (p, case)] = refrun.read_htk(os.path.join(d, "chroma_%s.htk" % p))[0]
                vals, hdr = refrun.read_htk(os.path.join(d, "cens_%s.htk" % p))
                out["cens_%s_%s" % (p, case)] = vals
                out["period_%s_%s" % (p, case)] = np.int64(hdr["period"])
                names, rows = csv_table(os.path.join(d, "cens_%s.csv" % p))
                out["names_%s_%s" % (p, case)] = np.array(names[1:])
                out["time_%s_%s" % (p, case)] = rows[:, 0]
            if case == "ds10":
                shutil.copy(os.path.join(d, "cens_fft.csv"), os.path.join(ROOT, "tests", "golden", "cens_fft_ds10.csv"))
                shutil.copy(os.path.join(d, "cens_fft.htk"), os.path.join(ROOT, "tests", "golden", "cens_fft_ds10.htk"))
        out["pcm_" + case] = pcm
        out["sr_" + case] = np.int64(sr)
        print(case, out["cens_fft_" + case].shape, out["cens_filt_" + case].shape, out["period_fft_" + case])
    for fc, (sig, ds) in FUNC_CASES.items():
        pcm, sr, nc = sigs[sig]
        with tempfile.TemporaryDirectory() as d:
            refrun.write_wav(os.path.join(d, "in.wav"), pcm, sr, nc)
            subprocess.run([refrun.SMILEXTRACT, "-C", FUNC, "-I", "in.wav", "-l", "0", "-downsampleRatio", str(ds)], cwd=d, check=True,
                           stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
            out["func_" + fc] = refrun.read_htk(os.path.join(d, "func.htk"))[0]
            out["names_func"] = np.array(csv_table(os.path.join(d, "func.csv"))[0])
        print(fc, out["func_" + fc].shape)
    # the pcm of the example recording is in egemaps_recordings.npz already
    for case, (sig, _) in CASES.items():
        if sig == "rec":
            del out["pcm_" + case]
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "cens_goldens.npz"), **out)


if __name__ == "__main__":
    main()
