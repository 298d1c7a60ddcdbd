"""Generate tests/golden/emo_large_goldens.npz with the UNMODIFIED reference (oracle/_ref/SMILExtract):

    python scripts/make_golden_emo_large.py        # needs `make -C oracle ref` and oracle/_ref/config/misc (build())

The shipped config/misc/emo_large.conf (centred frames: frameCenterSpecial = center) on three inputs: "rec" = the reference's
example-audio/opensmile.wav (44.1 kHz, pcm_opensmile_44k1 of tests/golden/egemaps_recordings.npz), "v" = voiced_pcm(32000,
seed=7), "m" = mixed_pcm(40000, seed=5), both 16 kHz.  Per input <k>:
  lld_<k> [T, 112], lldtime_<k> [T]   the -lldcsvoutput rows and their frame times
  func_<k> [1, 6552]                  the -csvoutput row
and names_lld (112), names_func (6552).
tests/configs/centred_frames.conf, every level <l> of c / r / s / f, on "v" (16 kHz mono) and on "st" = a 44.1 kHz stereo
input (stored as pcm_st [n, 2]):
  cf_<l>_<k> [T, n], cftime_<l>_<k> [T], cfcsv_<l>_<k> (the CSV file's bytes), cfnames_<l>
  frm_<l>_<k> [12, size], frmpe_<l>_<k> [12, size]   the first 12 frames (every padded frame and some after them) of the
                                                     cFramer level and of the cVectorPreemphasis level behind it, through HTK
                                                     taps (big-endian float32: the levels' values bit for bit)
"""
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import refrun  # noqa: E402
from opensmile_b200.synth import mixed_pcm, voiced_pcm  # noqa: E402


def csv_rows(path):
    lines = open(path).read().strip().split("\n")
    head = lines[0].split(";")
    lead = sum(1 for h in head[:3] if h in ("name", "frameIndex", "frameTime"))     # name [; frameIndex] ; frameTime
    names = head[lead:]
    cells = [ln.split(";") for ln in lines[1:]]
    rows = np.array([[float(x) for x in c[lead:]] for c in cells], np.float32).reshape(len(cells), len(names))
    times = np.array([float(c[lead - 1]) for c in cells], np.float64)
    return names, rows, times


def stereo_pcm():
    a = voiced_pcm(44100, 44100, seed=11).astype(np.int32)
    b = mixed_pcm(44100, 44100, seed=12).astype(np.int32)
    return np.stack([a, b], axis=1).astype(np.int16)


def run(d, conf, args):
    subprocess.run([refrun.SMILEXTRACT, "-C", conf, "-I", "in.wav", "-l", "0"] + args, cwd=d, check=True,
                   stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)


def main():
    assert refrun.available(), "build the reference first: make -C oracle ref"
    rec = np.load(os.path.join(ROOT, "tests", "golden", "egemaps_recordings.npz"))
    conf = os.path.join(refrun.CONFIG_DIR, "misc", "emo_large.conf")
    out = {}
    sigs = {"rec": (rec["pcm_opensmile_44k1"], 44100), "v": (voiced_pcm(32000, 16000, seed=7), 16000),
            "m": (mixed_pcm(40000, 16000, seed=5), 16000)}
    for key, (pcm, sr) in sigs.items():
        with tempfile.TemporaryDirectory() as d:
            refrun.write_wav(os.path.join(d, "in.wav"), pcm, sr, 1)
            run(d, conf, ["-lldcsvoutput", "l.csv", "-csvoutput", "f.csv"])
            n, out["lld_" + key], out["lldtime_" + key] = csv_rows(os.path.join(d, "l.csv"))
            out["names_lld"] = np.array(n)
            n, out["func_" + key], _ = csv_rows(os.path.join(d, "f.csv"))
            out["names_func"] = np.array(n)
    cf = os.path.join(ROOT, "tests", "configs", "centred_frames.conf")
    taps = open(cf).read()
    for lv in "crsf":
        taps = taps.replace("instance[csvout].type = cCsvSink\n", "instance[tf_%s].type = cHtkSink\ninstance[tp_%s].type = cHtkSink\n"
                            "instance[csvout].type = cCsvSink\n" % (lv, lv))
        taps += "\n[tf_%s:cHtkSink]\nreader.dmLevel = frames_%s\nfilename = frm_%s.htk\n" % (lv, lv, lv)
        taps += "\n[tp_%s:cHtkSink]\nreader.dmLevel = framespe_%s\nfilename = frmpe_%s.htk\n" % (lv, lv, lv)
    out["pcm_st"] = stereo_pcm()
    for key, (pcm, sr, nch) in {"v": (voiced_pcm(32000, 16000, seed=7), 16000, 1), "st": (out["pcm_st"], 44100, 2)}.items():
        for lv in "crsf":
            with tempfile.TemporaryDirectory() as d:
                refrun.write_wav(os.path.join(d, "in.wav"), pcm, sr, nch)
                run(d, cf, ["-level", "lld_" + lv, "-csvoutput", "o.csv"])
                n, out["cf_%s_%s" % (lv, key)], out["cftime_%s_%s" % (lv, key)] = csv_rows(os.path.join(d, "o.csv"))
                out["cfcsv_%s_%s" % (lv, key)] = np.frombuffer(open(os.path.join(d, "o.csv"), "rb").read(), np.uint8)
                out["cfnames_" + lv] = np.array(n)
        with tempfile.TemporaryDirectory() as d:
            refrun.write_wav(os.path.join(d, "in.wav"), pcm, sr, nch)
            open(os.path.join(d, "taps.conf"), "w").write(taps)
            run(d, "taps.conf", ["-csvoutput", "o.csv"])
            for lv in "crsf":
                for tap in ("frm", "frmpe"):
                    out["%s_%s_%s" % (tap, lv, key)] = refrun.read_htk(os.path.join(d, "%s_%s.htk" % (tap, lv)))[0][:12]
    for k, v in out.items():
        print(k, v.shape)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "emo_large_goldens.npz"), **out)


if __name__ == "__main__":
    main()
