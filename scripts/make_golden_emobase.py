"""Generate tests/golden/emobase_goldens.npz with the UNMODIFIED reference (oracle/_ref/SMILExtract):

    python scripts/make_golden_emobase.py        # needs `make -C oracle ref` (build container only)

Four inputs: "rec" = the reference's example-audio/opensmile.wav (44.1 kHz; its samples are pcm_opensmile_44k1 of
tests/golden/egemaps_recordings.npz, not stored twice), "v" = voiced_pcm(32000, seed=7), "m" = mixed_pcm(40000, seed=5)
(voiced / noise / silence), "x" = lsp_retry_pcm() (stored as pcm_x), the last three 16 kHz.  Per input <k>:
  lpc_<k> [T, 8]    level taps of tests/configs/emobase_taps.conf: lpc (cLpc p = 8, acf), lsp_<k> [T, 8] (cLsp),
  pitch_<k> [T40, 3] pitch (voiceProb, F0, F0env); cep_m [T40, 512] cepstrum40 (oldCompatCepstrum = 1) of "m" only
  lld_<k> [T, 52]   the -lldcsvoutput rows of the shipped config/emobase/emobase.conf
  func_<k> [1, 988] its -csvoutput row
and names_lld (52), names_func (988) from the two CSV headers.
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
    names = lines[0].split(";")[2:]
    rows = np.array([[float(x) for x in ln.split(";")[2:]] for ln in lines[1:]], np.float32)
    return names, rows


def lsp_retry_pcm():
    """a loud 100 Hz -> 8 kHz chirp and a 7.9 kHz tone: frames whose LSP pairs are too close for the 0.2 grid (cLsp retries
    with 0.05 and finds all roots) and frames where the 0.05 grid misses roots as well (zero fill)"""
    rng = np.random.default_rng(2)
    t = np.arange(32000) / 16000.0
    chirp = 30000 * np.sin(2 * np.pi * (100 * t + (7899 * t * t) / (2 * t[-1])))
    tone = 30000 * np.sin(2 * np.pi * 7900 * t[:8000])
    return np.clip(np.concatenate([chirp, tone]) + rng.normal(0, 1, 40000), -32768, 32767).astype(np.int16)


def main():
    assert refrun.available(), "build the reference first: make -C oracle ref"
    rec = np.load(os.path.join(ROOT, "tests", "golden", "egemaps_recordings.npz"))
    wav = os.path.join("/root/reference", "example-audio", "opensmile.wav")
    if os.path.exists(wav):
        assert np.array_equal(refrun.read_wav(wav)[0], rec["pcm_opensmile_44k1"])
    sigs = {"rec": (rec["pcm_opensmile_44k1"], 44100), "v": (voiced_pcm(32000, 16000, seed=7), 16000),
            "m": (mixed_pcm(40000, 16000, seed=5), 16000), "x": (lsp_retry_pcm(), 16000)}
    taps = open(os.path.join(ROOT, "tests", "configs", "emobase_taps.conf")).read().replace("REFCONF", refrun.CONFIG_DIR)
    conf = os.path.join(refrun.CONFIG_DIR, "emobase", "emobase.conf")
    out = {}
    for key, (pcm, sr) in sigs.items():
        with tempfile.TemporaryDirectory() as d:
            refrun.write_wav(os.path.join(d, "in.wav"), pcm, sr, 1)
            open(os.path.join(d, "t.conf"), "w").write(taps)
            subprocess.run([refrun.SMILEXTRACT, "-C", "t.conf", "-I", "in.wav", "-l", "0"], cwd=d, check=True,
                           stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
            for k in ("lpc", "lsp", "pitch") + (("cep",) if key == "m" else ()):
                out[k + "_" + key] = refrun.read_htk(os.path.join(d, k + ".htk"))[0]
            if key == "x":
                out["pcm_x"] = pcm
            subprocess.run([refrun.SMILEXTRACT, "-C", conf, "-I", "in.wav", "-lldcsvoutput", "l.csv", "-csvoutput", "f.csv",
                            "-l", "0"], cwd=d, check=True, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
            n, out["lld_" + key] = csv_rows(os.path.join(d, "l.csv"))
            out["names_lld"] = np.array(n)
            n, out["func_" + key] = csv_rows(os.path.join(d, "f.csv"))
            out["names_func"] = np.array(n)
    for k, v in out.items():
        print(k, v.shape)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "emobase_goldens.npz"), **out)


if __name__ == "__main__":
    main()
