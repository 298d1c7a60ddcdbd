"""Centred frame sampling in cFramer on the GPU, against the unmodified reference's rows (tests/golden/emo_large_goldens.npz,
scripts/make_golden_emo_large.py): the shipped config/misc/emo_large.conf (frameCenterSpecial = center), tests/configs/
centred_frames.conf (center / right / frameCenter = 0.004 / frameCenterFrames = 37) at 16 kHz mono and 44.1 kHz stereo with
the frame times of the CSV files, and ragged batches whose padded frames must only ever see their own utterance."""
import os

import numpy as np
import pytest

from opensmile_b200.session import Session
from opensmile_b200.synth import mixed_pcm, voiced_pcm
from test_centred_frames_cpu import CONF, EMO_LARGE, G, needs_conf

pytestmark = pytest.mark.gpu
REC = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "egemaps_recordings.npz"))


def _run(s, pcms, sr, nch=1):
    off = np.concatenate([[0], np.cumsum([len(x) for x in pcms])]).astype(np.int64)
    return s.extract_pcm(np.concatenate(pcms).astype(np.int16).reshape(-1), off, float(sr), nch)


def _lld_criterion(rows, ref):
    """the project's LLD criterion (smoke()): every column within 5e-5 of its scale, at most 0.1 % of the values beyond 1e-5"""
    assert rows.shape == ref.shape
    err = np.abs(rows - ref) / (np.abs(ref).max(axis=0) + 1e-30)
    return float(err.max()), float((err > 1e-5).mean()), int(err.max(axis=0).argmax())


def emo_signals():
    return {"rec": (REC["pcm_opensmile_44k1"], 44100), "v": (voiced_pcm(32000, 16000, seed=7), 16000),
            "m": (mixed_pcm(40000, 16000, seed=5), 16000)}


@needs_conf
@pytest.mark.parametrize("key", ["rec", "v", "m"])
def test_emo_large_lld_and_summary(key):
    pcm, sr = emo_signals()[key]
    s = Session(EMO_LARGE, {"lldcsvoutput": "x.csv"}, device=0)
    rows, _ = _run(s, [pcm], sr)
    s.close()
    worst, frac, col = _lld_criterion(rows, G["lld_" + key])
    assert worst < 5e-5 and frac <= 1e-3, (str(G["names_lld"][col]), worst, frac)
    s = Session(EMO_LARGE, {"csvoutput": "x.csv"}, device=0)
    summ, _ = _run(s, [pcm], sr)
    s.close()
    ref = G["func_" + key][0]
    # within 1e-4 of each value's magnitude; a summary of a contour that hovers around zero is held to 1e-5 of the scale of the
    # LLD column it summarises instead (as for emobase.conf).  The ΔΔ contours are not LLD columns: their summaries take the scale
    # of the Δ column.
    names_lld = [str(x) for x in G["names_lld"]]
    col_scale = np.abs(G["lld_" + key]).max(axis=0)

    def lld_col(f):
        f = f.replace("_de_de", "_de", 1)
        return max((j for j, n in enumerate(names_lld) if f.startswith(n + "_")), key=lambda j: len(names_lld[j]))
    floor = np.array([1e-1 * col_scale[lld_col(str(f))] for f in G["names_func"]])
    diff = np.abs(summ[0] - ref)
    rel = np.where(diff == 0, 0.0, diff / np.maximum(np.maximum(np.abs(ref), floor), 1e-30))   # all-zero contours: 0 / 0
    # nzgmean: exp of the mean log magnitude of the non-zero values; the Δ / ΔΔ contours cross zero, and their values next to
    # zero carry the rows' absolute error as a large relative one into the log (up to 2.7e-4 measured)
    tol = np.array([5e-4 if str(f).endswith("_nzgmean") else 1e-4 for f in G["names_func"]])
    bad = np.argsort(-(rel / tol))[:5]
    assert (rel < tol).all(), [(str(G["names_func"][j]), float(summ[0][j]), float(ref[j]), float(rel[j])) for j in bad]


def _cf_input(key):
    return (voiced_pcm(32000, 16000, seed=7), 16000, 1) if key == "v" else (G["pcm_st"], 44100, 2)


CENTRE_SAMPLES = {("c", 16000): 200, ("r", 16000): 399, ("s", 16000): 64, ("f", 16000): 37,
                  ("c", 44100): 551, ("r", 44100): 1102, ("s", 44100): 176, ("f", 44100): 37}


@pytest.mark.parametrize("lv", "crsf")
@pytest.mark.parametrize("key", ["v", "st"])
def test_padded_frames_bit_identical_to_left_frames_of_the_padded_input(lv, key, tmp_path):
    """The device's padded frames, bit for bit: the centred level of x equals, in every column, the left-framed level of x with
    c copies of its first sample frame in front (the same samples in every frame, tests/centred_framer.py, whose padded frames
    equal the reference's cFramer / cVectorPreemphasis levels bit for bit).  Covers the padded staging of lld_kernel (MFCC / PLP,
    spectral magnitudes) and the clamped frame reader of the time-domain kernels (energy, ZCR)."""
    pcm, sr, nch = _cf_input(key)
    c = CENTRE_SAMPLES[(lv, sr)]
    s = Session(CONF, {"level": "lld_" + lv, "csvoutput": "x.csv"}, device=0)
    centred, _ = _run(s, [pcm], sr, nch)
    s.close()
    text = open(CONF).read()
    for line in ("frameCenterSpecial = center", "frameCenterSpecial = right", "frameCenter = 0.004", "frameCenterFrames = 37"):
        text = text.replace(line, "frameCenterSpecial = left")
    left_conf = tmp_path / "left.conf"
    left_conf.write_text(text)
    padded = np.concatenate([np.repeat(pcm[:1], c, axis=0), pcm], axis=0)
    s = Session(str(left_conf), {"level": "lld_" + lv, "csvoutput": "x.csv"}, device=0)
    left, _ = _run(s, [padded], sr, nch)
    s.close()
    assert centred.shape == left.shape
    assert np.array_equal(centred, left), np.argwhere(centred != left)[:5]


@pytest.mark.parametrize("lv", "crsf")
@pytest.mark.parametrize("key", ["v", "st"])
def test_centred_frames_rows_and_csv_times(lv, key, tmp_path):
    """Rows against the reference's within the LLD criterion; of the CSV file the session writes, the header and the name /
    frameIndex / frameTime fields of every line equal the reference's file byte for byte.  The value fields are not compared
    as text: the device FFT's last-bit differences change the sixth significant digit of some values."""
    from oracle import refrun
    pcm, sr, nch = _cf_input(key)
    s = Session(CONF, {"level": "lld_" + lv, "csvoutput": "x.csv"}, device=0)
    rows, _ = _run(s, [pcm], sr, nch)
    worst, frac, col = _lld_criterion(rows, G["cf_%s_%s" % (lv, key)])
    assert worst < 5e-5 and frac <= 1e-3, (str(G["cfnames_" + lv][col]), worst, frac)
    wav = tmp_path / "in.wav"
    refrun.write_wav(str(wav), pcm, sr, nch)
    s.extract_files([str(wav)], csv_paths=[str(tmp_path / "o.csv")])
    s.close()
    got = (tmp_path / "o.csv").read_text().splitlines()
    exp = G["cfcsv_%s_%s" % (lv, key)].tobytes().decode().splitlines()
    assert len(got) == len(exp) and got[0] == exp[0]
    # name, frame index and frame time of every row as the reference prints them
    assert [";".join(g.split(";")[:3]) for g in got] == [";".join(e.split(";")[:3]) for e in exp]
    vals = np.array([[float(x) for x in g.split(";")[3:]] for g in got[1:]], np.float32)
    worst, frac, col = _lld_criterion(vals, G["cf_%s_%s" % (lv, key)])
    assert worst < 5e-5 and frac <= 1e-3, (str(G["cfnames_" + lv][col]), worst, frac)


@pytest.mark.parametrize("lv", "crsf")
def test_padded_frames_see_only_their_own_utterance(lv):
    """utterances of size - c - 1, size - c and size - c + step samples after an utterance with a loud tail: each utterance's
    rows equal its own single run; two runs of the batch are bit-identical"""
    size, step = 400, 160
    c = {"c": 200, "r": 399, "s": 64, "f": 37}[lv]
    rng = np.random.default_rng(3)
    loud = voiced_pcm(8000, 16000, seed=2).astype(np.int32)
    loud[-600:] = np.where(rng.random(600) < 0.5, 32000, -32000)
    utts = [loud.astype(np.int16)] + [voiced_pcm(n, 16000, seed=20 + i) for i, n in enumerate((size - c - 1, size - c, size - c + step))]
    utts += [voiced_pcm(size - c + 3 * step + 7, 16000, seed=30)]
    s = Session(CONF, {"level": "lld_" + lv, "csvoutput": "x.csv"}, device=0)
    rows, fo = _run(s, utts, 16000)
    rows2, _ = _run(s, utts, 16000)
    assert np.array_equal(rows, rows2)
    assert list(np.diff(fo)[1:4]) == [0, 1, 2]
    for u, x in enumerate(utts):
        one, _ = _run(s, [x], 16000)
        assert np.array_equal(rows[fo[u]:fo[u + 1]], one), u
    s.close()


def test_left_framed_rows_unchanged_by_the_centre_plumbing():
    """frameCenterSpecial = left and an explicit frameCenter = 0 give the rows of the default framer, bit for bit"""
    import tempfile
    pcm = voiced_pcm(16000, 16000, seed=4)
    base = open(CONF).read()
    outs = []
    for ctr in ("frameCenterSpecial = left", "frameCenter = 0", ""):
        with tempfile.NamedTemporaryFile("w", suffix=".conf", delete=False) as f:
            f.write(base.replace("frameCenterSpecial = center", ctr))
        s = Session(f.name, {"level": "lld_c", "csvoutput": "x.csv"}, device=0)
        outs.append(_run(s, [pcm], 16000)[0])
        s.close()
        os.unlink(f.name)
    assert np.array_equal(outs[0], outs[1]) and np.array_equal(outs[0], outs[2])
