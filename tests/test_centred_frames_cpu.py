"""Centred frame sampling in cFramer (frameCenterSpecial / frameCenter / frameCenterFrames) without a GPU:
  * frame counts of the graph compiler and the frame times of osm_b200_plan_row_time against a brute-force restatement of the
    reference's rules (core/winToVecProcessor.cpp:461-508 and :1076-1079, core/dataReader.cpp:618-633, core/dataMemoryLevel.cpp:
    1211-1212, noPostEOIprocessing = 1) over a grid of lengths, frame geometries, centre settings and sample rates, and against
    the times of the reference's CSV files;
  * the padded frames: tests/centred_framer.py (copies of sample 0, pre-emphasis over them) equals the reference's cFramer and
    cVectorPreemphasis levels, captured through HTK taps, bit for bit;
  * tests/configs/centred_frames.conf: every centre option parses, names and row counts equal the unmodified reference's
    (tests/golden/emo_large_goldens.npz, scripts/make_golden_emo_large.py);
  * consumers not verified on centred frames are refused by name;
  * the shipped config/misc/emo_large.conf opens unchanged with the reference's 6552 summary / 112 LLD names, in order."""
import os

import re
import shutil

import numpy as np
import pytest

import centred_framer as cfr
from opensmile_b200 import Plan, capi
from opensmile_b200.session import Session, SessionError
from opensmile_b200.synth import voiced_pcm

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
G = np.load(os.path.join(HERE, "golden", "emo_large_goldens.npz"))
CONF = os.path.join(HERE, "configs", "centred_frames.conf")
REC = np.load(os.path.join(HERE, "golden", "egemaps_recordings.npz"))
CF_CENTRES = {"c": ("special", "center"), "r": ("special", "right"), "s": ("sec", 0.004), "f": ("frames", 37)}   # centred_frames.conf
EMO_LARGE = os.path.join(ROOT, "oracle", "_ref", "config", "misc", "emo_large.conf")
needs_conf = pytest.mark.skipif(not os.path.exists(EMO_LARGE), reason="reference configuration files not built (make -C oracle ref)")

FRAMER = """
[componentInstances:cComponentManager]
instance[dataMemory].type = cDataMemory
instance[waveIn].type = cWaveSource
instance[fr].type = cFramer
instance[en].type = cEnergy
instance[csvout].type = cCsvSink
[waveIn:cWaveSource]
writer.dmLevel = wave
filename = \\cm[inputfile(I){test.wav}:input]
[fr:cFramer]
reader.dmLevel = wave
writer.dmLevel = frames
frameSize = %(size)s
frameStep = %(step)s
%(centre)s
[en:cEnergy]
reader.dmLevel = frames
writer.dmLevel = en
[csvout:cCsvSink]
reader.dmLevel = en
filename = \\cm[csvoutput{?}:out]
"""


def c_round(x):
    """C's round(): halves away from zero (Python's round() takes them to even)"""
    return int(np.floor(x + 0.5)) if x >= 0 else -int(np.floor(-x + 0.5))


def centre_frames(centre, size_sec, sr):
    """frameCenterFrames as the reference resolves it (winToVecProcessor.cpp:461-501)"""
    T = 1.0 / sr
    fsf = c_round(size_sec / T)
    kind, val = centre
    if kind == "special":
        fc, cf = 0.0, 0
        if val[:2].lower() in ("mi", "ce"):
            fc = size_sec / 2.0
        elif val[:2].lower() == "ri":
            cf = fsf - 1
        if cf == 0:
            cf = c_round(fc / T)
    elif kind == "frames":
        cf = val
    elif kind == "sec":
        cf = c_round(val / T)
    else:
        cf = 0
    return min(max(cf, 0), fsf - 1)


def centre_seconds(centre, size_sec, sr):
    """the frameCenter (seconds) added to a frame's time when the unclamped frameCenterFrames is > 0, else 0"""
    T = 1.0 / sr
    kind, val = centre
    if kind == "special":
        fc = size_sec / 2.0 if val[:2].lower() in ("mi", "ce") else 0.0
        cf = c_round(size_sec / T) - 1 if val[:2].lower() == "ri" else 0
        if cf == 0:
            cf = c_round(fc / T)
    elif kind == "frames":
        cf, fc = val, val * T
    elif kind == "sec":
        fc, cf = val, c_round(val / T)
    else:
        fc, cf = 0.0, 0
    return fc if cf > 0 else 0.0


def brute_force_time(t, size_sec, step_sec, step, sr, centre):
    """time of the first sample read (clamped at 0) + frameCenter; a time of exactly 0 becomes t * period when the frame is written"""
    c = centre_frames(centre, size_sec, sr)
    if c == 0 and centre_seconds(centre, size_sec, sr) == 0.0:
        return t * step_sec
    s = max(t * step - c, 0)
    tm = s * (1.0 / sr) + centre_seconds(centre, size_sec, sr)
    return t * step_sec if tm == 0.0 else tm


def row_times(conf, options, sr, n_rows, nch=1):
    s = Session(conf, options=options, device=-1)
    comps, level = s.components(float(sr), nch)
    s.close()
    plan = Plan(list(comps), level, device=-1)                     # description only: no device needed
    t = np.array([capi.lib().osm_b200_plan_row_time(plan._h, r) for r in range(n_rows)])
    plan.close()
    return t


def brute_force_frames(L, size, step, c):
    """frame t reads samples [t * step - c, t * step - c + size) and exists iff it ends inside the input"""
    t = 0
    while t * step - c + size <= L:
        t += 1
    return t


CENTRES = [("none", None), ("special", "left"), ("special", "center"), ("special", "MIDdle"), ("special", "right"),
           ("sec", 0.004), ("sec", 0.0123), ("frames", 37), ("frames", 5000), ("frames", -3)]


def centre_lines(centre):
    kind, val = centre
    if kind == "none":
        return ""
    return {"special": "frameCenterSpecial = %s", "sec": "frameCenter = %r", "frames": "frameCenterFrames = %d"}[kind] % val


@pytest.mark.parametrize("size_sec,step_sec", [(0.025, 0.010), (0.032, 0.016), (0.060, 0.010), (0.020, 0.025)])
@pytest.mark.parametrize("sr", [8000, 16000, 44100, 48000])
def test_frame_counts_match_the_rules(size_sec, step_sec, sr, tmp_path):
    size, step = c_round(size_sec / (1.0 / sr)), c_round(step_sec / (1.0 / sr))
    Ls = np.arange(0, 3 * size + 1, max(1, size // 97), dtype=np.int64)
    for centre in CENTRES:
        path = tmp_path / "f.conf"
        path.write_text(FRAMER % {"size": size_sec, "step": step_sec, "centre": centre_lines(centre)})
        s = Session(str(path), options={"csvoutput": "x.csv"}, device=-1)
        off = np.concatenate([[0], np.cumsum(Ls)]).astype(np.int64)
        got = np.diff(s.frame_offsets(off, float(sr), 1))
        s.close()
        c = centre_frames(centre, size_sec, sr)
        exp = np.array([brute_force_frames(int(L), size, step, c) for L in Ls])
        assert np.array_equal(got, exp), (centre, c, Ls[got != exp][:5], got[got != exp][:5], exp[got != exp][:5])


@pytest.mark.parametrize("size_sec,step_sec", [(0.025, 0.010), (0.032, 0.016), (0.060, 0.010)])
@pytest.mark.parametrize("sr", [8000, 16000, 44100, 48000])
def test_first_sample_pad_and_time_match_the_rules(size_sec, step_sec, sr, tmp_path):
    """osm_b200_plan_row_time against the time rule, and the first sample / pad count of every frame against the reference's
    frame level model (frames of a ramp: sample n = n, so a frame's first value is its first sample read, clamped at 0)"""
    step = c_round(step_sec / (1.0 / sr))
    size = c_round(size_sec / (1.0 / sr))
    n = 3 * size // step + 2
    for centre in CENTRES:
        path = tmp_path / "f.conf"
        path.write_text(FRAMER % {"size": size_sec, "step": step_sec, "centre": centre_lines(centre)})
        got = row_times(str(path), {"csvoutput": "x.csv"}, sr, n)
        exp = np.array([brute_force_time(t, size_sec, step_sec, step, sr, centre) for t in range(n)])
        assert np.array_equal(got, exp), (centre, got[got != exp][:3], exp[got != exp][:3])
        c = centre_frames(centre, size_sec, sr)
        ramp = np.arange(3 * size, dtype=np.int16)
        fr = cfr.frames(ramp, size, step, c) * np.float32(32767)
        t = np.arange(fr.shape[0])
        assert np.array_equal(np.rint(fr[:, 0]), np.maximum(t * step - c, 0))                      # first sample read
        pads = np.maximum(c - t * step, 0)
        assert np.array_equal((np.rint(fr) == 0).sum(axis=1), np.where(t * step - c <= 0, pads + 1, 0))   # pads + sample 0 itself


@pytest.mark.parametrize("lv", "crsf")
@pytest.mark.parametrize("key,sr,nch", [("v", 16000, 1), ("st", 44100, 2)])
def test_plan_row_times_equal_the_reference_csv_times(lv, key, sr, nch):
    ref = G["cftime_%s_%s" % (lv, key)]
    got = row_times(CONF, {"level": "lld_" + lv, "csvoutput": "x.csv"}, sr, ref.shape[0], nch)
    assert np.array_equal(np.array(["%f" % x for x in got]), np.array(["%f" % x for x in ref]))   # as the CSV sink prints them


@needs_conf
@pytest.mark.parametrize("key,sr", [("rec", 44100), ("v", 16000), ("m", 16000)])
def test_emo_large_row_times_equal_the_reference_csv_times(key, sr):
    """rows the smoothing / delta stages append at the end of input carry the last frame's time (the sinks clamp the row index
    at the framer level's frame count)"""
    ref = G["lldtime_" + key]
    L = {"rec": REC["pcm_opensmile_44k1"].shape[0], "v": 32000, "m": 40000}[key]
    size, step = c_round(0.025 * sr), c_round(0.010 * sr)
    T = brute_force_frames(L, size, step, centre_frames(("special", "center"), 0.025, sr))
    got = row_times(EMO_LARGE, {"lldcsvoutput": "x.csv"}, sr, T)[np.minimum(np.arange(ref.shape[0]), T - 1)]
    assert np.array_equal(np.array(["%f" % x for x in got]), np.array(["%f" % x for x in ref]))


@pytest.mark.parametrize("lv", "crsf")
@pytest.mark.parametrize("key", ["v", "st"])
def test_padded_frames_and_their_preemphasis_bit_identical_to_the_reference(lv, key):
    pcm, sr = (voiced_pcm(32000, 16000, seed=7), 16000) if key == "v" else (G["pcm_st"], 44100)
    size, step = c_round(0.025 * sr), c_round(0.010 * sr)
    c = centre_frames(CF_CENTRES[lv], 0.025, sr)
    ref, ref_pe = G["frm_%s_%s" % (lv, key)], G["frmpe_%s_%s" % (lv, key)]
    fr = cfr.frames(pcm, size, step, c, n_frames=ref.shape[0])
    assert c > 0 and fr.shape == ref.shape
    assert np.array_equal(fr, ref)
    assert np.array_equal(cfr.preemphasis(fr), ref_pe)


def test_mid_at_44k1_is_the_rounded_half_second_not_half_the_frame():
    assert centre_frames(("special", "center"), 0.025, 44100) == 551       # 1103 samples, 0.0125 s = 551.25 samples


@pytest.mark.parametrize("lv", "crsf")
@pytest.mark.parametrize("key,sr,nch", [("v", 16000, 1), ("st", 44100, 2)])
def test_centred_frames_conf_names_and_row_counts(lv, key, sr, nch):
    s = Session(CONF, options={"level": "lld_" + lv, "csvoutput": "x.csv"}, device=-1)
    assert s.element_names(float(sr), nch) == [str(x) for x in G["cfnames_" + lv]]
    n = 32000 if key == "v" else G["pcm_st"].shape[0]
    fo = s.frame_offsets(np.array([0, n], np.int64), float(sr), nch)
    s.close()
    assert fo[-1] == G["cf_%s_%s" % (lv, key)].shape[0]


@pytest.mark.parametrize("comp,extra", [
    ("cIntensity", "[x:cIntensity]\nreader.dmLevel = winframes_c\nwriter.dmLevel = x\n"),
    ("cLpc", "[x:cLpc]\nreader.dmLevel = framespe_c\nwriter.dmLevel = x\np = 8\n"),
    ("cPitchShs", "[sc:cSpecScale]\nreader.dmLevel = mag_c\nwriter.dmLevel = hps\n[x:cPitchShs]\nreader.dmLevel = hps\nwriter.dmLevel = x\n"),
])
def test_unverified_consumers_of_a_centred_stream_are_refused_by_name(comp, extra, tmp_path):
    text = open(CONF).read()
    inst = "instance[x].type = %s\n" % comp + ("instance[sc].type = cSpecScale\n" if comp == "cPitchShs" else "")
    text = text.replace("instance[csvout].type = cCsvSink\n", inst + "instance[csvout].type = cCsvSink\n") + "\n" + extra
    path = tmp_path / "r.conf"
    path.write_text(text)
    with pytest.raises(SessionError) as e:
        s = Session(str(path), options={"level": "x", "csvoutput": "x.csv"}, device=-1)
        s.element_names()
    assert "'x' (%s)" % comp in str(e.value) and "centred" in str(e.value)


def _centred_copy(name, tmp_path):
    """an existing test configuration with every framer switched to frameCenterSpecial = center"""
    text = open(os.path.join(HERE, "configs", name)).read().replace("REFCONF", os.path.join(ROOT, "oracle", "_ref", "config"))
    if os.path.isdir(os.path.join(HERE, "configs", "inc")):
        shutil.copytree(os.path.join(HERE, "configs", "inc"), tmp_path / "inc", dirs_exist_ok=True)
    text, n = re.subn(r"frameCenterSpecial\s*=\s*left", "frameCenterSpecial = center", text)
    path = tmp_path / name
    path.write_text(text)
    return str(path), n


@pytest.mark.parametrize("name,level,refused", [
    # cPitchJitter reads the wave at positions derived from frame times; its F0 source (the Viterbi-smoothed SHS chain) is the
    # first unverified component the graph compiler meets, and the open fails there
    ("pitch_variants.conf", "jitter", "cPitchSmootherViterbi"),
    ("formant_chain.conf", "formants", "cFormantLpc"),
    ("harmonics_taps.conf", "harmonics", "cPitchSmootherViterbi"),
    ("chroma_taps.conf", "tonespec", "cTonespec"),
    ("chroma_taps.conf", "chroma", "cChroma"),
    ("spectrogram_variants.conf", None, "cFFTmagphase"),
])
def test_centred_variants_of_the_test_configurations_are_refused_by_name(name, level, refused, tmp_path):
    path, n = _centred_copy(name, tmp_path)
    assert n >= 1
    with pytest.raises(SessionError) as e:
        s = Session(path, output_level=level, device=-1)
        s.element_names()
    assert "(%s) on a centred cFramer level" % refused in str(e.value), str(e.value)


@pytest.mark.parametrize("comp,extra", [
    ("cLsp", "[lp:cLpc]\nreader.dmLevel = framespe_c\nwriter.dmLevel = lpc\np = 8\n[x:cLsp]\nreader.dmLevel = lpc\nwriter.dmLevel = x\nprocessArrayFields = 0\n"),
    ("cPlp", "[x:cPlp]\nreader.dmLevel = mel_c\nwriter.dmLevel = x\nfirstCC = 0\nlpOrder = 5\nRASTA = 1\n"),
])
def test_lsp_and_rasta_plp_on_a_centred_stream_are_refused_by_name(comp, extra, tmp_path):
    text = open(CONF).read()
    inst = ("instance[lp].type = cLpc\n" if comp == "cLsp" else "") + "instance[x].type = %s\n" % comp
    text = text.replace("instance[csvout].type = cCsvSink\n", inst + "instance[csvout].type = cCsvSink\n") + "\n" + extra
    path = tmp_path / "r.conf"
    path.write_text(text)
    with pytest.raises(SessionError) as e:
        s = Session(str(path), options={"level": "x", "csvoutput": "x.csv"}, device=-1)
        s.element_names()
    assert "on a centred cFramer level" in str(e.value) and ("'lp' (cLpc)" in str(e.value) or "'x' (%s)" % comp in str(e.value)), str(e.value)


def test_the_same_consumer_on_a_left_framed_stream_still_opens(tmp_path):
    text = open(CONF).read().replace("frameCenterSpecial = center", "frameCenterSpecial = left")
    text = text.replace("instance[csvout].type = cCsvSink\n", "instance[x].type = cIntensity\ninstance[csvout].type = cCsvSink\n")
    path = tmp_path / "l.conf"
    path.write_text(text + "\n[x:cIntensity]\nreader.dmLevel = winframes_c\nwriter.dmLevel = x\n")
    s = Session(str(path), options={"level": "x", "csvoutput": "x.csv"}, device=-1)
    assert len(s.element_names()) >= 1
    s.close()


@needs_conf
@pytest.mark.parametrize("key,sr", [("rec", 44100), ("v", 16000), ("m", 16000)])
def test_emo_large_opens_unchanged_with_the_reference_names(key, sr):
    s = Session(EMO_LARGE, options={"csvoutput": "x.csv"}, device=-1)
    assert s.element_names(float(sr), 1) == [str(x) for x in G["names_func"]]
    s.close()
    s = Session(EMO_LARGE, options={"lldcsvoutput": "x.csv"}, device=-1)
    assert s.element_names(float(sr), 1) == [str(x) for x in G["names_lld"]]
    n = G["lld_" + key].shape[0]
    L = {"rec": REC["pcm_opensmile_44k1"].shape[0], "v": 32000, "m": 40000}[key]
    assert s.frame_offsets(np.array([0, L], np.int64), float(sr), 1)[-1] == n
    s.close()
