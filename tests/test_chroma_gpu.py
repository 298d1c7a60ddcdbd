"""cTonespec / cChroma on the device: the tone op of lld_kernel (opKind 2) against the unmodified reference's levels
(tests/golden/chroma_goldens.npz, tests/golden/chroma_fft_*.csv, scripts/make_golden_chroma.py) and against the CPU oracle
(oracle/chroma_oracle.py) applied to the device's own magnitude level.

Two checks per level, because the device FFT is not the reference's:
- the tone op's own arithmetic: its rows against the oracle's cTonespec / cChroma on the magnitude level the device computed (the
  plan with cFFTmagphase as output level) hold 1e-6 of the column scale (measured at most 2.4e-7 on every golden case, H100);
- against the reference: a value carries the FFT's round-off of its frame (the device magnitude differs from the reference's by
  ~1e-7 of the frame's spectral peak, tests/test_spectrogram_variants.py).  Notes far from every partial sit at that round-off:
  relative to their own column they differ by up to 5.7e-4 (pure tones, case between16), so the scale of an element is the larger
  of its column's and 1e-2 of its frame's largest value, and the bound is 1e-4 of that (measured at most 5.8e-5, case
  v_tri_p0_d1 chroma; 1e-5 of the plain column scale holds for the recording, noise and glissando cases).

silThresh: a chroma vector is zeroed when one unnormalised value lies below silThresh.  A frame whose smallest value lies within
the FFT's round-off of the threshold can decide differently from the reference; every such frame would be listed here by name with
its measured margin.  None of the goldens has one: the smallest distance of a frame's smallest chroma value from silThresh is
3.3 % of silThresh (case quiet16, computed from the reference's tonespec level), four orders of magnitude above the round-off."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from opensmile_b200 import Plan, Session, capi  # noqa: E402
from oracle import chroma_oracle as co  # noqa: E402
import make_golden_chroma as mg  # noqa: E402

pytestmark = pytest.mark.gpu

G = np.load(os.path.join(HERE, "golden", "chroma_goldens.npz"))
TAPS = os.path.join(HERE, "configs", "chroma_taps.conf")
SHIPPED = os.path.join(ROOT, "oracle", "_ref", "config", "chroma", "chroma_fft.conf")
SIGS = mg.signals()
OWN_TOL = 1e-6      # tone op vs the oracle on the device's magnitudes
REF_TOL = 1e-4      # vs the reference, per element scale max(column scale, 1e-2 x frame scale)


def col_err(got, ref):
    scale = np.maximum(np.abs(ref).max(axis=0), 1e-30)
    return float((np.abs(got - ref) / scale).max()) if ref.size else 0.0


def ref_err(got, ref):
    if not ref.size:
        return 0.0
    scale = np.maximum(np.maximum(np.abs(ref).max(axis=0, keepdims=True), 1e-2 * np.abs(ref).max(axis=1, keepdims=True)), 1e-30)
    return float((np.abs(got - ref) / scale).max())


def device_magnitudes(pcm, sr, nc=1):
    """the magnitude level the device computes for the chroma front end (cFFTmagphase as the output level)"""
    s = Session(TAPS, options={"toneoutput": "x.csv", "chromaoutput": "?"}, output_level="fftmag", device=-1)
    comps, lvl = s.components(float(sr), nc)
    s.close()
    plan = Plan(list(comps), lvl, device=0)
    m = run(plan, [pcm], nc)[0]
    plan.close()
    return m


def fft_frame_size_sec(sr):
    n = int(round(0.064 * sr))
    return 0.064 * (1 << int(np.ceil(np.log2(n)))) / n                  # cTransformFFT's rescale (dspcore/transformFft.cpp:79-83)


def tap_plan(level, sr, nc=1, fmt=0, **opts):
    o = {k: str(v) for k, v in opts.items()}
    o.update({"toneoutput": "x.csv" if level == "tonespec" else "?", "chromaoutput": "x.csv" if level == "chroma" else "?"})
    s = Session(TAPS, options=o, device=-1)
    comps, lvl = s.components(float(sr), nc)
    s.close()
    assert lvl == level
    for c in comps:
        if c.type == capi.C_WAVESOURCE:
            c.u.wavesource.format = fmt
    return Plan(list(comps), lvl, device=0)


def run(plan, utts, nc=1):
    pcm = np.concatenate([np.asarray(u).reshape(-1) for u in utts]) if utts else np.zeros(0, np.int16)
    off = np.concatenate([[0], np.cumsum([u.size // nc for u in utts])]).astype(np.int64)
    rows = plan.run_host(pcm, off)
    fo = plan.frame_offsets(off)
    return [rows[fo[i]:fo[i + 1]] for i in range(len(utts))]


def sil_margin(tone, octave_size, thresh):
    """per frame: min over the chroma values of |value - silThresh| / silThresh (the distance of the frame's decision)"""
    T, N = tone.shape
    s = tone.reshape(T, N // octave_size, octave_size).astype(np.float32).sum(axis=1)
    return np.abs(s.min(axis=1) - thresh) / thresh


@pytest.mark.parametrize("case", sorted(mg.CASES))
def test_levels_against_the_reference(case):
    sig = mg.CASES[case][0]
    pcm, sr, nc = SIGS[sig]
    o = mg.options(case)
    for level in ("tonespec", "chroma"):
        plan = tap_plan(level, sr, nc, **o)
        got = run(plan, [pcm], nc)[0]
        name = plan.last_lld_launch().kernel
        plan.close()
        ref = G[("tone_" if level == "tonespec" else "chroma_") + case]
        assert got.shape == ref.shape, (level, got.shape, ref.shape)
        assert name.startswith("lld_kernel<") and name.endswith(",GEN>"), name
        assert ref_err(got, ref) < REF_TOL, (level, ref_err(got, ref))
        own = co.tonespec(device_magnitudes(pcm, sr, nc), o["nOctaves"], o["firstNote"], o["filterType"], o["usePower"], o["dbA"],
                          fft_frame_size_sec(sr))
        if level == "chroma":
            own = co.chroma(own, o["octaveSize"], o["silThresh"])[0]
        assert col_err(got, own) < OWN_TOL, (level, col_err(got, own))
        zero = ref == 0
        if level == "tonespec":
            assert (got[:, -2:] == 0).all() and np.array_equal(got[zero], ref[zero])
        else:
            # frames the reference zeroed (silThresh / zero total) are zero here, and no other frame is
            rz, gz = (ref == 0).all(axis=1), (got == 0).all(axis=1)
            assert np.array_equal(rz, gz), np.flatnonzero(rz != gz)
            tone = G["tone_" + case]
            m = sil_margin(tone, o["octaveSize"], o["silThresh"])
            assert m.min() > 1e-3, float(m.min())          # every decision lies far outside the FFT's round-off


@pytest.mark.parametrize("fn,sig", [("chroma_fft_16k.csv", "mix16"), ("chroma_fft_44k1.csv", "rec")])
@pytest.mark.skipif(not os.path.exists(SHIPPED), reason="oracle/_ref/config (build()) not there")
def test_shipped_chroma_fft_csv(tmp_path, fn, sig):
    """config/chroma/chroma_fft.conf unchanged: the session writes the CSV file (no header, no index / time) the reference wrote"""
    from oracle import refrun
    pcm, sr, nc = SIGS[sig]
    wav, out = str(tmp_path / "in.wav"), str(tmp_path / "out.csv")
    refrun.write_wav(wav, pcm, sr, nc)
    s = Session(SHIPPED, options={"outputfile": out}, device=0)
    s.extract_files([wav], csv_paths=[out])
    s.close()
    ref_lines = open(os.path.join(HERE, "golden", fn)).read().strip().split("\n")
    got_lines = open(out).read().strip().split("\n")
    assert len(got_lines) == len(ref_lines)
    assert all(len(g.split(";")) == 12 for g in got_lines)
    got = np.array([[float(x) for x in ln.split(";")] for ln in got_lines], np.float32)
    ref = np.array([[float(x) for x in ln.split(";")] for ln in ref_lines], np.float32)
    assert ref_err(got, ref) < REF_TOL, ref_err(got, ref)
    assert np.array_equal((got == 0).all(axis=1), (ref == 0).all(axis=1))


def test_ragged_batch_with_short_and_empty_utterances():
    """1-, 2- and 3-frame utterances (1024 + k * 160 samples at 16 kHz), one too short for a frame and one empty, between
    long ones: every utterance has the oracle's row count and the rows it has when run alone, bit for bit"""
    pcm = SIGS["mix16"][0]
    lens = [16000, 1024, 0, 1184, 700, 1344, 9000]
    utts, at = [], 0
    for n in lens:
        utts.append(pcm[at:at + n].copy())
        at = (at + 997) % (pcm.size - 16000)
    for level in ("tonespec", "chroma"):
        plan = tap_plan(level, 16000)
        got = run(plan, utts)
        for u, x in zip(got, utts):
            T = (x.size - 1024) // 160 + 1 if x.size >= 1024 else 0
            assert u.shape == (T, 72 if level == "tonespec" else 12), (level, x.size, u.shape)
            if T:
                alone = run(plan, [x])[0]
                assert np.array_equal(u.view(np.uint32), alone.view(np.uint32))
                tone, ch, _ = co.extract(x, 16000)
                assert ref_err(u, tone if level == "tonespec" else ch) < REF_TOL
        plan.close()


def test_batch_invariance_2000_utterances():
    """the rows of an utterance do not depend on the batch around it: 2000 utterances of 0.1 .. 0.6 s in one run, against the
    same utterances run alone (bit for bit)"""
    rng = np.random.default_rng(21)
    src = np.concatenate([SIGS["mix16"][0], SIGS["gliss16"][0], SIGS["noise16"][0]])
    utts = []
    for _ in range(2000):
        n = int(rng.integers(1600, 9600))
        a = int(rng.integers(0, src.size - n))
        utts.append(src[a:a + n].copy())
    plan = tap_plan("chroma", 16000)
    big = run(plan, utts)
    for i in list(range(0, 2000, 97)) + [1999]:
        alone = run(plan, [utts[i]])[0]
        assert np.array_equal(big[i].view(np.uint32), alone.view(np.uint32)), i
    plan.close()
    assert sum(b.shape[0] for b in big) > 40000


def test_float_pcm_input_runs_the_f32_instance():
    """the same samples as 32-bit floats (s / 32767): lld_kernel_f32 sees identical samples (tests/test_pcm_float_kernels_gpu.py);
    its FFT is another compilation, so the rows hold the reference bound against the int16 run and the reference"""
    pcm = SIGS["mix16"][0]
    rows = []
    for fmt, x in ((0, pcm), (1, pcm.astype(np.float32) / np.float32(32767))):
        plan = tap_plan("chroma", 16000, fmt=fmt)
        rows.append(run(plan, [x])[0])
        name = plan.last_lld_launch().kernel
        plan.close()
        assert name.startswith("lld_kernel_f32<" if fmt else "lld_kernel<"), name
    assert rows[0].shape == rows[1].shape and ref_err(rows[1], rows[0]) < REF_TOL
    assert ref_err(rows[1], G["chroma_mix16"]) < REF_TOL


MIX = """[componentInstances:cComponentManager]
instance[dataMemory].type=cDataMemory
instance[w].type=cWaveSource
instance[fr].type=cFramer
instance[win].type=cWindower
instance[fft].type=cTransformFFT
instance[mag].type=cFFTmagphase
instance[mel].type=cMelspec
instance[mfcc].type=cMfcc
instance[ts].type=cTonespec
instance[cat].type=cVectorConcat
instance[s].type=cCsvSink
[w:cWaveSource]
writer.dmLevel=wave
[fr:cFramer]
reader.dmLevel=wave
writer.dmLevel=frames
frameSize=0.064
frameStep=0.01
[win:cWindower]
reader.dmLevel=frames
writer.dmLevel=winframes
winFunc=gauss
[fft:cTransformFFT]
reader.dmLevel=winframes
writer.dmLevel=fftc
[mag:cFFTmagphase]
reader.dmLevel=fftc
writer.dmLevel=fftmag
[mel:cMelspec]
reader.dmLevel=fftmag
writer.dmLevel=mel
[mfcc:cMfcc]
reader.dmLevel=mel
writer.dmLevel=mfcc
[ts:cTonespec]
reader.dmLevel=fftmag
writer.dmLevel=tonespec
usePower=1
[cat:cVectorConcat]
reader.dmLevel=%s
writer.dmLevel=out
processArrayFields=0
[s:cCsvSink]
reader.dmLevel=out
filename=x.csv
"""


def test_mfcc_and_tonespec_on_one_fft_chain(tmp_path):
    """two band ops of one FFT stream, one lld_kernel pass each: the concatenated rows equal the rows of each op alone"""
    pcm = SIGS["mix16"][0]
    out = {}
    for lv in ("mfcc;tonespec", "mfcc", "tonespec"):
        p = tmp_path / ("m%d.conf" % len(out))
        p.write_text(MIX % lv)
        s = Session(str(p), device=-1)
        comps, level = s.components(16000.0, 1)
        s.close()
        plan = Plan(list(comps), level, device=0)
        out[lv] = (run(plan, [pcm])[0], plan.element_names)
        plan.close()
    both, names = out["mfcc;tonespec"]
    nm = out["mfcc"][0].shape[1]
    assert names == out["mfcc"][1] + out["tonespec"][1]
    assert np.array_equal(both[:, :nm].view(np.uint32), out["mfcc"][0].view(np.uint32))
    assert np.array_equal(both[:, nm:].view(np.uint32), out["tonespec"][0].view(np.uint32))
    assert ref_err(out["tonespec"][0], G["tone_mix16"]) < REF_TOL
