"""Case table of the GeMAPS voice-quality kernels (formant_kernel in csrc/formant.cu, harmonics_kernel in csrc/harmonics.cu):
test infrastructure shared by test_formant_sweep_cpu.py and test_formant_sweep_gpu.py.  The anchor is the GeMAPSv01b chain of
tests/configs/harmonics_taps.conf: formants on 20 ms Hamming frames (cTransformFFT -> cSpecResample 11 kHz -> cLpc p = 11 ->
cFormantLpc), SHS pitch -> Viterbi -> cValbasedSelector on 60 ms Gaussian frames, and cHarmonics reading pitch, formants and the
60 ms magnitude level.  Every other case changes one axis from there, a few combine extremes.  One dict per case; the plan's
component list and the host build's arguments are both built from it.  Times are in seconds."""
import functools
import os
import re

import numpy as np

from opensmile_b200 import comp, components_frontend, pack_utterances
from opensmile_b200.synth import mixed_pcm, stereo_mixed_pcm, voiced_pcm
from oracle import oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

ANCHOR = dict(
    sr=16000, n_chan=1, f32=0,
    # formant stream: cFramer / cWindower / cTransformFFT
    frame=0.020, step=0.010, win="ham", zps=1,
    # cSpecResample / cLpc / cFormantLpc (nF = nFormants as configured; the graph clamps it to p - 1)
    target=11000.0, p=11, nF=5, minF=50.0, maxF=5450.0, nvalid=0, freqs=1, bws=1,
    # 60 ms Gaussian stream of the pitch chain and the magnitude level; sel: F0 through cValbasedSelector (else the Viterbi level)
    hframe=0.060, sel=1,
    # cHarmonics: hfmt = reads the formant level; diffs as in the configuration file; fa = formantAmplitudesStart / End
    hfmt=1, nHarm=100, diffs=("H1-H2", "H1-A3"), fa=(1, 3), hnr=1, floor=-201.0,
    # hz = 0: no 60 ms stream (its FFT would be larger than the pitch chain takes): the formant level alone
    hz=1,
)


def case(name, **kw):
    bad = set(kw) - set(ANCHOR)
    assert not bad, bad
    c = dict(ANCHOR, **kw)
    c["name"] = name
    return c


CASES = [
    case("anchor_gemaps"),
    # ---- formant geometry: the composed table (FFT size != 512, or up-sampling I >= K) ----
    case("c8k_20ms", sr=8000),
    case("c12k_20ms", sr=12000),
    case("c32k_20ms", sr=32000),
    case("c44k1_20ms", sr=44100),
    case("c48k_20ms", sr=48000),
    case("c96k_20ms", sr=96000, hz=0),
    case("c16k_to_32k", target=32000.0, maxF=15000.0),
    # ---- reference order, ungathered inverse sum (K = 512, kHalf > 136) ----
    case("u16k_25ms", frame=0.025),
    case("u16k_30ms", frame=0.030),
    case("u16k_to_16k", target=16000.0),
    case("u16k_to_20k", target=20000.0),
    # ---- reference order: no zero padding (N = K); odd padLeft ----
    case("r16k_32ms_nopad", frame=0.032),
    case("r22k05_odd_pad", sr=22050),
    # ---- frame steps, window, the v01a switches, stereo mix-down, float PCM ----
    case("step_5ms", step=0.005),
    case("step_7ms", step=0.007),
    case("step_20ms", step=0.020),
    case("win_hann", win="han"),
    case("v01a", zps=0, maxF=5500.0),
    case("stereo_44k1", sr=44100, n_chan=2),
    case("float32_pcm", f32=1),
    # ---- the 200 KB shared-memory limit: the largest composed geometry the graph pass accepts (48 kHz, 60 ms frames, I = 1536;
    # test_smem_limit_cases_sit_on_the_boundary shows that I = 1537 is refused) ----
    case("smem_largest_accepted", sr=48000, frame=0.060, target=25608.0, maxF=5450.0),
    # ---- predictor order and nFormants: p / 2, p - 1, above p - 1 (clamped); one frame per warp at p = 16 ----
    case("p2_n1", p=2, nF=1, hfmt=1, fa=(1, 1), diffs=("H1-H2", "H1-A1")),
    case("p4_n2", p=4, nF=2, fa=(1, 2), diffs=("H1-H2", "H1-A2")),
    case("p4_n9_clamped", p=4, nF=9, fa=(1, 3)),
    case("p6_n3", p=6, nF=3),
    case("p8_n4", p=8, nF=4),
    case("p8_n7", p=8, nF=7, fa=(1, -1)),
    case("p11_n10", p=11, nF=10, hfmt=0),
    case("p15_n7", p=15, nF=7),
    case("p15_n14", p=15, nF=14, hfmt=0),
    case("p16_n8", p=16, nF=8, fa=(1, -1), diffs=("H1-A8", "A1-A8", "H2-A7")),
    case("p16_n15", p=16, nF=15, hfmt=0),
    case("p16_n20_clamped", p=16, nF=20, hfmt=0),
    # ---- formant outputs ----
    case("o_nvalid_only", nvalid=1, freqs=0, bws=0, hfmt=0),
    case("o_freqs_no_bws", bws=0, hfmt=0),
    case("o_bws_only", freqs=0, hfmt=0),
    case("o_all_outputs", nvalid=1),
    case("o_200_3000", minF=200.0, maxF=3000.0),
    case("o_maxF_above_fs", maxF=12000.0),
    # ---- cHarmonics: magnitude spectra of 257, 1025 and 2049 bins ----
    case("h8k", sr=8000),
    case("h22k05", sr=22050),
    case("h44k1", sr=44100),
    case("h48k", sr=48000),
    # ---- cHarmonics: harmonics per frame (one pass of the lane loop, 33, 128; a difference naming harmonic 40) ----
    case("h_nharm_20", nHarm=20),
    case("h_nharm_33", nHarm=33),
    case("h_nharm_128", nHarm=128),
    case("h_diff_names_h40", nHarm=20, diffs=("H1-H40", "H2-A1")),
    # ---- cHarmonics options ----
    case("h_no_formant_level", hfmt=0),
    case("h_a0_and_beyond_nfmt", diffs=("H1-A0", "A0-A6", "A1-A2", "H3-H1")),
    case("h_fa_2_5", fa=(2, 5)),
    case("h_fa_all", fa=(1, -1)),
    case("h_fa_none", fa=(3, 2)),
    case("h_no_hnr_floor_100", hnr=0, floor=-100.0),
    case("h_no_diffs", diffs=()),
    case("h_viterbi_f0", sel=0),
    # ---- extremes combined ----
    case("x_48k_p16_n8_5ms", sr=48000, step=0.005, p=16, nF=8, nHarm=128, fa=(1, -1)),
    case("x_8k_p4_stereo", sr=8000, p=4, nF=2, n_chan=2, fa=(1, 2), diffs=("H1-A2",), hnr=0),
]
BY_NAME = {c["name"]: c for c in CASES}
assert len(BY_NAME) == len(CASES)

# the values every axis must reach (test_table_reaches_every_axis_value); `path` and `fpw` are read from the host build's path
# query (formant_harness.formant_path), nb from the 60 ms stream's FFT size
AXES = dict(
    sr={8000, 12000, 16000, 22050, 32000, 44100, 48000, 96000}, frame={0.020, 0.025, 0.030, 0.032, 0.060},
    step={0.005, 0.007, 0.010, 0.020}, win={"ham", "han"}, zps={0, 1}, n_chan={1, 2}, f32={0, 1},
    p={2, 4, 8, 11, 15, 16}, nvalid={0, 1}, freqs={0, 1}, bws={0, 1}, path={"composed", "gathered", "ungathered"}, fpw={1, 2},
    pad_parity={0, 1}, nopad={0, 1}, upsampled={0, 1}, nF_rule={"p/2", "p-1", "clamped"},
    nb={0, 257, 513, 1025, 2049}, nHarm={20, 33, 100, 128}, hfmt={0, 1}, hnr={0, 1}, sel={0, 1}, n_fmt_h={0, 1, 3, 8},
)


# ---------------------------------------------------------------- geometry
def geometry(c, hz=False):
    """(N, S, nfft) of the formant stream (hz = the 60 ms stream) as the graph computes them (graph.cpp: round(frameSize * sr))"""
    fe = oracle.frontend(float(c["sr"]), c["hframe"] if hz else c["frame"], c["step"], win="ham")
    N, S, nfft, _ = oracle.geometry(fe, 0)
    return N, S, nfft


def frames(c, n_samples, hz=False):
    N, S, _ = geometry(c, hz)
    return 0 if n_samples < N else (n_samples - N) // S + 1


def n_formants(c):
    """nFormants after the graph's clamp (tables.cpp build_formant)"""
    nF = c["nF"]
    if nF > c["p"] - 1 or nF <= 0:
        nF = c["p"] - 1
    return nF


def path(c):
    """formant_kernel's path for the case (composed / gathered / ungathered, frames per warp, ...) from the host build"""
    import formant_harness as fh
    N, S, nfft = geometry(c)
    return fh.formant_path(float(c["sr"]), N, nfft, c["frame"], c["zps"], c["target"], c["p"], c["nF"])


def axis_values(c):
    """the case's value on every axis of AXES"""
    info = path(c)
    N, S, nfft = geometry(c)
    nF = n_formants(c)
    v = {k: c[k] for k in AXES if k in c}
    v["path"] = "composed" if not info["ref_order"] else ("gathered" if info["gathered"] else "ungathered")
    v["fpw"] = info["fpw"]
    v["pad_parity"] = info["pad_left"] & 1
    v["nopad"] = int(N == nfft)
    v["upsampled"] = int(info["n_res"] >= nfft)
    v["nF_rule"] = "clamped" if c["nF"] > c["p"] - 1 else ("p-1" if nF == c["p"] - 1 else ("p/2" if nF == c["p"] // 2 else "other"))
    v["nb"] = geometry(c, hz=True)[2] // 2 + 1 if c["hz"] else 0
    v["n_fmt_h"] = nF if c["hfmt"] else 0
    return v


@functools.lru_cache(maxsize=None)
def _tile_rule():
    src = open(os.path.join(ROOT, "opensmile_b200", "csrc", "kernels.cu")).read()
    m = re.search(r"const int F = nfft == 4096 \? (\d+) : \(nfft == 2048 \? (\d+) : (\d+)\);", src)
    assert m, "lld_tile_frames changed: update formant_cases.tile_width"
    return tuple(int(g) for g in m.groups())


def tile_width(c):
    """frames per tile of the formant stream: lld_tile_frames (kernels.cu) of its FFT size, read from the source"""
    f4096, f2048, other = _tile_rule()
    nfft = geometry(c)[2]
    return f4096 if nfft == 4096 else (f2048 if nfft == 2048 else other)


# ---------------------------------------------------------------- plan side
def components(c):
    """wave -> 20 ms stream (`win` -> `fft` -> `res` -> `lpc` -> `formants`) and 60 ms Gaussian stream (`h_mag` -> `scale` ->
    `shs` -> `vit` [-> `pitch` through cValbasedSelector on the rms energy]) -> cHarmonics (`harm`)"""
    sr, nc = float(c["sr"]), c["n_chan"]
    cs = components_frontend(sr, c["frame"], c["step"], win=c["win"], n_channels=nc, with_fft=True, zero_pad_symmetric=c["zps"])
    cs = [x for x in cs if x.name != b"mag"]                                       # the formant stream has no magnitude level
    if c["f32"]:
        cs[0].u.wavesource.format = 1
    cs.append(comp("cSpecResample", "res", "fft", "res", targetFs=c["target"]))
    cs.append(comp("cLpc", "lpc", "res", "lpc", method=0, p=c["p"], saveLPCoeff=1, lpGain=0))
    cs.append(comp("cFormantLpc", "formants", "lpc", "formants", nFormants=c["nF"], saveFormants=c["freqs"], saveBandwidths=c["bws"],
                   saveNumberOfValidFormants=c["nvalid"], minF=c["minF"], maxF=c["maxF"]))
    if not c["hz"]:
        return cs
    hs = components_frontend(sr, c["hframe"], c["step"], win="gau", sigma=0.4, n_channels=nc, prefix="h_")
    cs += hs[1:]                                                                   # one wave source
    cs.append(comp("cSpecScale", "scale", "h_mag", "hps", scaleOctave=1, sourceLin=1, splineInterp=1, minF=25.0, maxF=-1.0,
                   nPointsTarget=0, specSmooth=1, specEnhance=1, auditoryWeighting=1))
    cs.append(comp("cPitchShs", "shs", "hps", "shs", maxPitch=1000.0, minPitch=55.0, nCandidates=6, scores=1, voicing=1, F0C1=0,
                   voicingC1=0, F0raw=1, voicingClip=1, voicingCutoff=0.70, octaveCorrection=0, nHarmonics=15, compressionFactor=0.85,
                   greedyPeakAlgo=1))
    cs.append(comp("cPitchSmootherViterbi", "vit", "shs", "vit", bufferLength=40, F0final=1, F0finalLog=1, F0finalEnv=0,
                   F0finalEnvLog=0, voicingFinalClipped=0, voicingFinalUnclipped=1, F0raw=0, voicingC1=0, voicingClip=0, wLocal=2.0,
                   wTvv=10.0, wTvvd=5.0, wTvuv=10.0, wThr=4.0, wRange=1.0, wTuu=0.0))
    if c["sel"]:
        cs.append(comp("cEnergy", "energy", "h_win", "e", htkcompatible=0, rms=1, energy2=0, log=0, escaleLog=1.0, escaleRms=1.0,
                       escaleSquare=1.0, ebiasLog=0.0, ebiasRms=0.0, ebiasSquare=0.0))
        cs.append(comp("cValbasedSelector", "sel", "e;vit", "pitch", threshold=0.001, idx=0, invert=0, allowEqual=0, removeIdx=1,
                       zeroVec=1, adaptiveThreshold=0, outputVal=0.0))
    readers = [f0_level(c)] + (["formants"] if c["hfmt"] else []) + ["h_mag"]
    h = comp("cHarmonics", "harm", ";".join(readers), "harm", f0ElementName="F0final", f0ElementNameIsFull=1,
             magSpecFieldName="pcm_fftMag", magSpecFieldNameIsFull=1, formantFrequencyFieldName="formantFreqLpc",
             formantFrequencyFieldNameIsFull=1, formantBandwidthFieldName="formantBandwidthLpc", formantBandwidthFieldNameIsFull=1,
             nHarmonics=c["nHarm"], harmonicDifferencesLog=1, formantAmplitudes=1, formantAmplitudesLogRel=1,
             formantAmplitudesStart=c["fa"][0], formantAmplitudesEnd=c["fa"][1], computeAcfHnrLogdB=c["hnr"],
             logRelValueFloorUnvoiced=c["floor"])
    hh = h.u.harmonics
    hh.nHarmonicDifferences = len(c["diffs"])
    for i, d in enumerate(c["diffs"]):
        hh.harmonicDifferences[i].value = d.encode()
    cs.append(h)
    return cs


def f0_level(c):
    return "pitch" if c["sel"] else "vit"


def _field(name, n, first=1):
    return [name] if n == 1 else ["%s[%d]" % (name, i) for i in range(first, first + n)]     # a one-element field has no index


def formant_names(c):
    """lld/formantLpc.cpp:113-136: fixed names, array indices from 1"""
    nF = n_formants(c)
    return ((["nFormants"] if c["nvalid"] else []) + (_field("formantFreqLpc", nF) if c["freqs"] else []) +
            (_field("formantBandwidthLpc", nF) if c["bws"] else []))


def diff_codes(c):
    """harmonicDifferences as (h1formant, h1idx, h2formant, h2idx) per difference (graph.cpp build_harmonics_op); formant
    differences are dropped without a formant level"""
    out = []
    for d in c["diffs"]:
        parts = []
        for t in d.split("-"):
            k = int(t[1:])
            parts += [-1, k] if t[0] == "H" else ([-1, 0] if k == 0 else [k, -1])
        out.append(tuple(parts))
    if not c["hfmt"] and any(p[0] > 0 or p[2] > 0 for p in out):
        return []
    return out


def harmonics_config(c):
    """(nHarm, diffs, (faStart, faEnd), hnr) after the graph's rules: nHarmonics raised to the highest named harmonic + 1;
    formant amplitudes only with a formant level, end = -1 -> nFmt, end < start -> none"""
    d = diff_codes(c)
    n_harm = max([c["nHarm"]] + [p[1] + 1 for p in d] + [p[3] + 1 for p in d])
    nF = n_formants(c) if c["hfmt"] else 0
    fa = (1, 0)
    if c["hfmt"]:
        end = nF if c["fa"][1] == -1 else min(c["fa"][1], nF)
        fa = (c["fa"][0], end) if end >= c["fa"][0] else (1, 0)
    return n_harm, d, fa, bool(c["hnr"])


def harmonics_names(c):
    _, d, fa, hnr = harmonics_config(c)
    names = ["HarmonicsToNoiseRatioACFLogdB"] if hnr else []
    names += ["HarmonicDifferenceLogRel" + x for x in c["diffs"]][:len(d)]
    return names + (_field("FormantAmplitudeByMaxHarmonicLogRelF0", fa[1] - fa[0] + 1, fa[0]) if fa[1] >= fa[0] else [])


# ---------------------------------------------------------------- signals
def _glide(n, sr, lo, hi, seed):
    """F0 glide from lo to hi and back, 40 harmonics, plus a little noise"""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / sr
    dur = max(n / sr, 1e-3)
    f0 = lo * (hi / lo) ** (1.0 - np.abs(2.0 * t / dur - 1.0))
    phi = 2 * np.pi * np.cumsum(f0) / sr
    x = np.zeros(n)
    for k in range(1, 41):
        x += np.where(k * f0 < sr / 2, np.sin(k * phi), 0.0) / (1.0 + 0.1 * k)
    x = 0.3 * x / max(np.abs(x).max(), 1e-9) + 0.005 * rng.standard_normal(n)
    return np.round(np.clip(x, -1, 1) * 32767).astype(np.int16)


VOWEL_FORMANTS = ((500.0, 80.0), (1500.0, 90.0), (2500.0, 120.0), (3500.0, 160.0))


def vowel(n, sr, seed, f0=125.0):
    """a pulse train at f0 (slight jitter) through a known all-pole filter: formants well apart, bandwidths >= 80 Hz"""
    from scipy.signal import lfilter
    rng = np.random.default_rng(seed)
    e = np.zeros(n)
    t = 0.0
    while t < n:
        e[int(t)] = 1.0
        t += sr / f0 * (1.0 + 0.01 * rng.standard_normal())
    a = np.array([1.0])
    for f, b in VOWEL_FORMANTS:
        if f < 0.45 * sr:
            r = np.exp(-np.pi * b / sr)
            a = np.convolve(a, [1.0, -2.0 * r * np.cos(2 * np.pi * f / sr), r * r])
    x = lfilter([1.0], a, e) + 1e-4 * rng.standard_normal(n)
    x = 0.5 * x / max(np.abs(x).max(), 1e-9)
    return np.round(x * 32767).astype(np.int16)


def signal(kind, n, c, seed):
    sr = int(c["sr"])
    rng = np.random.default_rng(seed)
    if kind == "voiced":
        x = voiced_pcm(n, sr, seed=seed)
    elif kind == "mixed":
        x = mixed_pcm(n, sr, seed=seed)
    elif kind == "silence":
        x = np.zeros(n, np.int16)
    elif kind == "noise":
        x = np.clip(np.round(rng.normal(0, 4000, n)), -32768, 32767).astype(np.int16)
    elif kind == "square":
        t = np.arange(n)
        x = np.where((t * 2 * 110 // sr) % 2 == 0, 32767, -32768).astype(np.int16)
    elif kind == "dc":
        x = (voiced_pcm(n, sr, seed=seed).astype(np.int64) // 4 + 12000).astype(np.int16)
    elif kind == "burst":
        x = np.zeros(n, np.int16)
        a, b = n // 3, 2 * n // 3
        x[a:b] = voiced_pcm(b - a, sr, seed=seed)
    elif kind == "glide":
        x = _glide(n, sr, 60.0, 600.0, seed)
    elif kind == "vowel":
        x = vowel(n, sr, seed)
    else:
        raise ValueError(kind)
    if c["n_chan"] == 2:
        if kind == "mixed":
            x = stereo_mixed_pcm(n, sr, seed=seed)
        else:
            x = np.stack([x, (x.astype(np.int64) * 4 // 5).astype(np.int16)], axis=1).reshape(-1)
    if c["f32"]:
        return (x.astype(np.float32) / np.float32(32767.0)).astype(np.float32)      # the float wave level as is (mono)
    return x


KINDS = ("voiced", "mixed", "silence", "noise", "burst", "dc", "square", "glide", "vowel")


def frame_counts(c):
    """formant-level frame counts of the ragged batch: the partial passes of formant_kernel (8 frames per transform batch, 16
    per per-frame phase) and of a tile (F = tile_width)"""
    F = tile_width(c)
    return sorted({1, 7, 8, 9, 15, 16, 17, F - 1, F, F + 1, 2 * F + 3})


def utterances(c, long_seconds=10.0):
    """the ragged batch of a case: empty; shorter than one 20 ms frame; between the 20 and 60 ms frame sizes (formant rows, no
    pitch or magnitude rows); T = frame_counts(c); every signal kind at about 3F frames; one long mixed utterance"""
    sr = int(c["sr"])
    N, S, _ = geometry(c)
    NH = geometry(c, hz=True)[0]
    F = tile_width(c)
    items = [("mixed", 0), ("voiced", N - 1), ("vowel", (N + NH) // 2)]
    for i, T in enumerate(frame_counts(c)):
        items.append((("voiced", "mixed", "vowel", "glide")[i % 4], N + (T - 1) * S + (i * 13) % S))
    for k in KINDS:
        items.append((k, N + (3 * F + 2) * S))
    items.append(("mixed", int(long_seconds * sr)))
    return [signal(k, n, c, seed=i) for i, (k, n) in enumerate(items)]


@functools.lru_cache(maxsize=None)
def _batch(name):
    c = BY_NAME[name]
    utts = utterances(c)
    if c["f32"]:
        off = np.concatenate([[0], np.cumsum([len(x) for x in utts])]).astype(np.int64)
        pcm = np.concatenate(utts + [np.zeros(8, np.float32)]).astype(np.float32)
        return utts, pcm, off
    pcm, off = pack_utterances(utts, n_chan=c["n_chan"])
    return utts, pcm, off


def batch(c):
    """(utterances, pcm, utt_offsets), built once per case: callers do not modify them"""
    return _batch(c["name"])


def n_samples(c, x):
    """sample frames of one utterance (float PCM is mono)"""
    return len(x) if c["f32"] else len(x) // c["n_chan"]
