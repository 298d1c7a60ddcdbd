"""Case table of the SHS pitch chain (shs_kernel, viterbi_kernel, jitter_kernel, seq_post_kernel in csrc/pitch.cu): test
infrastructure shared by test_pitch_sweep_cpu.py and test_pitch_sweep_gpu.py.  The anchor is the ComParE_2016 chain
(ComParE_2016_core.lld.conf.inc); every other case changes one axis from there, a few combine extremes.  One dict per case;
the plan's component list and the oracle's configuration structs are both built from it.  Times are in seconds."""
import functools

import numpy as np

from opensmile_b200 import comp, components_frontend, pack_utterances
from opensmile_b200.synth import mixed_pcm, stereo_mixed_pcm, voiced_pcm
from oracle import oracle

ANCHOR = dict(
    sr=16000, n_chan=1, frame=0.060, step=0.010,
    # cSpecScale
    minF=25.0, maxF=-1.0, nPts=0, smooth=1, enhance=1, audw=1,
    # cPitchShs
    maxPitch=620.0, minPitch=52.0, nCand=6, scores=1, voicing=1, F0C1=0, voicingC1=0, F0raw=1, voicingClip=1, cutoff=0.70,
    octave=0, nHarm=15, compression=0.85, greedy=1, lfCut=0.0,
    # cPitchSmootherViterbi: outputs F0final, F0finalLog, F0finalEnv, F0finalEnvLog, voicingFinalClipped, voicingFinalUnclipped;
    # weights wLocal, wTvv, wTvvd, wTvuv, wThr, wRange, wTuu
    bufLen=30, vout=(1, 0, 0, 0, 0, 1), w=(2.0, 10.0, 5.0, 10.0, 4.0, 1.0, 0.0),
    # cValbasedSelector on the rms energy of the frame in front of cPitchJitter
    sel=1,
    # cPitchJitter
    srr=0.25, jout=("jitterLocal", "jitterDDP", "shimmerLocal", "logHNR"), floor=-100.0, rms=0, mnp=2, minCC=0.5, p2p=0, broken=0,
)
JIT_OUT = ("jitterLocal", "jitterDDP", "jitterLocalEnv", "jitterDDPEnv", "shimmerLocal", "shimmerLocalDB", "shimmerLocalEnv",
           "shimmerLocalDBEnv", "harmonicERMS", "noiseERMS", "linearHNR", "logHNR", "refinedF0", "sourceQualityMean",
           "sourceQualityRange")
JIT_NAMES = dict(jitterLocalEnv="jitterLocEnv", jitterDDPEnv="jitterDEnv", shimmerLocalEnv="shimmerLocEnv",
                 shimmerLocalDBEnv="shimmerLocDBEnv", refinedF0="F0final")
VIT_NAMES = ("F0final", "F0finalLog", "F0finEnv", "F0finEnvLog", "voicingFinalClipped", "voicingFinalUnclipped")


def case(name, **kw):
    bad = set(kw) - set(ANCHOR)
    assert not bad, bad
    c = dict(ANCHOR, **kw)
    c["name"] = name
    return c


CASES = [
    case("anchor_compare16"),
    # ---- geometry: nMag 257 (FFT 512), 513, 1025 and 2049 (FFT 4096) ----
    case("g8k_60ms", sr=8000),
    case("g8k_40ms", sr=8000, frame=0.040, minPitch=80.0),
    case("g16k_40ms_5ms", frame=0.040, step=0.005),
    case("g16k_50ms_20ms", frame=0.050, step=0.020),
    case("g16k_60ms_step_7ms", step=0.007),
    case("g22k05_60ms", sr=22050),
    case("g32k_50ms", sr=32000, frame=0.050),
    case("g44k1_60ms", sr=44100),
    case("g44k1_25ms_10ms", sr=44100, frame=0.025),
    case("g48k_60ms", sr=48000),
    case("g48k_40ms_5ms", sr=48000, frame=0.040, step=0.005),
    case("g16k_stereo", n_chan=2),
    case("g44k1_stereo", sr=44100, n_chan=2),
    # ---- cSpecScale ----
    case("s_npts_100", nPts=100),
    case("s_npts_400", nPts=400, minF=30.0, maxF=4000.0),
    case("s_48k_npts_2049", sr=48000, nPts=2049),
    case("s_48k_npts_2050", sr=48000, nPts=2050),
    case("s_48k_npts_3000", sr=48000, nPts=3000),
    case("s_44k1_npts_4096", sr=44100, nPts=4096),
    case("s_48k_npts_4096_nongreedy", sr=48000, nPts=4096, greedy=0),
    case("s_minF_50_maxF_5000", minF=50.0, maxF=5000.0),
    case("s_plain_spectrum", smooth=0, enhance=0, audw=0),
    case("s_smooth_only", enhance=0, audw=0),
    case("s_enhance_only", smooth=0, audw=0),
    case("s_audw_only", smooth=0, enhance=0),
    case("s_lfcut_100", lfCut=100.0),
    # ---- cPitchShs ----
    case("p_1_candidate", nCand=1),
    case("p_3_candidates_nongreedy", nCand=3, greedy=0),
    case("p_8_candidates", nCand=8),
    case("p_8_candidates_nongreedy_octave", nCand=8, greedy=0, octave=1),
    case("p_octave_correction", octave=1),
    case("p_2_harmonics", nHarm=2),
    case("p_10_harmonics_comp_0_6", nHarm=10, compression=0.6),
    case("p_32_harmonics", nHarm=32),
    case("p_cutoff_0_5", cutoff=0.5),
    case("p_wide_30_1000", minPitch=30.0, maxPitch=1000.0),
    case("p_narrow_100_250", minPitch=100.0, maxPitch=250.0),
    case("p_all_outputs", F0C1=1, voicingC1=1),
    case("p_no_scores_no_raw", scores=0, F0raw=0, voicingClip=0),
    case("p_no_voicing_shs_only", voicing=0, F0C1=1),          # the cPitchShs level alone: cPitchSmootherViterbi needs voicing
    # ---- cPitchSmootherViterbi ----
    case("v_buf_2", bufLen=2),
    case("v_buf_8_all_outputs", bufLen=8, vout=(1, 1, 1, 1, 1, 1)),
    case("v_buf_63", bufLen=63),
    case("v_buf_64_wtuu", bufLen=64, w=(1.5, 8.0, 3.0, 6.0, 3.0, 2.0, 0.5)),
    case("v_no_selector", sel=0),
    # ---- cPitchJitter ----
    case("j_srr_0_05", srr=0.05),
    case("j_srr_0_5_mnp_4", srr=0.5, mnp=4),
    case("j_mnp_1", mnp=1),
    case("j_all_outputs_rms", jout=JIT_OUT, rms=1, floor=-50.0),
    case("j_all_outputs_p2p_broken", jout=JIT_OUT, p2p=1, broken=1, minCC=0.3),
    # ---- short frames and a low minPitch: the jitter reader's window (two longest periods) exceeds the frame and, in the last
    # frames, the input ----
    case("j_25ms_min30", frame=0.025, minPitch=30.0, jout=JIT_OUT),
    case("j_25ms_5ms_min30", frame=0.025, step=0.005, minPitch=30.0, srr=0.5),
    case("j_48k_25ms_min30", sr=48000, frame=0.025, minPitch=30.0, jout=JIT_OUT),
    # ---- extremes combined ----
    case("x_48k_8cand_buf64_npts_3000", sr=48000, nPts=3000, nCand=8, bufLen=64, minPitch=30.0, maxPitch=1000.0),
    case("x_8k_1cand_buf2_2harm", sr=8000, nCand=1, bufLen=2, nHarm=2, octave=1, vout=(1, 1, 1, 1, 1, 1)),
]
BY_NAME = {c["name"]: c for c in CASES}
assert len(BY_NAME) == len(CASES)

# The cPitchShs level is held to 2e-6 of the column scale, and a peak decision may differ only on a 1e-6 tie of the oracle's
# sub-harmonic sum, except in these cases.  Kernel, oracle and reference compute the magnitude spectrum with three different
# float FFTs (about 2.5e-7 of the frame maximum apart, each pair alike); the parabolic refinement of flat SHS peaks amplifies
# that.  Measured on a 4 s mixed signal, the oracle itself is 3.2e-6 from the reference at 2049 bins (48 kHz: 2 of 395 rows
# with another candidate list) and the kernel is as far from the reference as the oracle is.  The sweep's glides, square
# waves and fine target axes (up to 4096 points) reach further: value <- bound, tie <- relative tie tolerance, free <- rows
# whose decision differs without a tie the restated sum resolves (measured on the H100).
SHS_WIDE = {n: dict(value=2e-4, tie=1e-4, free=0) for n in (
    "g44k1_60ms", "g44k1_25ms_10ms", "g48k_60ms", "g48k_40ms_5ms", "g44k1_stereo", "s_48k_npts_2049", "s_48k_npts_2050",
    "s_48k_npts_3000", "s_44k1_npts_4096", "s_48k_npts_4096_nongreedy", "j_48k_25ms_min30", "x_48k_8cand_buf64_npts_3000")}
# 257- and 513-bin cases with single rows on flat peaks (16 kHz, 5 ms steps; 25 ms frames with F0 down to 30 Hz)
SHS_WIDE.update({n: dict(value=1e-4, tie=1e-6, free=0) for n in ("g16k_40ms_5ms", "j_25ms_min30", "j_25ms_5ms_min30")})
# one row of 3374 picks a sixth in-range candidate where the oracle's sixth lies outside the pitch range
SHS_WIDE["g16k_60ms_step_7ms"] = dict(value=2e-6, tie=1e-6, free=1)
SHS_STRICT = dict(value=2e-6, tie=1e-6, free=0)

# the values every axis must reach (test_every_axis_value_of_the_table_ran)
AXES = dict(sr={8000, 16000, 22050, 32000, 44100, 48000}, frame={0.060, 0.050, 0.040, 0.025}, step={0.005, 0.010, 0.020, 0.007},
            nPts={0, 100, 400, 2049, 2050, 3000, 4096}, nCand={1, 3, 6, 8}, greedy={0, 1}, octave={0, 1}, nHarm={2, 10, 15, 32},
            bufLen={2, 8, 30, 63, 64}, voicing={0, 1}, sel={0, 1}, srr={0.05, 0.25, 0.5}, mnp={1, 2, 4}, n_chan={1, 2}, smooth={0, 1},
            enhance={0, 1}, audw={0, 1}, rms={0, 1}, p2p={0, 1}, broken={0, 1})


# ---------------------------------------------------------------- plan side
def components(c):
    """ComParE-style graph: wave -> frame -> Gaussian window -> FFT -> magnitude -> cSpecScale -> cPitchShs (level `shs`) ->
    cPitchSmootherViterbi (`vit`) [-> cValbasedSelector on the frame's rms energy] (`pitch`); cPitchJitter (`jit`) on the F0 of
    `pitch`; cContourSmoother (noZeroSma) over `pitch;jit` (`smo`) and its onlyInSegments delta (`smo_de`), concatenated (`lld`)"""
    cs = components_frontend(float(c["sr"]), c["frame"], c["step"], win="gau", sigma=0.4, n_channels=c["n_chan"])
    cs.append(comp("cSpecScale", "scale", "mag", "hps", scaleOctave=1, sourceLin=1, splineInterp=1, minF=c["minF"], maxF=c["maxF"],
                   nPointsTarget=c["nPts"], specSmooth=c["smooth"], specEnhance=c["enhance"], auditoryWeighting=c["audw"]))
    cs.append(comp("cPitchShs", "shs", "hps", "shs", maxPitch=c["maxPitch"], minPitch=c["minPitch"], nCandidates=c["nCand"],
                   scores=c["scores"], voicing=c["voicing"], F0C1=c["F0C1"], voicingC1=c["voicingC1"], F0raw=c["F0raw"],
                   voicingClip=c["voicingClip"], voicingCutoff=c["cutoff"], octaveCorrection=c["octave"], nHarmonics=c["nHarm"],
                   compressionFactor=c["compression"], greedyPeakAlgo=c["greedy"], lfCut=c["lfCut"]))
    vo, w = c["vout"], c["w"]
    cs.append(comp("cPitchSmootherViterbi", "vit", "shs", "vit", bufferLength=c["bufLen"], F0final=vo[0], F0finalLog=vo[1],
                   F0finalEnv=vo[2], F0finalEnvLog=vo[3], voicingFinalClipped=vo[4], voicingFinalUnclipped=vo[5], F0raw=0, voicingC1=0,
                   voicingClip=0, wLocal=w[0], wTvv=w[1], wTvvd=w[2], wTvuv=w[3], wThr=w[4], wRange=w[5], wTuu=w[6]))
    if c["sel"]:
        cs.append(comp("cEnergy", "energy", "win", "e", htkcompatible=0, rms=1, energy2=0, log=0, escaleLog=1.0, escaleRms=1.0,
                       escaleSquare=1.0, ebiasLog=0.0, ebiasRms=0.0, ebiasSquare=0.0))
        cs.append(comp("cValbasedSelector", "sel", "e;vit", "pitch", threshold=0.001, idx=0, invert=0, allowEqual=0, removeIdx=1,
                       zeroVec=1, adaptiveThreshold=0, outputVal=0.0))
    f0lvl = "pitch" if c["sel"] else "vit"
    jo = {k: int(k in c["jout"]) for k in JIT_OUT}
    cs.append(comp("cPitchJitter", "jit", "wave", "jit", F0reader_dmLevel=f0lvl, F0field="F0final", searchRangeRel=c["srr"],
                   lgHNRfloor=c["floor"], shimmerUseRmsAmplitude=c["rms"], minNumPeriods=c["mnp"], minCC=c["minCC"],
                   usePeakToPeakPeriodLength=c["p2p"], useBrokenJitterThresh=c["broken"], onlyVoiced=0, **jo))
    cs.append(comp("cContourSmoother", "smo", f0lvl + ";jit", "smo", smaWin=3, noZeroSma=1))
    cs.append(comp("cDeltaRegression", "smo_de", "smo", "smo_de", deltawin=2, onlyInSegments=1))
    cs.append(comp("cVectorConcat", "lldconcat", "smo;smo_de", "lld", processArrayFields=0))
    return cs


def f0_level(c):
    return "pitch" if c["sel"] else "vit"


# ---------------------------------------------------------------- oracle side
def oracle_cfg(c):
    """(frontend, SpecScale, PitchShs, Viterbi, Jitter) of the oracle"""
    fe = oracle.frontend(float(c["sr"]), c["frame"], c["step"], win="gau", sigma=0.4, zero_pad_symmetric=1)
    sc = oracle.SpecScale(c["minF"], c["maxF"], c["nPts"], c["smooth"], c["enhance"], c["audw"])
    ps = oracle.PitchShs(c["maxPitch"], c["minPitch"], c["nCand"], c["scores"], c["voicing"], c["F0C1"], c["voicingC1"], c["F0raw"],
                         c["voicingClip"], c["cutoff"], c["octave"], c["nHarm"], c["compression"], c["greedy"], c["lfCut"])
    vc = oracle.Viterbi(c["bufLen"], *c["vout"], *c["w"])
    jo = [int(k in c["jout"]) for k in JIT_OUT]
    jc = oracle.Jitter(c["srr"], *jo[:12], c["floor"], c["rms"], c["mnp"], c["minCC"], jo[12], jo[14], jo[13], c["p2p"], c["broken"], 0)
    return fe, sc, ps, vc, jc


def n_mag(c):
    fe = oracle_cfg(c)[0]
    return oracle.geometry(fe, 0)[2] // 2 + 1


def n_pts(c):
    return c["nPts"] if c["nPts"] > 0 else n_mag(c)


def shs_names(c):
    n = min(max(c["nCand"], 1), 20)

    def field(f):
        return [f] if n == 1 else ["%s[%d]" % (f, i) for i in range(n)]     # a one-element field has no index
    names = ["nCandidates"] + field("F0Cand")
    if c["voicing"]:
        names += field("candVoicing")
    if c["scores"]:
        names += field("candScores")
    return names + [k for k in ("F0C1", "voicingC1", "F0raw", "voicingClip") if c[k]]


def vit_names(c):
    return [n for n, on in zip(VIT_NAMES, c["vout"]) if on]


def jit_names(c):
    return [JIT_NAMES.get(k, k) for k in JIT_OUT if k in c["jout"]]


def frames(c, n_samples):
    fe = oracle_cfg(c)[0]
    return max(oracle.geometry(fe, n_samples)[3], 0)


# ---------------------------------------------------------------- signals
def _glide(n, sr, lo, hi, seed):
    """F0 glide from lo to hi and back, 40 harmonics (the upper ones far above maxPitch), plus a little noise"""
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
        x = _glide(n, sr, c["minPitch"], c["maxPitch"], seed)
    else:
        raise ValueError(kind)
    if c["n_chan"] == 2:
        if kind == "mixed":
            return stereo_mixed_pcm(n, sr, seed=seed)
        y = np.stack([x, (x.astype(np.int64) * 4 // 5).astype(np.int16)], axis=1)
        return y.reshape(-1)
    return x


KINDS = ("voiced", "mixed", "silence", "noise", "square", "dc", "burst", "glide")


def utterances(c, long_seconds=10.0):
    """the ragged batch of a case: empty and shorter than one frame; T = 1, 2, bufLen - 1, bufLen, bufLen + 1, 2 bufLen + 3, a
    spread of lengths for the end-of-input lag rule, every signal kind at 3 * bufLen + 7 frames, and one long glide / mixed
    utterance"""
    sr = int(c["sr"])
    N = int(round(c["frame"] * sr))
    S = int(round(c["step"] * sr))
    B = c["bufLen"]
    Ts = [1, 2, max(B - 1, 1), B, B + 1, 2 * B + 3] + [B + 5 + 7 * i for i in range(6)]
    items = [("mixed", 0), ("voiced", N - 1)]
    for i, T in enumerate(Ts):
        items.append((("voiced", "mixed", "glide")[i % 3], N + (T - 1) * S + (i * 13) % S))
    for k in KINDS:
        items.append((k, N + (3 * B + 6) * S))
    items.append(("glide", int(long_seconds * sr) // 2))
    items.append(("mixed", int(long_seconds * sr)))
    return [signal(k, n, c, seed=i) for i, (k, n) in enumerate(items)]


@functools.lru_cache(maxsize=None)
def _batch(name):
    c = BY_NAME[name]
    utts = utterances(c)
    pcm, off = pack_utterances(utts, n_chan=c["n_chan"])
    return utts, pcm, off


def batch(c):
    """(utterances, pcm, utt_offsets), built once per case: callers do not modify them"""
    return _batch(c["name"])
