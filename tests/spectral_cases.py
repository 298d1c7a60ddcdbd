"""Case table of the standalone ops that read the magnitude level or the framed signal: spectral_kernel (cSpectral, csrc/ops.cu),
acf_pitch_kernel<N,F,NT> + pitch_smooth_kernel (cAcf x2 -> cPitchACF, csrc/kernels.cu), and energy_kernel / mzcr_kernel /
intensity_kernel (cEnergy, cMZcr, cIntensity, csrc/ops.cu): test infrastructure shared by test_spectral_sweep_cpu.py and
test_spectral_sweep_gpu.py.  The anchor is the ComParE_2016 cSpectral on 25 ms Hamming frames at 16 kHz; every other case changes
one axis from there, a few combine extremes.  One dict per case; the plan's component list and the oracle's configuration structs
are both built from it.  Times are in seconds."""
import functools

import numpy as np

from opensmile_b200 import comp, components_frontend, pack_utterances
from opensmile_b200.synth import mixed_pcm, stereo_mixed_pcm, voiced_pcm
from oracle import oracle

# cSpectral's descriptors in output order (lldcore/spectral.cpp:378-584), bands / slopes / roll-off aside
DESC = ("alphaRatio", "hammarbergIndex", "flux", "centroid", "maxPos", "minPos", "entropy", "standardDeviation", "variance",
        "skewness", "kurtosis", "slope", "sharpness", "harmonicity", "flatness")
PITCH_OUT = ("voiceProb", "HNR", "HNRdB", "linHNR", "voiceQual", "F0", "F0raw", "F0env")

ANCHOR = dict(
    op="spectral", sr=16000, n_chan=1, frame=0.025, step=0.010, win="ham", zps=1, center=0,
    # cSpectral (ComParE_2016_core.lld.conf.inc:283-302); desc = the descriptors switched on
    sq=1, log=0, norm=0, buggy=0, oldslope=1, bands=((250, 650), (1000, 4000)), slopes=(), rolloff=(0.25, 0.5, 0.75, 0.9),
    frange=(0, 0), desc=("flux", "centroid", "entropy", "variance", "skewness", "kurtosis", "slope", "harmonicity", "sharpness"),
    # cAcf (ACF), cAcf (cepstrum), cPitchACF
    acf_pow=1, cep_pow=0, norm_out=1, abs_cep=0, old_compat=0, max_pitch=500.0, cutoff=0.55, pout=PITCH_OUT,
    # cEnergy (htkcompatible, rms, energy2, log, escaleLog, escaleRms, escaleSquare, ebiasLog, ebiasRms, ebiasSquare)
    energy=(0, 1, 0, 1, 1.0, 1.0, 1.0, 0.0, 0.0, 0.0),
    # cMZcr (zcr, mcr, amax, maxmin, dc), cIntensity (intensity, loudness); windowed: the time op reads the windower level
    mzcr=(1, 1, 1, 1, 0), intensity=(1, 0), windowed=0,
)


def case(name, **kw):
    bad = set(kw) - set(ANCHOR)
    assert not bad, bad
    c = dict(ANCHOR, **kw)
    c["name"] = name
    return c


ALL_DESC = dict(desc=DESC, slopes=((0, 500), (500, 1500)))
PITCH = dict(op="pitch", win="gau", zps=0, frame=0.050)

CASES = [
    case("anchor_compare16"),
    # ---- geometry: FFT 512 / 1024 / 2048 / 4096, zero-padded and exact frames, hops, stereo (no centred frames: a device plan
    # refuses a magnitude level on a centred cFramer level) ----
    case("g8k_50ms", sr=8000, frame=0.050),
    case("g8k_64ms_exact", sr=8000, frame=0.064, step=0.005),
    case("g16k_32ms_exact", frame=0.032),
    case("g16k_hop1", step=1 / 16000),
    case("g16k_hop80", step=0.005),
    case("g16k_hop_beyond_frame", step=0.040),
    case("g16k_64ms_exact", frame=0.064),
    case("g22k05_25ms", sr=22050),
    case("g44k1_25ms", sr=44100),
    case("g44k1_stereo", sr=44100, n_chan=2),
    case("g48k_stereo_narrow", sr=48000, n_chan=2, step=0.010),
    case("g16k_128ms_exact", frame=0.128),
    case("g44k1_60ms", sr=44100, frame=0.060),
    case("g96k_25ms", sr=96000),
    case("g96k_hop8", sr=96000, frame=2056 / 96000, step=8 / 96000),
    case("g16k_256ms_exact", frame=0.256, step=0.020),
    # ---- cSpectral options ----
    case("s_magnitude_input", sq=0),
    case("s_log", log=1, **ALL_DESC),
    case("s_log_magnitude_input", log=1, sq=0, **ALL_DESC),
    case("s_norm_bands", norm=1, **ALL_DESC),
    case("s_log_norm", log=1, norm=1, **ALL_DESC),
    case("s_buggy_rolloff_16", buggy=1, rolloff=tuple(np.round(np.linspace(0.05, 0.99, 16), 3))),
    case("s_new_slope_scale", oldslope=0, **ALL_DESC),
    # 31.25 Hz bins; band edges are whole Hz (spectral.cpp:778)
    case("s_edges_on_and_between_bins", bands=((0, 31), (125, 250), (100, 110), (3990, 8000), (7000, 9000), (8000, 20000)),
         slopes=((0, 125), (40, 300), (7990, 12000))),
    case("s_range_narrowest", frange=(1000, 1150), **ALL_DESC),
    case("s_range_narrowest_log", frange=(1000, 1150), log=1, **ALL_DESC),
    case("s_range_0_5000", frange=(0, 5000), **ALL_DESC),
    case("s_all_44k1_log", sr=44100, log=1, norm=1, **ALL_DESC),
    case("s_all_4096_log", sr=96000, log=1, **ALL_DESC),
    case("s_all_4096_log_exact", frame=0.256, step=0.020, log=1, norm=1, **ALL_DESC),
    case("s_all_2048_log_stereo", sr=48000, n_chan=2, log=1, **ALL_DESC),
    case("s_all_1024_log", frame=0.050, log=1, **ALL_DESC),
    case("s_gemaps_logspectral", log=1, norm=1, oldslope=0, bands=(), rolloff=(), slopes=((0, 500), (500, 1500)), frange=(0, 5000),
         desc=("alphaRatio", "hammarbergIndex")),
] + [case("d_%s" % d, bands=(), rolloff=(), desc=(d,)) for d in DESC] + [
    case("d_log_%s" % d, bands=(), rolloff=(), log=1, desc=(d,)) for d in DESC if d != "flux"] + [
    case("d_bands_only", rolloff=(), desc=()),
    case("d_slopes_only", bands=(), rolloff=(), slopes=((0, 500), (500, 1500), (1500, 4000)), desc=()),
    case("d_rolloff_only", bands=(), desc=()),
    # ---- cAcf / cPitchACF ----
    case("p_anchor", **PITCH),
    case("p_25ms", **dict(PITCH, frame=0.025)),
    case("p_1024", **dict(PITCH, frame=0.060)),
    case("p_2048", **dict(PITCH, sr=44100, frame=0.040)),
    case("p_2048_stereo", **dict(PITCH, sr=48000, n_chan=2, frame=0.025)),
    case("p_2048_exact", **dict(PITCH, frame=0.128, step=0.020)),
    case("p_8k", **dict(PITCH, sr=8000, frame=0.064)),
    case("p_hop1", **dict(PITCH, step=1 / 16000)),
    case("p_acf_magnitude_cep_power", **dict(PITCH, acf_pow=0, cep_pow=1)),
    case("p_no_norm", **dict(PITCH, norm_out=0)),
    case("p_abs_cepstrum", **dict(PITCH, abs_cep=1)),
    case("p_old_compat_cepstrum", **dict(PITCH, old_compat=1, norm_out=0, cep_pow=1)),
    case("p_max_pitch_0", **dict(PITCH, max_pitch=0.0)),
    case("p_max_pitch_2000", **dict(PITCH, max_pitch=2000.0)),
    # FFT 1024 at 16 kHz: n = 512 lags; preskip = 16000 / maxPitch just below n, at n, and inside (n, 2n)
    case("p_preskip_below_n", **dict(PITCH, frame=0.060, max_pitch=31.3)),
    case("p_preskip_at_n", **dict(PITCH, frame=0.060, max_pitch=31.24)),
    case("p_preskip_between_n_2n", **dict(PITCH, frame=0.060, max_pitch=20.0)),
    case("p_preskip_between_n_2n_512", **dict(PITCH, frame=0.025, max_pitch=45.0, abs_cep=1)),
    case("p_cutoff_0", **dict(PITCH, cutoff=0.0)),
    case("p_cutoff_1", **dict(PITCH, cutoff=1.0)),
    case("p_cutoff_above_1", **dict(PITCH, cutoff=1.7)),
    case("p_cutoff_below_0", **dict(PITCH, cutoff=-0.3)),
    case("p_f0_only", **dict(PITCH, pout=("F0",))),
    case("p_hnr_outputs", **dict(PITCH, pout=("HNR", "HNRdB", "linHNR"))),
    case("p_f0raw_f0env", **dict(PITCH, pout=("voiceQual", "F0raw", "F0env"))),
    case("p_2048_old_compat_hop80", **dict(PITCH, sr=44100, frame=0.040, step=0.005, old_compat=1, norm_out=0)),
    # ---- time ops ----
    case("e_default", op="energy"),
    case("e_htk", op="energy", energy=(1, 1, 1, 0, 1.0, 1.0, 1.0, 0.0, 0.0, 0.0)),
    case("e_all_scaled", op="energy", energy=(0, 1, 1, 1, 0.5, 2.0, 3.0, -1.5, 0.25, 7.0)),
    case("e_windowed_stereo", op="energy", windowed=1, n_chan=2, sr=44100, energy=(0, 1, 1, 1, 1.0, 1.0, 1.0, 0.0, 0.0, 0.0)),
    case("e_hop1", op="energy", step=1 / 16000),
    case("z_framer", op="mzcr", mzcr=(1, 1, 1, 1, 1)),
    case("z_windowed", op="mzcr", windowed=1, mzcr=(1, 1, 1, 1, 1)),
    case("z_zcr_dc_only", op="mzcr", mzcr=(1, 0, 0, 0, 1), frame=0.060, step=0.005),
    case("z_mcr_only_8k", op="mzcr", mzcr=(0, 1, 0, 0, 0), sr=8000),
    case("z_amax_maxmin", op="mzcr", mzcr=(0, 0, 1, 1, 0), sr=48000, step=0.040),
    case("i_intensity", op="intensity"),
    case("i_both", op="intensity", intensity=(1, 1)),
    case("i_loudness_windowed", op="intensity", intensity=(0, 1), windowed=1),
]
BY_NAME = {c["name"]: c for c in CASES}
assert len(BY_NAME) == len(CASES)

# the values every axis must reach (test_table_reaches_every_axis_value)
AXES = dict(
    nfft={512, 1024, 2048, 4096}, sr={8000, 16000, 22050, 44100, 48000, 96000}, exact={0, 1}, n_chan={1, 2},
    hop={1, 80, 160, "beyond_frame"},
    sq={0, 1}, log={0, 1}, norm={0, 1}, buggy={0, 1}, oldslope={0, 1}, n_rolloff={0, 4, 16}, frange={"default", "narrowest", "0-5000"},
    edge={"on_bin", "between_bins", "zero", "above_nyquist"}, single_desc=set(DESC), all_desc={0, 1},
    acf_pow={0, 1}, cep_pow={0, 1}, norm_out={0, 1}, abs_cep={0, 1}, old_compat={0, 1},
    max_pitch={0.0, 500.0, 2000.0}, preskip={"<n", "=n", "(n,2n)"}, cutoff={0.0, 0.55, 1.0, "clamped"},
    pout=set(PITCH_OUT), pitch_nfft={512, 1024, 2048},
    energy={"htk", "rms", "log", "energy2", "scaled"}, mzcr={"zcr", "mcr", "amax", "maxmin", "dc"}, mzcr_level={0, 1},
    intensity={"intensity", "loudness"},
)


# ---------------------------------------------------------------- geometry
def frontend(c):
    return oracle.frontend(float(c["sr"]), c["frame"], c["step"], win=c["win"], zero_pad_symmetric=c["zps"])


def geometry(c):
    """(N, S, nfft) as the graph computes them"""
    N, S, nfft, _ = oracle.geometry(frontend(c), 0)
    return N, S, nfft


def centre(c):
    """samples before the frame's first sample that a centred frame reaches back (frameCenterSpecial = mid)"""
    return geometry(c)[0] // 2 if c["center"] == 2 else 0


def preskip(c):
    """the lags cPitchACF skips (lldcore/pitchACF.cpp:155-159) on the FFT level of the case"""
    fss = oracle.lib().osm_or_fft_frame_size_sec(oracle.C.byref(frontend(c)))
    nfft = geometry(c)[2]
    mp = max(c["max_pitch"], 0.0)
    return 0 if mp <= 0.0 else int(1.0 / (mp * (float(np.float32(fss)) / nfft)))


def axis_values(c):
    N, S, nfft = geometry(c)
    v = dict(sr=c["sr"], n_chan=c["n_chan"], nfft=nfft, exact=int(N == nfft))
    v["hop"] = "beyond_frame" if S > N else S
    if c["op"] == "spectral":
        v.update(sq=c["sq"], log=c["log"], norm=c["norm"], buggy=c["buggy"], oldslope=c["oldslope"], n_rolloff=len(c["rolloff"]))
        v["frange"] = ("default" if c["frange"] == (0, 0) else
                       "0-5000" if c["frange"] == (0, 5000) else "narrowest" if spectral_range(c)[1] - spectral_range(c)[0] == 4 else "other")
        v["all_desc"] = int(set(c["desc"]) == set(DESC))
        if len(c["desc"]) == 1:
            v["single_desc"] = c["desc"][0]
        binhz = float(c["sr"]) / nfft if N == nfft else 1.0 / (c["frame"] * nfft / N)
        for lo, hi in tuple(c["bands"]) + tuple(c["slopes"]):
            for f in (lo, hi):
                if f == 0:
                    v["edge"] = "zero"
                elif f > c["sr"] / 2:
                    v["edge_hi"] = "above_nyquist"
                elif abs(f / binhz - round(f / binhz)) < 1e-9:
                    v["edge_on"] = "on_bin"
                else:
                    v["edge_between"] = "between_bins"
    elif c["op"] == "pitch":
        n = nfft // 2
        ps = preskip(c)
        v.update(acf_pow=c["acf_pow"], cep_pow=c["cep_pow"], norm_out=c["norm_out"], abs_cep=c["abs_cep"], old_compat=c["old_compat"],
                 max_pitch=c["max_pitch"], pitch_nfft=nfft)
        v["preskip"] = "<n" if ps < n else ("=n" if ps == n else "(n,2n)")
        v["cutoff"] = c["cutoff"] if 0.0 <= c["cutoff"] <= 1.0 else "clamped"
    return v


def axis_sets(c):
    """axis -> set of values the case reaches (multi-valued axes: pitch outputs, energy / mzcr / intensity outputs, edges)"""
    v = axis_values(c)
    s = {k: {x} for k, x in v.items() if not k.startswith("edge")}
    s["edge"] = {x for k, x in v.items() if k.startswith("edge")}
    if c["op"] == "pitch":
        s["pout"] = set(c["pout"])
    if c["op"] == "energy":
        htk, rms, e2, lg = c["energy"][:4]
        s["energy"] = ({"htk"} if htk else set()) | ({"rms"} if rms and not htk else set()) | ({"energy2"} if e2 else set()) | \
                      ({"log"} if lg or htk else set()) | ({"scaled"} if c["energy"][4:] != (1.0, 1.0, 1.0, 0.0, 0.0, 0.0) else set())
    if c["op"] == "mzcr":
        s["mzcr"] = {k for k, on in zip(("zcr", "mcr", "amax", "maxmin", "dc"), c["mzcr"]) if on}
        s["mzcr_level"] = {c["windowed"]}
    if c["op"] == "intensity":
        s["intensity"] = {k for k, on in zip(("intensity", "loudness"), c["intensity"]) if on}
    return s


def spectral_range(c):
    """(loBin, hiBin) of cSpectral's freqRange (spectral.cpp:625-647)"""
    N, S, nfft = geometry(c)
    fss = oracle.lib().osm_or_fft_frame_size_sec(oracle.C.byref(frontend(c)))
    frq = np.arange(nfft // 2 + 1) * (1.0 / fss)
    lo, hi = int(c["frange"][0]), int(c["frange"][1])
    if lo == hi == 0:
        return 1, nfft // 2
    lb = max(int(np.nonzero(lo >= frq)[0].max()) if (lo >= frq).any() else -1, 0)
    hb = int(np.nonzero(hi > frq)[0].max()) if (hi > frq).any() else nfft // 2
    return lb, hb


# ---------------------------------------------------------------- plan side
def level(c):
    return dict(spectral="spec", pitch="pitch", energy="energy", mzcr="mzcr", intensity="intensity")[c["op"]]


def components(c):
    """wave -> frame -> win -> fft -> mag -> the op of the case (time ops read `frame`, or `win` when windowed)"""
    cs = components_frontend(float(c["sr"]), c["frame"], c["step"], win=c["win"], n_channels=c["n_chan"],
                             zero_pad_symmetric=c["zps"], with_fft=c["op"] in ("spectral", "pitch"))
    if c["center"]:
        cs[1].u.framer.frameCenterSpecial = c["center"]
    if c["op"] == "spectral":
        kw = {d: int(d in c["desc"]) for d in DESC}
        cs.append(comp("cSpectral", "spec", "mag", "spec", bands=list(c["bands"]), slopes=list(c["slopes"]),
                       rollOff=list(c["rolloff"]), freqRange=tuple(c["frange"]), squareInput=c["sq"], useLogSpectrum=c["log"],
                       normBandEnergies=c["norm"], buggyRollOff=c["buggy"], oldSlopeScale=c["oldslope"], **kw))
    elif c["op"] == "pitch":
        cs.append(comp("cAcf", "acf", "mag", "acf", usePower=c["acf_pow"], acfCepsNormOutput=c["norm_out"]))
        cs.append(comp("cAcf", "cep", "mag", "cepstrum", cepstrum=1, usePower=c["cep_pow"], acfCepsNormOutput=c["norm_out"],
                       absCepstrum=c["abs_cep"], oldCompatCepstrum=c["old_compat"]))
        cs.append(comp("cPitchACF", "pitch", "acf;cepstrum", "pitch", maxPitch=c["max_pitch"], voicingCutoff=c["cutoff"],
                       **{k: int(k in c["pout"]) for k in PITCH_OUT}))
    else:
        src = "win" if c["windowed"] else "frame"
        if c["op"] == "energy":
            e = c["energy"]
            cs.append(comp("cEnergy", "energy", src, "energy", htkcompatible=e[0], rms=e[1], energy2=e[2], log=e[3], escaleLog=e[4],
                           escaleRms=e[5], escaleSquare=e[6], ebiasLog=e[7], ebiasRms=e[8], ebiasSquare=e[9]))
        elif c["op"] == "mzcr":
            cs.append(comp("cMZcr", "mzcr", src, "mzcr", **dict(zip(("zcr", "mcr", "amax", "maxmin", "dc"), c["mzcr"]))))
        else:
            cs.append(comp("cIntensity", "intensity", src, "intensity", intensity=c["intensity"][0], loudness=c["intensity"][1]))
    return cs


def oracle_cfg(c):
    """the oracle's configuration struct of the case's op"""
    if c["op"] == "spectral":
        kw = {d: int(d in c["desc"]) for d in DESC}
        return oracle.spectral_cfg(bands=c["bands"], slopes=c["slopes"], rolloff=c["rolloff"], squareInput=c["sq"],
                                   useLogSpectrum=c["log"], normBandEnergies=c["norm"], buggyRollOff=c["buggy"],
                                   oldSlopeScale=c["oldslope"], freqRangeLo=c["frange"][0], freqRangeHi=c["frange"][1], **kw)
    if c["op"] == "pitch":
        return oracle.pitchacf_cfg(acfUsePower=c["acf_pow"], cepUsePower=c["cep_pow"], absCepstrum=c["abs_cep"],
                                   acfCepsNormOutput=c["norm_out"], maxPitch=c["max_pitch"], voicingCutoff=c["cutoff"],
                                   oldCompatCepstrum=c["old_compat"], **{k: int(k in c["pout"]) for k in PITCH_OUT})
    if c["op"] == "energy":
        return oracle.Energy(*c["energy"])
    if c["op"] == "mzcr":
        return oracle.MZcr(*c["mzcr"])
    return oracle.Intensity(*c["intensity"])


def oracle_rows(c, x):
    """the oracle's rows of one utterance from PCM (uncentred cases)"""
    fe, cfg = frontend(c), oracle_cfg(c)
    if c["op"] == "spectral":
        return oracle.spectral(x, fe, cfg, n_chan=c["n_chan"])
    if c["op"] == "pitch":
        return oracle.pitchacf(x, fe, cfg, n_chan=c["n_chan"])
    fn = dict(energy=oracle.energy, mzcr=oracle.mzcr, intensity=oracle.intensity)[c["op"]]
    return fn(x, fe, cfg, windowed=c["windowed"], n_chan=c["n_chan"])


def oracle_from_mag(c, mag):
    """the oracle's rows of one utterance on given magnitudes [T, nfft/2+1]"""
    if c["op"] == "spectral":
        return oracle.spectral_from_mag(mag, frontend(c), oracle_cfg(c))
    return oracle.pitchacf_from_mag(mag, frontend(c), oracle_cfg(c))


# ---------------------------------------------------------------- signals
KINDS = ("voiced", "mixed", "silence", "square", "impulses")


def signal(kind, n, c, seed):
    sr = int(c["sr"])
    if kind == "voiced":
        x = voiced_pcm(n, sr, seed=seed)
    elif kind == "mixed":
        x = mixed_pcm(n, sr, seed=seed)
    elif kind == "silence":
        x = np.zeros(n, np.int16)
    elif kind == "square":                                       # full scale, clipped
        x = np.where((np.arange(n) * 2 * 150 // sr) % 2 == 0, 32767, -32768).astype(np.int16)
    elif kind == "impulses":                                     # one impulse in every frame: a flat magnitude spectrum
        x = np.zeros(n, np.int16)
        x[3::geometry(c)[0]] = 20000
    else:
        raise ValueError(kind)
    if c["n_chan"] == 2:
        if kind == "mixed":
            return stereo_mixed_pcm(n, sr, seed=seed)
        return np.stack([x, (x.astype(np.int64) * 3 // 4).astype(np.int16)], axis=1).reshape(-1)
    return x


def tile_guess(c):
    """frames per tile of the magnitude level at full width (lld_tile_frames); narrow tiles are half of it"""
    nfft = geometry(c)[2]
    return 8 if nfft == 4096 else (16 if nfft == 2048 else 32)


def frame_counts(c):
    F = tile_guess(c)
    return sorted({1, 2, F - 1, F, F + 1, 2 * F + 3})


def utterances(c):
    """the ragged batch of a case: empty, shorter than one frame, T = frame_counts(c), every signal kind at about 3F frames"""
    N, S, _ = geometry(c)
    F, ctr = tile_guess(c), centre(c)
    items = [("mixed", 0), ("voiced", max(N - ctr - 1, 0))]
    for i, T in enumerate(frame_counts(c)):
        items.append((("voiced", "mixed")[i % 2], N - ctr + (T - 1) * S + (i * 7) % S))
    for k in KINDS:
        items.append((k, N - ctr + (3 * F + 2) * S))
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


def n_samples(c, x):
    return len(x) // c["n_chan"]

