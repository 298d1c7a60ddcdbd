"""ctypes binding of oracle/liboracle.so (the plain-C restatement, oracle/osm_oracle.c).

TEST INFRASTRUCTURE ONLY -- see oracle/osm_oracle.h for the parity-pinning statement.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

WIN = {"rect": 0, "han": 1, "ham": 2, "gau": 3, "sin": 4, "tri": 5, "bar": 6}


class Frontend(C.Structure):
    _fields_ = [("sample_rate", C.c_double), ("frame_size_sec", C.c_double),
                ("frame_step_sec", C.c_double), ("preemph_on", C.c_int),
                ("preemph_k", C.c_double), ("win_func", C.c_int), ("win_sigma", C.c_double),
                ("win_gain", C.c_double), ("win_offset", C.c_double),
                ("zero_pad_symmetric", C.c_int)]


class Melspec(C.Structure):
    _fields_ = [("n_bands", C.c_int), ("lofreq", C.c_double), ("hifreq", C.c_double),
                ("use_power", C.c_int), ("htkcompatible", C.c_int), ("spec_scale", C.c_int), ("scale_param", C.c_double)]


class Mfcc(C.Structure):
    _fields_ = [("first_mfcc", C.c_int), ("last_mfcc", C.c_int), ("cep_lifter", C.c_double),
                ("melfloor", C.c_double), ("htkcompatible", C.c_int)]


class Plp(C.Structure):
    _fields_ = [("lp_order", C.c_int), ("first_cc", C.c_int), ("last_cc", C.c_int),
                ("do_log", C.c_int), ("do_aud", C.c_int), ("do_inv_log", C.c_int),
                ("do_idft", C.c_int), ("do_lp", C.c_int), ("do_lp_to_ceps", C.c_int),
                ("rasta", C.c_int), ("new_rasta", C.c_int), ("rasta_upper", C.c_double),
                ("rasta_lower", C.c_double), ("cep_lifter", C.c_double),
                ("compression", C.c_double), ("melfloor", C.c_double),
                ("htkcompatible", C.c_int)]


MAX_LIST = 16


class Spectral(C.Structure):
    _fields_ = [("squareInput", C.c_int),
                ("nBands", C.c_int), ("bandLo", C.c_double * MAX_LIST), ("bandHi", C.c_double * MAX_LIST),
                ("nSlopes", C.c_int), ("slopeLo", C.c_double * MAX_LIST), ("slopeHi", C.c_double * MAX_LIST),
                ("nRollOff", C.c_int), ("rollOff", C.c_double * MAX_LIST),
                ("flux", C.c_int), ("centroid", C.c_int), ("maxPos", C.c_int), ("minPos", C.c_int),
                ("entropy", C.c_int), ("standardDeviation", C.c_int), ("variance", C.c_int),
                ("skewness", C.c_int), ("kurtosis", C.c_int), ("slope", C.c_int), ("alphaRatio", C.c_int),
                ("hammarbergIndex", C.c_int), ("sharpness", C.c_int), ("harmonicity", C.c_int),
                ("flatness", C.c_int), ("normBandEnergies", C.c_int), ("buggyRollOff", C.c_int),
                ("oldSlopeScale", C.c_int), ("useLogSpectrum", C.c_int),
                ("freqRangeLo", C.c_double), ("freqRangeHi", C.c_double), ("specFloor", C.c_double),
                ("logFlatness", C.c_int)]


class Energy(C.Structure):
    _fields_ = [("htkcompatible", C.c_int), ("rms", C.c_int), ("energy2", C.c_int), ("log", C.c_int),
                ("escaleLog", C.c_double), ("escaleRms", C.c_double), ("escaleSquare", C.c_double),
                ("ebiasLog", C.c_double), ("ebiasRms", C.c_double), ("ebiasSquare", C.c_double)]


class MZcr(C.Structure):
    _fields_ = [("zcr", C.c_int), ("mcr", C.c_int), ("amax", C.c_int), ("maxmin", C.c_int), ("dc", C.c_int)]


class PitchAcf(C.Structure):
    _fields_ = [("acfUsePower", C.c_int), ("cepUsePower", C.c_int), ("absCepstrum", C.c_int),
                ("acfCepsNormOutput", C.c_int), ("maxPitch", C.c_double),
                ("voiceProb", C.c_int), ("voiceQual", C.c_int), ("HNR", C.c_int), ("HNRdB", C.c_int),
                ("linHNR", C.c_int), ("F0", C.c_int), ("F0raw", C.c_int), ("F0env", C.c_int),
                ("voicingCutoff", C.c_double), ("oldCompatCepstrum", C.c_int)]


def pitchacf_cfg(**kw):
    """cAcf / cPitchACF defaults (SURVEY.md Appendix A) + overrides."""
    pc = PitchAcf(1, 0, 0, 1, 500.0, 1, 0, 0, 0, 0, 0, 0, 0, 0.55)
    for k, v in kw.items():
        assert hasattr(pc, k), k
        setattr(pc, k, v)
    return pc


def pitchacf(pcm, fe, cfg, n_chan=1, taps=False):
    pcm = np.ascontiguousarray(pcm, dtype=np.int16)
    nS = pcm.size // n_chan
    N, H, nfft, T = geometry(fe, nS)
    L = lib()
    L.osm_or_pitchacf.restype = C.c_long
    K = L.osm_or_pitchacf_num_out(C.byref(cfg))
    out = np.zeros((max(T, 0), K), np.float32)
    ta = np.zeros((max(T, 0), nfft // 2), np.float32) if taps else None
    tc = np.zeros((max(T, 0), nfft // 2), np.float32) if taps else None
    r = L.osm_or_pitchacf(C.byref(fe), C.byref(cfg), pcm.ctypes.data_as(C.POINTER(C.c_int16)), C.c_long(nS),
                          C.c_int(n_chan), _fp(out), _fp(ta), _fp(tc))
    assert r == max(T, 0)
    return (out, ta, tc) if taps else out


def pitchacf_from_mag(mag, fe, cfg, taps=False):
    """cAcf x2 -> cPitchACF on given magnitudes [T, nfft/2+1] of one utterance (fe gives the FFT size and frame length)"""
    mag = np.ascontiguousarray(mag, np.float32)
    T = mag.shape[0]
    L = lib()
    L.osm_or_pitchacf_from_mag.restype = C.c_long
    K = L.osm_or_pitchacf_num_out(C.byref(cfg))
    out = np.zeros((T, K), np.float32)
    n = mag.shape[1] - 1
    ta = np.zeros((T, n), np.float32) if taps else None
    tc = np.zeros((T, n), np.float32) if taps else None
    r = L.osm_or_pitchacf_from_mag(C.byref(fe), C.byref(cfg), _fp(mag), C.c_long(T), _fp(out), _fp(ta), _fp(tc))
    assert r == T, (r, T)
    return (out, ta, tc) if taps else out


def spectral_cfg(bands=(), slopes=(), rolloff=(), **kw):
    """cSpectral defaults (SURVEY.md Appendix A) + overrides."""
    sp = Spectral()
    sp.squareInput = 1; sp.flux = 1; sp.centroid = 1; sp.maxPos = 1; sp.minPos = 1
    sp.oldSlopeScale = 1; sp.specFloor = 1e-7
    sp.nBands = len(bands)
    for i, (a, b) in enumerate(bands):
        sp.bandLo[i], sp.bandHi[i] = a, b
    sp.nSlopes = len(slopes)
    for i, (a, b) in enumerate(slopes):
        sp.slopeLo[i], sp.slopeHi[i] = a, b
    sp.nRollOff = len(rolloff)
    for i, r in enumerate(rolloff):
        sp.rollOff[i] = r
    for k, v in kw.items():
        assert hasattr(sp, k), k
        setattr(sp, k, v)
    return sp


def compare16_spectral():
    """[is13_spectral:cSpectral] of config/compare16/ComParE_2016_core.lld.conf.inc:283-302"""
    return spectral_cfg(bands=[(250, 650), (1000, 4000)], rolloff=[0.25, 0.50, 0.75, 0.90], flux=1, centroid=1,
                        maxPos=0, minPos=0, entropy=1, variance=1, skewness=1, kurtosis=1, slope=1,
                        harmonicity=1, sharpness=1)


def gemaps_logspectral():
    """[gemapsv01b_logSpectral:cSpectral] of config/gemaps/v01b/GeMAPSv01b_core.lld.conf.inc:321-346"""
    return spectral_cfg(slopes=[(0, 500), (500, 1500)], flux=0, centroid=0, maxPos=0, minPos=0, alphaRatio=1,
                        hammarbergIndex=1, normBandEnergies=1, squareInput=1, useLogSpectrum=1,
                        freqRangeLo=0, freqRangeHi=5000, oldSlopeScale=0)


def frontend(sample_rate, frame_size, frame_step, win="ham", preemph=None, sigma=0.4, zero_pad_symmetric=1):
    return Frontend(sample_rate, frame_size, frame_step, 1 if preemph is not None else 0,
                    preemph if preemph is not None else 0.97, WIN[win], sigma, 1.0, 0.0, zero_pad_symmetric)


def _run_static(fn_name, nout_name, fe, cfg, pcm, n_chan, extra=()):
    pcm = np.ascontiguousarray(pcm, dtype=np.int16)
    nS = pcm.size // n_chan
    N, H, nfft, T = geometry(fe, nS)
    L = lib()
    getattr(L, fn_name).restype = C.c_long
    K = getattr(L, nout_name)(C.byref(cfg))
    out = np.zeros((max(T, 0), K), np.float32)
    r = getattr(L, fn_name)(C.byref(fe), C.byref(cfg), *extra, pcm.ctypes.data_as(C.POINTER(C.c_int16)),
                            C.c_long(nS), C.c_int(n_chan), _fp(out))
    assert r == max(T, 0), (r, T)
    return out


def spectral(pcm, fe, cfg, n_chan=1):
    return _run_static("osm_or_spectral", "osm_or_spectral_num_out", fe, cfg, pcm, n_chan)


def spectral_from_mag(mag, fe, cfg):
    """cSpectral on given magnitudes [T, nfft/2+1] of one utterance (fe gives the bin frequencies)"""
    mag = np.ascontiguousarray(mag, np.float32)
    T = mag.shape[0]
    L = lib()
    L.osm_or_spectral_from_mag.restype = C.c_long
    out = np.zeros((T, L.osm_or_spectral_num_out(C.byref(cfg))), np.float32)
    r = L.osm_or_spectral_from_mag(C.byref(fe), C.byref(cfg), _fp(mag), C.c_long(T), _fp(out))
    assert r == T, (r, T)
    return out


def energy(pcm, fe, cfg=None, windowed=0, n_chan=1):
    cfg = cfg or Energy(0, 1, 0, 1, 1.0, 1.0, 1.0, 0.0, 0.0, 0.0)
    return _run_static("osm_or_energy", "osm_or_energy_num_out", fe, cfg, pcm, n_chan, (C.c_int(windowed),))


def mzcr(pcm, fe, cfg=None, windowed=0, n_chan=1):
    cfg = cfg or MZcr(1, 1, 1, 1, 0)
    return _run_static("osm_or_mzcr", "osm_or_mzcr_num_out", fe, cfg, pcm, n_chan, (C.c_int(windowed),))


class Intensity(C.Structure):
    _fields_ = [("intensity", C.c_int), ("loudness", C.c_int)]


def intensity(pcm, fe, cfg=None, windowed=0, n_chan=1):
    cfg = cfg or Intensity(1, 0)
    return _run_static("osm_or_intensity", "osm_or_intensity_num_out", fe, cfg, pcm, n_chan, (C.c_int(windowed),))


def build(force=False):
    """Compile liboracle.so with gcc (oracle/Makefile)."""
    so = os.path.join(_HERE, "liboracle.so")
    src = [os.path.join(_HERE, f) for f in ("osm_oracle.c", "osm_oracle.h", "osm_oracle_pitch.c", "osm_oracle_pitch.h")]
    if force or not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in src):
        subprocess.check_call(["make", "-s", "-C", _HERE, "liboracle.so"])
    return so


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
        L = _LIB
        L.osm_or_frame_size_samples.restype = C.c_long
        L.osm_or_frame_step_samples.restype = C.c_long
        L.osm_or_fft_size.restype = C.c_long
        L.osm_or_fft_size.argtypes = [C.c_long]
        L.osm_or_num_frames.restype = C.c_long
        L.osm_or_num_frames.argtypes = [C.c_long, C.c_long, C.c_long]
        L.osm_or_fft_frame_size_sec.restype = C.c_double
        L.osm_or_mfcc_d_a.restype = C.c_long
        L.osm_or_plp_d_a.restype = C.c_long
        L.osm_or_delta.restype = C.c_long
        L.osm_or_sma.restype = C.c_long
        L.osm_or_delta_chained.restype = C.c_long
        L.osm_or_sma_chained.restype = C.c_long
    return _LIB


def _fp(a):
    return a.ctypes.data_as(C.POINTER(C.c_float)) if a is not None else None


# ---- config presets mirroring the shipped .conf files (values read from
# /root/reference/config/mfcc/MFCC12_0_D_A.conf, config/plp/PLP_0_D_A.conf) ----

def pcm_to_float(buf, fmt, n_chan=1):
    """a-1 for every sample format (osm_or_pcm_to_float): buf = the bytes of interleaved sample frames, fmt = osm_b200_pcm_format
    (0 int16, 1 float32, 2 int8, 3 packed 24 bit, 4 24 bit in 32, 5 int32) -> mono float32 samples"""
    raw = np.ascontiguousarray(np.frombuffer(bytes(buf), np.uint8))
    bps = {0: 2, 1: 4, 2: 1, 3: 3, 4: 4, 5: 4}[fmt]
    n = raw.size // (bps * n_chan)
    out = np.empty(n, np.float32)
    L = lib()
    L.osm_or_pcm_to_float.argtypes = [C.c_void_p, C.c_int, C.c_long, C.c_int, C.c_void_p]
    L.osm_or_pcm_to_float.restype = None
    L.osm_or_pcm_to_float(raw.ctypes.data, fmt, n, n_chan, out.ctypes.data)
    return out


def mfcc12_0_d_a(sample_rate):
    fe = Frontend(sample_rate, 0.025, 0.010, 1, 0.97, WIN["ham"], 0.4, 1.0, 0.0, 0)
    ms = Melspec(26, 0.0, 8000.0, 1, 1)
    mf = Mfcc(0, 12, 22.0, 1e-8, 1)
    return fe, ms, mf


def geometry(fe, n_samples):
    L = lib()
    N = L.osm_or_frame_size_samples(C.byref(fe))
    H = L.osm_or_frame_step_samples(C.byref(fe))
    nfft = L.osm_or_fft_size(N)
    T = L.osm_or_num_frames(n_samples, N, H)
    return N, H, nfft, T


def mfcc_d_a(pcm, sample_rate, n_chan=1, taps=False, cfg=None, delta_win=2, accel_win=2):
    """int16 PCM [L*n_chan] -> float32 [T, 3*nMfcc] (static | delta | accel)."""
    fe, ms, mf = cfg if cfg is not None else mfcc12_0_d_a(sample_rate)
    pcm = np.ascontiguousarray(pcm, dtype=np.int16)
    nS = pcm.size // n_chan
    N, H, nfft, T = geometry(fe, nS)
    K = mf.last_mfcc - mf.first_mfcc + 1
    out = np.zeros((max(T, 0), 3 * K), np.float32)
    tap_mag = np.zeros((max(T, 0), nfft // 2 + 1), np.float32) if taps else None
    tap_mel = np.zeros((max(T, 0), ms.n_bands), np.float32) if taps else None
    r = lib().osm_or_mfcc_d_a(C.byref(fe), C.byref(ms), C.byref(mf), C.c_int(delta_win),
                              C.c_int(accel_win), pcm.ctypes.data_as(C.POINTER(C.c_int16)),
                              C.c_long(nS), C.c_int(n_chan), _fp(out), _fp(tap_mag), _fp(tap_mel))
    assert r == max(T, 0), (r, T)
    return (out, tap_mag, tap_mel) if taps else out


def plp_0_d_a(sample_rate):
    """config/plp/PLP_0_D_A.conf"""
    fe = Frontend(sample_rate, 0.025, 0.010, 1, 0.97, WIN["ham"], 0.4, 1.0, 0.0, 0)
    ms = Melspec(26, 0.0, 8000.0, 1, 1)
    pl = Plp(5, 0, -1, 0, 1, 0, 1, 1, 1, 0, 0, 29.0, 1.0, 22.0, 0.33, 9.3e-10, 1)
    return fe, ms, pl


def plp_d_a(pcm, sample_rate, n_chan=1, cfg=None, delta_win=2, accel_win=2):
    """int16 PCM -> float32 [T, 3*nCeps] (PlpCC static | delta | accel)."""
    fe, ms, pl = cfg if cfg is not None else plp_0_d_a(sample_rate)
    pcm = np.ascontiguousarray(pcm, dtype=np.int16)
    nS = pcm.size // n_chan
    N, H, nfft, T = geometry(fe, nS)
    K = lib().osm_or_plp_num_out(C.byref(pl), C.c_int(ms.n_bands))
    out = np.zeros((max(T, 0), 3 * K), np.float32)
    r = lib().osm_or_plp_d_a(C.byref(fe), C.byref(ms), C.byref(pl), C.c_int(delta_win), C.c_int(accel_win),
                             pcm.ctypes.data_as(C.POINTER(C.c_int16)), C.c_long(nS), C.c_int(n_chan),
                             _fp(out), None)
    assert r == max(T, 0), (r, T)
    return out


def plp_static(pcm, sample_rate, cfg, n_chan=1):
    """cPlp static level only (with RASTA / newRASTA when configured): int16 PCM -> float32 [T, nOut]."""
    fe, ms, pl = cfg
    pcm = np.ascontiguousarray(pcm, dtype=np.int16)
    nS = pcm.size // n_chan
    N, H, nfft, T = geometry(fe, nS)
    K = lib().osm_or_plp_num_out(C.byref(pl), C.c_int(ms.n_bands))
    out = np.zeros((max(T, 0), K), np.float32)
    lib().osm_or_plp_static.restype = C.c_long
    r = lib().osm_or_plp_static(C.byref(fe), C.byref(ms), C.byref(pl), pcm.ctypes.data_as(C.POINTER(C.c_int16)),
                                C.c_long(nS), C.c_int(n_chan), _fp(out))
    assert r == max(T, 0), (r, T)
    return out


def cms(x):
    """cFullinputMean (default mode): subtract the per-column mean over all frames (float, frame order)."""
    x = np.ascontiguousarray(x, np.float32)
    out = np.zeros_like(x)
    lib().osm_or_cms(_fp(x), C.c_long(x.shape[0]), C.c_int(x.shape[1]), _fp(out))
    return out


def ll1(x):
    """cVectorOperation operation=ll1: per-row float sum / K."""
    x = np.ascontiguousarray(x, np.float32)
    out = np.zeros(x.shape[0], np.float32)
    lib().osm_or_ll1(_fp(x), C.c_long(x.shape[0]), C.c_int(x.shape[1]), _fp(out))
    return out


def delta(x, win):
    x = np.ascontiguousarray(x, np.float32)
    T, K = x.shape
    out = np.zeros((T + win, K), np.float32)
    r = lib().osm_or_delta(_fp(x), C.c_long(T), C.c_int(K), C.c_int(win), _fp(out))
    return out[:r]


def delta_variant(x, win, relative=0, abs_output=0, half_wave=0):
    """cDeltaRegression with relativeDelta / absOutput / halfWaveRect on a complete level"""
    x = np.ascontiguousarray(x, np.float32)
    T, K = x.shape
    out = np.zeros((T + win, K), np.float32)
    L = lib()
    L.osm_or_delta_variant.restype = C.c_long
    r = L.osm_or_delta_variant(_fp(x), C.c_long(T), C.c_int(K), C.c_int(win), C.c_int(relative), C.c_int(abs_output), C.c_int(half_wave), _fp(out))
    return out[:r]


def delta_chained(x, win, n0):
    """Stage reading a level of which only n0 frames exist when EOI is raised.
    Returns (out, c0) with c0 = the same quantity for the produced level."""
    x = np.ascontiguousarray(x, np.float32)
    T, K = x.shape
    out = np.zeros((T + win, K), np.float32)
    c0 = C.c_long(0)
    r = lib().osm_or_delta_chained(_fp(x), C.c_long(T), C.c_long(n0), C.c_int(K), C.c_int(win), _fp(out), C.byref(c0))
    return out[:r], c0.value


def sma_chained(x, sma_win, n0, no_zero_sma=0):
    x = np.ascontiguousarray(x, np.float32)
    T, K = x.shape
    out = np.zeros((T + sma_win // 2, K), np.float32)
    c0 = C.c_long(0)
    r = lib().osm_or_sma_chained(_fp(x), C.c_long(T), C.c_long(n0), C.c_int(K), C.c_int(sma_win), C.c_int(no_zero_sma),
                                 _fp(out), C.byref(c0))
    return out[:r], c0.value


def sma(x, sma_win=3, no_zero_sma=0):
    x = np.ascontiguousarray(x, np.float32)
    T, K = x.shape
    out = np.zeros((T + (sma_win - 1) // 2, K), np.float32)
    r = lib().osm_or_sma(_fp(x), C.c_long(T), C.c_int(K), C.c_int(sma_win), C.c_int(no_zero_sma), _fp(out))
    return out[:r]


# ---- SHS pitch chain (oracle/osm_oracle_pitch.c): cSpecScale -> cPitchShs -> cPitchSmootherViterbi ->
# cValbasedSelector -> cPitchJitter, values of config/compare16/ComParE_2016_core.lld.conf.inc ----

class SpecScale(C.Structure):
    _fields_ = [("minF", C.c_double), ("maxF", C.c_double), ("nPointsTarget", C.c_int), ("specSmooth", C.c_int),
                ("specEnhance", C.c_int), ("auditoryWeighting", C.c_int)]


class PitchShs(C.Structure):
    _fields_ = [("maxPitch", C.c_double), ("minPitch", C.c_double), ("nCandidates", C.c_int), ("scores", C.c_int),
                ("voicing", C.c_int), ("F0C1", C.c_int), ("voicingC1", C.c_int), ("F0raw", C.c_int), ("voicingClip", C.c_int),
                ("voicingCutoff", C.c_double), ("octaveCorrection", C.c_int), ("nHarmonics", C.c_int),
                ("compressionFactor", C.c_double), ("greedyPeakAlgo", C.c_int), ("lfCut", C.c_double)]


class Viterbi(C.Structure):
    _fields_ = [("bufferLength", C.c_int), ("F0final", C.c_int), ("F0finalLog", C.c_int), ("F0finalEnv", C.c_int),
                ("F0finalEnvLog", C.c_int), ("voicingFinalClipped", C.c_int), ("voicingFinalUnclipped", C.c_int),
                ("wLocal", C.c_double), ("wTvv", C.c_double), ("wTvvd", C.c_double), ("wTvuv", C.c_double),
                ("wThr", C.c_double), ("wRange", C.c_double), ("wTuu", C.c_double)]


class Jitter(C.Structure):
    _fields_ = [("searchRangeRel", C.c_double), ("jitterLocal", C.c_int), ("jitterDDP", C.c_int), ("jitterLocalEnv", C.c_int),
                ("jitterDDPEnv", C.c_int), ("shimmerLocal", C.c_int), ("shimmerLocalDB", C.c_int), ("shimmerLocalEnv", C.c_int),
                ("shimmerLocalDBEnv", C.c_int), ("harmonicERMS", C.c_int), ("noiseERMS", C.c_int), ("linearHNR", C.c_int),
                ("logHNR", C.c_int), ("lgHNRfloor", C.c_double), ("shimmerUseRmsAmplitude", C.c_int), ("minNumPeriods", C.c_int),
                ("minCC", C.c_double), ("refinedF0", C.c_int), ("sourceQualityRange", C.c_int), ("sourceQualityMean", C.c_int),
                ("usePeakToPeakPeriodLength", C.c_int), ("useBrokenJitterThresh", C.c_int), ("onlyVoiced", C.c_int)]


def compare16_pitch_cfg():
    """(frontend, SpecScale, PitchShs, Viterbi, Jitter) of ComParE_2016_core.lld.conf.inc:16-46,62-190"""
    fe = frontend(16000.0, 0.060, 0.010, win="gau", sigma=0.4, zero_pad_symmetric=1)
    sc = SpecScale(25.0, -1.0, 0, 1, 1, 1)
    ps = PitchShs(620.0, 52.0, 6, 1, 1, 0, 0, 1, 1, 0.70, 0, 15, 0.85, 1, 0.0)
    vc = Viterbi(30, 1, 0, 0, 0, 0, 1, 2.0, 10.0, 5.0, 10.0, 4.0, 1.0, 0.0)
    jc = Jitter(0.25, 1, 1, 0, 0, 1, 0, 0, 0, 0, 0, 0, 1, -100.0, 0, 2, 0.5, 0, 0, 0, 0, 0, 0)
    return fe, sc, ps, vc, jc


def pitch_shs(pcm, fe, sc, ps, n_chan=1, tap=False):
    pcm = np.ascontiguousarray(pcm, dtype=np.int16)
    nS = pcm.size // n_chan
    N, H, nfft, T = geometry(fe, nS)
    L = lib()
    L.osm_or_pitch_shs.restype = C.c_long
    K = L.osm_or_pitchshs_num_out(C.byref(ps))
    out = np.zeros((max(T, 0), K), np.float32)
    npts = sc.nPointsTarget if sc.nPointsTarget > 0 else nfft // 2 + 1
    hps = np.zeros((max(T, 0), npts), np.float32) if tap else None
    r = L.osm_or_pitch_shs(C.byref(fe), C.byref(sc), C.byref(ps), pcm.ctypes.data_as(C.POINTER(C.c_int16)), C.c_long(nS),
                           C.c_int(n_chan), _fp(out), _fp(hps))
    assert r == max(T, 0), (r, T)
    return (out, hps) if tap else out


def viterbi(shs, ps, vc, with_lag=False):
    """-> [T, K] (and V = frames the level holds before the end-of-input flush when with_lag)"""
    shs = np.ascontiguousarray(shs, np.float32)
    L = lib()
    L.osm_or_viterbi.restype = C.c_long
    K = L.osm_or_viterbi_num_out(C.byref(vc))
    out = np.zeros((shs.shape[0], K), np.float32)
    v = C.c_long(0)
    r = L.osm_or_viterbi(C.byref(ps), C.byref(vc), _fp(shs), C.c_long(shs.shape[0]), _fp(out), C.byref(v))
    assert r == shs.shape[0], (r, shs.shape)
    return (out, v.value) if with_lag else out


def sma_nz_lagged(x, V, lag_cols):
    """cContourSmoother (smaWin=3, noZeroSma=1) over a multi-level reader whose `lag_cols` come from a level
    that holds only V frames during the reference's first end-of-input pass (cPitchJitter does not run while
    EOI is set, lld/pitchJitter.cpp:593): output rows V-1 and V see that level padded with its row V-1
    (core/dataMemoryLevel.cpp:1020-1027,1698-1708); every other row is the plain clamp-at-the-ends result.
    Verified against oracle/_ref (scripts/make_golden_pitch.py)."""
    x = np.asarray(x, np.float32)
    T, K = x.shape
    out = np.zeros((T + 1, K), np.float32)
    for n in range(T + 1):
        for k in range(K):
            def g(i):
                i = min(max(i, 0), T - 1)
                if V >= 1 and k in lag_cols and n in (V - 1, V) and i > V - 1:     # V == 0: the lagging level is
                    i = V - 1                                                      # empty, nothing runs in the first pass
                return x[i, k]
            x0 = g(n)
            if x0 != 0:
                y, N = np.float32(x0), 1
                for v in (g(n - 1), g(n + 1)):
                    if v != 0:
                        y = np.float32(y + v)
                        N += 1
                out[n, k] = np.float32(y / np.float32(N))
    return out


def delta_segments_lagged(x, V, win=2):
    """cDeltaRegression (onlyInSegments=1) behind sma_nz_lagged: x = [T+1, K].  Rows V-1..V+2 are computed
    during the first end-of-input pass, when the input level ends at row V; row V+3 (if T-5 <= V <= T-2) is
    computed in the first tick of the second pass, when it ends at row T-1; the accumulating norm
    (dspcore/deltaRegression.cpp:123-141) runs through all rows in order."""
    x = np.asarray(x, np.float32)
    T1, K = x.shape
    T = T1 - 1
    out = np.zeros((T1 + win, K), np.float32)
    norm = np.float32(0)
    for i in range(1, win + 1):
        norm = np.float32(norm + np.float32(i) * np.float32(i))
    norm = np.float32(norm * 2)
    for n in range(T1 + win):
        last = T1 - 1
        if V >= 1 and V - 1 <= n <= V + 2:
            last = min(last, V)
        elif n == V + 3 and T - 5 <= V <= T - 2:
            last = T - 1
        for k in range(K):
            num = np.float32(0)
            for i in range(1, win + 1):
                a = x[min(max(n - i, 0), last), k]
                b = x[min(max(n + i, 0), last), k]
                if a != 0 and b != 0 and a == a and b == b:
                    num = np.float32(num + np.float32(i) * np.float32(b - a))
                    norm = np.float32(norm + np.float32(i) * np.float32(i))
            out[n, k] = np.float32(num / norm) if norm != 0 else np.float32(0)
    return out


def valbased_select(sel, x, threshold, output_val=0.0):
    sel = np.ascontiguousarray(sel, np.float32).reshape(-1)
    x = np.ascontiguousarray(x, np.float32)
    out = np.zeros_like(x)
    lib().osm_or_valbased_select(_fp(sel), _fp(x), C.c_long(x.shape[0]), C.c_int(x.shape[1]), C.c_double(threshold),
                                 C.c_double(output_val), _fp(out))
    return out


def pitch_jitter(pcm, fe, jc, f0, n_chan=1):
    pcm = np.ascontiguousarray(pcm, dtype=np.int16)
    nS = pcm.size // n_chan
    f0 = np.ascontiguousarray(f0, np.float32).reshape(-1)
    L = lib()
    L.osm_or_pitch_jitter.restype = C.c_long
    K = L.osm_or_jitter_num_out(C.byref(jc))
    out = np.zeros((f0.size, K), np.float32)
    r = L.osm_or_pitch_jitter(C.byref(fe), C.byref(jc), pcm.ctypes.data_as(C.POINTER(C.c_int16)), C.c_long(nS), C.c_int(n_chan),
                              _fp(f0), C.c_long(f0.size), _fp(out))
    return out[:r]


def delta_segments(x, win, n0=None):
    x = np.ascontiguousarray(x, np.float32)
    T, K = x.shape
    out = np.zeros((T + win, K), np.float32)
    L = lib()
    L.osm_or_delta_segments.restype = C.c_long
    r = L.osm_or_delta_segments(_fp(x), C.c_long(T), C.c_long(T if n0 is None else n0), C.c_int(K), C.c_int(win), _fp(out))
    return out[:r]


def compare16_pitch(pcm, n_chan=1, sample_rate=16000.0, with_lag=False):
    """The six `nz` columns of ComParE_2016 before smoothing: F0final, voicingFinalUnclipped, jitterLocal,
    jitterDDP, shimmerLocal, logHNR -> [T, 6]"""
    fe, sc, ps, vc, jc = compare16_pitch_cfg()
    fe.sample_rate = sample_rate
    shs = pitch_shs(pcm, fe, sc, ps, n_chan)
    vit, lag = viterbi(shs, ps, vc, with_lag=True)
    e60 = energy(pcm, fe, Energy(0, 1, 0, 0, 1.0, 1.0, 1.0, 0.0, 0.0, 0.0), windowed=1, n_chan=n_chan)
    sel = valbased_select(e60[:, 0], vit, 0.001)
    jit = pitch_jitter(pcm, fe, jc, sel[:, 0], n_chan)
    nz = np.concatenate([sel, jit], axis=1)
    return (nz, lag) if with_lag else nz


def compare16_nz_lld(pcm, n_chan=1, sample_rate=16000.0):
    """ComParE_2016 levels is13_lld_nzsmo [T+1, 6] and is13_lld_nzsmo_de [T+3, 6] (ComParE_2016_core.lld.conf.inc:331-341,392-398)"""
    nz, lag = compare16_pitch(pcm, n_chan, sample_rate, with_lag=True)
    sm = sma_nz_lagged(nz, lag, {2, 3, 4, 5})
    return sm, delta_segments_lagged(sm, lag, 2)


def pitch_variants_cfg():
    """tests/configs/pitch_variants.conf"""
    fe = frontend(16000.0, 0.050, 0.010, win="ham", zero_pad_symmetric=1)
    sc = SpecScale(30.0, 4000.0, 400, 1, 0, 0)
    ps = PitchShs(500.0, 60.0, 3, 1, 1, 1, 1, 1, 1, 0.65, 1, 10, 0.8, 0, 0.0)
    vc = Viterbi(8, 1, 1, 1, 1, 1, 1, 1.5, 8.0, 3.0, 6.0, 3.0, 2.0, 0.5)
    jc = Jitter(0.15, 1, 1, 1, 1, 1, 1, 1, 0, 1, 1, 1, 1, -100.0, 0, 2, 0.4, 1, 1, 1, 0, 1, 0)
    return fe, sc, ps, vc, jc


def pitch_variants_lld(pcm, n_chan=1):
    """levels smo ; smo_de of tests/configs/pitch_variants.conf -> [T+1, 36] (no energy gate, plain smoother)"""
    fe, sc, ps, vc, jc = pitch_variants_cfg()
    shs = pitch_shs(pcm, fe, sc, ps, n_chan)
    vit, lag = viterbi(shs, ps, vc, with_lag=True)
    jit = pitch_jitter(pcm, fe, jc, vit[:, 0], n_chan)
    x = np.concatenate([vit, jit], axis=1)
    nv = vit.shape[1]
    sm = sma_lagged(x, lag, set(range(nv, x.shape[1])), no_zero=False)
    de = delta_segments_lagged(sm, lag, 2)
    R = sm.shape[0]
    return np.concatenate([sm, de[:R]], axis=1), lag


def sma_lagged(x, V, lag_cols, no_zero):
    """sma_nz_lagged with the noZeroSma switch (dspcore/contourSmoother.cpp:84-117)"""
    if no_zero:
        return sma_nz_lagged(x, V, lag_cols)
    x = np.asarray(x, np.float32)
    T, K = x.shape
    out = np.zeros((T + 1, K), np.float32)
    for n in range(T + 1):
        for k in range(K):
            def g(i):
                i = min(max(i, 0), T - 1)
                if V >= 1 and k in lag_cols and n in (V - 1, V) and i > V - 1:
                    i = V - 1
                return x[i, k]
            y = np.float32(g(n))
            y = np.float32(y + g(n - 1))
            y = np.float32(y + g(n + 1))
            out[n, k] = np.float32(y / np.float32(3.0))
    return out
