"""The case table of tests/spectral_cases.py without a GPU:
  - every case opens on a description-only plan at its op's level, with the element count the oracle produces;
  - the table reaches every listed value of every axis;
  - the oracle's entry points on given magnitudes (osm_or_spectral_from_mag, osm_or_pitchacf_from_mag), fed the oracle's own
    magnitudes, reproduce its whole-chain functions bit for bit;
  - the oracle against the unmodified reference (tests/golden/spectral_variants.npz, scripts/make_golden_spectral_variants.py) under
    the cSpectral and cAcf / cPitchACF options the other goldens leave at their defaults;
  - the refusals of the graph pass, with their messages."""
import os
import ctypes as C

import numpy as np
import pytest

import spectral_cases as SC
from conftest import GOLD
from opensmile_b200 import Plan, comp, components_frontend
from oracle import oracle


def _plan_or_error(cs, level):
    try:
        p = Plan(cs, level, device=-1)
    except RuntimeError as e:
        return None, str(e)
    return p, None


@pytest.mark.parametrize("name", list(SC.BY_NAME))
def test_case_opens_on_a_description_only_plan(name):
    c = SC.BY_NAME[name]
    p, err = _plan_or_error(SC.components(c), SC.level(c))
    assert p is not None, err
    try:
        cfg = SC.oracle_cfg(c)
        fn = dict(spectral="osm_or_spectral_num_out", pitch="osm_or_pitchacf_num_out", energy="osm_or_energy_num_out",
                  mzcr="osm_or_mzcr_num_out", intensity="osm_or_intensity_num_out")[c["op"]]
        assert p.num_elements == getattr(oracle.lib(), fn)(C.byref(cfg))
        N, S, nfft = SC.geometry(c)
        assert (p.frame_size, p.frame_step) == (N, S)
        if c["op"] in ("spectral", "pitch"):
            assert p.fft_size == nfft
    finally:
        p.close()


def test_table_reaches_every_axis_value():
    seen = {k: set() for k in SC.AXES}
    for c in SC.CASES:
        for k, v in SC.axis_sets(c).items():
            if k in seen:
                seen[k] |= v
    for axis, values in SC.AXES.items():
        assert values <= seen[axis], (axis, values - seen[axis])


def _oracle_mags(c, x):
    """the oracle's own magnitudes of the case's frames (its MFCC chain's magnitude tap, same front end)"""
    fe = SC.frontend(c)
    ms = oracle.Melspec(26, 0.0, c["sr"] / 2, 1, 1, 0, 0.0)
    mf = oracle.Mfcc(0, 12, 22.0, 1e-8, 1)
    return oracle.mfcc_d_a(x, c["sr"], n_chan=c["n_chan"], taps=True, cfg=(fe, ms, mf))[1]


@pytest.mark.parametrize("name", [n for n, c in SC.BY_NAME.items() if c["op"] in ("spectral", "pitch") and c["step"] >= 0.005])
def test_oracle_entry_points_on_magnitudes_reproduce_the_chain(name):
    """the FFT front end split off: the same rows, bit for bit, for every signal kind (the pitch state machine included)"""
    c = SC.BY_NAME[name]
    utts = SC.batch(c)[0]
    for x in utts[-len(SC.KINDS):] + utts[2:4]:
        whole = SC.oracle_rows(c, x)
        mag = _oracle_mags(c, x)
        assert mag.shape[0] == whole.shape[0]
        part = SC.oracle_from_mag(c, mag)
        assert part.shape == whole.shape
        assert np.array_equal(part.view(np.uint32), whole.view(np.uint32))


def _pitch_components(sr, frame, max_pitch):
    return components_frontend(float(sr), frame, 0.010, win="gau", zero_pad_symmetric=0) + [
        comp("cAcf", "acf", "mag", "acf"),
        comp("cAcf", "cep", "mag", "cepstrum", cepstrum=1, usePower=0),
        comp("cPitchACF", "pitch", "acf;cepstrum", "pitch", maxPitch=max_pitch, F0=1)]


@pytest.mark.parametrize("cs,level,msg", [
    (components_frontend(8000.0, 0.025) + [comp("cSpectral", "spec", "mag", "spec")], "spec",
     "FFT size 256 not supported (512, 1024, 2048, 4096)"),
    (_pitch_components(16000, 0.010, 500.0), "pitch", "FFT size 256 not supported (512, 1024, 2048, 4096)"),
    (_pitch_components(16000, 0.060, 15.0), "pitch", "cPitchACF: maxPitch = 15 Hz skips 1066 lags, not fewer than the 1024 elements"),
    (_pitch_components(16000, 0.025, 31.0), "pitch", "cPitchACF: maxPitch = 31 Hz skips 516 lags, not fewer than the 512 elements"),
    (components_frontend(16000.0, 0.025) + [comp("cSpectral", "spec", "mag", "spec", freqRange=(1000, 1120))], "spec",
     "cSpectral: spectral range too narrow"),
    # oldCompatCepstrum drops acfCepsNormOutput on the cepstrum instance only (acf.cpp:104); acf_pitch_kernel normalises both
    # levels alike, so a normalised ACF next to it is refused (the oracle's rule is pinned against the reference by
    # test_oracle_pitchacf_against_the_reference[old_compat_acf_norm1])
    (SC.components(dict(SC.BY_NAME["p_old_compat_cepstrum"], norm_out=1)), "pitch", "cAcf.acfCepsNormOutput must agree on both instances"),
])
def test_refusals(cs, level, msg):
    """each refused on a description-only plan, with its message (FFT 4096 for cAcf is refused by a device plan:
    test_spectral_sweep_gpu.py::test_acf_refuses_fft4096_on_a_device_plan)"""
    p, err = _plan_or_error(cs, level)
    assert p is None, msg
    assert msg in err, err


def test_narrowest_accepted_range_is_the_boundary():
    """freqRange (1000, 1150) at 31.25 Hz bins: hiBin - loBin = 4, accepted; (1000, 1120) gives 3 and is refused above"""
    c = SC.BY_NAME["s_range_narrowest"]
    lo, hi = SC.spectral_range(c)
    assert hi - lo == 4
    assert SC.spectral_range(dict(c, frange=(1000, 1120)))[1] - lo == 3


def test_largest_accepted_preskip_is_the_boundary():
    """preskip = 2n - 1 opens, preskip = 2n is refused (FFT 1024 at 16 kHz: Tsamp = 1/16000 s, rounded through the float frame
    length)"""
    ok, _ = _plan_or_error(_pitch_components(16000, 0.060, 15.64), "pitch")
    assert ok is not None
    ok.close()
    c = dict(SC.BY_NAME["p_preskip_between_n_2n"], max_pitch=15.64)
    assert SC.preskip(c) == 1023
    p, err = _plan_or_error(_pitch_components(16000, 0.060, 15.62), "pitch")
    assert p is None and "skips 1024 lags" in err, err


# ---------------------------------------------------------------- the oracle against the reference (tests/configs/spectral_variants.conf)
VARIANTS = np.load(os.path.join(GOLD, "spectral_variants.npz"))
V_BANDS = ((0, 31), (125, 250), (100, 110), (3990, 8000), (7000, 9000), (8000, 20000))
V_SLOPES = ((0, 125), (40, 300), (7990, 12000), (0, 500), (500, 1500))
V_ROLL = (0.05, 0.11, 0.18, 0.24, 0.3, 0.36, 0.43, 0.49, 0.55, 0.61, 0.68, 0.74, 0.8, 0.86, 0.93, 0.99)
V_SPECTRAL = {
    "default": {}, "magnitude_input": dict(squareInput=0), "norm": dict(normBandEnergies=1), "log": dict(useLogSpectrum=1),
    "log_norm": dict(useLogSpectrum=1, normBandEnergies=1), "log_magnitude_input": dict(useLogSpectrum=1, squareInput=0),
    "buggy_rolloff": dict(buggyRollOff=1), "new_slope_scale": dict(oldSlopeScale=0), "range_narrowest": dict(freqRangeLo=1000, freqRangeHi=1150),
    "log_range_0_5000": dict(useLogSpectrum=1, freqRangeLo=0, freqRangeHi=5000, oldSlopeScale=0)}
# the oracle has one acfCepsNormOutput: oldCompatCepstrum drops it on the cepstrum instance only (acf.cpp:104), so
# old_compat_acf_norm1 (acfNorm = cepNorm = 1 in the configuration) checks that rule
V_PITCH = {
    "default": {}, "acf_magnitude_cep_power": dict(acfUsePower=0, cepUsePower=1), "no_norm": dict(acfCepsNormOutput=0),
    "abs_cepstrum": dict(absCepstrum=1), "old_compat_cep_power0": dict(oldCompatCepstrum=1, acfCepsNormOutput=0),
    "old_compat_cep_power1": dict(oldCompatCepstrum=1, acfCepsNormOutput=0, cepUsePower=1),
    "old_compat_acf_norm1": dict(oldCompatCepstrum=1, cepUsePower=1),
    "max_pitch_2000_cutoff_1": dict(maxPitch=2000.0, voicingCutoff=1.7), "max_pitch_0_cutoff_0": dict(maxPitch=0.0, voicingCutoff=-0.3)}
IMPULSE_ROWS = slice(94, 112)          # frames of the golden signal that hold one impulse each (samples 15000 .. 18200)


def test_variant_goldens_cover_the_option_sets():
    assert {"spec_" + k for k in V_SPECTRAL} | {"pitch_" + k for k in V_PITCH} | {"pcm"} == set(VARIANTS.files)


@pytest.mark.parametrize("name", list(V_SPECTRAL))
def test_oracle_spectral_against_the_reference(name):
    """every descriptor, 16 roll-off points, band and slope edges on bins, between bins, at 0 Hz and above Nyquist.  The oracle's
    FFT is not the reference's (they agree to ~2e-7 of the frame peak): continuous columns within 1e-5 of the column scale (5e-5
    with a log spectrum: dB values of bins far below the peak carry that rounding, measured 1.9e-5); roll-off points and max / min
    positions equal.  On the impulse-train frames every bin of the magnitude spectrum is the same value up to the FFT's rounding:
    there the max / min positions, the roll-off points and the log-spectral entropy decide between equal bins and are not compared"""
    fe = oracle.frontend(16000.0, 0.025, 0.010, "ham")
    d = dict(flux=1, centroid=1, maxPos=1, minPos=1, entropy=1, standardDeviation=1, variance=1, skewness=1, kurtosis=1, slope=1,
             alphaRatio=1, hammarbergIndex=1, sharpness=1, harmonicity=1, flatness=1)
    cfg = oracle.spectral_cfg(bands=V_BANDS, slopes=V_SLOPES, rolloff=V_ROLL, **dict(d, **V_SPECTRAL[name]))
    got, ref = oracle.spectral(VARIANTS["pcm"], fe, cfg), VARIANTS["spec_" + name]
    assert got.shape == ref.shape == (148, 42)
    log = V_SPECTRAL[name].get("useLogSpectrum", 0)
    dec = list(range(13, 29)) + [31, 32]                          # roll-off points, max / min position
    flat_excused = dec + ([33] if log else [])                    # + entropy of the log spectrum
    scale = np.abs(np.where(np.isfinite(ref), ref, 0)).max(axis=0)
    scale[scale == 0] = 1.0
    with np.errstate(invalid="ignore"):                          # -inf dB of silence on both sides: equal, not compared
        err = np.where(got == ref, 0.0, np.abs(got.astype(np.float64) - ref)) / scale
    flat = np.zeros(len(ref), bool)
    flat[IMPULSE_ROWS] = True
    for k in range(42):
        rows = ~flat if k in flat_excused else np.ones(len(ref), bool)
        if k in dec:
            assert np.array_equal(got[rows, k], ref[rows, k]), (k, np.nonzero(got[rows, k] != ref[rows, k])[0])
        else:
            assert err[rows, k].max() <= (5e-5 if log else 1e-5), (k, float(err[rows, k].max()))


@pytest.mark.parametrize("name", list(V_PITCH))
def test_oracle_pitchacf_against_the_reference(name):
    """cAcf x2 -> cPitchACF: lag decisions and the smoothed F0 / F0env equal; voicing, voiceQual within 1e-4 of the column scale,
    HNR / HNRdB / linHNR too except where the ACF at the chosen lag is below 1e-6 of its lag-0 value (HNRdB < -60 dB): that value
    sits at the rounding floor of the two FFTs (measured one such row of 146, -195.9 against -192.0)"""
    fe = oracle.frontend(16000.0, 0.050, 0.010, "gau", zero_pad_symmetric=0)
    cfg = oracle.pitchacf_cfg(**dict(dict(voiceProb=1, voiceQual=1, HNR=1, HNRdB=1, linHNR=1, F0=1, F0raw=1, F0env=1), **V_PITCH[name]))
    got, ref = oracle.pitchacf(VARIANTS["pcm"], fe, cfg), VARIANTS["pitch_" + name]
    assert got.shape == ref.shape == (146, 8)
    assert np.array_equal(got[:, 5:8], ref[:, 5:8])
    scale = np.maximum(np.abs(ref).max(axis=0), 1e-6)
    err = np.abs(got.astype(np.float64) - ref) / scale
    floor = ref[:, 2] < -60.0
    assert floor.sum() <= 2
    for k in range(5):
        rows = ~floor if k in (1, 2, 3) else np.ones(len(ref), bool)
        assert err[rows, k].max() <= 1e-4, (k, float(err[rows, k].max()))
