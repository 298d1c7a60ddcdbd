"""Generate tests/golden/spectral_variants.npz with the UNMODIFIED reference (oracle/_ref/SMILExtract): cSpectral and cAcf x2 ->
cPitchACF of tests/configs/spectral_variants.conf under each option set of SPECTRAL / PITCH, for one 1.5 s signal with digital
silence, a clipped square wave and an impulse train inside.  Build container only."""
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import refrun  # noqa: E402
from opensmile_b200.synth import mixed_pcm  # noqa: E402

# option set -> command line options of the configuration (defaults: squareInput 1, normBandEnergies 0, useLogSpectrum 0,
# buggyRollOff 0, oldSlopeScale 1, freqRange 0-0; acfUsePower 1, cepUsePower 0, acfNorm 1, cepNorm 1, oldCompatCepstrum 0,
# absCepstrum 0, maxPitch 500, voicingCutoff 0.55)
SPECTRAL = {
    "default": {},
    "magnitude_input": {"squareInput": "0"},
    "norm": {"normBandEnergies": "1"},
    "log": {"useLogSpectrum": "1"},
    "log_norm": {"useLogSpectrum": "1", "normBandEnergies": "1"},
    "log_magnitude_input": {"useLogSpectrum": "1", "squareInput": "0"},
    "buggy_rolloff": {"buggyRollOff": "1"},
    "new_slope_scale": {"oldSlopeScale": "0"},
    "range_narrowest": {"freqRange": "1000-1150"},
    "log_range_0_5000": {"useLogSpectrum": "1", "freqRange": "0-5000", "oldSlopeScale": "0"},
}
PITCH = {
    "default": {},
    "acf_magnitude_cep_power": {"acfUsePower": "0", "cepUsePower": "1"},
    "no_norm": {"acfNorm": "0", "cepNorm": "0"},
    "abs_cepstrum": {"absCepstrum": "1"},
    "old_compat_cep_power0": {"oldCompatCepstrum": "1", "acfNorm": "0"},
    "old_compat_cep_power1": {"oldCompatCepstrum": "1", "acfNorm": "0", "cepUsePower": "1"},
    "old_compat_acf_norm1": {"oldCompatCepstrum": "1", "cepUsePower": "1"},
    "max_pitch_2000_cutoff_1": {"maxPitch": "2000", "voicingCutoff": "1.7"},
    "max_pitch_0_cutoff_0": {"maxPitch": "0", "voicingCutoff": "-0.3"},
}


def signal():
    sr = 16000
    x = mixed_pcm(24000, sr, seed=21).astype(np.int64)
    x[6000:7600] = 0                                                         # digital silence
    t = np.arange(3200)
    x[10000:13200] = np.where((t * 2 * 150 // sr) % 2 == 0, 32767, -32768)    # full-scale square wave
    x[15000:18200] = 0
    x[15003:18200:400] = 20000                                               # one impulse per 25 ms frame
    return x.astype(np.int16)


def run(conf, wav, d, opts):
    so, po = os.path.join(d, "spec.htk"), os.path.join(d, "pitch.htk")
    args = [refrun.SMILEXTRACT, "-C", conf, "-I", wav, "-O", so, "-pitchO", po, "-l", "1"]
    for k, v in opts.items():
        args += ["-" + k, v]
    r = subprocess.run(args, capture_output=True, text=True)
    if r.returncode:
        print(r.stderr[-2000:])
        sys.exit(1)
    return refrun.read_htk(so)[0].astype(np.float32), refrun.read_htk(po)[0].astype(np.float32)


def main():
    pcm = signal()
    conf = os.path.join(ROOT, "tests", "configs", "spectral_variants.conf")
    out = {"pcm": pcm}
    with tempfile.TemporaryDirectory() as d:
        wav = os.path.join(d, "in.wav")
        refrun.write_wav(wav, pcm, 16000, 1)
        for name, opts in SPECTRAL.items():
            out["spec_" + name] = run(conf, wav, d, opts)[0]
            print("spec", name, out["spec_" + name].shape)
        for name, opts in PITCH.items():
            out["pitch_" + name] = run(conf, wav, d, opts)[1]
            print("pitch", name, out["pitch_" + name].shape)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "spectral_variants.npz"), **out)


if __name__ == "__main__":
    main()
