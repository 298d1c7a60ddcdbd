"""The float-input instances of the kernels that read PCM (energy, mzcr, intensity, jitter, formant, lpc and lld_kernel).

Inputs that are not 16-bit integer are converted to mono float samples by pcm_convert_kernel, and every kernel that reads PCM
has a second instance for that buffer.  Each graph below runs twice on the same signal: once from a 16-bit WAV file, once from a
32-bit float WAV file holding s / 32767 for every sample s.  pcm_convert_kernel passes mono float samples through unchanged and
div32767 equals that IEEE division for every int16 (tests/test_host_cpu.py), so both runs see identical samples:
- columns computed from the PCM and constant tables alone (energy, mzcr, intensity, lpc / lsp, formants) are bit-identical;
- the other columns pass the MFCC rule of tests/test_pcm_formats.py: the FFT of float input runs another lld_kernel instance."""
import os

import numpy as np
import pytest

from opensmile_b200 import capi
from opensmile_b200.synth import mixed_pcm
from test_pcm_formats import _close

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
EMOBASE = os.path.join(HERE, "..", "oracle", "_ref", "config", "emobase", "emobase.conf")
SR = 16000


def _both_formats(conf, options):
    """rows of the configuration's graph on int16 samples and on the same samples as float32 / 32767, and the element names"""
    from opensmile_b200 import Plan
    from opensmile_b200.session import Session
    s = Session(conf, options=options, device=-1)
    comps, level = s.components(float(SR), 1)
    s.close()
    s16 = mixed_pcm(48000, SR, seed=6)
    off = np.array([0, s16.size], np.int64)
    rows = []
    for fmt, pcm in ((0, s16), (1, s16.astype(np.float32) / np.float32(32767))):
        for c in comps:
            if c.type == capi.C_WAVESOURCE:
                c.u.wavesource.format = fmt
        plan = Plan(list(comps), level, device=0)
        rows.append(plan.run_host(pcm, off))
        names = plan.element_names
        plan.close()
    return rows[0], rows[1], names


def _check(conf, options, exact):
    a, b, names = _both_formats(conf, options)
    assert a.shape == b.shape and a.shape[0] > 100
    ex = [i for i, n in enumerate(names) if n.startswith(exact)]
    assert ex or not exact
    for i in ex:
        assert np.array_equal(a[:, i].view(np.uint32), b[:, i].view(np.uint32)), names[i]
    rest = [i for i in range(len(names)) if i not in ex]
    if rest:
        _close(b[:, rest], a[:, rest])


def test_energy_and_mzcr():
    _check(os.path.join(HERE, "configs", "lld_mix.conf"), None,
           ("pcm_RMSenergy", "pcm_LOGenergy", "pcm_zcr", "pcm_mcr", "pcm_absmax", "pcm_max", "pcm_min", "pcm_dc"))


def test_jitter():
    _check(os.path.join(HERE, "configs", "pitch_variants.conf"), {"O": "x.htk"}, ())


def test_formant():
    _check(os.path.join(HERE, "configs", "formant_chain.conf"), None, ("formant",))


def test_intensity_and_lpc_lsp():
    if not os.path.exists(EMOBASE):
        pytest.skip("reference configuration files not built (make -C oracle ref)")
    _check(EMOBASE, {"lldcsvoutput": "x.csv"}, ("pcm_intensity", "pcm_loudness", "lspFreq", "pcm_zcr"))


def test_float_input_runs_the_float_lld_kernel_instance():
    from opensmile_b200 import Plan, components_mfcc12_0_d_a
    x = mixed_pcm(16000, SR, seed=3).astype(np.float32) / np.float32(32767)
    plan = Plan(components_mfcc12_0_d_a(float(SR), 1, pcm_format=1), "lld", device=0)
    plan.run_host(x, np.array([0, x.size], np.int64))
    assert plan.last_lld_launch().kernel.startswith("lld_kernel_f32<")
