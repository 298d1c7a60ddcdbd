"""The shipped config/emobase/emobase.conf without a GPU: stand-alone cLpc (method acf) on the pre-emphasised 25 ms frames,
cLsp on it, and the cAcf cepstrum with oldCompatCepstrum = 1 in front of cPitchACF.
  * the restatement tests/native/emobase_oracle.c (tests/emobase_oracle.py) against level taps of the UNMODIFIED reference
    (tests/configs/emobase_taps.conf, scripts/make_golden_emobase.py -> tests/golden/emobase_goldens.npz): LPC and LSP
    bit-identical from the PCM, the compat cepstrum within 3e-7 of its scale, F0 / F0env equal, voiceProb within 1e-6;
  * the host build of the kernel's LSP statements (tests/native/lsp_host.cpp) bit-identical to that restatement, including the frames
    where cLsp retries with the 0.05 grid and zero-fills;
  * the graph: the reference's 988 summary / 52 LLD names in order, row counts, refusals by name."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from opensmile_b200 import capi
from opensmile_b200.session import Session, SessionError
from opensmile_b200.synth import mixed_pcm, voiced_pcm
import emobase_oracle as eo
from oracle import oracle

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
G = np.load(os.path.join(HERE, "golden", "emobase_goldens.npz"))
REC = np.load(os.path.join(HERE, "golden", "egemaps_recordings.npz"))
REFCONF = os.path.join(ROOT, "oracle", "_ref", "config")
EMOBASE = os.path.join(REFCONF, "emobase", "emobase.conf")
needs_conf = pytest.mark.skipif(not os.path.exists(EMOBASE), reason="reference configuration files not built (make -C oracle ref)")


def signals():
    return {"rec": (REC["pcm_opensmile_44k1"], 44100), "v": (voiced_pcm(32000, 16000, seed=7), 16000),
            "m": (mixed_pcm(40000, 16000, seed=5), 16000), "x": (G["pcm_x"], 16000)}


def lpc_frontend(sr):
    return oracle.frontend(sr, 0.025, 0.010, win="ham", preemph=0.97)     # emobase.conf [fr25] + [pe]


@pytest.mark.parametrize("key", ["rec", "v", "m", "x"])
def test_oracle_lpc_lsp_bit_identical_to_the_reference(key):
    pcm, sr = signals()[key]
    a, g, s, roots1 = eo.lpc_frames(pcm, sr, 8)
    assert np.array_equal(a, G["lpc_" + key])
    assert np.array_equal(s, G["lsp_" + key])
    s2, r2 = eo.lsp(G["lpc_" + key])                 # cLsp alone on the reference's own cLpc level
    assert np.array_equal(s2, G["lsp_" + key]) and np.array_equal(r2, roots1)


def test_the_goldens_pin_the_retry_and_zero_fill_paths():
    _, roots1 = eo.lsp(G["lpc_x"])
    zero = (G["lsp_x"] == 0).any(axis=1)
    assert ((roots1 != 8) & ~zero).sum() >= 1            # the 0.2 grid missed roots, the 0.05 grid found all
    assert ((roots1 != 8) & zero).sum() >= 1             # the 0.05 grid missed roots as well: zeros from the last root on


def test_oracle_compat_cepstrum_and_pitch():
    _, cep = eo.acf_pitch(mixed_pcm(40000, 16000, seed=5), 16000)
    ref = G["cep_m"]
    assert cep.shape == ref.shape
    scale = np.abs(ref).max(axis=1, keepdims=True) + 1e-30
    assert (np.abs(cep - ref) / scale).max() < 3e-7
    for key in ("m", "rec", "v", "x"):
        pcm, sr = signals()[key]
        got, _ = eo.acf_pitch(pcm, sr)
        ref = G["pitch_" + key]
        # F0 / F0env are lag decisions: equal; voiceProb is a ratio of ACF values (the oracle's ACF is an exact cosine sum,
        # the reference's a float FFT): within 1e-6
        assert np.array_equal(got[:, 1:], ref[:, 1:]), key
        assert np.abs(got[:, 0] - ref[:, 0]).max() < 1e-6, key


_HOST = None


def _host():
    global _HOST
    if _HOST is None:
        so = "/tmp/osm_lsp_host_%d.so" % os.getuid()
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", so,
                               os.path.join(HERE, "native", "lsp_host.cpp")])
        _HOST = C.CDLL(so)
        _HOST.lsph_lpc.restype = C.c_float
    return _HOST


def _fp(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


@pytest.mark.parametrize("key", ["rec", "v", "m", "x"])
def test_kernel_statements_bit_identical_to_the_oracle(key):
    L = _host()
    ref, roots1 = eo.lsp(G["lpc_" + key])
    for t, a in enumerate(np.ascontiguousarray(G["lpc_" + key])):
        got = np.zeros(8, np.float32)
        L.lsph_lsp(_fp(a), 8, _fp(got))
        assert np.array_equal(got, ref[t]), (key, t)
        first = np.zeros(8, np.float32)
        assert L.lsph_search(_fp(a), 8, _fp(first), C.c_float(0.2)) == roots1[t]
    pcm, sr = signals()[key]
    fe = lpc_frontend(sr)
    a_or, g_or, _, _ = eo.lpc_frames(pcm, sr, 8)
    x = pcm.astype(np.float32) / np.float32(32767.0)
    N, H, _, T = oracle.geometry(fe, len(pcm))
    k = np.float32(0.97)
    for t in range(0, T, 7):
        f = x[t * H:t * H + N]
        y = np.empty(N, np.float32)
        y[0] = (np.float32(1) - k) * f[0]
        y[1:] = f[1:] - k * f[:-1]
        a = np.zeros(8, np.float32)
        g = L.lsph_lpc(_fp(y), N, 8, _fp(a))
        assert np.array_equal(a, a_or[t]) and np.float32(g) == g_or[t], (key, t)


@needs_conf
def test_shipped_emobase_names_and_row_counts():
    s = Session(EMOBASE, {"csvoutput": "x.csv"}, device=-1)
    assert s.element_names() == [str(x) for x in G["names_func"]]
    s.close()
    s = Session(EMOBASE, {"lldcsvoutput": "x.csv"}, device=-1)
    assert s.element_names(44100.0) == [str(x) for x in G["names_lld"]]
    for key, (pcm, sr) in signals().items():
        fo = s.frame_offsets(np.array([0, len(pcm)], np.int64), float(sr))
        assert fo[1] - fo[0] == G["lld_" + key].shape[0], key
    s.close()


@needs_conf
def test_taps_names(tmp_path):
    path = tmp_path / "taps.conf"
    path.write_text(open(os.path.join(HERE, "configs", "emobase_taps.conf")).read().replace("REFCONF", REFCONF))
    assert Session(str(path), output_level="lpc", device=-1).element_names() == ["lpcCoeff[%d]" % i for i in range(8)]
    assert Session(str(path), output_level="lsp", device=-1).element_names() == ["lspFreq[%d]" % i for i in range(8)]


LPC_GRAPH = """
[componentInstances:cComponentManager]
instance[dataMemory].type=cDataMemory
instance[waveIn].type=cWaveSource
instance[fr25].type=cFramer
instance[pe].type=cVectorPreemphasis
instance[lpc].type=cLpc
instance[lsp].type=cLsp
[waveIn:cWaveSource]
writer.dmLevel=wave
filename=in.wav
monoMixdown = 1
[fr25:cFramer]
reader.dmLevel=wave
writer.dmLevel=frames
frameSize = 0.025
frameStep = 0.010
frameCenterSpecial = left
[pe:cVectorPreemphasis]
reader.dmLevel=frames
writer.dmLevel=framespe
k=0.97
[lpc:cLpc]
reader.dmLevel=framespe
writer.dmLevel=lpc
method = acf
p = 8
saveLPCoeff = 1
lpGain = 0
[lsp:cLsp]
reader.dmLevel=lpc
writer.dmLevel=lsp
processArrayFields = 0
"""


def _open(tmp_path, text, level):
    p = tmp_path / "g.conf"
    p.write_text(text)
    return Session(str(p), output_level=level, device=-1)


def test_lpc_lsp_graph_names_and_refusals(tmp_path):
    assert _open(tmp_path, LPC_GRAPH, "lsp").element_names() == ["lspFreq[%d]" % i for i in range(8)]
    assert _open(tmp_path, LPC_GRAPH.replace("lpGain = 0", "lpGain = 1"), "lpc").element_names() == \
        ["lpcCoeff[%d]" % i for i in range(8)] + ["lpGain"]
    assert _open(tmp_path, LPC_GRAPH.replace("p = 8", "p = 12"), "lpc").element_names() == ["lpcCoeff[%d]" % i for i in range(12)]
    for old, new, level, needle in (
            ("method = acf", "method = burg", "lsp", "method=acf"),
            ("lpGain = 0", "lpGain = 0\nsaveRefCoeff = 1", "lpc", "saveRefCoeff"),
            ("lpGain = 0", "lpGain = 0\nresidual = 1", "lpc", "residual"),
            ("lpGain = 0", "lpGain = 0\nforwardFilter = 1", "lpc", "forwardFilter"),
            ("lpGain = 0", "lpGain = 0\nlpSpectrum = 1", "lpc", "lpSpectrum"),
            ("p = 8", "p = 17", "lpc", "1..16"),
            ("lpGain = 0", "lpGain = 1", "lsp", "Ndst < Nsrc"),
            ("saveLPCoeff = 1", "saveLPCoeff = 0\nlpGain = 1", "lsp", "lpcCoeff"),
            ("reader.dmLevel=lpc", "reader.dmLevel=framespe", "lsp", "lpcCoeff"),
            ("processArrayFields = 0", "processArrayFields = 1", "lsp", "processArrayFields")):
        assert old in LPC_GRAPH
        with pytest.raises(SessionError) as e:
            _open(tmp_path, LPC_GRAPH.replace(old, new, 1), level)
        assert needle in str(e.value), (new, str(e.value))
    assert e.value.status == capi.ERR_UNSUPPORTED
