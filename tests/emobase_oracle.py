"""ctypes front of tests/native/emobase_oracle.c -- the restatement of the emobase pieces that the general oracle does not cover
(stand-alone cLpc, cLsp, the oldCompatCepstrum cAcf in front of cPitchACF).  The wave level as floats, the window table and the
cFFTmagphase level come from the general oracle (oracle/osm_oracle.c) unchanged.  Test infrastructure shared by the CPU and GPU
tests."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from oracle import oracle

HERE = os.path.dirname(os.path.abspath(__file__))
_L = None


def lib():
    global _L
    if _L is None:
        so = os.path.join(tempfile.mkdtemp(prefix="osm_emobase_oracle_"), "emobase_oracle.so")
        subprocess.check_call(["gcc", "-O2", "-std=c99", "-ffp-contract=off", "-shared", "-fPIC", "-o", so,
                               os.path.join(HERE, "native", "emobase_oracle.c"), "-lm"])
        _L = C.CDLL(so)
        _L.emo_lpc_frames.restype = C.c_long
        _L.emo_acf_pitch.restype = C.c_long
        _L.emo_lsp.restype = C.c_int
    return _L


def _fp(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def _wave(pcm):
    pcm = np.ascontiguousarray(pcm, np.int16)
    x = np.zeros(len(pcm), np.float32)
    oracle.lib().osm_or_pcm16_to_float(pcm.ctypes.data_as(C.POINTER(C.c_int16)), C.c_long(len(pcm)), C.c_int(1), _fp(x))
    return x


def lpc_frames(pcm, sample_rate, p=8, size_sec=0.025, step_sec=0.010, k=0.97):
    """cLpc (acf) on the pre-emphasised 25 ms frames + cLsp: (lpc [T, p], gain [T], lsp [T, p], roots of the 0.2 grid [T])"""
    fe = oracle.frontend(sample_rate, size_sec, step_sec, win="ham", preemph=k)
    N, H, _, T = oracle.geometry(fe, len(pcm))
    T = max(T, 0)
    a, g, s, r = np.zeros((T, p), np.float32), np.zeros(T, np.float32), np.zeros((T, p), np.float32), np.zeros(T, np.int32)
    if T:
        x = _wave(pcm)
        n = lib().emo_lpc_frames(_fp(x), C.c_long(len(x)), C.c_long(N), C.c_long(H), C.c_float(k), C.c_int(p),
                                 _fp(a), _fp(g), _fp(s), r.ctypes.data_as(C.POINTER(C.c_int)))
        assert n == T
    return a, g, s, r


def lsp(a):
    """cLsp on rows of LPC coefficients: (lsp [T, p], roots of the 0.2 grid [T])"""
    a = np.ascontiguousarray(np.atleast_2d(a), np.float32)
    out, roots = np.zeros_like(a), np.zeros(a.shape[0], np.int32)
    for t in range(a.shape[0]):
        roots[t] = lib().emo_lsp(_fp(a[t]), C.c_int(a.shape[1]), _fp(out[t]))
    return out, roots


def acf_pitch(pcm, sample_rate, max_pitch=500.0, voicing_cutoff=0.55):
    """emobase.conf's [fr40] -> [w40] (Hamming) -> [fft40] (zeroPadSymmetric = 0) -> [fftmagphase40] -> [acf40] + [cepstrum40]
    (oldCompatCepstrum) -> [pitchACF]: (pitch [T, 3] = voiceProb, F0, F0env ; cepstrum level [T, nfft / 2])"""
    fe = oracle.frontend(sample_rate, 0.040, 0.010, win="ham", zero_pad_symmetric=0)
    N, H, nfft, T = oracle.geometry(fe, len(pcm))
    T = max(T, 0)
    nb = nfft // 2 + 1
    OL = oracle.lib()
    x = _wave(pcm)
    w = np.zeros(N, np.float64)
    OL.osm_or_window_table(C.c_int(fe.win_func), C.c_long(N), C.c_double(fe.win_sigma), C.c_double(fe.win_gain),
                           w.ctypes.data_as(C.POINTER(C.c_double)))
    mag = np.zeros((T, nb), np.float32)
    for t in range(T):
        fr = np.ascontiguousarray(x[t * H:t * H + N])
        OL.osm_or_frame_to_mag(C.byref(fe), _fp(fr), C.c_long(N), C.c_long(nfft), w.ctypes.data_as(C.POINTER(C.c_double)),
                               None, _fp(mag[t]))
    OL.osm_or_fft_frame_size_sec.restype = C.c_double
    fs_sec = OL.osm_or_fft_frame_size_sec(C.byref(fe))
    out, cep = np.zeros((T, 3), np.float32), np.zeros((T, nb - 1), np.float32)
    if T:
        lib().emo_acf_pitch(_fp(mag), C.c_long(T), C.c_long(nb), C.c_float(fs_sec), C.c_double(max_pitch), C.c_double(voicing_cutoff),
                            _fp(out), _fp(cep))
    return out, cep
