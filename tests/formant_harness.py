"""Host build of the formant and harmonics kernels' arithmetic (tests/native/formant_host.cpp = opensmile_b200/csrc/
formant_math.cuh + harmonics_math.cuh + the product's table builder tables.cpp, compiled with g++): test infrastructure shared
by the CPU and GPU tests."""
import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_L = None


def lib():
    global _L
    if _L is None:
        so = "/tmp/osm_formant_host_%d.so" % os.getuid()
        srcs = [os.path.join(ROOT, "tests", "native", "formant_host.cpp"), os.path.join(ROOT, "opensmile_b200", "csrc", "tables.cpp")]
        cuda_inc = "/usr/local/cuda/include"
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-I" + cuda_inc, "-o", so] + srcs)
        _L = C.CDLL(so)
        _L.fmh_lpc.restype = C.c_float
    return _L


def _fp(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def lpc(x, p):
    a = np.zeros(p, np.float32)
    x = np.ascontiguousarray(x, np.float32)
    lib().fmh_lpc(_fp(x), x.size, p, _fp(a))
    return a


def formants(a, T, n_formants, min_f, max_f):
    a = np.ascontiguousarray(a, np.float32)
    f, b = np.zeros(n_formants, np.float32), np.zeros(n_formants, np.float32)
    lib().fmh_formants(_fp(a), a.size, C.c_double(T), n_formants, C.c_double(min_f), C.c_double(max_f), _fp(f), _fp(b))
    return np.concatenate([f, b])


def roots(c):
    c = np.ascontiguousarray(c, np.float64)
    zr, zi = np.zeros(16), np.zeros(16)
    dp = lambda v: v.ctypes.data_as(C.POINTER(C.c_double))
    it = lib().fmh_roots(dp(c), c.size, dp(zr), dp(zi))
    return zr[:c.size] + 1j * zi[:c.size], it


def resample(xw, sample_rate, nfft, frame_size_sec, target_fs, p=11, n_formants=5, zero_pad_symmetric=1):
    """xw [T, N] windowed frames -> (res [T, I], base period of the cLpc level) with the product's table"""
    xw = np.ascontiguousarray(xw, np.float32)
    T, N = xw.shape
    per = C.c_double()
    I = lib().fmh_resample(C.c_double(sample_rate), N, nfft, C.c_double(frame_size_sec), zero_pad_symmetric, C.c_double(target_fs),
                           p, n_formants, None, 0, None, C.byref(per))
    assert I > 0
    res = np.zeros((T, I), np.float32)
    lib().fmh_resample(C.c_double(sample_rate), N, nfft, C.c_double(frame_size_sec), zero_pad_symmetric, C.c_double(target_fs),
                       p, n_formants, _fp(xw), T, _fp(res), None)
    return res, per.value


def windowed_frames(pcm, sample_rate=16000.0, size_sec=0.020, step_sec=0.010, win="ham"):
    """the cWindower level of a mono int16 signal (float product with the float-cast window, dspcore/windower.cpp:226);
    window table and PCM scaling from the oracle (tests only)"""
    from oracle import oracle
    fe = oracle.frontend(sample_rate, size_sec, step_sec, win=win, zero_pad_symmetric=1)
    N, H, nfft, T = oracle.geometry(fe, len(pcm))
    OL = oracle.lib()
    pcm = np.ascontiguousarray(pcm, np.int16)
    x = np.zeros(len(pcm), np.float32)
    OL.osm_or_pcm16_to_float(pcm.ctypes.data_as(C.POINTER(C.c_int16)), C.c_long(len(pcm)), C.c_int(1), oracle._fp(x))
    w = np.zeros(N, np.float64)
    OL.osm_or_window_table(C.c_int(fe.win_func), C.c_long(N), C.c_double(fe.win_sigma), C.c_double(fe.win_gain),
                           w.ctypes.data_as(C.POINTER(C.c_double)))
    wf = w.astype(np.float32)
    xw = np.stack([x[t * H:t * H + N] * wf for t in range(max(T, 0))]).astype(np.float32) if T > 0 else np.zeros((0, N), np.float32)
    return xw, nfft


def formant_chain(pcm, sample_rate=16000.0, target_fs=11000.0, p=11, n_formants=5, min_f=50.0, max_f=5450.0):
    """PCM -> [T, 2 * n_formants] through the statements formant_kernel executes (20 ms Hamming frames, 10 ms step)"""
    xw, nfft = windowed_frames(pcm, sample_rate)
    res, per = resample(xw, sample_rate, nfft, 0.020, target_fs, p, n_formants)
    return np.stack([formants(lpc(x, p), per, n_formants, min_f, max_f) for x in res]) if len(res) else np.zeros((0, 2 * n_formants), np.float32)


def _ip(a):
    return a.ctypes.data_as(C.POINTER(C.c_int))


def formant_path(sample_rate, N, nfft, frame_size_sec, zero_pad_symmetric, target_fs, p, n_formants):
    """the path formant_kernel takes: dict(ref_order, gathered, k_half, pad_left, n_res, n_res_pad, fpw, smem), or None where
    the graph pass refuses the options"""
    info = np.zeros(8, np.int32)
    if lib().fmh_formant_path(C.c_double(sample_rate), N, nfft, C.c_double(frame_size_sec), zero_pad_symmetric, C.c_double(target_fs),
                              p, n_formants, _ip(info)) < 0:
        return None
    return dict(zip(("ref_order", "gathered", "k_half", "pad_left", "n_res", "n_res_pad", "fpw", "smem"), (int(v) for v in info)))


def formant_smem(ref_order, N, n_res_pad):
    """(shared memory of formant_kernel, the limit of the graph pass) in bytes"""
    L = lib()
    L.fmh_formant_smem.restype = L.fmh_formant_smem_limit.restype = C.c_long
    return int(L.fmh_formant_smem(int(ref_order), N, n_res_pad)), int(L.fmh_formant_smem_limit())


def window(win_func, N, sigma=0.4, gain=1.0):
    """the product's window table (tables.cpp build_window)"""
    w = np.zeros(N, np.float32)
    lib().fmh_window(win_func, N, C.c_double(sigma), C.c_double(gain), _fp(w))
    return w


def wave_level(pcm, n_chan=1):
    """the mono float samples formant_kernel reads (frame_reader.cuh td_pcm): float32 PCM as is; int16 mixed down as
    ((float) x0 + (float) x1) * 0.5f / 32767 (one channel: x / 32767)"""
    if pcm.dtype == np.float32:
        return np.ascontiguousarray(pcm)
    x = pcm.reshape(-1, n_chan).astype(np.float32)
    s = x[:, 0]
    for c in range(1, n_chan):
        s = (s + x[:, c]).astype(np.float32)
    if n_chan == 2:
        s = (s * np.float32(0.5)).astype(np.float32)
    elif n_chan > 2:
        s = (s / np.float32(n_chan)).astype(np.float32)
    return (s / np.float32(32767.0)).astype(np.float32)


def formant_rows(x, N, S, T, win, sample_rate, nfft, frame_size_sec, zero_pad_symmetric, target_fs, p, n_formants, min_f, max_f,
                 save_nvalid, save_formants, save_bandwidths, taps=False, win_offset=0.0):
    """mono float samples x -> the cFormantLpc rows [T, nOut] of formant_kernel's statements (fmh_formant_rows); with taps,
    also the resampled frames [T, I] and the LPC coefficients [T, p]"""
    x = np.ascontiguousarray(x, np.float32)
    win = np.ascontiguousarray(win, np.float32)
    info = formant_path(sample_rate, N, nfft, frame_size_sec, zero_pad_symmetric, target_fs, p, n_formants)
    assert info is not None
    nF = min(n_formants, p - 1) if n_formants > 0 else p - 1
    n_out = int(save_nvalid) + (nF if save_formants else 0) + (nF if save_bandwidths else 0)
    out = np.zeros((T, n_out), np.float32)
    res = np.zeros((T, info["n_res"]), np.float32) if taps else None
    a = np.zeros((T, p), np.float32) if taps else None
    if T > 0:
        assert x.size >= (T - 1) * S + N
        n = lib().fmh_formant_rows(_fp(x), N, S, T, _fp(win), C.c_float(win_offset), C.c_double(sample_rate), nfft,
                                   C.c_double(frame_size_sec), zero_pad_symmetric, C.c_double(target_fs), p, n_formants,
                                   C.c_double(min_f), C.c_double(max_f), int(save_nvalid), int(save_formants), int(save_bandwidths),
                                   _fp(out), _fp(res) if taps else None, _fp(a) if taps else None)
        assert n == n_out, (n, n_out)
    return (out, res, a) if taps else out


def harmonics_rows(F0, formants, mag, bin_hz, n_harm, diffs, fa, floor_unvoiced, hnr):
    """fmh_harmonics over rows: F0 [T], formants [T, nFmt], mag [T, nb] -> [T, nOut]; fa = (start, end), end < start: none"""
    F0 = np.ascontiguousarray(F0, np.float32)
    T = F0.size
    fm_ = np.ascontiguousarray(formants, np.float32).reshape(T, -1)
    mag = np.ascontiguousarray(mag, np.float32)
    d = np.ascontiguousarray(np.array(diffs, np.int32).reshape(-1))
    n_out = int(bool(hnr)) + len(diffs) + max(fa[1] - fa[0] + 1, 0)
    out = np.zeros((T, n_out), np.float32)
    if T:
        n = lib().fmh_harmonics_rows(T, _fp(F0), _fp(fm_), fm_.shape[1], _fp(mag), mag.shape[1], C.c_double(bin_hz), n_harm, len(diffs),
                                     _ip(d) if d.size else None, fa[0], fa[1], C.c_float(floor_unvoiced), 1 if hnr else 0, _fp(out))
        assert n == n_out
    return out


def harmonic_shortcut_fails(F0, nb, bin_hz, n_harm):
    """first harmonic whose closed-form predecessor check fails in harmonics_kernel (-1: the shortcut holds)"""
    return lib().fmh_harmonic_shortcut_fails(C.c_float(F0), nb, C.c_double(bin_hz), n_harm)


def harmonics(F0, formants, mag, bin_hz, n_harm=100, diffs=((-1, 1, -1, 2), (-1, 1, 3, -1)), fa=(1, 3), floor_unvoiced=-201.0, hnr=True):
    """one frame of cHarmonics -> [HNRdBACF] + differences + formant amplitudes (GeMAPS switch set by default)"""
    mag = np.ascontiguousarray(mag, np.float32)
    fm = np.ascontiguousarray(formants, np.float32)
    d = np.ascontiguousarray(np.array(diffs, np.int32).reshape(-1))
    out = np.zeros(1 + len(diffs) + fa[1] - fa[0] + 1, np.float32)
    n = lib().fmh_harmonics(C.c_float(F0), _fp(fm), fm.size, _fp(mag), mag.size, C.c_double(bin_hz), n_harm, len(diffs),
                            d.ctypes.data_as(C.POINTER(C.c_int)), fa[0], fa[1], C.c_float(floor_unvoiced), 1 if hnr else 0, _fp(out))
    return out[:n]
