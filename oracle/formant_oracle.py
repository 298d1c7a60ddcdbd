"""CPU restatement (numpy) of the formant chain of the GeMAPS graphs (SURVEY.md 8f-2):
cTransformFFT output -> cSpecResample -> cLpc (acf) -> cFormantLpc.

TEST INFRASTRUCTURE ONLY (same rules as oracle/osm_oracle.h): nothing in the product imports it.  Pinned against
the UNMODIFIED reference through level taps (tests/configs/formant_taps.conf, scripts/make_golden_formant.py ->
tests/golden/formant_goldens.npz).  Citations are relative to /root/reference/src.  float32 where the reference
computes in FLOAT_DMEM (sequential accumulation order kept), float64 where it computes in double.  The polynomial
roots come from numpy (LAPACK eigenvalues of the companion matrix) instead of the reference's own QR iteration on
the balanced companion matrix (smileutil/zerosolve.cpp): the same roots to ~1e-12, and cFormantLpc sorts the
resulting formants by frequency, so the order in which a solver returns them does not matter.
"""
import ctypes as C

import numpy as np

from . import oracle

f32 = np.float32


_FFT = None


def ref_fft_available():
    import os
    return os.path.exists(os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "libfftsg.so"))


def _ref_rdft(frames_padded):
    """rdft() of the reference's own FFT source (oracle/_ref/libfftsg.so, built by `make -C oracle ref` from
    src/dspcore/fftsg.c where it lies), forward transform in place on every row, work arrays sized like
    cTransformFFT (dspcore/transformFft.cpp:197-207)"""
    global _FFT
    import os
    if _FFT is None:
        _FFT = C.CDLL(os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "libfftsg.so"))
        _FFT.rdft.argtypes = [C.c_int, C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_int), C.POINTER(C.c_float)]
    a = np.ascontiguousarray(frames_padded, np.float32).copy()
    n = a.shape[1]
    ip = np.zeros(3 + int(np.ceil(np.sqrt(np.float32(n)))), np.int32)
    w = np.zeros(n // 2 + 1, np.float32)
    for row in a:
        _FFT.rdft(n, 1, row.ctypes.data_as(C.POINTER(C.c_float)), ip.ctypes.data_as(C.POINTER(C.c_int)),
                  w.ctypes.data_as(C.POINTER(C.c_float)))
    return a


def fft_frames_exact(pcm, fe, n_chan=1):
    """like fft_frames, but through the reference's FFT: bit-identical to the cTransformFFT level.  Windowing as in
    dspcore/windower.cpp:221-229 (float product with the float-cast double table), zero padding as in
    dspcore/transformFft.cpp:175-196"""
    pcm = np.ascontiguousarray(pcm, dtype=np.int16)
    nS = pcm.size // n_chan
    N, H, nfft, T = oracle.geometry(fe, nS)
    L = oracle.lib()
    x = np.zeros(nS, np.float32)
    L.osm_or_pcm16_to_float(pcm.ctypes.data_as(C.POINTER(C.c_int16)), C.c_long(nS), C.c_int(n_chan), oracle._fp(x))
    win = np.zeros(N, np.float64)
    L.osm_or_window_table(C.c_int(fe.win_func), C.c_long(N), C.c_double(fe.win_sigma), C.c_double(fe.win_gain),
                          win.ctypes.data_as(C.POINTER(C.c_double)))
    wf = win.astype(np.float32)
    pad = (nfft - N) // 2 if fe.zero_pad_symmetric else 0
    z = np.zeros((max(T, 0), nfft), np.float32)
    for t in range(max(T, 0)):
        z[t, pad:pad + N] = (x[t * H:t * H + N] * wf + np.float32(fe.win_offset)).astype(np.float32)
    return _ref_rdft(z)


def fft_frames(pcm, fe, n_chan=1):
    """packed real FFT of every frame (dspcore/transformFft.cpp:165-223, packing dspcore/fftsg.c:104-122) -> [T, nfft]"""
    pcm = np.ascontiguousarray(pcm, dtype=np.int16)
    nS = pcm.size // n_chan
    N, H, nfft, T = oracle.geometry(fe, nS)
    L = oracle.lib()
    x = np.zeros(nS, np.float32)
    L.osm_or_pcm16_to_float(pcm.ctypes.data_as(C.POINTER(C.c_int16)), C.c_long(nS), C.c_int(n_chan), oracle._fp(x))
    win = np.zeros(N, np.float64)
    L.osm_or_window_table(C.c_int(fe.win_func), C.c_long(N), C.c_double(fe.win_sigma), C.c_double(fe.win_gain),
                          win.ctypes.data_as(C.POINTER(C.c_double)))
    out = np.zeros((max(T, 0), nfft), np.float32)
    mag = np.zeros(nfft // 2 + 1, np.float32)
    for t in range(max(T, 0)):
        L.osm_or_frame_to_mag(C.byref(fe), oracle._fp(x[t * H:]), C.c_long(N), C.c_long(nfft),
                              win.ctypes.data_as(C.POINTER(C.c_double)), oracle._fp(out[t]), oracle._fp(mag))
    return out


class SpecResample:
    """cSpecResample (dsp/specResample.cpp:97-185) on a zero-padded FFT level; smileDsp_initIrdft / smileDsp_irdft
    (smileutil/smileUtil.c:1752-1820)"""

    def __init__(self, n_in, sample_rate, target_fs, frame_size_sec, last_frame_size_sec):
        bT = 1.0 / sample_rate
        sr = 1.0 / bT
        ratio = target_fs / sr                                                # :112-114
        self.base_period_out = 1.0 / target_fs                                # :120 (set before the adjustment below)
        fs, lfs = frame_size_sec, last_frame_size_sec
        if fs != lfs and lfs != 0.0 and lfs != bT:                            # :150-160 zero-padded input
            n_out0 = np.round(float(n_in) * ratio * lfs / fs)
            new_ratio = n_out0 / (float(n_in) * (lfs / fs))
            if new_ratio != ratio:
                ratio = new_ratio
            nd = float(n_in) * ratio
        else:
            n_out0 = np.round(float(n_in) * ratio)
            new_ratio = n_out0 / float(n_in)
            if new_ratio != ratio:
                ratio = new_ratio
            nd = n_out0
        self.K, self.I, self.nd = int(n_in), int(n_out0), nd
        k_max = min(self.K, self.I)                                           # antiAlias = 1
        if k_max & 1:
            k_max -= 1
        self.k_max = k_max
        i = np.arange(self.I, dtype=np.float64)[:, None]
        k2 = np.arange(1, k_max // 2, dtype=np.float64)[None, :]              # k = 2, 4, .. k_max-2
        kn = 2.0 * np.pi * (k2 * i) / nd
        self.cos = np.cos(kn).astype(f32)
        self.sin = np.sin(kn).astype(f32)
        self.nyq = np.cos((2.0 * np.pi * ((self.K // 2) * i[:, 0])) / nd).astype(f32) if self.I >= self.K else None

    def __call__(self, a):
        """a = one packed FFT frame [K] float32 -> [I] float32 (float accumulation in the reference's order)"""
        out = np.full(self.I, a[0], f32)
        if self.nyq is not None:
            out = (out + a[1] * self.nyq).astype(f32)
        for j in range(self.cos.shape[1]):
            k = 2 * (j + 1)
            out = (out + a[k] * self.cos[:, j]).astype(f32)
            out = (out + a[k + 1] * self.sin[:, j]).astype(f32)
        return (out / f32(self.K // 2)).astype(f32)


def autocorr(x, lags):
    """smileDsp_autoCorr (smileutil/smileUtil.c:1560-1569): float accumulation over i = lag .. n-1"""
    x = np.asarray(x, f32)
    n = x.size
    out = np.zeros(lags, f32)
    for lag in range(lags):
        acc = f32(0)
        prod = (x[lag:] * x[:n - lag]).astype(f32)
        for v in prod:
            acc = f32(acc + v)
        out[lag] = acc
    return out


def lpc_acf(r, p):
    """smileDsp_calcLpcAcf (smileutil/smileUtil.c:1572-1627): Durbin recursion in float -> (a[p], gain)"""
    a = np.zeros(p + 1, f32)
    if r[0] == 0:
        return a[:p], f32(0)
    e = f32(r[0])
    for m in range(1, p + 1):
        s = f32(f32(1.0) * r[m])
        for i in range(1, m):
            s = f32(s + f32(a[i - 1] * r[m - i]))
        k_m = f32(f32(f32(-1.0) / e) * s)
        a[m - 1] = k_m
        for i in range(1, m // 2 + 1):
            x = a[i - 1]
            a[i - 1] = f32(a[i - 1] + f32(k_m * a[m - i - 1]))
            if i < m // 2 or (m & 1) == 1:
                a[m - i - 1] = f32(a[m - i - 1] + f32(k_m * x))
        e = f32(e * f32(f32(1.0) - f32(k_m * k_m)))
        if e == 0:
            a[m:] = 0
            break
    return a[:p], e


def formants_from_lpc(a, T, n_formants, min_f, max_f):
    """cFormantLpc::processVector, root branch (lld/formantLpc.cpp:255-301) + smileMath_complexIntoUnitCircle
    (smileUtil.c:992-1004) + smileDsp_lpcrootsToFormants (:2019-2054) -> (freq[n], bandwidth[n]) float32"""
    p = len(a)
    poly = np.concatenate([-np.asarray(a, np.float64)[::-1], [1.0]])          # ascending powers, leading 1 (:258-262)
    roots = np.roots(poly[::-1])
    out = np.abs(roots) > 1.0
    roots = np.where(out, 1.0 / np.conj(np.where(out, roots, 1.0)), roots)    # 1 / conj(root)
    sp_pi = T * np.pi
    hi = max_f
    if hi < min_f or hi > 1.0 / T:
        hi = 0.5 / T - min_f
    fc, bc = [], []
    for r in roots:
        if r.imag < 0:
            continue
        f = abs(np.arctan2(r.imag, r.real)) / (2.0 * sp_pi)
        if min_f <= f <= hi:
            fc.append(f)
            bc.append(-np.log(abs(r)) / sp_pi)
            if len(fc) >= n_formants:
                break
    order = np.argsort(np.array(fc), kind="stable") if fc else []
    freq = np.zeros(n_formants, np.float64)
    bw = np.zeros(n_formants, np.float64)
    for j, o in enumerate(order):
        freq[j], bw[j] = fc[o], bc[o]
    return freq.astype(f32), bw.astype(f32)


def autocorr_rows(X, lags):
    """autocorr of every row of X [T, n] (the same float accumulation order per row, rows vectorised)"""
    X = np.asarray(X, f32)
    T, n = X.shape
    out = np.zeros((T, lags), f32)
    for lag in range(lags):
        prod = (X[:, lag:] * X[:, :n - lag]).astype(f32)
        acc = np.zeros(T, f32)
        for i in range(prod.shape[1]):
            acc = (acc + prod[:, i]).astype(f32)
        out[:, lag] = acc
    return out


def formant_levels(res, base_period, p, n_formants, min_f, max_f, save_nvalid=0, save_formants=1, save_bandwidths=1):
    """cLpc (acf, order p) + cFormantLpc on resampled frames res [T, I] -> (rows [T, nOut], lpc [T, p]).
    nFormants as lld/formantLpc.cpp:160-167 resolves it (above p - 1 or <= 0: p - 1); rows = [nValid] | freq[nF] | bw[nF]
    (:376-392), nValid = the candidates found before the slots ran out"""
    nF = n_formants if 0 < n_formants <= p - 1 else p - 1
    R = autocorr_rows(res, p + 1) if len(res) else np.zeros((0, p + 1), f32)
    n_out = int(bool(save_nvalid)) + (nF if save_formants else 0) + (nF if save_bandwidths else 0)
    rows = np.zeros((len(res), n_out), f32)
    lpcs = np.zeros((len(res), p), f32)
    for t in range(len(res)):
        a, _ = lpc_acf(R[t], p)
        lpcs[t] = a
        f, b = formants_from_lpc(a, base_period, nF, min_f, max_f)
        row = ([f32(np.count_nonzero(f))] if save_nvalid else []) + (list(f) if save_formants else []) + (list(b) if save_bandwidths else [])
        rows[t] = row
    return rows, lpcs


def formant_chain(pcm, sample_rate, frame, step, win, zero_pad_symmetric, target_fs, p, n_formants, min_f, max_f, save_nvalid=0,
                  save_formants=1, save_bandwidths=1, n_chan=1, exact_fft=False, taps=False):
    """cFramer -> cWindower -> cTransformFFT -> cSpecResample (target_fs) -> cLpc (p) -> cFormantLpc from int16 PCM, any geometry
    and option set; exact_fft: the reference's own FFT (needs oracle/_ref/libfftsg.so).  taps: also (res, lpc, base period)"""
    fe = oracle.frontend(float(sample_rate), frame, step, win=win, zero_pad_symmetric=zero_pad_symmetric)
    spec = fft_frames_exact(pcm, fe, n_chan) if exact_fft else fft_frames(pcm, fe, n_chan)
    N, H, nfft, T = oracle.geometry(fe, len(pcm) // n_chan)
    rs = SpecResample(nfft, float(sample_rate), target_fs, oracle.lib().osm_or_fft_frame_size_sec(C.byref(fe)), frame)
    res = np.stack([rs(a) for a in spec]) if T > 0 else np.zeros((0, rs.I), f32)
    rows, lpcs = formant_levels(res, rs.base_period_out, p, n_formants, min_f, max_f, save_nvalid, save_formants, save_bandwidths)
    return (rows, res, lpcs, rs.base_period_out) if taps else rows


def gemaps_formant_chain(pcm, sample_rate=16000.0, taps=False, exact_fft=False, v01a=False):
    """config/gemaps/v01b/GeMAPSv01b_core.lld.conf.inc:43-58,250-286 -> [T, 10] = formantFreqLpc[1..5] | formantBandwidthLpc[1..5];
    exact_fft: the FFT level through the reference's own FFT (bit-identical front end, needs oracle/_ref/libfftsg.so)"""
    # v01a (config/gemaps/v01a/GeMAPSv01a_core.lld.conf.inc): zeroPadSymmetric = 0 on both FFTs, maxF = 5500,
    # useBrokenJitterThresh = 1 -- otherwise the v01b graph
    fe = oracle.frontend(sample_rate, 0.020, 0.010, win="ham", zero_pad_symmetric=0 if v01a else 1)
    spec = fft_frames_exact(pcm, fe) if exact_fft else fft_frames(pcm, fe)
    N, H, nfft, T = oracle.geometry(fe, len(pcm))
    fs_sec = oracle.lib().osm_or_fft_frame_size_sec(C.byref(fe))
    rs = SpecResample(nfft, sample_rate, 11000.0, fs_sec, 0.020)
    res = np.stack([rs(a) for a in spec]) if T > 0 else np.zeros((0, rs.I), f32)
    lpcs = np.zeros((res.shape[0], 11), f32)
    fmt = np.zeros((res.shape[0], 10), f32)
    for t, x in enumerate(res):
        a, _ = lpc_acf(autocorr(x, 12), 11)
        lpcs[t] = a
        f, b = formants_from_lpc(a, rs.base_period_out, 5, 50.0, 5500.0 if v01a else 5450.0)
        fmt[t, :5], fmt[t, 5:] = f, b
    return (fmt, res, lpcs) if taps else fmt


# ------------------------------------------------------------------------------------------------------------
# cHarmonics (lld/harmonics.cpp): harmonic peaks of the 60 ms magnitude spectrum around multiples of F0, their
# log magnitudes relative to the fundamental, harmonic differences (H1-H2, H1-A3), formant amplitudes, HNR from
# the autocorrelation (inverse FFT of the power spectrum).  Restated for the switch set of the GeMAPS graphs
# (config/gemaps/v01b/GeMAPSv01b_core.lld.conf.inc:289-318); `frq` is the bin-frequency axis of the spectrum.

def _is_peak(x, n):                                                          # harmonics.cpp:369-390
    N = len(x)
    if n >= N or n < 0:
        return False
    if n + 1 < N:
        if n > 0:
            return x[n] > x[n - 1] and x[n] > x[n + 1]
        return x[0] > x[1]
    return n > 0 and x[n] > x[n - 1]


def _freq_to_bin(frq, freq, start):                                          # :403-415
    for b in range(start, len(frq)):
        if frq[b] > freq:
            return b - 1 if frq[b] - freq > freq - frq[b - 1] else b
    return 0


def _quad3(x1, y1, x2, y2, x3, y3):                                          # smileutil/smileUtil.c:1009-1034 -> (x, y)
    den = x1 * x1 * x2 + x2 * x2 * x3 + x3 * x3 * x1 - x3 * x3 * x2 - x2 * x2 * x1 - x1 * x1 * x3
    if den != 0.0:
        a = (y1 * x2 + y2 * x3 + y3 * x1 - y3 * x2 - y2 * x1 - y1 * x3) / den
        b = (x1 * x1 * y2 + x2 * x2 * y3 + x3 * x3 * y1 - x3 * x3 * y2 - x2 * x2 * y1 - x1 * x1 * y3) / den
        c = (x1 * x1 * x2 * y3 + x2 * x2 * x3 * y1 + x3 * x3 * x1 * y2 - x3 * x3 * x2 * y1 - x2 * x2 * x1 * y3 - x1 * x1 * x3 * y2) / den
        if a != 0.0:
            x = -b / (2.0 * a)
            return x, c - a * x * x
    if y1 > y2 and y1 > y3:
        return x1, y1
    if y2 > y1 and y2 > y3:
        return x2, y2
    if y3 > y1 and y3 > y2:
        return x3, y3
    return x1, y1


def find_harmonics(pitch, mag, frq, n_harm):
    """findHarmonicPeaks, branch with a frequency axis (:476-545) + postProcessHarmonics (:550-588)
    -> list of dicts (bin, freqInterpolated, magnitude, magnitudeInterpolated, magnitudeLogRelF0)"""
    nb = len(mag)
    pitch = f32(pitch)
    H = []
    last = _freq_to_bin(frq, f32(0.5) * pitch, 1)
    first = _freq_to_bin(frq, f32(0.5) * pitch, last)
    for i in range(n_harm):
        h = dict(bin=-1, fi=f32(0), mag=f32(0), magi=f32(0), lr=f32(-201.0), fe=f32(0))
        cand = _freq_to_bin(frq, f32(f32(i + 1) * pitch), last)
        if cand >= nb:
            H.append(h)
            continue
        peak = -1
        if _is_peak(mag, cand):
            peak = cand
        else:
            cl, cr = cand - 1, cand + 1
            lo = _freq_to_bin(frq, f32((f32(i) + f32(0.5)) * pitch), last)
            hi = _freq_to_bin(frq, f32((f32(i) + f32(1.5)) * pitch), cand)
            while (cl >= lo or cr <= hi) and peak == -1:
                if cr <= hi:
                    if _is_peak(mag, cr):
                        peak = cr
                        break
                    cr += 1
                if cl >= lo:
                    if _is_peak(mag, cl):
                        peak = cl
                        break
                    cl -= 1
        h["fe"] = f32(f32(i + 1) * pitch)
        if first <= peak < nb - 1:
            h["bin"] = peak
            h["mag"] = f32(mag[peak])
            x, y = _quad3(frq[peak - 1], float(mag[peak - 1]), frq[peak], float(mag[peak]), frq[peak + 1], float(mag[peak + 1]))
            h["fi"], h["magi"] = f32(x), f32(y)
        else:
            h["bin"] = cand
        last = cand
        H.append(h)
    # post processing, logRelMagnitude = true
    log_rel = True
    m0 = H[0]["mag"]
    if m0 == 0.0:
        log_rel = False
    else:
        m0 = f32(np.log10(m0))                   # float magnitudeF0 = log10(float)
    H[0]["lr"] = f32(0.0)                        # also when the fundamental has no magnitude (:560)
    for i in range(1, n_harm):
        if log_rel:
            if H[i]["magi"] > 0.0:
                tmp = np.log10(np.float64(H[i]["magi"]))
                v = f32(20.0 * (tmp - np.float64(m0)))
                H[i]["lr"] = v if v >= -200.0 else f32(-200.0)
            else:
                H[i]["lr"] = f32(-200.0)
        else:
            H[i]["lr"] = f32(-201.0)
        if H[i]["bin"] == H[i - 1]["bin"]:
            H[i] = dict(bin=0, fi=f32(0), mag=f32(0), magi=f32(0), lr=f32(-201.0), fe=f32(0))
    return H


def acf_hnr_db(mag, F0, frq):
    """computeAcf (:590-630, inverse FFT of the power spectrum; numpy's FFT instead of Ooura's) +
    getClosestPeak (:632-665) + computeAcfHnr_dB (:690-712)"""
    nb = len(mag)
    N = (nb - 1) * 2
    p = (np.asarray(mag, f32) * np.asarray(mag, f32)).astype(f32)
    spec = np.zeros(N // 2 + 1, np.complex128)
    spec[:] = p[:N // 2 + 1]
    # rdft(N, -1, a): a[j] = R_0/2 .. the Ooura inverse without the 2/N factor: x[j] = a0/2 + sum_k a_k cos + .. + aN/2 cos(pi j)/2
    k = np.arange(1, N // 2)
    j = np.arange(nb)[:, None]
    full = 0.5 * p[0] + 0.5 * p[N // 2] * np.cos(np.pi * j[:, 0]) + (p[k][None, :] * np.cos(2 * np.pi * j * k[None, :] / N)).sum(axis=1)
    acf = (np.abs(full).astype(f32) / f32(nb)).astype(f32)
    fs = frq[-1] * 2.0
    F0 = f32(F0)
    f0bin = int(np.floor(fs / F0)) if F0 > 0.0 else 0                       # freqToAcfBinLin (:393-401)
    ref = 0
    if f0bin > 0:
        ref = _closest_peak(acf, f0bin)
    if ref <= 0:
        return f32(0.0), acf
    hnr = float(acf[0]) - float(acf[ref])
    hnr = 10e10 if hnr == 0.0 else float(acf[ref]) / hnr
    if hnr > 10e10:
        ret = 10.0 * np.log10(10e10)
    elif hnr < 10e-10:
        ret = 10.0 * np.log10(10e-10)
    else:
        ret = 10.0 * np.log10(hnr)
    return f32(ret), acf


def _closest_peak(x, idx):
    N = len(x)
    if _is_peak(x, idx):
        return idx
    o = 1
    while idx - o > 0 or idx + o < N - 1:
        if idx - o > 0 and _is_peak(x, idx - o):
            return idx - o
        if idx + o < N - 1 and _is_peak(x, idx + o):
            return idx + o
        o += 1
    if x[0] > x[idx] and x[N - 1] <= x[idx]:
        return 0
    if x[0] <= x[idx] and x[N - 1] > x[idx]:
        return N - 1
    if x[0] > x[idx] and x[N - 1] > x[idx]:
        return 0 if idx < N // 2 else N - 1
    return idx


def parse_harmonic_differences(diffs, have_formants):
    """harmonicDifferences (lld/harmonics.cpp:84-160): "H<i>" = harmonic i (H0 the fundamental), "A<k>" = the strongest harmonic
    near formant k, "A0" = the fundamental -> (h1formant, h1idx, h2formant, h2idx) per difference, and the highest harmonic
    named.  Differences that name a formant are dropped, all of them, when there is no formant level (:296-300)"""
    out, top, formant = [], 0, False
    for d in diffs:
        parts = []
        for t in d.split("-"):
            k = int(t[1:])
            if t[0] == "H":
                parts += [-1, k]
                top = max(top, k)
            elif k == 0:
                parts += [-1, 0]
            else:
                parts += [k, -1]
                formant = True
        out.append(tuple(parts))
    if formant and not have_formants:
        out = []
    return out, top


def harmonics_row(F0, formant_freq, mag, frq, n_harmonics=100, diffs=("H1-H2", "H1-A3"), fa_start=1, fa_end=3, floor_unvoiced=-201.0,
                  hnr=True, taps=False):
    """cHarmonics::processVector for log-relative outputs (lld/harmonics.cpp:743-900): [HNRdBACF if hnr] | differences |
    formant amplitudes fa_start..fa_end (fa_end = -1: every formant; none without formants or when fa_end < fa_start).
    nHarmonics is raised to one above the highest harmonic a difference names (:212-217).  formant_freq = None: no formant
    level.  taps: also the ACF and its chosen lag (the HNR decision)"""
    have = formant_freq is not None
    fmt = list(formant_freq) if have else []
    d, top = parse_harmonic_differences(diffs, have)
    n_harm = max(n_harmonics, top + 1)
    if have:
        end = len(fmt) if fa_end == -1 else min(fa_end, len(fmt))
        fa_range = range(fa_start, end + 1)
    else:
        fa_range = range(0)
    out = []
    acf, lag = None, 0
    if hnr:
        v, acf, lag = _acf_hnr_tap(mag, F0, frq)
        out.append(v)
    if F0 > 0.0:
        H = find_harmonics(F0, mag, frq, n_harm)
        fa = []
        for f in fmt:
            lo, hi = f32(0.8) * f32(f), f32(1.2) * f32(f)
            best, bm = -1, f32(0.0)
            for h, hh in enumerate(H):
                if lo <= hh["fi"] <= hi and hh["mag"] > bm:
                    best, bm = h, hh["mag"]
            fa.append(best)
        for (h1f, h1i, h2f, h2i) in d:
            if h1f > 0:
                h1i = fa[h1f - 1] if h1f <= len(fa) else -1
            if h2f > 0:
                h2i = fa[h2f - 1] if h2f <= len(fa) else -1
            ok1, ok2 = 0 <= h1i < n_harm, 0 <= h2i < n_harm
            if ok1 and ok2:
                v = f32(H[h1i]["lr"] - H[h2i]["lr"])
            elif ok1:
                v = f32(H[h1i]["lr"] - f32(201.0))
            elif ok2:
                v = f32(-201.0 - np.float64(H[h2i]["lr"]))
            else:
                out.append(f32(0.0))
                continue
            out.append(f32(min(max(v, f32(-201.0)), f32(201.0))))
        for k in fa_range:
            out.append(H[fa[k - 1]]["lr"] if 1 <= k <= len(fa) and fa[k - 1] >= 0 else f32(0.0))
    else:
        out += [f32(0.0)] * len(d) + [f32(floor_unvoiced)] * len(fa_range)
    row = np.array(out, f32)
    return (row, acf, lag) if taps else row


def _acf_hnr_tap(mag, F0, frq):
    """acf_hnr_db with the chosen lag"""
    v, acf = acf_hnr_db(mag, F0, frq)
    fs = frq[-1] * 2.0
    f0bin = int(np.floor(fs / f32(F0))) if F0 > 0.0 else 0
    return v, acf, (_closest_peak(acf, f0bin) if 0 < f0bin < len(acf) else 0)


def harmonics_gemaps(F0, formant_freq, mag, frq, n_harm=100, floor_unvoiced=-201.0):
    """cHarmonics::processVector for the GeMAPS switch set -> [HNRdBACF, H1-H2, H1-A3, F1amp, F2amp, F3amp] (log rel. F0).
    Differences are parsed like the reference: "H1" is element 1 of the harmonics array whose element 0 is the
    fundamental (:98-104), "A3" the strongest harmonic within +-20 % of the third formant (:714-741)."""
    out = []
    hnr, _ = acf_hnr_db(mag, F0, frq)
    out.append(hnr)
    if F0 > 0.0:
        H = find_harmonics(F0, mag, frq, n_harm)
        fa = []
        for f in formant_freq:
            lo, hi = f32(0.8) * f32(f), f32(1.2) * f32(f)
            best, bm = -1, f32(0.0)
            for h, hh in enumerate(H):
                if lo <= hh["fi"] <= hi and hh["mag"] > bm:
                    best, bm = h, hh["mag"]
            fa.append(best)
        for (h1f, h1i, h2f, h2i) in ((-1, 1, -1, 2), (-1, 1, 3, -1)):       # H1-H2, H1-A3
            if h1f > 0:
                h1i = fa[h1f - 1]
            if h2f > 0:
                h2i = fa[h2f - 1]
            ok1, ok2 = 0 <= h1i < n_harm, 0 <= h2i < n_harm
            if ok1 and ok2:
                v = f32(H[h1i]["lr"] - H[h2i]["lr"])
            elif ok1:
                v = f32(H[h1i]["lr"] - f32(201.0))
            elif ok2:
                v = f32(-201.0 - np.float64(H[h2i]["lr"]))
            else:
                out.append(f32(0.0))
                continue
            out.append(f32(min(max(v, f32(-201.0)), f32(201.0))))
        for i in (1, 2, 3):                                                   # formantAmplitudesStart..End, log rel.
            out.append(H[fa[i - 1]]["lr"] if fa[i - 1] >= 0 else f32(0.0))
    else:
        out += [f32(0.0), f32(0.0)] + [f32(floor_unvoiced)] * 3
    return np.array(out, f32)


def gemaps_vq_levels(pcm, sample_rate=16000.0, exact_fft=False, v01a=False):
    """The four voice-quality levels of the shipped GeMAPS graph (config/gemaps/v01b/GeMAPSv01b_core.lld.conf.inc),
    end to end from PCM:
      logPitch  [T60, 3]  F0final, F0finalLog, voicingFinalUnclipped, gated by the 60 ms rms energy (:62-171)
      jitter    [T60, 2]  jitterLocal, shimmerLocalDB (:174-195)
      formants  [T25, 10] formantFreqLpc[1..5] | formantBandwidthLpc[1..5] (:250-286)
      harmonics [T60, 6]  HNRdBACF, H1-H2, H1-A3, F1..F3 amplitude (:289-318; frame t of the three input levels)"""
    fe60 = oracle.frontend(sample_rate, 0.060, 0.010, win="gau", sigma=0.4, zero_pad_symmetric=0 if v01a else 1)
    sc = oracle.SpecScale(25.0, -1.0, 0, 1, 1, 1)
    ps = oracle.PitchShs(1000.0, 55.0, 6, 1, 1, 0, 0, 1, 1, 0.70, 0, 15, 0.85, 1, 0.0)
    vc = oracle.Viterbi(40, 1, 1, 0, 0, 0, 1, 2.0, 10.0, 5.0, 10.0, 4.0, 1.0, 0.0)
    jc = oracle.Jitter(0.10, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0, -100.0, 0, 2, 0.5, 0, 0, 0, 0, 1 if v01a else 0, 0)
    shs = oracle.pitch_shs(pcm, fe60, sc, ps)
    vit = oracle.viterbi(shs, ps, vc)
    e60 = oracle.energy(pcm, fe60, oracle.Energy(0, 1, 0, 0, 1.0, 1.0, 1.0, 0.0, 0.0, 0.0), windowed=1)
    pitch = oracle.valbased_select(e60[:, 0], vit, 0.001)
    jit = oracle.pitch_jitter(pcm, fe60, jc, pitch[:, 0])
    fmt = gemaps_formant_chain(pcm, sample_rate, exact_fft=exact_fft, v01a=v01a)
    # 60 ms magnitude spectrum and its bin axis (dspcore/transformFft.cpp:111-115)
    N, H, nfft, T = oracle.geometry(fe60, len(pcm))
    spec = fft_frames_exact(pcm, fe60) if exact_fft else fft_frames(pcm, fe60)
    mag = np.zeros((spec.shape[0], nfft // 2 + 1), f32)
    mag[:, 0] = np.abs(spec[:, 0])
    mag[:, -1] = np.abs(spec[:, 1])
    re, im = spec[:, 2::2], spec[:, 3::2]
    mag[:, 1:-1] = np.sqrt((re * re + im * im).astype(f32)).astype(f32)
    fs_sec = oracle.lib().osm_or_fft_frame_size_sec(C.byref(fe60))
    frq = np.arange(nfft // 2 + 1, dtype=np.float64) * (1.0 / fs_sec)
    Th = min(pitch.shape[0], fmt.shape[0], mag.shape[0])
    harm = np.stack([harmonics_gemaps(pitch[t, 0], fmt[t, :5], mag[t], frq) for t in range(Th)]) if Th > 0 else np.zeros((0, 6), f32)
    return pitch, jit, fmt, harm


def gemaps_lld(pcm, sample_rate=16000.0, exact_fft=False, v01a=False):
    """Level `lld` of the shipped config/gemaps/v01b/GeMAPSv01b.conf (18 columns, T60 + 1 rows):
      lldsetE_smo: Loudness, alphaRatio, hammarbergIndex, slope0-500, slope500-1500 (sma3)
      lldsetF_smo: F0semitone, jitterLocal, shimmerLocaldB, HNRdBACF, logRelF0-H1-H2, logRelF0-H1-A3, F1 frequency /
                   bandwidth / amplitude, F2 frequency / amplitude, F3 frequency / amplitude (sma3nz)
    cDataSelector picks the elements in the order of its `selected` list (core/dataSelector.cpp:388-470).  The selector
    in front of the second smoother waits for the jitter level, which does not advance during the reference's first
    end-of-input pass: rows V-1 and V of ALL its columns are smoothed with the level padded at row V-1."""
    pitch, jit, fmt, harm = gemaps_vq_levels(pcm, sample_rate, exact_fft, v01a)
    fe60 = oracle.frontend(sample_rate, 0.060, 0.010, win="gau", sigma=0.4, zero_pad_symmetric=1)
    sc = oracle.SpecScale(25.0, -1.0, 0, 1, 1, 1)
    ps = oracle.PitchShs(1000.0, 55.0, 6, 1, 1, 0, 0, 1, 1, 0.70, 0, 15, 0.85, 1, 0.0)
    vc = oracle.Viterbi(40, 1, 1, 0, 0, 0, 1, 2.0, 10.0, 5.0, 10.0, 4.0, 1.0, 0.0)
    _, lag = oracle.viterbi(oracle.pitch_shs(pcm, fe60, sc, ps), ps, vc, with_lag=True)
    T = min(pitch.shape[0], jit.shape[0], harm.shape[0], fmt.shape[0])
    F = np.stack([pitch[:T, 1], jit[:T, 0], jit[:T, 1], harm[:T, 0], harm[:T, 1], harm[:T, 2], fmt[:T, 0], fmt[:T, 5], harm[:T, 3],
                  fmt[:T, 1], harm[:T, 4], fmt[:T, 2], harm[:T, 5]], axis=1).astype(f32)
    Fs = oracle.sma_nz_lagged(F, lag, set(range(F.shape[1])))
    # energy-related part on the 20 ms frames
    fe25 = oracle.Frontend(sample_rate, 0.020, 0.010, 0, 0.0, oracle.WIN["ham"], 0.4, 1.0, 0.0, 1)
    aud = oracle.plp_static(pcm, sample_rate, (fe25, oracle.Melspec(26, 20.0, 8000.0, 1, 0),
                                                oracle.Plp(5, 0, -1, 0, 1, 0, 0, 0, 0, 0, 0, 29.0, 1.0, 22.0, 0.33, 9.3e-10, 0)))
    loud = oracle.ll1(aud)
    spec = oracle.spectral(pcm, fe25, oracle.gemaps_logspectral())
    # cSpectral emits slopes before alphaRatio / hammarbergIndex (lldcore/spectral.cpp:378-584); the selector's order is
    # loudness, alphaRatioDB, hammarbergIndexDB, slope 0-500, slope 500-1500 (GeMAPSv01b_core.lld.conf.inc:177-181)
    E = np.stack([loud, spec[:, 2], spec[:, 3], spec[:, 0], spec[:, 1]], axis=1).astype(f32)
    Es = oracle.sma(E, 3, 0)
    R = min(Es.shape[0], Fs.shape[0])
    return np.concatenate([Es[:R], Fs[:R]], axis=1)


def gemaps_sel_lld(pcm, sample_rate=16000.0):
    """Level `lld` of tests/configs/gemaps_sel.conf: the shipped gemapsv01b_lldsetE (5 columns, sma3) next to a cDataSelector
    over the pitch and jitter / shimmer levels (shimmerLocalDB, F0finalLog, jitterLocal in this order; sma3nz, every column
    lagging with the jitter level).  No FFT-sensitive branch: none of the columns reads the formant chain."""
    fe60 = oracle.frontend(sample_rate, 0.060, 0.010, win="gau", sigma=0.4, zero_pad_symmetric=1)
    sc = oracle.SpecScale(25.0, -1.0, 0, 1, 1, 1)
    ps = oracle.PitchShs(1000.0, 55.0, 6, 1, 1, 0, 0, 1, 1, 0.70, 0, 15, 0.85, 1, 0.0)
    vc = oracle.Viterbi(40, 1, 1, 0, 0, 0, 1, 2.0, 10.0, 5.0, 10.0, 4.0, 1.0, 0.0)
    jc = oracle.Jitter(0.10, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0, -100.0, 0, 2, 0.5, 0, 0, 0, 0, 0, 0)
    vit, lag = oracle.viterbi(oracle.pitch_shs(pcm, fe60, sc, ps), ps, vc, with_lag=True)
    e60 = oracle.energy(pcm, fe60, oracle.Energy(0, 1, 0, 0, 1.0, 1.0, 1.0, 0.0, 0.0, 0.0), windowed=1)
    pitch = oracle.valbased_select(e60[:, 0], vit, 0.001)
    jit = oracle.pitch_jitter(pcm, fe60, jc, pitch[:, 0])
    T = min(pitch.shape[0], jit.shape[0])
    F = np.stack([jit[:T, 1], pitch[:T, 1], jit[:T, 0]], axis=1).astype(f32)
    Fs = oracle.sma_nz_lagged(F, lag, set(range(F.shape[1])))
    fe25 = oracle.Frontend(sample_rate, 0.020, 0.010, 0, 0.0, oracle.WIN["ham"], 0.4, 1.0, 0.0, 1)
    aud = oracle.plp_static(pcm, sample_rate, (fe25, oracle.Melspec(26, 20.0, 8000.0, 1, 0),
                                                oracle.Plp(5, 0, -1, 0, 1, 0, 0, 0, 0, 0, 0, 29.0, 1.0, 22.0, 0.33, 9.3e-10, 0)))
    spec = oracle.spectral(pcm, fe25, oracle.gemaps_logspectral())
    E = np.stack([oracle.ll1(aud), spec[:, 2], spec[:, 3], spec[:, 0], spec[:, 1]], axis=1).astype(f32)
    Es = oracle.sma(E, 3, 0)
    R = min(Es.shape[0], Fs.shape[0])
    return np.concatenate([Es[:R], Fs[:R]], axis=1)


EGEMAPS_LLD_NAMES = (["Loudness_sma3", "alphaRatio_sma3", "hammarbergIndex_sma3", "slope0-500_sma3", "slope500-1500_sma3",
                      "spectralFlux_sma3"] + ["mfcc%d_sma3" % i for i in range(1, 5)]
                     + ["F0semitoneFrom27.5Hz_sma3nz", "jitterLocal_sma3nz", "shimmerLocaldB_sma3nz", "HNRdBACF_sma3nz",
                        "logRelF0-H1-H2_sma3nz", "logRelF0-H1-A3_sma3nz"]
                     + ["F%d%s_sma3nz" % (k, w) for k in (1, 2, 3) for w in ("frequency", "bandwidth", "amplitudeLogRelF0")])


def egemaps_lld(pcm, sample_rate=16000.0, exact_fft=False):
    """Level `lld` of the shipped config/egemaps/v02/eGeMAPSv02.conf -- BASELINE configs[2] -- 25 columns, T60 + 1 rows:
      lldsetE_smo (sma3):   Loudness, alphaRatio, hammarbergIndex, slope0-500, slope500-1500, spectralFlux, mfcc1..4
      lldsetF_smo (sma3nz): F0semitone, jitterLocal, shimmerLocaldB, HNRdBACF, logRelF0-H1-H2, logRelF0-H1-A3,
                            F1 / F2 / F3 frequency, bandwidth, amplitude
    (eGeMAPSv02_core.lld.conf.inc:13-60,79-89 on top of the GeMAPS levels, see gemaps_lld)"""
    pitch, jit, fmt, harm = gemaps_vq_levels(pcm, sample_rate, exact_fft)
    fe60 = oracle.frontend(sample_rate, 0.060, 0.010, win="gau", sigma=0.4, zero_pad_symmetric=1)
    sc = oracle.SpecScale(25.0, -1.0, 0, 1, 1, 1)
    ps = oracle.PitchShs(1000.0, 55.0, 6, 1, 1, 0, 0, 1, 1, 0.70, 0, 15, 0.85, 1, 0.0)
    vc = oracle.Viterbi(40, 1, 1, 0, 0, 0, 1, 2.0, 10.0, 5.0, 10.0, 4.0, 1.0, 0.0)
    _, lag = oracle.viterbi(oracle.pitch_shs(pcm, fe60, sc, ps), ps, vc, with_lag=True)
    T = min(pitch.shape[0], jit.shape[0], harm.shape[0], fmt.shape[0])
    cols = [pitch[:T, 1], jit[:T, 0], jit[:T, 1], harm[:T, 0], harm[:T, 1], harm[:T, 2]]
    for k in range(3):
        cols += [fmt[:T, k], fmt[:T, 5 + k], harm[:T, 3 + k]]
    F = np.stack(cols, axis=1).astype(f32)
    Fs = oracle.sma_nz_lagged(F, lag, set(range(F.shape[1])))
    fe25 = oracle.Frontend(sample_rate, 0.020, 0.010, 0, 0.0, oracle.WIN["ham"], 0.4, 1.0, 0.0, 1)
    aud = oracle.plp_static(pcm, sample_rate, (fe25, oracle.Melspec(26, 20.0, 8000.0, 1, 0),
                                                oracle.Plp(5, 0, -1, 0, 1, 0, 0, 0, 0, 0, 0, 29.0, 1.0, 22.0, 0.33, 9.3e-10, 0)))
    spec = oracle.spectral(pcm, fe25, oracle.gemaps_logspectral())
    flux = oracle.spectral(pcm, fe25, oracle.spectral_cfg(flux=1, centroid=0, maxPos=0, minPos=0, normBandEnergies=1, squareInput=1,
                                                          useLogSpectrum=1, freqRangeLo=0, freqRangeHi=5000, oldSlopeScale=0))
    mf = oracle.mfcc_d_a(pcm, sample_rate, cfg=(fe25, oracle.Melspec(26, 20.0, 8000.0, 1, 1), oracle.Mfcc(1, 4, 22.0, 1e-8, 1)))[:, :4]
    E = np.concatenate([np.stack([oracle.ll1(aud), spec[:, 2], spec[:, 3], spec[:, 0], spec[:, 1], flux[:, 0]], axis=1), mf], axis=1).astype(f32)
    Es = oracle.sma(E, 3, 0)
    R = min(Es.shape[0], Fs.shape[0])
    return np.concatenate([Es[:R], Fs[:R]], axis=1)


def egemaps_v01_lld(pcm, sample_rate=16000.0, exact_fft=False, v01a=False):
    """Level `lld` of the shipped config/egemaps/v01a|v01b/eGeMAPSv01*.conf (23 columns): the ten sma3 columns of eGeMAPS
    (loudness, four log-spectral descriptors, spectral flux, MFCC 1-4) next to the thirteen sma3nz columns of the GeMAPS
    selector (v01a: the GeMAPSv01a switches in the voice-quality branch; the magnitude-based columns do not see
    zeroPadSymmetric)"""
    E = egemaps_lld(pcm, sample_rate, exact_fft)[:, :10]
    F = gemaps_lld(pcm, sample_rate, exact_fft, v01a)[:, 5:]
    R = min(len(E), len(F))
    return np.concatenate([E[:R], F[:R]], axis=1)
