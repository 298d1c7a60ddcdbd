"""Restatement of cTonespec and cChroma on the oracle's magnitude level (numpy, float32 / float64 as the reference casts).

TEST INFRASTRUCTURE ONLY.  Citations relative to the reference's src/:
  lld/tonespec.cpp:147-167   note frequencies          lld/tonespec.cpp:171-367   bin keys, bin counts, filter map
  dsp/dbA.cpp:110-126        dB(A) weights             lld/tonespec.cpp:390-441   per-frame tone values
  lld/chroma.cpp:86-117      chroma fold
The reference is C++: a float argument of pow / log / fabs / ceil / floor / round selects the float overload (powf, logf, ...),
so those calls go to the C library's float functions here (ctypes), the double ones to Python's math (the same libm).
"""
import ctypes as C
import ctypes.util
import math

import numpy as np

from oracle import formant_oracle, oracle

f32 = np.float32
_libm = C.CDLL(ctypes.util.find_library("m"))
_libm.logf.restype = C.c_float
_libm.logf.argtypes = [C.c_float]

FILTERS = {"gau": 0, "tri": 1, "trp": 2, "rec": 3}


def logf(x):
    return f32(_libm.logf(float(x)))


def dba(n, F0):
    """computeDBA (dsp/dbA.cpp:110-126)"""
    out = np.zeros(n, f32)
    curF = f32(0.0)
    for i in range(n):
        cf2 = f32(curF * curF)                        # the compiler's rewrite of powf(x, 2): x * x, one rounding
        tmp = f32(math.pow(12200.0, 2.0) * float(f32(cf2 * cf2))) / ((cf2 + f32(math.pow(20.6, 2.0))) * (cf2 + f32(math.pow(12200.0, 2.0))))
        tmp = f32(tmp / f32(math.sqrt(float(cf2) + math.pow(107.7, 2.0)) * math.sqrt(float(cf2) + math.pow(737.9, 2.0))))
        lg = float(logf(tmp)) if tmp > 0 else -math.inf
        out[i] = f32(math.pow(10.0, (10.0 * lg + 2.0) / 10.0)) if lg != -math.inf else f32(0.0)
        curF = f32(curF + F0)
    return out


def tables(n_octaves=6, first_note=55.0, filter_type="gau", db_a=1, n_bins=2049, frame_size_sec=4096 / 44100.0):
    """(pitchClassFreq [nNotes + 2], binKey [nBins], nbins [nNotes + 2], filterMap [nBins], firstBin, lastBin)"""
    nNotes = n_octaves * 12
    ft = FILTERS[filter_type] if isinstance(filter_type, str) else filter_type
    fn = f32(first_note)
    fn0 = f32(fn / f32(math.pow(2.0, 1.0 / 12.0)))
    pcf = np.zeros(nNotes + 2, f32)
    pcf[0] = fn0
    n = 0.0
    for i in range(1, nNotes + 2):
        n += 1.0
        pcf[i] = f32(fn0 * f32(math.pow(2.0, n / 12.0)))
    F0 = f32(1.0 / frame_size_sec)
    db = dba(n_bins, F0) if db_a else None
    firstBin = int(math.ceil(float(f32(pcf[0] + pcf[1])) / (2.0 * float(F0))))
    lastBin = int(math.floor(float(f32(pcf[nNotes] + pcf[nNotes + 1])) / (2.0 * float(F0))))
    firstBin = max(firstBin, 1)
    lastBin = min(lastBin, n_bins - 1)
    key = np.zeros(n_bins, np.int32)
    cur = 0
    for i in range(n_bins):
        if cur > nNotes:
            cur = nNotes
        fi = f32(f32(i) * F0)
        d0 = abs(f32(pcf[cur] - fi))
        n1 = cur + 1
        d1 = abs(f32(pcf[n1] - fi))
        while d0 > d1:
            if n1 > nNotes:
                break
            d0 = d1
            n1 += 1
            d1 = abs(f32(pcf[n1] - fi))
        cur = n1 - 1
        key[i] = cur
    nb = np.zeros(nNotes + 2, np.int32)
    for i in range(firstBin, lastBin + 1):
        if key[i] >= 0:
            nb[key[i]] += 1
    fm = np.zeros(n_bins, f32)
    if ft != 3:
        for b in range(1, nNotes - 1):
            sf = f32(f32(pcf[b - 1] + pcf[b]) / f32(2.0))
            ef = f32(f32(pcf[b] + pcf[b + 1]) / f32(2.0))
            sb, eb, mb = f32(sf / F0), f32(ef / F0), f32(pcf[b] / F0)
            i0, i1 = int(math.ceil(sb)), int(math.floor(eb))
            im = int(math.floor(float(mb) + 0.5))       # roundf of a positive float: half away from zero (exact in double)
            if i0 > i1:
                continue
            i1 = min(i1, n_bins - 1)
            i0 = min(i0, n_bins - 1)
            i0 = max(i0, 1)
            if ft in (1, 2):
                assert im <= n_bins, "the reference writes past its filter map"
                for i in range(i0, im):
                    v = f32(f32(1.0) - f32(f32(mb - f32(i)) / f32(mb - sb)))
                    fm[i] = f32(2.0) - v if v > 1.0 else v
                for i in range(im, i1 + 1):
                    v = f32(f32(1.0) - f32(f32(f32(i) - mb) / f32(eb - mb)))
                    fm[i] = f32(2.0) - v if v > 1.0 else v
            else:
                for i in range(i0, i1 + 1):
                    dist = float(f32(eb - sb))
                    if dist > 0.0:
                        x = float(i) - float(mb)
                        delta = dist / 15.0
                        fm[i] = f32((10.0 / 4.0) * (1.0 / math.sqrt(2.0 * math.pi)) * math.exp(-0.5 * (1.0 / delta) * (1.0 / delta) * math.pow(x, 2.0)))
    if ft == 2:
        fm = (fm * fm).astype(f32)
    fm[:firstBin] = 0
    fm[lastBin + 1:] = 0
    if db_a:
        fm[firstBin:lastBin + 1] = (fm[firstBin:lastBin + 1] * db[:lastBin + 1 - firstBin]).astype(f32)
    return pcf, key, nb, fm, firstBin, lastBin


def tonespec(mag, n_octaves=6, first_note=55.0, filter_type="gau", use_power=0, db_a=1, frame_size_sec=None):
    """[T, nBins] float32 magnitudes -> [T, nNotes] (lld/tonespec.cpp:403-434)"""
    mag = np.asarray(mag, f32)
    T, nBins = mag.shape
    pcf, key, nb, fm, fb, lb = tables(n_octaves, first_note, filter_type, db_a, nBins, frame_size_sec)
    nNotes = n_octaves * 12
    src = (mag * mag).astype(f32) if use_power else mag
    dst = np.zeros((T, nNotes), f32)
    for i in range(fb, lb + 1):
        k = key[i]
        if 0 < k <= nNotes:
            dst[:, k - 1] = dst[:, k - 1] + (src[:, i] * fm[i]).astype(f32)
    for i in range(nNotes):
        if nb[i + 1] > 0:
            dst[:, i] = dst[:, i] / f32(nb[i + 1])
            if use_power:
                dst[:, i] = np.where(dst[:, i] >= 0, np.sqrt(np.maximum(dst[:, i], 0)), 0).astype(f32)
        else:
            dst[:, i] = 0
    return dst


def chroma(tone, octave_size=12, sil_thresh=0.001):
    """[T, nNotes] -> [T, octaveSize] (lld/chroma.cpp:86-117)"""
    tone = np.asarray(tone, f32)
    T, N = tone.shape
    assert N % octave_size == 0
    no = N // octave_size
    dst = np.zeros((T, octave_size), f32)
    total = np.zeros(T, np.float64)
    sil = np.zeros(T, bool)
    for i in range(octave_size):
        s = np.zeros(T, f32)
        for j in range(no):
            s = (s + tone[:, j * octave_size + i]).astype(f32)
        sil |= s < f32(sil_thresh)
        total += s.astype(np.float64)
        dst[:, i] = s
    ok = (total != 0.0) & ~sil
    out = np.zeros_like(dst)
    out[ok] = (dst[ok] / total[ok].astype(f32)[:, None]).astype(f32)
    return out, sil


CHROMA_FE = dict(frame_size=0.064, frame_step=0.010, win="gau", sigma=0.4)


def magnitudes(pcm, sample_rate, n_chan=1, frame_size=0.064, frame_step=0.010, win="gau", sigma=0.4):
    """the cFFTmagphase level of the chroma front end: [T, nfft/2 + 1] float32, and frameSizeSec after cTransformFFT.  Through the
    reference's own FFT where oracle/_ref/libfftsg.so exists (bit-identical level: the quiet notes of a frame sit at the FFT's
    round-off, which would otherwise dominate their column), else through the oracle's C front end."""
    fe = oracle.frontend(sample_rate, frame_size, frame_step, win=win, sigma=sigma)
    L = oracle.lib()
    L.osm_or_fft_frame_size_sec.restype = C.c_double
    fss = float(L.osm_or_fft_frame_size_sec(C.byref(fe)))
    if formant_oracle.ref_fft_available():
        a = formant_oracle.fft_frames_exact(pcm, fe, n_chan)                     # packed rdft rows (dspcore/fftsg.c)
        n = a.shape[1]
        mag = np.zeros((a.shape[0], n // 2 + 1), f32)                             # dspcore/fftmagphase.cpp:215-221
        mag[:, 0] = np.abs(a[:, 0])
        re, im = a[:, 2::2], a[:, 3::2]
        mag[:, 1:n // 2] = np.sqrt((re * re + im * im).astype(f32))
        mag[:, n // 2] = np.abs(a[:, 1])
        return mag, fss
    pcm = np.ascontiguousarray(pcm, np.int16)
    nS = pcm.size // n_chan
    N, H, nfft, T = oracle.geometry(fe, nS)
    x = np.zeros(nS, f32)
    L.osm_or_pcm16_to_float(pcm.ctypes.data_as(C.POINTER(C.c_int16)), C.c_long(nS), C.c_int(n_chan), oracle._fp(x))
    w = np.zeros(N, np.float64)
    L.osm_or_window_table(C.c_int(fe.win_func), C.c_long(N), C.c_double(sigma), C.c_double(1.0), w.ctypes.data_as(C.POINTER(C.c_double)))
    mag = np.zeros((max(T, 0), nfft // 2 + 1), f32)
    pk = np.zeros(nfft, f32)
    for t in range(max(T, 0)):
        fr = np.ascontiguousarray(x[t * H:t * H + N])
        row = np.zeros(nfft // 2 + 1, f32)
        L.osm_or_frame_to_mag(C.byref(fe), oracle._fp(fr), C.c_long(N), C.c_long(nfft), w.ctypes.data_as(C.POINTER(C.c_double)),
                              oracle._fp(pk), oracle._fp(row))
        mag[t] = row
    return mag, fss


def extract(pcm, sample_rate, n_chan=1, n_octaves=6, first_note=55.0, filter_type="gau", use_power=1, db_a=1, octave_size=12,
            sil_thresh=0.001):
    """tonespec [T, nNotes], chroma [T, octaveSize] and the per-frame silThresh flags of one utterance"""
    mag, fss = magnitudes(pcm, sample_rate, n_chan)
    tone = tonespec(mag, n_octaves, first_note, filter_type, use_power, db_a, fss)
    ch, sil = chroma(tone, octave_size, sil_thresh)
    return tone, ch, sil
