"""Restatement of a centred cFramer level and of the cVectorPreemphasis level behind it, as the device kernels compute them
(lld_common.cuh stage_padded_tile, frame_reader.cuh), for the tests.  Frame t holds the samples t * step - c ... t * step - c +
size - 1 of its utterance; positions before 0 hold sample 0 (core/dataMemoryLevel.cpp:1651-1697).  Conversion
smileutil/smileUtil.c:2520-2534 ((sum_c (float)x_c) / nChan) / 32767, pre-emphasis dspcore/vectorPreemphasis.cpp:89-108 (de = 0):
(1 - k) x[0] for the first sample of a frame, x[n] - k x[n-1] after it, float arithmetic with separate roundings."""
import numpy as np

f32 = np.float32


def samples(pcm):
    """int16 [n] or [n, nChan] -> the mono float32 wave level"""
    x = np.asarray(pcm)
    if x.ndim == 1:
        return x.astype(f32) / f32(32767)
    s = x[:, 0].astype(f32)
    for c in range(1, x.shape[1]):
        s = s + x[:, c].astype(f32)
    return (s / f32(x.shape[1])) / f32(32767)


def frames(pcm, size, step, centre, n_frames=None):
    """[T, size] float32: the cFramer level (noPostEOIprocessing = 1: complete frames only)"""
    x = samples(pcm)
    L = x.shape[0]
    T = (L + centre - size) // step + 1 if L + centre >= size else 0
    if n_frames is not None:
        T = min(T, n_frames)
    idx = np.arange(T)[:, None] * step - centre + np.arange(size)[None, :]
    return x[np.maximum(idx, 0)]


def preemphasis(fr, k=0.97):
    k32 = f32(k)
    y = np.empty_like(fr)
    y[:, 0] = (f32(1) - k32) * fr[:, 0]
    y[:, 1:] = fr[:, 1:] - k32 * fr[:, :-1]
    return y
