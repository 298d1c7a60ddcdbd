"""Plain restatement of the reference's cCens (src/lld/cens.cpp) in numpy float32 / float64.

cens(chroma, window, winlength, l2norm) maps the rows [T, N] of one utterance's chroma level to its CENS rows [T, N]:
  1. quantise every value against the double constants 0.4 / 0.2 / 0.1 / 0.05 (chromaDiscretise, :139-149): 4 / 3 / 2 / 1 / 0;
  2. out[t][i] = sum_{j=0}^{W-1} q[t-j][i] * (float)win[j], accumulated in float with j ascending; rows before the start are 0
     (the calloc'd ring buffer, :152-187);
  3. l2norm: n = sum_i (double)out[i]^2 in double, dst = out / (float)sqrt(n); n == 0 gives (float)(1.0 / sqrt((float)N)) (:189-207).
downsampleRatio drops no row (dsidx is never incremented, :121,134,178); it only scales the level's period (configureWriter,
:107-114).  The window is smileDsp_winHan / winHam / winBar (smileutil/smileUtil.c:1260-1303) in libm double precision, any
other name falls back to Hanning (:68-80).
"""
import math

import numpy as np


def window(name, W):
    """(float) win[j] of the reference's window builders"""
    NN = float(W)
    w = []
    for n in range(W):
        i = float(n)
        if name.startswith("ham"):
            v = 0.54 - 0.46 * math.cos((2.0 * math.pi * i) / (NN - 1.0)) if W > 1 else float("nan")
        elif name.startswith("bar"):
            v = 2.0 * n / (W - 1) if n < W // 2 else (2.0 * (W - 1 - n) / (W - 1) if W > 1 else float("nan"))
        else:
            v = 0.5 * (1.0 - math.cos((2.0 * math.pi * i) / (NN - 1.0))) if W > 1 else float("nan")
        w.append(v)
    return np.array(w, np.float64).astype(np.float32)


def quantise(x):
    x = np.asarray(x, np.float32).astype(np.float64)
    q = np.zeros(x.shape, np.float32)
    q[x >= 0.05] = 1.0
    q[x >= 0.1] = 2.0
    q[x >= 0.2] = 3.0
    q[x >= 0.4] = 4.0
    return q


def unit_value(N):
    """(FLOAT_DMEM)(1.0 / sqrt((FLOAT_DMEM)N)): the float overload of sqrt, a double division"""
    return np.float32(1.0 / float(np.sqrt(np.float32(N))))


def cens(chroma, window_name="han", winlength=41, l2norm=1):
    x = np.asarray(chroma, np.float32)
    T, N = x.shape
    W = max(int(winlength), 1)
    w = window(window_name, W)
    q = np.concatenate([np.zeros((W - 1, N), np.float32), quantise(x)])
    acc = np.zeros((T, N), np.float32)
    with np.errstate(invalid="ignore"):
        for j in range(W):                                         # j ascending, float products and sums
            acc = (acc + q[W - 1 - j:W - 1 - j + T] * w[j]).astype(np.float32)
    if not l2norm:
        return acc
    n = np.zeros(T, np.float64)
    for i in range(N):                                             # element order, double
        n = n + acc[:, i].astype(np.float64) * acc[:, i].astype(np.float64)
    out = np.empty_like(acc)
    pos = n > 0.0
    out[pos] = acc[pos] / np.sqrt(n[pos]).astype(np.float32)[:, None]
    out[~pos] = unit_value(N)
    return out
