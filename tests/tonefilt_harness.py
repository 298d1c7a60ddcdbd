"""Shared pieces of the cTonefilt tests: the golden cases (scripts/make_golden_tonefilt.py), the literal C restatement of the
reference (tests/native/tonefilt_oracle.c), the host build of the kernel's block statements (tests/native/tonefilt_host.cpp) and
sessions on tests/configs/tonefilt_taps.conf with one level as the output level."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from opensmile_b200 import Session  # noqa: E402
from oracle import chroma_oracle as co  # noqa: E402
import make_golden_tonefilt as mg  # noqa: E402

G = np.load(os.path.join(HERE, "golden", "tonefilt_goldens.npz"))
TAPS = os.path.join(HERE, "configs", "tonefilt_taps.conf")
SHIPPED = os.path.join(ROOT, "oracle", "_ref", "config", "chroma", "chroma_filt.conf")
SIGS = mg.signals()
SINKS = ("tfoutput", "tfhtk", "choutput", "chhtk", "tsoutput", "smahtk", "deoutput", "dehtk")
LEVEL_SINK = {"tonefilt": "tfoutput", "chroma": "choutput", "chroma_sma": "smahtk", "chroma_sma_de": "deoutput"}


def _so(name, src, cc, extra=()):
    so = "/tmp/osm_%s_%d.so" % (name, os.getuid())
    srcp = os.path.join(HERE, "native", src)
    if not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(srcp):
        tmp = "%s.%d.tmp" % (so, os.getpid())
        subprocess.check_call([cc, "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", tmp, srcp] + list(extra))
        os.replace(tmp, so)
    return C.CDLL(so)


def wave_level(pcm, nc):
    """the float wave level: ((sum of channels) / nc) / 32767 in float (smileutil/smileUtil.c:2518-2534), float WAVs / nc"""
    if pcm.dtype == np.float32:
        x = pcm.reshape(-1, nc).astype(np.float32)
        s = x[:, 0].copy()
        for c in range(1, nc):
            s = (s + x[:, c]).astype(np.float32)
        return (s / np.float32(nc)).astype(np.float32)
    x = pcm.reshape(-1, nc).astype(np.float32)
    s = x[:, 0].copy()
    for c in range(1, nc):
        s = (s + x[:, c]).astype(np.float32)
    return ((s / np.float32(nc)).astype(np.float32) / np.float32(32767.0)).astype(np.float32)


def oracle_tf(x, sr, o):
    L = _so("tonefilt_oracle", "tonefilt_oracle.c", "gcc", ["-lm"])
    L.tfo_run.restype = C.c_long
    L.tfo_run.argtypes = [C.c_void_p, C.c_long, C.c_double, C.c_int, C.c_double, C.c_double, C.c_double, C.c_double, C.c_void_p]
    L.tfo_rows.restype = C.c_long
    L.tfo_rows.argtypes = [C.c_long, C.c_double, C.c_double, C.c_void_p]
    x = np.ascontiguousarray(x, np.float32)
    n = max(int(o["nNotes"]), 1)
    rows = L.tfo_rows(x.size, float(sr), float(o["outputPeriod"]), None)
    out = np.zeros((rows, n), np.float32)
    L.tfo_run(x.ctypes.data, x.size, float(sr), int(o["nNotes"]), float(o["firstNote"]), float(o["decayF0"]), float(o["decayFN"]),
              float(o["outputPeriod"]), out.ctypes.data)
    return out


def tables(sr, o):
    """block length and the tables after the reference's clamps (lld/tonefilt.cpp:65-134, 180-189)"""
    dN = min(max(float(o["decayFN"]), 0.0), 1.0)
    d0 = min(max(max(float(o["decayF0"]), dN), 0.0), 1.0)
    first = float(o["firstNote"]) if float(o["firstNote"]) > 0 else 1.0
    n = max(int(o["nNotes"]), 1)
    per = float(o["outputPeriod"]) if float(o["outputPeriod"]) > 0 else 0.1
    T = 1.0 / sr
    P = 1 if per < T else int(np.round(per / T))
    freq = np.array([first * 2.0 ** (k / 12.0) for k in range(n)])
    decay = np.array([dN + (d0 - dN) * (freq[k] - freq[0]) / freq[n - 1] for k in range(n)])
    return P, freq, decay


def host_tf(x, sr, o, seg=0):
    L = _so("tonefilt_host", "tonefilt_host.cpp", "g++")
    L.tfh_run.restype = C.c_long
    L.tfh_run.argtypes = [C.c_void_p, C.c_long, C.c_int, C.c_double, C.c_void_p, C.c_void_p, C.c_int, C.c_long, C.c_void_p]
    P, freq, decay = tables(sr, o)
    x = np.ascontiguousarray(x, np.float32)
    out = np.zeros(((x.size + P - 1) // P, freq.size), np.float32)
    L.tfh_run(x.ctypes.data, x.size, P, float(sr), freq.ctypes.data, decay.ctypes.data, freq.size, seg, out.ctypes.data)
    return out


def host_chroma(t, K, sil):
    L = _so("tonefilt_host", "tonefilt_host.cpp", "g++")
    L.tfh_chroma.argtypes = [C.c_void_p, C.c_long, C.c_int, C.c_int, C.c_float, C.c_void_p]
    t = np.ascontiguousarray(t, np.float32)
    out = np.zeros((t.shape[0], K), np.float32)
    L.tfh_chroma(t.ctypes.data, t.shape[0], t.shape[1], K, float(np.float32(sil)), out.ctypes.data)
    return out


def oracle_case(case):
    sig = mg.CASES[case][0]
    pcm, sr, nc = SIGS[sig]
    o = mg.options(case)
    tf = oracle_tf(wave_level(pcm, nc), sr, o)
    ch = co.chroma(tf, o["octaveSize"], o["silThresh"])[0] if o["nNotes"] > 1 else None
    return tf, ch


def col_err(got, ref):
    scale = np.maximum(np.abs(ref).max(axis=0), 1e-30)
    return float((np.abs(got - ref) / scale).max()) if ref.size else 0.0


def session(level, conf=TAPS, device=-1, **opts):
    o = {k: str(v) for k, v in opts.items()}
    o.update({k: "?" for k in SINKS})
    o[LEVEL_SINK[level]] = "x.csv"
    return Session(conf, options=o, device=device)
