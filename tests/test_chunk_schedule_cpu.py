"""The batch cut of the per-frame LLD kernels (opensmile_b200/csrc/chunk_schedule.hpp), built for the host: every CTA run
of the balanced schedule holds at most ctaTiles tiles, there are at most as many runs as resident CTAs, and the chunks
cover every output row of every utterance exactly once with the halo the kernel needs."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_L = []


def lib():
    if not _L:
        so = "/tmp/osm_chunk_schedule_host_%d.so" % os.getuid()
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I/usr/local/cuda/include", "-o", so,
                               os.path.join(ROOT, "tests", "native", "chunk_schedule_host.cpp")])
        _L.append(C.CDLL(so))
    return _L[0]


def balanced(T, F, H, KT, ctas):
    T = np.ascontiguousarray(T, np.int64)
    cap = 4 * (int(np.sum((T + F - 1) // F)) + len(T) + ctas) + 16
    out = np.zeros((cap, 5), np.int32)
    q = C.c_int64()
    n = lib().csh_balanced(T.ctypes.data_as(C.POINTER(C.c_int64)), len(T), F, H, KT, ctas,
                           out.ctypes.data_as(C.POINTER(C.c_int32)), cap, C.byref(q))
    assert n > 0
    return out[:n], q.value


def check(T, F, H, KT, ctas):
    ch, Q = balanced(T, F, H, KT, ctas)
    body, W = ch[:-1], int(ch[-1, 4])
    assert ch[-1, 0] == len(T)
    w0 = body[:, 4]
    assert np.all(np.diff(w0) > 0) and (len(w0) == 0 or w0[0] == 0)
    assert W <= Q * ctas
    covered = [np.zeros(t, np.int32) for t in T]
    runs = {}
    for k, (u, a, b, tile0, w) in enumerate(body):
        t = T[u]
        assert 0 <= a < b <= t
        s0, s1 = max(a - H, 0), min(b + H, t)
        nT = (s1 - s0 + F - 1) // F
        assert nT <= KT
        assert s1 - s0 <= nT * F
        assert (s1 == t) or (s1 - s0) % F == 0, (u, a, b)   # a whole number of tiles except at the utterance end
        nxt = int(w0[k + 1]) if k + 1 < len(w0) else W
        assert w + nT <= nxt                         # the schedule position counts the chunk's tiles
        covered[u][a:b] += 1
        runs.setdefault(w // Q, 0)
        runs[w // Q] += nT
    for c in covered:
        assert np.all(c == 1)
    assert len(runs) <= ctas
    assert max(runs.values(), default=0) <= Q + KT      # a run ends at its boundary, up to one chunk that starts in it
    return ch, Q, runs


@pytest.mark.parametrize("F,H", [(32, 4), (32, 0), (16, 4), (8, 4), (8, 2), (4, 2), (32, 16)])
@pytest.mark.parametrize("ctas", [1, 7, 132, 264])
def test_balanced_cut_covers_every_row_once(F, H, ctas):
    rng = np.random.default_rng(F * 1000 + H * 10 + ctas)
    T = np.concatenate([[0, 1, 2, H, H + 1, F, F + 1, 2 * F - 1, 16 * F, 16 * F + 1, 5000],
                        rng.integers(0, 40 * F, 300)])
    check(T, F, H, 16, ctas)


def test_bench_shape_is_balanced_without_extra_tiles():
    # mfcc12: 2000 utterances of 500 frames, 32-frame tiles, halo 4, 264 resident CTAs
    ch, Q, runs = check(np.full(2000, 500), 32, 4, 16, 264)
    assert int(ch[-1, 4]) == 2000 * 16                   # the cuts fit in each utterance's last tile
    assert Q == 122 and max(runs.values()) == Q and len(runs) == 263


def test_tiny_batch_runs_of_one_tile():
    # fewer tiles than CTAs: one-tile runs, and with F = 2H a single tile cannot hold a row beside the halo
    check(np.array([3, 9, 17, 40]), 8, 4, 16, 132)
    check(np.array([1, 1, 1]), 32, 4, 16, 264)
