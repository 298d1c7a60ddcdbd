"""cFunctionals on contours longer than 8 192 frames, the host-visible pieces (tests/native/long_contours_host.cpp): the percentile rank
selection's key and digit walk against np.sort order statistics on adversarial contours, the work space chunk plan on ragged batches,
and the sequential statements the long path shares with the short one (functionals_seq.cuh, host build) against the oracle at length."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle import functionals_oracle as fo
from test_functionals_cpu import SPEC_D, SPEC_E, SPEC_F, SPEC_G, SPEC_I, SPEC_J, SPEC_K, to_c_spec

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_L = []


def lib():
    if not _L:
        so = "/tmp/osm_long_contours_host_%d.so" % os.getuid()
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", so,
                               os.path.join(ROOT, "tests", "native", "long_contours_host.cpp")])
        L = C.CDLL(so)
        L.lch_key.argtypes, L.lch_key.restype = [C.c_float], C.c_uint32
        L.lch_value.argtypes, L.lch_value.restype = [C.c_uint32], C.c_float
        L.lch_select.argtypes, L.lch_select.restype = [C.c_void_p, C.c_int64, C.c_int64], C.c_float
        L.lch_pctl_block.argtypes, L.lch_pctl_block.restype = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p], C.c_int
        L.lch_plan.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int64, C.c_void_p, C.c_int, C.c_void_p, C.c_int,
                               C.POINTER(C.c_int), C.POINTER(C.c_int)]
        L.lch_plan.restype = C.c_int64
        L.lch_slice_floats.argtypes, L.lch_slice_floats.restype = [C.c_int64, C.c_int, C.c_int], C.c_int64
        L.lch_ws_cap.restype = C.c_int64
        _L.append(L)
    return _L[0]


def bit_sorted(x):
    """a full sort by the order the key defines: ascending values, -0 before +0"""
    u = x.view(np.uint32)
    k = np.where(u & 0x80000000, ~u, u | 0x80000000).astype(np.uint32)
    return np.sort(k).astype(np.uint32)


def key_to_value(k):
    k = np.asarray(k, np.uint32)
    return np.where(k & 0x80000000, k & 0x7fffffff, ~k).astype(np.uint32).view(np.float32)


def adversarial(rng):
    den = np.float32(1e-40)
    return {
        "one": np.array([3.5], np.float32),
        "two": np.array([2.0, -1.0], np.float32),
        "equal8193": np.full(8193, 0.75, np.float32),
        "twovalued8193": np.where(rng.random(8193) > 0.3, 1.0, -2.0).astype(np.float32),
        "dups8193": np.round(rng.standard_normal(8193) * 3).astype(np.float32),
        "signedzeros8193": np.where(rng.random(8193) > 0.5, np.float32(0.0), np.float32(-0.0)).astype(np.float32),
        "zeros_and_values": np.concatenate([np.zeros(3000, np.float32), -np.zeros(2000, np.float32), rng.standard_normal(3193).astype(np.float32)]),
        "infs_denormals": rng.permutation(np.concatenate([np.full(5, np.inf), np.full(7, -np.inf), [den, -den, np.float32(1.4e-45), -np.float32(1.4e-45)],
                                                          rng.standard_normal(8177) * 1e-38]).astype(np.float32)),
        "lld1e6": np.cumsum(rng.standard_normal(10 ** 6)).astype(np.float32),
    }


def test_key_orders_like_the_values():
    L = lib()
    xs = np.array([-np.inf, -3e38, -1.0, -1e-40, -1.4e-45, -0.0, 0.0, 1.4e-45, 1e-40, 1.0, 3e38, np.inf], np.float32)
    keys = [L.lch_key(float(x)) for x in xs]
    assert keys == sorted(keys) and len(set(keys)) == len(keys)            # strictly increasing, -0 just below +0
    for x, k in zip(xs, keys):
        y = np.float32(L.lch_value(k))
        assert y.view(np.uint32) == x.view(np.uint32)                     # the walk's prefix maps back to the value, sign of zero included


@pytest.mark.parametrize("name", ["one", "two", "equal8193", "twovalued8193", "dups8193", "signedzeros8193", "zeros_and_values",
                                  "infs_denormals", "lld1e6"])
def test_digit_walk_equals_np_sort_order_statistics(name):
    L = lib()
    x = adversarial(np.random.default_rng(7))[name]
    N = len(x)
    s = np.sort(x)
    sk = key_to_value(bit_sorted(x))
    ranks = sorted({0, N - 1, N // 2, N // 3, (N - 1) // 4, 3 * (N - 1) // 4, max(N - 2, 0), min(1, N - 1)})
    for r in ranks:
        got = np.float32(L.lch_select(x.ctypes.data, N, r))
        assert got == s[r] or (np.isnan(got) and np.isnan(s[r])), (name, r, got, s[r])
        assert got.view(np.uint32) == sk[r].view(np.uint32), (name, r)     # the bits of the key-ordered sort (zeros: -0 first)


def _interp_pctl(s, p):
    """getInterpPctl (functionalPercentiles.cpp:317-336) on a sorted float32 array, float32 arithmetic"""
    N = len(s)
    idx = p * (N - 1)
    i1, i2 = min(max(int(np.floor(idx)), 0), N - 1), min(max(int(np.ceil(idx)), 0), N - 1)
    if i1 != i2:
        return np.float32(s[i1] * np.float32(i2 - idx) + s[i2] * np.float32(idx - i1))
    return s[i1]


def _index_pctl(s, p):
    v = p * (len(s) - 1)
    r = int(np.floor(v + 0.5))                                            # C round() of a non-negative value
    return s[min(max(r, 0), len(s) - 1)]


def _expected_block(P, s):
    f = _interp_pctl if P["interp"] else _index_pctl
    q = [f(s, 0.25), f(s, 0.5), f(s, 0.75)]
    out = [q[0]] * P["quartile1"] + [q[1]] * P["quartile2"] + [q[2]] * P["quartile3"]
    out += [np.float32(q[1] - q[0])] * P["iqr12"] + [np.float32(q[2] - q[1])] * P["iqr23"] + [np.float32(q[2] - q[0])] * P["iqr13"]
    pc = [f(s, p) for p in P["percentile"]]
    out += pc + [np.float32(abs(np.float32(pc[b] - pc[a]))) for a, b in P["pctlrange"]]
    return np.array(out, np.float32)


PCTL_OPTIONS = [dict(quartile1=1, quartile2=1, quartile3=1, iqr12=1, iqr23=1, iqr13=1, percentile=[0.01, 0.2, 0.5, 0.8, 0.99, 0.0, 1.0, 0.333],
                     pctlrange=[(0, 4), (1, 3), (5, 6), (7, 2)]),
                dict(quartile1=0, quartile2=1, quartile3=0, iqr12=0, iqr23=0, iqr13=1, percentile=[0.95, 0.05], pctlrange=[(1, 0)]),
                dict(quartile1=0, quartile2=0, quartile3=0, iqr12=0, iqr23=0, iqr13=0, percentile=[0.5], pctlrange=[])]


@pytest.mark.parametrize("interp", [1, 0])
@pytest.mark.parametrize("opt", range(len(PCTL_OPTIONS)))
def test_percentile_block_equals_the_full_sort(interp, opt):
    """every quartile / iqr / percentile / pctlrange option, interpolated and indexed: the block assembled from the selected ranks equals
    the one read from a full sort, bit for bit (both neighbours of an interpolated percentile are selected)"""
    from opensmile_b200 import functionals as F
    L = lib()
    P = dict(PCTL_OPTIONS[opt], interp=interp)
    cs = F.spec(["Percentiles"], percentiles=P)
    for name, x in adversarial(np.random.default_rng(11)).items():
        if name == "lld1e6" and opt:
            continue
        out = np.zeros(32, np.float32)
        n = L.lch_pctl_block(C.byref(cs), x.ctypes.data, len(x), out.ctypes.data)
        exp = _expected_block(P, key_to_value(bit_sorted(x)))
        assert n == len(exp)
        assert np.array_equal(out[:n].view(np.uint32), exp.view(np.uint32)) or np.array_equal(out[:n], exp, equal_nan=True), (name, out[:n], exp)
        assert np.array_equal(out[:n], _expected_block(P, np.sort(x)), equal_nan=True), name    # value-equal to np.sort's order


def plan(T, nIn, listMul, lensFloats, cap):
    L = lib()
    T = np.ascontiguousarray(T, np.int64)
    maxC = int(np.sum(T > 8192)) * nIn + 1
    con = np.zeros((maxC, 3), np.int32)
    chk = np.zeros((maxC, 3), np.int32)
    nC, nK = C.c_int(), C.c_int()
    need = L.lch_plan(T.ctypes.data, len(T), nIn, listMul, lensFloats, cap, con.ctypes.data, maxC, chk.ctypes.data, maxC, C.byref(nC), C.byref(nK))
    assert need >= 0
    return need, con[:nC.value], chk[:nK.value]


def check_plan(T, nIn, listMul, lensFloats, cap):
    L = lib()
    need, con, chk = plan(T, nIn, listMul, lensFloats, cap)
    expected = [(u, e) for u, t in enumerate(T) if t > 8192 for e in range(nIn)]
    assert [tuple(x) for x in con[:, :2]] == expected                      # every long contour once, in order; no short one
    biggest = 0
    for k, (b, e, cp) in enumerate(chk):
        assert b < e and (k == 0 and b == 0 or b == chk[k - 1][1])
        assert np.all(con[b:e, 2] == k)
        assert cp == max((T[con[c, 0]] + 31) // 32 * 32 for c in range(b, e))   # every slice holds the chunk's longest copy
        size = (e - b) * L.lch_slice_floats(int(cp), listMul, lensFloats)
        assert size <= cap or e - b == 1                                   # only a contour that alone exceeds the cap exceeds it
        biggest = max(biggest, size)
    assert len(chk) == 0 or chk[-1][1] == len(con)
    assert need == biggest
    return need, chk


@pytest.mark.parametrize("listMul,lensFloats", [(2, 32), (0, 0), (0, 100), (2, 1000)])
def test_chunk_plan_covers_every_long_contour_once_within_the_cap(listMul, lensFloats):
    rng = np.random.default_rng(listMul * 1000 + lensFloats)
    T = np.concatenate([[0, 1, 8192, 8193, 8224, 8225, 60000, 360000], rng.integers(0, 200000, 60)])
    rng.shuffle(T)
    for nIn in (1, 7, 65):
        for cap in (lib().lch_ws_cap(), 4 << 20, 3 * 360032 + 5000, 100000):
            check_plan(T, nIn, listMul, lensFloats, cap)


def test_chunk_plan_of_one_utterance_larger_than_the_cap():
    # one 60-minute ComParE-sized utterance (130 contours of 360 000 frames, 12 bytes a frame = 560 MB) and a contour that alone
    # exceeds a small cap
    need, chk = check_plan(np.array([360000]), 130, 2, 100, lib().lch_ws_cap())
    assert len(chk) > 1 and need <= lib().lch_ws_cap()
    need, chk = check_plan(np.array([9000, 500000, 9000]), 3, 2, 32, 1 << 20)
    assert need == lib().lch_slice_floats(500000, 2, 32) and len(chk) >= 4


def test_chunk_plan_without_long_contours():
    need, con, chk = plan(np.array([0, 5, 8192]), 4, 2, 32, 1 << 20)
    assert need == 0 and len(con) == 0 and len(chk) == 0


@pytest.mark.parametrize("n", [10000, 50000])
def test_sequential_statements_at_length_equal_the_oracle(n):
    """functionals_seq.cuh compiled for the host (the statements both paths run) against the oracle on contours of 10^4 .. 5 10^4
    frames: a random walk, a contour with plateaus and pauses and (10^4) a zigzag, Peaks2's worst case, bit for bit"""
    import functionals_harness as fh
    rng = np.random.default_rng(n)
    walk = np.cumsum(rng.standard_normal(n)).astype(np.float32)
    zig = (np.where(np.arange(n) % 2, 1.0, -1.0) * (1 + 0.001 * np.arange(n))).astype(np.float32)
    plat = np.where(rng.random(n) > 0.7, 0, np.round(walk / 4)).astype(np.float32)
    for x in (walk, plat) + ((zig,) if n <= 10000 else ()):                     # the oracle's Peaks2 pruning of a zigzag is slow
        mn, mx = np.float32(x.min()), np.float32(x.max())
        mean = np.float32(x.astype(np.float64).sum() / len(x))
        for spec in (SPEC_D, SPEC_E, SPEC_F) + ((SPEC_G,) if n <= 10000 else ()):   # the oracle's dynRelThresh pruning is quadratic
            cs = to_c_spec(spec)
            if "Segments" in spec.enabled:
                nrm = fo._norm(spec.segments["norm"], spec.segments["norm_set"], spec.master_norm)
                assert np.array_equal(fh.segments(cs, x, 0.01, nrm), np.array(fo._segments(spec, x, mn, mx, mean, 0.01), np.float32))
            if "Peaks2" in spec.enabled:
                nrm = fo._norm(spec.peaks2["norm"], spec.peaks2["norm_set"], spec.master_norm)
                a, b = fh.peaks2(cs, x, 0.01, nrm), np.array(fo._peaks2(spec, x, mn, mx, mean, 0.01), np.float32)
                assert np.array_equal(a, b, equal_nan=True), (a, b)
            if "Lpc" in spec.enabled:
                a, b = fh.lpc(cs, x), np.array(fo._lpc(spec, x), np.float32)
                assert np.array_equal(a, b, equal_nan=True), (a, b)
        for spec in (SPEC_I, SPEC_J, SPEC_K):
            cs = to_c_spec(spec)
            nrm = fo._norm(spec.onset["norm"], spec.onset["norm_set"], spec.master_norm)
            assert np.array_equal(fh.onset(cs, x, 0.01, nrm), np.array(fo._onset(spec, x, 0.01), np.float32), equal_nan=True)
            nrm = fo._norm(spec.peaks["norm"], spec.peaks["norm_set"], spec.master_norm)
            assert np.array_equal(fh.peaks(cs, x, 0.01, nrm), np.array(fo._peaks_old(spec, x, 0.01), np.float32), equal_nan=True)
            assert np.array_equal(fh.crossings(cs, x), np.array(fo._crossings(spec, x), np.float32), equal_nan=True)
