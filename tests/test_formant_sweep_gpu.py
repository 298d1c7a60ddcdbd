"""formant_kernel and harmonics_kernel over the case table of tests/formant_cases.py, each kernel on its own inputs:
  1. the cFormantLpc level against the host build of the same statements (tests/native/formant_host.cpp) on the same PCM: every
     row bit-identical, except formant values that a device-vs-glibc ulp of atan2 / log in root_to_formant moves -- at most 1e-6
     of the column scale, counted and printed;
  2. the cHarmonics level against the host build run on the kernel's own F0, formant and magnitude levels (one plan per level over
     the same batch): every value, HNR included, within 1e-5 dB (or two float ulps of log10f near the -201 dB floor);
  3. batch shape: every utterance's rows equal its run alone, two runs are bit-identical, and 2 000 ragged utterances of 0 - 40
     frames equal the host build.
The wall time of every case is printed."""
import time

import numpy as np
import pytest

import formant_cases as FC
import formant_harness as fh
from opensmile_b200 import Plan, capi

pytestmark = pytest.mark.gpu
RAN = {}
ULPS = {}
_T0 = time.time()


def _bits_equal(a, b):
    return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32))


def _run(c, level, pcm, off):
    p = Plan(FC.components(c), level, device=0)
    try:
        return p.run_host(pcm, off), p.frame_offsets(off), p.element_names
    finally:
        p.close()


def _host_formants(c, x):
    N, S, nfft = FC.geometry(c)
    T = FC.frames(c, FC.n_samples(c, x))
    w = fh.window(capi.WIN_BY_NAME[c["win"]], N)
    return fh.formant_rows(fh.wave_level(x, 1 if c["f32"] else c["n_chan"]), N, S, T, w, float(c["sr"]), nfft, c["frame"], c["zps"],
                           c["target"], c["p"], c["nF"], c["minF"], c["maxF"], c["nvalid"], c["freqs"], c["bws"])


def _check_formants(c, got, want):
    """bit-identical, except formant / bandwidth values off by the atan2 / log ulp (<= 1e-6 of the column scale); returns the count"""
    assert got.shape == want.shape
    diff = got.view(np.uint32) != want.view(np.uint32)
    if not diff.any():
        return 0
    scale = np.abs(want).max(axis=0) + 1.0
    rel = np.abs(got - want) / scale
    if c["nvalid"]:
        assert not diff[:, 0].any(), "number of valid formants differs"
    bad = np.argwhere(diff & (rel > 1e-6))
    assert bad.size == 0, [(int(r), int(k), float(got[r, k]), float(want[r, k])) for r, k in bad[:8]]
    return int(diff.sum())


@pytest.mark.parametrize("name", list(FC.BY_NAME))
def test_case(name):
    t0 = time.time()
    c = FC.BY_NAME[name]
    utts, pcm, off = FC.batch(c)
    # 1. cFormantLpc level vs the host build on the same PCM
    fmt, fo, names = _run(c, "formants", pcm, off)
    assert names == FC.formant_names(c)
    n_ulp = 0
    for u, x in enumerate(utts):
        want = _host_formants(c, x)
        n_ulp += _check_formants(c, fmt[fo[u]:fo[u + 1]], want)
    ULPS[name] = n_ulp
    # 2. cHarmonics level vs the host build on the kernel's own F0, formant and magnitude levels
    n_rows = 0
    if c["hz"]:
        harm, fo_h, hnames = _run(c, "harm", pcm, off)
        assert hnames == FC.harmonics_names(c)
        f0, fo_p, _ = _run(c, FC.f0_level(c), pcm, off)
        mag, fo_m, _ = _run(c, "h_mag", pcm, off)
        assert np.array_equal(fo_h, fo_p) and np.array_equal(fo_h, fo_m)
        n_harm, diffs, fa, hnr = FC.harmonics_config(c)
        nF = FC.n_formants(c) if c["hfmt"] else 0
        Nh, _, nfft_h = FC.geometry(c, hz=True)
        bin_hz = 1.0 / (c["hframe"] * nfft_h / Nh if nfft_h != Nh else c["hframe"])
        for u in range(len(utts)):
            a, b = fo_h[u], fo_h[u + 1]
            if a == b:
                continue
            F = fmt[fo[u]:fo[u] + (b - a), int(c["nvalid"]):int(c["nvalid"]) + nF] if nF else np.zeros((b - a, 0), np.float32)
            want = fh.harmonics_rows(f0[a:b, 0], F, mag[a:b], bin_hz, n_harm, diffs, fa, c["floor"], hnr)
            got = harm[a:b]
            err = np.abs(got - want)
            # the log magnitudes take log10f: device and glibc differ by an ulp now and then, which is 1.5e-5 dB near the -201 dB
            # floor of a difference, so the bar is 1e-5 dB or two float ulps of the value
            tol = np.maximum(1e-5, 2 * np.spacing(np.abs(want)))
            bad = np.argwhere(err > tol)
            assert bad.size == 0, (u, [(int(r), int(k), float(got[r, k]), float(want[r, k])) for r, k in bad[:8]])
            n_rows += b - a
    RAN[name] = FC.axis_values(c)
    print("\n%s (%s, fpw %d): %d formant rows, %d values off by the atan2 / log ulp; %d harmonics rows; %.1f s" % (
        name, RAN[name]["path"], RAN[name]["fpw"], fmt.shape[0], n_ulp, n_rows, time.time() - t0))


@pytest.mark.parametrize("name", ["anchor_gemaps", "v01a"])
def test_end_to_end_against_the_oracle(name):
    """from PCM: the kernel's formant level against the oracle's cTransformFFT (the reference's own FFT) -> cSpecResample -> cLpc
    -> cFormantLpc, every row within 1e-5 of the column scale"""
    from oracle import formant_oracle as fo
    if not fo.ref_fft_available():
        pytest.skip("oracle/_ref/libfftsg.so not built (make -C oracle ref)")
    c = FC.BY_NAME[name]
    utts, pcm, off = FC.batch(c)
    fmt, fo_, _ = _run(c, "formants", pcm, off)
    refs = [fo.formant_chain(x, c["sr"], c["frame"], c["step"], c["win"], c["zps"], c["target"], c["p"], c["nF"], c["minF"], c["maxF"],
                             c["nvalid"], c["freqs"], c["bws"], exact_fft=True) for x in utts]
    ref = np.concatenate(refs)
    assert fmt.shape == ref.shape
    scale = np.abs(ref).max(axis=0)
    scale[scale == 0] = 1.0
    err = np.abs(fmt - ref) / scale
    assert err.max() <= 1e-5, (np.argwhere(err > 1e-5)[:4], err.max())
    print("\n%s: %d rows end to end, worst %.2g of the column scale" % (name, fmt.shape[0], err.max()))


# ---------------------------------------------------------------- batch shape
@pytest.mark.parametrize("name", ["anchor_gemaps", "c44k1_20ms", "u16k_25ms", "p16_n8"])
def test_rows_do_not_depend_on_the_batch(name):
    """every utterance's rows equal its run alone and a second run, at the formant and harmonics levels"""
    c = FC.BY_NAME[name]
    utts, pcm, off = FC.batch(c)
    nc = 1 if c["f32"] else c["n_chan"]
    for level in ("formants", "harm") if c["hz"] else ("formants",):
        p = Plan(FC.components(c), level, device=0)
        try:
            rows = p.run_host(pcm, off)
            assert _bits_equal(p.run_host(pcm, off), rows)
            fo = p.frame_offsets(off)
            for u, x in enumerate(utts):
                if len(x) == 0:
                    assert fo[u + 1] == fo[u]
                    continue
                alone = p.run_host(x, np.array([0, len(x) // nc], np.int64))
                assert _bits_equal(alone, rows[fo[u]:fo[u + 1]]), (level, u)
        finally:
            p.close()


@pytest.mark.parametrize("name", ["anchor_gemaps", "c48k_20ms", "p16_n15"])
def test_two_thousand_ragged_utterances_equal_the_host_build(name):
    c = FC.BY_NAME[name]
    rng = np.random.default_rng(11)
    N, S, _ = FC.geometry(c)
    T = rng.integers(0, 41, 2000)
    L = np.where(T > 0, N + (T - 1) * S + rng.integers(0, S, T.size), rng.integers(0, N, T.size))
    base = FC.signal("mixed", int(L.max()) + 40_000, c, 3)
    vow = FC.signal("vowel", int(L.max()) + 40_000, c, 4)
    starts = rng.integers(0, 40_000, T.size)
    nc = c["n_chan"]
    utts = [(vow if u % 2 else base)[s * nc:(s + n) * nc] for u, (s, n) in enumerate(zip(starts, L))]
    from opensmile_b200 import pack_utterances
    pcm, off = pack_utterances(utts, n_chan=nc)
    rows, fo, _ = _run(c, "formants", pcm, off)
    n_ulp = 0
    for u, x in enumerate(utts):
        n_ulp += _check_formants(c, rows[fo[u]:fo[u + 1]], _host_formants(c, x))
    print("\n%s: 2000 utterances, %d rows, %d values off by the atan2 / log ulp" % (name, rows.shape[0], n_ulp))


def test_every_axis_value_of_the_table_ran():
    if set(RAN) != set(FC.BY_NAME):
        pytest.skip("only %d of %d cases ran" % (len(RAN), len(FC.BY_NAME)))
    for axis, values in FC.AXES.items():
        seen = {r[axis] for r in RAN.values()}
        assert values <= seen, (axis, values - seen)
    print("\nformant values off by the atan2 / log ulp: %d in %d cases; %.0f s" % (
        sum(ULPS.values()), sum(1 for v in ULPS.values() if v), time.time() - _T0))
