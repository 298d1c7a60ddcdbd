"""The SHS pitch chain over the case table of tests/pitch_cases.py, each stage on its own inputs:
  1. the cPitchShs level (shs_kernel) against the oracle's cSpecScale + cPitchShs: rows with the oracle's peak decisions within
     2e-4 of the column scale (within 2e-6 for all but 0.1 % of them up to 513 bins); rows whose decisions differ only on a
     near tie of the oracle's sub-harmonic sum or at the margin of the candidate list, at most 0.5 % of them, counted
  2. the Viterbi / selector level (viterbi_kernel) bit for bit against the oracle's Viterbi on the kernel's own cPitchShs rows
     (the semitone columns to 2 ulps: the host's logf is not correctly rounded)
  3. the cPitchJitter level (jitter_kernel) against the oracle on the kernel's own F0: 1e-6 of the column scale, one row per
     frame (zeros where the reference drops a last frame) and the same voiced / unvoiced and period decisions
  4. the smoothed level and its onlyInSegments delta (seq_post_kernel) bit for bit against the oracle's end-of-input lag model
     on the kernel's own Viterbi and jitter rows
plus batch invariance over thousands of ragged utterances, the workspace refusals, and coverage of every axis value."""
import time

import numpy as np
import pytest

import pitch_cases as PC
from opensmile_b200 import Plan, capi, pack_utterances
from oracle import oracle

pytestmark = pytest.mark.gpu
RAN = {}              # case -> axis values
LAGS = set()          # T - V seen (V = rows of the Viterbi level before the end-of-input flush)
EXCUSED = {}          # case -> rows excused at the cPitchShs level
DROPPED = {}          # case -> jitter frames the reference drops (read window past the input)
LOG_ULPS = {}         # case -> semitone values off the host's logf (by at most 2 ulps)
_T0 = time.time()


def _bits_equal(a, b):
    return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32))


def _run(c, level, pcm, off):
    p = Plan(PC.components(c), level, device=0)
    try:
        return p.run_host(pcm, off), p.frame_offsets(off), p.element_names
    finally:
        p.close()


def _col_scale(ref):
    s = np.abs(ref).max(axis=0) if ref.shape[0] else np.ones(ref.shape[1], np.float32)
    s[s == 0] = 1.0
    return s


# ---------------------------------------------------------------- vectorised oracle of the smoother and the segment delta
def sma_lagged(x, V, lag_cols, no_zero):
    """oracle.sma_lagged without the Python loop (same float32 operations in the same order)"""
    x = np.asarray(x, np.float32)
    T, K = x.shape
    n = np.arange(T + 1)

    def g(d):
        idx = np.repeat(np.clip(n + d, 0, T - 1)[:, None], K, axis=1)
        if V >= 1:
            rows = (n == V - 1) | (n == V)
            for k in lag_cols:
                idx[rows, k] = np.minimum(idx[rows, k], V - 1)
        return np.take_along_axis(x, idx, axis=0)
    x0, a, b = g(0), g(-1), g(1)
    if not no_zero:
        return ((x0 + a) + b) / np.float32(3.0)
    y, N = x0.copy(), np.ones_like(x0)
    y = np.where(a != 0, y + a, y)
    N = np.where(a != 0, N + 1, N)
    y = np.where(b != 0, y + b, y)
    N = np.where(b != 0, N + 1, N)
    return np.where(x0 == 0, np.float32(0), y / N).astype(np.float32)


def delta_segments_lagged(x, V, win=2):
    """oracle.delta_segments_lagged without the Python loop: the running norm is an integer prefix sum (exact in float32)"""
    x = np.asarray(x, np.float32)
    T1, K = x.shape
    T = T1 - 1
    n = np.arange(T1 + win)
    last = np.full(n.size, T1 - 1)
    if V >= 1:
        m = (n >= V - 1) & (n <= V + 2)
        last[m] = np.minimum(last[m], V)
    if T - 5 <= V <= T - 2:
        last[(n == V + 3) & ~((V >= 1) & (n >= V - 1) & (n <= V + 2))] = T - 1
    num = np.zeros((n.size, K), np.float32)
    cnt = np.zeros((n.size, K), np.int64)
    for i in range(1, win + 1):
        a = x[np.minimum(np.maximum(n - i, 0), last)]
        b = x[np.minimum(np.maximum(n + i, 0), last)]
        ok = (a != 0) & (b != 0) & (a == a) & (b == b)
        num = np.where(ok, num + np.float32(i) * (b - a), num).astype(np.float32)
        cnt += ok * i * i
    norm = (2 * sum(i * i for i in range(1, win + 1)) + np.cumsum(cnt.ravel())).reshape(cnt.shape).astype(np.float32)
    return (num / norm).astype(np.float32)


def test_vectorised_lag_model_is_the_oracle():
    """the two helpers above are bit-identical to oracle.sma_lagged / delta_segments_lagged, every lag position included"""
    rng = np.random.default_rng(3)
    for T in (1, 2, 3, 6, 9, 14):
        x = rng.normal(size=(T, 4)).astype(np.float32)
        x[rng.random(x.shape) < 0.3] = 0
        for V in range(0, T + 1):
            for nz in (0, 1):
                sm = oracle.sma_lagged(x, V, {2, 3}, no_zero=nz)
                assert _bits_equal(sma_lagged(x, V, {2, 3}, nz), sm), (T, V, nz)
                assert _bits_equal(delta_segments_lagged(sm, V, 2), oracle.delta_segments_lagged(sm, V, 2)), (T, V, nz)


# ---------------------------------------------------------------- the near ties of the peak picker
def _ss_peaks_tied(c, hps, tol=1e-6):
    """rows where two of the nCandidates + 1 highest local maxima of the oracle's sub-harmonic sum are within `tol` relative
    (pitchShs.cpp:238-318; the sum restated in double from the oracle's scaled-spectrum tap)"""
    fe = PC.oracle_cfg(c)[0]
    nfft = oracle.geometry(fe, 0)[2]
    nMag, M = nfft // 2 + 1, hps.shape[1]
    fs = float(np.float32(nfft / c["sr"]))
    minF = max(c["minF"], 1.0)
    maxF = c["maxF"] if minF < c["maxF"] <= (nMag - 1) / fs else (nMag - 1) / fs
    ppo = float(np.float32(M / (np.log(maxF / minF) / np.log(2.0))))
    ss = hps.astype(np.float64).copy()
    scale = c["compression"]
    for h in range(2, c["nHarm"] + 1):
        sh = int(np.floor(ppo * np.log(h) / np.log(2.0)))
        if sh < M:
            ss[:, :M - sh] += hps[:, sh:] * scale
        scale *= c["compression"]
    ss = np.maximum(ss / c["nHarm"], 0)
    tied = np.zeros(hps.shape[0], bool)
    k = max(c["nCand"], 1) + 1
    for r in range(hps.shape[0]):
        s = ss[r]
        mid, lo, hi = s[1:-1], s[:-2], s[2:]
        strict = (lo < mid) & (mid > hi)
        weak = (lo < mid * (1 + tol)) & (mid * (1 + tol) > hi)          # maxima that a rounding of `tol` could create
        top_s = np.argsort(-np.where(strict, mid, -1))[:k]
        top_w = np.argsort(-np.where(weak, mid, -1))[:k]
        pk = np.sort(mid[weak])[::-1][:k]
        tied[r] = set(top_s[strict[top_s]]) != set(top_w[weak[top_w]]) or (
            pk.size > 1 and bool((np.abs(np.diff(pk)) <= tol * np.maximum(pk[:-1], 1e-30)).any()))
    return tied


def _check_reference_goldens(c):
    """the kernel's cPitchShs level against the reference's own tap of it (tests/golden/pitch_goldens.npz: ComParE_2016 on four
    signals, scripts/make_golden_pitch.py): candidate count exact, 2e-6 of the column scale"""
    import os
    from opensmile_b200.synth import mixed_pcm, voiced_pcm
    G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pitch_goldens.npz"))
    sigs = {"v32k": voiced_pcm(32000, 16000, seed=7), "m48k": mixed_pcm(48000, 16000, seed=2),
            "m30k": mixed_pcm(30000, 16000, seed=4), "m64k": mixed_pcm(64000, 16000, seed=3)}
    keys = sorted(sigs)
    pcm, off = pack_utterances([sigs[k] for k in keys])
    got, fo, _ = _run(c, "shs", pcm, off)
    for u, k in enumerate(keys):
        g, r = got[fo[u]:fo[u + 1]], G[k + "_shs"]
        assert g.shape == r.shape and np.array_equal(g[:, 0], r[:, 0]), k
        assert (np.abs(g - r) / _col_scale(r)).max() < 2e-6, k


# ---------------------------------------------------------------- the case table
@pytest.mark.parametrize("name", list(PC.BY_NAME))
def test_case(name):
    c = PC.BY_NAME[name]
    fe, sc, ps, vc, jc = PC.oracle_cfg(c)
    utts, pcm, off = PC.batch(c)
    nc = c["n_chan"]
    # 1. cPitchShs level
    shs, fo, names = _run(c, "shs", pcm, off)
    assert names == PC.shs_names(c)
    refs, taps = [], []
    for u, x in enumerate(utts):
        T = int(fo[u + 1] - fo[u])
        assert T == PC.frames(c, len(x) // nc), u
        r, h = oracle.pitch_shs(x, fe, sc, ps, nc, tap=True) if T else (np.zeros((0, shs.shape[1]), np.float32), None)
        refs.append(r)
        taps.append(h)
    ref = np.concatenate(refs)
    nC = max(c["nCand"], 1)
    err = (np.abs(shs - ref) / _col_scale(ref)).max(axis=1)
    same = (shs[:, 0] == ref[:, 0]) & (np.abs(shs[:, 1:1 + nC] - ref[:, 1:1 + nC]) <= 1e-4 * np.maximum(np.abs(ref[:, 1:1 + nC]), 1)).all(axis=1)
    # rows with the oracle's peak decisions: the values; rows where a decision differs: only on a near tie of the oracle's
    # sub-harmonic sum (two competing maxima, or a maximum that exists only by that margin).  2e-6 and 1e-6 except in the cases
    # of pitch_cases.SHS_WIDE, which says why
    tol = PC.SHS_WIDE.get(name, PC.SHS_STRICT)
    over = np.nonzero(same & (err > tol["value"]))[0]
    assert over.size == 0, "cPitchShs rows with the oracle's peaks beyond %g of the column scale: %s (err %s)" % (
        tol["value"], over[:8], err[over[:8]])
    flip = np.nonzero(~same)[0]
    if flip.size:
        tied = np.concatenate([_ss_peaks_tied(c, h, tol["tie"]) if h is not None else np.zeros(0, bool) for h in taps])
        worse = flip[~tied[flip]]
        assert worse.size <= tol["free"], "cPitchShs rows whose peak decisions differ without a near tie: %s\n%s\n%s" % (
            worse[:4], shs[worse[:2]], ref[worse[:2]])
        assert flip.size <= max(2, shs.shape[0] // 200), flip.size
    EXCUSED[name] = int(flip.size)
    if name == "anchor_compare16":
        _check_reference_goldens(c)
    if not c["voicing"]:                              # the chain behind it is refused (test_pitch_sweep_cpu.py)
        RAN[name] = {k: c[k] for k in PC.AXES}
        return
    # 2. Viterbi (+ selector) level on the kernel's own cPitchShs rows: exact
    vit, fo2, names = _run(c, PC.f0_level(c), pcm, off)
    assert np.array_equal(fo2, fo) and vit.shape[1] == len(PC.vit_names(c))
    lags, n_log = [], 0
    for u, x in enumerate(utts):
        a, b = fo[u], fo[u + 1]
        if a == b:
            lags.append(0)
            continue
        rv, V = oracle.viterbi(shs[a:b], ps, vc, with_lag=True)
        lags.append(V)
        LAGS.add(int(b - a - V))
        if c["sel"]:
            e = oracle.energy(x, fe, oracle.Energy(0, 1, 0, 0, 1.0, 1.0, 1.0, 0.0, 0.0, 0.0), windowed=1, n_chan=nc)
            rv = oracle.valbased_select(e[:, 0], rv, 0.001)
        ulps = np.abs(vit[a:b].view(np.int32).astype(np.int64) - rv.view(np.int32))
        # the semitone columns take a float logarithm: the host's logf (glibc) is within 1 ulp of the rounded double logarithm
        # the kernel uses, and differs from it on about 0.1 % of arguments; 12 log(f / 27.5) / log(2) turns that into at most
        # 2 ulps of the semitone value.  Every other column is exact
        log_cols = [k for k, nm in enumerate(PC.vit_names(c)) if nm.endswith("Log")]
        LOG_ULPS[name] = LOG_ULPS.get(name, 0) + int((ulps[:, log_cols] > 0).sum())
        n_log += int((rv[:, log_cols] > 0).sum())
        ulps[:, log_cols] = np.maximum(ulps[:, log_cols] - 2, 0)
        bad = np.nonzero(ulps.any(axis=1))[0]
        assert bad.size == 0, "Viterbi level of utterance %d (T = %d): %d rows differ, first %s" % (u, b - a, bad.size, bad[:8])
    # CUDA's logf put ~5 % of these values off glibc's (188 of ~3900 in v_buf_8_all_outputs); the rounded double logarithm
    # ~0.1 % of the arguments (each appears in F0finalLog and F0finEnvLog)
    assert LOG_ULPS.get(name, 0) <= max(4, n_log // 200), (LOG_ULPS.get(name, 0), n_log)
    # 3. cPitchJitter on the kernel's own F0
    jit, fo3, names = _run(c, "jit", pcm, off)
    assert names == PC.jit_names(c) and np.array_equal(fo3, fo)
    jrefs = []
    for u, x in enumerate(utts):
        a, b = fo[u], fo[u + 1]
        rj = oracle.pitch_jitter(x, fe, jc, vit[a:b, 0], nc) if b > a else np.zeros((0, jit.shape[1]), np.float32)
        # the reference drops a frame whose read window runs past the input (lld/pitchJitter.cpp:668-673); that can only be one
        # of the last frames (the window length rounds up to frameSize + 1).  The plan keeps one row per frame and writes zeros
        dropped = (b - a) - rj.shape[0]
        assert 0 <= dropped <= 1, (u, rj.shape, b - a)
        if dropped:
            assert not jit[b - 1].any(), u
            rj = np.concatenate([rj, np.zeros((dropped, jit.shape[1]), np.float32)])
        DROPPED[name] = DROPPED.get(name, 0) + dropped
        jrefs.append(rj)
    jref = np.concatenate(jrefs)
    jerr = np.abs(jit - jref) / _col_scale(jref)
    bad = np.argwhere(jerr > 1e-6)
    assert bad.size == 0, [(names[k], int(r), float(jit[r, k]), float(jref[r, k])) for r, k in bad[:8]]
    for k, nm in enumerate(names):
        if nm == "F0final" or nm == "sourceQualityRange":             # voiced / unvoiced and period-found decisions
            assert np.array_equal(jit[:, k] > 0, jref[:, k] > 0), nm
    # 4. smoothed level and its onlyInSegments delta on the kernel's own Viterbi and jitter rows: exact
    lld, fo4, _ = _run(c, "lld", pcm, off)
    nv, nj = vit.shape[1], jit.shape[1]
    for u in range(len(utts)):
        a, b = fo[u], fo[u + 1]
        if a == b:
            assert fo4[u + 1] == fo4[u]
            continue
        x = np.concatenate([vit[a:b], jit[a:b]], axis=1)
        V = lags[u]
        sm = sma_lagged(x, V, set(range(nv, nv + nj)), True)
        de = delta_segments_lagged(sm, V, 2)
        want = np.concatenate([sm, de[:sm.shape[0]]], axis=1)
        got = lld[fo4[u]:fo4[u + 1]]
        assert got.shape == want.shape, (u, got.shape, want.shape)
        bad = np.nonzero((got.view(np.uint32) != want.view(np.uint32)).any(axis=1))[0]
        assert bad.size == 0, "smoothed / delta rows of utterance %d (T = %d, V = %d): %d differ, first %s" % (u, b - a, V, bad.size, bad[:8])
    RAN[name] = {k: c[k] for k in PC.AXES}
    print("\n%s: %d rows, %d cPitchShs rows excused (near ties)" % (name, shs.shape[0], EXCUSED[name]))


# ---------------------------------------------------------------- batch invariance
def _big_batch(c, n_utt, seed):
    rng = np.random.default_rng(seed)
    sr = int(c["sr"])
    N, S = int(round(c["frame"] * sr)), int(round(c["step"] * sr))
    T = np.where(rng.random(n_utt) < 0.05, rng.integers(200, 600, n_utt), rng.integers(0, 2 * c["bufLen"] + 8, n_utt))
    L = np.where(T > 0, N + (T - 1) * S + rng.integers(0, S, n_utt), rng.integers(0, N, n_utt))
    base = PC.signal("mixed", int(L.max()) + 50_000, c, seed)
    glide = PC.signal("glide", int(L.max()) + 50_000, c, seed + 1)
    nc = c["n_chan"]
    starts = rng.integers(0, int(L.max()) + 50_000 - L, n_utt)
    return [(glide if u % 3 == 0 else base)[s * nc:(s + n) * nc] for u, (s, n) in enumerate(zip(starts, L))]


@pytest.mark.parametrize("name,n_utt", [("anchor_compare16", 3000), ("v_no_selector", 2000), ("x_48k_8cand_buf64_npts_3000", 2000)])
def test_rows_do_not_depend_on_the_batch(name, n_utt):
    import torch
    c = PC.BY_NAME[name]
    utts = _big_batch(c, n_utt, seed=len(name))
    pcm, off = pack_utterances(utts, n_chan=c["n_chan"])
    p = Plan(PC.components(c), "lld", device=0)
    try:
        fo = p.frame_offsets(off)
        dev = p.run_device(torch.from_numpy(pcm).cuda(), off)
        torch.cuda.synchronize()
        dev = dev.cpu().numpy()
        assert _bits_equal(p.run_host(pcm, off), dev)
        rpcm, roff = pack_utterances(utts[::-1], n_chan=c["n_chan"])
        rev = p.run_host(rpcm, roff)
        rfo = p.frame_offsets(roff)
        for u in range(n_utt):
            r = n_utt - 1 - u
            assert _bits_equal(rev[rfo[r]:rfo[r + 1]], dev[fo[u]:fo[u + 1]]), u
        for u in np.random.default_rng(7).choice(n_utt, 40, replace=False):
            alone = p.run_host(utts[u], np.array([0, len(utts[u]) // c["n_chan"]], np.int64))
            assert _bits_equal(alone, dev[fo[u]:fo[u + 1]]), u
    finally:
        p.close()
    print("\n%s: %d utterances, %d rows" % (name, n_utt, dev.shape[0]))


# ---------------------------------------------------------------- limits of the kernels' workspaces
@pytest.mark.parametrize("kw,msg", [
    (dict(sr=8000, nPts=600), "cSpecScale: spectrum too long for the SHS kernel's workspace"),
    (dict(sr=48000, minPitch=3.0), "cPitchJitter: frame size / pitch range need more workspace than the kernel has"),
])
def test_workspace_limits_are_refused_when_the_plan_is_created(kw, msg):
    c = PC.case("refused", **kw)
    with pytest.raises(RuntimeError) as e:
        Plan(PC.components(c), "lld", device=0)
    assert "(%d): %s" % (capi.ERR_UNSUPPORTED, msg) in str(e.value), str(e.value)


def test_every_axis_value_of_the_table_ran():
    """every value of every axis ran (coverage is checked, not assumed), and the end-of-input lag rule's rows were reached"""
    if set(RAN) != set(PC.BY_NAME):
        pytest.skip("only %d of %d cases ran" % (len(RAN), len(PC.BY_NAME)))
    for axis, values in PC.AXES.items():
        seen = {r[axis] for r in RAN.values()}
        assert values <= seen, (axis, values - seen)
    print("\nT - V seen: %s; cPitchShs rows excused: %d in %d cases; jitter frames the reference drops: %d; semitone values "
          "off the host's logf: %d; %.0f s" % (sorted(LAGS), sum(EXCUSED.values()), sum(1 for v in EXCUSED.values() if v),
                                         sum(DROPPED.values()), sum(LOG_ULPS.values()), time.time() - _T0))
    assert LAGS & {2, 3, 4, 5}, LAGS
