"""spectral_kernel, acf_pitch_kernel<N,F,NT> + pitch_smooth_kernel and the time ops over the case table of tests/spectral_cases.py.
Per case:
  1. stage by stage: the plan's magnitude level (mag_rows_kernel) and its op level come from the same LLD instance; the oracle's
     cSpectral / cAcf -> cPitchACF runs on those very magnitudes, so the tolerances below are the kernel's alone:
       - cSpectral on the linear spectrum: float statements (alpha ratio, Hammarberg index, sharpness, harmonicity, flatness)
         within 2 float ulps; roll-off points and spectral max / min positions (bin frequencies chosen by comparisons) equal;
         double-accumulated descriptors within 1e-6 of the column scale over the case's rows (only the summation order and the
         FMA contraction of the device's double sums differ; equal values, -inf dB of silence among them, pass);
       - cSpectral on the log spectrum (useLogSpectrum = 1): the kernel's log tile is its own logf of each bin, which differs
         from the C library's by up to one ulp on some bins (measured on the H100: flatness 6 ulps, skewness / kurtosis 1e-5 of
         the column scale apart).  Every column is held to 1e-5 of the column scale, and max / min positions (comparisons of
         dB values that can be equal to within that ulp) may differ on 1 % of the frames; the impulse train is not compared:
         its flat log spectrum turns entropy, positions and harmonicity peaks into decisions between values equal up to that
         ulp (measured up to 0.37 of the column scale for the entropy);
       - cPitchACF: the lag decisions (F0raw) and the smoothed F0 / F0env equal, unless the oracle's cepstrum has a near-tie at the
         frame (a lag within 1e-6 of the threshold or of its neighbour, relative to the cepstrum's peak), counted, at most 0.1 % of
         the frames; the per-frame values (voicing, HNR, voiceQual) within 1e-4 of the column scale, as test_parity_gpu.py holds
         them: they go through the kernel's own float FFT of the spectrum, which the oracle computes as a double sum;
  2. time ops: bit for bit against the oracle on the PCM;
  3. from PCM, the whole chain against the oracle's (sanity: the tolerances of test_parity_gpu.py on the voiced / mixed signals;
     the log-spectral skewness and kurtosis, third and fourth moments of dB values that carry the two FFTs' rounding, only in 1.).
Then batch invariance over ragged batches of about 2 000 utterances that run_host cuts into pieces, the two defects this table
found (FFT 4096 with a log spectrum, preskip past the ACF's lags), and a final check that every kernel instance and staging path
of the table ran."""
import time

import numpy as np
import pytest

import spectral_cases as SC
from opensmile_b200 import Plan, pack_utterances
from opensmile_b200.synth import mixed_pcm, stereo_mixed_pcm

pytestmark = pytest.mark.gpu
OBSERVED = {}        # case -> (kernel, staged, tile width) or (kernel, FFT size)
_T0 = time.time()
FLOAT_COLS = ("alphaRatio", "hammarberg", "Sharpness", "Harmonicity", "Flatness")
POS_COLS = ("RollOff", "MaxPos", "MinPos")


def _bits_equal(a, b):
    return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32))


def _ulps(a, b):
    ia = np.ascontiguousarray(a, np.float32).view(np.int32).astype(np.int64)
    ib = np.ascontiguousarray(b, np.float32).view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7fffffff), ia)
    ib = np.where(ib < 0, -(ib & 0x7fffffff), ib)
    return np.abs(ia - ib)


def _tile_width(kernel):
    return 32 if kernel.startswith("lld512") else int(kernel.split("<")[1].split(",")[1])


def _run(c, level, pcm, off, profile=False):
    import torch
    p = Plan(SC.components(c), level, device=0)
    try:
        fo = p.frame_offsets(off)
        if profile:
            p.set_profiling(True)
            out = p.run_device(torch.from_numpy(pcm).cuda(), off)
            torch.cuda.synchronize()
            out = out.cpu().numpy()
            names = [n for n, _ in p.kernel_profile()]
        else:
            out, names = p.run_host(pcm, off), []
        _run.info = p.last_run_info()
        return out, fo, p.last_lld_launch().kernel, names, p.element_names
    finally:
        p.close()


def _check_spectral(c, got, ref, names, flat):
    """-> list of failures (column, kind, worst); got / ref = every row of the case, flat = rows of the impulse signal"""
    bad = []
    scale = np.abs(np.where(np.isfinite(ref), ref, 0)).max(axis=0) if ref.size else np.ones(ref.shape[1])
    scale = np.where(scale > 0, scale, 1.0)
    for k, nm in enumerate(names):
        g, r = got[:, k], ref[:, k]
        if c["log"]:
            g, r = g[~flat], r[~flat]
        same = (g == r) | (np.isnan(g) & np.isnan(r))
        if any(s in nm for s in POS_COLS):
            if (~same).sum() > (max(1, len(g) // 100) if c["log"] else 0):
                bad.append((nm, "frames differ", int((~same).sum())))
        elif any(s in nm for s in FLOAT_COLS) and not c["log"]:
            u = int(np.where(same, 0, _ulps(g, r)).max(initial=0))
            if u > 2:
                bad.append((nm, "ulps", u))
        else:
            e = float(np.where(same, 0.0, np.abs(g.astype(np.float64) - r) / scale[k]).max(initial=0))
            if not e <= (1e-5 if c["log"] else 1e-6):
                bad.append((nm, "rel", e))
    return bad


def _cep_near_tie(cep, n, skip, t):
    """the oracle's cepstrum of frame t has a lag within 1e-6 (of its peak) of pitchPeak's threshold or of a neighbour"""
    a = cep[t].astype(np.float64)
    mx = max(a[n - 1], a[skip:].max(initial=-np.inf))
    thr = (mx + np.abs(a).sum() / n) * 0.6
    eps = 1e-6 * max(np.abs(a).max(), 1e-30)
    seg = a[skip + 1:n - 1]
    return bool((np.abs(seg - thr) <= eps).any() or (np.abs(np.diff(a[skip:n])) <= eps).any())


def _check_pitch(c, got, ref, cep, names):
    """-> (failures, excused frames)"""
    bad, excused = [], 0
    col = {nm: k for k, nm in enumerate(names)}
    n, skip = cep.shape[1], SC.preskip(c) + 1
    dec = [col[x] for x in ("F0raw", "F0", "F0env") if x in col]
    flip = np.zeros(len(got), bool)
    if "F0raw" in col:
        flip = got[:, col["F0raw"]] != ref[:, col["F0raw"]]
    elif dec:
        flip = (got[:, dec] != ref[:, dec]).any(axis=1)
    for t in np.nonzero(flip)[0]:
        if _cep_near_tie(cep, n, skip, t):
            excused += 1
        else:
            bad.append(("lag decision", "frame", int(t)))
    if not flip.any() and dec and not np.array_equal(got[:, dec], ref[:, dec]):
        bad.append(("F0 / F0env", "differ without a lag flip", int((got[:, dec] != ref[:, dec]).any(axis=1).sum())))
    keep = ~flip
    for nm, k in col.items():
        if k in dec:
            continue
        scale = max(float(np.abs(ref[:, k]).max(initial=0)), 1e-6)
        e = float(np.abs(got[keep, k] - ref[keep, k]).max(initial=0)) / scale
        if not e <= 1e-4:
            bad.append((nm, "rel", e))
    return bad, excused


SPEC_PITCH = [n for n, c in SC.BY_NAME.items() if c["op"] in ("spectral", "pitch")]
TIME = [n for n, c in SC.BY_NAME.items() if c["op"] not in ("spectral", "pitch")]


@pytest.mark.parametrize("name", SPEC_PITCH)
def test_case_stage_by_stage(name):
    c = SC.BY_NAME[name]
    utts, pcm, off = SC.batch(c)
    mag, fo_m, k_mag, _, _ = _run(c, "mag", pcm, off)
    out, fo, k_op, kernels, names = _run(c, SC.level(c), pcm, off, profile=True)
    assert k_mag == k_op, (k_mag, k_op)                     # one LLD instance produced the magnitudes both runs read
    assert np.array_equal(fo, fo_m)
    N, S, nfft = SC.geometry(c)
    if c["op"] == "spectral":
        assert "spectral_kernel" in kernels, kernels
        staged = _run.info.spectral_staged                           # the path the launcher took, reported by the plan
        assert staged in (0, 1) and _run.info.spectral_smem <= 232448
        OBSERVED[name] = ("spectral_kernel", staged, _tile_width(k_op))
    else:
        assert "acf_pitch_kernel" in kernels and "pitch_smooth_kernel" in kernels, kernels
        OBSERVED[name] = ("acf_pitch_kernel", nfft)
    failures, excused, frames, refs = [], 0, 0, []
    flat = np.zeros(len(out), bool)
    flat[fo[-2]:fo[-1]] = True                                    # the last utterance is the impulse train
    for u in range(len(utts)):
        m = mag[fo[u]:fo[u + 1]]
        got = out[fo[u]:fo[u + 1]]
        frames += len(got)
        if c["op"] == "spectral":
            refs.append(SC.oracle_from_mag(c, m) if len(got) else np.zeros((0, out.shape[1]), np.float32))
        elif len(got):
            from oracle import oracle
            ref, _, cep = oracle.pitchacf_from_mag(m, SC.frontend(c), SC.oracle_cfg(c), taps=True)
            refs.append(ref)
            f, e = _check_pitch(c, got, ref, cep, names)
            failures += [x for x in f if x[1] != "rel"]
            excused += e
    if c["op"] == "spectral":
        failures = _check_spectral(c, out, np.concatenate(refs), names, flat)
    else:
        ref = np.concatenate(refs)
        scale = np.maximum(np.abs(ref).max(axis=0), 1e-6)
        dec = [k for k, nm in enumerate(names) if nm.startswith("F0")]
        keep = (out[:, dec] == ref[:, dec]).all(axis=1) if dec else np.ones(len(ref), bool)
        for k, nm in enumerate(names):
            if k not in dec:
                e = float((np.abs(out[keep, k] - ref[keep, k]) / scale[k]).max(initial=0))
                if not e <= 1e-4:
                    failures.append((nm, "rel", e))
    assert not failures, failures[:12]
    assert excused <= frames // 1000, (excused, frames)
    print("\n%s: %s, %d frames, %d near-ties excused" % (name, OBSERVED[name], frames, excused))


@pytest.mark.parametrize("name", TIME)
def test_time_op_bit_exact(name):
    c = SC.BY_NAME[name]
    utts, pcm, off = SC.batch(c)
    out, fo, _, kernels, _ = _run(c, SC.level(c), pcm, off, profile=True)
    assert "%s_kernel" % c["op"] in kernels, kernels
    OBSERVED[name] = ("%s_kernel" % c["op"],)
    for u, x in enumerate(utts):
        ref = SC.oracle_rows(c, x)
        got = out[fo[u]:fo[u + 1]]
        assert _bits_equal(got, ref), (u, got.shape, ref.shape, np.abs(got - ref).max(axis=0) if got.shape == ref.shape else None)


@pytest.mark.parametrize("name", SPEC_PITCH)
def test_case_end_to_end(name):
    """from PCM against the oracle's whole chain, on the voiced and mixed utterances: continuous columns within 2e-5 (1e-4 with a
    log spectrum, whose dB values of bins far below the peak carry the FFT's rounding, see test_parity_gpu.py) of the column scale;
    bin-frequency and lag decisions may differ on at most 1 % of the frames"""
    c = SC.BY_NAME[name]
    utts, pcm, off = SC.batch(c)
    out, fo, _, _, names = _run(c, SC.level(c), pcm, off)
    tol = 1e-4 if (c["op"] == "pitch" or c["log"]) else 2e-5
    dec = [k for k, nm in enumerate(names) if any(s in nm for s in POS_COLS + ("F0",))]
    skip = [k for k, nm in enumerate(names) if c["op"] == "spectral" and c["log"] and ("Skewness" in nm or "Kurtosis" in nm)]
    differ, frames = 0, 0
    for u, x in enumerate(utts):
        if not (u < 2 + len(SC.frame_counts(c)) or u == len(utts) - len(SC.KINDS)):     # voiced / mixed only
            continue
        ref = SC.oracle_rows(c, x)
        got = out[fo[u]:fo[u + 1]]
        assert got.shape == ref.shape
        if not len(ref):
            continue
        frames += len(ref)
        flip = (got[:, dec] != ref[:, dec]).any(axis=1) if dec else np.zeros(len(ref), bool)
        differ += int(flip.sum())
        for k in range(ref.shape[1]):
            if k in dec or k in skip:
                continue
            g, r = got[~flip, k], ref[~flip, k]
            scale = max(float(np.abs(r[np.isfinite(r)]).max(initial=0)), 1e-30)
            err = np.where(g == r, 0.0, np.abs(g.astype(np.float64) - r))
            assert float(err.max(initial=0)) <= tol * scale, (u, names[k])
    assert differ <= max(1, frames // 100), (differ, frames)


# ---------------------------------------------------------------- batch invariance
def _big_batch(c, n_utt, seed):
    """ragged lengths: 0, shorter than a frame, one tile and one tile +- 1 frame, mostly up to 3 tiles, 8 % of 30 to 50 tiles (the
    batch passes 24 MB of PCM, so run_host cuts it into pieces); slices of one long signal at every start residue"""
    rng = np.random.default_rng(seed)
    N, S, _ = SC.geometry(c)
    F = SC.tile_guess(c)
    T = np.where(rng.random(n_utt) < 0.08, rng.integers(30 * F, 50 * F, n_utt), rng.integers(0, 3 * F, n_utt))
    T[:6] = [0, 0, F, F - 1, F + 1, 1]
    L = np.where(T > 0, N + (T - 1) * S + rng.integers(0, S, n_utt), rng.integers(0, N, n_utt))
    L[:2] = [0, N - 1]
    nc, n_base = c["n_chan"], int(L.max()) + 100_000
    base = (stereo_mixed_pcm if nc == 2 else mixed_pcm)(n_base, int(c["sr"]), seed=seed)
    starts = rng.integers(0, n_base - L, n_utt)
    return [base[s * nc:(s + n) * nc] for s, n in zip(starts, L)]


@pytest.mark.parametrize("name,n_utt", [("anchor_compare16", 2000), ("s_all_4096_log", 1500), ("s_all_2048_log_stereo", 1500),
                                        ("p_anchor", 2000), ("p_2048", 1500)])
def test_rows_do_not_depend_on_the_batch(name, n_utt):
    """every utterance's rows alone equal its rows inside the ragged batch, reversed too: spectral flux reads the previous frame
    across tile and piece boundaries, and the pitch smoothing runs per utterance"""
    c = SC.BY_NAME[name]
    utts = _big_batch(c, n_utt, seed=len(name))
    pcm, off = pack_utterances(utts, n_chan=c["n_chan"])
    p = Plan(SC.components(c), SC.level(c), device=0)
    try:
        fo = p.frame_offsets(off)
        out = p.run_host(pcm, off)
        assert p.last_run_info().pieces >= 2, p.last_run_info()      # piece boundaries are crossed
        rpcm, roff = pack_utterances(utts[::-1], n_chan=c["n_chan"])
        rev = p.run_host(rpcm, roff)
        rfo = p.frame_offsets(roff)
        for u in range(n_utt):
            r = n_utt - 1 - u
            assert _bits_equal(rev[rfo[r]:rfo[r + 1]], out[fo[u]:fo[u + 1]]), u
        for u in list(range(6)) + list(np.random.default_rng(7).choice(n_utt, 30, replace=False)):
            alone = p.run_host(utts[u], np.array([0, len(utts[u]) // c["n_chan"]], np.int64))
            assert _bits_equal(alone, out[fo[u]:fo[u + 1]]), u
    finally:
        p.close()


# ---------------------------------------------------------------- the defects the table found
def test_fft4096_log_spectrum_runs_and_matches_the_oracle():
    """useLogSpectrum = 1 on 25 ms frames at 96 kHz (FFT 4096): the log tile holds one column per frame of the 8-frame tile
    (64 KB); sized for 32 frames it needed 262 272 B, beyond the 232 448 B a block may opt into, and the run failed"""
    c = SC.BY_NAME["s_all_4096_log"]
    utts, pcm, off = SC.batch(c)
    mag, fo, _, _, _ = _run(c, "mag", pcm, off)
    out, fo2, _, _, names = _run(c, SC.level(c), pcm, off)
    ref = np.concatenate([SC.oracle_from_mag(c, mag[fo[u]:fo[u + 1]]) for u in range(len(utts))])
    flat = np.zeros(len(out), bool)
    flat[fo[-2]:fo[-1]] = True
    assert not _check_spectral(c, out, ref, names, flat)


@pytest.mark.parametrize("name", ["p_preskip_at_n", "p_preskip_between_n_2n"])
def test_preskip_past_n_reads_the_cepstrum(name):
    """maxPitch below sr / n: preskip >= n, and the voicing mean starts with element preskip of [acf ; cepstrum], a cepstrum value.
    The mean only reaches the rows through voiceQual, which is 0 whenever the cepstral peak search (from lag preskip + 2) finds no
    lag, as it cannot here: the rows equal the oracle's, but this does not tell the cepstrum value from the mirrored ACF value
    the kernel used to read.  The change that shows is the refusal from preskip = 2n on (test_spectral_sweep_cpu.py), where the
    kernel read past its FFT tile"""
    from oracle import oracle
    c = SC.BY_NAME[name]
    utts, pcm, off = SC.batch(c)
    mag, fo, _, _, _ = _run(c, "mag", pcm, off)
    out, _, _, _, names = _run(c, SC.level(c), pcm, off)
    k = names.index("voiceQual")
    for u in range(len(utts)):
        ref = oracle.pitchacf_from_mag(mag[fo[u]:fo[u + 1]], SC.frontend(c), SC.oracle_cfg(c))
        got = out[fo[u]:fo[u + 1]]
        scale = max(float(np.abs(ref[:, k]).max(initial=0)), 1e-6)
        assert float(np.abs(got[:, k] - ref[:, k]).max(initial=0)) <= 1e-4 * scale, u


def test_acf_refuses_fft4096_on_a_device_plan():
    """acf_pitch_kernel has instances for FFT 512, 1024 and 2048: 25 ms frames at 96 kHz (FFT 4096) are refused when the plan is
    opened on the device, with the message"""
    from opensmile_b200 import comp, components_frontend
    cs = components_frontend(96000.0, 0.025, 0.010, win="gau", zero_pad_symmetric=0) + [
        comp("cAcf", "acf", "mag", "acf"), comp("cAcf", "cep", "mag", "cepstrum", cepstrum=1, usePower=0),
        comp("cPitchACF", "pitch", "acf;cepstrum", "pitch", F0=1)]
    with pytest.raises(RuntimeError, match="cAcf / cPitchACF: FFT size must be 512, 1024 or 2048"):
        Plan(cs, "pitch", device=0)


def test_every_instance_and_path_of_the_table_ran():
    """acf_pitch_kernel at FFT 512 / 1024 / 2048; spectral_kernel staged (a log spectrum up to FFT 1024) and unstaged, at the tile
    widths 32, 16 and 8 (and the narrow 4 of FFT 4096); each time op"""
    if set(OBSERVED) != set(SC.BY_NAME):
        pytest.skip("only %d of %d cases ran" % (len(OBSERVED), len(SC.BY_NAME)))
    seen = set(OBSERVED.values())
    print("\ninstances covered (%d cases, %.0f s): %s" % (len(OBSERVED), time.time() - _T0, sorted(seen, key=str)))
    assert {("acf_pitch_kernel", n) for n in (512, 1024, 2048)} <= seen
    spec = {v for v in seen if v[0] == "spectral_kernel"}
    assert {v[1] for v in spec} == {0, 1}
    assert {v[2] for v in spec if v[1] == 0} >= {32, 16, 8}
    assert {v[2] for v in spec if v[1] == 1} >= {32}
    assert {("energy_kernel",), ("mzcr_kernel",), ("intensity_kernel",)} <= seen
