"""Every per-frame LLD kernel instance (lld512_kernel<13|16>, the lld_kernel family) over the case table of tests/lld_cases.py:
frame geometries, band and cepstrum layouts, regression windows, ragged batches with misaligned starts, and batches of more
chunks than CTAs.  Per case: the instance that ran, the statics against the oracle, the delta / delta-delta columns bit for bit
against the oracle's regression chain on the kernel's own statics, the fused regression against post_kernel, the fast instance
against lld_kernel, and batch invariance of every utterance's rows."""
import os
import subprocess
import sys
import time

import numpy as np
import pytest

import lld_cases as LC
from conftest import ROOT, assert_columns_close, rel_to_frame_scale
from opensmile_b200 import Plan, pack_utterances
from opensmile_b200.synth import mixed_pcm, stereo_mixed_pcm
from oracle import oracle

pytestmark = pytest.mark.gpu
TOL = 1e-5
OBSERVED = {}        # case -> instance that ran
ROWS = {}            # case -> rows of the default run
_STATIC = {}         # (configuration, signal) -> the oracle's statics
_T0 = time.time()


def _bits_equal(a, b):
    return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32))


def _oracle_static(c, x):
    cfg = tuple((k, v) for k, v in sorted(c.items()) if k not in ("name", "expect", "windows", "extremes"))
    key = (cfg, len(x), hash(x.tobytes()))
    if key not in _STATIC:
        ref = LC.oracle_rows(c, x)
        _STATIC[key] = np.ascontiguousarray(ref[:, :ref.shape[1] // 3])
    return _STATIC[key]


def _run(c, pcm, off):
    p = Plan(LC.components(c), "lld", device=0)
    try:
        out = p.run_host(pcm, off)
        return out, p.frame_offsets(off), p.last_lld_launch(), p.last_launch_count()
    finally:
        p.close()


def _check_statics(c, utts, out, fo):
    """shape = the oracle's T; statics within 1e-5 of the frame scale and to the MFCC / PLP column rule over the batch"""
    K = out.shape[1] // 3
    got_all, ref_all = [], []
    for u, x in enumerate(utts):
        ref = _oracle_static(c, x)
        got = out[fo[u]:fo[u + 1]]
        assert got.shape == (ref.shape[0], 3 * K), (u, got.shape, ref.shape)
        if ref.shape[0]:
            assert rel_to_frame_scale(got[:, :K], ref) < TOL, (u, ref.shape[0], rel_to_frame_scale(got[:, :K], ref))
            got_all.append(got[:, :K])
            ref_all.append(ref)
    assert_columns_close(np.concatenate(got_all), np.concatenate(ref_all))


@pytest.mark.parametrize("name", list(LC.BY_NAME))
def test_case(name, monkeypatch):
    c = LC.BY_NAME[name]
    utts, pcm, off = LC.batch(c)
    out, fo, info, launches = _run(c, pcm, off)
    OBSERVED[name] = info.kernel
    ROWS[name] = out, fo
    # statics against the oracle
    _check_statics(c, utts, out, fo)
    # the regression columns are exact: the oracle's chain (n0 = T, then the produced level's c0) on the kernel's statics
    K = out.shape[1] // 3
    w1, w2 = c["windows"]
    for u in range(len(utts)):
        got = out[fo[u]:fo[u + 1]]
        T = got.shape[0]
        if T == 0:
            continue
        d, c0 = oracle.delta_chained(got[:, :K], w1, T)
        dd, _ = oracle.delta_chained(d, w2, c0)
        for lo, ref, what in ((K, d[:T], "delta"), (2 * K, dd[:T], "delta-delta")):
            bad = np.nonzero((got[:, lo:lo + K].view(np.uint32) != ref.view(np.uint32)).any(axis=1))[0]
            assert bad.size == 0, "%s of utterance %d (T = %d): %d rows differ, first %s" % (what, u, T, bad.size, bad[:8])
    # the instance the table names, fused into it or followed by post_kernel as the halo rule says
    assert info.kernel == c["expect"]
    assert launches == (1 if LC.expect_fused(c) else 2), launches
    # the fused regression against the two-kernel path
    if LC.expect_fused(c):
        monkeypatch.setenv("OSM_B200_NO_FUSE", "1")
        two, _, _, launches2 = _run(c, pcm, off)
        assert launches2 == 2
        assert _bits_equal(out, two)


# ---------------------------------------------------------------- lld512_kernel against lld_kernel
FAST = [n for n, c in LC.BY_NAME.items() if LC.is_fast(c)]
_CHILD = r"""
import sys
import numpy as np
sys.path[:0] = [sys.argv[2], sys.argv[3]]
import lld_cases as LC
from opensmile_b200 import Plan
res = {}
for name in sys.argv[4:]:
    c = LC.BY_NAME[name]
    _, pcm, off = LC.batch(c)
    p = Plan(LC.components(c), "lld", device=0)
    res["rows_" + name] = p.run_host(pcm, off)
    res["kernel_" + name] = np.array(p.last_lld_launch().kernel)
    p.close()
np.savez(sys.argv[1], **res)
"""


@pytest.fixture(scope="module")
def generic_rows(tmp_path_factory):
    """the fast-path cases in a child process with OSM_B200_LLD_FAST=0 (read once per process)"""
    path = str(tmp_path_factory.mktemp("lld_generic") / "rows.npz")
    env = dict(os.environ, OSM_B200_LLD_FAST="0")
    subprocess.run([sys.executable, "-c", _CHILD, path, ROOT, os.path.join(ROOT, "tests")] + FAST, env=env, check=True, cwd=ROOT)
    with np.load(path) as z:
        return {k: z[k] for k in z.files}


@pytest.mark.parametrize("name", FAST)
def test_fast_and_generic_instances_both_meet_the_oracle(name, generic_rows):
    """Not bit-identical by design: lld512 forms the power with one FMA where lld_kernel rounds twice, and the two factor the FFT
    differently.  Both are held to the oracle; the largest difference between them is printed."""
    c = LC.BY_NAME[name]
    utts, pcm, off = LC.batch(c)
    fast, fo = ROWS[name] if name in ROWS else _run(c, pcm, off)[:2]
    gen = generic_rows["rows_" + name]
    assert str(generic_rows["kernel_" + name]) == LC.G512
    _check_statics(c, utts, fast, fo)
    _check_statics(c, utts, gen, fo)
    K = fast.shape[1] // 3
    scale = np.abs(fast[:, :K]).max(axis=1, keepdims=True)
    scale[scale == 0] = 1.0
    print("\n%s: lld512 vs lld_kernel, statics: max |diff| = %.3g, max |diff| / frame scale = %.3g, all columns: %.3g"
          % (name, float(np.abs(fast[:, :K] - gen[:, :K]).max()), float((np.abs(fast[:, :K] - gen[:, :K]) / scale).max()),
             float(np.abs(fast - gen).max())))


# ---------------------------------------------------------------- batch invariance with more chunks than CTAs
def _big_batch(c, n_utt, seed):
    """seeded ragged lengths: mostly up to 3 tiles, 8 % of one to two and a half chunks, every start residue; slices of one
    long signal"""
    rng = np.random.default_rng(seed)
    N, S, F = c["frame"], c["hop"], LC.tile_frames(c)
    long_ = rng.random(n_utt) < 0.08
    T = np.where(long_, rng.integers(16 * F, 40 * F, n_utt), rng.integers(0, 3 * F, n_utt))
    L = np.where(T > 0, N + (T - 1) * S + rng.integers(0, S, n_utt), rng.integers(0, N, n_utt))
    nc, n_base = c["n_chan"], int(L.max()) + 100_000
    base = (stereo_mixed_pcm if nc == 2 else mixed_pcm)(n_base, int(c["sr"]), seed=seed)
    starts = rng.integers(0, n_base - L, n_utt)
    return [base[s * nc:(s + n) * nc] for s, n in zip(starts, L)]


BIG = [("fast_anchor_400_160", 2500), ("fast_8k_480_80", 2500), ("gen2048_48k_mono", 2500), ("win22_48k_stereo", 2000),
       ("win33_48k_stereo", 2000)]


@pytest.mark.parametrize("name,n_utt", BIG)
def test_rows_do_not_depend_on_the_batch(name, n_utt):
    import torch
    c = LC.BY_NAME[name]
    utts = _big_batch(c, n_utt, seed=len(name))
    pcm, off = pack_utterances(utts, n_chan=c["n_chan"])
    p = Plan(LC.components(c), "lld", device=0)
    try:
        fo = p.frame_offsets(off)
        dev = p.run_device(torch.from_numpy(pcm).cuda(), off)
        torch.cuda.synchronize()
        info = p.last_lld_launch()
        dev = dev.cpu().numpy()
        assert info.kernel == c["expect"]
        assert info.n_chunks >= 4 * info.grid, info
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
    print("\n%s: %d utterances, %d rows, %d chunks on %d CTAs" % (name, n_utt, dev.shape[0], info.n_chunks, info.grid))


def test_every_instance_of_the_table_ran():
    """the set of instances observed equals the set the table names (coverage is checked, not assumed)"""
    if set(OBSERVED) != set(LC.BY_NAME):
        pytest.skip("only %d of %d cases ran" % (len(OBSERVED), len(LC.BY_NAME)))
    seen = set(OBSERVED.values())
    print("\ninstances covered (%d cases, %.0f s): %s" % (len(OBSERVED), time.time() - _T0, ", ".join(sorted(seen))))
    assert seen == {c["expect"] for c in LC.CASES}
