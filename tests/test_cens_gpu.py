"""cCens on the device, on both chroma paths (tests/configs/cens_taps.conf):
- the device's CENS rows equal, bit for bit, the restatement (tests/cens_oracle.py) applied to the device's own chroma rows (the same
  configuration with the chroma level as the output level), over a ragged batch with empty, 1-row, W - 1, W and W + 1 row
  utterances and one of 600 s;
- the rows are the same alone, in the batch and on a rerun;
- against the reference end to end (tests/golden/cens_goldens.npz): quantisation turns round-off near 0.05 / 0.1 / 0.2 / 0.4 into
  steps, so rows whose window holds a reference chroma value within 1e-4 of a threshold are excluded, the rest agree within 1e-6;
- cFunctionals over the CENS level (FFT path, tests/configs/cens_func.conf) against the reference's summaries, with values in seconds
  at downsampleRatio 1, 3 and 10."""
import os

import numpy as np
import pytest

from cens_harness import G, HERE, case_input, cens_oracle, mg, session
from opensmile_b200 import Session

pytestmark = pytest.mark.gpu

W = 41
FUNC = os.path.join(HERE, "configs", "cens_func.conf")


def lengths(path):
    """sample counts at 16 kHz that give 0, 1, W - 1, W, W + 1 rows and 600 s (FFT rows: 1024-sample frames, hop 160; filter rows:
    blocks of 160 samples)"""
    if path == "fft":
        rows = lambda r: 0 if r == 0 else 1024 + (r - 1) * 160      # noqa: E731
    else:
        rows = lambda r: r * 160 - 37 if r else 0                    # noqa: E731
    return [rows(0), rows(1), rows(W - 1), rows(W), rows(W + 1), 600 * 16000, rows(3), rows(2 * W + 5)]


def batch_pcm(lens, seed=0):
    rng = np.random.default_rng(seed)
    t = np.arange(max(lens)) / 16000.0
    parts = []
    for i, n in enumerate(lens):
        f = 110.0 * 2 ** (i / 5.0)
        x = 6000 * np.sin(2 * np.pi * f * t[:n]) + 3000 * np.sin(2 * np.pi * 1.5 * f * t[:n]) + rng.normal(0, 300, n)
        x[: n // 7] *= 0.0                                            # a silent start: zero-norm rows
        parts.append(np.clip(np.round(x), -32768, 32767).astype(np.int16))
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    return np.concatenate(parts), off


def run(level, pcm, off, sr=16000, **opts):
    s = session(level, device=0, **opts)
    rows, fo = s.extract_pcm(pcm, off, float(sr))
    s.close()
    return rows, fo


VARIANTS = [dict(), dict(window="ham", winlength=101, downsampleRatio=10), dict(window="bar", winlength=7, l2norm=0),
            dict(winlength=512), dict(winlength=1)]


@pytest.mark.parametrize("path", ["fft", "filt"])
@pytest.mark.parametrize("vi", range(len(VARIANTS)))
def test_device_rows_equal_the_restatement_of_the_device_chroma(path, vi):
    o = dict(mg.BASE)
    o.update(VARIANTS[vi])
    lens = lengths(path)
    pcm, off = batch_pcm(lens)
    ch, fo = run("chroma_" + path, pcm, off, **o)
    ce, fo2 = run("cens_" + path, pcm, off, **o)
    assert np.array_equal(fo, fo2)
    counts = np.diff(fo)
    assert list(counts[:5]) == [0, 1, W - 1, W, W + 1], counts
    for u in range(len(lens)):
        a, b = fo[u], fo[u + 1]
        want = cens_oracle.cens(ch[a:b], o["window"], o["winlength"], o["l2norm"])
        assert np.array_equal(ce[a:b].view(np.uint32), want.view(np.uint32)), (u, np.argwhere(ce[a:b].view(np.uint32) != want.view(np.uint32))[:5])
    # alone, in the batch, on a rerun
    again, _ = run("cens_" + path, pcm, off, **o)
    assert np.array_equal(again.view(np.uint32), ce.view(np.uint32))
    for u in (1, 3, 5):
        alone, fa = run("cens_" + path, pcm[off[u]:off[u + 1]], np.array([0, lens[u]], np.int64), **o)
        assert np.array_equal(alone.view(np.uint32), ce[fo[u]:fo[u + 1]].view(np.uint32))


def near_threshold_rows(chroma, winlength, tol=1e-4):
    """rows whose window (the row and the winlength - 1 before it) holds a chroma value within tol of a quantisation threshold"""
    x = chroma.astype(np.float64)
    near = np.zeros(x.shape[0], bool)
    for th in (0.05, 0.1, 0.2, 0.4):
        near |= (np.abs(x - th) < tol).any(axis=1)
    idx = np.flatnonzero(near)
    out = np.zeros_like(near)
    for i in idx:
        out[i:i + max(int(winlength), 1)] = True
    return out


@pytest.mark.parametrize("path", ["fft", "filt"])
@pytest.mark.parametrize("case", sorted(mg.CASES))
def test_against_the_reference_end_to_end(case, path):
    pcm, sr = case_input(case)
    o = mg.options(case)
    got, fo = run("cens_" + path, pcm, np.array([0, pcm.size], np.int64), sr, **o)
    ref = G["cens_%s_%s" % (path, case)]
    assert got.shape == ref.shape
    skip = near_threshold_rows(G["chroma_%s_%s" % (path, case)], o["winlength"])
    keep = ~skip
    nan = np.isnan(ref)
    assert np.array_equal(np.isnan(got[keep]), nan[keep])
    err = np.abs(np.where(nan, 0, got) - np.where(nan, 0, ref))[keep]
    assert err.size == 0 or err.max() <= 1e-6, (err.max(), int(skip.sum()), ref.shape[0])
    print("%s/%s: %d of %d rows excluded" % (case, path, int(skip.sum()), ref.shape[0]))


@pytest.mark.parametrize("fc", sorted(mg.FUNC_CASES))
def test_functionals_over_cens_against_the_reference(fc):
    """cFunctionals over the FFT path's CENS level (tests/configs/cens_func.conf): Means, and Extremes / Times in seconds, whose
    values scale with the level period (its input's times downsampleRatio); within 1e-4 of each value's magnitude"""
    sig, ds = mg.FUNC_CASES[fc]
    pcm, sr = G["pcm_" + sig], int(G["sr_" + sig])
    s = Session(FUNC, options={"downsampleRatio": str(ds), "funchtk": "?", "funccsv": "x.csv"}, device=0)
    names = s.element_names(float(sr))
    got, _ = s.extract_pcm(pcm, np.array([0, pcm.size], np.int64), float(sr))
    s.close()
    ref = G["func_" + fc]
    assert names == [str(x) for x in G["names_func"]]
    assert got.shape == ref.shape
    err = np.abs(got.astype(np.float64) - ref) / np.maximum(np.abs(ref), 1e-6)
    assert err.max() <= 1e-4, (names[int(err.argmax())], got.reshape(-1)[int(err.argmax())], ref.reshape(-1)[int(err.argmax())])
