"""The shipped config/emobase/emobase.conf on the GPU, through the C ABI: the stand-alone cLpc / cLsp kernel (lsp.cu) and the
oldCompatCepstrum input stage of acf_pitch_kernel, against the UNMODIFIED reference's rows (tests/golden/emobase_goldens.npz,
scripts/make_golden_emobase.py)."""
import os

import numpy as np
import pytest

import emobase_oracle as eo
from test_emobase_cpu import EMOBASE, G, HERE, REFCONF, needs_conf, signals

pytestmark = [pytest.mark.gpu, needs_conf]


def _session(options=None, level=None, tmp_path=None):
    from opensmile_b200.session import Session
    if level is not None:
        path = tmp_path / "taps.conf"
        path.write_text(open(os.path.join(HERE, "configs", "emobase_taps.conf")).read().replace("REFCONF", REFCONF))
        return Session(str(path), output_level=level, device=0)
    return Session(EMOBASE, options, device=0)


def _run(s, pcms, sr):
    off = np.concatenate([[0], np.cumsum([len(x) for x in pcms])]).astype(np.int64)
    return s.extract_pcm(np.concatenate(pcms).astype(np.int16), off, float(sr), 1)


@pytest.mark.parametrize("key", ["rec", "v", "m", "x"])
def test_lpc_and_lsp_levels(key, tmp_path):
    pcm, sr = signals()[key]
    s = _session(level="lpc", tmp_path=tmp_path)
    lpc, _ = _run(s, [pcm], sr)
    s.close()
    assert np.array_equal(lpc, G["lpc_" + key])              # the reference's float statements, uncontracted: bit-identical
    s = _session(level="lsp", tmp_path=tmp_path)
    lsp, _ = _run(s, [pcm], sr)
    s.close()
    ref = G["lsp_" + key]
    assert lsp.shape == ref.shape
    assert np.array_equal(lsp == 0, ref == 0)                 # zero-filled entries exactly where the reference's are
    scale = np.abs(ref).max(axis=0) + 1e-30
    assert (np.abs(lsp - ref) / scale).max() < 1e-5           # acosf of the device vs the host's libm


@pytest.mark.parametrize("key", ["rec", "v", "m"])
def test_shipped_emobase_lld_and_summary(key):
    pcm, sr = signals()[key]
    s = _session({"lldcsvoutput": "x.csv"})
    rows, fo = _run(s, [pcm], sr)
    s.close()
    ref = G["lld_" + key]
    assert rows.shape == ref.shape
    scale = np.abs(ref).max(axis=0) + 1e-30
    err = np.abs(rows - ref) / scale
    # the project's LLD criterion (smoke()): every column within 5e-5 of its scale, at most 0.1 % of the values beyond 1e-5 (the Δ of
    # MFCC 1 of "v" has one value at 1.1e-5: the MFCC path's own FFT, not the new kernels)
    assert err.max() < 5e-5 and (err > 1e-5).mean() <= 1e-3, (G["names_lld"][int(err.max(axis=0).argmax())], float(err.max()))
    s = _session({"csvoutput": "x.csv"})
    summ, _ = _run(s, [pcm], sr)
    s.close()
    ref = G["func_" + key][0]
    # within 1e-4 of each value's magnitude (the eGeMAPS summaries' tolerance); a summary of a contour that hovers around zero
    # (the median of a delta column) is held to 1e-5 of the scale of the LLD column it summarises instead
    names_lld = [str(x) for x in G["names_lld"]]
    col_scale = np.abs(G["lld_" + key]).max(axis=0)
    floor = np.array([1e-1 * col_scale[max((j for j, n in enumerate(names_lld) if str(f).startswith(n + "_")), key=lambda j: len(names_lld[j]))]
                      for f in G["names_func"]])
    rel = np.abs(summ[0] - ref) / np.maximum(np.abs(ref), floor)
    # skewness / kurtosis of the LSP contours: the device's acosf and glibc's differ by an ulp or two in some lspFreq values, and
    # the third / fourth central moments of a contour with little spread amplify that to ~2e-4
    tol = np.array([5e-4 if "lspFreq" in str(f) and str(f).endswith(("_skewness", "_kurtosis")) else 1e-4 for f in G["names_func"]])
    bad = np.argsort(-(rel / tol))[:5]
    assert (rel < tol).all(), [(str(G["names_func"][j]), float(summ[0][j]), float(ref[j]), float(rel[j])) for j in bad]


def test_ragged_batch_short_utterances_and_run_to_run_identity(tmp_path):
    """1-4 frame utterances between longer ones: every utterance's rows equal its own single run (and the oracle's LPC / LSP),
    and two runs of the batch are bit-identical"""
    pcm, _ = signals()["v"]
    utts = [pcm[:400], pcm[1000:1560], pcm[2000:2720], pcm[3000:3880], pcm, pcm[5000:5800], pcm[:399]]
    for level in ("lpc", "lsp"):
        s = _session(level=level, tmp_path=tmp_path)
        rows, fo = _run(s, utts, 16000)
        again, _ = _run(s, utts, 16000)
        assert np.array_equal(rows, again)
        assert [fo[i + 1] - fo[i] for i in range(len(utts))] == [1, 2, 3, 4, 198, 3, 0]
        for u, x in enumerate(utts):
            a, _, l, _ = eo.lpc_frames(x, 16000, 8)
            got = rows[fo[u]:fo[u + 1]]
            if level == "lpc":
                assert np.array_equal(got, a), u
            else:
                assert np.array_equal(got == 0, l == 0) and (np.abs(got - l) <= 1e-5 * np.pi).all(), u
        s.close()
    s = _session({"lldcsvoutput": "x.csv"})
    rows, fo = _run(s, utts, 16000)
    again, _ = _run(s, utts, 16000)
    assert np.array_equal(rows, again)
    for u in (1, 3, 4, 5):
        one, _ = _run(s, [utts[u]], 16000)
        assert np.array_equal(one, rows[fo[u]:fo[u + 1]]), u
    s.close()


def test_device_sinks_byte_identical_to_host_writers(tmp_path):
    import wave
    pcm, _ = signals()["m"]
    wav = tmp_path / "in.wav"
    with wave.open(str(wav), "wb") as w:
        w.setnchannels(1)
        w.setsampwidth(2)
        w.setframerate(16000)
        w.writeframes(np.ascontiguousarray(pcm, dtype="<i2").tobytes())
    for opts, kind in (({"lldcsvoutput": "x.csv", "lldhtkoutput": "x.htk"}, "lld"), ({"csvoutput": "x.csv"}, "func")):
        s = _session(opts)
        csv_dev, htk_dev = str(tmp_path / (kind + "_d.csv")), str(tmp_path / (kind + "_d.htk"))
        frames = s.extract_files([str(wav)], [htk_dev] if kind == "lld" else None, [csv_dev])
        rows, fo = _run(s, [pcm], 16000)
        csv_host, htk_host = str(tmp_path / (kind + "_h.csv")), str(tmp_path / (kind + "_h.htk"))
        s.write_files(rows, fo, 16000.0, 1, n_samples=np.array([len(pcm)], np.int64),
                      htk_paths=[htk_host] if kind == "lld" else None, csv_paths=[csv_host])
        s.close()
        assert list(frames) == [rows.shape[0]]
        assert open(csv_dev, "rb").read() == open(csv_host, "rb").read()
        if kind == "lld":
            assert open(htk_dev, "rb").read() == open(htk_host, "rb").read()
