"""cTonefilt / cChroma on a cTonefilt level on the device (tonefilt.cu) against the unmodified reference's levels
(tests/golden/tonefilt_goldens.npz, tests/golden/chroma_filt_*.csv, scripts/make_golden_tonefilt.py) and against the C
restatement of the reference (tests/native/tonefilt_oracle.c).  Bound: 1e-6 of the column scale everywhere.

silThresh: a chroma vector is zeroed when one unnormalised value lies below silThresh.  A frame whose smallest value lies within
1e-6 (relative) of the threshold could decide differently from the reference; test_levels_against_the_reference lists every such
frame of the goldens with its margin (none is expected)."""
import os

import numpy as np
import pytest

from tonefilt_harness import G, SHIPPED, SIGS, col_err, mg, oracle_tf, session, wave_level
from opensmile_b200 import Plan, Session
from oracle import chroma_oracle as co

pytestmark = pytest.mark.gpu
TOL = 1e-6


def tap_plan(level, sr, nc=1, fmt=0, **opts):
    s = session(level, **opts)
    comps, lvl = s.components(float(sr), nc)
    s.close()
    assert lvl == level
    for c in comps:
        if c.type == 0:
            c.u.wavesource.format = fmt
    return Plan(list(comps), lvl, device=0)


def run(plan, utts, nc=1):
    pcm = np.concatenate([np.asarray(u).reshape(-1) for u in utts])
    off = np.concatenate([[0], np.cumsum([u.size // nc for u in utts])]).astype(np.int64)
    rows = plan.run_host(pcm, off)
    fo = plan.frame_offsets(off)
    return [rows[fo[i]:fo[i + 1]] for i in range(len(utts))]


def sil_margin(tf, K, thresh):
    T, N = tf.shape
    s = tf.reshape(T, N // K, K).astype(np.float32).sum(axis=1)
    return np.abs(s.min(axis=1) - thresh) / thresh


@pytest.mark.parametrize("case", sorted(mg.CASES))
def test_levels_against_the_reference(case):
    sig = mg.CASES[case][0]
    pcm, sr, nc = SIGS[sig]
    o = mg.options(case)
    fmt = 1 if pcm.dtype == np.float32 else 0
    levels = [("tonefilt", "tf")] if o["nNotes"] == 1 else [("tonefilt", "tf"), ("chroma", "chroma"), ("chroma_sma", "sma"),
                                                             ("chroma_sma_de", "de")]
    for level, key in levels:
        plan = tap_plan(level, sr, nc, fmt, **o)
        data = pcm.view(np.int16) if fmt else pcm
        got = run(plan, [data], nc * (2 if fmt else 1))[0] if fmt else run(plan, [pcm], nc)[0]
        plan.close()
        ref = G["%s_%s" % (key, case)]
        assert got.shape == ref.shape, (level, got.shape, ref.shape)
        assert col_err(got, ref) < TOL, (level, col_err(got, ref))
        if level == "chroma":
            rz, gz = (ref == 0).all(axis=1), (got == 0).all(axis=1)
            assert np.array_equal(rz, gz), np.flatnonzero(rz != gz)
            m = sil_margin(G["tf_" + case], o["octaveSize"], o["silThresh"])
            close = np.flatnonzero(m < 1e-6)
            assert close.size == 0, [("%s frame %d" % (case, i), float(m[i])) for i in close]


def ragged_lengths():
    P = 160
    rng = np.random.default_rng(3)
    base = [1, 2, 100, P - 1, P, P + 1, 2 * P - 1, 2 * P, 2 * P + 1]
    more = [int(k * P + r) for k, r in zip(rng.integers(1, 400, 300), rng.integers(0, P, 300))]
    more += [1024 * P + 5, 1025 * P, 1500 * P + 17]             # past one segment: the carry across segments
    return base + more


def test_ragged_batch_matches_the_oracle():
    noise = np.round(np.random.default_rng(9).normal(0, 3000, 1600 * 160)).clip(-32768, 32767).astype(np.int16)
    lens = ragged_lengths()
    rng = np.random.default_rng(4)
    utts = [noise[s:s + n] for s, n in zip(rng.integers(0, noise.size - max(lens), len(lens)), lens)]
    o = dict(mg.BASE)
    plan = tap_plan("tonefilt", 16000, **o)
    got = run(plan, utts)
    plan.close()
    pick = list(range(12)) + list(range(12, len(utts), 17)) + list(range(len(utts) - 3, len(utts)))
    for i in pick:
        ref = oracle_tf(wave_level(utts[i], 1), 16000, o)
        assert got[i].shape == ref.shape and col_err(got[i], ref) < TOL, (i, lens[i], col_err(got[i], ref))


def test_long_utterance_alone_in_a_batch_and_again():
    """one 150 s utterance: 1172 segments' carries, block phases up to 2 pi 3.3 kHz 150 s; bit-identical rows alone, inside a batch
    and from run to run, and within the bound of the restatement"""
    sr = 16000
    t = np.arange(150 * sr) / sr
    x = 6000 * np.sin(2 * np.pi * 440.0 * t) + 3000 * np.sin(2 * np.pi * (200 + 20 * t) * t)
    x = np.round(x + np.random.default_rng(1).normal(0, 500, t.size)).clip(-32768, 32767).astype(np.int16)
    o = dict(mg.BASE)
    plan = tap_plan("chroma", sr, **o)
    alone = run(plan, [x])[0]
    again = run(plan, [x])[0]
    other = [np.round(np.random.default_rng(s).normal(0, 2000, 48000 + 37 * s)).astype(np.int16) for s in range(5)]
    batch = run(plan, other[:2] + [x] + other[2:])[2]
    plan.close()
    assert np.array_equal(alone.view(np.int32), again.view(np.int32))
    assert np.array_equal(alone.view(np.int32), batch.view(np.int32))
    tfp = tap_plan("tonefilt", sr, **o)
    tf = run(tfp, [x])[0]
    tfp.close()
    ref = oracle_tf(wave_level(x, 1), sr, o)
    assert tf.shape == ref.shape and col_err(tf, ref) < TOL, col_err(tf, ref)
    ch = co.chroma(ref, 12, 0.001)[0]
    assert col_err(alone, ch) < TOL, col_err(alone, ch)


@pytest.mark.parametrize("fn,sig", [("chroma_filt_16k.csv", "mix16"), ("chroma_filt_44k1.csv", "rec")])
@pytest.mark.skipif(not os.path.exists(SHIPPED), reason="oracle/_ref/config (build()) not there")
def test_shipped_chroma_filt_csv(tmp_path, fn, sig):
    """config/chroma/chroma_filt.conf unchanged: the session writes the CSV layout the reference wrote (no header, ';', no index or
    time, the same rows), every value within 1e-6 of its column scale"""
    from oracle import refrun
    pcm, sr, nc = SIGS[sig]
    wav, out = str(tmp_path / "in.wav"), str(tmp_path / "out.csv")
    refrun.write_wav(wav, pcm, sr, nc)
    s = Session(SHIPPED, options={"outputfile": out}, device=0)
    s.extract_files([wav], csv_paths=[out])
    s.close()
    ref_lines = open(os.path.join(os.path.dirname(__file__), "golden", fn)).read().strip().split("\n")
    got_lines = open(out).read().strip().split("\n")
    assert len(got_lines) == len(ref_lines)
    ref = np.array([[float(v) for v in ln.split(";")] for ln in ref_lines])
    got = np.array([[float(v) for v in ln.split(";")] for ln in got_lines])
    assert got.shape == ref.shape == (len(ref_lines), 12)
    # the reference's CSV holds 7 significant digits: half a unit of the last one is 5e-7 of the value
    assert col_err(got, ref) < TOL + 5e-7, col_err(got, ref)
