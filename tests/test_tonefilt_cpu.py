"""cTonefilt / cChroma on a cTonefilt level without a GPU: the C restatement (tests/native/tonefilt_oracle.c) against the
unmodified reference's levels (tests/golden/tonefilt_goldens.npz, scripts/make_golden_tonefilt.py), the host build of the kernel's
block statements against the restatement, names / row counts / time stamps of description-only sessions, and the refusals."""
import os

import numpy as np
import pytest

from tonefilt_harness import (G, SHIPPED, SIGS, TAPS, col_err, host_chroma, host_tf, mg, oracle_case, oracle_tf,
                              session, wave_level)
from opensmile_b200 import Plan, Session, capi
from opensmile_b200.session import SessionError
from oracle import chroma_oracle as co


def ulps(a, b):
    ia = a.astype(np.float32).view(np.int32).astype(np.int64)
    ib = b.astype(np.float32).view(np.int32).astype(np.int64)
    return int(np.abs(ia - ib).max()) if a.size else 0


@pytest.mark.parametrize("case", sorted(mg.CASES))
def test_oracle_matches_the_reference_levels(case):
    """measured: at most 1 float ulp on the cTonefilt level (libm's sin / cos here and in the reference's build), the chroma,
    smoothing and delta levels within 1e-6 of their column scale"""
    tf, ch = oracle_case(case)
    rt = G["tf_" + case]
    assert tf.shape == rt.shape, (tf.shape, rt.shape)
    assert ulps(tf, rt) <= 1, ulps(tf, rt)
    if ch is None:
        return
    rc = G["chroma_" + case]
    assert ch.shape == rc.shape and col_err(ch, rc) < 1e-6, col_err(ch, rc)
    assert np.array_equal((ch == 0).all(axis=1), (rc == 0).all(axis=1))


@pytest.mark.parametrize("seg", [0, 1, 7, 128])
@pytest.mark.parametrize("case", sorted(mg.CASES))
def test_host_block_statements_match_the_oracle(case, seg):
    """the block form (in-block sums, block phase from the reference's argument, decay d^P per block, segment carries) against
    the per-sample loop, padded last blocks included"""
    sig = mg.CASES[case][0]
    pcm, sr, nc = SIGS[sig]
    o = mg.options(case)
    tf, ch = oracle_case(case)
    got = host_tf(wave_level(pcm, nc), sr, o, seg)
    assert got.shape == tf.shape and col_err(got, tf) < 1e-6, col_err(got, tf)
    if ch is not None:
        gc = host_chroma(got, o["octaveSize"], o["silThresh"])
        assert col_err(gc, ch) < 1e-6 and np.array_equal((gc == 0).all(axis=1), (ch == 0).all(axis=1))


def test_chroma_fold_matches_the_python_oracle():
    tf = G["tf_mix16"]
    assert np.array_equal(host_chroma(tf, 12, 0.001), co.chroma(tf, 12, 0.001)[0])


@pytest.mark.parametrize("case", sorted(mg.CASES))
def test_names_and_rows_of_the_taps(case):
    sig = mg.CASES[case][0]
    pcm, sr, nc = SIGS[sig]
    o = mg.options(case)
    opts = dict(o)
    levels = [("tonefilt", "tf")] if o["nNotes"] == 1 else [("tonefilt", "tf"), ("chroma", "chroma"), ("chroma_sma_de", "de")]
    for level, key in levels:
        s = session(level, **opts)
        assert s.element_names(float(sr), nc) == [str(x) for x in G["names_%s_%s" % (key, case)]]
        fo = s.frame_offsets(np.array([0, pcm.size // nc], np.int64), float(sr), nc)
        assert int(fo[1]) == G["%s_%s" % (key, case)].shape[0]
        s.close()


@pytest.mark.parametrize("case", sorted(c for c in mg.CASES if mg.options(c)["nNotes"] > 1))
def test_row_time_stamps(case):
    """the time of a row is that of its first sample, (double)(r P) / fs, printed "%f"; with outputPeriod 0.0125 at 44.1 kHz
    (P = 551) it is not r * 0.0125"""
    sig = mg.CASES[case][0]
    pcm, sr, nc = SIGS[sig]
    s = session("chroma", **mg.options(case))
    comps, lvl = s.components(float(sr), nc)
    s.close()
    plan = Plan(list(comps), lvl, device=-1)
    L = capi.lib()
    ts = G["ts_" + case]
    got = np.array([float("%f" % L.osm_b200_plan_row_time(plan._h, r)) for r in range(ts.shape[0])])
    plan.close()
    assert np.array_equal(ts[:, 0], np.arange(ts.shape[0])) and np.array_equal(got, ts[:, 1]), np.flatnonzero(got != ts[:, 1])[:5]
    if case == "per0125":
        assert abs(ts[1, 1] - 0.012494) < 1e-9


@pytest.mark.parametrize("L,rows", [(0, 0), (1, 1), (159, 1), (160, 1), (161, 2), (6400, 40), (6401, 41), (6559, 41)])
def test_row_count_rule(L, rows):
    s = session("chroma")
    assert int(s.frame_offsets(np.array([0, L], np.int64), 16000.0, 1)[1]) == rows
    s.close()


@pytest.mark.skipif(not os.path.exists(SHIPPED), reason="oracle/_ref/config (build()) not there")
def test_shipped_chroma_filt_names_and_rows():
    s = Session(SHIPPED, options={"outputfile": "x.csv"}, device=-1)
    assert s.element_names(44100.0) == ["chroma[%d]" % i for i in range(12)]
    for fn, sig in (("chroma_filt_44k1.csv", "rec"), ("chroma_filt_16k.csv", "mix16")):
        pcm, sr, nc = SIGS[sig]
        rows = open(os.path.join(os.path.dirname(TAPS), "..", "golden", fn)).read().strip().split("\n")
        fo = s.frame_offsets(np.array([0, pcm.size // nc], np.int64), float(sr), nc)
        assert int(fo[1]) == len(rows)
    for L in (0, 1, 159, 160, 161, 16000):
        assert int(s.frame_offsets(np.array([0, L], np.int64), 16000.0, 1)[1]) == (L + 159) // 160
    s.close()


HEAD = ("[componentInstances:cComponentManager]\ninstance[dataMemory].type=cDataMemory\ninstance[w].type=cWaveSource\n"
        "instance[fr].type=cFramer\ninstance[tf].type=cTonefilt\ninstance[ch].type=cChroma\ninstance[s].type=cCsvSink\n%s"
        "[w:cWaveSource]\nwriter.dmLevel=wave\n%s\n[fr:cFramer]\nreader.dmLevel=wave\nwriter.dmLevel=frames\nframeSize=0.064\n"
        "frameStep=0.01\n[tf:cTonefilt]\nreader.dmLevel=%s\nwriter.dmLevel=tonefilt\n%s\n[ch:cChroma]\nreader.dmLevel=tonefilt\n"
        "writer.dmLevel=chroma\n%s\n[s:cCsvSink]\nreader.dmLevel=chroma\nfilename=x.csv\n%s")
FUNC = ("instance[f].type=cFunctionals\ninstance[fs].type=cCsvSink\n",
        "[f:cFunctionals]\nreader.dmLevel=chroma\nwriter.dmLevel=func\nframeMode=full\nfunctionalsEnabled=Means\n"
        "Means.amean=1\n[fs:cCsvSink]\nreader.dmLevel=func\nfilename=y.csv\n")


@pytest.mark.parametrize("wave,tfin,tf,ch,func,status,needle", [
    ("", "frames", "", "", False, capi.ERR_UNSUPPORTED, "cTonefilt must read the cWaveSource level"),
    # the channel count comes with the input: the session reports the plan's refusal as an invalid input there
    ("monoMixdown=0", "wave", "", "", False, capi.ERR_INVALID, "cTonefilt: a multi-element wave level"),
    ("", "wave", "nNotes=30", "", False, capi.ERR_UNSUPPORTED, "cChroma.octaveSize must divide the number of cTonefilt notes"),
    ("", "wave", "", "octaveSize=7", False, capi.ERR_UNSUPPORTED, "cChroma.octaveSize must divide the number of cTonefilt notes"),
    ("", "wave", "nNotes=1", "octaveSize=1", False, capi.ERR_UNSUPPORTED, "one-note cTonefilt level"),
    ("", "wave", "nNotes=200", "", False, capi.ERR_UNSUPPORTED, "cTonefilt.nNotes above 128"),
    ("", "wave", "", "", True, capi.ERR_UNSUPPORTED, "cFunctionals reading a level behind cTonefilt 'tf'"),
    ("", "wave", "outputBuffersize=10", "", False, capi.ERR_INVALID, "unknown field 'outputBuffersize'"),
    ("", "wave", "bogus=1", "", False, capi.ERR_INVALID, "unknown field 'bogus'"),
])
def test_refusals(tmp_path, wave, tfin, tf, ch, func, status, needle):
    p = tmp_path / "c.conf"
    text = HEAD % (FUNC[0] if func else "", wave, tfin, tf, ch, FUNC[1] if func else "")
    p.write_text(text.replace("filename=x.csv", "filename=?") if func else text)
    with pytest.raises(SessionError) as e:
        s = Session(str(p), device=-1)
        if wave:                                        # the channel count is known per input
            s.element_names(16000.0, 2)
    assert e.value.status == status and needle in str(e.value), str(e.value)


def test_clamps_and_defaults():
    c = capi.Component()
    assert capi.lib().osm_b200_component_defaults(capi.C_TONEFILT, C_ref(c)) == 0
    q = c.u.tonefilt
    assert (q.nNotes, q.firstNote, q.decayF0, q.decayFN, q.outputPeriod) == (48, 55.0, 0.9995, 0.998, 0.1)
    # decayF0 < decayFN is raised to decayFN; outputPeriod below 1 / fs gives one sample per row at period 1 / fs
    s = session("tonefilt", outputPeriod=0.00001)
    comps, lvl = s.components(16000.0, 1)
    s.close()
    plan = Plan(list(comps), lvl, device=-1)
    assert plan.frame_period == 1.0 / 16000 and plan.num_frames(100) == 100
    plan.close()


def C_ref(c):
    import ctypes
    return ctypes.byref(c)
