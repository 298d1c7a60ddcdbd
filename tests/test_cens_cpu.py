"""cCens without a GPU: the restatement (tests/cens_oracle.py) applied to the reference's own chroma level against the reference's
CENS level (tests/golden/cens_goldens.npz, scripts/make_golden_cens.py), names / row counts / level period of description-only
sessions on both chroma paths, the CSV and HTK files written from the reference's values against the reference's files, and the
refusals."""
import os

import numpy as np
import pytest

from cens_harness import G, TAPS, case_input, cens_oracle, mg, session
from opensmile_b200 import Plan, Session, capi
from opensmile_b200.session import SessionError

PATHS = ("fft", "filt")


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("case", sorted(mg.CASES))
def test_restatement_matches_the_reference_bit_for_bit(case, path):
    """zero-norm rows (silence, the silent start of quiet16) and the rows before W included"""
    o = mg.options(case)
    got = cens_oracle.cens(G["chroma_%s_%s" % (path, case)], o["window"], o["winlength"], o["l2norm"])
    ref = G["cens_%s_%s" % (path, case)]
    assert got.shape == ref.shape
    assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), np.argwhere(got.view(np.uint32) != ref.view(np.uint32))[:5]


def test_the_goldens_cover_zero_norm_rows_and_short_utterances():
    assert (G["chroma_fft_silence16"] == 0).all() and np.all(G["cens_fft_silence16"] == cens_oracle.unit_value(12))
    assert (G["chroma_fft_quiet16"][:20] == 0).all()
    for p in PATHS:
        assert G["cens_%s_short16" % p].shape[0] < 41 and G["cens_%s_short16b" % p].shape[0] < 41


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("case", sorted(mg.CASES))
def test_names_rows_and_period(case, path):
    """the level period is the chroma level's times downsampleRatio (values < 1 are 1); every input row is an output row"""
    pcm, sr = case_input(case)
    o = mg.options(case)
    s = session("cens_" + path, **o)
    assert s.element_names(float(sr)) == [str(x) for x in G["names_%s_%s" % (path, case)]]
    fo = s.frame_offsets(np.array([0, pcm.size], np.int64), float(sr))
    assert int(fo[1]) == G["cens_%s_%s" % (path, case)].shape[0] == G["chroma_%s_%s" % (path, case)].shape[0]
    comps, lvl = s.components(float(sr))
    s.close()
    plan = Plan(list(comps), lvl, device=-1)
    assert int(round(plan.frame_period * 1e7)) == int(G["period_%s_%s" % (path, case)])
    # the rows keep the time stamps of their chroma rows: the period scale does not enter them
    L = capi.lib()
    t = G["time_%s_%s" % (path, case)]
    got = np.array([float("%f" % L.osm_b200_plan_row_time(plan._h, r)) for r in range(t.size)])
    plan.close()
    assert np.array_equal(got, t)


@pytest.mark.parametrize("htk", [False, True])
def test_files_written_from_the_reference_values_are_byte_identical(tmp_path, htk):
    """downsampleRatio = 10: the CSV time column keeps the chroma rows' times, the HTK header carries the period 0.1 s"""
    case = "ds10"
    pcm, sr = case_input(case)
    rows = G["cens_fft_" + case]
    s = session("cens_fft", htk=htk, **mg.options(case))
    out = str(tmp_path / ("o.htk" if htk else "o.csv"))
    s.write_files(rows, np.array([0, rows.shape[0]], np.int64), float(sr), 1, np.array([pcm.size], np.int64),
                  htk_paths=[out] if htk else None, csv_paths=None if htk else [out])
    s.close()
    ref = os.path.join(os.path.dirname(TAPS), "..", "golden", "cens_fft_ds10." + ("htk" if htk else "csv"))
    assert open(out, "rb").read() == open(ref, "rb").read()


def test_functionals_names_and_period():
    """cFunctionals over the CENS level (tests/configs/cens_func.conf): the reference's names; the period its seconds are taken in"""
    fconf = os.path.join(os.path.dirname(TAPS), "cens_func.conf")
    for ds in (1, 10):
        s = Session(fconf, options={"downsampleRatio": str(ds), "funchtk": "?", "funccsv": "x.csv"}, device=-1)
        assert s.element_names() == [str(x) for x in G["names_func"]]
        s.close()


def test_defaults():
    c = capi.Component()
    import ctypes
    assert capi.lib().osm_b200_component_defaults(capi.C_CENS, ctypes.byref(c)) == 0
    q = c.u.cens
    assert (q.window, q.winlength, q.l2norm, q.downsampleRatio, q.winlength_sec, q.winlength_secSet) == (1, 41, 1, 10, 0.41, 0)
    assert c.copyInputName == 0


FFT = ("[componentInstances:cComponentManager]\ninstance[dataMemory].type=cDataMemory\ninstance[w].type=cWaveSource\n"
       "instance[fr].type=cFramer\ninstance[win].type=cWindower\ninstance[fft].type=cTransformFFT\ninstance[mag].type=cFFTmagphase\n"
       "instance[ts].type=cTonespec\ninstance[ch].type=cChroma\ninstance[ce].type=cCens\ninstance[s].type=cCsvSink\n%s"
       "[w:cWaveSource]\nwriter.dmLevel=wave\n[fr:cFramer]\nreader.dmLevel=wave\nwriter.dmLevel=frames\nframeSize=0.064\n"
       "frameStep=0.01\n[win:cWindower]\nreader.dmLevel=frames\nwriter.dmLevel=winframes\nwinFunc=Gau\n"
       "[fft:cTransformFFT]\nreader.dmLevel=winframes\nwriter.dmLevel=fftc\n[mag:cFFTmagphase]\nreader.dmLevel=fftc\n"
       "writer.dmLevel=fftmag\n[ts:cTonespec]\nreader.dmLevel=fftmag\nwriter.dmLevel=tonespec\n[ch:cChroma]\n"
       "reader.dmLevel=tonespec\nwriter.dmLevel=chroma\n[ce:cCens]\nreader.dmLevel=%s\nwriter.dmLevel=cens\n%s\n"
       "[s:cCsvSink]\nreader.dmLevel=%s\nfilename=x.csv\n%s")
EXTRA_MFCC = ("instance[mel].type=cMelspec\n", "[mel:cMelspec]\nreader.dmLevel=fftmag\nwriter.dmLevel=mel\n")


@pytest.mark.parametrize("src,opts,extra,out,status,needle", [
    ("tonespec", "", False, "cens", capi.ERR_UNSUPPORTED, "cCens 'ce' must read a cChroma level"),
    ("fftmag", "", False, "cens", capi.ERR_UNSUPPORTED, "cCens 'ce' must read a cChroma level"),
    ("chroma;tonespec", "", False, "cens", capi.ERR_UNSUPPORTED, "cCens 'ce': a multi-field input"),
    ("chroma", "winlength=513", False, "cens", capi.ERR_UNSUPPORTED, "cCens 'ce': winlength 513 is above 512 taps"),
    ("chroma", "winlength_sec=0.41", False, "cens", capi.ERR_UNSUPPORTED, "cCens 'ce': winlength_sec is not supported"),
    ("chroma", "bogus=1", False, "cens", capi.ERR_INVALID, "unknown field 'bogus' in section [ce:cCens]"),
])
def test_refusals(tmp_path, src, opts, extra, out, status, needle):
    p = tmp_path / "c.conf"
    p.write_text(FFT % ("", src, opts, out, ""))
    with pytest.raises(SessionError) as e:
        Session(str(p), device=-1)
    assert e.value.status == status and needle in str(e.value), str(e.value)


def test_winlength_bound_and_clamps_are_accepted(tmp_path):
    for opts, period in (("winlength=512\ndownsampleRatio=0", 0.01), ("winlength=0\ndownsampleRatio=3", 0.03)):
        p = tmp_path / "c.conf"
        p.write_text(FFT % ("", "chroma", opts, "cens", ""))
        s = Session(str(p), device=-1)
        assert s.element_names() == ["CENS[%d]" % i for i in range(12)]
        comps, lvl = s.components()
        s.close()
        plan = Plan(list(comps), lvl, device=-1)
        assert abs(plan.frame_period - period) < 1e-15
        plan.close()


def test_names_with_copy_input_name(tmp_path):
    p = tmp_path / "c.conf"
    p.write_text(FFT % ("", "chroma", "copyInputName=1\nnameAppend=cens", "cens", ""))
    s = Session(str(p), device=-1)
    assert s.element_names() == ["chroma_cens[%d]" % i for i in range(12)]
    s.close()


def test_mixed_periods_in_one_output_level_are_refused(tmp_path):
    p = tmp_path / "c.conf"
    text = FFT % ("instance[cc].type=cVectorConcat\n", "chroma", "downsampleRatio=10", "both",
                  "[cc:cVectorConcat]\nreader.dmLevel=cens;chroma\nwriter.dmLevel=both\n")
    p.write_text(text)
    with pytest.raises(SessionError) as e:
        Session(str(p), device=-1)
    assert "levels of different periods" in str(e.value)
