"""cTonespec / cChroma without a GPU: the oracle (oracle/chroma_oracle.py) against the unmodified reference's levels
(tests/golden/chroma_goldens.npz, scripts/make_golden_chroma.py), the library's tables against the oracle's bit for bit, names
and row counts of the shipped chroma_fft.conf, and the configurations that are refused."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from opensmile_b200 import Session, capi  # noqa: E402
from opensmile_b200.session import SessionError  # noqa: E402
from oracle import chroma_oracle as co  # noqa: E402
import make_golden_chroma as mg  # noqa: E402

G = np.load(os.path.join(HERE, "golden", "chroma_goldens.npz"))
TAPS = os.path.join(HERE, "configs", "chroma_taps.conf")
SHIPPED = os.path.join(ROOT, "oracle", "_ref", "config", "chroma", "chroma_fft.conf")
SIGS = mg.signals()


def oracle_case(case):
    sig = mg.CASES[case][0]
    pcm, sr, nc = SIGS[sig]
    o = mg.options(case)
    return co.extract(pcm, sr, nc, o["nOctaves"], o["firstNote"], o["filterType"], o["usePower"], o["dbA"], o["octaveSize"], o["silThresh"])


def col_err(got, ref):
    scale = np.maximum(np.abs(ref).max(axis=0), 1e-30)
    return float((np.abs(got - ref) / scale).max()) if ref.size else 0.0


@pytest.mark.parametrize("case", sorted(mg.CASES))
def test_oracle_matches_the_reference_levels(case):
    tone, ch, _ = oracle_case(case)
    rt, rc = G["tone_" + case], G["chroma_" + case]
    assert tone.shape == rt.shape and ch.shape == rc.shape, (tone.shape, rt.shape, ch.shape, rc.shape)
    # the reference's CSV holds 7 significant digits (%e): half a unit of the last one is 5e-7 of the value
    assert col_err(tone, rt) < 1e-6, col_err(tone, rt)
    assert col_err(ch, rc) < 1e-6, col_err(ch, rc)
    # zeros where the reference writes zeros: the top two notes, filterType = rec, frames below silThresh
    assert np.array_equal(tone[rt == 0], rt[rt == 0]) and np.array_equal(ch[rc == 0], rc[rc == 0])
    assert (rt[:, -2:] == 0).all()
    if mg.options(case)["filterType"] == "rec":
        assert (rt == 0).all()


def test_quiet_signal_trips_silthresh():
    _, ch, sil = oracle_case("quiet16")
    assert sil.any() and (~sil).any()
    assert (G["chroma_quiet16"][sil] == 0).all() and (ch[sil] == 0).all()


def lib_tables(cfg, n_bins, fss):
    nN = 12 * cfg.nOctaves
    pcf = np.zeros(nN + 2, np.float32); key = np.zeros(n_bins, np.int32); cnt = np.zeros(nN + 2, np.int32)
    fm = np.zeros(n_bins, np.float32); fl = np.zeros(2, np.int32)
    st = capi.lib().osm_b200_tone_tables(C.byref(cfg), n_bins, fss, pcf.ctypes.data, key.ctypes.data, cnt.ctypes.data,
                                         fm.ctypes.data, fl.ctypes.data)
    return st, pcf, key, cnt, fm, fl


@pytest.mark.parametrize("geom", [(16000, 1024, 1024), (44100, 4096, 2822), (8000, 512, 512), (48000, 4096, 3072), (22050, 2048, 1411)])
@pytest.mark.parametrize("ft", ["gau", "tri", "trp", "rec"])
def test_library_tables_equal_the_oracle_bit_for_bit(geom, ft):
    sr, nfft, N = geom
    fss = 0.064 * nfft / N                        # cTransformFFT's frameSizeSec: 1 / fss = sr / nfft
    for no, fn, dba in ((6, 55.0, 1), (6, 55.0, 0), (1, 220.0, 1), (8, 65.406, 1)):
        st, *got = lib_tables(capi.Tonespec(no, fn, co.FILTERS[ft], 0, dba), nfft // 2 + 1, fss)
        if ft in ("tri", "trp") and 55.0 * 2 ** ((12 * no - 2) / 12.0) > sr / 2:
            assert st == capi.ERR_UNSUPPORTED and "past its filter map" in capi.last_error()     # the reference's write past the map
            continue
        assert st == capi.OK, capi.last_error()
        ref = co.tables(no, fn, ft, dba, nfft // 2 + 1, fss)
        for g, r in zip(got[:4], ref[:4]):
            assert g.dtype == r.dtype and np.array_equal(g.view(np.int32), np.asarray(r).view(np.int32))
        assert list(got[4]) == list(ref[4:])


def test_bin_spacing_at_44k1():
    """64 ms at 44.1 kHz is 2822 samples, N = 4096.  cTransformFFT scales the level's frameSizeSec -- the framer's nominal 0.064 s,
    not 2822 / 44100 -- by 4096 / 2822 (dspcore/transformFft.cpp:79-83), so the bin spacing F0 = 2822 / (0.064 * 4096) is
    10.7651 Hz, 0.014 % below fs / N = 10.7666 Hz.  The first bin of the 6-octave bank differs between the two; the goldens of the
    44.1 kHz recording (test_oracle_matches_the_reference_levels[rec]) hold only with the first."""
    s = Session(TAPS, options={"toneoutput": "x.csv", "chromaoutput": "?"}, device=-1)
    comps = s.components(44100.0, 1)[0]
    s.close()
    assert any(c.type == capi.C_TONESPEC for c in comps)
    fss = 0.064 * 4096 / 2822
    st, pcf, key, cnt, fm, fl = lib_tables(capi.Tonespec(6, 55.0, 0, 0, 1), 2049, fss)
    assert st == capi.OK
    F0 = float(np.float32(1.0 / fss))
    assert abs(F0 - 10.7651) < 1e-4 and abs(F0 - 44100 / 4096.0) > 1e-3
    assert fl[0] == int(np.ceil(float(np.float32(pcf[0] + pcf[1])) / (2.0 * F0)))


def test_tap_names_follow_the_reference_header():
    s = Session(TAPS, options={"toneoutput": "x.csv", "chromaoutput": "?"}, device=-1)
    assert s.element_names() == [str(x) for x in G["names_tone_mix16"]]
    s.close()
    s = Session(TAPS, options={"chromaoutput": "x.csv", "toneoutput": "?", "octaveSize": "24"}, device=-1)
    assert s.element_names() == [str(x) for x in G["names_chroma_os24"]]
    s.close()


@pytest.mark.skipif(not os.path.exists(SHIPPED), reason="oracle/_ref/config (build()) not there")
def test_shipped_chroma_fft_names_and_rows():
    s = Session(SHIPPED, options={"outputfile": "x.csv"}, device=-1)
    assert s.element_names(44100.0) == [str(x) for x in G["names_chroma_rec"]] == ["chroma[%d]" % i for i in range(12)]
    for fn, sig in (("chroma_fft_44k1.csv", "rec"), ("chroma_fft_16k.csv", "mix16")):
        pcm, sr, nc = SIGS[sig]
        rows = open(os.path.join(HERE, "golden", fn)).read().strip().split("\n")
        fo = s.frame_offsets(np.array([0, pcm.size // nc], np.int64), float(sr), nc)
        assert int(fo[1]) == len(rows) == G["chroma_" + sig].shape[0]
    s.close()


HEAD = ("[componentInstances:cComponentManager]\ninstance[dataMemory].type=cDataMemory\ninstance[w].type=cWaveSource\n"
        "instance[fr].type=cFramer\ninstance[win].type=cWindower\ninstance[fft].type=cTransformFFT\ninstance[mag].type=cFFTmagphase\n"
        "instance[ts].type=cTonespec\ninstance[ch].type=cChroma\ninstance[s].type=cCsvSink\n"
        "[w:cWaveSource]\nwriter.dmLevel=wave\n[fr:cFramer]\nreader.dmLevel=wave\nwriter.dmLevel=frames\nframeSize=0.064\nframeStep=0.01\n"
        "[win:cWindower]\nreader.dmLevel=frames\nwriter.dmLevel=winframes\nwinFunc=gauss\n[fft:cTransformFFT]\nreader.dmLevel=winframes\n"
        "writer.dmLevel=fftc\n[mag:cFFTmagphase]\nreader.dmLevel=fftc\nwriter.dmLevel=fftmag\n%s\n[ts:cTonespec]\nreader.dmLevel=fftmag\n"
        "writer.dmLevel=tonespec\n%s\n[ch:cChroma]\nreader.dmLevel=%s\nwriter.dmLevel=chroma\n%s\n[s:cCsvSink]\nreader.dmLevel=chroma\n"
        "filename=x.csv\n")


@pytest.mark.parametrize("mag,ts,chin,ch,status,needle", [
    ("", "", "fftmag", "", capi.ERR_UNSUPPORTED, "cChroma must read a cTonespec level"),
    ("", "", "frames", "", capi.ERR_UNSUPPORTED, "cChroma must read a cTonespec level"),
    ("dBpsd=1", "", "tonespec", "", capi.ERR_UNSUPPORTED, "cTonespec: cFFTmagphase: normalise / power / dBpsd"),
    ("", "nOctaves=5", "tonespec", "octaveSize=24", capi.ERR_UNSUPPORTED, "octaveSize must divide"),
    ("", "", "tonespec", "octaveSize=7", capi.ERR_UNSUPPORTED, "octaveSize must divide"),
    ("", "printBinMap=1", "tonespec", "", capi.ERR_INVALID, "unknown field 'printBinMap'"),
    ("", "printFilterMap=0", "tonespec", "", capi.ERR_INVALID, "unknown field 'printFilterMap'"),
    ("", "", "tonespec", "bogus=1", capi.ERR_INVALID, "unknown field 'bogus'"),
])
def test_refusals(tmp_path, mag, ts, chin, ch, status, needle):
    p = tmp_path / "c.conf"
    p.write_text(HEAD % (mag, ts, chin, ch))
    with pytest.raises(SessionError) as e:
        Session(str(p), device=-1)
    assert e.value.status == status and needle in str(e.value), str(e.value)


@pytest.mark.parametrize("spelling,kind", [("gau", 0), ("Gaussian", 0), ("Tri", 1), ("triangular", 1), ("TrP", 2),
                                           ("Triangular-Powered", 2), ("Rec", 3), ("rectangular", 3), ("box", 0)])
def test_filter_type_spellings(tmp_path, spelling, kind):
    p = tmp_path / "c.conf"
    p.write_text(HEAD % ("", "filterType=" + spelling, "tonespec", ""))
    s = Session(str(p), device=-1)
    ts = [c for c in s.components()[0] if c.type == capi.C_TONESPEC][0]
    s.close()
    assert ts.u.tonespec.filterType == kind
