"""CPU tests of sessions whose active sinks read a summary level and an LLD level (description only, device = -1): every shipped
summary configuration opens with each summary sink option combined with each LLD sink option; the summary's names and row counts,
and the LLD part's names and row counts, are those of the two sessions with one of the options each.  Other mixes of levels keep
their refusal."""
import ctypes as C
import os

import numpy as np
import pytest

from opensmile_b200 import Session, SessionError, capi
from combined_sinks_cases import CONFS, LLD_OPTS, ROOT, SUMMARY_OPTS, conf_path, have_confs

needs_conf = pytest.mark.skipif(not have_confs(), reason="reference configuration files not built (make -C oracle ref)")
i64p = C.POINTER(C.c_int64)
LENGTHS = np.array([16000, 0, 1, 399, 400, 1103, 61 * 16000, 37000], np.int64)
DIFFERENT = "the active sinks read different levels"


def lld_query(s, lengths, sr=16000.0, nch=1):
    """osm_b200_session_extract_device_lld with no samples and no buffers: (status, summary offsets, LLD offsets)"""
    lens = np.ascontiguousarray(lengths, dtype=np.int64)
    fo = np.zeros(len(lens) + 1, dtype=np.int64)
    lfo = np.zeros(len(lens) + 1, dtype=np.int64)
    st = s._L.osm_b200_session_extract_device_lld(s._h, None, 0, int(lens.max()), lens.ctypes.data_as(i64p), len(lens), float(sr), nch,
                                                  fo.ctypes.data_as(i64p), None, 0, lfo.ctypes.data_as(i64p), None, 0, None)
    return st, fo, lfo


def test_new_symbols_are_exported():
    L = C.CDLL(capi.LIB_PATH)
    for sym in ("osm_b200_session_extract_device_lld", "osm_b200_session_extract_files_lld", "osm_b200_session_lld_num_elements",
                "osm_b200_session_lld_element_name", "osm_b200_device_gather_rows"):
        assert sym in capi.EXPORTS and hasattr(L, sym), sym


@needs_conf
@pytest.mark.parametrize("lld_opt", LLD_OPTS)
@pytest.mark.parametrize("sum_opt", SUMMARY_OPTS)
@pytest.mark.parametrize("name", sorted(CONFS))
def test_summary_and_lld_sinks_open_together(name, sum_opt, lld_opt):
    both = Session(conf_path(name), options={sum_opt: "f.out", lld_opt: "l.out"}, device=-1)
    summ = Session(conf_path(name), options={sum_opt: "f.out"}, device=-1)
    lld = Session(conf_path(name), options={lld_opt: "l.out"}, device=-1)
    for sr, nch in ((16000, 1), (44100, 2)):
        assert both.element_names(sr, nch) == summ.element_names(sr, nch)
        assert both.lld_element_names(sr, nch) == lld.element_names(sr, nch)
        assert summ.lld_element_names(sr, nch) == [] and lld.lld_element_names(sr, nch) == []
    off = np.concatenate([[0], np.cumsum(LENGTHS)])
    st, fo, lfo = lld_query(both, LENGTHS)
    assert st == capi.OK, capi.lib().osm_b200_host_last_error()
    assert list(fo) == list(summ.frame_offsets(off, 16000)) == list(both.frame_offsets(off, 16000))
    assert list(lfo) == list(lld.frame_offsets(off, 16000))
    for s in (both, summ, lld):
        s.close()


@needs_conf
def test_lld_sink_options_are_those_of_its_own_session():
    # the summary's CSV sink (number = 0, timestamp = 1) and the LLD CSV sink (timestamp = \cm[timestampcsvlld]) keep their options
    opts = {"csvoutput": "f.csv", "lldcsvoutput": "l.csv", "timestampcsvlld": "0", "instname": "utt"}
    both = Session(conf_path("egemaps"), options=opts, device=-1)
    summ = Session(conf_path("egemaps"), options={k: v for k, v in opts.items() if k != "lldcsvoutput"}, device=-1)
    assert both.sink_options() == summ.sink_options()
    both.close()
    summ.close()


@needs_conf
def test_queries_without_an_lld_part():
    s = Session(conf_path("egemaps"), options={"csvoutput": "f.csv"}, device=-1)
    st, _, _ = lld_query(s, LENGTHS)
    assert st == capi.ERR_INVALID and "no LLD part" in capi.lib().osm_b200_host_last_error().decode()
    with pytest.raises(SessionError, match="no LLD part"):
        s.extract_files(["a.wav"], lld_csv_paths=["l.csv"])
    s.close()


@needs_conf
def test_two_lld_levels_and_two_summary_levels_stay_refused():
    with pytest.raises(SessionError, match=DIFFERENT) as e:
        Session(os.path.join(ROOT, "tests", "configs", "cens_taps.conf"), device=-1)
    assert e.value.status == capi.ERR_UNSUPPORTED
    av = os.path.join(os.path.dirname(conf_path("is09")), "..", "audiovisual", "audiovideo.conf")
    if os.path.exists(av):
        with pytest.raises(SessionError, match=DIFFERENT):
            Session(av, device=-1)
