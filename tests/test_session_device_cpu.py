"""CPU tests of osm_b200_session_extract_device (include/osm_b200_host.h) and Session.extract_tensor: the row-count query
(d_out = NULL) of a padded batch needs no device and gives the offsets Session.frame_offsets gives for the same lengths, for the
shipped LLD and summary configurations; malformed arguments are refused, in C and in Python, before anything runs.
Description-only sessions (device = -1)."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from opensmile_b200 import Session, SessionError, capi
from session_device_cases import LLD, SUMMARY, conf_path, ragged_lengths

needs_conf = pytest.mark.skipif(not os.path.isdir(os.path.dirname(conf_path(LLD["mfcc"]))),
                                reason="reference configuration files not built (make -C oracle ref)")
i64p = C.POINTER(C.c_int64)
NEW_SYMBOLS = ["osm_b200_session_extract_device", "osm_b200_plan_run_device_padded", "osm_b200_plan_copy_seq_lag_stream",
               "osm_b200_plan_check_device_flags"]


def device_query(s, lengths, stride, sr, nch, fmt=0, d_out=None, max_rows=0):
    """osm_b200_session_extract_device with no samples: (status, frame offsets)"""
    lens = np.ascontiguousarray(lengths, dtype=np.int64)
    fo = np.zeros(len(lens) + 1, dtype=np.int64)
    st = s._L.osm_b200_session_extract_device(s._h, None, fmt, stride, lens.ctypes.data_as(i64p), len(lens), float(sr), nch,
                                              fo.ctypes.data_as(i64p), d_out, max_rows, None)
    return st, fo


def test_new_symbols_are_exported():
    L = C.CDLL(capi.LIB_PATH)
    for sym in NEW_SYMBOLS:
        assert sym in capi.EXPORTS and hasattr(L, sym), sym


@needs_conf
@pytest.mark.parametrize("name", sorted(LLD) + sorted(SUMMARY))
def test_row_count_query_needs_no_device_and_matches_frame_offsets(name):
    conf, opts, sr, nch = {**LLD, **SUMMARY}[name]
    s = Session(conf_path((conf,)), options=opts, device=-1)
    lens = ragged_lengths(s, sr, nch)
    want = s.frame_offsets(np.concatenate([[0], np.cumsum(lens)]), sr, nch)
    for fmt in (0, 1):                                    # int16, float32: the row counts do not depend on the sample format
        st, fo = device_query(s, lens, int(lens.max()) + 5, sr, nch, fmt)
        assert st == capi.OK, capi.lib().osm_b200_host_last_error()
        assert list(fo) == list(want)
    n = np.diff(want)
    assert n[1] == 0 and n[3] == 0 and n[4] >= 1                # lengths 0 and one row's worth - 1 give no row, one row's worth does
    s.close()


@needs_conf
@pytest.mark.parametrize("name", ["mfcc", "egemaps"])
def test_refusals_of_the_c_entry_point(name):
    conf, opts, sr, nch = {**LLD, **SUMMARY}[name]
    s = Session(conf_path((conf,)), options=opts, device=-1)
    lens = np.array([16000, 0, 32000], np.int64)
    err = lambda: capi.lib().osm_b200_host_last_error().decode()
    for fmt in (2, 3, 4, 5, -1):                          # int8, 24-bit, 24-in-32, int32, nonsense
        assert device_query(s, lens, 32000, sr, nch, fmt)[0] == capi.ERR_INVALID and "pcm_format" in err()
    assert device_query(s, lens, 31999, sr, nch)[0] == capi.ERR_INVALID and "stride" in err()
    assert device_query(s, np.array([-1], np.int64), 10, sr, nch)[0] == capi.ERR_INVALID and "stride" in err()
    fo = np.zeros(4, np.int64)
    assert s._L.osm_b200_session_extract_device(s._h, None, 0, 32000, None, 3, float(sr), nch, fo.ctypes.data_as(i64p), None, 0,
                                                None) == capi.ERR_INVALID
    # too small an output buffer is refused before anything runs (the pointer is never used)
    st, fo = device_query(s, lens, 32000, sr, nch)
    assert st == capi.OK and fo[-1] > 0
    st, _ = device_query(s, lens, 32000, sr, nch, d_out=C.c_void_p(256), max_rows=int(fo[-1]) - 1)
    assert st == capi.ERR_INVALID and "too small" in err()
    s.close()


@needs_conf
def test_configurations_the_session_refuses_are_refused_with_the_same_message():
    conf, opts, sr, nch = LLD["compare_lld"]
    s = Session(conf_path((conf,)), options=opts, device=-1)
    for rate in (96000, 8000):                            # the SHS pitch chain's cSpecScale, and a 256-point FFT: not supported
        with pytest.raises(SessionError) as host:
            s.frame_offsets([0, 16000], rate, nch)
        for fmt in (0, 1):
            st, _ = device_query(s, [16000], 16000, rate, nch, fmt)
            assert st == host.value.status == capi.ERR_UNSUPPORTED
            assert capi.lib().osm_b200_host_last_error().decode() == str(host.value)
    s.close()


def _session():
    conf, opts, sr, nch = LLD["mfcc"]
    if not os.path.exists(conf_path((conf,))):
        pytest.skip("reference configuration files not built (make -C oracle ref)")
    return Session(conf_path((conf,)), options=opts, device=-1)


def test_extract_tensor_refuses_malformed_input():
    s = _session()
    x = torch.zeros((2, 16000), dtype=torch.int16)
    with pytest.raises(TypeError, match="int16 or float32"):
        s.extract_tensor(x.double(), [16000, 100], 16000)
    with pytest.raises(TypeError, match="torch tensor"):
        s.extract_tensor(x.numpy(), [16000, 100], 16000)
    with pytest.raises(ValueError, match=r"\[B, L\] or \[B, C, L\]"):
        s.extract_tensor(x[0], [16000], 16000)
    with pytest.raises(ValueError, match=r"\[B, L\] or \[B, C, L\]"):
        s.extract_tensor(x.reshape(1, 1, 2, 16000), [16000], 16000)
    with pytest.raises(ValueError, match="contiguous"):
        s.extract_tensor(torch.zeros((16000, 2), dtype=torch.int16).t(), [16000, 100], 16000)
    with pytest.raises(ValueError, match="on the host"):
        s.extract_tensor(x, torch.tensor([16000, 100], device="meta"), 16000)
    with pytest.raises(ValueError, match="2 entries"):
        s.extract_tensor(x, [16000], 16000)
    with pytest.raises(ValueError, match=r"0 \.\. 16000"):
        s.extract_tensor(x, [16001, 0], 16000)
    with pytest.raises(ValueError, match=r"0 \.\. 16000"):
        s.extract_tensor(x, torch.tensor([-1, 0]), 16000)
    with pytest.raises(ValueError, match="CUDA tensor"):             # well-formed, but in host memory: extract_pcm's input
        s.extract_tensor(x, torch.tensor([16000, 100]), 16000)
    s.close()
