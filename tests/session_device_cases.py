"""The shipped configuration files the tests of osm_b200_session_extract_device / Session.extract_tensor run, and the ragged batch
shape they use (tests/test_session_device_cpu.py, tests/test_session_device_gpu.py)."""
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REFCONF = os.path.join(ROOT, "oracle", "_ref", "config")

# name: (configuration file under the reference's config/, options, sample rate, channels)
LLD = {
    "mfcc": ("mfcc/MFCC12_0_D_A.conf", {"O": "x.htk"}, 16000, 1),
    "plp_stereo": ("plp/PLP_0_D_A.conf", {"O": "x.htk"}, 44100, 2),
    "compare_lld": ("compare16/ComParE_2016.conf", {"lldcsvoutput": "x.csv"}, 16000, 1),
    "chroma_filt": ("chroma/chroma_filt.conf", {"outputfile": "x.csv"}, 16000, 1),
    "emo_large": ("misc/emo_large.conf", {"lldcsvoutput": "x.csv"}, 16000, 1),
}
SUMMARY = {
    "is09": ("is09-13/IS09_emotion.conf", {"csvoutput": "x.csv"}, 16000, 1),
    "egemaps": ("egemaps/v02/eGeMAPSv02.conf", {"csvoutput": "x.csv"}, 16000, 1),
    "compare": ("compare16/ComParE_2016.conf", {"csvoutput": "x.csv"}, 16000, 1),
}


def conf_path(case):
    return os.path.join(REFCONF, case[0])


def first_row_length(session, sr, nch):
    """the fewest sample frames that give an utterance one output row (bisection over Session.frame_offsets)"""
    lo, hi = 0, 10 * int(sr)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if session.frame_offsets([0, mid], sr, nch)[-1] > 0:
            hi = mid
        else:
            lo = mid
    return hi


def ragged_lengths(session, sr, nch, long_s=61.0):
    """lengths 0, 1, one row's worth - 1, one row's worth, a long utterance and two ordinary ones"""
    f = first_row_length(session, sr, nch)
    return np.array([int(0.9 * sr), 0, 1, f - 1, f, int(long_s * sr), int(2.3 * sr)], np.int64)
