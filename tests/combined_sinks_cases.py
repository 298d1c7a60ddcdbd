"""The shipped summary configurations whose summary and LLD sinks one session serves together, and the options that enable each
(tests/test_combined_sinks_cpu.py, tests/test_combined_sinks_gpu.py).  Every file includes shared/standard_data_output*.conf.inc:
-csvoutput / -O (output) / -htkoutput enable the summary's CSV / ARFF / HTK sink, -lld*output the LLD sinks."""
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REFCONF = os.path.join(ROOT, "oracle", "_ref", "config")

CONFS = {
    "is09": "is09-13/IS09_emotion.conf",
    "is13": "is09-13/IS13_ComParE.conf",
    "compare": "compare16/ComParE_2016.conf",
    "emobase": "emobase/emobase.conf",
    "emo_large": "misc/emo_large.conf",
    "gemaps": "gemaps/v01b/GeMAPSv01b.conf",
    "egemaps": "egemaps/v02/eGeMAPSv02.conf",
}
SUMMARY_OPTS = ("csvoutput", "O", "htkoutput")
LLD_OPTS = ("lldcsvoutput", "lldhtkoutput", "lldarffoutput")


def conf_path(name):
    return os.path.join(REFCONF, CONFS[name])


def have_confs():
    return os.path.isdir(REFCONF)
