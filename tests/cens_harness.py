"""Shared pieces of the cCens tests: the golden cases (scripts/make_golden_cens.py), the restatement (tests/cens_oracle.py) and
sessions on tests/configs/cens_taps.conf with one level as the output level."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, HERE)
from opensmile_b200 import Session  # noqa: E402
import cens_oracle  # noqa: E402
import make_golden_cens as mg  # noqa: E402

G = np.load(os.path.join(HERE, "golden", "cens_goldens.npz"))
TAPS = os.path.join(HERE, "configs", "cens_taps.conf")
SINKS = ("chromafft", "censfft", "censfftcsv", "chromafilt", "censfilt", "censfiltcsv")
# output level -> the sink that keeps it (the other sinks are switched off)
LEVEL_SINK = {"chroma_fft": "chromafft", "cens_fft": "censfftcsv", "chroma_filt": "chromafilt", "cens_filt": "censfiltcsv"}
LEVEL_HTK = {"cens_fft": "censfft", "cens_filt": "censfilt"}
REC = np.load(os.path.join(HERE, "golden", "egemaps_recordings.npz"))["pcm_opensmile_44k1"]


def case_input(case):
    """(int16 pcm, sample rate) of a golden case"""
    sig = mg.CASES[case][0]
    if sig == "rec":
        return REC, 44100
    return G["pcm_" + case], int(G["sr_" + case])


def session(level, device=-1, htk=False, **opts):
    o = {k: str(v) for k, v in opts.items()}
    o.update({k: "?" for k in SINKS})
    o[LEVEL_HTK[level] if htk else LEVEL_SINK[level]] = "x.htk" if htk else "x.csv"
    return Session(TAPS, options=o, device=device)
