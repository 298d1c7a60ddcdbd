"""The long recordings the full-input summaries are pinned on (scripts/make_golden_long_summaries.py, tests/test_long_contours_gpu.py):
both regenerated from committed data, their sha256 recorded next to the reference's values so that a drift in a generator fails
loudly.  Above 8 192 frames (81.9 s at 10 ms) every contour takes the long path of cFunctionals."""
import hashlib
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REFCONF = os.path.join(ROOT, "oracle", "_ref", "config")
GOLDEN = os.path.join(ROOT, "tests", "golden", "long_summaries.npz")

CONFS = {
    "egemaps": "egemaps/v02/eGeMAPSv02.conf",
    "gemaps": "gemaps/v01b/GeMAPSv01b.conf",
    "compare": "compare16/ComParE_2016.conf",
}


def synth_10min():
    """10 minutes of opensmile_b200.synth.mixed_pcm at 16 kHz (voiced, noise and near-silence stretches)"""
    from opensmile_b200.synth import mixed_pcm
    return mixed_pcm(600 * 16000, 16000, seed=21)


def tiled_3min():
    """35 tiles (3 min 4 s) of the 5.2 s recording pcm_media_interpretation_16k, each scaled by its own gain"""
    rec = np.load(os.path.join(ROOT, "tests", "golden", "egemaps_recordings.npz"))["pcm_media_interpretation_16k"].astype(np.float64)
    gains = np.random.default_rng(5).uniform(0.3, 1.8, 35)
    return np.concatenate([np.clip(np.round(rec * g), -32768, 32767) for g in gains]).astype(np.int16)


INPUTS = {"synth10": synth_10min, "tiled3": tiled_3min}


def sha256(pcm):
    return hashlib.sha256(np.ascontiguousarray(pcm, "<i2").tobytes()).hexdigest()
