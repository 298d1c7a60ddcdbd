"""GPU check of the GeMAPS / eGeMAPS summary path against the reference dumps (tests/golden/gemaps_func*.npz): the seven input levels
of the functionals row by row, then the 88 / 62 summary values."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from opensmile_b200.session import Session  # noqa: E402
from opensmile_b200.synth import mixed_pcm, voiced_pcm  # noqa: E402

REFCONF = os.path.join(ROOT, "oracle", "_ref", "config")
GL = np.load(os.path.join(ROOT, "tests", "golden", "gemaps_func_levels.npz"))
GF = np.load(os.path.join(ROOT, "tests", "golden", "gemaps_func.npz"))
rec = np.load(os.path.join(ROOT, "tests", "golden", "egemaps_recordings.npz"))["pcm_opensmile_16k"]
pcms = {"m24k": mixed_pcm(24000, 16000, seed=3), "v32k": voiced_pcm(32000, 16000, seed=7), "rec": rec}
keys = list(pcms)
off = np.concatenate([[0], np.cumsum([len(pcms[k]) for k in keys])]).astype(np.int64)
allpcm = np.concatenate([pcms[k] for k in keys])
conf = os.path.join(REFCONF, "egemaps", "v02", "eGeMAPSv02.conf")
levels = sorted({k.split("_", 1)[1] for k in GL.files if not k.startswith("names_")})
for lv in levels:
    s = Session(conf, output_level=lv, device=0)
    names = s.element_names()
    rows, fo = s.extract_pcm(allpcm, off, 16000.0, 1)
    s.close()
    assert names == [str(x) for x in GL["names_" + lv]], (names, GL["names_" + lv])
    for u, k in enumerate(keys):
        ref = GL["%s_%s" % (k, lv)]
        got = rows[fo[u]:fo[u + 1]]
        if got.shape != ref.shape:
            print("LEVEL", lv, k, "SHAPE", got.shape, ref.shape)
            n = min(len(got), len(ref))
            got, ref = got[:n], ref[:n]
        scale = np.abs(ref).max(axis=0) + 1e-12
        err = np.abs(got - ref) / scale
        worst = err.max(axis=0)
        bad = [(names[c], float(worst[c]), int(np.argmax(err[:, c]))) for c in range(len(names)) if worst[c] > 1e-4]
        print("LEVEL", lv, k, got.shape, "max err/scale %.2e" % worst.max(), bad[:6])
for tag, cf in (("egemaps", "egemaps/v02/eGeMAPSv02.conf"), ("gemaps", "gemaps/v01b/GeMAPSv01b.conf")):
    s = Session(os.path.join(REFCONF, cf), options={"csvoutput": "f.csv"}, device=0)
    names = s.element_names()
    rows, fo = s.extract_pcm(allpcm, off, 16000.0, 1)
    s.close()
    print(tag, rows.shape, list(fo))
    for u, k in enumerate(keys):
        ref = GF["%s_%s" % (tag, k)][0]
        got = rows[u]
        rel = np.abs(got - ref) / (np.abs(ref) + 1e-6)
        nb = int((rel > 1e-4).sum())
        print(tag, k, "values with rel err > 1e-4:", nb, " > 1e-3:", int((rel > 1e-3).sum()), " > 1e-2:", int((rel > 1e-2).sum()))
        for i in np.argsort(-rel)[:12]:
            if rel[i] > 1e-4: print("   %-45s got %-14.7g ref %-14.7g rel %.2e" % (names[i], got[i], ref[i], rel[i]))
