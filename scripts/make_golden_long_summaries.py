"""Generate tests/golden/long_summaries.npz with the UNMODIFIED reference (oracle/_ref/SMILExtract): the -csvoutput rows of the
shipped eGeMAPSv02, GeMAPSv01b and ComParE_2016 configurations for the long inputs of tests/long_summary_cases.py (10 minutes of
synthetic speech-like signal, 3 minutes of a tiled recording), with each input's sha256 and the reference's LLD row count.  Only names,
values and counts are stored.  The LLD CSV sink is enabled beside the summary, and nothing is written when the LLD level holds fewer
rows than the input has 10 ms frames (the reference did not read the whole input).  On eGeMAPSv02 the reference warns that
egemapsv02_smoE "could not perform any work because destination levels are full ... Processing will possibly be incomplete": its
level waits for lldconcat, which reads it together with the F0 level behind it; the LLD rows show the level complete, and the
functionals do not read it.  Build container only."""
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import refrun  # noqa: E402
from long_summary_cases import CONFS, GOLDEN, INPUTS, REFCONF, sha256  # noqa: E402
from make_golden_functionals import csv_rows  # noqa: E402


def main():
    assert refrun.available()
    out = {}
    for key, make in INPUTS.items():
        pcm = make()
        out["sha256_" + key] = np.array(sha256(pcm))
        with tempfile.TemporaryDirectory() as d:
            wav = os.path.join(d, "in.wav")
            refrun.write_wav(wav, pcm, 16000, 1)
            for conf, rel in CONFS.items():
                csv, lld = os.path.join(d, conf + ".csv"), os.path.join(d, conf + "_lld.csv")
                r = subprocess.run([refrun.SMILEXTRACT, "-C", os.path.join(REFCONF, rel), "-I", wav, "-csvoutput", csv, "-lldcsvoutput", lld],
                                   check=True, capture_output=True, text=True)
                n_lld = len(open(lld).read().strip().split("\n")) - 1
                if n_lld < len(pcm) // 160 - 5:
                    raise SystemExit("%s on %s: the reference did not summarise the whole input (%d LLD rows):\n%s" % (conf, key, n_lld, (r.stdout + r.stderr)[-2000:]))
                out["lld_rows_%s_%s" % (conf, key)] = np.array(n_lld)
                names, rows = csv_rows(csv)
                assert rows.shape[0] == 1, rows.shape
                out["names_" + conf] = np.array(names)
                out[conf + "_" + key] = rows[0]
                print(key, conf, rows.shape, n_lld, "LLD rows", len(pcm) / 16000.0, "s", flush=True)
    np.savez_compressed(GOLDEN, **out)


if __name__ == "__main__":
    main()
