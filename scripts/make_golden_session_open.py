"""Write tests/golden/session_open.json: what every configuration file lowers to when a session opens it.

    python scripts/make_golden_session_open.py      # needs oracle/_ref/config (make -C oracle ref) and libosm_b200.so

Every .conf under the reference's config tree (oracle/_ref/config) and under tests/configs, opened with device = -1 under
each option set of tests/session_open_cases.py: the status and message of a refusal, or the output level, a hash of the
component array, the element names' count and hash at 16 kHz mono and 44.1 kHz stereo, the sink options and the frame offsets
of a small ragged batch.  The file pins the behaviour of the host front end; tests/test_session_open_cpu.py checks it.
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from session_open_cases import TREES, conf_files, describe_file  # noqa: E402


def main():
    assert os.path.isdir(TREES["ref"]), "build the reference's config tree first: make -C oracle ref"
    os.chdir(ROOT)
    out = {}
    for tree in TREES:
        for rel in conf_files(tree):
            out[tree + ":" + rel] = describe_file(tree, rel)
    with open(os.path.join(ROOT, "tests", "golden", "session_open.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    cases = [r for recs in out.values() for r in recs.values()]
    print("%d files, %d cases: %d open, %d refused" % (len(out), len(cases), sum("output_level" in r for r in cases),
                                                       sum("status" in r for r in cases)))


if __name__ == "__main__":
    main()
