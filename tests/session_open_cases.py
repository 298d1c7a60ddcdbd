"""What a configuration file lowers to when a session opens it (osm_b200_session_open, description only: device = -1), as
one JSON-ready record per file and option set.  scripts/make_golden_session_open.py writes these records for every .conf under
the reference's config tree and under tests/configs into tests/golden/session_open.json; tests/test_session_open_cpu.py
compares the library against that file.  Both run from the repository root: includes that are not found next to the including
file are looked up relative to the working directory."""
import glob
import hashlib
import os

from opensmile_b200 import Session, SessionError

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# fixture key prefix -> directory whose .conf files (recursively) are pinned
TREES = {"ref": os.path.join(ROOT, "oracle", "_ref", "config"), "tests": os.path.join(ROOT, "tests", "configs")}
# option set name -> command line options (-O, -csvoutput, ...) given to the configuration
OPTION_SETS = {
    "none": {},
    "O": {"O": "out.htk"},
    "csvoutput": {"csvoutput": "out.csv"},
    "lldcsvoutput": {"lldcsvoutput": "lld.csv"},
    "arffoutput": {"arffoutput": "out.arff"},
    "lldhtkoutput": {"lldhtkoutput": "lld.htk"},
    "lldarffoutput": {"lldarffoutput": "lld.arff"},
    "htkoutput": {"htkoutput": "out.htk"},
}
UTT_OFFSETS = [0, 0, 400, 16400, 64523]


def conf_files(tree):
    """the .conf files of one tree, relative to it, sorted"""
    base = TREES[tree]
    return sorted(os.path.relpath(p, base) for p in glob.glob(os.path.join(base, "**", "*.conf"), recursive=True))


def _portable(text, tree):
    return text.replace(TREES[tree], "<" + tree + ">").replace(ROOT, "<root>")


def _sha(data):
    return hashlib.sha256(data).hexdigest()


def _refused(e, tree):
    return {"status": e.status, "message": _portable(str(e), tree)}


def _names(s, sr, nch, tree):
    try:
        names = s.element_names(sr, nch)
    except SessionError as e:
        return _refused(e, tree)
    return {"count": len(names), "sha256": _sha("\n".join(names).encode())}


def describe(tree, rel, options):
    """the record of configuration `rel` of `tree` opened with `options`"""
    try:
        s = Session(os.path.join(TREES[tree], rel), options=options, device=-1)
    except SessionError as e:
        return _refused(e, tree)
    try:
        comps, level = s.components(16000, 1)
        rec = {"output_level": level, "components_sha256": _sha(bytes(comps)),
               "names_16k_mono": _names(s, 16000, 1, tree), "names_44k1_stereo": _names(s, 44100, 2, tree),
               "sink_options": s.sink_options()}
        try:
            rec["frame_offsets"] = [int(x) for x in s.frame_offsets(UTT_OFFSETS, 16000)]
        except SessionError as e:
            rec["frame_offsets"] = _refused(e, tree)
        return rec
    finally:
        s.close()


def describe_file(tree, rel):
    """records of one configuration file under every option set"""
    return {name: describe(tree, rel, opts) for name, opts in OPTION_SETS.items()}
