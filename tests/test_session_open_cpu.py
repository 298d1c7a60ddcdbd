"""Every configuration file opens to what tests/golden/session_open.json pins (scripts/make_golden_session_open.py): the
refusal, or the output level, component array, element names, sink options and frame offsets, under each option set.
Description-only sessions (device = -1): no compute.  The shipped files need oracle/_ref/config (make -C oracle ref)."""
import json
import os

import pytest

from conftest import GOLD
from opensmile_b200 import Session, SessionError, capi
from session_open_cases import ROOT, TREES, describe_file

PINNED = json.load(open(os.path.join(GOLD, "session_open.json")))


def _keys(tree):
    return sorted(k.split(":", 1)[1] for k in PINNED if k.startswith(tree + ":"))


def _check(tree, rel, monkeypatch):
    monkeypatch.chdir(ROOT)                      # includes fall back to paths relative to the working directory
    assert os.path.exists(os.path.join(TREES[tree], rel)), "a pinned configuration file is missing"
    assert describe_file(tree, rel) == PINNED[tree + ":" + rel]


@pytest.mark.parametrize("rel", _keys("tests"))
def test_test_configs_open_as_pinned(rel, monkeypatch):
    _check("tests", rel, monkeypatch)


@pytest.mark.skipif(not os.path.isdir(TREES["ref"]), reason="oracle/_ref/config not built (make -C oracle ref)")
@pytest.mark.parametrize("rel", _keys("ref"))
def test_shipped_configs_open_as_pinned(rel, monkeypatch):
    _check("ref", rel, monkeypatch)


def _energy_sink_conf(path, n_levels):
    """a cCsvSink that reads n_levels cEnergy levels of one framer (an implicit concat of n_levels inputs)"""
    text = "[componentInstances:cComponentManager]\ninstance[waveIn].type = cWaveSource\ninstance[fr].type = cFramer\n"
    text += "".join("instance[e%d].type = cEnergy\n" % i for i in range(n_levels)) + "instance[csv].type = cCsvSink\n\n"
    text += "[waveIn:cWaveSource]\nwriter.dmLevel = wave\nfilename = in.wav\n\n"
    text += "[fr:cFramer]\nreader.dmLevel = wave\nwriter.dmLevel = fr\nframeSize = 0.025\nframeStep = 0.010\n\n"
    text += "".join("[e%d:cEnergy]\nreader.dmLevel = fr\nwriter.dmLevel = e%d\n\n" % (i, i) for i in range(n_levels))
    text += "[csv:cCsvSink]\nreader.dmLevel = %s\nfilename = out.csv\n" % ";".join("e%d" % i for i in range(n_levels))
    path.write_text(text)
    return str(path)


def test_sink_reading_more_levels_than_a_concat_holds_is_refused(tmp_path):
    """a sink reader of up to 8 levels opens with every level's elements; a ninth level is refused, not dropped"""
    per_level = len(Session(_energy_sink_conf(tmp_path / "e1.conf", 1), device=-1).element_names())
    assert len(Session(_energy_sink_conf(tmp_path / "e8.conf", 8), device=-1).element_names()) == 8 * per_level
    with pytest.raises(SessionError) as e:
        Session(_energy_sink_conf(tmp_path / "e9.conf", 9), device=-1)
    assert e.value.status == capi.ERR_UNSUPPORTED and str(e.value) == "more than 8 levels in one reader"
