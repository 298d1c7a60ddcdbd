"""The SHS pitch chain's case table (tests/pitch_cases.py) on description-only plans: every case opens at every level of the chain,
the cPitchShs level carries the reference's field names (lldcore/pitchBase.cpp:132-154), the row offsets of the case's ragged batch
are the oracle's frame counts, and the limits of the kernels are refused when the plan is created."""
import re

import numpy as np
import pytest

import pitch_cases as PC
from opensmile_b200 import Plan, capi


@pytest.mark.parametrize("name", list(PC.BY_NAME))
def test_case_opens_with_the_oracle_geometry_and_names(name):
    c = PC.BY_NAME[name]
    utts, _, off = PC.batch(c)
    T = [PC.frames(c, len(x) // c["n_chan"]) for x in utts]
    want = np.concatenate([[0], np.cumsum(T)])
    expect = {"shs": PC.shs_names(c), PC.f0_level(c): PC.vit_names(c), "jit": PC.jit_names(c)}
    if not c["voicing"]:
        for level in (PC.f0_level(c), "jit", "lld"):
            assert "cPitchShs.voicing=0 below cPitchSmootherViterbi is not supported" in _refused(c, level)
        expect = {"shs": expect["shs"]}
    for level, names in expect.items():
        p = Plan(PC.components(c), level, device=-1)
        try:
            assert p.element_names == names, level
            assert np.array_equal(p.frame_offsets(off), want), level
        finally:
            p.close()
    if not c["voicing"]:
        return
    p = Plan(PC.components(c), "lld", device=-1)
    try:
        n = len(PC.vit_names(c)) + len(PC.jit_names(c))
        assert p.num_elements == 2 * n
        # the smoothed level has one row more than the frames, its delta two more again; the concatenation ends with the first
        assert np.array_equal(np.diff(p.frame_offsets(off)), [t + 1 if t else 0 for t in T])
    finally:
        p.close()


def test_table_reaches_every_spectrum_length():
    """nMag 257, 513, 1025 and 2049 (FFT 512 .. 4096); target axes beyond the 64 strides of one lane's peak mask"""
    assert {PC.n_mag(c) for c in PC.CASES} >= {257, 513, 1025, 2049}
    assert max(PC.n_pts(c) for c in PC.CASES) == 4096 and any(2049 < PC.n_pts(c) < 4096 for c in PC.CASES)
    for axis, values in PC.AXES.items():
        got = {c[axis] for c in PC.CASES}
        assert values <= got, (axis, values - got)


def _refused(c, level="lld"):
    with pytest.raises(RuntimeError) as e:
        Plan(PC.components(c), level, device=-1)
    return str(e.value)


@pytest.mark.parametrize("kw,msg", [
    (dict(nCand=9), r"cPitchShs\.nCandidates > 8 is not supported"),
    (dict(nCand=20), r"cPitchShs\.nCandidates > 8 is not supported"),
    (dict(bufLen=65), r"cPitchSmootherViterbi\.bufferLength must be 2\.\.64"),
    (dict(bufLen=1), r"cPitchSmootherViterbi\.bufferLength must be 2\.\.64"),
    (dict(nHarm=33), r"cPitchShs\.nHarmonics out of range"),
    (dict(sr=48000, nPts=4097), r"cSpecScale: unsupported number of points"),
    (dict(sr=96000), r"cSpecScale: unsupported number of points"),          # ComParE's 60 ms frames at 96 kHz: nMag = 4097
])
def test_limits_are_refused_when_the_plan_is_created(kw, msg):
    c = PC.case("refused", **kw)
    for level in ("lld", "shs", "jit"):
        if level == "shs" and "bufLen" in kw:
            Plan(PC.components(c), level, device=-1).close()     # the cPitchShs level alone has no Viterbi stage
            continue
        text = _refused(c, level)
        assert re.search(r"\(%d\): .*%s" % (capi.ERR_UNSUPPORTED, msg), text), text


def test_shs_level_feeds_no_jitter_or_gate():
    """cPitchJitter and the cValbasedSelector gates need the Viterbi-smoothed F0: pointed at the cPitchShs level they are refused"""
    c = PC.BY_NAME["anchor_compare16"]
    cs = [x for x in PC.components(c) if x.name != b"jit"]
    from opensmile_b200 import comp
    cs.append(comp("cPitchJitter", "jit", "wave", "jit", F0reader_dmLevel="shs", F0field="F0raw", jitterLocal=1))
    with pytest.raises(RuntimeError, match="cPitchJitter: the F0 level must come from cPitchSmootherViterbi"):
        Plan(cs, "jit", device=-1)
