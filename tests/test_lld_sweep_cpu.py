"""The LLD case table (tests/lld_cases.py) on description-only plans: every case opens, and the plan's frame geometry, FFT size,
element count and row offsets of the case's ragged batch are the oracle's."""
import numpy as np
import pytest

import lld_cases as LC
from opensmile_b200 import Plan
from oracle import oracle


@pytest.mark.parametrize("name", list(LC.BY_NAME))
def test_case_opens_with_the_oracle_geometry(name):
    c = LC.BY_NAME[name]
    p = Plan(LC.components(c), "lld", device=-1)
    try:
        (fe, _, _), _ = LC.oracle_cfg(c)
        utts, pcm, off = LC.batch(c)
        N, H, nfft, _ = oracle.geometry(fe, 0)
        assert (p.frame_size, p.frame_step, p.fft_size) == (c["frame"], c["hop"], nfft) == (N, H, nfft)
        assert p.num_elements == 3 * LC.n_static(c)
        T = [max(oracle.geometry(fe, len(x) // c["n_chan"])[3], 0) for x in utts]
        assert np.array_equal(p.frame_offsets(off), np.concatenate([[0], np.cumsum(T)]))
    finally:
        p.close()


def test_batches_cover_every_start_residue_and_the_chunk_edges():
    """the first samples of the utterances take every residue mod 8 (the bulk copy lands at every misalignment), and the lengths
    reach one chunk of 16 tiles on both sides and an utterance of more than five chunks"""
    for c in LC.CASES:
        utts, _, off = LC.batch(c)
        (fe, _, _), _ = LC.oracle_cfg(c)
        T = [oracle.geometry(fe, len(x) // c["n_chan"])[3] for x in utts]
        starts = {int(off[i]) % 8 for i in range(len(utts)) if T[i] > 0}
        assert starts == set(range(8)), (c["name"], starts)
        C = 16 * LC.tile_frames(c)
        assert {C - 1, C, C + 1} <= set(T) and max(T) > 5 * C, c["name"]


def test_expected_instances_name_every_launcher_shape():
    """the table reaches both lld512 instances, every full-width lld_kernel FFT size, the narrow 2048 / 4096 tiles, scalar and
    pair loads, and the general (PLP) back end"""
    kinds = {c["expect"] for c in LC.CASES}
    assert {LC.FAST13, LC.FAST16} <= kinds
    for m in (256, 512, 1024, 2048):
        assert any(k.startswith("lld_kernel<%d," % m) for k in kinds), m
    assert LC.gen(1024, 8, 256, 1) in kinds and LC.gen(2048, 4, 128, 1) in kinds
    assert any(",SCALAR," in k for k in kinds) and any(k.endswith(",GEN>") for k in kinds)
    fused = {c["windows"] for c in LC.CASES if LC.expect_fused(c)}
    assert {(1, 1), (1, 2), (2, 1), (2, 2), (3, 3), (4, 4), (5, 3)} <= fused
    assert not any(LC.expect_fused(c) for c in LC.CASES if sum(c["windows"]) > 8)
