"""cFunctionals on contours longer than 8 192 frames on the GPU (the long path of opensmile_b200/csrc/functionals.cu: per-warp kernel on
a work space slice in HBM, radix rank selection for the percentiles): the kernel against the oracle on long synthetic contours of
every shape and functional family, ragged batches mixing both paths through run_device_cols, the shipped summary configurations on
10-minute / 3-minute recordings against the reference's rows (tests/golden/long_summaries.npz), a real-length combined LLD + summary
session, and a 60-minute utterance with the work space bounded."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import functionals_oracle as fo
from opensmile_b200 import capi
from opensmile_b200 import functionals as F
from test_functionals_cpu import SPEC_A, SPEC_B, SPEC_C, SPEC_D, SPEC_E, SPEC_F, SPEC_G, SPEC_H, SPEC_I, SPEC_J, SPEC_K, SPEC_L, to_c_spec
from long_summary_cases import CONFS, GOLDEN, INPUTS, REFCONF, sha256

pytestmark = pytest.mark.gpu
ALL_SPECS = {"is09": fo.IS09, "A": SPEC_A, "B": SPEC_B, "C": SPEC_C, "D": SPEC_D, "E": SPEC_E, "F": SPEC_F, "G": SPEC_G, "H": SPEC_H,
             "I": SPEC_I, "J": SPEC_J, "K": SPEC_K, "L": SPEC_L}
PCTL_NAMES = ("quartile", "iqr", "percentile", "pctlrange")


def contours(T, rng):
    """[T, 6]: zigzag (Peaks2's worst case: T - 4 extrema), constant, all-zero, mostly zero (N <= 8192 after nonZeroFuncts while
    T > 8192), a LLD-like random walk with positive and negative values, a smoothed pitch-like contour with unvoiced zeros"""
    t = np.arange(T)
    x = np.zeros((T, 6), np.float32)
    x[:, 0] = np.where(t % 2, 1.0, -1.0) * (1.0 + 1e-4 * t)
    x[:, 1] = 2.5
    nz = rng.random(T) < min(0.9, 4000.0 / max(T, 1))
    x[:, 3] = np.where(nz, rng.standard_normal(T) + 0.5, 0.0)
    x[:, 4] = np.cumsum(rng.standard_normal(T)) * 0.1
    f0 = 150 + 30 * np.sin(2 * np.pi * t / 800.0) + rng.standard_normal(T)
    x[:, 5] = np.where(np.sin(2 * np.pi * t / 137.0) > -0.3, f0, 0.0)
    return x


def check_against_oracle(spec, rows, got, exact_pctl=True):
    names = F.Functionals(to_c_spec(spec), ["c%d" % i for i in range(rows.shape[1])], 0.01, device=0)
    nm = names.element_names()
    names.close()
    ora = fo.functionals(spec, rows, 0.01)
    ok = (np.abs(got - ora) <= 2e-6 * np.abs(ora) + 1e-9) | (np.isnan(got) & np.isnan(ora))
    assert np.all(ok), [(nm[i], float(got[i]), float(ora[i])) for i in np.nonzero(~ok)[0][:8]]
    if exact_pctl:
        for i, n in enumerate(nm):
            if any(k in n.rsplit("_", 1)[1] for k in PCTL_NAMES):
                assert got[i].view(np.uint32) == ora[i].view(np.uint32) or got[i] == ora[i], (n, got[i], ora[i])


@pytest.mark.parametrize("T", [8192, 8193, 20000])
def test_long_contours_every_family_against_the_oracle(T):
    rows = contours(T, np.random.default_rng(T))
    for tag, spec in ALL_SPECS.items():
        f = F.Functionals(to_c_spec(spec), ["c%d" % i for i in range(rows.shape[1])], 0.01, device=0)
        got = f.run_host(rows, [0], [T])[0]
        f.close()
        check_against_oracle(spec, rows, got)


@pytest.mark.parametrize("T", [100000, 360000])
def test_longest_contours_against_the_oracle(T):
    """10^5 and 3.6 10^5 frames (1 h at 10 ms): every family whose oracle runs in seconds at that length (the Peaks2 pruning with
    dynRelThresh of SPEC_G is quadratic in the oracle; its statements are compared with the host build at length on the CPU)"""
    rows = contours(T, np.random.default_rng(T))
    specs = ["is09", "A", "B", "C", "H", "L"] + (["D", "I", "J", "K"] if T <= 100000 else [])
    for tag in specs:
        spec = ALL_SPECS[tag]
        f = F.Functionals(to_c_spec(spec), ["c%d" % i for i in range(rows.shape[1])], 0.01, device=0)
        got = f.run_host(rows, [0], [T])[0]
        f.close()
        check_against_oracle(spec, rows, got)


def _bind_cols():
    L = capi.lib()
    i64p = C.POINTER(C.c_int64)
    L.osm_b200_functionals_run_device_cols.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(C.c_int32), i64p, i64p, C.c_int32,
                                                       C.c_void_p, C.c_int64, C.c_void_p]
    return L


def test_ragged_batch_of_both_paths_through_run_device_cols():
    """empty, 1-frame, 8192-row, 8193-row and 10-minute utterances in one matrix, three instances on column subsets writing side by
    side into one summary row: every utterance's values equal its own single run bit for bit, and a rerun gives the same bits"""
    L = _bind_cols()
    lens = [0, 1, 8192, 8193, 60000, 37, 8193]
    rng = np.random.default_rng(9)
    rows = np.concatenate([contours(n, rng) for n in lens])
    off = np.concatenate([[0], np.cumsum(lens)])[:-1].astype(np.int64)
    nr = np.array(lens, np.int64)
    inst = [(SPEC_B, [0, 3, 4]), (SPEC_G, [5, 0]), (fo.IS09, [4, 1, 2, 3])]
    fs = [F.Functionals(to_c_spec(sp), ["c%d" % c for c in cols], 0.01, device=0) for sp, cols in inst]
    widths = [f.num_elements for f in fs]
    stride = sum(widths)
    d_rows = torch.from_numpy(rows).cuda()
    i64p = C.POINTER(C.c_int64)

    def run(u_sel):
        o, n = off[u_sel].copy(), nr[u_sel].copy()
        out = torch.full((len(o), stride), float("nan"), device="cuda")
        at = 0
        for f, (sp, cols), w in zip(fs, inst, widths):
            cc = np.array(cols, np.int32)
            st = L.osm_b200_functionals_run_device_cols(f._h, C.c_void_p(d_rows.data_ptr()), rows.shape[1], cc.ctypes.data_as(C.POINTER(C.c_int32)),
                                                        o.ctypes.data_as(i64p), n.ctypes.data_as(i64p), len(o),
                                                        C.c_void_p(out.data_ptr() + 4 * at), stride, None)
            assert st == capi.OK, capi.last_error()
            at += w
        torch.cuda.synchronize()
        return out.cpu().numpy()

    every = np.arange(len(lens))
    a, b = run(every), run(every)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    assert not np.isnan(a).any()
    for u in range(len(lens)):
        one = run(np.array([u]))
        assert np.array_equal(one[0].view(np.uint32), a[u].view(np.uint32)), (u, lens[u])
    # and against the oracle per instance
    at = 0
    for (sp, cols), w in zip(inst, widths):
        for u, n in enumerate(lens):
            if n and (n <= 8193 or sp is not SPEC_G):
                check_against_oracle(sp, rows[off[u]:off[u] + n][:, cols], a[u, at:at + w])
        at += w
    for f in fs:
        f.close()


def _golden():
    if not os.path.exists(GOLDEN):
        pytest.skip("tests/golden/long_summaries.npz missing")
    return np.load(GOLDEN)


@pytest.mark.skipif(not os.path.isdir(REFCONF), reason="reference configuration files not built (make -C oracle ref)")
@pytest.mark.parametrize("conf", sorted(CONFS))
def test_shipped_summaries_of_long_recordings_against_the_reference(conf):
    """eGeMAPSv02 / GeMAPSv01b: every value within 1e-4 of its own magnitude; ComParE_2016: the per-family rule of
    test_shipped_compare16_functionals_end_to_end (1e-5 of the family's scale, <= 0.5 % discontinuous flips, lpc / lpgain 2e-2) --
    the criteria the same configurations meet on short inputs"""
    from opensmile_b200.session import Session
    GL = _golden()
    names = [str(x) for x in GL["names_" + conf]]
    pcms = {k: make() for k, make in INPUTS.items()}
    for k, pcm in pcms.items():
        assert sha256(pcm) == str(GL["sha256_" + k]), "the generator of %s drifted" % k
    s = Session(os.path.join(REFCONF, CONFS[conf]), options={"csvoutput": "f.csv"}, device=0)
    assert s.element_names() == names
    keys = sorted(pcms)
    off = np.concatenate([[0], np.cumsum([len(pcms[k]) for k in keys])]).astype(np.int64)
    rows, fo_ = s.extract_pcm(np.concatenate([pcms[k] for k in keys]), off, 16000.0, 1)
    # the same through extract_tensor, audio resident on the GPU
    L = max(len(p) for p in pcms.values())
    pad = torch.zeros((len(keys), L), dtype=torch.int16)
    for i, k in enumerate(keys):
        pad[i, :len(pcms[k])] = torch.from_numpy(pcms[k])
    trow, tfo = s.extract_tensor(pad.cuda(), [len(pcms[k]) for k in keys], 16000.0)
    s.close()
    assert list(fo_) == list(range(len(keys) + 1)) and list(tfo) == list(fo_)
    assert np.array_equal(trow.cpu().numpy().view(np.uint32), rows.view(np.uint32))
    suffix = np.array([n.rsplit("_", 1)[-1] for n in names])
    report = {}
    for u, key in enumerate(keys):
        ref = GL["%s_%s" % (conf, key)]
        if conf != "compare":
            rel = np.abs(rows[u] - ref) / (np.abs(ref) + 1e-6)
            assert rel.max() < 1e-4, (key, names[int(np.argmax(rel))], float(rows[u][int(np.argmax(rel))]), float(ref[int(np.argmax(rel))]))
            continue
        bad_total = 0
        for sfx in np.unique(suffix):
            idx = np.nonzero(suffix == sfx)[0]
            scale = np.abs(ref[idx]).max() + 1e-12
            err = np.abs(rows[u, idx] - ref[idx]) / scale
            if sfx.startswith("lpc") or sfx == "lpgain":
                assert err.max() < 2e-2, (key, sfx, float(err.max()))
                continue
            bad = idx[err > 1e-5]
            if bad.size:
                report[(key, sfx)] = (int(bad.size), float(err.max()), names[int(bad[0])])
                bad_total += int(bad.size)
        assert bad_total <= 0.005 * len(names), (key, bad_total, sorted(report.items(), key=lambda kv: -kv[1][0])[:12])
    print(conf, "long recordings: values beyond 1e-5 of their family's scale:", report)


@pytest.mark.skipif(not os.path.isdir(REFCONF), reason="reference configuration files not built (make -C oracle ref)")
def test_ten_minute_combined_session_writes_the_single_level_files(tmp_path):
    import scipy.io.wavfile
    from opensmile_b200 import Session
    wav = str(tmp_path / "talk.wav")
    scipy.io.wavfile.write(wav, 16000, INPUTS["synth10"]())
    conf = os.path.join(REFCONF, CONFS["egemaps"])
    both = Session(conf, options={"csvoutput": "f.csv", "lldcsvoutput": "l.csv"}, device=0)
    summ = Session(conf, options={"csvoutput": "f.csv"}, device=0)
    lld = Session(conf, options={"lldcsvoutput": "l.csv"}, device=0)
    p = {k: str(tmp_path / (k + ".csv")) for k in ("bf", "bl", "sf", "sl")}
    both.extract_files([wav], csv_paths=[p["bf"]], lld_csv_paths=[p["bl"]])
    summ.extract_files([wav], csv_paths=[p["sf"]])
    lld.extract_files([wav], csv_paths=[p["sl"]])
    for s in (both, summ, lld):
        s.close()
    assert open(p["bf"], "rb").read() == open(p["sf"], "rb").read()
    assert open(p["bl"], "rb").read() == open(p["sl"], "rb").read()
    assert len(open(p["sl"]).read().strip().split("\n")) > 59000


@pytest.mark.skipif(not os.path.isdir(REFCONF), reason="reference configuration files not built (make -C oracle ref)")
def test_sixty_minute_utterance_with_a_bounded_work_space():
    """a 60-minute eGeMAPSv02 utterance through extract_tensor: finite values, the same bits on a second call, and the second call
    allocates no device memory (the work spaces have reached their size; a functionals object's is at most 256 MB)"""
    from opensmile_b200 import Session
    from opensmile_b200.synth import mixed_pcm
    pcm = torch.from_numpy(mixed_pcm(3600 * 16000, 16000, seed=4)).reshape(1, -1).cuda()
    s = Session(os.path.join(REFCONF, CONFS["egemaps"]), options={"csvoutput": "f.csv"}, device=0)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    rows, fo_ = s.extract_tensor(pcm, [pcm.shape[1]], 16000.0)
    torch.cuda.synchronize()
    free1 = torch.cuda.mem_get_info()[0]
    rows2, _ = s.extract_tensor(pcm, [pcm.shape[1]], 16000.0)
    torch.cuda.synchronize()
    free2 = torch.cuda.mem_get_info()[0]
    s.close()
    r = rows.cpu().numpy()
    assert r.shape == (1, 88) and np.isfinite(r).all()
    assert np.array_equal(r.view(np.uint32), rows2.cpu().numpy().view(np.uint32))
    assert free2 >= free1 - (2 << 20), (free1 - free2)
    print("60-minute eGeMAPSv02: device memory taken by the first call %.0f MB" % ((free0 - free1) / 2 ** 20))
