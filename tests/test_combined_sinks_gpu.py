"""GPU tests of sessions whose active sinks read a summary level and an LLD level: one combined run writes, byte for byte, the
files the two single-level sessions write (every LLD sink kind, append mode across two calls, an instance name, ragged batches
with utterances of a few 60 ms frames, a long one and stereo 44.1 kHz), and Session.extract_tensor(..., with_lld=True) gives, bit
for bit, the rows of the two single-level extract_tensor calls, on int16 and float32 input, without host <-> device copies of the
samples or the rows."""
import json

import numpy as np
import pytest
import scipy.io.wavfile
import torch

from opensmile_b200 import Session
from opensmile_b200.synth import mixed_pcm, stereo_mixed_pcm
from combined_sinks_cases import CONFS, conf_path, have_confs

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not have_confs(), reason="reference configuration files not built (make -C oracle ref)")]
# 1 - 5 frames of the 60 ms pitch level (10 ms step), a long utterance (81 s: the cFunctionals percentile path takes contours of at
# most 8192 frames) and an ordinary one
MONO = [960 + 160 * k for k in range(5)] + [81 * 16000, 37003]
LLD_SINKS = {"csv": ("lldcsvoutput", "lld_csv_paths", ".csv"), "htk": ("lldhtkoutput", "lld_htk_paths", ".htk"),
             "arff": ("lldarffoutput", "lld_arff_paths", ".arff")}


def write_batch(tmp_path):
    wavs = []
    for u, n in enumerate(MONO):
        p = str(tmp_path / ("m%d.wav" % u))
        scipy.io.wavfile.write(p, 16000, mixed_pcm(n, 16000, seed=u))
        wavs.append(p)
    p = str(tmp_path / "s.wav")
    scipy.io.wavfile.write(p, 44100, stereo_mixed_pcm(int(1.7 * 44100), 44100, seed=7).reshape(-1, 2))
    return wavs + [p]


def outputs(tmp_path, tag, n, ext, shared):
    """per-input paths, or one path for every input (append mode)"""
    return [str(tmp_path / ("%s%s" % (tag, ext) if shared else "%s%d%s" % (tag, u, ext))) for u in range(n)]


@pytest.mark.parametrize("kind", sorted(LLD_SINKS))
@pytest.mark.parametrize("name", sorted(CONFS))
def test_combined_files_are_the_single_level_files(name, kind, tmp_path):
    opt, arg, ext = LLD_SINKS[kind]
    wavs = write_batch(tmp_path)
    base = {"instname": "utt_1", "relation": "rel"}
    both = Session(conf_path(name), options={**base, "csvoutput": "f.csv", opt: "l" + ext}, device=0)
    summ = Session(conf_path(name), options={**base, "csvoutput": "f.csv"}, device=0)
    lld = Session(conf_path(name), options={**base, opt: "l" + ext}, device=0)
    shared = kind == "arff"                                  # cArffSink appends every input to one file (appendarfflld = 1)
    got_f, want_f = outputs(tmp_path, "bf", len(wavs), ".csv", False), outputs(tmp_path, "sf", len(wavs), ".csv", False)
    got_l, want_l = outputs(tmp_path, "bl", len(wavs), ext, shared), outputs(tmp_path, "sl", len(wavs), ext, shared)
    for _ in range(2):                                       # a second call appends to the ARFF files, rewrites the others
        fb = both.extract_files(wavs, csv_paths=got_f, **{arg: got_l})
        fs = summ.extract_files(wavs, csv_paths=want_f)
        lld.extract_files(wavs, **{arg.replace("lld_", ""): want_l})
        assert list(fb) == list(fs)
    for g, w in zip(got_f + got_l, want_f + want_l):
        assert open(g, "rb").read() == open(w, "rb").read(), (name, kind, g)
    for s in (both, summ, lld):
        s.close()


def padded(lengths, fmt, seed=0):
    """a mono CUDA batch [B, L] with garbage padding, and the same samples as int16 for reference"""
    rng = np.random.default_rng(seed)
    x = rng.integers(-32768, 32767, size=(len(lengths), max(lengths) + 11)).astype(np.int16)
    for u, n in enumerate(lengths):
        x[u, :n] = mixed_pcm(n, 16000, seed=seed + u)
    t = torch.from_numpy(x)
    return (t if fmt == "int16" else (t.float() / 32768.0)).contiguous().cuda()


def same_bits(a, b):
    a, b = a.cpu().numpy(), b.cpu().numpy()
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.mark.parametrize("fmt", ["int16", "float32"])
@pytest.mark.parametrize("name", sorted(CONFS))
def test_combined_tensor_rows_are_the_single_level_rows(name, fmt):
    lens = np.array([0, 1] + MONO, np.int64)
    x = padded(lens, fmt)
    both = Session(conf_path(name), options={"csvoutput": "f.csv", "lldcsvoutput": "l.csv"}, device=0)
    summ = Session(conf_path(name), options={"csvoutput": "f.csv"}, device=0)
    lld = Session(conf_path(name), options={"lldcsvoutput": "l.csv"}, device=0)
    rows, fo, lrows, lfo = both.extract_tensor(x, lens, 16000, with_lld=True)
    want, wfo = summ.extract_tensor(x, lens, 16000)
    lwant, wlfo = lld.extract_tensor(x, lens, 16000)
    assert list(fo) == list(wfo) and list(lfo) == list(wlfo)
    assert same_bits(rows, want) and same_bits(lrows, lwant), name
    for s in (both, summ, lld):
        s.close()


PROFILE = r"""
import json, sys, tempfile
import numpy as np, torch
sys.path.insert(0, sys.argv[1])
from opensmile_b200 import Session
from test_combined_sinks_gpu import padded
s = Session(sys.argv[2], options={"csvoutput": "f.csv", "lldcsvoutput": "l.csv"}, device=0)
lens = np.array([3 * 16000 - 5 * u for u in range(16)], np.int64)
x = padded(lens, "int16")
s.extract_tensor(x, lens, 16000, with_lld=True)                       # warm-up: plans, buffers, schedule
torch.cuda.synchronize()
with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]) as prof:
    rows, _, lrows, _ = s.extract_tensor(x, lens, 16000, with_lld=True)
    torch.cuda.synchronize()
with tempfile.TemporaryDirectory() as tmp:
    prof.export_chrome_trace(tmp + "/trace.json")
    ev = json.load(open(tmp + "/trace.json"))["traceEvents"]
print(json.dumps({"copies": [(e["name"], int(e.get("args", {}).get("bytes", 0))) for e in ev
                             if e.get("cat") == "gpu_memcpy" and ("HtoD" in e["name"] or "DtoH" in e["name"])],
                  "kernels": [e["name"] for e in ev if e.get("cat") == "kernel"], "n_utt": len(lens), "samples": x.numel(),
                  "rows": rows.numel(), "lld_rows": lrows.numel(), "lld_cols": lrows.shape[1]}))
"""


@pytest.mark.parametrize("name", ["egemaps", "compare"])
def test_no_host_device_copy_of_samples_or_rows(name):
    # its own process: a torch.profiler session leaves the profiler of the process that ran it in a state later traces depend on
    import os
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    out = subprocess.run([sys.executable, "-c", PROFILE, here, conf_path(name)], capture_output=True, text=True, timeout=600,
                         env={**os.environ, "PYTHONPATH": os.pathsep.join([os.path.dirname(here), here])})
    assert out.returncode == 0, out.stderr[-3000:]
    r = json.loads(out.stdout.strip().splitlines()[-1])
    assert any("gather_rows_kernel" in k for k in r["kernels"]), r["kernels"]
    # offsets and counts (a few int64 per utterance), and the gather's column list
    limit = 64 * (r["n_utt"] + 1) + 8 * r["lld_cols"]
    assert all(b <= limit for _, b in r["copies"]), (r["copies"], limit)
    assert limit < min(r["samples"] * 2, r["rows"] * 4, r["lld_rows"] * 4)


def test_cli_writes_both_levels_from_one_run(tmp_path):
    import os
    import subprocess
    cli = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "opensmile_b200", "SMILExtract_b200")
    wav = str(tmp_path / "a.wav")
    scipy.io.wavfile.write(wav, 16000, mixed_pcm(37003, 16000, seed=3))
    t = lambda n: str(tmp_path / n)
    run = lambda *a: subprocess.run([cli, "-C", conf_path("egemaps"), "-I", wav, *a], check=True, capture_output=True, timeout=300)
    run("-csvoutput", t("bf.csv"), "-lldcsvoutput", t("bl.csv"), "-lldhtkoutput", t("bl.htk"))
    run("-csvoutput", t("sf.csv"))
    run("-lldcsvoutput", t("sl.csv"))
    run("-lldhtkoutput", t("sl.htk"))
    for g, w in (("bf.csv", "sf.csv"), ("bl.csv", "sl.csv"), ("bl.htk", "sl.htk")):
        assert open(t(g), "rb").read() == open(t(w), "rb").read(), g
