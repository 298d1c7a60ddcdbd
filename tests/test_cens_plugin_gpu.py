"""GPU box: the reference's SMILExtract (dynamic build of the unmodified sources) with the B200 plugin runs the FFT path of
tests/configs/cens_taps.conf up to its CENS level (downsampleRatio = 10) inside cLldBlockB200, and the reference's own CSV / HTK sinks
write the rows.  The CSV must carry the reference's header and time column (the chroma rows' times, 10 ms apart, although the
level period is 0.1 s), the HTK header the period 0.1 s, and the values those of the reference's file
(tests/golden/cens_fft_ds10.csv) away from quantisation thresholds."""
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from cens_harness import G, ROOT, TAPS, case_input, mg  # noqa: E402
from oracle import refrun  # noqa: E402  (HTK reader and WAV writer only)
from test_cens_gpu import near_threshold_rows  # noqa: E402

PLUG = os.path.join(ROOT, "plugin")
SMILE = os.path.join(ROOT, "oracle", "_ref_dyn", "SMILExtract")

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not (os.access(SMILE, os.X_OK) and os.path.exists(os.path.join(PLUG, "plugins", "libosm_b200_plugin.so"))),
                                 reason="dynamic reference build / plugin not built")]

WRAP = """[componentInstances:cComponentManager]
instance[dataMemory].type=cDataMemory
instance[waveIn].type=cWaveSource
instance[b200].type=cLldBlockB200
instance[csv].type=cCsvSink
instance[htk].type=cHtkSink
printLevelStats=0
nThreads=1

[waveIn:cWaveSource]
writer.dmLevel=wave
filename=\\cm[inputfile(I){test.wav}:name of input file]
monoMixdown=1

[b200:cLldBlockB200]
reader.dmLevel=wave
writer.dmLevel=cens
graphConf=%s
captureTo=cens_fft
graphOption[0]=downsampleRatio=10
device=0

[csv:cCsvSink]
reader.dmLevel=cens
filename=\\cm[csvoutput{o.csv}:CSV output]
delimChar=;
timestamp=1
number=0
printHeader=1

[htk:cHtkSink]
reader.dmLevel=cens
filename=\\cm[htkoutput{o.htk}:HTK output]
"""


def test_plugin_writes_the_reference_cens_files(tmp_path):
    case = "ds10"
    pcm, sr = case_input(case)
    wav, conf = str(tmp_path / "in.wav"), str(tmp_path / "cens_b200.conf")
    csv, htk = str(tmp_path / "o.csv"), str(tmp_path / "o.htk")
    refrun.write_wav(wav, pcm, sr)
    open(conf, "w").write(WRAP % TAPS)
    r = subprocess.run([SMILE, "-C", conf, "-I", wav, "-csvoutput", csv, "-htkoutput", htk, "-l", "1"], cwd=PLUG,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
    assert r.returncode == 0 and "(ERR)" not in r.stdout, r.stdout
    got = open(csv).read().strip().split("\n")
    ref = open(os.path.join(HERE, "golden", "cens_fft_ds10.csv")).read().strip().split("\n")
    assert got[0] == ref[0] and len(got) == len(ref)
    assert [ln.split(";")[0] for ln in got[1:]] == [ln.split(";")[0] for ln in ref[1:]]      # 0.000000, 0.010000, ...
    gv = np.array([[float(x) for x in ln.split(";")[1:]] for ln in got[1:]])
    rv = np.array([[float(x) for x in ln.split(";")[1:]] for ln in ref[1:]])
    keep = ~near_threshold_rows(G["chroma_fft_" + case], mg.options(case)["winlength"])
    assert keep.sum() > 0 and np.abs(gv - rv)[keep].max() <= 2e-6          # the CSV prints 7 significant digits
    rows, hdr = refrun.read_htk(htk)
    assert hdr["period"] == int(G["period_fft_" + case]) == 1000000 and rows.shape == G["cens_fft_" + case].shape
