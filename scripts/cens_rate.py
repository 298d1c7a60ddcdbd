"""Device-resident rate of the shipped config/chroma/chroma_fft.conf with and without a cCens level behind its chroma level: PCM and
rows stay in device memory, the time is CUDA events around run_device after a warm-up on the same batch.

    python scripts/cens_rate.py [--frames 1000000] [--reps 7] [--out /tmp/cens_rate.json]

One workload: a batch of 10 s, 16 kHz mono utterances holding at least --frames output rows, run once with the chroma level as the
output level and once with a default cCens (winlength 41, Hanning, l2norm) behind it.  The difference of the two medians is what the
CENS stage adds; kernels_ms splits one profiled run by kernel.  Prints one JSON line per graph with the card's name, power limit and clocks."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CENS = ("[censDev:cCens]\nreader.dmLevel = chroma\nwriter.dmLevel = cens\ndownsampleRatio = 1\n")


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm,temperature.gpu", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split("\n")[0]
        return [x.strip() for x in q.split(",")]
    except Exception as e:                          # measured numbers are still printed, the card columns say why they are missing
        return ["unknown (%s)" % e] + ["unknown"] * 4


def cens_conf(conf, d):
    """chroma_fft.conf with a cCens behind the chroma level, the CSV sink reading it"""
    text = open(conf).read()
    text = text.replace("instance[chroma].type = cChroma", "instance[chroma].type = cChroma\ninstance[censDev].type = cCens", 1)
    i = text.index("[csvSink:cCsvSink]")
    text = text[:i] + CENS + "\n" + text[i:]
    j = text.index("reader.dmLevel", text.index("[csvSink:cCsvSink]"))
    k = text.index("\n", j)
    text = text[:j] + "reader.dmLevel = cens" + text[k:]
    p = os.path.join(d, "chroma_cens.conf")
    open(p, "w").write(text)
    return p


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from opensmile_b200 import Plan, Session
    conf = os.path.join(ROOT, "oracle", "_ref", "config", "chroma", "chroma_fft.conf")
    assert os.path.exists(conf), "oracle/_ref/config/chroma (build()) is missing"
    res = []
    sr = 16000
    with tempfile.TemporaryDirectory() as d:
        for graph, path in (("chroma_fft.conf", conf), ("chroma_fft.conf + cCens", cens_conf(conf, d))):
            s = Session(path, options={"outputfile": "x.csv"}, device=-1)
            comps, level = s.components(float(sr), 1)
            names = s.element_names(float(sr))
            s.close()
            plan = Plan(list(comps), level, device=0)
            n_utt_len = 10 * sr
            per = plan.num_frames(n_utt_len)
            n_utt = (a.frames + per - 1) // per
            rng = np.random.default_rng(1)
            t = np.arange(n_utt_len) / sr
            base = (6000 * np.sin(2 * np.pi * 220 * t) + 3000 * np.sin(2 * np.pi * 330 * t) + rng.normal(0, 300, t.size)).astype(np.int16)
            d_pcm = torch.from_numpy(np.tile(base, n_utt)).cuda()
            off = (np.arange(n_utt + 1, dtype=np.int64) * n_utt_len)
            fo = plan.frame_offsets(off)
            d_out = plan.run_device(d_pcm, off, frame_offsets=fo)            # warm-up (sizes the plan's buffers)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ms = []
            for _ in range(a.reps):
                e0.record()
                plan.run_device(d_pcm, off, d_out=d_out, frame_offsets=fo)
                e1.record()
                torch.cuda.synchronize()
                ms.append(e0.elapsed_time(e1))
            rows = int(fo[-1])
            # per-kernel split: one profiled run (an event after every launch, everything on one stream)
            plan.set_profiling(True)
            plan.run_device(d_pcm, off, d_out=d_out, frame_offsets=fo)
            torch.cuda.synchronize()
            kernels = [(k, round(v, 4)) for k, v in plan.kernel_profile()]
            plan.set_profiling(False)
            plan.close()
            name, plim, clk, cur, temp = card()
            r = dict(workload=graph + " %d Hz mono" % sr, first_element=names[0], utterances=int(n_utt), rows=rows,
                     ms_median=float(np.median(ms)), ms_all=[round(x, 3) for x in ms], kernels_ms=kernels, rows_per_s=rows / (np.median(ms) / 1e3),
                     gpu=name, power_limit=plim, max_sm_clock=clk, sm_clock_after=cur, temperature=temp)
            print(json.dumps(r))
            res.append(r)
            del d_pcm, d_out
            torch.cuda.empty_cache()
    print(json.dumps(dict(cens_stage_ms=res[1]["ms_median"] - res[0]["ms_median"],
                          cens_share_of_chroma=(res[1]["ms_median"] - res[0]["ms_median"]) / res[0]["ms_median"])))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        json.dump(res, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
