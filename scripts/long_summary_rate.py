"""Full-input summaries of long recordings through Session.extract_tensor: the shipped eGeMAPSv02 and ComParE_2016 -csvoutput on
8 x 10-minute utterances and on 1 x 60-minute utterance (16 kHz mono int16, already on the GPU), where every cFunctionals contour
takes the long path (work space slices in HBM, radix rank selection for the percentiles).

    python scripts/long_summary_rate.py [--reps 3] [--out results.json]

Timing: every shape is warmed up first; CUDA events on the current stream around each call, then a synchronise.  A separate run of
one call per shape under torch.profiler (CUDA activities) gives the kernel time by family: the functionals' share, and within it the
per-warp kernel (functionals_kernel) against the rank selection (pctl_select_kernel), beside the LLD graph's kernels.  Prints one
JSON line per workload with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CONFS = [("eGeMAPSv02", "egemaps/v02/eGeMAPSv02.conf"), ("ComParE_2016", "compare16/ComParE_2016.conf")]
SHAPES = [("8 x 10 min", 8, 600), ("1 x 60 min", 1, 3600)]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split("\n")[0]
        return [x.strip() for x in q.split(",")]
    except Exception as e:
        return ["unknown (%s)" % e, "unknown"]


def kernel_split(prof):
    with tempfile.TemporaryDirectory() as tmp:
        trace = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(trace)
        ev = json.load(open(trace))["traceEvents"]
    ms = {"functionals_kernel<long>": 0.0, "functionals_kernel<short>": 0.0, "pctl_select_kernel": 0.0, "other": 0.0}
    for e in ev:
        if e.get("cat") != "kernel":
            continue
        n, d = e["name"], e["dur"] / 1000.0
        if "pctl_select_kernel" in n:
            ms["pctl_select_kernel"] += d
        elif "functionals_kernel<true>" in n or "functionals_kernelILb1" in n:
            ms["functionals_kernel<long>"] += d
        elif "functionals_kernel" in n:
            ms["functionals_kernel<short>"] += d
        else:
            ms["other"] += d
    total = sum(ms.values())
    fn = total - ms["other"]
    return {k: round(v, 3) for k, v in ms.items()}, round(total, 3), round(fn / total, 4) if total else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from opensmile_b200 import Session
    from opensmile_b200.synth import mixed_pcm
    from torch.profiler import ProfilerActivity, profile
    ref = os.path.join(ROOT, "oracle", "_ref", "config")
    assert os.path.isdir(ref), "oracle/_ref/config (build()) is missing"
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing is measured")
    name, plim = card()
    sr = 16000
    res = []
    for shape, n_utt, secs in SHAPES:
        n = secs * sr
        pcm = torch.from_numpy(np.stack([mixed_pcm(n, sr, seed=30 + u) for u in range(n_utt)])).cuda()
        lens = [n] * n_utt
        for label, conf in CONFS:
            s = Session(os.path.join(ref, conf), options={"csvoutput": "x.csv"}, device=0)
            s.extract_tensor(pcm, lens, sr)                                     # warm-up: sizes the plan, work spaces and row buffers
            torch.cuda.synchronize()
            times = []
            for _ in range(a.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                rows, fo = s.extract_tensor(pcm, lens, sr)
                e1.record()
                torch.cuda.synchronize()
                times.append(e0.elapsed_time(e1))
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                s.extract_tensor(pcm, lens, sr)
                torch.cuda.synchronize()
            split, kernel_ms, fn_share = kernel_split(prof)
            s.close()
            r = dict(workload="%s %s, int16 mono 16 kHz, extract_tensor" % (label, shape), audio_s=n_utt * secs, values_per_row=int(rows.shape[1]),
                     ms_per_call=[round(t, 2) for t in times], ms_per_call_median=round(float(np.median(times)), 2),
                     profiled_kernel_ms=kernel_ms, functionals_share_of_kernel_time=fn_share, kernel_ms_by_family=split,
                     finite=bool(torch.isfinite(rows).all().item()), gpu=name, power_limit=plim)
            print(json.dumps(r), flush=True)
            res.append(r)
        del pcm
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
