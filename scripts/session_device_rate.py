"""Session.extract_tensor (audio held as a padded CUDA tensor, rows left in device memory) against Session.extract_pcm (the same
samples in host memory, rows copied back to host memory), on one workload: 1000 utterances of about 3 s (ragged, 2.7 .. 3.3 s) at
16 kHz, mono int16, for the shipped MFCC12_0_D_A (LLD), eGeMAPSv02 -csvoutput (88 values) and ComParE_2016 -csvoutput (6373 values).

    python scripts/session_device_rate.py [--reps 7] [--out results.json]
    python scripts/session_device_rate.py --profile [--out ...]

Timing: every shape is warmed up first, then the two paths alternate.  Device path: CUDA events on the current stream around the
call, then a stream synchronise.  Host path: a host clock around the blocking call; its PCM sits in page-locked memory (the
pipelined H2D copies of extract_pcm are then asynchronous).  --profile is a separate run under torch.profiler (CUDA activities):
the packing kernel's time and achieved bytes/s against the H100 SXM's 3.35 TB/s, and the memcpy list of one extract_tensor call.
Prints one JSON line per configuration with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CONFS = [("MFCC12_0_D_A", "mfcc/MFCC12_0_D_A.conf", {"O": "x.htk"}),
         ("eGeMAPSv02", "egemaps/v02/eGeMAPSv02.conf", {"csvoutput": "x.csv"}),
         ("ComParE_2016", "compare16/ComParE_2016.conf", {"csvoutput": "x.csv"})]
HBM_BYTES_PER_S = 3.35e12


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split("\n")[0]
        return [x.strip() for x in q.split(",")]
    except Exception as e:                          # measured numbers are still printed, the card columns say why they are missing
        return ["unknown (%s)" % e, "unknown"]


def workload(torch, n_utt=1000, sr=16000):
    from opensmile_b200.synth import voiced_pcm
    rng = np.random.default_rng(0)
    lens = rng.integers(int(2.7 * sr), int(3.3 * sr) + 1, size=n_utt).astype(np.int64)
    base = voiced_pcm(int(lens.max()) + 4096, sr, seed=1)
    x = np.zeros((n_utt, int(lens.max())), np.int16)
    for u, n in enumerate(lens):
        s0 = int(rng.integers(0, 4096))
        x[u, :n] = base[s0:s0 + n]
    host = torch.empty(int(lens.sum()), dtype=torch.int16).pin_memory().numpy()
    host[:] = np.concatenate([x[u, :n] for u, n in enumerate(lens)])
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    return lens, torch.from_numpy(x).cuda(), host, off


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from opensmile_b200 import Session
    ref = os.path.join(ROOT, "oracle", "_ref", "config")
    assert os.path.isdir(ref), "oracle/_ref/config (build()) is missing"
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing is measured")
    name, plim = card()
    sr = 16000
    lens, d_pcm, host, off = workload(torch)
    audio_s = float(lens.sum()) / sr
    res = []
    for label, conf, opts in CONFS:
        s = Session(os.path.join(ref, conf), options=opts, device=0)
        d_rows, fo = s.extract_tensor(d_pcm, lens, sr)                  # warm-up of both paths on this shape
        h_rows, fo_h = s.extract_pcm(host, off, sr, 1)
        torch.cuda.synchronize()
        r = dict(workload="%s, %d x ~3 s int16 mono at 16 kHz" % (label, len(lens)), rows=int(fo[-1]), values_per_row=int(h_rows.shape[1]),
                 audio_s=audio_s, gpu=name, power_limit=plim,
                 rows_equal=bool(np.array_equal(d_rows.cpu().numpy().view(np.uint32), h_rows.view(np.uint32)) and list(fo) == list(fo_h)))
        if a.profile:
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                s.extract_tensor(d_pcm, lens, sr)
                torch.cuda.synchronize()
            with tempfile.TemporaryDirectory() as tmp:
                trace = os.path.join(tmp, "trace.json")
                prof.export_chrome_trace(trace)
                ev = json.load(open(trace))["traceEvents"]
            pack = [e for e in ev if e.get("cat") == "kernel" and "pcm_pack_kernel" in e["name"]]
            pack_us = sum(float(e["dur"]) for e in pack)
            moved = 2 * 2 * int(lens.sum())                                 # int16 samples read once and written once
            r.update(pack_kernel_us=pack_us, pack_bytes=moved, pack_bytes_per_s=moved / (pack_us * 1e-6) if pack_us else None,
                     pack_share_of_3_35TBps=(moved / (pack_us * 1e-6)) / HBM_BYTES_PER_S if pack_us else None,
                     memcpys=[(e["name"], int(e.get("args", {}).get("bytes", -1))) for e in ev if e.get("cat") == "gpu_memcpy"],
                     kernels=len([e for e in ev if e.get("cat") == "kernel"]))
        else:
            dev_ms, host_ms = [], []
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            stream = torch.cuda.current_stream()
            for _ in range(a.reps):
                e0.record(stream)
                s.extract_tensor(d_pcm, lens, sr)
                e1.record(stream)
                stream.synchronize()
                dev_ms.append(e0.elapsed_time(e1))
                t0 = time.perf_counter()
                s.extract_pcm(host, off, sr, 1)
                host_ms.append((time.perf_counter() - t0) * 1e3)
            dm, hm = float(np.median(dev_ms)), float(np.median(host_ms))
            r.update(extract_tensor_ms_median=dm, extract_pcm_ms_median=hm, extract_tensor_ms=[round(x, 3) for x in dev_ms],
                     extract_pcm_ms=[round(x, 3) for x in host_ms], extract_tensor_rows_per_s=fo[-1] / (dm * 1e-3),
                     extract_pcm_rows_per_s=fo[-1] / (hm * 1e-3), extract_tensor_audio_s_per_s=audio_s / (dm * 1e-3),
                     extract_pcm_audio_s_per_s=audio_s / (hm * 1e-3), speedup=hm / dm)
        s.close()
        print(json.dumps(r))
        res.append(r)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        json.dump(res, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
