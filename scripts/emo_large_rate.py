"""Device-resident LLD rate of the shipped config/misc/emo_large.conf (centred 25 ms frames, 112 LLD columns): PCM and rows stay in
device memory, the time is CUDA events around run_device after a warm-up on the same batch.

    python scripts/emo_large_rate.py [--frames 1000000] [--reps 5] [--out /tmp/emo_large_rate.json]

One workload: a batch of 10 s utterances, 16 kHz mono, holding at least --frames output rows.  Prints one JSON line with the
card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split("\n")[0]
        return [x.strip() for x in q.split(",")]
    except Exception as e:                          # measured numbers are still printed, the card columns say why they are missing
        return ["unknown (%s)" % e, "unknown", "unknown"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from opensmile_b200 import Plan, Session
    conf = os.path.join(ROOT, "oracle", "_ref", "config", "misc", "emo_large.conf")
    assert os.path.exists(conf), "oracle/_ref/config/misc (build()) is missing"
    name, plim, clk = card()
    res = []
    for sr in (16000,):
        s = Session(conf, options={"lldcsvoutput": "x.csv"}, device=-1)
        comps, level = s.components(float(sr), 1)
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
        lk = plan.last_lld_launch()
        plan.close()
        r = dict(workload="emo_large.conf LLD %d Hz mono" % sr, utterances=int(n_utt), rows=rows, audio_s=float(n_utt * 10),
                 ms_median=float(np.median(ms)), ms_all=[round(x, 3) for x in ms], rows_per_s=rows / (np.median(ms) / 1e3),
                 realtime_factor=float(n_utt * 10) / (np.median(ms) / 1e3), kernel=lk.kernel,
                 gpu=name, power_limit=plim, max_sm_clock=clk)
        print(json.dumps(r))
        res.append(r)
        del d_pcm, d_out
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        json.dump(res, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
