"""Device-resident rate of the shipped config/chroma/chroma_filt.conf (cTonefilt -> cChroma on the wave level, tonefilt.cu): PCM
and rows stay in device memory, the time is CUDA events around run_device after a warm-up on the same batch.

    python scripts/tonefilt_rate.py [--reps 5] [--out /tmp/tonefilt_rate.json]

Workloads: 10 000 utterances of 3 s at 16 kHz and at 44.1 kHz, and one 600 s utterance at 16 kHz.  Prints one JSON line per
workload with the card's name and power limit, and the FP64 bound of the block products computed from shapes (4 P nNotes flops per
row, P rounded up to whole k-steps of 4 and the note columns to whole tiles, as the kernel runs them) at the data sheet's 67 TFLOP/s
(H100 SXM, FP64 tensor cores).  A long utterance runs its products twice (aggregate and output passes)."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from chroma_rate import card  # noqa: E402

FP64_TC = 67e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--utts", type=int, default=10000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from opensmile_b200 import Plan, Session
    conf = os.path.join(ROOT, "oracle", "_ref", "config", "chroma", "chroma_filt.conf")
    assert os.path.exists(conf), "oracle/_ref/config/chroma (build()) is missing"
    name, plim, clk = card()
    res = []
    for sr, secs, n_utt in ((16000, 3, a.utts), (44100, 3, a.utts), (16000, 600, 1)):
        s = Session(conf, options={"outputfile": "x.csv"}, device=-1)
        comps, level = s.components(float(sr), 1)
        s.close()
        plan = Plan(list(comps), level, device=0)
        n_len = secs * sr
        rng = np.random.default_rng(1)
        t = np.arange(n_len) / sr
        base = (6000 * np.sin(2 * np.pi * 220 * t) + 3000 * np.sin(2 * np.pi * 330 * t) + rng.normal(0, 300, t.size)).astype(np.int16)
        d_pcm = torch.from_numpy(np.tile(base, n_utt)).cuda()
        off = np.arange(n_utt + 1, dtype=np.int64) * n_len
        fo = plan.frame_offsets(off)
        d_out = plan.run_device(d_pcm, off, frame_offsets=fo)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ms = []
        for _ in range(a.reps):
            e0.record()
            plan.run_device(d_pcm, off, d_out=d_out, frame_offsets=fo)
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        plan.close()
        rows = int(fo[-1])
        P, nN = int(round(0.01 * sr)), 72
        flops = 4.0 * ((P + 3) // 4 * 4) * ((2 * nN + 7) // 8 * 8) / 2 * rows * (2 if rows // n_utt > 1024 else 1)
        med = float(np.median(ms))
        r = dict(workload="chroma_filt.conf %d Hz, %d x %d s" % (sr, n_utt, secs), rows=rows, ms_median=med,
                 ms_all=[round(x, 3) for x in ms], rows_per_s=rows / (med / 1e3), fp64_flops=flops,
                 fp64_bound_ms=flops / FP64_TC * 1e3, fp64_tflops_achieved=flops / (med / 1e3) / 1e12,
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
