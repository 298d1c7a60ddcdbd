"""One combined Session.extract_tensor(..., with_lld=True) call (summary and LLD rows of one plan run) against the two single-level
calls it replaces (a summary session and an LLD session, each running its own plan), on one workload: 1000 utterances of about 3 s
(ragged, 2.7 .. 3.3 s) at 16 kHz, mono int16, for the shipped eGeMAPSv02 and ComParE_2016 (-csvoutput with -lldcsvoutput).

    python scripts/combined_sinks_rate.py [--reps 7] [--out results.json]

Every session is warmed up on the shape first, then the combined call and the pair of single calls alternate; each is timed with
CUDA events on the current stream around the call(s), then a stream synchronise.  The rows of both ways are compared bit for bit.
Prints one JSON line per configuration with the card's name and power limit."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from session_device_rate import card, workload  # noqa: E402

CONFS = [("eGeMAPSv02", "egemaps/v02/eGeMAPSv02.conf"), ("ComParE_2016", "compare16/ComParE_2016.conf")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
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
    lens, d_pcm, _, _ = workload(torch)
    res = []
    for label, conf in CONFS:
        path = os.path.join(ref, conf)
        both = Session(path, options={"csvoutput": "f.csv", "lldcsvoutput": "l.csv"}, device=0)
        summ = Session(path, options={"csvoutput": "f.csv"}, device=0)
        lld = Session(path, options={"lldcsvoutput": "l.csv"}, device=0)
        rows, fo, lrows, lfo = both.extract_tensor(d_pcm, lens, sr, with_lld=True)      # warm-up of every session on this shape
        want, wfo = summ.extract_tensor(d_pcm, lens, sr)
        lwant, wlfo = lld.extract_tensor(d_pcm, lens, sr)
        torch.cuda.synchronize()
        same = lambda x, y: x.shape == y.shape and bool(torch.equal(x.view(torch.int32), y.view(torch.int32)))
        equal = same(rows, want) and same(lrows, lwant) and list(fo) == list(wfo) and list(lfo) == list(wlfo)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        stream = torch.cuda.current_stream()
        comb_ms, pair_ms = [], []
        for _ in range(a.reps):
            e0.record(stream)
            both.extract_tensor(d_pcm, lens, sr, with_lld=True)
            e1.record(stream)
            stream.synchronize()
            comb_ms.append(e0.elapsed_time(e1))
            e0.record(stream)
            summ.extract_tensor(d_pcm, lens, sr)
            lld.extract_tensor(d_pcm, lens, sr)
            e1.record(stream)
            stream.synchronize()
            pair_ms.append(e0.elapsed_time(e1))
        cm, pm = float(np.median(comb_ms)), float(np.median(pair_ms))
        r = dict(workload="%s -csvoutput -lldcsvoutput, %d x ~3 s int16 mono at 16 kHz" % (label, len(lens)), summary_values=int(rows.shape[1]),
                 lld_rows=int(lfo[-1]), lld_values=int(lrows.shape[1]), gpu=name, power_limit=plim, rows_equal=equal,
                 combined_ms_median=cm, two_calls_ms_median=pm, saving=1.0 - cm / pm,
                 combined_ms=[round(x, 3) for x in comb_ms], two_calls_ms=[round(x, 3) for x in pair_ms])
        for s in (both, summ, lld):
            s.close()
        print(json.dumps(r))
        res.append(r)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        json.dump(res, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
