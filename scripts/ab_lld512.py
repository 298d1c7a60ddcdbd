"""A/B timing of the cfg-2 fused kernel across library variants (opensmile_b200/variants/lib_*.so, e.g. the parent commit's
library or builds with -D switches) and the default library: 1 M frames device-resident, CUDA events over 20 launches after
5 warm-ups, one subprocess per library (OSM_B200_LIB) and round.  The libraries alternate round by round, so that a drift
of the card's clock or of the neighbours' load over the run reaches every library alike.

    python scripts/ab_lld512.py [--rounds R]       # default 5 rounds

Prints every run (time, rate, checksum of the output rows) and per library the median, the range and the spread
(max - min over median) of the per-launch times."""
import argparse
import glob
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHILD = r'''
import os, sys
sys.path.insert(0, %r)
import numpy as np, torch
from opensmile_b200 import Plan, components_mfcc12_0_d_a
n_utt, L = 2000, 80240
plan = Plan(components_mfcc12_0_d_a(16000.0), "lld", 0)
g = torch.Generator(device="cuda").manual_seed(0)
pcm = (torch.randn(n_utt * L, device="cuda", generator=g) * 3000).clamp(-32768, 32767).to(torch.int16)
off = np.arange(n_utt + 1, dtype=np.int64) * L
out = plan.run_device(pcm, off)
for _ in range(5):
    plan.run_device(pcm, off, d_out=out)
torch.cuda.synchronize()
a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
a.record()
for _ in range(20):
    plan.run_device(pcm, off, d_out=out)
b.record()
torch.cuda.synchronize()
ms = a.elapsed_time(b) / 20
print("RESULT %%.4f %%.1f %%.6e" %% (ms, out.shape[0] / ms / 1e3, float(out.double().abs().sum())))
''' % ROOT


def main(argv):
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args(argv)
    libs = [("default", None)] + [(os.path.basename(p), p) for p in
                                  sorted(glob.glob(os.path.join(ROOT, "opensmile_b200", "variants", "lib_*.so")))]
    times = {name: [] for name, _ in libs}
    sums = {name: set() for name, _ in libs}
    for rnd in range(args.rounds):
        order = libs if rnd % 2 == 0 else libs[::-1]
        for name, path in order:
            env = dict(os.environ)
            if path:
                env["OSM_B200_LIB"] = path
            r = subprocess.run([sys.executable, "-c", CHILD], env=env, capture_output=True, text=True)
            line = [s for s in r.stdout.splitlines() if s.startswith("RESULT ")]
            if r.returncode != 0 or not line:
                raise SystemExit("%s failed:\n%s" % (name, r.stderr[-2000:]))
            ms, rate, chk = line[-1].split()[1:]
            times[name].append(float(ms))
            sums[name].add(chk)
            print("round %d  %-28s %s ms  %s M frames/s  checksum %s" % (rnd, name, ms, rate, chk), flush=True)
    print("\n%-28s %10s %10s %10s %8s  %s" % ("library", "median ms", "min", "max", "spread", "checksum"))
    for name, _ in libs:
        t = times[name]
        med = statistics.median(t)
        print("%-28s %10.4f %10.4f %10.4f %7.2f%%  %s" % (name, med, min(t), max(t), 100 * (max(t) - min(t)) / med,
                                                        " ".join(sorted(sums[name]))))


if __name__ == "__main__":
    main(sys.argv[1:])
