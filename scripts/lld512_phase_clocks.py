"""Cycles per frame of each lld512_kernel phase at the bench shape (mfcc12: MFCC12_0_D_A, 2000 utterances x 500 frames,
16 kHz mono), read from the phase-clock variant library (lld_fast.cu: OSM_LLD_PHASE_CLOCKS).

    make -C opensmile_b200/csrc phase-clocks          # -> opensmile_b200/variants/lib_phase_clocks.so
    python scripts/lld512_phase_clocks.py [LIB ...]

Each library runs in its own process (OSM_B200_LIB).  The counts are CTA cycles: thread 0 of every CTA sums the cycles
between the phase boundaries of its tiles, and the sums of all CTAs are divided by the frames of the launch.  Two CTAs
share an SM, so an SM spends about half of the summed count per frame.  'kernel' is the CTAs' whole lifetime (the
phases plus the start-up and the tail); 'busiest CTA' is the longest single CTA, i.e. the kernel's critical path, in
cycles per launch.  The clock instrumentation itself costs a few instructions per phase, so compare variants with each
other, not with the default library's time."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PHASES = ("stage", "pass 1", "pass 2 + split", "mel", "DCT", "emit", "store")
CHILD = r'''
import ctypes, os, sys
sys.path.insert(0, %r)
import numpy as np, torch
from opensmile_b200 import Plan, capi, components_mfcc12_0_d_a
n_utt, L, steps = 2000, 400 + 160 * 499, 10
plan = Plan(components_mfcc12_0_d_a(16000.0), "lld", 0)
g = torch.Generator(device="cuda").manual_seed(0)
pcm = (torch.randn(n_utt * L, device="cuda", generator=g) * 3000).clamp(-32768, 32767).to(torch.int16)
off = np.arange(n_utt + 1, dtype=np.int64) * L
lib = capi.lib()
buf = (ctypes.c_ulonglong * 11)()
out = plan.run_device(pcm, off)
for _ in range(3):
    plan.run_device(pcm, off, d_out=out)
torch.cuda.synchronize()
assert lib.osm_b200_lld512_phase_clocks(buf) == 0
name = [str(x) for x in plan.last_lld_launch()]
per_launch_max = []
tot = np.zeros(11)
for _ in range(steps):
    plan.run_device(pcm, off, d_out=out)
    torch.cuda.synchronize()
    assert lib.osm_b200_lld512_phase_clocks(buf) == 0
    tot += np.array(list(buf), dtype=np.float64)
    per_launch_max.append(buf[8])
frames = out.shape[0] * steps
print("RESULT", repr({"kernel": name, "frames": frames, "sums": tot.tolist(), "busiest": per_launch_max}))
''' % ROOT


def main(argv):
    libs = argv or [os.path.join(ROOT, "opensmile_b200", "variants", "lib_phase_clocks.so")]
    rows = []
    for path in libs:
        env = dict(os.environ, OSM_B200_LIB=os.path.abspath(path))
        r = subprocess.run([sys.executable, "-c", CHILD], env=env, capture_output=True, text=True)
        line = [s for s in r.stdout.splitlines() if s.startswith("RESULT ")]
        if r.returncode != 0 or not line:
            raise SystemExit("%s failed:\n%s" % (path, r.stderr[-2000:]))
        res = eval(line[-1][7:])
        rows.append((os.path.basename(path), res))
    print("lld512_kernel phase clocks, CTA cycles per frame (%s)" % ", ".join("%s: %s" % (n, r["kernel"][0]) for n, r in rows))
    print("%-22s" % "phase" + "".join("%16s" % n[:15] for n, _ in rows))
    for k, ph in enumerate(PHASES + ("sum of phases", "kernel")):
        vals = []
        for _, r in rows:
            s, fr = r["sums"], r["frames"]
            v = sum(s[:7]) if ph == "sum of phases" else (s[7] if ph == "kernel" else s[k])
            vals.append(v / fr)
        print("%-22s" % ph + "".join("%16.1f" % v for v in vals))
    print("%-22s" % "tiles per launch" + "".join("%16.0f" % (r["sums"][9] / len(r["busiest"])) for _, r in rows))
    print("%-22s" % "busiest CTA (cycles)" + "".join("%16.0f" % (sum(r["busiest"]) / len(r["busiest"])) for _, r in rows))
    print("%-22s" % "mean CTA (cycles)" + "".join(
        "%16.0f" % (r["sums"][7] / len(r["busiest"]) / int(r["kernel"][1])) for _, r in rows))


if __name__ == "__main__":
    main(sys.argv[1:])
