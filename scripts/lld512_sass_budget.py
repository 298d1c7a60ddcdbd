"""Static instruction budget of lld512_kernel<13> at the bench geometry (hop 160, frame 400, F = 32, K = 13, 26 bands),
without a GPU:

    python scripts/lld512_sass_budget.py [-D...]      # extra arguments go to nvcc

1. compiles opensmile_b200/csrc/lld_fast.cu for sm_90a (-lineinfo) and disassembles it with inline line information;
2. gives every instruction of the kernel the lld_fast.cu line it was inlined into and keeps the per-tile loop, split into
   the phases the source's "// =====" headers and its phase-clock marks delimit (the same phases as
   scripts/lld512_phase_clocks.py); code under `if (tid == 0)` (prefetch, load_chunk) and the set-up before the loop are
   left out, and the barriers (BAR.SYNC) of each phase are listed;
3. counts each phase by class: FP32, shared memory, integer / address, control, other (global, constant, conversion);
4. multiplies the bodies of the loops it finds (backward branches) by their trip counts at the bench geometry, averaged
   over the 8 warps of a tile, and prints warp-instructions per frame (a tile = 32 frames).

Straight-line code counts once per warp, branches included (warp 0's extra work in pass 2, the DCT warp left idle),\nexcept the loops of the unfused store and of the utterance-edge emission, which count zero:
the figures are an issue budget, not a measurement.  The mel trip counts come from mel-spaced band edges (0-8 kHz,
26 bands, 512-point FFT), the others from the loop bounds in the source."""
import math
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "opensmile_b200", "csrc", "lld_fast.cu")
HOP, FRAME, F, K, NB, NT, NW = 160, 400, 32, 13, 26, 256, 8
PHASES = ("stage", "pass 1", "pass 2 + split", "mel", "DCT", "emit", "store")

FP32 = {"FFMA", "FADD", "FMUL", "MUFU", "FSEL", "FSETP", "FMNMX", "FCHK", "FSWZADD"}
SHARED = {"LDS", "STS", "LDSM", "ATOMS"}
CONTROL = {"BRA", "BAR", "EXIT", "SYNCS", "WARPSYNC", "BSSY", "BSYNC", "CALL", "RET", "NOP", "YIELD", "BREAK", "JMP"}
OTHER = {"LDG", "STG", "LDC", "ULDC", "LDL", "STL", "I2F", "F2I", "F2F", "I2FP", "F2IP", "S2R", "S2UR", "CS2R", "UBLKCP",
         "UTMALDG", "ATOMG", "RED", "MEMBAR", "ERRBAR", "CCTL", "DEPBAR"}


def klass(op):
    base = op.split(".")[0]
    if base in FP32:
        return "fp32"
    if base in SHARED:
        return "shared"
    if base in CONTROL:
        return "control"
    if base in OTHER:
        return "other"
    return "int/addr"


def warp_trips(n, step, start_of_warp):
    """mean over the warps of the trips of `for (i = first(lane); i < n; i += step)`; start_of_warp(w) = warp w's lane 0"""
    return sum(max(0, math.ceil((n - start_of_warp(w)) / step)) for w in range(NW)) / NW


def mel_trips():
    """(band iterations, 4-bin groups) per warp of the mel loop: bins of each range between mel-spaced edges, padded to x4"""
    mel = lambda f: 1127.0 * math.log(1.0 + f / 700.0)
    imel = lambda m: 700.0 * (math.exp(m / 1127.0) - 1.0)
    edges = [imel(i * mel(8000.0) / (NB + 1)) for i in range(NB + 2)]
    binhz = 16000.0 / 512
    groups = 0
    for r in range(NB + 1):
        lo, hi = math.ceil(edges[r] / binhz), math.ceil(edges[r + 1] / binhz)
        groups += (max(hi - lo, 0) + 3) // 4
    return (NB + NW) / NW, groups / NW


def trip_table():
    """source text of a loop's `for` line -> trips per warp and tile of each of its back edges, in address order (the DCT
    loop is unrolled by four: a main loop and a remainder)"""
    count = (F - 1) * HOP + FRAME
    dr = F + 4
    bands, groups = mel_trips()
    stage = [warp_trips(count, NT * 8, lambda w: 256 * w)]
    return [
        ("for (int i = tid * 8; i < count", "stage", stage),
        ("for (int base = warp * 256; base < count", "stage", stage),
        ("for (int t = warp; t < 16; t += NW)", "pass 1", [16 / NW]),
        ("for (int r = melBs; r <= melBe; r++)", "mel", [bands]),
        ("for (int q = (sVB[r + 1] - v0) >> 2", "mel", [groups]),
        # unrolled by four, the remainder straight-line; warps 0..6 own coefficients
        ("for (int m = 0; m < p.nBands; m++, lp += F", "DCT", [NB // 4 * 7 / NW]),
        ("for (int item = tid; item < K * DR; item += NT)", "emit", [warp_trips(K * dr, NT, lambda w: 32 * w)]),
        ("// statics -> outS", "emit", [warp_trips(K * F, NT, lambda w: 32 * w)]),
        ("// delta-delta rows", "emit", [warp_trips(K * F, NT, lambda w: 32 * w)]),
        ("for (int i = tid; i < n; i += NT) o[i] = outS[i]", "store", [warp_trips(F * 3 * K, NT, lambda w: 32 * w)]),
    ]


# loops off the bench path (the unfused store; emit_edge, which runs on an utterance's first and last tiles only): their
# bodies count zero, like the other branches the interior tiles do not take
COLD = ("for (int idx = tid; idx < tot", "for (int i = 1; i <= W1", "for (int tt = lane; tt < d1 - d0",
        "for (int rr = lane; rr < nr", "for (int c = warp; c < K; c += NW)", "for (int i = 1; i <= W2")


def phase_lines(src):
    """lld_fast.cu line -> phase, and the set of lines under `if (tid == 0) {`"""
    lines = src.splitlines()
    marks = []
    t0 = set()
    for i, s in enumerate(lines, 1):
        if "// ================= stage" in s: marks.append((i, "stage"))
        elif "// ================= FFT pass 1" in s: marks.append((i, "pass 1"))
        elif "// ================= FFT pass 2" in s: marks.append((i, "pass 2 + split"))
        elif "// ================= mel filterbank" in s: marks.append((i, "mel"))
        elif "// ================= DCT-II" in s: marks.append((i, "DCT"))
        elif "// ================= store" in s: marks.append((i, "emit"))
        elif "OSM_PHASE(kPhEmit)" in s: marks.append((i, "store"))
        elif "OSM_PHASE(kPhStore)" in s: marks.append((i + 1, None))
        if re.match(r"\s*if \(tid == 0\) \{", s):
            depth, j = 0, i
            while True:
                depth += lines[j - 1].count("{") - lines[j - 1].count("}")
                t0.add(j)
                if depth <= 0 and j > i - 1 and "}" in lines[j - 1]:
                    break
                j += 1

    def phase_of(line):
        ph = None
        for ln, name in marks:
            if line >= ln:
                ph = name
        return ph
    return phase_of, t0


def disassemble(extra):
    with tempfile.TemporaryDirectory() as td:
        cub = os.path.join(td, "lld_fast.cubin")
        subprocess.check_call(["nvcc", "-std=c++17", "-O3", "-lineinfo", "-gencode", "arch=compute_90a,code=sm_90a", "-cubin",
                               "-I" + os.path.dirname(SRC), *extra, "-o", cub, SRC])
        return subprocess.check_output(["nvdisasm", "-gi", "-c", cub], text=True)


def main(extra):
    sass = disassemble(extra)
    src = open(SRC).read()
    src_lines = src.splitlines()
    phase_of, t0 = phase_lines(src)
    body = sass.split("lld512_kernelILi13EEEvNS_9LldParamsE:\n", 1)[1].split("\n\t.section", 1)[0]
    srcs = {}
    insts = []            # (addr, op, phase, back-edge target label, innermost source text)
    labels, pending = {}, []
    line, inner, fresh = 0, "", True
    for s in body.splitlines():
        m = re.search(r'//## File "(.*?)", line (\d+)', s)
        if m:
            if fresh:             # the first line of an inline chain is the innermost one
                fn = m.group(1)
                if fn not in srcs:
                    srcs[fn] = open(fn).read().splitlines() if os.path.exists(fn) else []
                ln = int(m.group(2))
                inner = srcs[fn][ln - 1] if 0 < ln <= len(srcs[fn]) else ""
                fresh = False
            m2 = re.search(r'//## File ".*lld_fast\.cu", line (\d+)$', s)
            if m2:
                line = int(m2.group(1))
            continue
        m = re.match(r"(\.L_x_\d+):", s)
        if m:
            pending.append(m.group(1))
            continue
        m = re.match(r"\s*/\*([0-9a-f]+)\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)(.*);", s)
        if not m:
            continue
        fresh = True
        addr, op, rest = int(m.group(1), 16), m.group(2), m.group(3)
        for lb in pending:
            labels[lb] = addr
        pending = []
        ph = None if line in t0 else phase_of(line)
        mt = re.search(r"\((\.L_x_\d+)\)", rest) if op.startswith("BRA") else None
        insts.append((addr, op, ph, mt.group(1) if mt else None, inner))
    # loops: backward branches whose innermost line is a `for` of the table; each back edge takes the next trip count of
    # its line (address order).  Other backward branches (the mbarrier wait, out-of-line fix-ups) are not tile loops.
    edges = {}
    for addr, op, ph, tgt, text in insts:
        t = labels.get(tgt)
        if ph is not None and t is not None and t < addr and "for (" in text:
            edges.setdefault(text, []).append((t, addr, ph))
    mult = {}
    notes = []
    table = trip_table()
    for text, es in edges.items():
        row = [r for r in table if r[0] in text]
        if any(c in text for c in COLD):
            for lo, hi, ph in es:
                for a, _, p, _, _ in insts:
                    if lo <= a <= hi and p == ph:
                        mult.setdefault(a, 0.0)
            continue
        if not row:
            notes.append("unknown loop, body counted once: " + text.strip()[:70])
            continue
        _, ph, want = row[0]
        if len(es) != len(want) or any(e[2] != ph for e in es):
            notes.append("%s: %d back edges for %d trip counts, body counted once where unmatched: %s"
                         % (ph, len(es), len(want), text.strip()[:60]))
        for (lo, hi, _), n in zip(sorted(es), want):
            for a, _, p, _, _ in insts:
                if lo <= a <= hi and p == ph:
                    # nested loops (mel): the inner body's count replaces the outer's
                    mult[a] = max(n, mult.get(a, 0))
    insts = [(a, op, ph, t) for a, op, ph, t, _ in insts]
    classes = ("fp32", "shared", "int/addr", "control", "other")
    static = {ph: dict.fromkeys(classes, 0) for ph in PHASES}
    dyn = {ph: dict.fromkeys(classes, 0.0) for ph in PHASES}
    fpops = {ph: {} for ph in PHASES}
    bars = dict.fromkeys(PHASES, 0)
    for addr, op, ph, _ in insts:
        if ph not in static:
            continue
        c = klass(op)
        static[ph][c] += 1
        dyn[ph][c] += mult.get(addr, 1.0)
        if op.startswith("BAR.SYNC"):
            bars[ph] += 1
        base = op.split(".")[0]
        if base in ("FFMA", "FADD", "FMUL", "MUFU"):
            fpops[ph][base] = fpops[ph].get(base, 0) + 1
    print("lld512_kernel<13> SASS budget (sm_90a%s), bench geometry hop %d, frame %d, F = %d, K = %d, %d bands"
          % ((", " + " ".join(extra)) if extra else "", HOP, FRAME, F, K, NB))
    print("\nstatic instructions per phase (every-thread code of the tile loop)")
    print("%-16s" % "phase" + "".join("%10s" % c for c in classes) + "%8s%6s   FFMA/FADD/FMUL/MUFU" % ("total", "bars"))
    for ph in PHASES:
        fp = fpops[ph]
        print("%-16s" % ph + "".join("%10d" % static[ph][c] for c in classes) + "%8d%6d   %d/%d/%d/%d" % (
            sum(static[ph].values()), bars[ph], fp.get("FFMA", 0), fp.get("FADD", 0), fp.get("FMUL", 0), fp.get("MUFU", 0)))
    print("\nestimated warp-instructions per frame (loop bodies x trip counts, 8 warps / 32 frames)")
    print("%-16s" % "phase" + "".join("%10s" % c for c in classes) + "%8s" % "total")
    tot = dict.fromkeys(classes, 0.0)
    for ph in PHASES:
        row = {c: dyn[ph][c] * NW / F for c in classes}
        for c in classes:
            tot[c] += row[c]
        print("%-16s" % ph + "".join("%10.1f" % row[c] for c in classes) + "%8.1f" % sum(row.values()))
    print("%-16s" % "all" + "".join("%10.1f" % tot[c] for c in classes) + "%8.1f" % sum(tot.values()))
    print("\ntrip counts per warp and tile: " + "; ".join("%s %s" % (ph, "/".join("%.3g" % x for x in v)) for _, ph, v in trip_table()))
    for n in notes:
        print("note: " + n)


if __name__ == "__main__":
    main(sys.argv[1:])
