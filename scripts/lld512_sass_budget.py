"""Instruction budget of lld512_kernel at the bench geometry (hop 160, frame 400, F = 32, K = 13, 26 bands), without a GPU:

    python scripts/lld512_sass_budget.py [--src path/lld_fast.cu] [--lines PHASE] [-D...]   # other arguments go to nvcc

1. compiles opensmile_b200/csrc/lld_fast.cu (or --src, e.g. another checkout's) for sm_90a (-lineinfo) and disassembles
   it with inline line information; the instance is lld512_kernel<13, 13> (lld512_kernel<13> before the K = 13 emission);
2. gives every instruction of the kernel the lld_fast.cu line it was inlined into and keeps the per-tile loop, split into
   the phases the source's "// =====" headers and its phase-clock marks delimit (the same phases as
   scripts/lld512_phase_clocks.py); code under `if (tid == 0)` (prefetch, load_chunk) and the set-up before the loop are
   left out, and the barriers (BAR.SYNC) of each phase are listed;
3. counts each phase by class: FP32, shared memory, integer / address, control, other (global, constant, conversion);
4. static table: every instruction once.  Estimated table (the earlier issue budget): the bodies of the loops it finds
   (backward branches) times their trip counts, straight-line code once per warp with every branch, except the loops of
   the unfused store and of the utterance-edge emission, which count zero;
5. executed table: what a warp executes at the bench geometry, per frame.  Loops: the trips of each warp (exec_loops), the
   unroll factor read from the back edge (a signature instruction each trip executes once), remainder copies counted by
   the trips they take; nested loops multiply.  Branches (exec_branches): the warp-uniform ones are resolved from the
   bench layout and the plan, each with its reason printed -- aligned staging, pre-emphasis on, the unfused store off,
   interior / edge emission 14 / 2 of the 16 tiles of an utterance, warp 0's extra pass-2 work 1 of 8, the DCT's 7 of 8
   warps, IEEE division slow paths never taken; the edge emission and other out-of-line code count by the tiles that
   call them.  --lines PHASE lists a phase's executed instructions by source line.

All tables are warp-instructions per frame (a tile = 32 frames, 8 warps): an issue budget read from the SASS and the
source, not a measurement.  The mel trip counts come from mel-spaced band edges (0-8 kHz, 26 bands, 512-point FFT), the
others from the loop bounds in the source."""
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


def per_warp(n, step=NT, lane0=32):
    """trips of `for (i = tid; i < n; i += step)` for each warp (warp w starts at lane0 * w)"""
    return [max(0, math.ceil((n - lane0 * w) / step)) for w in range(NW)]


def exec_loops():
    """the executed path's loops: (file, `for` line text, trips of each warp per tile, signature op, signature ops per trip).
    The signature is an instruction every trip executes exactly once (or `per trip` times): the number of signatures inside a
    back edge gives the loop's unroll factor, those outside it the remainder copies.  None: the loop is not unrolled.
    Trips are per pass of the enclosing loop, except the mel groups: their count is the warp's total over its bands."""
    count = (F - 1) * HOP + FRAME
    _, groups = mel_trips()
    bands = (NB + NW) / NW
    return [
        ("lld_fast.cu", "for (int i = tid * 8; i < count", per_warp(count // 8, NT, 32), "LDS.128", 1),
        ("lld_fast.cu", "for (int t = warp; t < 16; t += NW)", [16 // NW] * NW, None, 1),
        ("lld_fast.cu", "for (int r = melBs; r <= melBe; r++)", [bands] * NW, None, 1),
        ("lld_fast.cu", "for (int q = (sVB[r + 1] - v0) >> 2", [groups] * NW, None, 1),
        ("lld_fast.cu", "for (int m = 0; m < p.nBands; m++, lp += F", [NB] * NW, "FFMA", 2),
        ("lld_fast.cu", "for (int i = tid; i < n; i += NT) o[i] = outS[i]", per_warp(F * 3 * K), "STG", 1),
        ("lld_fast.cu", "for (int i = tid; i < nv; i += NT) gv[i] = sv[i]", per_warp(F * 3 * K // 4), "STG", 1),
        ("lld_common.cuh", "for (int item = tid; item < K * DR; item += NT)", per_warp(K * (F + 4)), "FSETP.GT", 1),
        ("lld_common.cuh", "// statics -> outS", per_warp(K * F), "LDS", 1),
        ("lld_common.cuh", "// delta-delta rows", per_warp(K * F), "FSETP.GT", 1),
        # emit_edge (first / last tile of an utterance): coefficients by warp, rows by lane, the two regression windows
        ("lld_common.cuh", "for (int c = warp; c < K; c += NW) {\n    const float *rc", per_warp(K, NW, 1), None, 1),
        ("lld_common.cuh", "for (int tt = lane; tt < d1 - d0", [2] * NW, "FSETP.GT", 1),
        ("lld_common.cuh", "for (int i = 1; i <= W1", [2] * NW, "FMUL", 1),
        ("lld_common.cuh", "for (int rr = lane; rr < nr; rr += 32) outS", [1] * NW, "STS", 1),
        ("lld_common.cuh", "for (int c = warp; c < K; c += NW) {\n    const float *dc", per_warp(K, NW, 1), None, 1),
        ("lld_common.cuh", "for (int rr = lane; rr < nr; rr += 32) {\n      const int t = r0", [1] * NW, "FSETP.GT", 1),
        ("lld_common.cuh", "for (int i = 1; i <= W2", [2] * NW, "FMUL", 1),
    ]


EDGE_SHARE = 2 / 16    # emit_edge: the first and the last of the 16 tiles of a 500-frame utterance


def exec_branches(src):
    """warp-uniform branches of the tile loop, resolved at the bench geometry: (file, text of the line, 'block' = the
    { } block opened on that line / 'line' = that line, share of the warps x tiles that execute it, how it was resolved)"""
    return [
        ("lld_fast.cu", "} else {\n          const unsigned short *up", "block", 0.0,
         "staging: tg.mis == 0 (utterances of 80 240 samples from a 16-byte aligned buffer: every tile fetch is aligned)"),
        ("lld_fast.cu", "else w4 = load8_unaligned(rp + i);", "line", 0.0,
         "staging: mis == 0 (utterances of 80 240 samples from a 16-byte aligned buffer: every tile fetch is aligned)"),
        ("lld_fast.cu", "} else {\n#pragma unroll\n          for (int jj = 0; jj < 8; jj++) y[jj] = x[jj];", "block", 0.0,
         "staging: p.preemph = 1 (MFCC12_0_D_A pre-emphasis k = 0.97)"),
        ("lld_fast.cu", "if (t == 0 && p.preemph)", "line", 1 / 16, "pass 1: first-sample fix-up, butterfly t = 0 (1 of 16)"),
        ("lld_fast.cu", "if (warp == 0) {\n        // a = butterfly 0", "block", 1 / NW, "pass 2: warp 0's register reorder (1 warp of 8)"),
        ("lld_fast.cu", "if (warp == 0) {\n        // k = 0", "block", 1 / NW, "pass 2: warp 0's k = 0 / M bins (1 warp of 8)"),
        ("lld_fast.cu", "if (r > melBs) {", "block", 1 - NW / (NB + NW),
         "mel: band output, every range but the warp's first (4.25 ranges per warp)"),
        ("lld_fast.cu", "if (i < p.nStat) {", "block", 7 / NW, "DCT: warps with a coefficient (7 of 8 at K = 13)"),
        ("lld_fast.cu", "if (i + 1 < p.nStat)", "line", 6 / 7, "DCT: second coefficient (6 of the 7 warps)"),
        ("lld_fast.cu", "if (!p.fused) {", "block", 0.0, "store: p.fused = 1 (the unfused store is off the path)"),
        ("lld_fast.cu", "emit_interior", "line", 1 - EDGE_SHARE, "emit: interior tiles (14 of 16 per utterance)"),
        ("lld_fast.cu", "emit_edge<F, NW, KC, 2>(ring", "line", EDGE_SHARE, "emit: first / last tile of an utterance (2 of 16)"),
        # where the kernel has the compile-time edge emission, the generic one serves windows other than 2 / 2 only
        ("lld_fast.cu", "emit_edge<F, NW>(ring", "line", 0.0 if "emit_edge<F, NW, KC, 2>(ring" in src else EDGE_SHARE,
         "emit: first / last tile of an utterance (2 of 16), unless the K = 13 / windows 2 / 2 edge emission takes them"),
        ("lld_fast.cu", "if (tid < K * DR - NT) delta_item", "line", 7 / NW,
         "emit (K = 13): second delta item, tid < 13 x 36 - 256 (warps 0..6)"),
        ("lld_fast.cu", "if (warp + NW < K) outS", "line", 5 / NW, "emit (K = 13): second static column, warps 0..4"),
        ("lld_fast.cu", "if (warp + NW < K) delta2_item", "line", 5 / NW, "emit (K = 13): second delta-delta column, warps 0..4"),
        ("lld_fast.cu", "if (tid < head) o[tid]", "line", 1 / NW, "store: leading floats, tid < 3 (warp 0)"),
        ("lld_fast.cu", "if (tid < n - tail) o[tail + tid]", "line", 1 / NW, "store: trailing floats, tid < 3 (warp 0)"),
        ("lld_common.cuh", "return __fdiv_rn(x, d);", "line", 0.0,
         "div_exact: IEEE division only for |x| outside (1e-30, 1e30), never for the bench deltas"),
    ]


def block_end(lines, ln):
    """last line of the statement that starts on line ln (1-based): its { } block, or the line itself (a `}` that opens
    the line, as in `} else {`, closes the previous block)"""
    depth, opened = 0, False
    for j in range(ln, len(lines) + 1):
        t = re.sub(r"//.*", "", lines[j - 1])
        if j == ln:
            t = t.lstrip().lstrip("}")
        for ch in t:
            if ch == "{":
                depth, opened = depth + 1, True
            elif ch == "}":
                depth -= 1
                if opened and depth == 0:
                    return j
        if not opened and t.rstrip().endswith(";"):
            return j
    return ln


def find_line(lines, text):
    """1-based line where `text` (which may span lines: '\n') starts"""
    parts = text.split("\n")
    for i in range(len(lines) - len(parts) + 1):
        if all(parts[k].strip() in lines[i + k] for k in range(len(parts))):
            return i + 1
    return None


def executed_weights(insts, chains, funcs, labels, srcs):
    """addr -> (executed count per warp and tile, phase) on the bench geometry's path, and notes on how it was resolved"""
    files = {os.path.basename(k): v for k, v in srcs.items()}
    notes = []

    def region(fn, text, kind):
        lines = files.get(fn, [])
        ln = find_line(lines, text)
        if ln is None:
            return None
        return (fn, ln, ln if kind == "line" else block_end(lines, ln))

    def inside(a, rg):
        fn, lo, hi = rg
        return any(f == fn and lo <= ln <= hi for f, ln in chains.get(a, ()))

    # the phase an instruction executes in: the kernel's own code by its lld_fast.cu line, emit_edge in the emit phase;
    # the other out-of-line code (IEEE division and 64-bit integer division slow paths) is off the path
    phase = {}
    for a, op, ph, tgt, text in insts:
        fn = funcs.get(a, "")
        phase[a] = ph if fn == "" else ("emit" if "emit_edge" in fn else None)
    loops = []
    for fn, text, trips, sig, per in exec_loops():
        rg = region(fn, text, "block")
        if rg is None:
            notes.append("loop not in the source, skipped: " + text.split("\n")[0])
            continue
        loops.append((rg, text.split("\n")[0], sum(trips) / NW, sig, per, "for (int q = " in text))
    # innermost loop of every instruction (the smallest body that contains one of its chain's lines) and its parent
    owner = {}
    for a, *_ in insts:
        best = None
        for k, (rg, *_) in enumerate(loops):
            if inside(a, rg) and (best is None or rg[2] - rg[1] < loops[best][0][2] - loops[best][0][1]):
                best = k
        owner[a] = best
    parent = {}
    for k, (rg, *_) in enumerate(loops):
        cands = [j for j, (r2, *_) in enumerate(loops)
                 if j != k and r2[0] == rg[0] and r2[1] <= rg[1] and rg[2] <= r2[2] and (r2[1], r2[2]) != (rg[1], rg[2])]
        parent[k] = min(cands, key=lambda j: loops[j][0][2] - loops[j][0][1]) if cands else None
    def passes(k):          # passes of loop k's set-up: the trips of every enclosing loop
        j = parent[k]
        return 1.0 if j is None else loops[j][2] * passes(j)
    weight = {a: 1.0 for a, *_ in insts}
    for k, (rg, text, trips, sig, per, total) in enumerate(loops):
        mine = [(a, op) for a, op, ph, tgt, _ in insts if owner[a] == k and phase[a] is not None]
        if not mine:
            continue
        addrs = {a for a, _ in mine}
        edges = sorted((labels[t], a) for a, op, ph, t, _ in insts
                       if a in addrs and op.startswith("BRA") and t in labels and labels[t] < a)
        outer = passes(k)
        body = trips if total else outer * trips
        if not edges:
            for a, _ in mine:
                weight[a] = outer
            notes.append("%-48s no back edge: straight-line, x %.3g" % (text.strip()[:48], outer))
            continue
        nsig = lambda ops: sum(1 for op in ops if sig is not None and op.split(" ")[0] == sig or
                               (sig is not None and op.startswith(sig + ".") and sig != "LDS"))
        span = []
        for lo, hi in edges:
            ops = [op for a, op in mine if lo <= a <= hi]
            u = max(1, round(nsig(ops) / per)) if sig else 1
            span.append((u, lo, hi, len(ops)))
        u, lo, hi, nbody = min(span)                                   # the least unrolled back edge carries the trips
        c = nbody / u
        in_edge = lambda a: any(l <= a <= h for _, l, h, _ in span)
        out = [(a, op) for a, op in mine if not in_edge(a)]
        rem = (nsig([op for _, op in out]) / per) if sig else 0.0
        keep = max(0.0, len(out) - rem * c) / len(out) if out else 0.0
        for a, _ in mine:
            if lo <= a <= hi:
                weight[a] = body / u
            elif in_edge(a):
                weight[a] = 0.0                                        # a wider unroll the trips never reach
            else:
                weight[a] = outer * keep
        notes.append("%-48s %.3g trips x %.1f instructions (unrolled x%d, %d remainder copies), set-up x %.3g"
                     % (text.strip()[:48], body, c, u, round(rem), outer))
    rules = []
    for fn, text, kind, share, why in exec_branches("\n".join(files.get("lld_fast.cu", []))):
        rg = region(fn, text, kind)
        if rg is None:
            notes.append("branch not in the source, not applied: " + text.split("\n")[0])
            continue
        rules.append((rg, share))
        notes.append("%-48s x %.3g  %s" % (text.split("\n")[0].strip()[:48], share, why))
    # edge tiles run the K = 13 / windows 2 / 2 instance of emit_edge where the kernel has one, else the generic emit_edge
    special = "emit_edgeILi32ELi8ELi13ELi2E"
    has_special = any(special in fn for fn in funcs.values())
    out = {}
    for a, op, ph, tgt, _ in insts:
        w = weight[a]
        fn = funcs.get(a, "")
        if "emit_edge" in fn:
            w *= EDGE_SHARE if (special in fn) == has_special else 0.0
        for rg, share in rules:
            if inside(a, rg):
                w *= share
        out[a] = (w, phase[a])
    return out, notes


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


def main(argv):
    global SRC
    if "--src" in argv:             # another checkout's lld_fast.cu (e.g. the parent commit's, for a before / after)
        k = argv.index("--src")
        SRC = os.path.abspath(argv[k + 1])
        argv = argv[:k] + argv[k + 2:]
    lines_of = None
    if "--lines" in argv:
        k = argv.index("--lines")
        lines_of = argv[k + 1]
        argv = argv[:k] + argv[k + 2:]
    extra = argv
    sass = disassemble(extra)
    src = open(SRC).read()
    src_lines = src.splitlines()
    phase_of, t0 = phase_lines(src)
    # the K = 13 instance where the kernel has one (lld512_kernel<NZR, KC>), else lld512_kernel<13>
    name = re.search(r"^(_Z\S*lld512_kernelILi13E(?:Li13E)?EEvNS_9LldParamsE):$", sass, re.M).group(1)
    body = sass.split(name + ":\n", 1)[1].split("\n\t.section", 1)[0]
    srcs = {}
    insts = []            # (addr, op, phase, back-edge target label, innermost source text)
    chains = {}           # addr -> [(source file name, line)] of the inline chain, innermost first
    funcs = {}            # addr -> the out-of-line function the instruction lies in ("" = the kernel itself)
    labels, pending = {}, []
    line, inner, fresh, chain, func = 0, "", True, [], ""
    for s in body.splitlines():
        m = re.search(r'//## File "(.*?)", line (\d+)', s)
        if m:
            if fresh:             # the first line of an inline chain is the innermost one
                fn = m.group(1)
                if fn not in srcs:
                    srcs[fn] = open(fn).read().splitlines() if os.path.exists(fn) else []
                ln = int(m.group(2))
                inner = srcs[fn][ln - 1] if 0 < ln <= len(srcs[fn]) else ""
                chain = []
                fresh = False
            chain += [(os.path.basename(a), int(b)) for a, b in re.findall(r'File "(.*?)", line (\d+)', s)]
            m2 = re.search(r'//## File ".*lld_fast\.cu", line (\d+)$', s)
            if m2:
                line = int(m2.group(1))
            continue
        m = re.match(r"\$(\S+):$", s)
        if m:
            func = m.group(1)
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
        chains[addr] = list(dict.fromkeys(chain))
        funcs[addr] = func
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
    exe, exe_notes = executed_weights(insts, chains, funcs, labels, srcs)
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
    print("%s SASS budget (sm_90a%s), bench geometry hop %d, frame %d, F = %d, K = %d, %d bands"
          % ("lld512_kernel<13, 13>" if "Li13ELi13E" in name else "lld512_kernel<13>",
             (", " + " ".join(extra)) if extra else "", HOP, FRAME, F, K, NB))
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
    print("\nexecuted warp-instructions per frame (branches resolved at the bench geometry, loops by their executed trips,\n"
          "remainders of unrolled loops by the trips they take; 8 warps / 32 frames)")
    print("%-16s" % "phase" + "".join("%10s" % c for c in classes) + "%8s" % "total")
    ex = {ph: dict.fromkeys(classes, 0.0) for ph in PHASES}
    for addr, op, ph, _ in insts:
        w, eph = exe.get(addr, (0.0, None))
        if eph in ex:
            ex[eph][klass(op)] += w
    tot = dict.fromkeys(classes, 0.0)
    for ph in PHASES:
        row = {c: ex[ph][c] * NW / F for c in classes}
        for c in classes:
            tot[c] += row[c]
        print("%-16s" % ph + "".join("%10.1f" % row[c] for c in classes) + "%8.1f" % sum(row.values()))
    print("%-16s" % "all" + "".join("%10.1f" % tot[c] for c in classes) + "%8.1f" % sum(tot.values()))
    non_fft = sum(sum(ex[ph].values()) for ph in ("stage", "mel", "emit", "store")) * NW / F
    print("%-16s%58.1f" % ("stage+mel+emit+store", non_fft))
    for n in exe_notes:
        print("executed: " + n)
    if lines_of:
        # executed warp-instructions per frame of one phase by the innermost source line of each instruction
        per = {}
        for addr, op, ph, _ in insts:
            w, eph = exe.get(addr, (0.0, None))
            if eph == lines_of and w > 0:
                key = "%s:%d" % chains[addr][0] if chains.get(addr) else "?"
                per[key] = per.get(key, 0.0) + w * NW / F
        print("\n%s, executed warp-instructions per frame by source line:" % lines_of)
        for key, v in sorted(per.items(), key=lambda kv: -kv[1]):
            print("  %-24s %6.2f" % (key, v))
    print("\ntrip counts per warp and tile: " + "; ".join("%s %s" % (ph, "/".join("%.3g" % x for x in v)) for _, ph, v in trip_table()))
    for n in notes:
        print("note: " + n)


if __name__ == "__main__":
    main(sys.argv[1:])
