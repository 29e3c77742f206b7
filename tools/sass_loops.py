#!/usr/bin/env python3
"""Static SASS helper: per-function opcode histogram and the backward-branch loops with their opcode mix.
usage: sass_loops.py <file.sass | lib.so> <function-substring> [--loop N]
       sass_loops.py --regions <file.cubin | nvdisasm -gi listing> <function-substring> <source-file-substring> name=lo-hi[,lo-hi...] ...
                     [--within lo-hi]
The --regions form needs line info (-lineinfo): each instruction is charged to the first named region whose line range holds a line of
<source-file> in its inline chain (its own line and every call site it was inlined through); an instruction without line info inherits
the region of the one before it.  --within counts only instructions whose chain passes through that line range (e.g. the call sites
in one loop) and lists the rest as "outside".  Counts are static, split by issue pipe."""
import re, sys, subprocess, collections
def load(path):
    if path.endswith(".so") or path.endswith(".cubin"):
        return subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True).stdout
    return open(path).read()
def funcs(txt):
    out = {}; cur = None
    for ln in txt.splitlines():
        m = re.search(r"Function : (\S+)", ln)
        if m: cur = m.group(1); out[cur] = []; continue
        m = re.match(r"\s+/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;", ln)
        if m and cur is not None:
            ins = m.group(2); ins = re.sub(r"^@!?U?P\d+\s+", "", ins)
            out[cur].append((int(m.group(1), 16), ins))
    return out
def op(ins): return ins.split()[0]
def pipe(o):
    """Issue pipe of an opcode on sm_90 (the ones this project's kernels use): FMA takes every IMAD form (moves and shifts the compiler
    writes as IMAD included), MIO the shared / global / constant memory and warp-shuffle traffic, ALU the rest of the integer and logic ops."""
    b = o.split(".")[0]
    if b in ("IMAD", "IMUL", "FFMA", "FMUL", "FADD", "HFMA2"): return "FMA"
    if b in ("LDS", "STS", "LDG", "STG", "LDL", "STL", "LD", "ST", "LDC", "LDSM", "ATOMS", "ATOMG", "RED", "SHFL", "UBLKCP", "SYNCS"): return "MIO"
    if b in ("MUFU", "BREV", "FLO", "POPC", "I2F", "F2I", "I2FP", "F2IP"): return "XU"
    if b in ("BRA", "BSSY", "BSYNC", "EXIT", "RET", "CALL", "WARPSYNC", "ENDCOLLECTIVE", "BAR", "NOP", "YIELD", "VOTE", "VOTEU", "BMOV",
             "S2R", "S2UR", "CS2R", "ULDC", "UMOV", "UIADD3", "ULEA", "UISETP", "USHF", "ULOP3", "R2UR", "MATCH", "REDUX", "CREDUX", "WARPGROUP"):
        return "other"
    return "ALU"
def regions(argv):
    within = None
    if "--within" in argv:
        i = argv.index("--within"); within = tuple(int(v) for v in argv[i + 1].split("-")); argv = argv[:i] + argv[i + 2:]
    path, fsub, src = argv[0], argv[1], argv[2]
    spans = []
    for a in argv[3:]:
        name, rng = a.split("=")
        for r in rng.split(","):
            lo, hi = r.split("-"); spans.append((name, int(lo), int(hi)))
    txt = subprocess.run(["nvdisasm", "-gi", path], capture_output=True, text=True).stdout if path.endswith(".cubin") else open(path).read()
    count = collections.defaultdict(collections.Counter); cur = None; reg = None; chain = []
    for ln in txt.splitlines():
        if ln.startswith(".text."): cur = fsub in ln; reg = None; chain = []; continue
        if not cur: continue
        if ln.lstrip().startswith("//## File"):        # one line per inline frame, innermost first, the kernel's own line last
            chain += [int(n) for f, n in re.findall(r'"([^"]+)", line (\d+)', ln) if src in f]
            continue
        m = re.match(r"\s+/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;", ln)
        if not m: continue
        if chain:
            if within and not any(within[0] <= l <= within[1] for l in chain): reg = "outside"
            else: reg = next((nm for nm, lo, hi in spans if any(lo <= l <= hi for l in chain)), "rest")
            chain = []
        ins = re.sub(r"^@!?U?P\w+\s+", "", m.group(2))
        count[reg or "rest"][pipe(op(ins))] += 1
    cols = ("ALU", "FMA", "MIO", "XU", "other")
    print("%-14s %6s %6s %6s %6s %6s %7s" % (("region",) + cols + ("total",)))
    for name in [s[0] for s in spans if s[0] in count] + ["rest", "outside"]:
        if name not in count: continue
        c = count.pop(name)
        print("%-14s %6d %6d %6d %6d %6d %7d" % ((name,) + tuple(c[k] for k in cols) + (sum(c.values()),)))
def main():
    if sys.argv[1] == "--regions": return regions(sys.argv[2:])
    txt = load(sys.argv[1]); F = funcs(txt)
    for name, body in F.items():
        if sys.argv[2] not in name: continue
        print("==", name, len(body), "instructions")
        addr = {a: i for i, (a, _) in enumerate(body)}
        loops = []
        for i, (a, ins) in enumerate(body):
            m = re.search(r"\bBRA\S*\s+.*?(0x[0-9a-f]+)", ins)
            if m and int(m.group(1), 16) in addr and addr[int(m.group(1), 16)] <= i:
                loops.append((addr[int(m.group(1), 16)], i))
        for k, (s, e) in enumerate(loops):
            h = collections.Counter(op(x) for _, x in body[s:e + 1])
            print(" loop %d: [%x..%x] %d instr; top: %s" % (k, body[s][0], body[e][0], e - s + 1, ", ".join("%s %d" % kv for kv in h.most_common(14))))
        if "--loop" in sys.argv:
            k = int(sys.argv[sys.argv.index("--loop") + 1]); s, e = loops[k]
            for a, x in body[s:e + 1]: print("  %05x  %s" % (a, x))
if __name__ == "__main__": main()
