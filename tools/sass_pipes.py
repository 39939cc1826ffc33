"""Per-pipe SASS budget of a kernel's loop bodies, and the issue-cost estimate of one Poseidon permutation.

    python tools/sass_pipes.py <file.cubin|lib.so|file.sass|file.cu> [kernel-substring] [-D...]

A `.cu` file is compiled here for sm_90a (nvcc -cubin, extra -D switches passed through) so `ptxas -v`'s register and
spill report comes with it; a cubin / library is disassembled with cuobjdump. Runs on the CPU, no GPU needed.

Loop bodies are found from their back-edges (a branch to a lower address); nested loops are reported separately and an
outer body's counts exclude the inner ones. Each body is counted per pipe:
  wide   IMAD.WIDE(.U32)(.X)                        fma    other IMAD forms (IMAD, IMAD.X, IMAD.IADD, IMAD.SHL, IMAD.HI)
  mov    IMAD.MOV(.U32), MOV                        alu    IADD3(.X), LOP3, SHF, SEL, LEA(.HI), ISETP, PRMT, ...
  fp64   DFMA, DADD, DMUL, DSETP                    xu     I2F, F2I, MUFU
  ldc    LDC                                        mem    LDG / STG / LDS / STS; spill = STL / LDL (listed apart)
Cost model (tools/pipe_mix.cu, tools/pipe_mix2.cu on the H100; DESIGN.md §4): an IMAD.WIDE takes WIDE_CLK issue clocks
and overlaps with nothing, every other instruction takes one issue slot, and the ALU, FMA (moves included) and FP64 pipes
each accept one warp instruction every 2 clocks per SM sub-partition, the XU pipe one every XU_CLK. A body costs
    max(WIDE_CLK * wide + other, 2 * alu, 2 * (fma + mov), 2 * fp64, XU_CLK * xu)
clocks per warp. With the leaf-hash permutation's trip counts (8 full rounds, 11 partial-round pairs, one stretch after
the pairs) the per-permutation estimate is printed; it is a static figure, not a measurement."""
import collections
import os
import re
import subprocess
import sys
import tempfile

WIDE_CLK, XU_CLK = 5.0, 8.0
PIPES = ["wide", "fma", "mov", "alu", "fp64", "xu", "ldc", "mem", "spill", "ctrl"]


def pipe_of(op):
    base = op.split(".")[0]
    if base == "IMAD":
        if ".WIDE" in op:
            return "wide"
        if ".MOV" in op:
            return "mov"
        return "fma"
    if base == "MOV":
        return "mov"
    if base in ("DFMA", "DADD", "DMUL", "DSETP", "DMNMX"):
        return "fp64"
    if base in ("I2F", "F2I", "MUFU", "F2F", "I2FP", "F2IP"):
        return "xu"
    if base == "LDC":
        return "ldc"
    if base in ("STL", "LDL"):
        return "spill"
    if base in ("LDG", "STG", "LDS", "STS", "LD", "ST", "ATOM", "ATOMS", "RED", "LDSM"):
        return "mem"
    if base in ("BRA", "BAR", "EXIT", "RET", "CALL", "BSSY", "BSYNC", "WARPSYNC", "NOP", "YIELD", "BPT", "JMP"):
        return "ctrl"
    return "alu"


def clocks(c):
    other = sum(c[p] for p in PIPES if p not in ("wide", "ctrl")) + c["ctrl"]
    return max(WIDE_CLK * c["wide"] + other, 2 * c["alu"], 2 * (c["fma"] + c["mov"]), 2 * c["fp64"], XU_CLK * c["xu"])


def disassemble(path, defines):
    ptxas = ""
    if path.endswith(".sass"):
        return open(path).read(), ptxas
    if path.endswith(".cu"):
        tmp = tempfile.mkdtemp()
        cubin = os.path.join(tmp, "k.cubin")
        r = subprocess.run(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-cubin",
                            "-Xptxas", "-v", "-o", cubin, path] + defines, capture_output=True, text=True)
        if r.returncode:
            raise SystemExit(r.stderr[-3000:])
        ptxas, path = r.stderr, cubin
    sass = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True, check=True).stdout
    return sass, ptxas


def parse(sass):
    """kernel name -> list of (address, opcode, text)."""
    out, cur = collections.OrderedDict(), None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            out[cur] = []
            continue
        m = re.match(r"\s+/\*([0-9a-f]{4,})\*/\s+((?:@!?U?P[T\d]+\s+)?)([A-Z][A-Z0-9_.]*)([^;]*);", line)
        if m and cur:
            out[cur].append((int(m.group(1), 16), m.group(3), (m.group(2) + m.group(3) + m.group(4)).strip()))
    return out


def loops(ins):
    """[(start, end)] of every back-edge (branch target <= branch address), innermost first."""
    res = []
    for addr, op, text in ins:
        if op.startswith("BRA"):
            m = re.search(r"0x([0-9a-f]+)", text.split("BRA", 1)[1])
            if m and int(m.group(1), 16) <= addr:
                res.append((int(m.group(1), 16), addr))
    return sorted(set(res), key=lambda r: r[1] - r[0])


def body_counts(ins, lo, hi, inner):
    c = collections.Counter()
    ops = collections.Counter()
    for addr, op, _ in ins:
        if lo <= addr <= hi and not any(a <= addr <= b for a, b in inner):
            if op == "NOP":
                continue
            c[pipe_of(op)] += 1
            ops[op] += 1
    return c, ops


def ptxas_summary(ptxas, name):
    m = re.search(r"Compiling entry function '%s'.*?Used (\d+) registers" % re.escape(name), ptxas, re.S)
    s = re.search(r"Function properties for %s\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes "
                  r"spill loads" % re.escape(name), ptxas)
    if not m:
        return ""
    return "%s registers, %s B spill stores, %s B spill loads" % (m.group(1), s.group(2) if s else "?",
                                                                   s.group(3) if s else "?")


def report(name, ins, ptxas, verbose):
    print("== %s: %d instructions%s" % (name, len([i for i in ins if i[1] != "NOP"]),
                                        ("  (" + ptxas_summary(ptxas, name) + ")") if ptxas else ""))
    lps = loops(ins)
    bodies = []
    for k, (lo, hi) in enumerate(lps):
        inner = [l for l in lps[:k] if lo <= l[0] and l[1] <= hi and l != (lo, hi)]
        c, ops = body_counts(ins, lo, hi, inner)
        bodies.append(((lo, hi), c, ops))
    hdr = "   %-15s %5s " % ("body", "instr") + " ".join("%5s" % p for p in PIPES) + "  clocks"
    print(hdr)
    for (lo, hi), c, ops in sorted(bodies, key=lambda b: b[0][0]):
        print("   %04x-%04x%6s %5d " % (lo, hi, "", sum(c.values())) + " ".join("%5d" % c[p] for p in PIPES)
              + "  %6.0f" % clocks(c))
        if verbose:
            print("      " + ", ".join("%s %d" % kv for kv in ops.most_common(24)))
    return bodies


def permutation_estimate(ins, bodies):
    """The leaf-hash nest: the loop that contains another is the full-round loop (8 trips), the nested one the
    partial-round pair loop (11 trips). The forward branch in the full-round body that jumps over the pair loop (the
    r == 3 block) bounds the code around the pairs that runs once per permutation; it is split off the full round."""
    nested = [(b, o) for b in bodies for o in bodies if b is not o and o[0][0] <= b[0][0] and b[0][1] <= o[0][1]]
    if not nested:
        return None
    pair, full = nested[0]
    (flo, fhi), (plo, phi) = full[0], pair[0]
    once_rng = None
    for addr, op, text in ins:
        if op.startswith("BRA") and flo <= addr < plo:
            m = re.search(r"0x([0-9a-f]+)", text.split("BRA", 1)[1])
            if m and phi < int(m.group(1), 16) <= fhi:
                once_rng = (addr + 16, int(m.group(1), 16) - 16)
    once = collections.Counter()
    if once_rng:
        once, _ = body_counts(ins, once_rng[0], once_rng[1], [pair[0]])
        full = (full[0], full[1] - once, None)
    return full, pair, once, 8 * clocks(full[1]) + 11 * clocks(pair[1]) + clocks(once)


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("-")]
    defines = [a for a in sys.argv[1:] if a.startswith("-D")]
    verbose = "-v" in sys.argv[1:]
    if not args:
        raise SystemExit(__doc__)
    sass, ptxas = disassemble(args[0], defines)
    pat = args[1] if len(args) > 1 else ""
    for name, ins in parse(sass).items():
        if pat not in name:
            continue
        bodies = report(name, ins, ptxas, verbose)
        est = permutation_estimate(ins, bodies)
        if est:
            full, pair, once, total = est
            for label, c in (("full round (x8)", full[1]), ("partial-round pair (x11)", pair[1]), ("around the pairs (x1)", once)):
                print("   %-26s %5d instr " % (label, sum(c.values())) + " ".join("%5d" % c[p] for p in PIPES)
                      + "  %6.0f" % clocks(c))
            print("   estimate: %.1f k clocks per warp-permutation (cost model, not measured)" % (total / 1e3))
            sp = sum(b[1]["spill"] for b in (full, pair))
            mv = full[1]["mov"]
            print("   spills in the loop bodies: %d, moves in the full-round body: %d" % (sp, mv))


if __name__ == "__main__":
    main()
