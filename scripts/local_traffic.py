#!/usr/bin/env python3
"""Local-memory traffic of the Viterbi kernels, per source region, from the SASS (no GPU).

Compiles kiwi_b200/csrc/viterbi.cu for sm_90a with the flags of csrc/Makefile (or takes objects that were built already), disassembles
them with line information (cuobjdump -xelf, nvdisasm -g) and counts, per function of viterbi.cu, the instructions and the LDL / STL
sites among them.  An instruction is charged to the function whose source lines contain its line; code inlined from a header is
charged to the viterbi.cu line that precedes it.  Functions inlined into another one (evaluate into findBestPath) keep their own row.
The ptxas report (registers, stack frame, spills) of each kernel comes along.

  python scripts/local_traffic.py [--builds knlm,cong,sbg] [--lines N] [--json OUT]
  python scripts/local_traffic.py --obj build/viterbi.o [--obj ...]"""
import argparse, json, os, re, subprocess, sys, tempfile
from collections import Counter

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "kiwi_b200", "csrc")
SRC = os.path.join(CSRC, "viterbi.cu")
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")
# build -> (Makefile variable with the build's flags, the defines csrc/Makefile adds in front of them)
BUILDS = {"knlm": ("KNLM_FLAGS", []), "cong": ("CONG_FLAGS", ["-DKB_CONG=1"]), "sbg": ("SBG_FLAGS", ["-DKB_SBG=1"])}
REGIONS = ["flushItems", "evaluate", "evalCand", "knProgressV", "findBestPath", "KB_VIT_KERNEL"]


def make_var(name):
    out = subprocess.run(["make", "-s", "--no-print-directory", "-C", CSRC, "--eval", "print-%: ; @echo $($*)", "print-" + name],
                         check=True, capture_output=True, text=True).stdout
    return out.split()


def compile_build(build, tmp):
    var, extra = BUILDS[build]
    obj = os.path.join(tmp, "viterbi_%s.o" % build)
    cmd = [os.path.join(CUDA, "bin", "nvcc")] + make_var("FLAGS") + ["-fmad=false"] + extra + make_var(var) + ["-Xptxas", "-v", "-c", SRC, "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode:
        sys.stderr.write(r.stdout + r.stderr)
        raise SystemExit("nvcc failed for the %s build" % build)
    return obj, ptxas_report(r.stderr + r.stdout)


def ptxas_report(log):
    """registers / stack frame / spills of the viterbi kernel from `-Xptxas -v`"""
    rep = {}
    lines = log.splitlines()
    for i, l in enumerate(lines):
        if "Function properties for" in l and "viterbi" in l and "kernel" in l and i + 2 < len(lines):
            m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", lines[i + 1])
            r = re.search(r"Used (\d+) registers", lines[i + 2])
            if m and r:
                rep = {"stack_frame": int(m.group(1)), "spill_stores": int(m.group(2)), "spill_loads": int(m.group(3)), "registers": int(r.group(1))}
    return rep


def function_ranges(path):
    """[first line, last line] of every function in REGIONS (1-based, by brace matching from its definition)"""
    src = open(path).read().split("\n")
    ranges = {}
    for name in REGIONS:
        pat = re.compile(r"__(device|global)__.*\b%s\s*\(" % name)
        start = next((i for i, l in enumerate(src) if pat.search(l)), None)
        if start is None:
            continue
        depth, seen = 0, False
        for j in range(start, len(src)):
            code = re.sub(r"//.*", "", src[j])
            code = re.sub(r"'(\\.|[^'\\])'", "''", code)
            depth += code.count("{") - code.count("}")
            seen = seen or "{" in code
            if seen and depth == 0:
                ranges[name] = (start + 1, j + 1)
                break
    return ranges


def region_of(line, ranges):
    best = None
    for name, (a, b) in ranges.items():
        if a <= line <= b and (best is None or b - a < ranges[best][1] - ranges[best][0]):
            best = name
    return best or "other"


def disassemble(obj, tmp):
    d = tempfile.mkdtemp(dir=tmp)
    subprocess.run([os.path.join(CUDA, "bin", "cuobjdump"), "-xelf", "all", os.path.abspath(obj)], cwd=d, check=True, capture_output=True)
    cubins = [f for f in os.listdir(d) if f.endswith(".cubin")]
    if len(cubins) != 1:
        raise SystemExit("%s: expected one sm_90a cubin, found %s" % (obj, cubins))
    return subprocess.run([os.path.join(CUDA, "bin", "nvdisasm"), "-g", "-c", os.path.join(d, cubins[0])],
                          check=True, capture_output=True, text=True).stdout


def count(sass, ranges):
    per = {}
    lines = Counter()
    cur = 0
    for l in sass.splitlines():
        m = re.match(r'\s*//## File "([^"]+)", line (\d+)', l)
        if m:
            if os.path.basename(m.group(1)) == "viterbi.cu":
                cur = int(m.group(2))
            continue
        m = re.match(r"\s*/\*[0-9a-f]+\*/\s+(@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)", l)
        if not m:
            continue
        op = m.group(2).split(".")[0]
        reg = region_of(cur, ranges)
        c = per.setdefault(reg, Counter())
        c["instr"] += 1
        if op in ("LDL", "STL"):
            c[op] += 1
            lines[(cur, op)] += 1
    return per, lines


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--builds", default="knlm,cong,sbg", help="comma-separated subset of " + ",".join(BUILDS))
    ap.add_argument("--obj", action="append", default=[], help="analyse this object instead of compiling (repeatable)")
    ap.add_argument("--src", default=SRC, help="the viterbi.cu the objects were compiled from (for the function ranges)")
    ap.add_argument("--lines", type=int, default=0, help="also list the N source lines with the most LDL + STL sites")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    ranges = function_ranges(a.src)
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        jobs = [(os.path.basename(o), o, {}) for o in a.obj] if a.obj else [(b,) + compile_build(b, tmp) for b in a.builds.split(",")]
        for name, obj, rep in jobs:
            per, lines = count(disassemble(obj, tmp), ranges)
            out[name] = {"ptxas": rep, "regions": {k: dict(v) for k, v in per.items()},
                         "top_lines": [[ln, op, n] for (ln, op), n in lines.most_common(a.lines)] if a.lines else []}
    for name, r in out.items():
        p = r["ptxas"]
        print("== %s" % name + ("  (%d registers, %d B stack frame, %d B spill stores, %d B spill loads)" %
                                (p["registers"], p["stack_frame"], p["spill_stores"], p["spill_loads"]) if p else ""))
        print("  %-14s %-13s %7s %5s %5s" % ("region", "lines", "instr", "LDL", "STL"))
        tot = Counter()
        for reg in REGIONS + ["other"]:
            c = r["regions"].get(reg)
            if not c:
                continue
            tot.update(c)
            span = "%d-%d" % ranges[reg] if reg in ranges else ""
            print("  %-14s %-13s %7d %5d %5d" % (reg.replace("KB_VIT_KERNEL", "kernel body"), span, c["instr"], c.get("LDL", 0), c.get("STL", 0)))
        print("  %-14s %-13s %7d %5d %5d" % ("total", "", tot["instr"], tot["LDL"], tot["STL"]))
        for ln, op, n in r["top_lines"]:
            print("    line %5d (%s): %d %s" % (ln, region_of(ln, ranges), n, op))
    if a.json:
        json.dump({"function_ranges": ranges, "builds": out}, open(a.json, "w"), indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
