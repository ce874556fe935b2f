#!/usr/bin/env python
"""Static SASS counts of the narrow-band affine-gap rows (`sg_warp_ag_rows_banded4`) in one kernel of a built libsnapgpu.so, per
source-line range: the row loop outside the units, the unit body outside the lazy-F loop, and the lazy-F round.  No GPU.

    python tools/sass_loops.py [--lib snap_b200/csrc/libsnapgpu.so] [--kernel 'sg_align_kernelILi4ELi2E'] [--counts counts.json]

The library is built with -lineinfo (the Makefile's flags), so `nvdisasm --print-line-info-inline` puts every instruction on a line
of the source, through the inlining chain.  An instruction belongs to the innermost of the three loops whose lines hold it (a call
into an inlined helper counts where it is called from).  The loop ranges come from the source in this tree, found by brace matching
from the function's signature: the row loop is the first `for` of the body, the unit loop the first `for` inside it, the lazy-F
loop the first `for` inside that.  For each range it prints the instruction count, LDL / STL (local memory: spills or the stack),
generic LD / ST and global LDG / STG, and BSSY (convergence barriers).  When the kernel holds more than one copy of the function
(one per caller), each copy is printed.

--counts takes the JSON line of tools/narrow_band_counts.py (rows, units and lazy-F rounds of the second pass on bench.py's
headline workload) and adds the predicted instruction total of the function: units x unit + rounds x round + rows x row.
Static counts are not a GPU measurement.
"""
from __future__ import annotations

import argparse
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "snap_b200", "csrc", "sg_warp_ag.cuh")
FUNC = "sg_warp_ag_rows_banded4"
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")

ANNOT = re.compile(r'File "([^"]+)", line (\d+)')
INSN = re.compile(r"^\s*/\*[0-9a-f]+\*/\s+(@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)")


def _block_end(lines, start):
    """Index of the line closing the brace block opened at or after line `start`."""
    depth, opened = 0, False
    for k in range(start, len(lines)):
        code = lines[k].split("//")[0]
        for ch in code:
            if ch == "{":
                depth += 1
                opened = True
            elif ch == "}":
                depth -= 1
                if opened and depth == 0:
                    return k
    raise ValueError("unbalanced braces from line %d" % (start + 1))


def _first_for(lines, beg, end):
    for k in range(beg, end):
        if re.match(r"\s*for\s*\(", lines[k].split("//")[0]):
            return k
    raise ValueError("no for loop in lines %d..%d" % (beg + 1, end + 1))


def loop_ranges(path=SRC):
    """1-based inclusive line ranges {func, row, unit, lazy} of the function and its three nested loops."""
    lines = open(path).read().split("\n")
    sig = next(k for k, s in enumerate(lines) if re.search(r"\b%s\s*\(" % FUNC, s) and "void" in s)
    fend = _block_end(lines, sig)
    out = {"func": (sig + 1, fend + 1)}
    beg = sig + 1
    for name in ("row", "unit", "lazy"):
        k = _first_for(lines, beg, fend)
        e = _block_end(lines, k)
        out[name] = (k + 1, e + 1)
        beg, fend = k + 1, e
    return out


def disassemble(lib, kernel):
    """Lines of the SASS section of the one kernel whose mangled name contains `kernel`."""
    with tempfile.TemporaryDirectory() as d:
        subprocess.run([os.path.join(CUDA, "bin", "cuobjdump"), "-xelf", "all", os.path.abspath(lib)], cwd=d, check=True,
                       stdout=subprocess.DEVNULL)
        for cub in sorted(os.listdir(d)):
            txt = subprocess.run([os.path.join(CUDA, "bin", "nvdisasm"), "-c", "-gi", os.path.join(d, cub)], check=True,
                                 capture_output=True, text=True).stdout
            out, inside, names = [], False, set()
            for s in txt.split("\n"):
                if s.startswith("\t.section\t.text."):
                    name = s.split("\t.section\t.text.")[1].split(",")[0]
                    inside = kernel in name
                    if inside:
                        names.add(name)
                    continue
                if inside:
                    out.append(s)
            if len(names) > 1:
                raise SystemExit("--kernel %r matches %d kernels: %s" % (kernel, len(names), sorted(names)))
            if out:
                return out, names.pop()
    raise SystemExit("no kernel matching %r in %s" % (kernel, lib))


def classify(sass, ranges, src_name):
    """[(copy, category, opcode)] for the instructions of the function; category one of row / unit / lazy / call.

    The source lines find the loops; the loops' extents come from the code: a loop is the span from a backward branch's target to
    the branch.  The lazy-F loop is the smallest such span mostly made of lazy-F lines, the unit loop the smallest span around it, the
    row loop the smallest span around that.  So an instruction the compiler hoisted out of a loop counts where it runs."""
    f0, f1 = ranges["func"]

    def category(line):
        for name in ("lazy", "unit", "row"):
            a, b = ranges[name]
            if a <= line <= b:
                return name
        return "call"

    cur = None                 # the function's line the current annotation maps to, or None
    insns, labels, copy, gap = [], {}, -1, 10 ** 9      # insns: (index, copy or None, line category or None, opcode, branch target)
    for s in sass:
        if "//##" in s:
            cur = None
            for f, ln in ANNOT.findall(s):      # innermost first: the first frame in this file inside the function
                if os.path.basename(f) == src_name and f0 <= int(ln) <= f1:
                    cur = int(ln)
                    break
            continue
        lab = re.match(r"^(\.L_x_\d+):", s)
        if lab:
            labels[lab.group(1)] = len(insns)
            continue
        m = INSN.match(s)
        if not m:
            continue
        tgt = re.search(r"`\((\.L_x_\d+)\)", s) if m.group(2).startswith("BRA") else None
        if cur is None:
            gap += 1
            insns.append((len(insns), None, None, m.group(2), tgt and tgt.group(1)))
            continue
        if gap > 64:           # a new copy of the function (copies are far apart; one function's instructions are contiguous)
            copy += 1
        gap = 0
        insns.append((len(insns), copy, category(cur), m.group(2), tgt and tgt.group(1)))

    res = []
    for c in sorted({x[1] for x in insns if x[1] is not None}):
        idx = [x[0] for x in insns if x[1] == c]
        lo, hi = min(idx), max(idx)
        spans = sorted({(labels[x[4]], x[0]) for x in insns[lo:hi + 1] if x[4] in labels and lo <= labels[x[4]] <= x[0]},
                       key=lambda p: p[1] - p[0])

        def mostly(span, cat):
            cats = [x[2] for x in insns[span[0]:span[1] + 1] if x[2] is not None]
            return cats and sum(1 for k in cats if k == cat) * 2 > len(cats)

        lazy = next((p for p in spans if mostly(p, "lazy")), None)
        unit = next((p for p in spans if lazy and p[0] <= lazy[0] and p[1] >= lazy[1] and p != lazy), None)
        row = next((p for p in spans if unit and p[0] <= unit[0] and p[1] >= unit[1] and p != unit), None)
        if not (lazy and unit and row):
            raise SystemExit("copy %d: could not find the three nested loops in the code (spans %s)" % (c, spans[:8]))
        for x in insns[lo:hi + 1]:
            k = x[0]
            cat = ("lazy" if lazy[0] <= k <= lazy[1] else "unit" if unit[0] <= k <= unit[1] else
                   "row" if row[0] <= k <= row[1] else "call")
            res.append((c, cat, x[3]))
    return res


def tally(insns):
    t = {}
    for copy, cat, op in insns:
        d = t.setdefault(copy, {}).setdefault(cat, {"insns": 0, "LDL": 0, "STL": 0, "LD_generic": 0, "ST_generic": 0,
                                                    "LDG": 0, "STG": 0, "BSSY": 0})
        d["insns"] += 1
        base = op.split(".")[0]
        if base in ("LDL", "STL", "LDG", "STG", "BSSY"):
            d[base] += 1
        elif base == "LD":
            d["LD_generic"] += 1
        elif base == "ST":
            d["ST_generic"] += 1
    return t


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--lib", default=os.path.join(ROOT, "snap_b200", "csrc", "libsnapgpu.so"))
    ap.add_argument("--kernel", default="sg_align_kernelILi4ELi2E", help="substring of the mangled kernel name")
    ap.add_argument("--src", default=SRC, help="the sg_warp_ag.cuh the library was built from")
    ap.add_argument("--counts", help="JSON output of tools/narrow_band_counts.py")
    ap.add_argument("--json", action="store_true", help="print one JSON line instead of the table")
    args = ap.parse_args()

    ranges = loop_ranges(args.src)
    sass, name = disassemble(args.lib, args.kernel)
    t = tally(classify(sass, ranges, os.path.basename(args.src)))
    if not t:
        raise SystemExit("%s has no instructions on lines %d..%d of %s" % (name, *ranges["func"], args.src))
    counts = None
    if args.counts:
        with open(args.counts) as f:
            c = json.loads(f.read().strip().split("\n")[-1])
        counts = {"rows": int(c["narrow_rows"]), "units": int(c["rows"]["warp_steps"]), "rounds": int(c["rows"]["lazy_f_rounds"])}
        for copy in t.values():
            z = {"insns": 0}
            copy["predicted_insns"] = (counts["units"] * copy.get("unit", z)["insns"] + counts["rounds"] * copy.get("lazy", z)["insns"]
                                       + counts["rows"] * copy.get("row", z)["insns"])
    if args.json:
        print(json.dumps({"kernel": name, "lines": ranges, "copies": t, "counts": counts}))
        return
    print("%s: %s lines %d-%d (row loop %d-%d, unit %d-%d, lazy-F %d-%d)" % (name, FUNC, *ranges["func"], *ranges["row"], *ranges["unit"],
                                                                           *ranges["lazy"]))
    cols = ["insns", "LDL", "STL", "LD_generic", "ST_generic", "LDG", "STG", "BSSY"]
    labels = {"call": "per call, outside the rows", "row": "per row, outside the units", "unit": "per unit, outside lazy F",
              "lazy": "per lazy-F round"}
    for copy in sorted(t):
        print("copy %d" % copy)
        print("  %-28s" % "" + "".join("%11s" % c for c in cols))
        for cat in ("call", "row", "unit", "lazy"):
            if cat in t[copy]:
                print("  %-28s" % labels[cat] + "".join("%11d" % t[copy][cat][c] for c in cols))
        if counts:
            print("  predicted: %d units x %d + %d rounds x %d + %d rows x %d = %.3f G instructions" % (
                counts["units"], t[copy].get("unit", {"insns": 0})["insns"], counts["rounds"], t[copy].get("lazy", {"insns": 0})["insns"],
                counts["rows"], t[copy].get("row", {"insns": 0})["insns"], t[copy]["predicted_insns"] / 1e9))


if __name__ == "__main__":
    sys.exit(main())
