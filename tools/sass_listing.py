#!/usr/bin/env python
"""Per-kernel SASS evidence for the shipped library.

  python tools/sass_listing.py [--out sass_listing.txt]

Runs `cuobjdump -sass` on gangealing_b200/libgg_b200.so (no GPU needed) and prints, for every kernel, the count of the
Hopper-specific / memory-path mnemonics that show wgmma / TMA / bulk-copy use:

  HGMMA (wgmma.mma_async), DMMA (fp64 mma.sync), UTMALDG (cp.async.bulk.tensor = TMA tensor map),
  UBLKCP (cp.async.bulk = 1-D bulk TMA), SYNCS (mbarrier), REDG (red.global), MATCH (match.any),
  LDG/STG.E.128 and LDS.128 (16-byte accesses), plus register count per kernel from `cuobjdump -res-usage`.
"""
import argparse
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MNEMONICS = ["HGMMA", "DMMA", "UTMALDG", "UBLKCP", "SYNCS", "REDG", "MATCH", "LDG.E.128", "STG.E.128",
             "LDS.128", "STS.128", "SHFL", "MUFU"]


def demangle(names):
    try:
        out = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True, check=True).stdout
        return out.strip().split("\n")
    except Exception:
        return names


def short(name):
    name = re.sub(r"\(anonymous namespace\)::", "", name)
    name = re.sub(r"^void ", "", name)
    name = re.sub(r"\(.*$", "", name)          # drop the parameter list
    return name


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=os.path.join(ROOT, "gangealing_b200", "libgg_b200.so"))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    sass = subprocess.run(["cuobjdump", "-sass", args.lib], capture_output=True, text=True, check=True).stdout
    res = subprocess.run(["cuobjdump", "-res-usage", args.lib], capture_output=True, text=True).stdout
    regs = {}
    cur = None
    for line in res.split("\n"):
        m = re.search(r"Function (\S+):", line)
        if m:
            cur = m.group(1)
        m = re.search(r"REG:(\d+).*?SHARED:(\d+)", line)
        if m and cur:
            regs[cur] = (int(m.group(1)), int(m.group(2)))
    counts = collections.OrderedDict()
    instr = {}
    arch = None
    cur = None
    for line in sass.split("\n"):
        m = re.search(r"arch = (sm_\w+)", line)
        if m:
            arch = m.group(1)
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            counts[cur] = collections.Counter()
            instr[cur] = 0
            continue
        if cur is None or "/*" not in line:
            continue
        body = line.split("/*")[1] if line.lstrip().startswith("/*") else line
        m = re.search(r"\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_.]+)", line)
        if not m:
            continue
        op = m.group(1)
        instr[cur] += 1
        for mn in MNEMONICS:
            if op.startswith(mn) or (("." in mn) and mn in op):
                counts[cur][mn] += 1
    names = list(counts)
    pretty = [short(n) for n in demangle(names)]
    lines = ["# SASS mnemonic counts per kernel: cuobjdump -sass %s  (arch %s, %d kernels)" % (
        os.path.relpath(args.lib, ROOT), arch, len(names)),
        "# columns: instructions, registers/thread, static smem bytes, then the count of each listed mnemonic (zeros omitted)", ""]
    total = collections.Counter()
    order = sorted(range(len(names)), key=lambda i: pretty[i])
    for i in order:
        n = names[i]
        c = counts[n]
        total.update(c)
        r = regs.get(n, (None, None))
        tags = "  ".join("%s=%d" % (k, c[k]) for k in MNEMONICS if c[k])
        lines.append("%-110s instr=%-6d regs=%-4s smem=%-6s %s" % (pretty[i][:110], instr[n], r[0], r[1], tags))
    lines += ["", "# totals over the library: " + "  ".join("%s=%d" % (k, total[k]) for k in MNEMONICS if total[k])]
    text = "\n".join(lines) + "\n"
    if args.out:
        with open(args.out, "w") as f:
            f.write(text)
        print("wrote %s (%d kernels)" % (args.out, len(names)))
    else:
        sys.stdout.write(text)


if __name__ == "__main__":
    main()
