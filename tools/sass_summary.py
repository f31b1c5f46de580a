#!/usr/bin/env python
"""Opcode histogram per kernel from `cuobjdump -sass` (static instruction counts).

    python tools/sass_summary.py [path/to/lib.so | file.o] [--filter substring] [--top N]

Prints, per kernel: total SASS instructions, the share of FP32 (FFMA / FMUL / FADD), shuffles, shared- and global-memory
instructions, and the TMA / mbarrier / cp.async mnemonics that prove which hardware paths a kernel uses (UTMALDG = TMA load,
SYNCS = mbarrier, LDGSTS = cp.async, HGMMA = wgmma -- none expected here: the path has no dense contraction).
"""
import argparse
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def demangle(name):
    try:
        out = subprocess.run(["c++filt", name], capture_output=True, text=True, check=True).stdout.strip()
        return re.sub(r"\(anonymous namespace\)::", "", out).split("(")[0]
    except Exception:
        return name


def histogram(path):
    txt = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True, check=True).stdout
    kernels, cur = collections.OrderedDict(), None
    for line in txt.splitlines():
        mfun = re.search(r"Function : (\S+)", line)
        if mfun:
            cur = demangle(mfun.group(1))
            kernels[cur] = collections.Counter()
            continue
        mins = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+(?:\.[A-Z0-9_]+)*)", line)
        if mins and cur is not None:
            kernels[cur][mins.group(1)] += 1
    return kernels


GROUPS = [
    ("fp32", ("FFMA", "FMUL", "FADD")),
    ("mufu", ("MUFU",)),
    ("shfl", ("SHFL",)),
    ("lds/sts", ("LDS", "STS", "LDSM")),
    ("ldg/stg", ("LDG", "STG", "LD", "ST", "RED", "ATOM", "ATOMG")),
    ("ldc", ("LDC", "LDCU", "ULDC")),
    ("tma", ("UTMALDG", "UTMASTG", "UBLKCP", "UTMAPF")),
    ("mbarrier", ("SYNCS",)),
    ("cp.async", ("LDGSTS",)),
    ("bar", ("BAR",)),
    ("wgmma", ("HGMMA", "IGMMA", "QGMMA", "BGMMA")),
]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("path", nargs="?", default=os.path.join(ROOT, "mppi_isaac_b200", "libmppib.so"))
    ap.add_argument("--filter", default="")
    ap.add_argument("--top", type=int, default=12)
    args = ap.parse_args()
    ks = histogram(args.path)
    print(f"# cuobjdump -sass {os.path.relpath(args.path, ROOT)}: static SASS instruction counts per kernel")
    for name, c in ks.items():
        if args.filter and args.filter not in name:
            continue
        total = sum(c.values())
        by_base = collections.Counter()
        for op, n in c.items():
            by_base[op.split(".")[0]] += n
        parts = []
        for label, bases in GROUPS:
            n = sum(by_base[b] for b in bases)
            if n:
                parts.append(f"{label} {n}")
        print(f"\n{name}\n  total {total} | " + " | ".join(parts))
        full = ", ".join(f"{op} {n}" for op, n in sorted(c.items(), key=lambda kv: -kv[1])[: args.top])
        print(f"  top: {full}")
        flagged = {op: n for op, n in c.items() if op.split(".")[0] in ("UTMALDG", "UTMASTG", "SYNCS", "LDGSTS", "UBLKCP", "SHFL") or op.startswith("LDG.E.128") or op.startswith("UTC")}
        if flagged:
            print("  hw paths: " + ", ".join(f"{op} x{n}" for op, n in sorted(flagged.items())))


if __name__ == "__main__":
    sys.exit(main())
