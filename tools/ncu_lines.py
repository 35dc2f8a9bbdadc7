#!/usr/bin/env python3
"""Attribute the warp-stall samples of an ncu report to CUDA source lines.

    ncu -i prof.ncu-rep --page source --csv > prof_sass.csv
    cuobjdump -xelf all libkarpsolve.so ; nvdisasm -g -c kp_api.sm_90a.cubin > k.sass
    python tools/ncu_lines.py prof_sass.csv k.sass k_solve [top]

ncu's CSV source page is per SASS instruction; nvdisasm -g interleaves `//## File "...", line N` markers with the same
instruction stream, so the two are joined by instruction order inside the kernel's .text section.
"""
import csv
import re
import sys
from collections import defaultdict


def sass_lines(path, kernel):
    out, cur, active = [], ("?", 0), False
    inl = None
    for ln in open(path, errors="replace"):
        if ln.startswith("//---") and ".text." in ln:
            active = kernel in ln
            continue
        if not active:
            continue
        m = re.search(r'//## File "([^"]+)", line (\d+)(.*)', ln)
        if m:
            cur = (m.group(1).split("/")[-1], int(m.group(2)))
            continue
        if re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+\S", ln):
            out.append(cur)
    return out


def main():
    csv_path, sass_path, kernel = sys.argv[1:4]
    top = int(sys.argv[4]) if len(sys.argv) > 4 else 40
    rows = list(csv.reader(open(csv_path)))
    hdr = rows[1]
    si, ii = hdr.index("# Samples"), hdr.index("Instructions Executed")
    stall_cols = [i for i, h in enumerate(hdr) if h.startswith("stall_") and "Not Issued" not in h]
    insts = rows[2:]
    lines = sass_lines(sass_path, kernel)
    if len(lines) != len(insts):
        print(f"warning: {len(insts)} profiled instructions vs {len(lines)} disassembled", file=sys.stderr)
    agg = defaultdict(lambda: [0, 0, defaultdict(int)])
    for r, loc in zip(insts, lines):
        a = agg[loc]
        a[0] += int(r[si] or 0)
        a[1] += int(r[ii] or 0)
        for c in stall_cols:
            v = int(r[c] or 0)
            if v:
                a[2][hdr[c][6:]] += v
    tot = sum(a[0] for a in agg.values()) or 1
    toti = sum(a[1] for a in agg.values()) or 1
    print(f"total samples {tot}, warp instructions {toti}")
    for loc, a in sorted(agg.items(), key=lambda kv: -kv[1][0])[:top]:
        why = ",".join(f"{k}:{v}" for k, v in sorted(a[2].items(), key=lambda kv: -kv[1])[:3])
        print(f"{100 * a[0] / tot:5.1f}% smp {100 * a[1] / toti:5.1f}% ins  {loc[0]}:{loc[1]:<5} {why}")


if __name__ == "__main__":
    main()
