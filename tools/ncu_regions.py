#!/usr/bin/env python3
"""Per-region instruction / stall-sample shares of k_wsolve from an ncu source-page CSV.
usage: ncu_regions.py prof_source.csv k.sass kp_wsolve.cuh(kernel version) kp_kernels.cuh n_pods"""
import csv
import sys
from collections import defaultdict

sys.path.insert(0, __file__.rsplit("/", 1)[0])
from ncu_lines import sass_lines

csvp, sassp, wsrc, ksrc, npods = sys.argv[1:6]
npods = float(npods)
rows = list(csv.reader(open(csvp)))
hdr = rows[1]
si, ii = hdr.index("# Samples"), hdr.index("Instructions Executed")
lines = sass_lines(sassp, "k_wsolve")
src = open(wsrc).read().split("\n")
ks = open(ksrc).read().split("\n")


def find(lines_, txt):
    for i, l in enumerate(lines_):
        if txt in l:
            return i + 1
    return 10 ** 9


marks = [("claim rows", find(src, "void claim_load(")), ("migrate", find(src, "void migrate_small")),
         ("stager", find(src, "void stager_run")), ("head", find(src, "template <bool CONSOL")),
         ("pop/stage", find(src, "// ---- Queue.Pop")), ("existing", find(src, "addToExistingNode (scheduler.go")),
         ("sort stage", find(src, "sort.Slice(newNodeClaims")), ("inflight scan", find(src, "addToInflightNode (scheduler.go")),
         ("inflight eval+commit", find(src, "const int cpos = base + l;")), ("new claim", find(src, "addToNewNodeClaim (scheduler.go")),
         ("requeue/tail", find(src, "scheduler.go:415-421: record the error"))]
kmarks = [("fits_word", find(ks, "uint64_t fits_word(")), ("compat_off_word", find(ks, "uint64_t compat_off_word(")),
          ("topo_domains", find(ks, "Slot topo_domains(")), ("eval_candidate", find(ks, "struct Eval {")),
          ("class regs", find(ks, "struct ClassRegs {")), ("topo_record", find(ks, "void topo_record(")),
          ("k_feas", find(ks, "k_feasibility("))]


def region(f, l):
    if f == "kp_gosort.cuh":
        return "gosort"
    if f == "kp_slot.hpp":
        return "slot algebra"
    if f == "kp_kernels.cuh":
        r = "k: head"
        for name, ln in kmarks:
            if l >= ln:
                r = "k: " + name
        return r
    if f == "kp_wsolve.cuh":
        r = "w: top"
        for name, ln in marks:
            if l >= ln:
                r = "w: " + name
        return r
    return f


agg = defaultdict(lambda: [0, 0])
for r, (f, l) in zip(rows[2:], lines):
    a = agg[region(f, l)]
    a[0] += int(r[si] or 0)
    a[1] += int(r[ii] or 0)
tot = sum(a[0] for a in agg.values()) or 1
toti = sum(a[1] for a in agg.values()) or 1
print(f"warp instructions / pod: {toti / npods:.0f}")
for k, a in sorted(agg.items(), key=lambda kv: -kv[1][0]):
    print(f"{100 * a[0] / tot:5.1f}% smp {100 * a[1] / toti:5.1f}% ins ({a[1] / npods:6.0f}/pod) {k}")
