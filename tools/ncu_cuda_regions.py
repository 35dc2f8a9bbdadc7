#!/usr/bin/env python3
"""Per-region instruction / stall-sample shares from `ncu --page source --csv --print-source sass,cuda`: regions are the
function bodies (and the stages of wsolve_run) found by text markers in the CURRENT sources, so run it against the
sources the profiled binary was built from.
usage: ncu_cuda_regions.py file.csv n_pods [srcdir]"""
import csv
import os
import sys
from collections import defaultdict

path, npods = sys.argv[1], float(sys.argv[2])
srcdir = sys.argv[3] if len(sys.argv) > 3 else os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "karpenter_b200", "csrc")
MARKS = {
    "kp_wsolve.cuh": [("ov_find", "int ov_find("), ("claim rows", "void claim_load("), ("scan", "struct ScanCtx {"),
                      ("migrate", "void migrate_small"), ("stager", "struct StageRing {"), ("head", "template <bool CONSOL"),
                      ("pop/stage", "// ---- Queue.Pop"), ("existing", "addToExistingNode (scheduler.go"),
                      ("sort stage", "sort.Slice(newNodeClaims"), ("inflight", "addToInflightNode (scheduler.go"),
                      ("new claim", "addToNewNodeClaim (scheduler.go"), ("requeue/tail", "scheduler.go:415-421: record the error")],
    "kp_kernels.cuh": [("fits_word", "uint64_t fits_word("), ("compat_off_word", "uint64_t compat_off_word("),
                       ("topo_domains", "Slot topo_domains("), ("eval_candidate", "struct Eval {"),
                       ("class regs", "struct ClassRegs {"), ("topo_record", "void topo_record("),
                       ("min_values", "bool min_values_ok("), ("k_feas", "k_feasibility(")],
}
marks = {}
for f, ms in MARKS.items():
    try:
        src = open(os.path.join(srcdir, f)).read().split("\n")
    except OSError:
        continue
    out = []
    for name, txt in ms:
        ln = next((i + 1 for i, l in enumerate(src) if txt in l), 10 ** 9)
        out.append((ln, name))
    marks[f] = sorted(out)


def region(f, ln):
    if f in marks:
        r = f[3:-4] + ": top"
        for l0, name in marks[f]:
            if ln >= l0:
                r = f[3] + ": " + name
        return r
    return f


rows = list(csv.reader(open(path, errors="replace")))
cur, hdr = "?", None
agg = defaultdict(lambda: [0, 0, defaultdict(int)])
for r in rows:
    if not r:
        continue
    if r[0] == "File Path":
        cur = r[1].split("/")[-1]
        continue
    if r[0] == "Line No":
        hdr = r
        si, ii = hdr.index("# Samples"), hdr.index("Instructions Executed")
        stall_cols = [i for i, h in enumerate(hdr) if h.startswith("stall_") and "Not Issued" not in h]
        continue
    if hdr is None or r[0] in ("", "Function Name"):
        continue
    try:
        ln = int(r[0])
    except ValueError:
        continue
    a = agg[region(cur, ln)]
    a[0] += int(r[si] or 0)
    a[1] += int(r[ii] or 0)
    for c in stall_cols:
        v = int(r[c] or 0)
        if v:
            a[2][hdr[c][6:]] += v
tot = sum(a[0] for a in agg.values()) or 1
toti = sum(a[1] for a in agg.values()) or 1
print(f"warp instructions / pod: {toti / npods:.0f}")
for k, a in sorted(agg.items(), key=lambda kv: -kv[1][0]):
    why = ",".join(f"{n}:{100 * v / max(a[0], 1):.0f}%" for n, v in sorted(a[2].items(), key=lambda kv: -kv[1])[:3])
    print(f"{100 * a[0] / tot:5.1f}% smp {100 * a[1] / toti:5.1f}% ins ({a[1] / npods:7.0f}/pod) {k:22s} {why}")
