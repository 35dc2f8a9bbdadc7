"""Workloads whose pods name hosts, each next to the same workload without hostname requirements.  Prints one JSON line.

(a) Provisioning against a live cluster: config_existing at 2 000 nodes / 40 000 pods with 5 % of the pods selecting one
    of 500 nodes by hostname and 10 % keeping off three nodes (NotIn).  Device ms (resident solves, the library's CUDA
    events), end-to-end ms of kp_solve, host prep ms, the k_node_cand time (torch.profiler, a run of its own), the solver
    plan line (KP_DEBUG), and whether the result equals the oracle's.
(b) Consolidation: C4's cluster (10 000 nodes, 200 000 running pods, 166 750 candidate subsets) with one pod pinned to its
    own node on 1 000 nodes, ten of them candidates.  Device and end-to-end ms of kp_consolidate, the decision
    histogram, the k_consolidate plan line (KP_DEBUG: its staged tables against the 110 KB cut-off), and equality with
    the oracle on 100 evenly spaced subsets.

    python tools/hostname_bench.py [--steps 10] [--warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def plan_line(problem):
    """the KP_DEBUG solver plan line of one upload (the library prints it on stderr)"""
    from karpenter_b200 import _native
    os.environ["KP_DEBUG"] = "1"
    with tempfile.TemporaryFile(mode="w+") as f:
        saved = os.dup(2)
        os.dup2(f.fileno(), 2)
        try:
            h = _native.Handle()
            h.upload(problem)
            h.close()
        finally:
            os.dup2(saved, 2)
            os.close(saved)
            del os.environ["KP_DEBUG"]
        f.seek(0)
        return [l.strip() for l in f if "solver plan" in l]


def node_cand_ms(h, problem, torch):
    from torch.profiler import ProfilerActivity, profile
    h.upload(problem)
    h.solve_resident()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            h.solve_resident()
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.name.startswith("k_node_cand") or "k_node_cand" in e.name]
    return round(sum(e.device_time for e in ev) / 3 / 1000.0, 4) if ev else None


def measure(name, enc, args, torch, oracle):
    from karpenter_b200 import _native
    from tests.parity import assert_same
    h = _native.Handle()
    try:
        h.upload(enc.problem)
        dev = []
        for i in range(args.warmup + args.steps):
            torch.cuda.synchronize()
            h.solve_resident()
            if i >= args.warmup:
                dev.append(h.stats()["solve_ms"])
        e2e = []
        for i in range(4):
            t0 = time.perf_counter()
            res = h.solve(enc.problem)
            if i:
                e2e.append(1000 * (time.perf_counter() - t0))
        st = h.stats()
        kc = node_cand_ms(h, enc.problem, torch)
    finally:
        h.close()
    out = {"device_ms": round(float(np.mean(dev)), 3), "device_ms_all": [round(float(x), 3) for x in dev],
           "e2e_ms": round(float(np.mean(e2e)), 3), "prep_ms": round(st["prep_ms"], 3), "k_node_cand_ms": kc,
           "n_claims": int(res["n_claims"]), "unscheduled": int((res["pod_target"] == -1).sum()),
           "plan": plan_line(enc.problem)}
    if oracle:
        from tests import oracle_lib
        try:
            assert_same(res, oracle_lib.solve(enc.problem, threads=os.cpu_count() or 1), f"{name} ")
            out["identical_to_oracle"] = True
        except AssertionError as e:
            out["identical_to_oracle"] = False
            out["mismatch"] = str(e)[:300]
    return out


def consolidation(pin_own, args, oracle):
    from karpenter_b200 import _abi, _native, workloads
    from tests import oracle_lib
    enc, consol = workloads.config_c4(pin_own=pin_own)
    ci = _abi.ConsolInput(**consol)
    os.environ["KP_DEBUG"] = "1"
    with tempfile.TemporaryFile(mode="w+") as f:
        saved = os.dup(2)
        os.dup2(f.fileno(), 2)
        h = _native.Handle()
        try:
            dev, e2e = [], []
            for i in range(args.warmup + args.steps):
                t0 = time.perf_counter()
                res = h.consolidate(enc.problem, ci)
                if i >= args.warmup:
                    e2e.append(1000 * (time.perf_counter() - t0))
                    dev.append(res["solve_ms"])
            # the same subsets the oracle checks, through the library
            S, off, nodes = consol["n_subsets"], consol["subset_off"], consol["subset_nodes"]
            pick = np.linspace(0, S - 1, 100).astype(np.int64)
            sizes = (off[1:] - off[:-1])[pick]
            smp = _abi.ConsolInput(**dict(consol, n_subsets=len(pick),
                                          subset_off=np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32),
                                          subset_nodes=np.concatenate([nodes[off[i]:off[i + 1]] for i in pick]).astype(np.int32)))
            sub = h.consolidate(enc.problem, smp)
        finally:
            h.close()
            os.dup2(saved, 2)
            os.close(saved)
            del os.environ["KP_DEBUG"]
        f.seek(0)
        plan = sorted({l.strip() for l in f if "consolidate plan" in l})
    d = np.bincount(res["decision"], minlength=3)
    out = {"device_ms": round(float(np.mean(dev)), 3), "e2e_ms": round(float(np.mean(e2e)), 3),
           "decisions": {"noop": int(d[0]), "delete": int(d[1]), "replace": int(d[2])}, "plan": plan}
    if oracle:
        orc = oracle_lib.consolidate(enc.problem, smp, threads=os.cpu_count() or 1)
        out["identical_to_oracle_on_100_subsets"] = all(np.array_equal(sub[k], orc[k]) for k in _abi.CONSOL_PARITY_KEYS)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-oracle", action="store_true")
    args = ap.parse_args()
    import torch
    from karpenter_b200 import workloads
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    torch.cuda.init()
    out = {"card": card}
    for name, kw in (("plain", {}), ("pinned", dict(pin_in=0.05, pin_not_in=0.10))):
        enc = workloads.config_existing(n_nodes=2000, n_pods=40_000, **kw)
        out[f"a_{name}"] = measure(name, enc, args, torch, not args.no_oracle)
    for name, pin in (("c4", 0), ("c4_pinned", 1000)):
        out[f"b_{name}"] = consolidation(pin, args, not args.no_oracle)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
