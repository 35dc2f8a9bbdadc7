"""Consolidation of C4's cluster (10 000 nodes, 200 000 running pods, 166 750 candidate subsets) as it is and with one pod
on 1 000 nodes that has two zone alternatives (workloads.config_c4(vol_alts=1000), ten of them candidates).  The two
are timed alternately in one run: device ms (the library's CUDA events) and end-to-end ms of kp_consolidate, the decision
histogram, the k_consolidate plan line (KP_DEBUG: instantiation and staged tables), and equality with the oracle on 100
evenly spaced subsets.  Prints one JSON line, with the card's name, power limit and max SM clock.

    python tools/volume_consolidation_bench.py [--steps 10] [--warmup 3] [--no-oracle]
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


def plan_line(h, problem, ci):
    """the KP_DEBUG consolidate plan line of one kp_consolidate call (the library prints it on stderr)"""
    os.environ["KP_DEBUG"] = "1"
    with tempfile.TemporaryFile(mode="w+") as f:
        saved = os.dup(2)
        os.dup2(f.fileno(), 2)
        try:
            h.consolidate(problem, ci)
        finally:
            os.dup2(saved, 2)
            os.close(saved)
            del os.environ["KP_DEBUG"]
        f.seek(0)
        return sorted({l.strip() for l in f if "consolidate plan" in l})


def sample(consol, n=100):
    """the ConsolInput kwargs of `n` evenly spaced subsets"""
    S, off, nodes = consol["n_subsets"], consol["subset_off"], consol["subset_nodes"]
    pick = np.linspace(0, S - 1, n).astype(np.int64)
    sizes = (off[1:] - off[:-1])[pick]
    return pick, dict(consol, n_subsets=len(pick), subset_off=np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32),
                      subset_nodes=np.concatenate([nodes[off[i]:off[i + 1]] for i in pick]).astype(np.int32))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-oracle", action="store_true")
    args = ap.parse_args()
    import torch
    from karpenter_b200 import _abi, _native, workloads
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    torch.cuda.init()
    cases = {}
    for name, vol in (("c4", 0), ("c4_vol_alts", 1000)):
        enc, consol = workloads.config_c4(vol_alts=vol)
        cases[name] = dict(enc=enc, consol=consol, ci=_abi.ConsolInput(**consol), dev=[], e2e=[])
    h = _native.Handle()
    out = {"card": card}
    try:
        for c in cases.values():
            c["plan"] = plan_line(h, c["enc"].problem, c["ci"])
        for i in range(args.warmup + args.steps):
            for c in cases.values():  # alternating, so both see the same machine state
                t0 = time.perf_counter()
                res = h.consolidate(c["enc"].problem, c["ci"])
                if i >= args.warmup:
                    c["e2e"].append(1000 * (time.perf_counter() - t0))
                    c["dev"].append(res["solve_ms"])
                c["res"] = res
        for name, c in cases.items():
            pick, smp = sample(c["consol"])
            sub = h.consolidate(c["enc"].problem, _abi.ConsolInput(**smp))
            d = np.bincount(c["res"]["decision"], minlength=3)
            o = {"device_ms": round(float(np.mean(c["dev"])), 3), "device_ms_all": [round(float(x), 3) for x in c["dev"]],
                 "e2e_ms": round(float(np.mean(c["e2e"])), 3),
                 "decisions": {"noop": int(d[0]), "delete": int(d[1]), "replace": int(d[2])}, "plan": c["plan"]}
            o["sample_equals_full_run"] = all(np.array_equal(sub[k], c["res"][k][pick])
                                              for k in ("decision", "n_new_claims", "n_unscheduled", "replacement_its"))
            if not args.no_oracle:
                from tests import oracle_lib
                orc = oracle_lib.consolidate(c["enc"].problem, _abi.ConsolInput(**smp), threads=os.cpu_count() or 1)
                o["identical_to_oracle_on_100_subsets"] = all(np.array_equal(sub[k], orc[k]) for k in _abi.CONSOL_PARITY_KEYS)
            out[name] = o
    finally:
        h.close()
    out["device_ratio_vol_over_plain"] = round(out["c4_vol_alts"]["device_ms"] / out["c4"]["device_ms"], 3)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
