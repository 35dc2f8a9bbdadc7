"""Per-phase cycle profile of the solver warp on C3 and on one C5 NodePool shard.

Needs the profiling build of the library (make -C karpenter_b200/csrc prof), loaded through KP_LIB_PATH:

    KP_LIB_PATH=karpenter_b200/csrc/libkarpsolve_prof.so python tools/phase_profile.py [--apps 1000] [--json OUT]

Each workload is uploaded once, solved once to warm up and once more for the profile.  Prints, per phase of wsolve_run
(see KP_PROF_LAP in kp_wsolve.cuh), the solver warp's SM cycles per pod, the phases' sum and the pod loop's total.
The clock64() reads themselves cost cycles, so compare profiles with each other, not with the default build's times.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PHASES = ["pop", "sort", "domain_mask", "scan", "fast_commit", "record", "full_eval", "new_claim", "other"]
# the in-flight scan's counters: steps (the first 32-wide step, each later step), positions from the scan start up to each
# result (what a position-by-position walk visits), cycles of the first steps (the rest of the scan phase: later steps)
SCAN = ["steps", "positions", "first_step_cycles"]


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
        return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"
    except OSError:
        return "unknown"


def profile(h, lib, problem, n_pods):
    h.upload(problem)
    h.solve_resident()  # warm-up
    res = h.solve_resident()
    st = h.stats()
    buf = np.zeros(len(PHASES) + 1 + len(SCAN), dtype=np.int64)
    n = lib.kp_phase_profile(h._h, -1, buf.ctypes.data_as(C.c_void_p), len(buf))
    if n != len(buf):
        raise RuntimeError("kp_phase_profile failed: is KP_LIB_PATH the profiling build (libkarpsolve_prof.so)?")
    per_pod = {p: float(buf[i]) / n_pods for i, p in enumerate(PHASES)}
    scan = {s: float(buf[len(PHASES) + 1 + i]) / n_pods for i, s in enumerate(SCAN)}
    scan["later_step_cycles"] = per_pod["scan"] - scan["first_step_cycles"]
    return {
        "pods": n_pods,
        "claims": int(res["n_claims"]),
        "solve_ms": st["solve_ms"],
        "cycles_per_pod": per_pod,
        "sum_cycles_per_pod": float(buf[:len(PHASES)].sum()) / n_pods,
        "total_cycles_per_pod": float(buf[len(PHASES)]) / n_pods,
        "scan_per_pod": scan,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--apps", type=int, default=1000, help="C3 apps of 1000 replicas (bench.py: 1000)")
    ap.add_argument("--c5-pods", type=int, default=10_000_000, help="C5 total pods; pool 0's shard is profiled")
    ap.add_argument("--json", default=None, help="also write the profiles here")
    args = ap.parse_args()
    from karpenter_b200 import _native, workloads
    lib = _native.lib()
    lib.kp_phase_profile.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32]
    lib.kp_phase_profile.restype = C.c_int
    print(f"library {_native.LIB_PATH}; GPU {gpu_info()}", flush=True)
    h = _native.Handle(0)
    out = {"gpu": gpu_info()}
    try:
        c3 = workloads.config_c3(n_apps=args.apps, replicas=1000, n_its=1000)
        out["c3"] = profile(h, lib, c3.problem, args.apps * 1000)
        del c3
        c5 = workloads.config_c5_shards(n_pods=args.c5_pods, n_pools=8, n_its=1000, app_replicas=1000, pool_groups=[[0]])[0]
        out["c5_shard0"] = profile(h, lib, c5.problem, int(c5.problem.n_pods))
    finally:
        h.close()
    for name in ("c3", "c5_shard0"):
        r = out[name]
        print(f"{name}: {r['pods']} pods, {r['claims']} claims, solve {r['solve_ms']:.1f} ms (profiling build)")
        for p in PHASES:
            c = r["cycles_per_pod"][p]
            print(f"  {p:12s} {c:9.1f} cycles/pod  {100 * c / r['total_cycles_per_pod']:5.1f} %")
        print(f"  {'sum':12s} {r['sum_cycles_per_pod']:9.1f}   total {r['total_cycles_per_pod']:.1f} cycles/pod")
        s = r["scan_per_pod"]
        print(f"  scan: {s['steps']:.2f} steps/pod, {s['positions']:.1f} positions/pod, first steps "
              f"{s['first_step_cycles']:.1f} cycles/pod, later steps {s['later_step_cycles']:.1f} cycles/pod")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
