"""C4 consolidation with the stock library (2 CTAs / SM) and with a -DCONSOL_MIN_CTAS=1 build: which occupancy wins.

    nvcc ... -DCONSOL_MIN_CTAS=1 -shared -o tools/libkarpsolve_occ1.so kp_api.cu kp_prep.cpp -lcudart   (in karpenter_b200/csrc)
    python tools/run_c4_occ.py; python tools/run_c4_occ.py tools/libkarpsolve_occ1.so"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from karpenter_b200 import _abi, _native, workloads
if len(sys.argv) > 1:
    _native.LIB_PATH = sys.argv[1]
enc, consol = workloads.config_c4()
h = _native.Handle()
for _ in range(4):
    res = h.consolidate(enc.problem, _abi.ConsolInput(**consol))
    print(sys.argv[1:] or "stock", res["solve_ms"])
h.close()
