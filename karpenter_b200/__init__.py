"""karpenter_b200: an H100-native solver for Karpenter's provisioning hot path (Scheduler.Solve + consolidation search).

Layout: `csrc/` CUDA kernels + the C ABI (libkarpsolve.so, include/karpsolve.h), `model.py` / `encode.py` /
`scheduler.py` the host-side mirror of the reference's Scheduler API, `kwok.py` / `workloads.py` the KWOK catalogs and
benchmark configurations.
"""
from . import model  # noqa: F401
