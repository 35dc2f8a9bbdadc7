"""ctypes binding of libkarpsolve.so (the CUDA product path). There is no CPU fallback: if the library is missing
or no CUDA device is usable every call raises."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from . import _abi

CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc")
LIB_PATH = os.environ.get("KP_LIB_PATH") or os.path.join(CSRC, "libkarpsolve.so")  # KP_LIB_PATH: experiment builds only
_LIB = None

STATUS = {0: "OK", 1: "DEADLINE", 2: "INVALID", 3: "CUDA", 4: "CAPACITY", 5: "UNSUPPORTED"}


class SolverError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"karpsolve: {STATUS.get(code, code)}: {msg}")
        self.code = code


def build(verbose=False):
    """Compile every CUDA source for sm_90a (nvcc cross-compiles without a GPU)."""
    out = subprocess.run(["make", "-C", CSRC], capture_output=True, text=True)
    if out.returncode != 0:
        raise RuntimeError("building libkarpsolve.so failed:\n" + out.stdout[-4000:] + out.stderr[-4000:])
    if verbose:
        print(out.stdout[-2000:])


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                               "(the product path has no CPU fallback)")
        L = C.CDLL(LIB_PATH)
        L.kp_create.argtypes = [C.c_int, C.POINTER(C.c_void_p)]
        L.kp_destroy.argtypes = [C.c_void_p]
        L.kp_last_error.argtypes = [C.c_void_p]
        L.kp_last_error.restype = C.c_char_p
        L.kp_solve.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
        L.kp_upload.argtypes = [C.c_void_p, C.c_void_p]
        L.kp_solve_resident.argtypes = [C.c_void_p, C.c_int64, C.c_void_p]
        L.kp_result_free.argtypes = [C.c_void_p]
        L.kp_solve_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_void_p]
        L.kp_upload_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_int32]
        L.kp_solve_batch_resident.argtypes = [C.c_void_p, C.c_int64, C.c_void_p]
        L.kp_comm_unique_id.argtypes = [C.c_void_p]
        L.kp_comm_init.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32]
        L.kp_comm_counter_slots.argtypes = [C.c_void_p, C.c_int32]
        L.kp_comm_counter_slots.restype = C.c_int64
        L.kp_comm_set_counter_layout.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int32]
        L.kp_comm_global_counts.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
        L.kp_comm_last_allreduce_ms.argtypes = [C.c_void_p]
        L.kp_comm_last_allreduce_ms.restype = C.c_double
        L.kp_comm_destroy.argtypes = [C.c_void_p]
        L.kp_debug_slot_algebra.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p, C.c_int32, C.c_void_p]
        L.kp_go_sort_f64.argtypes = [C.c_void_p, C.c_int32, C.c_void_p]
        L.kp_go_sort_i64.argtypes = [C.c_void_p, C.c_int32, C.c_void_p]
        L.kp_consolidate.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
        L.kp_consol_result_free.argtypes = [C.c_void_p]
        L.kp_feasibility.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.kp_get_stats.argtypes = [C.c_void_p, C.c_void_p]
        _LIB = L
    return _LIB


SLOT_CASE = np.dtype([("mask_a", "<u8"), ("mask_b", "<u8"), ("gte_a", "<i8"), ("lte_a", "<i8"), ("gte_b", "<i8"), ("lte_b", "<i8"),
                      ("flags_a", "<u4"), ("flags_b", "<u4"), ("value", "<i4"), ("well_known", "<i4"), ("allow_undefined", "<i4"),
                      ("_pad", "<i4")])
SLOT_OUT = np.dtype([("mask", "<u8"), ("gte", "<i8"), ("lte", "<i8"), ("flags", "<u4"), ("op", "<i4"), ("has_intersection", "<i4"),
                     ("has_value", "<i4"), ("compatible", "<i4"), ("_pad", "<i4")])

EXPORTS = ["kp_version", "kp_create", "kp_destroy", "kp_last_error", "kp_solve", "kp_result_free", "kp_upload",
           "kp_solve_resident", "kp_consolidate", "kp_consol_result_free", "kp_feasibility", "kp_get_stats",
           "kp_solve_batch", "kp_upload_batch", "kp_solve_batch_resident", "kp_comm_unique_id", "kp_comm_init",
           "kp_comm_counter_slots", "kp_comm_set_counter_layout", "kp_comm_global_counts", "kp_comm_last_allreduce_ms",
           "kp_comm_destroy", "kp_go_sort_f64", "kp_go_sort_i64", "kp_debug_slot_algebra"]


def go_sort_order(keys) -> np.ndarray:
    """Order Go's sort.Slice(less = <) leaves `keys` in (indices into keys); host code of the library, no device needed."""
    k = np.ascontiguousarray(keys)
    perm = np.zeros(len(k), np.int32)
    if k.dtype.kind == "f":
        k = k.astype(np.float64)
        rc = lib().kp_go_sort_f64(k.ctypes.data_as(C.c_void_p), len(k), perm.ctypes.data_as(C.c_void_p))
    else:
        k = k.astype(np.int64)
        rc = lib().kp_go_sort_i64(k.ctypes.data_as(C.c_void_p), len(k), perm.ctypes.data_as(C.c_void_p))
    if rc != 0:
        raise SolverError(rc, "kp_go_sort failed")
    return perm


class Handle:
    """kp_handle: one CUDA stream + device arena. Single caller at a time (like one reference Scheduler)."""

    def __init__(self, device: int = -1):
        self._h = C.c_void_p()
        rc = lib().kp_create(device, C.byref(self._h))
        if rc != 0:
            raise SolverError(rc, "kp_create failed (no usable CUDA device; there is no CPU fallback)")

    def close(self):
        if self._h:
            lib().kp_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != 0:
            raise SolverError(rc, lib().kp_last_error(self._h).decode())

    def solve(self, problem: _abi.Problem, deadline_ms: int = 0) -> dict:
        """kp_solve.  On KP_DEADLINE the partial result is returned with out["deadline"] = True (the reference returns
        partial Results plus ctx.Err(), scheduler.go:411-414)."""
        r = _abi.kp_result()
        rc = lib().kp_solve(self._h, problem.ref(), deadline_ms, C.byref(r))
        if rc != 1:
            self._check(rc)
        out = _abi.result_to_dict(r, problem.n_resources)
        out["deadline"] = rc == 1
        lib().kp_result_free(C.byref(r))
        return out

    def upload(self, problem: _abi.Problem):
        self._n_resources = problem.n_resources
        self._batch_resources = None
        self._check(lib().kp_upload(self._h, problem.ref()))

    def solve_resident(self, deadline_ms: int = 0) -> dict:
        r = _abi.kp_result()
        self._check(lib().kp_solve_resident(self._h, deadline_ms, C.byref(r)))
        out = _abi.result_to_dict(r, self._n_resources)
        lib().kp_result_free(C.byref(r))
        return out

    @staticmethod
    def _problem_array(problems):
        arr = (C.c_void_p * len(problems))()
        for i, p in enumerate(problems):
            arr[i] = C.addressof(p.c)
        return arr

    def _batch_out(self, rc, results, n_resources):
        if rc != 1:
            self._check(rc)
        outs = []
        for r, nr in zip(results, n_resources):
            o = _abi.result_to_dict(r, nr)
            o["deadline"] = rc == 1
            lib().kp_result_free(C.byref(r))
            outs.append(o)
        return outs

    def solve_batch(self, problems, deadline_ms: int = 0) -> list:
        """kp_solve_batch: independent Scheduler instances (NodePool shards, candidate sets), one CTA each."""
        n = len(problems)
        results = (_abi.kp_result * max(n, 1))()
        rc = lib().kp_solve_batch(self._h, self._problem_array(problems), n, deadline_ms, results)
        return self._batch_out(rc, results[:n], [p.n_resources for p in problems])

    def upload_batch(self, problems):
        self._batch_resources = [p.n_resources for p in problems]
        self._check(lib().kp_upload_batch(self._h, self._problem_array(problems), len(problems)))

    def solve_batch_resident(self, deadline_ms: int = 0) -> list:
        n = len(self._batch_resources)
        results = (_abi.kp_result * max(n, 1))()
        rc = lib().kp_solve_batch_resident(self._h, deadline_ms, results)
        return self._batch_out(rc, results[:n], self._batch_resources)

    # ---- multi-GPU (NodePool shards): the global topology-domain counter table, reduced inside the library
    @staticmethod
    def comm_unique_id() -> bytes:
        buf = (C.c_uint8 * 128)()
        if lib().kp_comm_unique_id(buf) != 0:
            raise SolverError(3, "ncclGetUniqueId failed (NCCL not available)")
        return bytes(buf)

    def comm_init(self, unique_id: bytes, rank: int, world: int):
        buf = (C.c_uint8 * 128).from_buffer_copy(unique_id)
        self._check(lib().kp_comm_init(self._h, buf, rank, world))

    def counter_slots(self, instance: int = -1) -> int:
        n = lib().kp_comm_counter_slots(self._h, instance)
        if n < 0:
            raise SolverError(2, "no such uploaded instance")
        return int(n)

    def set_counter_layout(self, total_slots: int, offsets):
        """offsets: start slot of each kp_upload_batch instance (or of the kp_upload instance: one entry, batch=False)."""
        off = np.ascontiguousarray(offsets, np.int64)
        n = len(self._batch_resources) if getattr(self, "_batch_resources", None) is not None else 0
        if n and n != len(off):
            raise ValueError("one offset per uploaded batch instance")
        self._check(lib().kp_comm_set_counter_layout(self._h, int(total_slots), off.ctypes.data, n))
        self._gcnt = int(total_slots)

    def global_counts(self) -> np.ndarray:
        out = np.zeros(self._gcnt, np.int32)
        self._check(lib().kp_comm_global_counts(self._h, out.ctypes.data, self._gcnt))
        return out

    def last_allreduce_ms(self) -> float:
        return float(lib().kp_comm_last_allreduce_ms(self._h))

    def consolidate(self, problem: _abi.Problem, consol: _abi.ConsolInput, deadline_ms: int = 0) -> dict:
        r = _abi.kp_consol_result()
        rc = lib().kp_consolidate(self._h, problem.ref(), consol.ref(), deadline_ms, C.byref(r))
        if rc != 1:  # KP_DEADLINE: the subsets that finished are valid, the rest read KP_DECISION_UNKNOWN
            self._check(rc)
        out = _abi.consol_result_to_dict(r)
        out["deadline"] = rc == 1
        lib().kp_consol_result_free(C.byref(r))
        return out

    def feasibility(self, problem: _abi.Problem) -> np.ndarray:
        itw = (problem.n_its + 63) // 64
        out = np.zeros((problem.n_classes, problem.n_templates, itw), np.uint64)
        w = C.c_int32()
        self._check(lib().kp_feasibility(self._h, problem.ref(), out.ctypes.data, C.byref(w)))
        return out

    def slot_algebra(self, value_int, is_int: int, universe: int, cases: np.ndarray) -> np.ndarray:
        """kp_debug_slot_algebra: structured arrays in the layout of kp_slot_case / kp_slot_out."""
        vi = np.zeros(64, np.int64)
        vi[:len(value_int)] = value_int
        cases = np.ascontiguousarray(cases, SLOT_CASE)
        out = np.zeros(len(cases), SLOT_OUT)
        self._check(lib().kp_debug_slot_algebra(self._h, vi.ctypes.data, is_int, universe, cases.ctypes.data, len(cases),
                                                out.ctypes.data))
        return out

    def stats(self) -> dict:
        s = _abi.kp_stats()
        lib().kp_get_stats(self._h, C.byref(s))
        return {n: getattr(s, n) for n, _ in s._fields_}
