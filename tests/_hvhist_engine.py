"""``ShimHVEngine`` -- ``TPEEngine.hypervolume_history`` answered on the host (TEST INFRASTRUCTURE).

The order-level steps of tpe_hvhist.cuh (eligibility, added trials, death, the scan) are restated here in NumPy; the
per-trial hypervolume HV(max(front_i, v_i)) comes from ``shim_hvhist_trial`` in tests/csrc/hvhist_shim.cu, the host
build of the same gather / clip / filter / order code and the same exact hypervolume the kernels run.  Plugged into
``optuna_b200.analysis``, it lets the CPU suite check the arithmetic and the Python glue against the live reference.
"""
from __future__ import annotations

import ctypes
import os

import numpy as np

LIB = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc", "libhvhist_shim.so")


def _p(a: np.ndarray):
    return a.ctypes.data_as(ctypes.c_void_p)


class ShimHVEngine:
    def __init__(self, device: int = 0) -> None:
        self._lib = ctypes.CDLL(LIB)
        fn = self._lib.shim_hvhist_trial
        fn.restype = ctypes.c_double
        fn.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                       ctypes.POINTER(ctypes.c_int)]

    def close(self) -> None:
        pass

    def hypervolume_history(self, values, feasible, ref) -> np.ndarray:
        v = np.ascontiguousarray(values, dtype=np.float64)
        r = np.ascontiguousarray(ref, dtype=np.float64).reshape(-1)
        n, M = v.shape
        if np.isnan(r).any() or np.isnan(v).any():
            raise ValueError("NaN in the values or the reference point")
        feas = np.ones(n, bool) if feasible is None else np.asarray(feasible, bool)
        elig = feas & ~(v > r).any(axis=1)
        added = np.zeros(n, bool)
        for i in range(n):
            if elig[i]:
                earlier = v[:i][elig[:i]]
                added[i] = not (earlier <= v[i]).all(axis=1).any()
        lst = np.flatnonzero(added).astype(np.int32)
        K = lst.size
        death = np.full(K, n, np.int32)
        for p in range(K):
            later = np.flatnonzero((v[lst[p + 1:]] <= v[lst[p]]).all(axis=1))
            if later.size:
                death[p] = lst[p + 1 + later[0]]
        out = np.zeros(n)
        h, kept = 0.0, ctypes.c_int()
        for p in range(K):
            pr = r[0] - v[lst[p], 0]
            for j in range(1, M):
                pr *= r[j] - v[lst[p], j]
            h += pr
            if p > 0:
                h -= self._lib.shim_hvhist_trial(_p(v), _p(lst), _p(death), p, M, _p(r), ctypes.byref(kept))
            out[lst[p]:] = h
        return out
