"""``NumpyParetoEngine`` -- ``TPEEngine.pareto_front`` answered on the host (TEST INFRASTRUCTURE).

The steps of tpe_pareto.cuh restated in NumPy: a stable order by coordinate 0, chunks of ``chunk`` sorted rows whose
cuts move to the end of a tie run of coordinate 0 (compared with ==, so -0.0 ties with +0.0), and per chunk a test
of every row against the front found so far (from coordinate 1 on: those rows are strictly smaller in coordinate 0)
and against every row of the chunk, after which the rows nothing dominates join the front.  The chunk is small, so
that the cases' tie runs reach across the nominal cut points.  Plugged into ``optuna_b200.analysis``, it lets the
CPU suite check the algorithm and the Python glue against the live reference.
"""
from __future__ import annotations

import numpy as np

MAX_OBJECTIVES = 16   # kMoMaxM


class NumpyParetoEngine:
    chunk = 5

    def __init__(self, device: int = 0) -> None:
        pass

    def close(self) -> None:
        pass

    def pareto_front(self, values) -> np.ndarray:
        v = np.ascontiguousarray(values, dtype=np.float64)
        n, M = v.shape
        if not 1 <= M <= MAX_OBJECTIVES:
            raise ValueError(f"n_objectives must be in [1, {MAX_OBJECTIVES}]")
        if np.isnan(v).any():
            raise ValueError("objective values hold NaN")
        order = np.argsort(v[:, 0], kind="stable")
        s = v[order]
        on_front = np.zeros(n, dtype=bool)
        front = np.empty((0, M))
        c0 = 0
        while c0 < n:
            c1 = min(n, c0 + self.chunk)
            while c1 < n and s[c1, 0] == s[c1 - 1, 0]:
                c1 += 1
            rows = s[c0:c1]
            dom = (front[None, :, 1:] <= rows[:, None, 1:]).all(axis=2).any(axis=1)
            le = (rows[None, :, :] <= rows[:, None, :]).all(axis=2)
            lt = (rows[None, :, :] < rows[:, None, :]).any(axis=2)
            dom |= (le & lt).any(axis=1)
            front = np.concatenate([front, rows[~dom]])
            on_front[order[c0:c1][~dom]] = True
            c0 = c1
        return on_front
