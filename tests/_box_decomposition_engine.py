"""``NumpyBoxDecompositionEngine`` -- ``NumpyEHVIEngine`` (tests/_gp_sampler_ehvi_engine.py) with the engine call of
``GPSampler``'s device box decomposition: ``box_decomposition`` (tpe_box_decomposition) (TEST INFRASTRUCTURE).

It restates tpe_boxdec.cuh's algorithm, not optuna's code:
- the rows in unique-lexsorted order by stable sorts on the columns, last first, of keys that fold -0.0 onto +0.0;
  the rows that differ (!=) from their predecessor; their Pareto front;
- each pass keeps an append-only pool of bounds with a live flag and an active list in pool order.  A step scans the
  active list only: the dominated bounds die, those with u_0 <= z_0 retire (they stay live), the rest stay active.
  Each dominated bound appends its children in (pool index, j) order; all but the dimension-0 child join the active
  list after the kept bounds.  The result of a pass is the live bounds in pool order;
- the boxes of the final bounds with numpy's maximum rule ``a if a >= b else b``, the empty ones dropped.
"""
from __future__ import annotations

import numpy as np

from tests._gp_sampler_ehvi_engine import NumpyEHVIEngine

_BD_MAX_M = 24


def _lexsorted_unique_front(rows: np.ndarray) -> np.ndarray:
    n, M = rows.shape
    keys = np.where(rows == 0.0, 0.0, rows)
    order = np.arange(n)
    for j in range(M - 1, -1, -1):
        order = order[np.argsort(keys[order, j], kind="stable")]
    s = rows[order]
    keep = np.ones(len(s), dtype=bool)
    keep[1:] = np.any(s[1:] != s[:-1], axis=1)
    u = s[keep]
    # Pareto front: no other row <= everywhere and < somewhere (the rows are unique under ==)
    on_front = np.ones(len(u), dtype=bool)
    for i in range(len(u)):
        le = np.all(u <= u[i], axis=1)
        lt = np.any(u < u[i], axis=1)
        on_front[i] = not np.any(le & lt)
    return u[on_front]


def _pass(front: np.ndarray, ref: np.ndarray) -> tuple[np.ndarray, np.ndarray, int]:
    M = front.shape[1]
    ub = [ref.copy()]
    d0 = np.full((M, M), -np.inf)
    d0[np.arange(M), np.arange(M)] = ref
    dp = [d0]
    live = [True]
    active = [0]
    for z in front:
        kept, dom = [], []
        for a in active:
            if np.all(z < ub[a]):
                dom.append(a)
                live[a] = False
            elif ub[a][0] > z[0]:
                kept.append(a)
        born = []
        for a in dom:
            for j in range(M):
                if j > 0 and not z[j] >= max(dp[a][k, j] for k in range(M) if k != j):
                    continue
                u = ub[a].copy()
                u[j] = z[j]
                d = dp[a].copy()
                d[j] = z
                ub.append(u)
                dp.append(d)
                live.append(True)
                if j > 0:
                    born.append(len(ub) - 1)
        active = kept + born
    idx = np.flatnonzero(live)
    return np.asarray(ub)[idx], np.asarray(dp)[idx], len(ub) - 1


def _boxes(ub: np.ndarray, dp: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
    B, M = ub.shape
    lower = np.empty((B, M))
    upper = np.empty((B, M))
    lower[:, 0] = dp[:, 0, 0]
    upper[:, 0] = np.inf
    for r in range(B):
        for c in range(1, M):
            acc = dp[r, 0, c]
            for k in range(1, c):
                x = dp[r, k, c]
                acc = acc if acc >= x else x
            lower[r, c] = acc
    upper[:, 1:] = ub[:, 1:]
    keep = ~np.any(upper <= lower, axis=1)
    return -upper[keep], -lower[keep]


def box_decomposition(loss_vals: np.ndarray, ref_point: np.ndarray) -> tuple[tuple[np.ndarray, np.ndarray], dict]:
    front = _lexsorted_unique_front(loss_vals)
    ub1, _, born1 = _pass(front, ref_point)
    front2 = _lexsorted_unique_front(-ub1)
    ub2, dp2, born2 = _pass(front2, np.full(ref_point.size, np.inf))
    stats = {"front": len(front), "born1": born1, "bounds1": len(ub1), "front2": len(front2), "born2": born2,
             "bounds2": len(ub2)}
    return _boxes(ub2, dp2), stats


class NumpyBoxDecompositionEngine(NumpyEHVIEngine):
    def box_decomposition(self, loss_vals, ref_point):
        v = np.array(loss_vals, dtype=np.float64)
        r = np.array(ref_point, dtype=np.float64).reshape(-1)
        if v.ndim != 2 or v.shape[1] != r.size:
            raise ValueError(f"loss_vals must be [n, {r.size}] for a reference point of {r.size} objectives, got "
                             f"shape {v.shape}")
        n, M = v.shape
        if M < 2 or M > _BD_MAX_M:
            raise ValueError(f"box decomposition needs 2 <= M <= {_BD_MAX_M} objectives, got {M}")
        if n < 1:
            raise ValueError(f"box decomposition needs 1 <= n < 2^31 - 4096 rows, got {n}")
        if not np.all(np.isfinite(v)):
            raise ValueError("box decomposition: loss values must be finite")
        if np.isnan(r).any():
            raise ValueError("box decomposition: the reference point holds a NaN")
        (lower, upper), self.last_box_stats = box_decomposition(v, r)
        return lower, upper
