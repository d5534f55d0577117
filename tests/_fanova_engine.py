"""``NumpyFanovaEngine`` -- ``TPEEngine.fanova_variances`` answered on the host (TEST INFRASTRUCTURE).

The steps of tpe_fanova.cuh restated in NumPy, tree by tree: boxes top-down (a child's box is its parent's with one
bound replaced), leaf weights as the product of the box widths, weighted means bottom-up, the subtree parameter
sets, the tree variance over the leaves, the sorted unique thresholds per feature with the two bounds as edges, and
per (tree, parameter) the terminals -- nodes whose parent's subtree splits on the parameter while their own does
not -- each adding (w / prod width, v w / prod width) to the grid cells its box covers: through the canonical ranges
of a segment tree for one column, cell by cell for several.  Only additions form a cell's sums.  Plugged into
``optuna_b200.importance``, it lets the CPU suite check the algorithm and the Python glue against the live
reference.
"""
from __future__ import annotations

import numpy as np

MAX_CELLS = 1 << 20   # kFaMaxCells


def _validate(off, left, right, feature, thr, bounds, po, cols):
    F = bounds.shape[0]
    if off[0] != 0 or np.any(np.diff(off) <= 0):
        raise ValueError("bad node offsets")
    if np.any(~(bounds[:, 0] <= bounds[:, 1])):
        raise ValueError("bad bounds")
    if po[0] != 0 or np.any(np.diff(po) <= 0):
        raise ValueError("a parameter has no raw features")
    if np.any((cols < 0) | (cols >= F)) or np.unique(cols).size != cols.size:
        raise ValueError("raw feature out of range or repeated")
    for t in range(off.size - 1):
        a, n = off[t], off[t + 1] - off[t]
        parents = np.zeros(n, dtype=np.int64)
        for i in range(n):
            f = feature[a + i]
            if f < 0:
                continue
            if f >= F:
                raise ValueError("feature out of range")
            th = thr[a + i]
            if np.isnan(th) or th < bounds[f, 0] or th > bounds[f, 1]:
                raise ValueError("threshold is NaN or outside its feature's bounds")
            for c in (left[a + i], right[a + i]):
                if c <= i or c >= n:
                    raise ValueError("child out of range")
                parents[c] += 1
        if np.any(parents[1:] != 1):
            raise ValueError("a node has no or two parents")


class NumpyFanovaEngine:
    def __init__(self, device: int = 0) -> None:
        pass

    def close(self) -> None:
        pass

    def fanova_variances(self, node_offsets, left, right, feature, threshold, value, bounds, param_offsets,
                         raw_features):
        off = np.asarray(node_offsets, dtype=np.int64)
        left, right, feature = (np.asarray(a, dtype=np.int64) for a in (left, right, feature))
        thr, value = np.asarray(threshold, dtype=np.float64), np.asarray(value, dtype=np.float64)
        bounds = np.asarray(bounds, dtype=np.float64)
        po, cols = np.asarray(param_offsets, dtype=np.int64), np.asarray(raw_features, dtype=np.int64)
        _validate(off, left, right, feature, thr, bounds, po, cols)
        T, n_params = off.size - 1, po.size - 1
        tree_var = np.empty(T)
        marg = np.empty((n_params, T))
        for t in range(T):
            sl = slice(off[t], off[t + 1])
            tree_var[t], marg[:, t] = _tree(left[sl], right[sl], feature[sl], thr[sl], value[sl], bounds,
                                            [cols[po[p]:po[p + 1]] for p in range(n_params)])
        return tree_var, marg


def _tree(left, right, feature, thr, value, bounds, params):
    n, F = feature.size, bounds.shape[0]
    parent = np.full(n, -1)
    box = np.empty((n, F, 2))
    box[0] = bounds
    for i in range(n):
        if feature[i] >= 0:
            f = feature[i]
            for c, side in ((left[i], 1), (right[i], 0)):
                parent[c] = i
                box[c] = box[i]
                box[c, f, side] = thr[i]
    param_of = np.full(F, -1)
    for p, c in enumerate(params):
        param_of[c] = p
    stat = np.empty((n, 2))
    has = np.zeros((n, len(params)), dtype=bool)
    for i in reversed(range(n)):
        if feature[i] < 0:
            w = box[i, 0, 1] - box[i, 0, 0]
            for f in range(1, F):
                w *= box[i, f, 1] - box[i, f, 0]
            stat[i] = value[i], w
        else:
            (vl, wl), (vr, wr) = stat[left[i]], stat[right[i]]
            stat[i] = (vl * wl + vr * wr) / (wl + wr), wl + wr
            has[i] = has[left[i]] | has[right[i]]
            if param_of[feature[i]] >= 0:
                has[i, param_of[feature[i]]] = True
    leaves = feature < 0
    v, w = stat[leaves, 0], stat[leaves, 1]
    mean = (v * w).sum() / w.sum()
    tvar = (w * (v - mean) ** 2).sum() / w.sum()
    # split midpoints and sizes per feature
    mids, sizes = [], []
    for f in range(F):
        e = np.concatenate([[bounds[f, 0]], np.unique(thr[feature == f]), [bounds[f, 1]]])
        mids.append(0.5 * (e[1:] + e[:-1]))
        sizes.append(e[1:] - e[:-1])
    out = np.empty(len(params))
    for p, A in enumerate(params):
        out[p] = _marginal(p, A, parent, has, stat, box, mids, sizes)
    return tvar, out


def _marginal(p, A, parent, has, stat, box, mids, sizes):
    Ks = [mids[c].size for c in A]
    cells = int(np.prod(Ks))
    if cells > MAX_CELLS:
        raise ValueError("more than 2^20 grid cells")
    if cells == 1:
        return 0.0
    P = 1 << (cells - 1).bit_length()
    acc = np.zeros((2 * P if len(A) == 1 else cells, 2))
    strides = [int(np.prod(Ks[j + 1:])) for j in range(len(A))]
    for i in range(parent.size):
        q = parent[i]
        if (q >= 0 and not has[q, p]) or has[i, p]:
            continue
        card = 1.0
        for c in A:
            card *= box[i, c, 1] - box[i, c, 0]
        W = stat[i, 1] / card
        V = stat[i, 0] * W
        # index range of the midpoints inside (lo, hi] per column; a column the tree never splits on is never tested
        ranges = []
        for j, c in enumerate(A):
            if Ks[j] == 1:
                ranges.append(range(1))
            else:
                ranges.append(range(np.searchsorted(mids[c], box[i, c, 0], side="right"),
                                    np.searchsorted(mids[c], box[i, c, 1], side="right")))
        if len(A) == 1:
            lo, hi = P + ranges[0].start, P + ranges[0].stop
            while lo < hi:
                if lo & 1:
                    acc[lo] += W, V
                    lo += 1
                if hi & 1:
                    hi -= 1
                    acc[hi] += W, V
                lo >>= 1
                hi >>= 1
        else:
            for idx in np.ndindex(*[len(r) for r in ranges]):
                acc[sum((r.start + k) * s for r, k, s in zip(ranges, idx, strides))] += W, V
    vals, wts = np.empty(cells), np.empty(cells)
    for cell in range(cells):
        if len(A) == 1:
            W = V = 0.0
            j = P + cell
            while j >= 1:
                W += acc[j, 0]
                V += acc[j, 1]
                j >>= 1
            size = sizes[A[0]][cell]
        else:
            W, V = acc[cell]
            size = 1.0
            for j, c in enumerate(A):
                size *= sizes[c][(cell // strides[j]) % Ks[j]]
        vals[cell], wts[cell] = V / W, W * size
    mean = (vals * wts).sum() / wts.sum()
    return (wts * (vals - mean) ** 2).sum() / wts.sum()
