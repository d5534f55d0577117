"""``NumpyGPBatchEngine`` -- ``TPEEngine.gp_batch_set`` / ``gp_batch_loss`` / ``gp_batch_bounds`` answered on the
host (TEST INFRASTRUCTURE).

The batch kernels (tpe_gpbatch.cuh) compute, per GP, what the single-GP kernels compute; this engine restates them
by looping ``NumpyGPEngine`` (tests/_gp_engine.py) over the GPs of a call.  A failed factorisation is a per-job
status, the bounds are the three maxima with ``np.max``'s NaN propagation.
"""
from __future__ import annotations

import numpy as np

from optuna_b200.engine import GPCholeskyError
from tests._gp_engine import NumpyGPEngine


class NumpyGPBatchEngine(NumpyGPEngine):
    def gp_batch_set(self, offsets, X, y, is_categorical) -> None:
        off = np.asarray(offsets, dtype=np.int64)
        X, y = np.asarray(X, dtype=np.float64), np.asarray(y, dtype=np.float64)
        if off.size < 2:
            raise ValueError("no GPs in the batch")
        if np.any(np.diff(off) < 1) or off[0] != 0 or off[-1] != X.shape[0]:
            raise ValueError("a GP of the batch has no rows")
        self._gps = []
        for a, b in zip(off[:-1], off[1:]):
            e = NumpyGPEngine()
            e.gp_set_data(X[a:b], y[a:b], is_categorical)
            self._gps.append(e)

    def _gp(self, i):
        if not 0 <= i < len(self._gps):
            raise ValueError(f"GP index {i} out of range ({len(self._gps)} GPs)")
        return self._gps[i]

    def gp_batch_loss(self, gp_idx, raw, minimum_noise):
        raw = np.asarray(raw, dtype=np.float64)
        k = len(gp_idx)
        loss, grad, status = np.full(k, np.nan), np.full(raw.shape, np.nan), np.zeros(k, dtype=np.int32)
        for b, i in enumerate(gp_idx):
            try:
                loss[b], grad[b] = self._gp(int(i)).gp_loss(raw[b], minimum_noise)
            except GPCholeskyError:
                status[b] = 1
        return loss, grad, status

    def gp_batch_bounds(self, gp_idx, params, beta, samples):
        k = len(gp_idx)
        out, status = np.full((k, 3), np.nan), np.zeros(k, dtype=np.int32)
        for b, i in enumerate(gp_idx):
            e = self._gp(int(i))
            n = e._X.shape[0]
            try:
                ucb, lcb = e.gp_posterior(params[b], np.concatenate([e._X, samples[b]]), beta[b])
            except GPCholeskyError:
                status[b] = 1
                continue
            out[b] = [ucb[:n].max(), ucb[n:].max(), np.max(lcb[:n])]
        return out, status
