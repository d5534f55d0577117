"""``NumpyEMMRBatchEngine`` -- ``NumpyGPBatchEngine`` (tests/_gp_batch_engine.py) with the two batch calls the EMMR
improvement curve adds, answered on the host (TEST INFRASTRUCTURE):
- ``gp_batch_loss(..., deterministic=True)`` (tpe_gp_batch_loss_fixed_noise): ``NumpyEMMREngine``'s fixed-noise loss
  per job;
- ``gp_batch_moments`` (tpe_gp_batch_moments): ``NumpyEMMREngine.gp_posterior_moments`` per job at the job's own
  train rows.
A failed factorisation is a per-job status with NaN outputs, as on the device.  The single-GP calls are
``NumpyEMMREngine``'s, so the drop-in's per-prefix path runs on this engine too.
"""
from __future__ import annotations

import numpy as np

from optuna_b200.engine import GPCholeskyError
from tests._emmr_engine import NumpyEMMREngine
from tests._gp_batch_engine import NumpyGPBatchEngine


class NumpyEMMRBatchEngine(NumpyGPBatchEngine, NumpyEMMREngine):
    def gp_batch_set(self, offsets, X, y, is_categorical) -> None:
        super().gp_batch_set(offsets, X, y, is_categorical)
        gps = []
        for e in self._gps:
            g = NumpyEMMREngine()
            g.gp_set_data(e._X, e._y, e._cat)
            gps.append(g)
        self._gps = gps

    def gp_batch_loss(self, gp_idx, raw, minimum_noise, deterministic=False):
        if not deterministic:
            return super().gp_batch_loss(gp_idx, raw, minimum_noise)
        raw = np.asarray(raw, dtype=np.float64)
        k = len(gp_idx)
        loss, grad, status = np.full(k, np.nan), np.full(raw.shape, np.nan), np.zeros(k, dtype=np.int32)
        for b, i in enumerate(gp_idx):
            try:
                loss[b], grad[b] = self._gp(int(i)).gp_loss(raw[b], minimum_noise, deterministic=True)
            except GPCholeskyError:
                status[b] = 1
        return loss, grad, status

    def gp_batch_moments(self, gp_idx, params, rows, n_joint=0):
        rows = np.asarray(rows, dtype=np.int64)
        k, m = rows.shape
        if not 1 <= m <= 3:
            raise ValueError(f"batched GP moments take 1 .. 3 rows per job, got m = {m}")
        if n_joint != 0 and not 2 <= n_joint <= m:
            raise ValueError(f"bad joint covariance request (n_joint {n_joint}, m {m})")
        mean, var = np.full((k, m), np.nan), np.full((k, m), np.nan)
        cov = np.full((k, n_joint, n_joint), np.nan)
        status = np.zeros(k, dtype=np.int32)
        for b, i in enumerate(gp_idx):
            e = self._gp(int(i))
            if np.any(rows[b] < 0) or np.any(rows[b] >= e._X.shape[0]):
                raise ValueError(f"row index of job {b} out of range (GP {i} has {e._X.shape[0]} rows)")
            try:
                mean[b], var[b], c = e.gp_posterior_moments(params[b], e._X[rows[b]], n_joint)
            except GPCholeskyError:
                status[b] = 1
                continue
            cov[b] = c
        return mean, var, cov, status
