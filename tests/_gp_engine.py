"""``NumpyGPEngine`` -- ``TPEEngine.gp_set_data`` / ``gp_loss`` / ``gp_posterior`` answered on the host (TEST
INFRASTRUCTURE).

The steps of tpe_gp.cuh restated in NumPy: the covariance from the squared differences (Hamming in categorical
columns), its Cholesky factor, L^-1 and C^-1 = L^-T L^-1, the loss from sum log L_ii and u = L^-1 y, the gradient as
one pass over the lower triangle with W = C^-1 - alpha alpha^T and optuna's saved Matern derivative, and the
posterior variance as ks - |L^-1 k*|^2.  Plugged into ``optuna_b200.terminator``, it lets the CPU suite check the
algorithm and the Python glue against the live reference.
"""
from __future__ import annotations

import math

import numpy as np
import scipy.linalg

from optuna_b200.engine import GPCholeskyError


def _matern52(r):
    s = np.sqrt(5.0 * r)
    e = np.exp(-s)
    return e * ((5.0 / 3.0) * r + s + 1.0), (-5.0 / 6.0) * (s + 1.0) * e


class NumpyGPEngine:
    def __init__(self, device: int = 0) -> None:
        self._X = None

    def close(self) -> None:
        pass

    def gp_set_data(self, X, y, is_categorical) -> None:
        X, y = np.asarray(X, dtype=np.float64), np.asarray(y, dtype=np.float64)
        cat = np.asarray(is_categorical, dtype=bool)
        if X.ndim != 2 or y.shape != (X.shape[0],) or cat.shape != (X.shape[1],) or X.shape[0] < 1 or X.shape[1] < 1:
            raise ValueError("bad GP data")
        if not (np.all(np.isfinite(X)) and np.all(np.isfinite(y))):
            raise ValueError("GP data hold a non-finite value")
        self._X, self._y, self._cat = X, y, cat

    def _sqd(self, A, B):
        sqd = (A[:, None, :] - B[None, :, :]) ** 2
        sqd[..., self._cat] = (sqd[..., self._cat] > 0.0).astype(np.float64)
        return sqd

    def _factor(self, ell, ks, noise):
        n = self._X.shape[0]
        sqd = self._sqd(self._X, self._X)
        val, der = _matern52(sqd @ ell)
        C = val * ks
        C[np.diag_indices(n)] += noise
        try:
            L = np.linalg.cholesky(C)
        except np.linalg.LinAlgError as e:
            raise GPCholeskyError(str(e)) from e
        Linv = scipy.linalg.solve_triangular(L, np.eye(n), lower=True)
        u = Linv @ self._y
        return sqd, val, der, L, Linv, u, Linv.T @ u

    def gp_loss(self, raw_params, minimum_noise):
        raw = np.asarray(raw_params, dtype=np.float64)
        P = self._X.shape[1]
        ell, ks = np.exp(raw[:P]), np.exp(raw[P])
        noise_excess = np.exp(raw[P + 1])
        if not (np.all(np.isfinite(ell)) and np.isfinite(ks) and np.isfinite(noise_excess + minimum_noise)):
            raise GPCholeskyError("non-finite kernel parameters")
        sqd, val, der, L, Linv, u, alpha = self._factor(ell, ks, noise_excess + minimum_noise)
        n = L.shape[0]
        mll = (-np.log(np.diag(L)).sum() + -0.5 * n * math.log(2 * math.pi)) + -0.5 * (u @ u)
        W = Linv.T @ Linv - np.outer(alpha, alpha)
        off = ~np.eye(n, dtype=bool)
        Wd = (W * der)[off]
        grad = np.empty(P + 2)
        grad[:P] = ks * ell * (0.5 * (Wd @ sqd[off]))   # both triangles: 1/2 sum_{i != j} = sum_{i > j}
        sdiag = np.trace(W)
        grad[P] = ks * ((W * val)[np.tril(off)].sum() + 0.5 * sdiag)
        grad[P + 1] = 0.5 * noise_excess * sdiag
        return float(-mll), grad

    def gp_posterior(self, params, Xq, beta):
        prm = np.asarray(params, dtype=np.float64)
        P = self._X.shape[1]
        ell, ks, noise = prm[:P], prm[P], prm[P + 1]
        _, _, _, _, Linv, _, alpha = self._factor(ell, ks, noise)
        K = _matern52(self._sqd(np.asarray(Xq, dtype=np.float64), self._X) @ ell)[0] * ks
        mean = K @ alpha
        V = K @ Linv.T
        var = np.maximum(ks - (V * V).sum(axis=1), 0.0)
        h = np.sqrt(beta * var)
        return mean + h, mean - h
