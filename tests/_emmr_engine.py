"""``NumpyEMMREngine`` -- ``NumpyGPEngine`` (tests/_gp_engine.py) with the two engine calls ``EMMREvaluator`` adds:
the loss with the noise held fixed (``gp_loss(..., deterministic=True)``, tpe_gp_loss_fixed_noise) and the posterior
moments with the joint covariance of a few points (``gp_posterior_moments``, tpe_gp_posterior_moments) (TEST
INFRASTRUCTURE).

The same NumPy restatement of tpe_gp.cuh: with the noise fixed, the covariance's noise is ``minimum_noise`` and the raw
noise gradient is 1/2 * 0 * sum_i W_ii; the moments are mean = k* . alpha, var = ks - |L^-1 k*|^2 clamped at 0, and
the joint covariance ks Matern52(r(x_a, x_b)) - V_a . V_b with V = K L^-T, its diagonal clamped at 0
(k_gp_joint_cov).
"""
from __future__ import annotations

import math

import numpy as np

from optuna_b200.engine import GPCholeskyError
from tests._gp_engine import NumpyGPEngine, _matern52


class NumpyEMMREngine(NumpyGPEngine):
    def gp_loss(self, raw_params, minimum_noise, deterministic=False):
        if not deterministic:
            return super().gp_loss(raw_params, minimum_noise)
        raw = np.asarray(raw_params, dtype=np.float64)
        P = self._X.shape[1]
        ell, ks = np.exp(raw[:P]), np.exp(raw[P])
        if not (np.all(np.isfinite(ell)) and np.isfinite(ks)):
            raise GPCholeskyError("non-finite kernel parameters")
        sqd, val, der, L, Linv, u, alpha = self._factor(ell, ks, minimum_noise)
        n = L.shape[0]
        mll = (-np.log(np.diag(L)).sum() + -0.5 * n * math.log(2 * math.pi)) + -0.5 * (u @ u)
        W = Linv.T @ Linv - np.outer(alpha, alpha)
        off = ~np.eye(n, dtype=bool)
        Wd = (W * der)[off]
        grad = np.empty(P + 2)
        grad[:P] = ks * ell * (0.5 * (Wd @ sqd[off]))   # both triangles: 1/2 sum_{i != j} = sum_{i > j}
        sdiag = np.trace(W)
        grad[P] = ks * ((W * val)[np.tril(off)].sum() + 0.5 * sdiag)
        grad[P + 1] = 0.5 * 0.0 * sdiag
        return float(-mll), grad

    def gp_posterior_moments(self, params, Xq, n_joint=0):
        prm, xq = np.asarray(params, dtype=np.float64), np.asarray(Xq, dtype=np.float64)
        P = self._X.shape[1]
        ell, ks, noise = prm[:P], prm[P], prm[P + 1]
        if n_joint != 0 and not 2 <= n_joint <= min(64, xq.shape[0]):
            raise ValueError("bad joint covariance request")
        _, _, _, _, Linv, _, alpha = self._factor(ell, ks, noise)
        K = _matern52(self._sqd(xq, self._X) @ ell)[0] * ks
        mean = K @ alpha
        V = K @ Linv.T
        var = np.maximum(ks - (V * V).sum(axis=1), 0.0)
        J = xq[:n_joint]
        cov = _matern52(self._sqd(J, J) @ ell)[0] * ks - V[:n_joint] @ V[:n_joint].T
        cov[np.diag_indices(n_joint)] = np.maximum(np.diag(cov), 0.0)
        return mean, var, cov
