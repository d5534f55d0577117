"""``NumpyGPSamplerEngine`` -- ``NumpyEMMREngine`` (tests/_emmr_engine.py) with the two engine calls ``GPSampler``
adds: ``gp_condition`` (tpe_gp_condition) and ``gp_query`` (tpe_gp_query) (TEST INFRASTRUCTURE).

The same NumPy restatement of tpe_gp.cuh: conditioning keeps L^-1 and alpha = C^-1 y at the given parameters, and a
query returns mean = k* . alpha and var = ks - |L^-1 k*|^2 clamped at 0 and, with gradients, with w = L^-T L^-1 k*,
  dmean/dx_d = 2 l_d ks sum_i alpha_i M'(r_i) (x_d - X_id),  dvar/dx_d = -2 (2 l_d ks sum_i w_i M'(r_i) (x_d - X_id)),
0 in categorical columns and, for dvar, where the variance was clamped (k_gp_post_grad).  Any other GP call undoes
the conditioning.
"""
from __future__ import annotations

import numpy as np

from tests._emmr_engine import NumpyEMMREngine
from tests._gp_engine import _matern52


class NumpyGPSamplerEngine(NumpyEMMREngine):
    _cond = None

    def gp_set_data(self, X, y, is_categorical):
        self._cond = None
        return super().gp_set_data(X, y, is_categorical)

    def gp_loss(self, raw_params, minimum_noise, deterministic=False):
        self._cond = None
        return super().gp_loss(raw_params, minimum_noise, deterministic)

    def gp_posterior(self, params, Xq, beta):
        self._cond = None
        return super().gp_posterior(params, Xq, beta)

    def gp_posterior_moments(self, params, Xq, n_joint=0):
        self._cond = None
        return super().gp_posterior_moments(params, Xq, n_joint)

    def gp_condition(self, params):
        self._cond = None
        prm = np.asarray(params, dtype=np.float64)
        P = self._X.shape[1]
        ell, ks, noise = prm[:P], prm[P], prm[P + 1]
        _, _, _, _, Linv, _, alpha = self._factor(ell, ks, noise)
        self._cond = (ell, ks, Linv, alpha)

    def gp_query(self, Xq, grad=False):
        if self._cond is None:
            raise RuntimeError("the GP is not conditioned")
        ell, ks, Linv, alpha = self._cond
        xq = np.asarray(Xq, dtype=np.float64)
        val, der = _matern52(self._sqd(xq, self._X) @ ell)
        K = val * ks
        mean = K @ alpha
        V = K @ Linv.T
        raw_var = ks - (V * V).sum(axis=1)
        var = np.maximum(raw_var, 0.0)
        if not grad:
            return mean, var
        w = V @ Linv
        diff = xq[:, None, :] - self._X[None, :, :]
        dmean = 2.0 * ell * ks * np.einsum("mn,mnp->mp", alpha * der, diff)
        dvar = -2.0 * (2.0 * ell * ks * np.einsum("mn,mnp->mp", w * der, diff))
        dmean[:, self._cat] = 0.0
        dvar[:, self._cat] = 0.0
        dvar[raw_var < 0.0] = 0.0
        return mean, var, dmean, dvar
