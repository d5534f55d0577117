"""The terminator's improvement evaluators on the GPU: drop-in ``RegretBoundEvaluator`` and ``EMMREvaluator``.

``optuna.terminator.Terminator``, ``TerminatorCallback`` and ``plot_terminator_improvement`` default to optuna's
``RegretBoundEvaluator``.  Each ``evaluate`` fits a Gaussian process to the top trials by L-BFGS-B over the kernel
parameters; every loss evaluation builds an n x n x P tensor of squared differences, a Cholesky factor and a torch
autograd pass (optuna/_gp/gp.py:287-409).  This evaluator keeps optuna's steps, its L-BFGS-B (scipy, with optuna's
arguments), its prior and its random stream, and computes the negative marginal log-likelihood, its gradient and the
posterior bounds on the device (optuna_b200/csrc/tpe_gp.cuh): the covariance is built on the fly, factorised and
inverted by blocked fp64 tensor-core kernels.

``EMMREvaluator`` (optuna/terminator/improvement/emmr.py) fits two such GPs per ``evaluate``, to all complete trials
but the last and then to all of them, warm-started from the first; with ``deterministic_objective`` the noise is held
at its minimum.  Its drop-in does the same on the device, and takes from it the posterior mean and variance and the
joint covariance of two points.

One difference: the device holds two n x n fp64 matrices (n = the number of trials fitted), and ``evaluate`` raises
``ValueError`` naming the need when the device lacks that memory.  The reference keeps an n x n x P tensor on the
host and cannot run at those sizes at all.
"""
from __future__ import annotations

import math
import sys

import numpy as np
import scipy.stats
import torch
from optuna._gp import gp, prior
from optuna._gp import search_space as gp_search_space
from optuna._gp.scipy_blas_thread_patch import single_blas_thread_if_scipy_v1_15_or_newer
from optuna._warnings import optuna_warn
from optuna.logging import get_logger
from optuna.search_space import intersection_search_space
from optuna.study import StudyDirection
from optuna.terminator import EMMREvaluator as _OptunaEMMREvaluator
from optuna.terminator import RegretBoundEvaluator as _OptunaRegretBoundEvaluator
from optuna.terminator.improvement.emmr import MARGIN_FOR_NUMARICAL_STABILITY
from optuna.terminator.improvement.evaluator import _get_beta
from optuna.trial import FrozenTrial, TrialState

from .engine import GPCholeskyError, TPEEngine

# the engine class that answers the computation (tests substitute a host implementation)
_engine_cls = TPEEngine

_logger = get_logger("optuna.terminator.optuna_b200")  # a child of optuna's root logger: same handlers / verbosity


class _KernelParams:
    """What ``default_log_prior`` reads of a ``GPRegressor`` (optuna/_gp/prior.py:19-33)."""

    def __init__(self, inverse_squared_lengthscales: torch.Tensor, kernel_scale: torch.Tensor,
                 noise_var: torch.Tensor) -> None:
        self.inverse_squared_lengthscales = inverse_squared_lengthscales
        self.kernel_scale = kernel_scale
        self.noise_var = noise_var


def _loss_and_grad(engine, raw_params: np.ndarray, n_params: int, log_prior, minimum_noise: float,
                   deterministic_objective: bool = False) -> tuple[float, np.ndarray]:
    """``loss_func`` of ``_fit_kernel_params`` (gp.py:312-327): -log p(y) - log_prior and its gradient in the raw
    parameters.  The likelihood part comes from the engine, the prior part (O(P)) from torch autograd.  With
    ``deterministic_objective`` the noise is the constant ``minimum_noise``: the prior sees it as a constant tensor, so
    it adds to the loss and nothing to the gradient, and the raw noise gradient is 0."""
    if deterministic_objective:
        neg_mll, grad = engine.gp_loss(raw_params, minimum_noise, deterministic=True)
    else:   # the call RegretBoundEvaluator has always made
        neg_mll, grad = engine.gp_loss(raw_params, minimum_noise)
    raw_params_tensor = torch.from_numpy(raw_params).requires_grad_(True)
    with torch.enable_grad():
        prior = log_prior(_KernelParams(
            torch.exp(raw_params_tensor[:n_params]),
            torch.exp(raw_params_tensor[n_params]),
            torch.tensor(minimum_noise, dtype=torch.float64) if deterministic_objective
            else torch.exp(raw_params_tensor[n_params + 1]) + minimum_noise,
        ))
        (-prior).backward()
    return neg_mll - prior.item(), grad + raw_params_tensor.grad.detach().cpu().numpy()


def _fit_kernel_params(engine, n_params: int, log_prior, minimum_noise: float, initial_params: np.ndarray,
                       deterministic_objective: bool = False, gtol: float = 1e-2) -> np.ndarray:
    """``GPRegressor._fit_kernel_params`` (gp.py:287-351) from ``initial_params`` = (inverse squared lengthscales,
    kernel scale, noise_var): returns the fitted parameters in the same form, as the GP stores them.  The negative
    marginal log-likelihood and its gradient come from the device, the prior term from ``log_prior`` with torch
    autograd."""
    import scipy.optimize

    # gp.py:301-310: the lengthscales as one array, the kernel scale and noise as Python floats
    initial_raw_params = np.concatenate([
        np.log(initial_params[:n_params]),
        [np.log(float(initial_params[n_params])), np.log(float(initial_params[n_params + 1]) - 0.99 * minimum_noise)],
    ])

    def loss_func(raw_params: np.ndarray) -> tuple[float, np.ndarray]:
        return _loss_and_grad(engine, raw_params, n_params, log_prior, minimum_noise, deterministic_objective)

    with single_blas_thread_if_scipy_v1_15_or_newer():
        res = scipy.optimize.minimize(loss_func, initial_raw_params, jac=True, method="l-bfgs-b",
                                      options={"gtol": gtol})
    if not res.success:
        raise RuntimeError(f"Optimization failed: {res.message}")
    raw = torch.from_numpy(res.x)
    noise_var = minimum_noise if deterministic_objective else (minimum_noise + torch.exp(raw[n_params + 1])).item()
    return np.concatenate([torch.exp(raw[:n_params]).numpy(), [torch.exp(raw[n_params]).item(), noise_var]])


def _fit(engine, n_params: int, log_prior, minimum_noise: float, gpr_cache: np.ndarray | None = None,
         deterministic_objective: bool = False) -> np.ndarray:
    """``fit_kernel_params`` (gp.py:354-409): a first attempt from ``gpr_cache`` (the parameters an earlier fit
    returned; the default parameters when None), a second from the default parameters, then the warning and the
    default GP, whose noise_var is 1 whatever ``deterministic_objective`` is."""
    default_params = np.ones(n_params + 2)
    error = None
    for initial_params in (default_params if gpr_cache is None else gpr_cache, default_params):
        try:
            return _fit_kernel_params(engine, n_params, log_prior, minimum_noise, initial_params,
                                      deterministic_objective)
        except RuntimeError as e:
            error = e
    _logger.warning(
        f"The optimization of kernel parameters failed: \n{error}\n"
        "The default initial kernel parameters will be used instead."
    )
    return np.ones(n_params + 2)


class RegretBoundEvaluator(_OptunaRegretBoundEvaluator):
    """Regret-bound improvement evaluator whose Gaussian process is fitted and queried on the GPU.

    A drop-in for ``optuna.terminator.RegretBoundEvaluator``: pass it as ``improvement_evaluator=`` to
    ``Terminator``, ``TerminatorCallback`` or ``plot_terminator_improvement``.  For the same seed it consumes the
    random stream as the reference does and returns the reference's bound.

    The device holds two n x n fp64 matrices, n being the number of top trials the GP is fitted to.  When it lacks
    that memory, ``evaluate`` raises ``ValueError`` naming the need; this is the one difference from the reference,
    which cannot run at those sizes at all.

    Args:
        top_trials_ratio: A ratio of top trials to be considered when estimating the regret.
        min_n_trials: A minimum number of complete trials to estimate the regret.
        seed: Seed for random number generator.
        device: CUDA device to compute on.
    """

    def __init__(self, top_trials_ratio: float = 0.5, min_n_trials: int = 20, seed: int | None = None, *,
                 device: int = 0) -> None:
        super().__init__(top_trials_ratio=top_trials_ratio, min_n_trials=min_n_trials, seed=seed)
        self._device = device

    def evaluate(self, trials: list[FrozenTrial], study_direction: StudyDirection) -> float:
        # optuna/terminator/improvement/evaluator.py:142-177, with the fit and the bounds on the device
        optuna_search_space = intersection_search_space(trials)
        self._validate_input(trials, optuna_search_space)

        complete_trials = [t for t in trials if t.state == TrialState.COMPLETE]

        sign = -1 if study_direction == StudyDirection.MINIMIZE else 1
        values = np.array([t.value for t in complete_trials]) * sign
        search_space = gp_search_space.SearchSpace(optuna_search_space)
        normalized_params = search_space.get_normalized_params(complete_trials)
        normalized_top_n_params, top_n_values = self._get_top_n(normalized_params, values)
        top_n_values_mean = top_n_values.mean()
        top_n_values_std = max(1e-10, top_n_values.std())
        standarized_top_n_values = (top_n_values - top_n_values_mean) / top_n_values_std

        n_trials, n_params = normalized_top_n_params.shape
        engine = _engine_cls(self._device)
        try:
            engine.gp_set_data(normalized_top_n_params, standarized_top_n_values, search_space.is_categorical)
            params = _fit(engine, n_params, self._log_prior, self._minimum_noise)
            # _compute_standardized_regret_bound (evaluator.py:50-84): UCB over the top trials and over the 2048
            # samples of optimize_acqf_sample, LCB over the top trials
            beta = _get_beta(n_params, n_trials)
            xs = search_space.sample_normalized_params(self._optimize_n_samples, rng=self._rng.rng)
            try:
                ucb, lcb = engine.gp_posterior(params, np.concatenate([normalized_top_n_params, xs]), beta)
            except GPCholeskyError as e:
                # the reference factorises the final covariance with NumPy (gp.py:132)
                raise np.linalg.LinAlgError("Matrix is not positive definite") from e
        finally:
            engine.close()
        standardized_ucb_value = max(ucb[:n_trials].max(), ucb[n_trials:].max())
        standardized_lcb_value = np.max(lcb[:n_trials])
        return (standardized_ucb_value - standardized_lcb_value) * top_n_values_std


def _posterior_moments(engine, params: np.ndarray, Xq: np.ndarray, n_joint: int = 0):
    try:
        return engine.gp_posterior_moments(params, Xq, n_joint)
    except GPCholeskyError as e:
        # the reference factorises the final covariance with NumPy (gp.py:132)
        raise np.linalg.LinAlgError("Matrix is not positive definite") from e


class EMMREvaluator(_OptunaEMMREvaluator):
    """Expected Minimum Model Regret (EMMR) improvement evaluator whose two Gaussian processes are fitted and queried
    on the GPU.

    A drop-in for ``optuna.terminator.EMMREvaluator``: pass it as ``improvement_evaluator=`` to ``Terminator``,
    ``TerminatorCallback`` or ``plot_terminator_improvement``, or as the evaluator of optuna's
    ``MedianErrorEvaluator``.  For the same seed it consumes the random stream as the reference does and returns the
    reference's criterion.

    The device holds two n x n fp64 matrices, n being the number of complete trials.  When it lacks that memory,
    ``evaluate`` raises ``ValueError`` naming the need; this is the one difference from the reference.

    Args:
        deterministic_objective: Whether the objective function is deterministic (the GP noise is then fixed at its
            minimum).
        delta: The confidence parameter of the regret bound's beta.
        min_n_trials: A minimum number of complete trials to compute the criterion.
        seed: Seed for random number generator.
        device: CUDA device to compute on.
    """

    def __init__(self, deterministic_objective: bool = False, delta: float = 0.1, min_n_trials: int = 2,
                 seed: int | None = None, *, device: int = 0) -> None:
        super().__init__(deterministic_objective=deterministic_objective, delta=delta, min_n_trials=min_n_trials,
                         seed=seed)
        self._device = device

    def evaluate(self, trials: list[FrozenTrial], study_direction: StudyDirection) -> float:
        # optuna/terminator/improvement/emmr.py:123-237, with both fits and the posterior on the device
        optuna_search_space = intersection_search_space(trials)
        complete_trials = [t for t in trials if t.state == TrialState.COMPLETE]

        if len(complete_trials) < self.min_n_trials:
            return sys.float_info.max * MARGIN_FOR_NUMARICAL_STABILITY  # Do not terminate.

        search_space = gp_search_space.SearchSpace(optuna_search_space)
        normalized_params = search_space.get_normalized_params(complete_trials)
        if not search_space.dim:
            optuna_warn(
                f"{self.__class__.__name__} cannot consider any search space."
                "Termination will never occur in this study."
            )
            return sys.float_info.max * MARGIN_FOR_NUMARICAL_STABILITY  # Do not terminate.

        sign = -1 if study_direction == StudyDirection.MINIMIZE else 1
        score_vals = np.array([t.value for t in complete_trials]) * sign
        score_vals = gp.warn_and_convert_inf(score_vals)
        standarized_score_vals = (score_vals - score_vals.mean()) / max(sys.float_info.min, score_vals.std())

        n_params = normalized_params.shape[1]
        X_t1, y_t1 = normalized_params[:-1, :], standarized_score_vals[:-1]
        theta_t_star_index = int(np.argmax(standarized_score_vals))
        theta_t1_star_index = int(np.argmax(y_t1))
        minimum_noise = prior.DEFAULT_MINIMUM_NOISE_VAR
        engine = _engine_cls(self._device)
        try:
            # the GP over the first t - 1 trials, and the regret bound of _compute_standardized_regret_bound
            # (evaluator.py:50-84) from it: UCB over those trials and the 2048 samples, LCB over those trials.  Its
            # mean at theta*_{t-1} is the training-point row of that trial.
            engine.gp_set_data(X_t1, y_t1, search_space.is_categorical)
            params_t1 = _fit(engine, n_params, prior.default_log_prior, minimum_noise,
                             deterministic_objective=self._deterministic)
            beta = _get_beta(n_params, len(y_t1), self._delta)
            xs = search_space.sample_normalized_params(2048, rng=self._rng.rng)
            mean_t1, var_t1, _ = _posterior_moments(engine, params_t1, np.concatenate([X_t1, xs]))
            h = np.sqrt(beta * var_t1)
            ucb, lcb = mean_t1 + h, mean_t1 - h
            kappa_t1 = max(ucb[: len(y_t1)].max(), ucb[len(y_t1):].max()) - np.max(lcb[: len(y_t1)])
            mu_t1_theta_t1_star = float(mean_t1[theta_t1_star_index])

            # the GP over all t trials, warm-started from the first, at theta*_t, theta*_{t-1} and x_t
            engine.gp_set_data(normalized_params, standarized_score_vals, search_space.is_categorical)
            params_t = _fit(engine, n_params, prior.default_log_prior, minimum_noise, gpr_cache=params_t1,
                            deterministic_objective=self._deterministic)
            mean_t, var_t, cov_t = _posterior_moments(
                engine, params_t,
                normalized_params[[theta_t_star_index, theta_t1_star_index, len(standarized_score_vals) - 1]], 2)
        finally:
            engine.close()

        # emmr.py:249-250: for one point the reference takes the variance of the non-joint posterior
        cov_t_between_theta_t_star_and_theta_t1_star = float(
            var_t[0] if theta_t_star_index == theta_t1_star_index else cov_t[0, 1])
        mu_t_theta_t_star, variance_t_theta_t_star = float(mean_t[0]), float(var_t[0])
        variance_t_theta_t1_star = float(var_t[1])
        mu_t1_theta_t_with_nu_t, variance_t1_theta_t_with_nu_t = float(mean_t[2]), float(var_t[2])
        y_t = standarized_score_vals[-1]

        # emmr.py:198-237
        theorem1_delta_mu_t_star = mu_t1_theta_t1_star - mu_t_theta_t_star
        alg1_delta_r_tilde_t_term1 = theorem1_delta_mu_t_star
        theorem1_v = math.sqrt(
            max(
                1e-10,
                variance_t_theta_t_star
                - 2.0 * cov_t_between_theta_t_star_and_theta_t1_star
                + variance_t_theta_t1_star,
            )
        )
        theorem1_g = (mu_t_theta_t_star - mu_t1_theta_t1_star) / theorem1_v
        alg1_delta_r_tilde_t_term2 = theorem1_v * scipy.stats.norm.pdf(theorem1_g)
        alg1_delta_r_tilde_t_term3 = theorem1_v * theorem1_g * scipy.stats.norm.cdf(theorem1_g)

        _lambda = prior.DEFAULT_MINIMUM_NOISE_VAR**-1
        eq4_rhs_term1 = 0.5 * math.log(1.0 + _lambda * variance_t1_theta_t_with_nu_t)
        eq4_rhs_term2 = -0.5 * variance_t1_theta_t_with_nu_t / (variance_t1_theta_t_with_nu_t + _lambda**-1)
        eq4_rhs_term3 = (
            0.5
            * variance_t1_theta_t_with_nu_t
            * (y_t - mu_t1_theta_t_with_nu_t) ** 2
            / (variance_t1_theta_t_with_nu_t + _lambda**-1) ** 2
        )
        alg1_delta_r_tilde_t_term4 = kappa_t1 * math.sqrt(0.5 * (eq4_rhs_term1 + eq4_rhs_term2 + eq4_rhs_term3))

        return min(
            sys.float_info.max * 0.5,
            alg1_delta_r_tilde_t_term1
            + alg1_delta_r_tilde_t_term2
            + alg1_delta_r_tilde_t_term3
            + alg1_delta_r_tilde_t_term4,
        )

