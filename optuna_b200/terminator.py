"""The terminator's regret bound on the GPU: a drop-in ``RegretBoundEvaluator``.

``optuna.terminator.Terminator``, ``TerminatorCallback`` and ``plot_terminator_improvement`` default to optuna's
``RegretBoundEvaluator``.  Each ``evaluate`` fits a Gaussian process to the top trials by L-BFGS-B over the kernel
parameters; every loss evaluation builds an n x n x P tensor of squared differences, a Cholesky factor and a torch
autograd pass (optuna/_gp/gp.py:287-409).  This evaluator keeps optuna's steps, its L-BFGS-B (scipy, with optuna's
arguments), its prior and its random stream, and computes the negative marginal log-likelihood, its gradient and the
posterior bounds on the device (optuna_b200/csrc/tpe_gp.cuh): the covariance is built on the fly, factorised and
inverted by blocked fp64 tensor-core kernels.

One difference: the device holds two n x n fp64 matrices (n = the number of top trials), and ``evaluate`` raises
``ValueError`` naming the need when the device lacks that memory.  The reference keeps an n x n x P tensor on the
host and cannot run at those sizes at all.
"""
from __future__ import annotations

import numpy as np
import torch
from optuna._gp import search_space as gp_search_space
from optuna._gp.scipy_blas_thread_patch import single_blas_thread_if_scipy_v1_15_or_newer
from optuna.logging import get_logger
from optuna.search_space import intersection_search_space
from optuna.study import StudyDirection
from optuna.terminator import RegretBoundEvaluator as _OptunaRegretBoundEvaluator
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


def _loss_and_grad(engine, raw_params: np.ndarray, n_params: int, log_prior,
                   minimum_noise: float) -> tuple[float, np.ndarray]:
    """``loss_func`` of ``_fit_kernel_params`` (gp.py:312-327): -log p(y) - log_prior and its gradient in the raw
    parameters.  The likelihood part comes from the engine, the prior part (O(P)) from torch autograd."""
    neg_mll, grad = engine.gp_loss(raw_params, minimum_noise)
    raw_params_tensor = torch.from_numpy(raw_params).requires_grad_(True)
    with torch.enable_grad():
        prior = log_prior(_KernelParams(
            torch.exp(raw_params_tensor[:n_params]),
            torch.exp(raw_params_tensor[n_params]),
            torch.exp(raw_params_tensor[n_params + 1]) + minimum_noise,
        ))
        (-prior).backward()
    return neg_mll - prior.item(), grad + raw_params_tensor.grad.detach().cpu().numpy()


def _fit_kernel_params(engine, n_params: int, log_prior, minimum_noise: float, gtol: float = 1e-2) -> np.ndarray:
    """``GPRegressor._fit_kernel_params`` from the default parameters (gp.py:287-351, deterministic_objective=False):
    returns (inverse squared lengthscales, kernel scale, noise_var).  The negative marginal log-likelihood and its
    gradient come from the device, the prior term from ``log_prior`` with torch autograd."""
    import scipy.optimize

    # gp.py:301-310 with inverse_squared_lengthscales = kernel_scale = noise_var = 1
    initial_raw_params = np.concatenate([np.log(np.ones(n_params)), [np.log(1.0), np.log(1.0 - 0.99 * minimum_noise)]])

    def loss_func(raw_params: np.ndarray) -> tuple[float, np.ndarray]:
        return _loss_and_grad(engine, raw_params, n_params, log_prior, minimum_noise)

    with single_blas_thread_if_scipy_v1_15_or_newer():
        res = scipy.optimize.minimize(loss_func, initial_raw_params, jac=True, method="l-bfgs-b",
                                      options={"gtol": gtol})
    if not res.success:
        raise RuntimeError(f"Optimization failed: {res.message}")
    raw = torch.from_numpy(res.x)
    return np.concatenate([
        torch.exp(raw[:n_params]).numpy(),
        [torch.exp(raw[n_params]).item(), (minimum_noise + torch.exp(raw[n_params + 1])).item()],
    ])


def _fit(engine, n_params: int, log_prior, minimum_noise: float) -> np.ndarray:
    """``fit_kernel_params`` with ``gpr_cache=None`` (gp.py:354-409): two attempts from the default parameters, then
    the warning and the default GP."""
    error = None
    for _ in range(2):
        try:
            return _fit_kernel_params(engine, n_params, log_prior, minimum_noise)
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

