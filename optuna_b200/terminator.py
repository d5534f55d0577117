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

import contextlib
import math
import sys
import threading

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
                       deterministic_objective: bool = False, gtol: float = 1e-2,
                       single_blas: bool = True) -> np.ndarray:
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

    # single_blas=False: the caller (the lock-step batch, which runs many fits in threads) holds the limit
    with single_blas_thread_if_scipy_v1_15_or_newer() if single_blas else contextlib.nullcontext():
        res = scipy.optimize.minimize(loss_func, initial_raw_params, jac=True, method="l-bfgs-b",
                                      options={"gtol": gtol})
    if not res.success:
        raise RuntimeError(f"Optimization failed: {res.message}")
    raw = torch.from_numpy(res.x)
    noise_var = minimum_noise if deterministic_objective else (minimum_noise + torch.exp(raw[n_params + 1])).item()
    return np.concatenate([torch.exp(raw[:n_params]).numpy(), [torch.exp(raw[n_params]).item(), noise_var]])


def _fit(engine, n_params: int, log_prior, minimum_noise: float, gpr_cache: np.ndarray | None = None,
         deterministic_objective: bool = False, single_blas: bool = True) -> np.ndarray:
    """``fit_kernel_params`` (gp.py:354-409): a first attempt from ``gpr_cache`` (the parameters an earlier fit
    returned; the default parameters when None), a second from the default parameters, then the warning and the
    default GP, whose noise_var is 1 whatever ``deterministic_objective`` is."""
    default_params = np.ones(n_params + 2)
    error = None
    for initial_params in (default_params if gpr_cache is None else gpr_cache, default_params):
        try:
            return _fit_kernel_params(engine, n_params, log_prior, minimum_noise, initial_params,
                                      deterministic_objective, single_blas=single_blas)
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
        return _emmr_criterion(kappa_t1, mu_t1_theta_t1_star, mean_t, var_t,
                               cov_t_between_theta_t_star_and_theta_t1_star, standarized_score_vals[-1])


def _emmr_criterion(kappa_t1: float, mu_t1_theta_t1_star: float, mean_t, var_t,
                    cov_t_between_theta_t_star_and_theta_t1_star: float, y_t: float) -> float:
    """The closing arithmetic of ``EMMREvaluator.evaluate`` (emmr.py:198-237): ``mean_t`` and ``var_t`` are the
    posterior of the GP over all t trials at theta*_t, theta*_{t-1} and x_t, ``kappa_t1`` and
    ``mu_t1_theta_t1_star`` come from the GP over the first t - 1 trials."""
    mu_t_theta_t_star, variance_t_theta_t_star = float(mean_t[0]), float(var_t[0])
    variance_t_theta_t1_star = float(var_t[1])
    mu_t1_theta_t_with_nu_t, variance_t1_theta_t_with_nu_t = float(mean_t[2]), float(var_t[2])

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


# ---- the whole improvement curve at once ------------------------------------------------------------------------------
# Upper bound on the device memory one wave of batched fits may take (data, workspace and sample rows).  A private
# module constant so that tests can make every wave a single GP.
_WAVE_BYTES = 4 << 30


def _wave_bytes(n: int, P: int, n_samples: int) -> int:
    """Device bytes one GP of n rows adds to a wave: its rows, the workspace of tpe_gpbatch.cuh (an n x n matrix and
    three n-vectors above 160 rows, and n x 256 doubles of cross covariance for the bounds) and its samples."""
    ws = (n * n + 3 * n if n > 160 else 0) + n * 256
    return 8 * (n * (P + 1) + ws + n_samples * P + 2 * (P + 2) + 8)


class _Prefix:
    """What ``RegretBoundEvaluator.evaluate`` forms for one trial prefix before its fit (evaluator.py:142-163)."""

    __slots__ = ("X", "y", "std", "is_categorical", "beta", "samples", "gp", "failed")


class _LockStep:
    """Lock-step evaluation for one thread per task (scipy's L-BFGS-B or Brent searches).  A thread's ``post`` hands
    over its payload and blocks; ``run`` evaluates everything posted in one ``evaluate(payloads)`` call (the payloads
    in key order, one result each), then releases the threads one at a time and waits for each to post again or
    finish.  So one thread runs at a time (the host work is serial under the GIL anyway) and the threads do not
    contend for the GIL; a thread that calls ``leave`` drops out of the batch."""

    def __init__(self, evaluate) -> None:
        self._evaluate = evaluate
        self._cond = threading.Condition()
        self._posted: dict[int, object] = {}
        self._left: set[int] = set()
        self._results: dict[int, object] = {}
        self._events: dict[int, threading.Event] = {}
        self.rounds = 0
        self.device_seconds = 0.0

    def join(self, key: int) -> None:
        """Registers the thread of ``key`` before it starts."""
        self._events[key] = threading.Event()

    def post(self, key: int, payload):
        ev = self._events[key]
        with self._cond:
            self._posted[key] = payload
            self._cond.notify()
        ev.wait()
        ev.clear()
        return self._results.pop(key)

    def leave(self, key: int) -> None:
        with self._cond:
            self._left.add(key)
            self._cond.notify()

    def _wait(self, key: int) -> None:
        with self._cond:
            while key not in self._posted and key not in self._left:
                self._cond.wait()

    def run(self, threads: list) -> None:
        """Starts ``threads[k]`` (the thread of key k) and serves their posts until every one has left."""
        import time
        for key, th in enumerate(threads):
            th.start()
            self._wait(key)
        while self._posted:
            batch, self._posted = self._posted, {}
            keys = sorted(batch)
            t0 = time.perf_counter()
            results = self._evaluate([batch[k] for k in keys])
            self.device_seconds += time.perf_counter() - t0
            self.rounds += 1
            for k, r in zip(keys, results):
                self._results[k] = r
                self._events[k].set()
                self._wait(k)


def _batch_loss(engine, minimum_noise: float, deterministic: bool):
    """The lock-step evaluation of the batched fits: one ``gp_batch_loss`` over the posted (GP, raw parameters)."""
    def evaluate(posted: list) -> list:
        gps = [gp for gp, _ in posted]
        raws = np.stack([raw for _, raw in posted])
        if deterministic:
            loss, grad, status = engine.gp_batch_loss(gps, raws, minimum_noise, deterministic=True)
        else:
            loss, grad, status = engine.gp_batch_loss(gps, raws, minimum_noise)
        return [(float(loss[i]), grad[i].copy(), int(status[i])) for i in range(len(posted))]
    return evaluate


class _Slot:
    """The engine a fit thread sees: ``gp_loss`` answered by the lock-step batch, for the GP ``gp`` of the wave
    (the thread's own index unless its task sets another)."""

    def __init__(self, lockstep: _LockStep, key: int, deterministic: bool) -> None:
        self._ls = lockstep
        self._key = key
        self._deterministic = deterministic
        self.gp = key
        lockstep.join(key)

    def gp_loss(self, raw_params, minimum_noise: float, deterministic: bool = False):
        if deterministic != self._deterministic:
            raise ValueError("a fit's noise model differs from its lock-step batch's")
        loss, grad, status = self._ls.post(self._key, (self.gp, np.array(raw_params, dtype=np.float64)))
        if status:
            raise GPCholeskyError("the GP covariance is not positive definite")
        return loss, grad


def _in_waves(device: int, units: list[tuple[int, int]], run_wave, stats: dict | None) -> None:
    """The driver both batched evaluators use.  ``units`` holds (P, device bytes) per unit of work (a distinct
    complete set); the units are grouped by P in first-seen order and packed into waves of at most ``_WAVE_BYTES``
    (a unit larger than that gets a wave of its own), and ``run_wave(engine, wave)`` runs each wave's unit indices on
    one engine, under one BLAS thread limit."""
    import time
    by_p: dict[int, list[int]] = {}
    for i, (P, _) in enumerate(units):
        by_p.setdefault(P, []).append(i)
    engine = _engine_cls(device)
    t_all = time.perf_counter()
    try:
        with single_blas_thread_if_scipy_v1_15_or_newer():
            for members in by_p.values():
                waves: list[list[int]] = [[]]
                used = 0
                for i in members:
                    need = units[i][1]
                    if waves[-1] and used + need > _WAVE_BYTES:
                        waves.append([])
                        used = 0
                    waves[-1].append(i)
                    used += need
                for wave in waves:
                    run_wave(engine, wave)
    finally:
        engine.close()
    if stats is not None:
        stats["wall_seconds"] = time.perf_counter() - t_all


def _fit_wave(engine, data: list[tuple[np.ndarray, np.ndarray]], is_categorical, minimum_noise: float, tasks: list,
              stats: dict | None, deterministic: bool = False) -> list:
    """Uploads a wave's GPs (GP i fitted to ``data[i]`` = (X, y)) and runs ``tasks[k](slot)`` for every k, each in its
    own thread, in lock step.  A task fits through its slot, choosing the GP by ``slot.gp``.  Returns the tasks'
    results in order; an exception of a task is re-raised, the first task's first."""
    offsets = np.zeros(len(data) + 1, dtype=np.int64)
    offsets[1:] = np.cumsum([X.shape[0] for X, _ in data])
    engine.gp_batch_set(offsets, np.concatenate([X for X, _ in data]), np.concatenate([y for _, y in data]),
                        is_categorical)
    ls = _LockStep(_batch_loss(engine, minimum_noise, deterministic))
    results: dict[int, object] = {}
    errors: dict[int, BaseException] = {}

    def work(k: int, slot: _Slot) -> None:
        try:
            results[k] = tasks[k](slot)
        except BaseException as e:   # re-raised below, in task order
            errors[k] = e
        finally:
            ls.leave(k)

    threads = [threading.Thread(target=work, args=(k, _Slot(ls, k, deterministic)), daemon=True)
               for k in range(len(tasks))]
    ls.run(threads)
    for th in threads:
        th.join()
    if errors:
        raise errors[min(errors)]
    if stats is not None:
        stats["rounds"] = stats.get("rounds", 0) + ls.rounds
        stats["device_seconds"] = stats.get("device_seconds", 0.0) + ls.device_seconds
    return [results[k] for k in range(len(tasks))]


def _prepare_prefixes(evaluator: "RegretBoundEvaluator", study) -> tuple[list[int], list[_Prefix]]:
    """The host pre-pass, in the reference's trial order: per prefix the data of ``evaluate`` and its 2048 samples
    from the evaluator's own stream.  Prefixes whose complete trials are the same share one GP."""
    trial_numbers: list[int] = []
    prefixes: list[_Prefix] = []
    completed: list[FrozenTrial] = []
    last: _Prefix | None = None
    last_n = -1
    rng = evaluator._rng.rng
    direction = study.direction
    for trial in study.trials:
        if trial.state == TrialState.COMPLETE:
            completed.append(trial)
        if not completed:
            continue
        trial_numbers.append(trial.number)
        p = _Prefix()
        if len(completed) == last_n:
            p.X, p.y, p.std, p.is_categorical, p.beta = last.X, last.y, last.std, last.is_categorical, last.beta
            space = last_space
        else:
            trials = list(completed)
            optuna_search_space = intersection_search_space(trials)
            evaluator._validate_input(trials, optuna_search_space)
            sign = -1 if direction == StudyDirection.MINIMIZE else 1
            values = np.array([t.value for t in trials]) * sign
            space = gp_search_space.SearchSpace(optuna_search_space)
            normalized_params = space.get_normalized_params(trials)
            p.X, top_n_values = evaluator._get_top_n(normalized_params, values)
            top_n_values_mean = top_n_values.mean()
            p.std = max(1e-10, top_n_values.std())
            p.y = (top_n_values - top_n_values_mean) / p.std
            p.is_categorical = space.is_categorical
            p.beta = _get_beta(p.X.shape[1], p.X.shape[0])
        p.samples = space.sample_normalized_params(evaluator._optimize_n_samples, rng=rng)
        p.failed = False
        prefixes.append(p)
        last, last_n, last_space = p, len(completed), space
    return trial_numbers, prefixes


def _batched_improvements(evaluator: "RegretBoundEvaluator", study, stats: dict | None = None) -> tuple[list, list]:
    rng = evaluator._rng.rng
    start_state = rng.get_state()
    trial_numbers, prefixes = _prepare_prefixes(evaluator, study)
    if not prefixes:
        return [], []
    # the distinct GPs (one per distinct complete set), grouped by P, in waves bounded by _WAVE_BYTES
    gps: list[_Prefix] = []
    for p in prefixes:
        if not gps or p.X is not gps[-1].X:
            gps.append(p)
        p.gp = len(gps) - 1
    params: list[np.ndarray | None] = [None] * len(gps)
    n_samples = evaluator._optimize_n_samples
    out = np.empty((len(prefixes), 3))
    users = [[] for _ in gps]
    for j, p in enumerate(prefixes):
        users[p.gp].append(j)
    units = [(g.X.shape[1], _wave_bytes(g.X.shape[0], g.X.shape[1], n_samples * len(users[i])))
             for i, g in enumerate(gps)]
    _in_waves(evaluator._device, units,
              lambda engine, wave: _run_wave(engine, evaluator, gps, wave, users, prefixes, params, out, stats), stats)
    # the reference raises at the first prefix whose final covariance is not positive definite, after drawing that
    # prefix's samples: leave the stream there
    for j, p in enumerate(prefixes):
        if p.failed:
            rng.set_state(start_state)
            _prepare_prefixes_upto(evaluator, study, j)
            raise np.linalg.LinAlgError("Matrix is not positive definite")
    improvements = []
    for j, p in enumerate(prefixes):
        standardized_ucb_value = max(out[j, 0], out[j, 1])
        standardized_lcb_value = out[j, 2]
        improvements.append((standardized_ucb_value - standardized_lcb_value) * p.std)
    return trial_numbers, improvements


def _prepare_prefixes_upto(evaluator, study, last: int) -> None:
    """Redraws the samples of the prefixes 0 .. last, so that the stream is where the reference leaves it when it
    raises at prefix ``last``."""
    rng = evaluator._rng.rng
    completed = []
    j = -1
    space = None
    last_n = -1
    for trial in study.trials:
        if trial.state == TrialState.COMPLETE:
            completed.append(trial)
        if not completed:
            continue
        j += 1
        if len(completed) != last_n:
            space = gp_search_space.SearchSpace(intersection_search_space(list(completed)))
            last_n = len(completed)
        space.sample_normalized_params(evaluator._optimize_n_samples, rng=rng)
        if j == last:
            return


def _run_wave(engine, evaluator, gps, wave, users, prefixes, params, out, stats) -> None:
    """Fits the GPs of one wave in lock step, then the bounds of every prefix that uses them."""
    P = gps[wave[0]].X.shape[1]

    def task(slot: _Slot) -> np.ndarray:
        return _fit(slot, P, evaluator._log_prior, evaluator._minimum_noise, single_blas=False)

    fitted = _fit_wave(engine, [(gps[i].X, gps[i].y) for i in wave], gps[wave[0]].is_categorical,
                       evaluator._minimum_noise, [task] * len(wave), stats)
    jobs = [(k, j) for k, i in enumerate(wave) for j in users[i]]
    idx = np.array([k for k, _ in jobs], dtype=np.int32)
    prm = np.stack([fitted[k] for k, _ in jobs])
    beta = np.array([prefixes[j].beta for _, j in jobs])
    samples = np.stack([prefixes[j].samples for _, j in jobs])
    res, status = engine.gp_batch_bounds(idx, prm, beta, samples)
    for r, (k, j), st in zip(res, jobs, status):
        out[j] = r
        prefixes[j].failed = bool(st)


# ---- EMMR: both Gaussian processes of every prefix ----------------------------------------------------------------

_EMMR_N_SAMPLES = 2048   # the samples of _compute_standardized_regret_bound that EMMREvaluator.evaluate draws


def _emmr_wave_bytes(t: int, P: int, n_users: int) -> int:
    """Device bytes one complete set of t trials adds to a wave: the rows of both its GPs (t - 1 and t), their loss
    workspace (tpe_gpbatch.cuh: an n x n matrix and three n-vectors above 160 rows), per prefix that uses the set the
    bounds workspace of the first GP (that again, n x 256 doubles of cross covariance) and its samples, and the two
    moments jobs (the loss workspace and three n-vectors of cross covariance, tpe_gpemmr.cuh)."""
    def ws(n: int) -> int:
        return n * n + 3 * n if n > 160 else 0
    rows = (2 * t - 1) * (P + 1)
    loss = ws(t - 1) + ws(t)
    bounds = n_users * (ws(t - 1) + 256 * (t - 1) + _EMMR_N_SAMPLES * P + 4)
    moments = ws(t - 1) + ws(t) + 3 * (2 * t - 1) + 2 * (P + 2) + 24
    return 8 * (rows + loss + bounds + moments + 4 * (P + 2) + 16)


class _EMMRSet:
    """What ``EMMREvaluator.evaluate`` forms from one complete set before its fits (emmr.py:141-186): the data of
    both GPs, the two argmax rows and beta; after the fits, what it reads from them."""

    __slots__ = ("X", "y", "is_categorical", "theta_t_star", "theta_t1_star", "beta", "users", "failed",
                 "mu_t1_theta_t1_star", "mean_t", "var_t", "cov_t")


class _EMMRPrefix:
    """One trial prefix of the EMMR curve: a constant (too few complete trials, or no search space), or a set, its
    own samples, and the stream state just after drawing them."""

    __slots__ = ("value", "set", "samples", "state", "kappa", "failed")


def _prepare_emmr(evaluator: "EMMREvaluator", study, error_evaluator=None):
    """The host pre-pass, in trial order: per prefix what ``EMMREvaluator.evaluate`` does before its fits, with the
    same warnings and the same draws from the evaluator's stream.  With ``error_evaluator`` it is called after each
    prefix, as the reference loop calls it, so that an error evaluator sharing the stream (``MedianErrorEvaluator``
    of this evaluator) draws where it draws there."""
    trial_numbers: list[int] = []
    prefixes: list[_EMMRPrefix] = []
    errors: list[float] = []
    completed: list[FrozenTrial] = []
    rng = evaluator._rng.rng
    direction = study.direction
    last_n = -1
    space = score_vals_raw = cur = None
    for trial in study.trials:
        if trial.state == TrialState.COMPLETE:
            completed.append(trial)
        if not completed:
            continue
        trial_numbers.append(trial.number)
        p = _EMMRPrefix()
        p.value, p.set, p.failed = None, None, False
        t = len(completed)
        if t < evaluator.min_n_trials:
            p.value = sys.float_info.max * MARGIN_FOR_NUMARICAL_STABILITY  # Do not terminate.
        else:
            if t != last_n:
                space = gp_search_space.SearchSpace(intersection_search_space(completed))
                sign = -1 if direction == StudyDirection.MINIMIZE else 1
                score_vals_raw = np.array([tr.value for tr in completed]) * sign
                cur = None
                last_n = t
            if not space.dim:
                optuna_warn(
                    f"{evaluator.__class__.__name__} cannot consider any search space."
                    "Termination will never occur in this study."
                )
                p.value = sys.float_info.max * MARGIN_FOR_NUMARICAL_STABILITY  # Do not terminate.
            else:
                # the reference converts (and warns) at every evaluate, shared set or not
                score_vals = gp.warn_and_convert_inf(score_vals_raw)
                if cur is None:
                    cur = _EMMRSet()
                    cur.X = space.get_normalized_params(completed)
                    cur.y = (score_vals - score_vals.mean()) / max(sys.float_info.min, score_vals.std())
                    cur.is_categorical = space.is_categorical
                    cur.theta_t_star = int(np.argmax(cur.y))
                    cur.theta_t1_star = int(np.argmax(cur.y[:-1]))
                    cur.beta = _get_beta(cur.X.shape[1], t - 1, evaluator._delta)
                    cur.users = []
                    cur.failed = False
                p.set = cur
                cur.users.append(len(prefixes))
                p.samples = space.sample_normalized_params(_EMMR_N_SAMPLES, rng=rng)
                p.state = rng.get_state()
        prefixes.append(p)
        if error_evaluator is not None:
            errors.append(error_evaluator.evaluate(trials=completed, study_direction=direction))
    return trial_numbers, prefixes, errors


def _run_emmr_wave(engine, evaluator, sets: list[_EMMRSet], wave: list[int], prefixes, stats) -> None:
    """Fits both GPs of every set of one wave in lock step (GP 2k over the first t - 1 trials of set k, GP 2k + 1 over
    all t, warm-started from the first), then every prefix's kappa in one bounds launch and every set's posterior
    terms in one moments launch."""
    P = sets[wave[0]].X.shape[1]
    minimum_noise = prior.DEFAULT_MINIMUM_NOISE_VAR
    det = evaluator._deterministic

    def task(k: int):
        def fit_both(slot: _Slot):
            slot.gp = 2 * k
            params_t1 = _fit(slot, P, prior.default_log_prior, minimum_noise, deterministic_objective=det,
                             single_blas=False)
            slot.gp = 2 * k + 1
            params_t = _fit(slot, P, prior.default_log_prior, minimum_noise, gpr_cache=params_t1,
                            deterministic_objective=det, single_blas=False)
            return params_t1, params_t
        return fit_both

    data = []
    for i in wave:
        s = sets[i]
        data += [(s.X[:-1], s.y[:-1]), (s.X, s.y)]
    fitted = _fit_wave(engine, data, sets[wave[0]].is_categorical, minimum_noise,
                       [task(k) for k in range(len(wave))], stats, deterministic=det)

    # kappa of every prefix: the regret bound of the first GP over its train rows and the prefix's samples
    jobs = [(k, j) for k, i in enumerate(wave) for j in sets[i].users]
    res, status = engine.gp_batch_bounds(np.array([2 * k for k, _ in jobs], dtype=np.int32),
                                         np.stack([fitted[k][0] for k, _ in jobs]),
                                         np.array([sets[wave[k]].beta for k, _ in jobs]),
                                         np.stack([prefixes[j].samples for _, j in jobs]))
    for r, (_, j), st in zip(res, jobs, status):
        prefixes[j].kappa = max(r[0], r[1]) - r[2]
        prefixes[j].failed = bool(st)
    # the first GP at theta*_{t-1}; the second at theta*_t, theta*_{t-1} and x_t, with the joint covariance of the
    # first two
    idx, prm, rows = [], [], []
    for k, i in enumerate(wave):
        s = sets[i]
        idx += [2 * k, 2 * k + 1]
        prm += [fitted[k][0], fitted[k][1]]
        rows += [[s.theta_t1_star] * 3, [s.theta_t_star, s.theta_t1_star, s.X.shape[0] - 1]]
    mean, var, cov, status = engine.gp_batch_moments(np.array(idx, dtype=np.int32), np.stack(prm),
                                                     np.array(rows, dtype=np.int32), 2)
    for k, i in enumerate(wave):
        s = sets[i]
        s.failed = bool(status[2 * k] or status[2 * k + 1])
        s.mu_t1_theta_t1_star = float(mean[2 * k, 0])
        s.mean_t, s.var_t, s.cov_t = mean[2 * k + 1], var[2 * k + 1], cov[2 * k + 1]


def _batched_emmr(evaluator: "EMMREvaluator", study, error_evaluator=None,
                  stats: dict | None = None) -> tuple[list, list, list]:
    """``_get_improvement_info``'s walk with ``EMMREvaluator.evaluate`` at every prefix: the pre-pass, both fits of
    every distinct complete set in lock step, then the closing arithmetic per prefix."""
    trial_numbers, prefixes, errors = _prepare_emmr(evaluator, study, error_evaluator)
    sets: list[_EMMRSet] = []
    for p in prefixes:
        if p.set is not None and (not sets or p.set is not sets[-1]):
            sets.append(p.set)
    if sets:
        units = [(s.X.shape[1], _emmr_wave_bytes(s.X.shape[0], s.X.shape[1], len(s.users))) for s in sets]
        _in_waves(evaluator._device, units,
                  lambda engine, wave: _run_emmr_wave(engine, evaluator, sets, wave, prefixes, stats), stats)
    improvements = []
    for p in prefixes:
        if p.set is None:
            improvements.append(p.value)
            continue
        if p.failed or p.set.failed:
            # the per-prefix evaluator raises after drawing this prefix's samples (between its two fits)
            evaluator._rng.rng.set_state(p.state)
            raise np.linalg.LinAlgError("Matrix is not positive definite")
        s = p.set
        # emmr.py:249-250: for one point the reference takes the variance of the non-joint posterior
        cov_t_between = float(s.var_t[0] if s.theta_t_star == s.theta_t1_star else s.cov_t[0, 1])
        improvements.append(_emmr_criterion(p.kappa, s.mu_t1_theta_t1_star, s.mean_t, s.var_t, cov_t_between,
                                            s.y[-1]))
    return trial_numbers, improvements, errors


def terminator_improvement_history(study, improvement_evaluator=None, error_evaluator=None, get_error: bool = False):
    """The terminator's improvement after every trial of ``study``: what
    ``optuna.visualization._terminator_improvement._get_improvement_info`` returns, with the same trial walk, the
    same arguments and the same errors.

    With the default evaluator, or an evaluator whose type is exactly ``optuna_b200.RegretBoundEvaluator``, the
    Gaussian processes of every trial prefix are fitted together: the host forms each prefix's data and draws its
    samples from the evaluator's stream in the reference's order, then one device launch per L-BFGS-B round
    evaluates every live fit (``tpe_gp_batch_loss``) and one more gives every prefix's bounds.  Error evaluators are
    then called per prefix.

    With an evaluator whose type is exactly ``optuna_b200.EMMREvaluator``, both Gaussian processes of every prefix
    (over all complete trials but the last, then over all of them, warm-started from the first) are fitted in lock
    step: the host forms each prefix's data, emits the reference's warnings and draws its samples in trial order, one
    launch per L-BFGS-B round evaluates every live fit of either kind (``tpe_gp_batch_loss``, or
    ``tpe_gp_batch_loss_fixed_noise`` with ``deterministic_objective``), then one bounds launch gives every prefix's
    regret bound and one moments launch (``tpe_gp_batch_moments``) every posterior term the criterion reads.  The
    error evaluator is called after each prefix's draws, as the reference loop calls it, so that a
    ``MedianErrorEvaluator`` paired with the same evaluator draws from the shared stream where it draws there.

    Any other improvement evaluator (optuna's own, or a subclass of these) takes optuna's per-prefix loop
    unchanged."""
    from optuna.terminator import CrossValidationErrorEvaluator, StaticErrorEvaluator
    from optuna.terminator.improvement.evaluator import BestValueStagnationEvaluator
    from optuna.visualization._terminator_improvement import _get_improvement_info, _ImprovementInfo

    if study._is_multi_objective():
        raise ValueError("This function does not support multi-objective optimization study.")
    if improvement_evaluator is None:
        improvement_evaluator = RegretBoundEvaluator()
    if error_evaluator is None:
        if isinstance(improvement_evaluator, BestValueStagnationEvaluator):
            error_evaluator = StaticErrorEvaluator(constant=0)
        else:
            error_evaluator = CrossValidationErrorEvaluator()
    if type(improvement_evaluator) is EMMREvaluator:
        trial_numbers, improvements, errors = _batched_emmr(improvement_evaluator, study,
                                                            error_evaluator if get_error else None)
        return _ImprovementInfo(trial_numbers=trial_numbers, improvements=improvements, errors=errors or None)
    if type(improvement_evaluator) is not RegretBoundEvaluator:
        return _get_improvement_info(study, get_error, improvement_evaluator, error_evaluator)
    trial_numbers, improvements = _batched_improvements(improvement_evaluator, study)
    errors = []
    if get_error:
        completed: list[FrozenTrial] = []
        for trial in study.trials:
            if trial.state == TrialState.COMPLETE:
                completed.append(trial)
            if not completed:
                continue
            errors.append(error_evaluator.evaluate(trials=completed, study_direction=study.direction))
    return _ImprovementInfo(trial_numbers=trial_numbers, improvements=improvements, errors=errors or None)
