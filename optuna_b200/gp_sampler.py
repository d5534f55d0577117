"""optuna's Bayesian-optimisation sampler with its Gaussian processes on the GPU: a drop-in ``GPSampler``.

``optuna.samplers.GPSampler`` does two costly things per trial (optuna/samplers/_gp/sampler.py:358-485):
- it fits one Gaussian process per objective and one per constraint by L-BFGS-B over the kernel parameters; every
  loss evaluation builds an n x n x P tensor and runs autograd through a Cholesky factor (optuna/_gp/gp.py:287-409);
- it maximises the acquisition function (optuna/_gp/optim_mixed.py): 2 048 QMC points, then up to 10 local searches
  of L-BFGS-B and discrete steps.  Every evaluation calls ``GPRegressor.posterior``, two triangular solves against the
  n x n factor plus torch autograd for the gradient in x.

This sampler subclasses optuna's and keeps every host step: the standardisation, the cache handling, the choice of
starting points, the random stream, optuna's acquisition functions and ``optimize_acqf_mixed``.  The GPs move to the
device.  Each GP is fitted by the terminator's device fit (``terminator._fit``: the loss and its gradient on the
device, scipy's L-BFGS-B and the prior on the host), factorised once, and queried with its posterior and the
posterior's gradient in x against that factor (``TPEEngine.gp_condition`` / ``gp_query``).

With two or more objectives the log-EHVI of ``LogEHVI`` (acqf.py:45-62, 245-300), and of ``ConstrainedLogEHVI``'s
objective part, also runs on the device (``TPEEngine.ehvi_set`` / ``ehvi``): optuna builds a (points, 128 samples,
boxes, objectives) fp64 tensor per evaluation, which at four objectives and a thousand trials is tens of GB.  So does
the non-dominated box decomposition ``LogEHVI.__init__`` computes once per ask (``TPEEngine.box_decomposition``):
optuna's (optuna/_hypervolume/box_decomposition.py) costs seconds to minutes from five objectives on.  The device
returns the reference's boxes bit for bit and in its order, so the acquisition is the one optuna builds.  optuna still
computes the Pareto filter and reference point before the decomposition, the QMC samples and the constraints' ``LogPI``
terms on the host; the other acquisition functions run unchanged over the device GPs.  Beyond 24 objectives optuna's
host ``LogEHVI`` is kept.

The acquisition search is optuna's ``optimize_acqf_mixed`` restated step for step (``_acqf_search``) over a fused
device acquisition (``TPEEngine.acqf_set`` / ``acqf_eval``): the GPs' posteriors, LogEI / LogPI / log-EHVI and the
gradient in x in one call, and every round of the live local searches gathered into that call.  A row's value does
not depend on its batch, so the suggestion is the bits of optuna's own search over the same acquisition.

One difference: the device holds two n x n fp64 matrices per GP and a pool of the decomposition's bounds, and
``sample_relative`` raises ``ValueError`` naming the need when the device lacks that memory.
"""
from __future__ import annotations

import os
import sys
import threading
import warnings
from typing import Any

import numpy as np
import torch
from optuna._gp import acqf as acqf_module
from optuna._gp import search_space as gp_search_space
from optuna._warnings import _OPTUNA_MODULE_ROOT, optuna_warn
from optuna.samplers import GPSampler as _OptunaGPSampler
from optuna.samplers._gp.sampler import EPS, _get_constraint_vals_and_feasibility, _standardize_values
from optuna.study import StudyDirection
from optuna.study._multi_objective import _is_pareto_front

from . import _acqf_search
from .engine import GPCholeskyError, TPEEngine
from .terminator import _fit

# the engine class that answers the computation (tests substitute a host implementation)
_engine_cls = TPEEngine
# objectives the device log-EHVI takes at most (tpe_ehvi_set); beyond, optuna's host LogEHVI runs
_EHVI_MAX_OBJECTIVES = 24


def _answers_ehvi(engine_cls) -> bool:
    """Whether ``engine_cls`` answers the log-EHVI calls (``ehvi_set`` / ``ehvi``) as well as the GP calls.
    ``TPEEngine`` always does: its library refuses to load without the EHVI entry points, so on the device a missing
    kernel is an error.  A substitute engine that restates only the GP calls (a host implementation of them) leaves the
    acquisition to optuna's host ``LogEHVI``, as before the device log-EHVI existed."""
    return callable(getattr(engine_cls, "ehvi_set", None)) and callable(getattr(engine_cls, "ehvi", None))


def _answers_acqf(engine_cls) -> bool:
    """Whether ``engine_cls`` answers the fused acquisition calls (``acqf_set`` / ``acqf_eval``).  ``TPEEngine``
    always does; with a substitute engine without them the acquisition search stays optuna's, over the per-GP
    queries."""
    return callable(getattr(engine_cls, "acqf_set", None)) and callable(getattr(engine_cls, "acqf_eval", None))


def _answers_box_decomposition(engine_cls) -> bool:
    """Whether ``engine_cls`` answers the box decomposition (``box_decomposition``).  ``TPEEngine`` always does; a
    substitute engine without it leaves the decomposition to optuna's host ``LogEHVI``."""
    return callable(getattr(engine_cls, "box_decomposition", None))


_PACKAGE_ROOT = os.path.dirname(os.path.abspath(__file__)) + os.sep
_BOX_DECOMPOSITION_WARNING = ("Box decomposition (typically used by `GPSampler`) might be significantly slow for "
                              "n_objectives > 4. Please consider using another sampler instead.")


def _warn_box_decomposition() -> None:
    """The warning optuna's ``get_non_dominated_box_bounds`` emits for more than four objectives
    (box_decomposition.py:151-155), attributed as ``optuna_warn`` attributes it: to the first frame outside optuna and
    outside this package, so that warning filters match it as they match the reference's."""
    if sys.version_info >= (3, 12):
        warnings.warn(_BOX_DECOMPOSITION_WARNING, UserWarning, skip_file_prefixes=(_OPTUNA_MODULE_ROOT, _PACKAGE_ROOT))
    else:  # pragma: no cover
        optuna_warn(_BOX_DECOMPOSITION_WARNING)


def _condition(engine, params: np.ndarray) -> None:
    try:
        engine.gp_condition(params)
    except GPCholeskyError as e:
        # the reference factorises the final covariance with NumPy (gp.py:132)
        raise np.linalg.LinAlgError("Matrix is not positive definite") from e


class _Posterior(torch.autograd.Function):
    """``GPRegressor.posterior(x)`` (gp.py:215-250) from one device query; the backward is
    ``g_mean dmean/dx + g_var dvar/dx`` with the gradients that query returned."""

    @staticmethod
    def forward(ctx: Any, x: torch.Tensor, gpr: _DeviceGP) -> tuple[torch.Tensor, torch.Tensor]:
        want_grad = ctx.needs_input_grad[0]
        xs = x.detach().cpu().numpy().reshape(-1, x.shape[-1])
        out = gpr._engine.gp_query(xs, grad=want_grad)
        if want_grad:
            ctx.save_for_backward(torch.from_numpy(out[2]).reshape(x.shape), torch.from_numpy(out[3]).reshape(x.shape))
        return torch.from_numpy(out[0]).reshape(x.shape[:-1]), torch.from_numpy(out[1]).reshape(x.shape[:-1])

    @staticmethod
    def backward(ctx: Any, g_mean: torch.Tensor, g_var: torch.Tensor) -> tuple[torch.Tensor, None]:
        dmean, dvar = ctx.saved_tensors
        return g_mean[..., None] * dmean + g_var[..., None] * dvar, None


class _DeviceGP:
    """What optuna's acquisition functions (optuna/_gp/acqf.py) and ``GPSampler`` read of a fitted ``GPRegressor``,
    answered by an engine conditioned at the fitted parameters."""

    def __init__(self, engine, X: np.ndarray, y: np.ndarray, is_categorical: np.ndarray, params: np.ndarray) -> None:
        P = X.shape[1]
        self._engine = engine
        self._X_train, self._is_categorical, self._params = X, is_categorical, params
        self._y_train = torch.from_numpy(y)
        self.inverse_squared_lengthscales = torch.from_numpy(params[:P].copy())
        self.kernel_scale = torch.tensor(params[P], dtype=torch.float64)
        self.noise_var = torch.tensor(params[P + 1], dtype=torch.float64)
        _condition(engine, params)

    @property
    def length_scales(self) -> np.ndarray:
        return 1.0 / np.sqrt(self.inverse_squared_lengthscales.detach().cpu().numpy())

    def append_running_data(self, X_running: torch.Tensor, y_running: torch.Tensor) -> None:
        # gp.py:151-183 extends the factor block-wise; the factor of the stacked train and running rows at the same
        # parameters is of the same matrix
        X = np.concatenate([self._X_train, X_running.detach().cpu().numpy()])
        y = np.concatenate([self._y_train.numpy(), y_running.detach().cpu().numpy()])
        self._engine.gp_set_data(X, y, self._is_categorical)
        _condition(self._engine, self._params)

    def posterior(self, x: torch.Tensor, joint: bool = False) -> tuple[torch.Tensor, torch.Tensor]:
        if joint:
            raise NotImplementedError("GPSampler's acquisition functions do not ask for the joint posterior")
        return _Posterior.apply(x, self)


class _EHVI(torch.autograd.Function):
    """``logehvi`` of the stacked posteriors (acqf.py:45-62, 282-300) from one device call; the backward is
    ``g dvalue/dmean`` and ``g dvalue/dsd`` with the gradients that call returned."""

    @staticmethod
    def forward(ctx: Any, mean: torch.Tensor, sd: torch.Tensor, engine) -> torch.Tensor:
        want_grad = ctx.needs_input_grad[0] or ctx.needs_input_grad[1]
        M = mean.shape[-1]
        m = mean.detach().cpu().numpy().reshape(-1, M)
        s = sd.detach().cpu().numpy().reshape(-1, M)
        out = engine.ehvi(m, s, grad=want_grad)
        if not want_grad:
            return torch.from_numpy(out).reshape(mean.shape[:-1])
        ctx.save_for_backward(torch.from_numpy(out[1]).reshape(mean.shape), torch.from_numpy(out[2]).reshape(sd.shape))
        return torch.from_numpy(out[0]).reshape(mean.shape[:-1])

    @staticmethod
    def backward(ctx: Any, g: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor, None]:
        dmean, dsd = ctx.saved_tensors
        return g[..., None] * dmean, g[..., None] * dsd, None


class _DeviceLogEHVI(acqf_module.BaseAcquisitionFunc):
    """optuna's ``LogEHVI`` (acqf.py:245-300) with its ``logehvi`` on the device.  It takes an already-built host
    ``LogEHVI``, so the box decomposition and the QMC samples are the reference's bits, uploads them to ``engine``
    once, and keeps that object's GPs, stabilising noise, ``length_scales`` and ``search_space``.  ``eval_acqf``
    forms each objective's standard deviation as the reference does and evaluates log-EHVI and its gradient in one
    device call."""

    def __init__(self, host: acqf_module.LogEHVI, engine) -> None:
        self._host = host
        self._gpr_list = host._gpr_list
        self._stabilizing_noise = host._stabilizing_noise
        self._engine = engine
        engine.ehvi_set(host._non_dominated_box_lower_bounds.numpy(), host._non_dominated_box_intervals.numpy(),
                        host._fixed_samples.numpy())
        super().__init__(host.length_scales, host.search_space)

    def eval_acqf(self, x: torch.Tensor) -> torch.Tensor:
        means, sds = [], []
        for gpr in self._gpr_list:
            mean, var = gpr.posterior(x)
            means.append(mean)
            sds.append(torch.sqrt(var + self._stabilizing_noise))
        return _EHVI.apply(torch.stack(means, dim=-1), torch.stack(sds, dim=-1), self._engine)


class _AcqfValue(torch.autograd.Function):
    """``eval_acqf`` from one ``acqf_eval``; the backward is ``g dvalue/dx`` with the gradient that call returned."""

    @staticmethod
    def forward(ctx: Any, x: torch.Tensor, acqf: _DeviceAcqf) -> torch.Tensor:
        want_grad = ctx.needs_input_grad[0]
        xs = x.detach().cpu().numpy().reshape(-1, x.shape[-1])
        out = acqf.evaluate(xs, want_grad)
        if not want_grad:
            return torch.from_numpy(out).reshape(x.shape[:-1])
        ctx.save_for_backward(torch.from_numpy(out[1]).reshape(x.shape))
        return torch.from_numpy(out[0]).reshape(x.shape[:-1])

    @staticmethod
    def backward(ctx: Any, g: torch.Tensor) -> tuple[torch.Tensor, None]:
        (dx,) = ctx.saved_tensors
        return g[..., None] * dx, None


class _DeviceAcqf(acqf_module.BaseAcquisitionFunc):
    """GPSampler's acquisition function (LogEI, ConstrainedLogEI, LogEHVI, ConstrainedLogEHVI) evaluated by one
    ``acqf_eval`` of ``engine`` per call, value and gradient, over the conditioned device GPs of the host object it
    replaces, with that object's thresholds, stabilising noise, boxes, samples, length scales and search space.
    ``calls`` counts the device calls."""

    def __init__(self, engine, kind: int, n_obj: int, gprs: list[_DeviceGP], thresholds: list[float], noise: float,
                 host: acqf_module.BaseAcquisitionFunc, ehvi: acqf_module.LogEHVI | None = None) -> None:
        self._engine = engine
        self.calls = 0
        boxes = {} if ehvi is None else dict(lower=ehvi._non_dominated_box_lower_bounds.numpy(),
                                             intervals=ehvi._non_dominated_box_intervals.numpy(),
                                             samples=ehvi._fixed_samples.numpy())
        engine.acqf_set(kind, [gpr._engine for gpr in gprs], n_obj, thresholds, noise, **boxes)
        super().__init__(host.length_scales, host.search_space)

    @classmethod
    def build(cls, engine, acqf: acqf_module.BaseAcquisitionFunc) -> _DeviceAcqf | None:
        """The device form of the acquisition function ``GPSampler`` built, or None when it has none: optuna's host
        ``LogEHVI`` (beyond 24 objectives, or an engine class without the log-EHVI calls) stays on optuna's path."""
        cons: list = []
        ehvi = None
        if type(acqf) is acqf_module.LogEI:
            kind, objs, thr = TPEEngine.ACQF_LOGEI, [acqf], [acqf._threshold]
        elif type(acqf) is acqf_module.ConstrainedLogEI:
            kind, objs, thr = TPEEngine.ACQF_LOGEI, [acqf._acqf], [acqf._acqf._threshold]
            cons = acqf._constraints_acqf_list
        elif type(acqf) is _DeviceLogEHVI:
            kind, objs, thr, ehvi = TPEEngine.ACQF_LOGEHVI, [acqf], [], acqf._host
        elif type(acqf) is acqf_module.ConstrainedLogEHVI and acqf._acqf is None:
            kind, objs, thr = TPEEngine.ACQF_LOGPI, [], []
            cons = acqf._constraints_acqf_list
        elif type(acqf) is acqf_module.ConstrainedLogEHVI and type(acqf._acqf) is _DeviceLogEHVI:
            kind, objs, thr, ehvi = TPEEngine.ACQF_LOGEHVI, [acqf._acqf], [], acqf._acqf._host
            cons = acqf._constraints_acqf_list
        else:
            return None
        gprs = [o._gpr for o in objs if hasattr(o, "_gpr")] + [g for o in objs for g in getattr(o, "_gpr_list", [])]
        gprs += [c._gpr for c in cons]
        thr = thr + [0.0] * (len(gprs) - len(cons) - len(thr)) + [c._threshold for c in cons]
        noises = {o._stabilizing_noise for o in objs + cons}
        if len(noises) != 1 or not all(isinstance(g, _DeviceGP) for g in gprs):
            return None
        n_obj = len(gprs) - len(cons)
        return cls(engine, kind, n_obj, gprs, [float(t) for t in thr], noises.pop(), acqf, ehvi)

    def evaluate(self, x: np.ndarray, grad: bool):
        self.calls += 1
        return self._engine.acqf_eval(x, grad=grad)

    def eval_acqf(self, x: torch.Tensor) -> torch.Tensor:
        return _AcqfValue.apply(x, self)


class GPSampler(_OptunaGPSampler):
    """Gaussian-process Bayesian-optimisation sampler whose Gaussian processes are fitted and queried on the GPU.

    A drop-in for ``optuna.samplers.GPSampler`` with the same arguments and ``device``.  For the same seed and history
    it consumes the random stream as the reference does and suggests the reference's parameters, up to the rounding
    of the device's fp64 sums.  Its engines (one per objective and per constraint) are kept across trials; ``close``
    frees them.  Under ``study.optimize(n_jobs > 1)`` the relative sampling of concurrent trials runs one at a time,
    since the trials share those engines.

    With 2 to 24 objectives the log-EHVI acquisition (with constraints, its hypervolume part) is also evaluated on
    the device, by one more engine kept across trials, which also computes the acquisition's non-dominated box
    decomposition: the reference's boxes, bit for bit.  optuna's other acquisition functions run unchanged over the
    device GPs.

    The device holds two n x n fp64 matrices per GP, n being the number of complete trials (plus the running ones in a
    single-objective study without constraints), and the bounds of the box decomposition.  When it lacks that memory,
    ``sample_relative`` raises ``ValueError`` naming the need; this is the one difference from the reference.

    Args:
        seed: Random seed.
        independent_sampler: Sampler for the startup trials and for conditional parameters.
        n_startup_trials: Number of initial trials.
        deterministic_objective: Whether the objective function is deterministic (the GP noise is then fixed at its
            minimum).
        constraints_func: A function that computes the constraints of a trial.
        warn_independent_sampling: Whether to warn when a parameter is sampled by the independent sampler.
        device: CUDA device to compute on.
    """

    def __init__(self, *, seed: int | None = None, independent_sampler=None, n_startup_trials: int = 10,
                 deterministic_objective: bool = False, constraints_func=None, warn_independent_sampling: bool = True,
                 device: int = 0) -> None:
        super().__init__(seed=seed, independent_sampler=independent_sampler, n_startup_trials=n_startup_trials,
                         deterministic_objective=deterministic_objective, constraints_func=constraints_func,
                         warn_independent_sampling=warn_independent_sampling)
        self._device = device
        self._engines: list = []   # one per GP: the objectives', then the constraints'
        self._ehvi_engine = None   # the log-EHVI acquisition's, created on the first multi-objective ask
        self._acqf_engine = None   # the fused acquisition's (acqf_set / acqf_eval), created on the first search
        # study.optimize(n_jobs > 1) samples on several threads, and a trial's fits, conditioning and queries on the
        # shared engines must not interleave with another trial's
        self._lock = threading.RLock()

    def close(self) -> None:
        with self._lock:
            for engine in self._engines:
                engine.close()
            self._engines = []
            if self._ehvi_engine is not None:
                self._ehvi_engine.close()
                self._ehvi_engine = None
            if self._acqf_engine is not None:
                self._acqf_engine.close()
                self._acqf_engine = None

    def __del__(self) -> None:  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass

    def _fit_gp(self, k: int, X: np.ndarray, y: np.ndarray, is_categorical: np.ndarray,
                cache: _DeviceGP | None) -> _DeviceGP:
        """``gp.fit_kernel_params`` (gp.py:354-409) on engine ``k``, warm-started from ``cache``'s parameters."""
        while len(self._engines) <= k:
            self._engines.append(_engine_cls(self._device))
        engine = self._engines[k]
        engine.gp_set_data(X, y, is_categorical)
        params = _fit(engine, X.shape[1], self._log_prior, self._minimum_noise,
                      None if cache is None else cache._params, self._deterministic)
        return _DeviceGP(engine, X, y, is_categorical, params)

    def _device_ehvi(self, host: acqf_module.LogEHVI) -> acqf_module.BaseAcquisitionFunc:
        """``host`` with its log-EHVI on the device, or ``host`` itself beyond the device's 24 objectives or when the
        engine class answers only the GP calls (``_answers_ehvi``)."""
        if host._fixed_samples.shape[-1] > _EHVI_MAX_OBJECTIVES or not _answers_ehvi(_engine_cls):
            return host
        if self._ehvi_engine is None:
            self._ehvi_engine = _engine_cls(self._device)
        return _DeviceLogEHVI(host, self._ehvi_engine)

    def _log_ehvi(self, gpr_list: list[_DeviceGP], search_space: gp_search_space.SearchSpace, Y_train: np.ndarray,
                  qmc_seed: int) -> acqf_module.BaseAcquisitionFunc:
        """``LogEHVI(gpr_list, search_space, Y_train, 128, qmc_seed)`` through ``_device_ehvi``.  When the engine class
        answers the box decomposition and the EHVI calls and there are at most 24 objectives, the ``LogEHVI`` is built
        as acqf.py:255-280 builds it, with the decomposition on the device: the same Pareto filter and reference point
        on the host, the device's boxes flipped back to maximisation, the same clamp, samples and length scales."""
        M = Y_train.shape[-1]
        if M > _EHVI_MAX_OBJECTIVES or not (_answers_ehvi(_engine_cls) and _answers_box_decomposition(_engine_cls)):
            return self._device_ehvi(acqf_module.LogEHVI(gpr_list=gpr_list, search_space=search_space,
                                                         Y_train=torch.from_numpy(Y_train), n_qmc_samples=128,
                                                         qmc_seed=qmc_seed))
        if self._ehvi_engine is None:
            self._ehvi_engine = _engine_cls(self._device)
        host = acqf_module.LogEHVI.__new__(acqf_module.LogEHVI)
        host._stabilizing_noise = 1e-12
        host._gpr_list = gpr_list
        host._fixed_samples = acqf_module._sample_from_normal_sobol(dim=M, n_samples=128, seed=qmc_seed)
        # acqf.py:257-263: Y is maximised, loss_vals minimised
        loss_vals = -Y_train
        pareto_sols = loss_vals[_is_pareto_front(loss_vals, assume_unique_lexsorted=False)]
        ref_point = np.max(loss_vals, axis=0)
        ref_point = np.nextafter(np.maximum(1.1 * ref_point, 0.9 * ref_point), np.inf)
        if M > 4:
            _warn_box_decomposition()
        lbs, ubs = self._ehvi_engine.box_decomposition(pareto_sols, ref_point)
        host._non_dominated_box_lower_bounds = torch.from_numpy(-ubs)
        upper = torch.from_numpy(-lbs)
        host._non_dominated_box_intervals = (upper - host._non_dominated_box_lower_bounds).clamp_min_(acqf_module._EPS)
        acqf_module.BaseAcquisitionFunc.__init__(host, np.mean([gpr.length_scales for gpr in gpr_list], axis=0),
                                                 search_space)
        return self._device_ehvi(host)

    def _optimize_acqf(self, acqf: acqf_module.BaseAcquisitionFunc, best_params: np.ndarray | None) -> np.ndarray:
        """optuna's ``_optimize_acqf`` (optuna/samplers/_gp/sampler.py:237-252).  When the engine class answers the
        fused acquisition calls (``_answers_acqf``), ``optimize_acqf_mixed`` runs as ``_acqf_search`` restates it
        over the device acquisition (``_DeviceAcqf``): every round of the live local searches is one device call, and
        the suggestion is the bits optuna's own search over that acquisition returns.  Otherwise, and for optuna's
        host ``LogEHVI``, optuna's search runs unchanged."""
        device = None
        if _answers_acqf(_engine_cls):
            if self._acqf_engine is None:
                self._acqf_engine = _engine_cls(self._device)
            device = _DeviceAcqf.build(self._acqf_engine, acqf)
        if device is None:
            return super()._optimize_acqf(acqf, best_params)
        assert best_params is None or len(best_params.shape) == 2
        normalized_params, _acqf_val = _acqf_search.optimize_acqf_mixed(
            device, device.evaluate, warmstart_normalized_params_array=best_params,
            n_preliminary_samples=self._n_preliminary_samples, n_local_search=self._n_local_search, tol=self._tol,
            rng=self._rng.rng)
        self.last_acqf_calls = device.calls
        return normalized_params

    def _get_constraints_acqf_args(self, constraint_vals: np.ndarray,
                                   internal_search_space: gp_search_space.SearchSpace,
                                   normalized_params: np.ndarray) -> tuple[list[_DeviceGP], list[float]]:
        # optuna/samplers/_gp/sampler.py:254-292, with the fits on the device
        standardized_constraint_vals, means, stds = _standardize_values(-constraint_vals)
        if (
            self._gprs_cache_list is not None
            and len(self._gprs_cache_list[0].inverse_squared_lengthscales) != internal_search_space.dim
        ):
            self._constraints_gprs_cache_list = None

        is_categorical = internal_search_space.is_categorical
        constraints_threshold_list = (-means / np.maximum(EPS, stds)).tolist()
        first = len(self._gprs_cache_list)   # the objectives' engines come first
        constraints_gprs = []
        for i, vals in enumerate(standardized_constraint_vals.T):
            cache = self._constraints_gprs_cache_list[i] if self._constraints_gprs_cache_list is not None else None
            constraints_gprs.append(self._fit_gp(first + i, normalized_params, vals, is_categorical, cache))

        self._constraints_gprs_cache_list = constraints_gprs
        return constraints_gprs, constraints_threshold_list

    def _sample_relative_impl(self, study, completed_trials, trials, search_space) -> dict[str, Any]:
        with self._lock:
            return self._sample_relative_locked(study, completed_trials, trials, search_space)

    def _sample_relative_locked(self, study, completed_trials, trials, search_space) -> dict[str, Any]:
        # optuna/samplers/_gp/sampler.py:358-485, with the fits on the device
        internal_search_space = gp_search_space.SearchSpace(search_space)
        normalized_params = internal_search_space.get_normalized_params(completed_trials)

        _sign = np.array([-1.0 if d == StudyDirection.MINIMIZE else 1.0 for d in study.directions])
        standardized_score_vals, _, _ = _standardize_values(
            _sign * np.array([trial.values for trial in completed_trials])
        )

        if (
            self._gprs_cache_list is not None
            and len(self._gprs_cache_list[0].inverse_squared_lengthscales) != internal_search_space.dim
        ):
            self._gprs_cache_list = None

        gprs_list = []
        n_objectives = standardized_score_vals.shape[-1]
        is_categorical = internal_search_space.is_categorical
        for i in range(n_objectives):
            cache = self._gprs_cache_list[i] if self._gprs_cache_list is not None else None
            gprs_list.append(self._fit_gp(i, normalized_params, standardized_score_vals[:, i], is_categorical, cache))
        self._gprs_cache_list = gprs_list

        best_params: np.ndarray | None
        acqf: acqf_module.BaseAcquisitionFunc
        if self._constraints_func is None:
            if n_objectives == 1:
                acqf = acqf_module.LogEI(
                    gpr=gprs_list[0],
                    search_space=internal_search_space,
                    threshold=standardized_score_vals[:, 0].max(),
                    normalized_params_of_running_trials=(
                        self._get_normalized_params_of_running_trials(trials, internal_search_space)
                    ),
                )
                best_params = normalized_params[np.argmax(standardized_score_vals), np.newaxis]
            else:
                acqf = self._log_ehvi(gprs_list, internal_search_space, standardized_score_vals,
                                      self._rng.rng.randint(1 << 30))
                best_params = self._get_best_params_for_multi_objective(normalized_params, standardized_score_vals)
        else:
            constraint_vals, is_feasible = _get_constraint_vals_and_feasibility(study, completed_trials)
            constr_gpr_list, constr_threshold_list = self._get_constraints_acqf_args(
                constraint_vals, internal_search_space, normalized_params
            )
            if n_objectives == 1:
                y_with_neginf = np.where(is_feasible, standardized_score_vals[:, 0], -np.inf)
                i_opt = np.argmax(y_with_neginf)
                best_feasible_y = y_with_neginf[i_opt]
                acqf = acqf_module.ConstrainedLogEI(
                    gpr=gprs_list[0],
                    search_space=internal_search_space,
                    threshold=best_feasible_y,
                    constraints_gpr_list=constr_gpr_list,
                    constraints_threshold_list=constr_threshold_list,
                )
                best_params = None if np.isneginf(best_feasible_y) else normalized_params[i_opt, np.newaxis]
            else:
                is_all_infeasible = not any(is_feasible)
                qmc_seed = self._rng.rng.randint(1 << 30)
                # built without its LogEHVI, which _log_ehvi builds as ConstrainedLogEHVI would (acqf.py:318-322)
                acqf = acqf_module.ConstrainedLogEHVI(
                    gpr_list=gprs_list,
                    search_space=internal_search_space,
                    Y_feasible=None,
                    n_qmc_samples=128,
                    qmc_seed=qmc_seed,
                    constraints_gpr_list=constr_gpr_list,
                    constraints_threshold_list=constr_threshold_list,
                )
                if not is_all_infeasible:   # else the LogPI terms alone
                    acqf._acqf = self._log_ehvi(gprs_list, internal_search_space,
                                                standardized_score_vals[is_feasible], qmc_seed)
                best_params = (
                    self._get_best_params_for_multi_objective(
                        normalized_params[is_feasible], standardized_score_vals[is_feasible]
                    )
                    if not is_all_infeasible
                    else None
                )

        normalized_param = self._optimize_acqf(acqf, best_params)
        return internal_search_space.get_unnormalized_param(normalized_param)
