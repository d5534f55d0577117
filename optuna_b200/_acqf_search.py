"""GPSampler's acquisition search with every live local search evaluated in one call per round.

A restatement of optuna's ``optimize_acqf_mixed`` and ``local_search_mixed_batched`` (optuna/_gp/optim_mixed.py:
232-329), step for step: the same random-stream consumption, the same start points, the same scipy L-BFGS-B and Brent
runs per start point with the same arguments, the same exhaustive steps and the same log warnings.  What changes is
how the acquisition is evaluated:
- L-BFGS-B (``_gradient_ascent_batched``, :29-94): each start point runs ``fmin_l_bfgs_b`` with ``batched_lbfgsb``'s
  arguments in a thread of its own, and each round of evaluations across the live runs is one call (optuna's greenlet
  path, batched_lbfgsb.py:34-86, on threads; ``terminator._LockStep``);
- exhaustive steps (:97-118): the neighbour sets of all start points in one call;
- line searches (:121-186): optuna's own ``_discrete_line_search`` per start point, each in a thread, one call per
  round of their evaluations.
Each search's trajectory depends only on the values of its own rows.  With an evaluation whose rows do not depend on
the rest of the batch (``TPEEngine.acqf_eval``), the result is the bits of optuna's sequential run, and of its
greenlet run.

``evaluate(x, grad)`` answers the acquisition at the rows of ``x`` [k, dim]: the values [k], and with ``grad`` also
their gradient in x [k, dim].
"""
from __future__ import annotations

import math
import threading

import numpy as np
import scipy.optimize as so
from optuna._gp import optim_mixed
from optuna._gp.scipy_blas_thread_patch import single_blas_thread_if_scipy_v1_15_or_newer

from .terminator import _LockStep

# optuna/_gp/optim_mixed.py:199
_MAX_INT_EXHAUSTIVE_SEARCH_PARAMS = 16


def _run_lockstep(evaluate_posted, tasks: list) -> list:
    """Runs ``tasks[k](post)`` for every k, each in its own thread, in lock step: ``post(payload)`` blocks until the
    round's ``evaluate_posted(payloads)`` answers it.  Returns the tasks' results in order; an exception of a task is
    re-raised, the first task's first."""
    ls = _LockStep(evaluate_posted)
    results: dict[int, object] = {}
    errors: dict[int, BaseException] = {}

    def work(k: int) -> None:
        try:
            results[k] = tasks[k](lambda payload: ls.post(k, payload))
        except BaseException as e:   # re-raised below, in task order
            errors[k] = e
        finally:
            ls.leave(k)

    threads = []
    for k in range(len(tasks)):
        ls.join(k)
        threads.append(threading.Thread(target=work, args=(k,), daemon=True))
    ls.run(threads)
    for th in threads:
        th.join()
    if errors:
        raise errors[min(errors)]
    return [results[k] for k in range(len(tasks))]


def _gradient_ascent_lockstep(evaluate, initial_params_batched: np.ndarray, initial_fvals: np.ndarray,
                              continuous_indices: np.ndarray, lengthscales: np.ndarray,
                              tol: float) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """``_gradient_ascent_batched`` (optim_mixed.py:29-94) with the L-BFGS-B runs in lock step."""
    assert initial_params_batched.ndim == 2
    if len(continuous_indices) == 0:
        return initial_params_batched, initial_fvals, np.zeros(len(initial_fvals), dtype=bool)

    def evaluate_posted(rows: list) -> list:
        fvals, grads = evaluate(np.stack(rows), True)
        return [(fvals[i], grads[i]) for i in range(len(rows))]

    x0_batched = initial_params_batched[:, continuous_indices] / lengthscales
    fixed = [param for param in initial_params_batched.copy()]
    bounds = [(0, 1 / s) for s in lengthscales]

    def task(i: int):
        def run(post):
            def func_and_grad(scaled_x: np.ndarray, fixed_params: np.ndarray) -> tuple[float, np.ndarray]:
                # batched_lbfgsb's wrapper around negative_acqf_with_grad for one row: scipy minimises -acqf, whose
                # gradient in the scaled point is -dacqf/dx * lengthscale
                next_params = np.array(fixed_params)
                next_params[continuous_indices] = scaled_x * lengthscales
                fval, grad = post(next_params)
                return float(-fval), (-grad)[continuous_indices] * lengthscales

            x_opt, fval_opt, info = so.fmin_l_bfgs_b(func=func_and_grad, x0=x0_batched[i], args=(fixed[i],),
                                                     bounds=bounds, m=10, factr=1e7, pgtol=math.sqrt(tol),
                                                     maxfun=15000, maxiter=200, maxls=20)
            return x_opt, fval_opt, info["nit"]
        return run

    with single_blas_thread_if_scipy_v1_15_or_newer():
        runs = _run_lockstep(evaluate_posted, [task(i) for i in range(len(x0_batched))])
    scaled_cont_xs_opt = np.empty_like(x0_batched)
    neg_fvals_opt = np.empty(len(x0_batched), dtype=float)
    n_iterations = np.empty(len(x0_batched), dtype=int)
    for i, (x_opt, fval_opt, nit) in enumerate(runs):
        scaled_cont_xs_opt[i], neg_fvals_opt[i], n_iterations[i] = x_opt, fval_opt, nit

    xs_opt = initial_params_batched.copy()
    xs_opt[:, continuous_indices] = scaled_cont_xs_opt * lengthscales
    fvals_opt = -neg_fvals_opt
    is_updated_batch = (fvals_opt > initial_fvals) & (n_iterations > 0)
    return (
        np.where(is_updated_batch[:, None], xs_opt, initial_params_batched),
        np.where(is_updated_batch, fvals_opt, initial_fvals),
        is_updated_batch,
    )


def _exhaustive_search_batched(evaluate, initial_params_batched: np.ndarray, initial_fvals: np.ndarray,
                               param_idx: int, choices: np.ndarray) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """``_exhaustive_search`` (optim_mixed.py:97-118) for every start point, the neighbour sets in one call."""
    best_xs = initial_params_batched.copy()
    best_fvals = initial_fvals.copy()
    is_updated = np.zeros(len(initial_fvals), dtype=bool)
    if len(choices) == 1:
        return best_xs, best_fvals, is_updated
    sets = []
    for params in initial_params_batched:
        others = choices[choices != params[param_idx]]
        all_params = np.repeat(params[None, :], len(others), axis=0)
        all_params[:, param_idx] = others
        sets.append(all_params)
    fvals_all = evaluate(np.concatenate(sets), False)
    at = 0
    for b, all_params in enumerate(sets):
        fvals = fvals_all[at:at + len(all_params)]
        at += len(all_params)
        best_idx = np.argmax(fvals)
        if fvals[best_idx] > initial_fvals[b]:
            best_xs[b], best_fvals[b], is_updated[b] = all_params[best_idx, :], fvals[best_idx], True
    return best_xs, best_fvals, is_updated


class _PostedAcqf:
    """What ``_discrete_line_search`` reads of its acquisition function: ``eval_acqf_no_grad`` of one row, answered
    by the lock-step round."""

    def __init__(self, post) -> None:
        self._post = post

    def eval_acqf_no_grad(self, x: np.ndarray) -> np.ndarray:
        return self._post(np.array(x))


def _line_search_lockstep(evaluate, initial_params_batched: np.ndarray, initial_fvals: np.ndarray, param_idx: int,
                          grids: np.ndarray, xtol: float) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """optuna's ``_discrete_line_search`` (optim_mixed.py:121-186) for every start point, in lock step."""
    def evaluate_posted(rows: list) -> list:
        return list(evaluate(np.stack(rows), False))

    def task(b: int):
        return lambda post: optim_mixed._discrete_line_search(_PostedAcqf(post), initial_params_batched[b],
                                                               initial_fvals[b], param_idx, grids, xtol)

    runs = _run_lockstep(evaluate_posted, [task(b) for b in range(len(initial_fvals))])
    best_xs = initial_params_batched.copy()
    best_fvals = initial_fvals.copy()
    is_updated = np.zeros(len(initial_fvals), dtype=bool)
    for b, (params, fval, updated) in enumerate(runs):
        best_xs[b], best_fvals[b], is_updated[b] = params, fval, updated
    return best_xs, best_fvals, is_updated


def _local_search_mixed(acqf, evaluate, xs0: np.ndarray, *, tol: float = 1e-4,
                        max_iter: int = 100) -> tuple[np.ndarray, np.ndarray]:
    """``local_search_mixed_batched`` (optim_mixed.py:232-277) over the lock-step steps."""
    lengthscales = acqf.length_scales[(cont_inds := acqf.search_space.continuous_indices)]
    discrete_indices = acqf.search_space.discrete_indices
    choices_of_discrete_params = acqf.search_space.get_choices_of_discrete_params()
    discrete_xtols = [np.min(np.diff(choices), initial=np.inf) / 4 for choices in choices_of_discrete_params]
    best_fvals = evaluate((best_xs := xs0.copy()), False)
    CONTINUOUS = -1
    last_changed_dims = np.full(len(best_xs), CONTINUOUS, dtype=int)
    remaining_inds = np.arange(len(best_xs))
    for _ in range(max_iter):
        best_xs[remaining_inds], best_fvals[remaining_inds], updated = _gradient_ascent_lockstep(
            evaluate, best_xs[remaining_inds], best_fvals[remaining_inds], cont_inds, lengthscales, tol
        )
        last_changed_dims = np.where(updated, CONTINUOUS, last_changed_dims)
        for i, choices, xtol in zip(discrete_indices, choices_of_discrete_params, discrete_xtols):
            last_changed_dims = last_changed_dims[~(is_converged := last_changed_dims == i)]
            remaining_inds = remaining_inds[~is_converged]
            if remaining_inds.size == 0:
                return best_xs, best_fvals
            if acqf.search_space.is_categorical[i] or len(choices) <= _MAX_INT_EXHAUSTIVE_SEARCH_PARAMS:
                step = _exhaustive_search_batched(evaluate, best_xs[remaining_inds], best_fvals[remaining_inds], i,
                                                  choices)
            else:
                step = _line_search_lockstep(evaluate, best_xs[remaining_inds], best_fvals[remaining_inds], i,
                                             choices, xtol)
            best_xs[remaining_inds], best_fvals[remaining_inds], updated = step
            last_changed_dims = np.where(updated, i, last_changed_dims)

        remaining_inds = remaining_inds[~(is_converged := last_changed_dims == CONTINUOUS)]
        last_changed_dims = last_changed_dims[~is_converged]
        if remaining_inds.size == 0:
            return best_xs, best_fvals
    else:
        optim_mixed._logger.warning("local_search_mixed: Local search did not converge.")
    return best_xs, best_fvals


def optimize_acqf_mixed(acqf, evaluate, *, warmstart_normalized_params_array: np.ndarray | None = None,
                        n_preliminary_samples: int = 2048, n_local_search: int = 10, tol: float = 1e-4,
                        rng: np.random.RandomState | None = None) -> tuple[np.ndarray, float]:
    """``optimize_acqf_mixed`` (optim_mixed.py:280-329) with ``acqf``'s values from ``evaluate``.  ``acqf`` gives
    the search space and the length scales."""
    rng = rng or np.random.RandomState()

    if warmstart_normalized_params_array is None:
        warmstart_normalized_params_array = np.empty((0, acqf.search_space.dim))

    assert len(warmstart_normalized_params_array) <= n_local_search - 1, (
        "We must choose at least 1 best sampled point + given_initial_xs as start points."
    )

    sampled_xs = acqf.search_space.sample_normalized_params(n_preliminary_samples, rng=rng)
    f_vals = evaluate(sampled_xs, False)
    max_i = np.argmax(f_vals)

    probs = np.exp(f_vals - f_vals[max_i])
    probs[max_i] = 0.0
    probs /= probs.sum()
    n_non_zero_probs_improvement = int(np.count_nonzero(probs > 0.0))
    n_additional_warmstart = min(
        n_local_search - len(warmstart_normalized_params_array) - 1, n_non_zero_probs_improvement
    )
    if n_additional_warmstart == n_non_zero_probs_improvement:
        optim_mixed._logger.warning("Study already converged, so the number of local search is reduced.")
    chosen_idxs = np.array([max_i])
    if n_additional_warmstart > 0:
        additional_idxs = rng.choice(len(sampled_xs), size=n_additional_warmstart, replace=False, p=probs)
        chosen_idxs = np.append(chosen_idxs, additional_idxs)

    x_warmstarts = np.vstack([sampled_xs[chosen_idxs, :], warmstart_normalized_params_array])
    best_xs, best_fvals = _local_search_mixed(acqf, evaluate, x_warmstarts, tol=tol)
    best_idx = np.argmax(best_fvals).item()
    return best_xs[best_idx], best_fvals[best_idx]
