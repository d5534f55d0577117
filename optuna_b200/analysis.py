"""Study analysis on the GPU: the hypervolume history and the Pareto front of a multi-objective study.

``hypervolume_history`` returns what optuna's ``_get_hypervolume_history_info``
(optuna/visualization/_hypervolume_history.py:83-138) returns, computed by ``tpe_hypervolume_history``
(optuna_b200/csrc/tpe_hvhist.cuh); ``plot_hypervolume_history`` is the drop-in for
``optuna.visualization.plot_hypervolume_history`` and draws with optuna's own plot code.

``best_trials`` is the drop-in for ``Study.best_trials`` (optuna/study/study.py:158-175), ``pareto_front_info``
returns what ``_get_pareto_front_info`` (optuna/visualization/_pareto_front.py:177-328) returns and
``plot_pareto_front`` is the drop-in for ``optuna.visualization.plot_pareto_front``; the front is computed by
``tpe_pareto_front`` (optuna_b200/csrc/tpe_pareto.cuh).
"""
from __future__ import annotations

import copy
from collections.abc import Sequence as _SequenceABC
from typing import Callable, Sequence

import numpy as np

from ._compat import CONSTRAINTS_KEY, StudyDirection, TrialState, get_logger
from .engine import TPEEngine

from optuna.visualization._hypervolume_history import _get_hypervolume_history_plot, _HypervolumeHistoryInfo  # noqa: I001

_logger = get_logger("optuna.visualization.optuna_b200")  # a child of optuna's root logger: same handlers / verbosity

# the engine class that answers the computation (tests substitute a host implementation)
_engine_cls = TPEEngine


def hypervolume_history(study, reference_point: Sequence[float], *, device: int = 0) -> _HypervolumeHistoryInfo:
    """Hypervolume of the feasible COMPLETE trials after each of them, in trial order.

    Returns ``(trial_numbers, values)`` as ``_get_hypervolume_history_info`` does, with the same trial walk, the
    same constraint test and the same errors and warnings.  Raises ``ValueError`` for a single-objective study, a
    reference point whose dimension is not the number of objectives, and a reference point holding NaN.  The
    reference raises on a NaN reference point only once it reaches the second feasible trial inside the box
    (optuna/_hypervolume/wfg.py:144); here it is rejected before any work.  Objective values holding NaN are
    rejected the same way.

    Args:
        study: a multi-objective ``optuna.Study``.
        reference_point: the reference point, one coordinate per objective, in the objectives' own directions.
        device: CUDA device to compute on.
    """
    if not study._is_multi_objective():
        raise ValueError(
            "Study must be multi-objective. For single-objective optimization, "
            "please use plot_optimization_history instead."
        )
    if len(reference_point) != len(study.directions):
        raise ValueError(
            "The dimension of the reference point must be the same as the number of objectives."
        )
    ref = np.asarray(reference_point, dtype=np.float64)
    if np.isnan(ref).any():
        raise ValueError("The reference point must not contain NaN.")

    trials = study.get_trials(deepcopy=False, states=(TrialState.COMPLETE,))
    if len(trials) == 0:
        _logger.warning("Your study does not have any completed trials.")

    signs = np.asarray([1 if d == StudyDirection.MINIMIZE else -1 for d in study.directions])
    M = signs.size
    values = np.asarray([t.values for t in trials], dtype=np.float64).reshape(len(trials), M) * signs
    ref = signs * ref
    feasible = np.asarray([not (CONSTRAINTS_KEY in t.system_attrs
                                and any(c > 0.0 for c in t.system_attrs[CONSTRAINTS_KEY])) for t in trials],
                          dtype=bool)
    if np.isnan(values).any():
        raise ValueError("The objective values of the completed trials must not contain NaN.")

    engine = _engine_cls(device)
    try:
        hv = engine.hypervolume_history(values, feasible, ref)
    finally:
        engine.close()

    if not (feasible & ~(values > ref).any(axis=1)).any():
        _logger.warning("Your study does not have any feasible trials.")
    return _HypervolumeHistoryInfo([t.number for t in trials], hv.tolist())


def plot_hypervolume_history(study, reference_point: Sequence[float], *, device: int = 0):
    """Drop-in for ``optuna.visualization.plot_hypervolume_history``: the same ``plotly`` figure, with the
    hypervolume history computed on the GPU (``hypervolume_history``).  Needs plotly, as optuna's does."""
    from optuna.visualization._plotly_imports import _imports

    _imports.check()
    return _get_hypervolume_history_plot(hypervolume_history(study, reference_point, device=device))


def _front_mask(trials, directions, device: int) -> np.ndarray:
    """Pareto-front flags of ``trials`` (COMPLETE) under the study's directions, computed on the device."""
    M = len(directions)
    if any(len(t.values) != M for t in trials):
        raise ValueError("The number of the values and the number of the objectives must be identical.")
    if not trials:
        return np.zeros(0, dtype=bool)
    signs = np.asarray([1.0 if d == StudyDirection.MINIMIZE else -1.0 for d in directions])
    values = np.asarray([t.values for t in trials], dtype=np.float64).reshape(len(trials), M) * signs
    if np.isnan(values).any():
        raise ValueError("The objective values of the completed trials must not contain NaN.")
    engine = _engine_cls(device)
    try:
        return engine.pareto_front(values)
    finally:
        engine.close()


def best_trials(study, *, device: int = 0) -> list:
    """Drop-in for ``Study.best_trials``: deep copies of the trials on the Pareto front, in trial order.

    As in the reference, a study counts as constrained when any of its trials, in any state, carries constraint
    values; then only the COMPLETE trials whose constraint values are all <= 0 are considered, otherwise every
    COMPLETE trial.  A single-objective study returns every trial tied at the best value.  Objective values holding
    NaN are rejected with ``ValueError`` before any work (``Study.tell`` never stores them), and so are studies of
    more than 16 objectives.

    Args:
        study: an ``optuna.Study``.
        device: CUDA device to compute on.
    """
    trials = study.get_trials(deepcopy=False)
    constrained = any(CONSTRAINTS_KEY in t.system_attrs for t in trials)
    considered = []
    for t in trials:
        if t.state != TrialState.COMPLETE:
            continue
        if constrained:
            c = t.system_attrs.get(CONSTRAINTS_KEY)
            if c is None or any(x > 0.0 for x in c):
                continue
        considered.append(t)
    mask = _front_mask(considered, study.directions, device)
    return copy.deepcopy([t for t, f in zip(considered, mask) if f])


def _deprecated_argument(name: str, deprecated: str, removed: str) -> None:
    from optuna._deprecated import _DEPRECATION_WARNING_TEMPLATE
    from optuna._warnings import optuna_warn

    optuna_warn(_DEPRECATION_WARNING_TEMPLATE.format(name=name, d_ver=deprecated, r_ver=removed), FutureWarning)


def _with_targets(trials, targets) -> list:
    pairs = [(t, targets(t)) for t in trials]
    for _, v in pairs:
        if not isinstance(v, _SequenceABC):
            raise ValueError(f"`targets` should return a sequence of target values. your `targets` returns {type(v)}")
    return [(t, list(v)) for t, v in pairs]


def pareto_front_info(study, *, target_names: list[str] | None = None, include_dominated_trials: bool = True,
                      axis_order: list[int] | None = None,
                      constraints_func: Callable | None = None, targets: Callable | None = None, device: int = 0):
    """The ``_ParetoFrontInfo`` that optuna's ``_get_pareto_front_info`` returns, with the front on the GPU.

    The same trial walk: COMPLETE trials, feasible when they carry no constraint values or all of them are <= 0
    (or, with the deprecated ``constraints_func``, when all its values are <= 0); the front of the feasible trials;
    best and non-best trials in trial order.  The same ``FutureWarning``s, ``ValueError``s and "does not have any
    completed (and feasible) trials" warning.  One difference: objective values of feasible trials holding NaN are
    rejected with ``ValueError`` before the front is computed (``Study.tell`` never stores them); so are studies of
    more than 16 objectives.
    """
    from optuna.visualization._pareto_front import _ParetoFrontInfo

    if axis_order is not None:
        _deprecated_argument("`axis_order`", "3.0.0", "5.0.0")
    if constraints_func is not None:
        _deprecated_argument("`constraints_func`", "4.0.0", "6.0.0")
    if targets is not None and axis_order is not None:
        raise ValueError("Using both `targets` and `axis_order` is not supported. "
                         "Use either `targets` or `axis_order`.")

    feasible, infeasible = [], []
    has_constraints = constraints_func is not None
    for t in study.get_trials(deepcopy=False, states=(TrialState.COMPLETE,)):
        if constraints_func is not None:
            ok = all(x <= 0.0 for x in constraints_func(t))
        else:
            c = t.system_attrs.get(CONSTRAINTS_KEY)
            has_constraints = has_constraints or c is not None
            ok = c is None or all(x <= 0.0 for x in c)
        (feasible if ok else infeasible).append(t)

    mask = _front_mask(feasible, study.directions, device)
    best = [t for t, f in zip(feasible, mask) if f]
    non_best = [t for t, f in zip(feasible, mask) if not f] if include_dominated_trials else []
    if not best:
        _logger.warning("Your study does not have any %s trials. "
                        % ("completed and feasible" if has_constraints else "completed"))

    if targets is None and len(study.directions) not in (2, 3):
        raise ValueError("`plot_pareto_front` function only supports 2 or 3 objective studies when using "
                         "`targets` is `None`. Please use `targets` if your objective studies have more than 3 "
                         "objectives.")
    get = targets if targets is not None else (lambda t: t.values)
    best_wv, non_best_wv, infeasible_wv = (_with_targets(x, get) for x in (best, non_best, infeasible))

    # the number of targets: from the first best (or else infeasible) trial, then target_names, then the study
    n_targets = (len(best_wv[0][1]) if best_wv else None) or (len(infeasible_wv[0][1]) if infeasible_wv else None)
    if n_targets is None:
        if target_names is not None:
            n_targets = len(target_names)
        elif targets is None:
            n_targets = len(study.directions)
        else:
            raise ValueError("If `targets` is specified for empty studies, `target_names` must be specified.")
    if n_targets not in (2, 3):
        raise ValueError(f"`plot_pareto_front` function only supports 2 or 3 targets. you used {n_targets} "
                         "targets now.")

    if target_names is None:
        names = study.metric_names
        target_names = names if names is not None else [f"Objective {i}" for i in range(n_targets)]
    elif len(target_names) != n_targets:
        raise ValueError(f"The length of `target_names` is supposed to be {n_targets}.")

    if axis_order is None:
        axis_order = list(range(n_targets))
    elif len(axis_order) != n_targets:
        raise ValueError(f"Size of `axis_order` {axis_order}. Expect: {n_targets}, Actual: {len(axis_order)}.")
    elif len(set(axis_order)) != n_targets:
        raise ValueError(f"Elements of given `axis_order` {axis_order} are not unique!.")
    elif max(axis_order) > n_targets - 1:
        raise ValueError(f"Given `axis_order` {axis_order} contains invalid index {max(axis_order)} higher than "
                         f"{n_targets - 1}.")
    elif min(axis_order) < 0:
        raise ValueError(f"Given `axis_order` {axis_order} contains invalid index {min(axis_order)} lower than 0.")

    return _ParetoFrontInfo(n_targets=n_targets, target_names=target_names, best_trials_with_values=best_wv,
                            non_best_trials_with_values=non_best_wv, infeasible_trials_with_values=infeasible_wv,
                            axis_order=axis_order, include_dominated_trials=include_dominated_trials,
                            has_constraints=has_constraints)


def plot_pareto_front(study, *, target_names: list[str] | None = None, include_dominated_trials: bool = True,
                      axis_order: list[int] | None = None, constraints_func: Callable | None = None,
                      targets: Callable | None = None, device: int = 0):
    """Drop-in for ``optuna.visualization.plot_pareto_front``: the same ``plotly`` figure, with the Pareto front
    computed on the GPU (``pareto_front_info``).  Needs plotly, as optuna's does."""
    from optuna.visualization._pareto_front import _get_pareto_front_plot
    from optuna.visualization._plotly_imports import _imports

    _imports.check()
    return _get_pareto_front_plot(pareto_front_info(
        study, target_names=target_names, include_dominated_trials=include_dominated_trials, axis_order=axis_order,
        constraints_func=constraints_func, targets=targets, device=device))
