"""Study analysis on the GPU: the hypervolume history of a multi-objective study.

``hypervolume_history`` returns what optuna's ``_get_hypervolume_history_info``
(optuna/visualization/_hypervolume_history.py:83-138) returns, computed by ``tpe_hypervolume_history``
(optuna_b200/csrc/tpe_hvhist.cuh); ``plot_hypervolume_history`` is the drop-in for
``optuna.visualization.plot_hypervolume_history`` and draws with optuna's own plot code.
"""
from __future__ import annotations

from typing import Sequence

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
