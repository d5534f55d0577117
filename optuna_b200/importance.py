"""fANOVA parameter importances on the GPU: a drop-in ``FanovaImportanceEvaluator``.

``optuna.importance.get_param_importances`` and ``optuna.visualization.plot_param_importances`` default to optuna's
``FanovaImportanceEvaluator``.  It fits a random forest with scikit-learn, then, for every tree and parameter, walks
the tree once per split midpoint of the parameter in Python (optuna/importance/_fanova/_tree.py:47-142), which grows
faster than the square of the number of trials.  This evaluator is optuna's, with only the ``_Fanova`` object it
keeps in ``self._evaluator`` replaced: the same forest is fitted with the same arguments and seed on the host, and
one ``tpe_fanova_variances`` call (optuna_b200/csrc/tpe_fanova.cuh) computes every tree's variance and every
(tree, parameter) marginal variance.  ``evaluate`` -- the trial filtering, the encoding, ``target``, the errors and
the result order -- is optuna's own.

One difference: a categorical whose one-hot columns split one tree into more than 2^20 grid cells (more than 20 of
its columns split in that tree) raises ``ValueError``; the reference would walk that tree 2^20 times.
"""
from __future__ import annotations

import numpy as np
from optuna.importance import FanovaImportanceEvaluator as _OptunaFanovaImportanceEvaluator

from .engine import TPEEngine

# the engine class that answers the computation (tests substitute a host implementation)
_engine_cls = TPEEngine


class _Fanova:
    """``fit`` / ``get_importance`` of optuna's ``_Fanova`` (optuna/importance/_fanova/_fanova.py:53-108)."""

    def __init__(self, n_trees: int, max_depth: int, seed: int | None, device: int) -> None:
        from sklearn.ensemble import RandomForestRegressor

        self._forest = RandomForestRegressor(
            n_estimators=n_trees,
            max_depth=max_depth,
            min_samples_split=2,
            min_samples_leaf=1,
            random_state=seed,
        )
        self._device = device
        self._tree_variances: np.ndarray | None = None
        self._marginal_variances: np.ndarray | None = None

    def fit(self, X: np.ndarray, y: np.ndarray, search_spaces: np.ndarray,
            column_to_encoded_columns: list[np.ndarray]) -> None:
        assert X.shape[0] == y.shape[0]
        assert X.shape[1] == search_spaces.shape[0]
        assert search_spaces.shape[1] == 2

        self._forest.fit(X, y)
        trees = [e.tree_ for e in self._forest.estimators_]
        node_offsets = np.concatenate([[0], np.cumsum([t.node_count for t in trees])])
        param_offsets = np.concatenate([[0], np.cumsum([len(c) for c in column_to_encoded_columns])])
        raw_features = (np.concatenate(column_to_encoded_columns) if column_to_encoded_columns
                        else np.empty(0, dtype=np.int64))
        engine = _engine_cls(self._device)
        try:
            tree_var, marginal_var = engine.fanova_variances(
                node_offsets,
                np.concatenate([t.children_left for t in trees]),
                np.concatenate([t.children_right for t in trees]),
                np.concatenate([t.feature for t in trees]),
                np.concatenate([t.threshold for t in trees]),
                np.concatenate([t.value[:, 0, 0] for t in trees]),
                search_spaces, param_offsets, raw_features)
        finally:
            engine.close()
        if np.all(tree_var == 0):
            # If all trees have 0 variance, we cannot assess any importances.
            raise RuntimeError("Encountered zero total variance in all trees.")
        self._tree_variances = tree_var
        self._marginal_variances = np.clip(marginal_var, 0.0, None)

    def get_importance(self, feature: int) -> tuple[float, float]:
        assert self._tree_variances is not None and self._marginal_variances is not None
        keep = self._tree_variances > 0.0
        fractions = self._marginal_variances[feature][keep] / self._tree_variances[keep]
        return float(fractions.mean()), float(fractions.std())


class FanovaImportanceEvaluator(_OptunaFanovaImportanceEvaluator):
    """fANOVA importance evaluator whose tree marginals are computed on the GPU.

    A drop-in for ``optuna.importance.FanovaImportanceEvaluator``: pass it as ``evaluator=`` to
    ``optuna.importance.get_param_importances`` or ``optuna.visualization.plot_param_importances``.  For the same
    seed it fits the same forest and returns the reference's importances.

    Args:
        n_trees: The number of trees in the forest.
        max_depth: The maximum depth of the trees in the forest.
        seed: Controls the randomness of the forest (``random_state`` of scikit-learn's ``RandomForestRegressor``).
        device: CUDA device to compute on.
    """

    def __init__(self, *, n_trees: int = 64, max_depth: int = 64, seed: int | None = None, device: int = 0) -> None:
        super().__init__(n_trees=n_trees, max_depth=max_depth, seed=seed)
        # optuna's evaluate() (optuna/importance/_fanova/_evaluator.py:73-130) fits and queries self._evaluator
        if not hasattr(self, "_evaluator"):
            raise RuntimeError("optuna's FanovaImportanceEvaluator no longer keeps its _Fanova in _evaluator")
        self._evaluator = _Fanova(n_trees=n_trees, max_depth=max_depth, seed=seed, device=device)
