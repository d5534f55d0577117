"""Writes tests/golden/fanova.npz: two seeded forests and the live reference's fANOVA variances of them.

For each case ("num": a float, a log float and an int; "cat": a float, an int and a 5-choice categorical) the
reference's ``_Fanova`` (optuna/importance/_fanova/_fanova.py) fits its forest on a seeded RandomSampler study, encoded
as ``FanovaImportanceEvaluator.evaluate`` encodes it.  Stored per case, under the prefix ``<case>_``:
  node_offsets, left, right, feature, threshold, value  -- the flattened trees (children indexed within their tree);
  bounds, param_offsets, raw_features                   -- the search space and the parameters' raw features;
  tree_variance [T], marginal_variance [n_params, T]    -- ``_FanovaTree.variance`` and ``get_marginal_variance``.

    python oracle/gen_fanova_fixture.py      # needs oracle/_ref (oracle/build_ref.py) and scikit-learn
"""
from __future__ import annotations

import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(ROOT, "tests", "golden", "fanova.npz")


def _study(optuna, case: str, n_trials: int):
    def objective(t):
        x = t.suggest_float("x", -2.0, 3.0)
        z = t.suggest_int("z", 0, 12)
        if case == "num":
            y = t.suggest_float("y", 1e-3, 1e2, log=True)
            return x * x + 0.5 * np.log(y) + 0.2 * z
        c = t.suggest_categorical("c", ["a", "b", "c", "d", "e"])
        return x * x + 0.2 * z + {"a": 0.0, "b": 1.0, "c": 2.5, "d": 0.3, "e": -1.0}[c]

    study = optuna.create_study(sampler=optuna.samplers.RandomSampler(seed=11 if case == "num" else 12))
    study.optimize(objective, n_trials=n_trials)
    return study


def main() -> None:
    sys.path.insert(0, ROOT)
    from oracle import build_ref, ref
    build_ref.build()
    assert ref.enable()
    import optuna
    from optuna._transform import _SearchSpaceTransform
    from optuna.importance._base import _get_distributions, _get_filtered_trials, _get_target_values, _get_trans_params
    from optuna.importance._fanova._fanova import _Fanova

    out = {}
    for case, n_trials, n_trees in (("num", 300, 8), ("cat", 300, 8)):
        study = _study(optuna, case, n_trials)
        dists = _get_distributions(study, params=None)
        trials = _get_filtered_trials(study, params=list(dists), target=None)
        trans = _SearchSpaceTransform(dists, transform_log=False, transform_step=False)
        X, y = _get_trans_params(trials, trans), _get_target_values(trials, None)
        fa = _Fanova(n_trees=n_trees, max_depth=64, min_samples_split=2, min_samples_leaf=1, seed=5)
        fa.fit(X, y, trans.bounds, trans.column_to_encoded_columns)
        trees = [e.tree_ for e in fa._forest.estimators_]
        cols = trans.column_to_encoded_columns
        out[f"{case}_node_offsets"] = np.concatenate([[0], np.cumsum([t.node_count for t in trees])])
        out[f"{case}_left"] = np.concatenate([t.children_left for t in trees]).astype(np.int32)
        out[f"{case}_right"] = np.concatenate([t.children_right for t in trees]).astype(np.int32)
        out[f"{case}_feature"] = np.concatenate([t.feature for t in trees]).astype(np.int32)
        out[f"{case}_threshold"] = np.concatenate([t.threshold for t in trees])
        out[f"{case}_value"] = np.concatenate([t.value[:, 0, 0] for t in trees])
        out[f"{case}_bounds"] = trans.bounds
        out[f"{case}_param_offsets"] = np.concatenate([[0], np.cumsum([len(c) for c in cols])]).astype(np.int32)
        out[f"{case}_raw_features"] = np.concatenate(cols).astype(np.int32)
        out[f"{case}_tree_variance"] = np.array([t.variance for t in fa._trees])
        out[f"{case}_marginal_variance"] = np.array([[t.get_marginal_variance(c) for t in fa._trees] for c in cols])
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
