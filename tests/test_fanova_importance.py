"""``optuna_b200.FanovaImportanceEvaluator`` against the live reference's ``FanovaImportanceEvaluator``
(optuna/importance/_fanova) and against tests/golden/fanova.npz (oracle/gen_fanova_fixture.py).

Every case runs twice: through ``NumpyFanovaEngine`` (tests/_fanova_engine.py: the terminal sweep in NumPy, runs
anywhere) and, with ``-m gpu``, through libtpe_b200.so.  Tolerances: importances within 1e-9 absolute (and 1e-9
relative above 1e-3), per tree |marginal variance difference| <= 1e-9 * tree variance, and the reference's key order
wherever its values differ by more than 1e-8.
"""
from __future__ import annotations

import inspect
import math
import os

import numpy as np
import pytest

optuna = pytest.importorskip("optuna")

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fanova.npz")


@pytest.fixture(params=[pytest.param("numpy", id="numpy-engine"),
                        pytest.param("cuda", id="cuda-engine", marks=pytest.mark.gpu)])
def engine_cls(request, monkeypatch):
    """The engine class behind optuna_b200.importance: the NumPy restatement or the CUDA library."""
    from optuna_b200 import TPEEngine
    from tests._fanova_engine import NumpyFanovaEngine
    cls = NumpyFanovaEngine if request.param == "numpy" else TPEEngine
    if request.param == "numpy":
        pytest.importorskip("sklearn")
    from optuna_b200 import importance
    monkeypatch.setattr(importance, "_engine_cls", cls)
    return cls


def _check(want: dict, got: dict) -> None:
    assert set(want) == set(got)
    for k in want:
        assert abs(want[k] - got[k]) <= 1e-9, (k, want[k], got[k])
        if want[k] > 1e-3:
            assert abs(want[k] - got[k]) <= 1e-9 * want[k], (k, want[k], got[k])
    wk, gk = list(want), list(got)
    for i in range(len(wk) - 1):
        if want[wk[i]] - want[wk[i + 1]] > 1e-8:
            assert gk.index(wk[i]) < gk.index(wk[i + 1]), (wk, gk)


def _compare(study, seed=0, n_trees=64, max_depth=64, **kw):
    import optuna_b200
    want = optuna.importance.get_param_importances(
        study, evaluator=optuna.importance.FanovaImportanceEvaluator(n_trees=n_trees, max_depth=max_depth, seed=seed),
        **kw)
    got = optuna.importance.get_param_importances(
        study, evaluator=optuna_b200.FanovaImportanceEvaluator(n_trees=n_trees, max_depth=max_depth, seed=seed), **kw)
    _check(want, got)
    return got


_WEIGHTS = {2: [0.0, 1.0], 3: [0.0, 2.0, -1.0], 4: [0.0, 1.0, 3.0, 0.5], 5: [1.0, 0.0, 0.2, 2.0, -0.5],
            6: [0.0, 0.1, 0.2, 0.3, 0.4, 2.0]}


def _mixed_study(n_trials, seed, n_choices=4, directions=None, single=False, duplicates=False):
    def objective(t):
        x = t.suggest_float("x", -3.0, 3.0)
        y = t.suggest_float("y", 1e-3, 10.0, log=True)
        s = t.suggest_float("s", 0.0, 1.0, step=0.1)
        z = t.suggest_int("z", -4, 9)
        c = t.suggest_categorical("c", list(range(n_choices)))
        # a categorical with almost no influence: some trees never split on it
        q = t.suggest_categorical("q", ["u", "v", "w"])
        if single:
            t.suggest_float("one", 2.0, 2.0)
        v = x * x + 0.4 * math.log(y) + 0.5 * s + 0.1 * z + _WEIGHTS[n_choices][c] + (1e-4 if q == "w" else 0.0)
        return v if directions is None else (v, -x + 0.1 * z)

    sampler = optuna.samplers.RandomSampler(seed=seed)
    study = (optuna.create_study(sampler=sampler) if directions is None
             else optuna.create_study(directions=directions, sampler=sampler))
    if duplicates:
        rs = np.random.RandomState(seed)
        base = [dict(x=float(rs.uniform(-3, 3)), y=float(rs.uniform(1e-3, 10)), s=0.1 * rs.randint(11),
                     z=int(rs.randint(-4, 10)), c=int(rs.randint(n_choices)), q="u") for _ in range(40)]
        for i in range(200):
            study.enqueue_trial(base[i % 40])
    study.optimize(objective, n_trials=n_trials)
    return study


@pytest.mark.parametrize("n_choices", [2, 3, 4, 5, 6])
def test_mixed_parameters(engine_cls, n_choices):
    pytest.importorskip("sklearn")
    _compare(_mixed_study(250, n_choices, n_choices), seed=n_choices)


def test_single_value_distribution_and_params_subset(engine_cls):
    pytest.importorskip("sklearn")
    study = _mixed_study(200, 21, single=True)
    got = _compare(study, seed=3)
    assert got["one"] == 0.0
    _compare(study, seed=4, params=["x", "c", "one"])
    _compare(study, seed=4, params=["z"])
    _compare(study, seed=5, params=["one"])


def test_target_normalize_and_forest_shape(engine_cls):
    pytest.importorskip("sklearn")
    study = _mixed_study(200, 31)
    _compare(study, seed=7, target=lambda t: t.params["x"] + t.params["z"])
    _compare(study, seed=8, normalize=False)
    _compare(study, seed=9, n_trees=7, max_depth=3)
    _compare(study, seed=10, n_trees=16, max_depth=9)


def test_multi_objective(engine_cls):
    pytest.importorskip("sklearn")
    import optuna_b200
    study = _mixed_study(200, 41, directions=["minimize", "maximize"])
    _compare(study, seed=1, target=lambda t: t.values[1])
    with pytest.raises(ValueError, match="please specify the `target`"):
        optuna.importance.get_param_importances(study, evaluator=optuna_b200.FanovaImportanceEvaluator(seed=0))


def test_constant_objective_raises(engine_cls):
    pytest.importorskip("sklearn")
    import optuna_b200
    study = optuna.create_study(sampler=optuna.samplers.RandomSampler(seed=0))
    study.optimize(lambda t: t.suggest_float("x", 0, 1) * 0.0 + t.suggest_int("z", 0, 3) * 0 + 1.5, n_trials=50)
    for ev in (optuna.importance.FanovaImportanceEvaluator(seed=0), optuna_b200.FanovaImportanceEvaluator(seed=0)):
        with pytest.raises(RuntimeError, match="Encountered zero total variance in all trees."):
            optuna.importance.get_param_importances(study, evaluator=ev)


def test_duplicate_parameter_vectors(engine_cls):
    pytest.importorskip("sklearn")
    _compare(_mixed_study(200, 51, duplicates=True), seed=2)


def test_per_tree_variances(engine_cls):
    """Per tree and parameter, the engine's marginal variance against the reference's _FanovaTree on the same forest."""
    pytest.importorskip("sklearn")
    from optuna._transform import _SearchSpaceTransform
    from optuna.importance._base import _get_distributions, _get_filtered_trials, _get_target_values, _get_trans_params
    from optuna.importance._fanova._fanova import _Fanova

    study = _mixed_study(200, 61, n_choices=5)
    dists = _get_distributions(study, params=None)
    trials = _get_filtered_trials(study, params=list(dists), target=None)
    trans = _SearchSpaceTransform(dists, transform_log=False, transform_step=False)
    fa = _Fanova(n_trees=12, max_depth=64, min_samples_split=2, min_samples_leaf=1, seed=0)
    fa.fit(_get_trans_params(trials, trans), _get_target_values(trials, None), trans.bounds,
           trans.column_to_encoded_columns)
    arrays = _flatten([e.tree_ for e in fa._forest.estimators_], trans.bounds, trans.column_to_encoded_columns)
    _check_arrays(engine_cls, arrays, np.array([t.variance for t in fa._trees]),
                  np.array([[t.get_marginal_variance(c) for t in fa._trees] for c in trans.column_to_encoded_columns]))


def _flatten(trees, bounds, cols):
    return dict(node_offsets=np.concatenate([[0], np.cumsum([t.node_count for t in trees])]),
                left=np.concatenate([t.children_left for t in trees]),
                right=np.concatenate([t.children_right for t in trees]),
                feature=np.concatenate([t.feature for t in trees]),
                threshold=np.concatenate([t.threshold for t in trees]),
                value=np.concatenate([t.value[:, 0, 0] for t in trees]), bounds=bounds,
                param_offsets=np.concatenate([[0], np.cumsum([len(c) for c in cols])]),
                raw_features=np.concatenate(cols))


def _variances(engine_cls, arrays):
    eng = engine_cls(0)
    try:
        return eng.fanova_variances(**arrays)
    finally:
        eng.close()


def _check_arrays(engine_cls, arrays, want_tree, want_marginal):
    tree_var, marg = _variances(engine_cls, arrays)
    np.testing.assert_allclose(tree_var, want_tree, rtol=1e-12, atol=0)
    assert marg.shape == want_marginal.shape
    assert np.all(np.abs(marg - want_marginal) <= 1e-9 * want_tree[None, :])


@pytest.mark.parametrize("case", ["num", "cat"])
def test_golden_fixture(engine_cls, case):
    z = np.load(GOLDEN)
    arrays = {k: z[f"{case}_{k}"] for k in ("node_offsets", "left", "right", "feature", "threshold", "value", "bounds",
                                            "param_offsets", "raw_features")}
    _check_arrays(engine_cls, arrays, z[f"{case}_tree_variance"], z[f"{case}_marginal_variance"])


def _golden_arrays():
    z = np.load(GOLDEN)
    return {k: z[f"cat_{k}"].copy() for k in ("node_offsets", "left", "right", "feature", "threshold", "value",
                                               "bounds", "param_offsets", "raw_features")}


def _corrupt(kind):
    a = _golden_arrays()
    internal = np.nonzero(a["feature"] >= 0)[0]
    i = int(internal[3])
    if kind == "child_not_after_parent":
        a["left"][i] = 0
    elif kind == "child_out_of_range":
        a["right"][i] = int(a["node_offsets"][1]) + 5
    elif kind == "two_parents":
        j = int(internal[4])
        a["left"][j] = a["left"][i]
    elif kind == "feature_out_of_range":
        a["feature"][i] = a["bounds"].shape[0]
    elif kind == "nan_threshold":
        a["threshold"][i] = np.nan
    elif kind == "threshold_outside_bounds":
        a["threshold"][i] = a["bounds"][a["feature"][i], 1] + 1.0
    elif kind == "raw_feature_repeated":
        a["raw_features"][1] = a["raw_features"][0]
    elif kind == "empty_tree":
        a["node_offsets"][1] = 0
    return a


@pytest.mark.parametrize("kind", ["child_not_after_parent", "child_out_of_range", "two_parents",
                                  "feature_out_of_range", "nan_threshold", "threshold_outside_bounds",
                                  "raw_feature_repeated", "empty_tree"])
def test_invalid_tree_arrays(engine_cls, kind):
    with pytest.raises(ValueError):
        _variances(engine_cls, _corrupt(kind))


def _one_hot_tree(n_split):
    """One tree splitting n_split one-hot columns at 0.5 along a chain; the last leaf carries the value 1."""
    n = 2 * n_split + 1
    left, right = np.full(n, -1), np.full(n, -1)
    feature, thr, value = np.full(n, -2), np.full(n, -2.0), np.zeros(n)
    for k in range(n_split):
        node = 2 * k
        feature[node], thr[node] = k, 0.5
        left[node], right[node] = node + 1, node + 2
        value[node + 1] = float(k % 3)
    value[n - 1] = 1.0
    return dict(node_offsets=np.array([0, n]), left=left, right=right, feature=feature, threshold=thr, value=value,
                bounds=np.tile([0.0, 1.0], (n_split + 1, 1)), param_offsets=np.array([0, n_split + 1]),
                raw_features=np.arange(n_split + 1))


def test_categorical_cell_cap(engine_cls):
    tree_var, marg = _variances(engine_cls, _one_hot_tree(12))   # 2^12 cells
    assert tree_var[0] > 0 and 0 < marg[0, 0] <= tree_var[0] * (1 + 1e-12)
    if engine_cls.__name__ == "NumpyFanovaEngine":
        return   # 2^21 cells cell by cell in Python: only the library's refusal is worth the time
    with pytest.raises(ValueError, match="2\\^20"):
        _variances(engine_cls, _one_hot_tree(21))


def test_categorical_cell_cap_numpy():
    from tests._fanova_engine import NumpyFanovaEngine
    with pytest.raises(ValueError, match="2\\^20"):
        _variances(NumpyFanovaEngine, _one_hot_tree(21))


def test_subclass_hooks_into_optuna_evaluator():
    """The drop-in replaces only ``_evaluator``; this fails if optuna renames the attribute evaluate() uses."""
    pytest.importorskip("sklearn")
    import optuna_b200
    from optuna.importance import FanovaImportanceEvaluator
    assert "self._evaluator" in inspect.getsource(FanovaImportanceEvaluator.evaluate)
    assert "_evaluator" in vars(FanovaImportanceEvaluator(seed=0))
    ev = optuna_b200.FanovaImportanceEvaluator(seed=0)
    assert isinstance(ev, FanovaImportanceEvaluator)
    assert type(ev._evaluator).__module__ == "optuna_b200.importance"
    assert optuna_b200.FanovaImportanceEvaluator.evaluate is FanovaImportanceEvaluator.evaluate


@pytest.mark.gpu
def test_large_forest_against_reference_trees():
    """5 000 trials x 8 parameters: a few (tree, parameter) marginals against _FanovaTree.get_marginal_variance."""
    pytest.importorskip("sklearn")
    from optuna_b200 import TPEEngine
    from optuna.importance._fanova._fanova import _Fanova
    from optuna.importance._fanova._tree import _FanovaTree

    rs = np.random.RandomState(0)
    X = rs.uniform(0, 1, (5000, 8))
    y = ((X - 0.3) ** 2 * np.arange(1, 9)).sum(1) + 0.1 * rs.randn(5000)
    bounds = np.tile([0.0, 1.0], (8, 1))
    cols = [np.array([j]) for j in range(8)]
    fa = _Fanova(n_trees=4, max_depth=64, min_samples_split=2, min_samples_leaf=1, seed=0)
    fa._forest.fit(X, y)
    trees = [e.tree_ for e in fa._forest.estimators_]
    tree_var, marg = _variances(TPEEngine, _flatten(trees, bounds, cols))
    for t, p in ((0, 7), (2, 3)):
        ft = _FanovaTree(trees[t], bounds)
        assert abs(tree_var[t] - ft.variance) <= 1e-12 * ft.variance
        assert abs(marg[p, t] - ft.get_marginal_variance(cols[p])) <= 1e-9 * ft.variance


@pytest.mark.gpu
def test_engine_suggestion_unchanged_by_fanova():
    from optuna_b200 import ParamSpec, TPEEngine
    N, P, C = 500, 4, 32
    rs = np.random.RandomState(0)
    X = rs.uniform(0, 1, (N, P))
    key = np.stack([((X - 0.5) ** 2).sum(1), np.zeros(N)], 1)
    u = np.random.RandomState(1).rand(C * (1 + P))
    eng = TPEEngine(0)
    try:
        eng.set_space([ParamSpec(kind=0, low=0.0, high=1.0) for _ in range(P)])
        eng.set_history(X, np.zeros(N, np.int8), key)
        cfg = dict(n_below=25, n_candidates=C, multivariate=True)
        before = eng.suggest(list(range(P)), u, 1, **cfg)
        z = np.load(GOLDEN)
        tree_var, marg = eng.fanova_variances(**{k: z[f"cat_{k}"] for k in (
            "node_offsets", "left", "right", "feature", "threshold", "value", "bounds", "param_offsets",
            "raw_features")})
        np.testing.assert_allclose(tree_var, z["cat_tree_variance"], rtol=1e-12)
        after = eng.suggest(list(range(P)), u, 1, **cfg)
        for a, b in zip(before, after):
            np.testing.assert_array_equal(a, b)
    finally:
        eng.close()
