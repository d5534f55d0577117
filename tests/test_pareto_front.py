"""``optuna_b200.best_trials`` / ``pareto_front_info`` / ``plot_pareto_front`` against the live reference
(``Study.best_trials``, optuna.visualization._pareto_front._get_pareto_front_info,
optuna.study._multi_objective._is_pareto_front).

Every case runs twice: through ``NumpyParetoEngine`` (tests/_pareto_engine.py: the sort-then-filter steps in NumPy
with a small chunk, runs anywhere) and, with ``-m gpu``, through libtpe_b200.so.  Front flags are exact, so the
results must be equal.
"""
from __future__ import annotations

import logging
import math
import warnings

import numpy as np
import pytest

optuna = pytest.importorskip("optuna")


@pytest.fixture(params=[pytest.param("numpy", id="numpy-engine"),
                        pytest.param("cuda", id="cuda-engine", marks=pytest.mark.gpu)])
def engine_cls(request, monkeypatch):
    """The engine class behind optuna_b200.analysis: the NumPy restatement or the CUDA library."""
    from optuna_b200 import TPEEngine, analysis
    if request.param == "numpy":
        from tests._pareto_engine import NumpyParetoEngine
        cls = NumpyParetoEngine
    else:
        cls = TPEEngine
    monkeypatch.setattr(analysis, "_engine_cls", cls)
    return cls


def _study(directions, rows, constraints=None, states=None):
    """rows[i]: objective values of trial i; constraints[i]: its constraint values (None: no attr); states[i]: its
    TrialState (default COMPLETE; the others carry no values)."""
    from optuna.samplers._base import _CONSTRAINTS_KEY
    from optuna.trial import TrialState, create_trial

    study = optuna.create_study(directions=directions)
    trials = []
    for i, row in enumerate(rows):
        state = states[i] if states is not None else TrialState.COMPLETE
        attrs = {}
        if constraints is not None and constraints[i] is not None:
            attrs[_CONSTRAINTS_KEY] = list(constraints[i])
        vals = [float(x) for x in row] if state == TrialState.COMPLETE else None
        trials.append(create_trial(state=state, values=vals, system_attrs=attrs))
    study.add_trials(trials)
    return study


def _converging(n, M, seed):
    from tools.bench_hv_history import dtlz2_values
    return dtlz2_values(n, M, seed)


def _reference_mask(values):
    from optuna.study._multi_objective import _is_pareto_front
    return _is_pareto_front(np.asarray(values, dtype=np.float64), assume_unique_lexsorted=False)


def _engine_mask(engine_cls, values):
    eng = engine_cls(0)
    try:
        return eng.pareto_front(values)
    finally:
        eng.close()


def _check_study(study, **info_kwargs):
    """best_trials and pareto_front_info equal the reference's on this study."""
    from optuna.visualization._pareto_front import _get_pareto_front_info

    from optuna_b200 import analysis
    got = analysis.best_trials(study)
    want = study.best_trials
    assert [t.number for t in got] == [t.number for t in want]
    assert got == want
    if len(study.directions) in (2, 3) or "targets" in info_kwargs:
        for dominated in (True, False):
            got_info = analysis.pareto_front_info(study, include_dominated_trials=dominated, **info_kwargs)
            want_info = _get_pareto_front_info(study, include_dominated_trials=dominated, **info_kwargs)
            assert got_info == want_info
    return got


@pytest.mark.parametrize("M,n", [(1, 300), (2, 600), (3, 500), (4, 400), (6, 300), (16, 120)])
def test_objectives(engine_cls, M, n):
    values = _converging(n, M, M)
    study = _study(["minimize"] * M, values)
    kw = {} if M in (2, 3) else {"targets": lambda t: [t.values[0], t.values[-1]]}
    front = _check_study(study, **kw)
    assert 0 < len(front) < n or M == 16
    np.testing.assert_array_equal(_engine_mask(engine_cls, values), _reference_mask(values))


def test_single_objective_ties(engine_cls):
    study = _study(["minimize"], [[3.0], [1.0], [2.0], [1.0], [-0.0], [0.0], [0.0]])
    assert [t.number for t in _check_study(study)] == [4, 5, 6]
    study = _study(["maximize"], [[3.0], [1.0], [3.0], [math.inf], [math.inf]])
    assert [t.number for t in _check_study(study)] == [3, 4]


@pytest.mark.parametrize("directions", [["maximize"] * 3, ["minimize", "maximize", "minimize"],
                                        ["maximize", "minimize"], ["maximize", "minimize", "maximize", "minimize"]])
def test_directions(engine_cls, directions):
    M = len(directions)
    signs = np.array([1.0 if d == "minimize" else -1.0 for d in directions])
    study = _study(directions, _converging(400, M, 7) * signs)
    _check_study(study, **({} if M <= 3 else {"targets": lambda t: t.values[1:3]}))


@pytest.mark.parametrize("M", [2, 3, 4])
def test_duplicate_vectors(engine_cls, M):
    rs = np.random.RandomState(19 + M)
    rows = rs.randint(0, 4, (250, M)).astype(float)
    study = _study(["minimize"] * M, rows)
    front = _check_study(study, **({} if M <= 3 else {"targets": lambda t: t.values[:3]}))
    # copies of front vectors are all on the front, copies of dominated ones all off it
    on = {tuple(t.values) for t in front}
    assert sum(tuple(r) in on for r in rows) == len(front)
    np.testing.assert_array_equal(_engine_mask(engine_cls, rows), _reference_mask(rows))


def test_signed_zero(engine_cls):
    # the +0.0 row dominates the -0.0 row: same coordinate 0 under ==, smaller coordinate 1
    rows = np.array([[-0.0, 1.0], [0.0, 0.5], [0.0, 1.0], [1.0, 0.0]])
    want = _reference_mask(rows)
    np.testing.assert_array_equal(want, [False, True, False, True])
    np.testing.assert_array_equal(_engine_mask(engine_cls, rows), want)
    # the same with the -0.0 rows placed across the chunk cuts of the NumPy engine, and through the study
    rs = np.random.RandomState(3)
    rows = np.concatenate([np.stack([np.where(rs.rand(40) < 0.5, -0.0, 0.0), rs.randint(0, 6, 40) * 0.5], 1),
                           np.stack([rs.randint(1, 4, 20) * 1.0, rs.randint(-3, 3, 20) * 1.0], 1)])
    rows = rows[rs.permutation(len(rows))]
    np.testing.assert_array_equal(_engine_mask(engine_cls, rows), _reference_mask(rows))
    _check_study(_study(["minimize", "minimize"], rows))
    # a maximised 0.0 becomes -0.0 after sign normalisation
    _check_study(_study(["maximize", "minimize"], -rows))


@pytest.mark.parametrize("M", [2, 3, 4])
def test_infinite_values(engine_cls, M):
    rs = np.random.RandomState(23 + M)
    rows = _converging(200, M, 29 + M)
    rows[rs.rand(*rows.shape) < 0.05] = -np.inf
    rows[rs.rand(*rows.shape) < 0.05] = np.inf
    rows[5] = np.inf
    rows[6] = -np.inf
    rows[7] = -np.inf
    np.testing.assert_array_equal(_engine_mask(engine_cls, rows), _reference_mask(rows))
    _check_study(_study(["minimize"] * M, rows), **({} if M <= 3 else {"targets": lambda t: t.values[:2]}))


def test_trial_states_are_ignored(engine_cls):
    from optuna.trial import TrialState
    rs = np.random.RandomState(5)
    n = 300
    kinds = [TrialState.COMPLETE, TrialState.PRUNED, TrialState.FAIL, TrialState.RUNNING, TrialState.WAITING]
    states = [kinds[k] for k in rs.choice(5, n, p=[0.6, 0.1, 0.1, 0.1, 0.1])]
    study = _study(["minimize"] * 3, _converging(n, 3, 13), states=states)
    front = _check_study(study)
    assert all(t.state == TrialState.COMPLETE for t in front)


def test_constraints(engine_cls):
    rs = np.random.RandomState(3)
    n = 300
    cons = []
    for _ in range(n):
        k = rs.randint(4)
        cons.append([None, list(rs.uniform(-1, 0, 2)), [rs.uniform(-1, 0), 0.5], [0.0]][k])
    study = _study(["minimize"] * 3, _converging(n, 3, 11), constraints=cons)
    front = _check_study(study)
    # best_trials: a trial without constraint values is infeasible in a constrained study
    assert all(cons[t.number] is not None for t in front)
    from optuna_b200 import pareto_front_info
    info = pareto_front_info(study)
    assert info.has_constraints and len(info.infeasible_trials_with_values) > 0


def test_constraint_attr_only_on_unfinished_trials(engine_cls):
    from optuna.trial import TrialState
    n = 60
    states = [TrialState.COMPLETE] * n
    cons = [None] * n
    for i in (3, 17, 40):
        states[i] = [TrialState.PRUNED, TrialState.FAIL, TrialState.RUNNING][i % 3]
        cons[i] = [-1.0]
    study = _study(["minimize", "minimize"], _converging(n, 2, 12), constraints=cons, states=states)
    # the study is constrained, and no COMPLETE trial carries constraint values: best_trials is empty
    assert _check_study(study) == []
    from optuna_b200 import pareto_front_info
    assert len(pareto_front_info(study).best_trials_with_values) > 0


def test_constraints_func(engine_cls):
    from optuna.visualization._pareto_front import _get_pareto_front_info

    from optuna_b200 import analysis
    study = _study(["minimize", "maximize"], _converging(200, 2, 14) * [1.0, -1.0])

    def cf(t):
        return [t.values[0] - 0.8, -1.0]

    with pytest.warns(FutureWarning, match="constraints_func"):
        got = analysis.pareto_front_info(study, constraints_func=cf)
    with pytest.warns(FutureWarning, match="constraints_func"):
        want = _get_pareto_front_info(study, constraints_func=cf)
    assert got == want and got.has_constraints
    assert len(got.infeasible_trials_with_values) > 0


def _outcome(fn):
    """(exception type and text or None, FutureWarning texts, result) of fn()."""
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        try:
            res, err = fn(), None
        except ValueError as e:
            res, err = None, (type(e), str(e))
    return err, [str(x.message) for x in w if issubclass(x.category, FutureWarning)], res


@pytest.mark.parametrize("kwargs", [
    dict(axis_order=[1, 0]),
    dict(axis_order=[0, 1, 2]),
    dict(axis_order=[0, 0]),
    dict(axis_order=[0, 2]),
    dict(axis_order=[-1, 0]),
    dict(axis_order=[1, 0], targets=lambda t: t.values),
    dict(targets=lambda t: t.values[0]),
    dict(targets=lambda t: [t.values[0]]),
    dict(targets=lambda t: [t.values[0], t.values[1], 1.0]),
    dict(target_names=["a"]),
    dict(target_names=["a", "b"]),
    dict(target_names=["a", "b"], axis_order=[1, 0]),
])
def test_arguments_match_reference(engine_cls, kwargs):
    from optuna.visualization._pareto_front import _get_pareto_front_info

    from optuna_b200 import analysis
    study = _study(["minimize", "minimize"], _converging(100, 2, 15))
    got = _outcome(lambda: analysis.pareto_front_info(study, **kwargs))
    want = _outcome(lambda: _get_pareto_front_info(study, **kwargs))
    assert got == want


@pytest.mark.filterwarnings("ignore::optuna.exceptions.ExperimentalWarning")
def test_objectives_beyond_three_need_targets(engine_cls):
    from optuna.visualization._pareto_front import _get_pareto_front_info

    from optuna_b200 import analysis
    study = _study(["minimize"] * 4, _converging(50, 4, 16))
    got = _outcome(lambda: analysis.pareto_front_info(study))
    assert got[0] is not None and got == _outcome(lambda: _get_pareto_front_info(study))
    study.set_metric_names(["a", "b", "c", "d"])
    got = _outcome(lambda: analysis.pareto_front_info(study, targets=lambda t: t.values[1:]))
    assert got == _outcome(lambda: _get_pareto_front_info(study, targets=lambda t: t.values[1:]))


def _warnings_of(fn, caplog):
    optuna.logging.enable_propagation()
    try:
        caplog.clear()
        with caplog.at_level(logging.WARNING):
            out = _outcome(fn)
    finally:
        optuna.logging.disable_propagation()
    return out, [r.getMessage() for r in caplog.records]


@pytest.mark.parametrize("kind", ["empty", "no-complete", "all-infeasible"])
def test_empty_and_infeasible_studies(engine_cls, kind, caplog):
    from optuna.trial import TrialState
    from optuna.visualization._pareto_front import _get_pareto_front_info

    from optuna_b200 import analysis
    if kind == "empty":
        study = _study(["minimize", "minimize"], [])
    elif kind == "no-complete":
        study = _study(["minimize", "minimize"], [[1.0, 2.0]] * 3, states=[TrialState.PRUNED] * 3)
    else:
        study = _study(["minimize", "minimize"], _converging(30, 2, 17), constraints=[[1.0]] * 30)
    assert analysis.best_trials(study) == study.best_trials == []
    for kw in ({}, {"targets": lambda t: t.values}, {"targets": lambda t: t.values, "target_names": ["a", "b"]}):
        got, got_log = _warnings_of(lambda: analysis.pareto_front_info(study, **kw), caplog)
        want, want_log = _warnings_of(lambda: _get_pareto_front_info(study, **kw), caplog)
        assert got == want
        assert any("does not have any" in m for m in want_log)
        assert [m for m in got_log if "does not have any" in m] == [m for m in want_log if "does not have any" in m]


def test_errors(engine_cls):
    from optuna_b200 import analysis
    study = _study(["minimize", "minimize"], [[1.0, 2.0], [0.5, 1.0], [2.0, 1.0]])
    # optuna refuses NaN values when a trial is told or created; plant one in the stored trial itself
    study.get_trials(deepcopy=False)[1].values[0] = math.nan
    with pytest.raises(ValueError, match="NaN"):
        analysis.best_trials(study)
    with pytest.raises(ValueError, match="NaN"):
        analysis.pareto_front_info(study)
    many = _study(["minimize"] * 17, _converging(20, 17, 18))
    with pytest.raises(ValueError, match="n_objectives"):
        analysis.best_trials(many)
    with pytest.raises(ValueError, match="NaN"):
        _engine_mask(engine_cls, np.array([[1.0, 2.0], [np.nan, 1.0]]))
    with pytest.raises(ValueError, match="n_objectives"):
        _engine_mask(engine_cls, np.zeros((3, 17)))


def test_best_trials_are_copies(engine_cls):
    from optuna_b200 import analysis
    study = _study(["minimize", "minimize"], _converging(50, 2, 19))
    before = study.best_trials
    got = analysis.best_trials(study)
    got[0].values[0] = 123.0
    got[0].user_attrs["x"] = 1
    got[0].system_attrs["y"] = 2
    got.pop()
    assert study.best_trials == before
    assert analysis.best_trials(study) == before


def test_plot_matches_optuna(monkeypatch):
    pytest.importorskip("plotly")
    from optuna_b200 import analysis
    from tests._pareto_engine import NumpyParetoEngine
    monkeypatch.setattr(analysis, "_engine_cls", NumpyParetoEngine)
    for directions, cons in ((["minimize", "maximize"], None), (["minimize"] * 3, [[0.0], [1.0]] * 60)):
        M = len(directions)
        study = _study(directions, _converging(120, M, 20 + M), constraints=cons)
        got = analysis.plot_pareto_front(study)
        want = optuna.visualization.plot_pareto_front(study)
        assert got.to_json() == want.to_json()


def test_lazy_exports():
    import optuna_b200
    from optuna_b200 import analysis
    assert optuna_b200.best_trials is analysis.best_trials
    assert optuna_b200.pareto_front_info is analysis.pareto_front_info
    assert optuna_b200.plot_pareto_front is analysis.plot_pareto_front
    assert {"best_trials", "pareto_front_info", "plot_pareto_front"} <= set(optuna_b200.__all__)


@pytest.mark.gpu
@pytest.mark.parametrize("n,M", [(100000, 3), (30000, 6)])
def test_full_size_against_is_pareto_front(n, M):
    from optuna_b200 import TPEEngine
    values = _converging(n, M, 1)
    eng = TPEEngine(0)
    try:
        got = eng.pareto_front(values)
    finally:
        eng.close()
    np.testing.assert_array_equal(got, _reference_mask(values))


@pytest.mark.gpu
def test_engine_suggestion_unchanged_by_pareto_front():
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
        vals = _converging(20000, 4, 2)
        front = eng.pareto_front(vals)
        np.testing.assert_array_equal(front, _reference_mask(vals))
        after = eng.suggest(list(range(P)), u, 1, **cfg)
        for a, b in zip(before, after):
            np.testing.assert_array_equal(a, b)
    finally:
        eng.close()
