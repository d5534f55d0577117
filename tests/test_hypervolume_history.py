"""``optuna_b200.hypervolume_history`` / ``plot_hypervolume_history`` against the live reference
(optuna.visualization._hypervolume_history._get_hypervolume_history_info).

Every case runs twice: through ``ShimHVEngine`` (tests/_hvhist_engine.py: the host build of the per-trial code,
runs anywhere) and, with ``-m gpu``, through libtpe_b200.so.  Finite values agree within 1e-12 of the largest
|hypervolume|: the 2-D / 3-D hypervolumes may differ from the reference's BLAS dot products by a few ulp.
"""
from __future__ import annotations

import logging
import math

import numpy as np
import pytest

optuna = pytest.importorskip("optuna")


@pytest.fixture(params=[pytest.param("shim", id="shim-engine"),
                        pytest.param("cuda", id="cuda-engine", marks=pytest.mark.gpu)])
def hvh(request, monkeypatch):
    """optuna_b200.hypervolume_history answered by the host shim or by the CUDA library."""
    from optuna_b200 import analysis
    if request.param == "shim":
        from tests._hvhist_engine import ShimHVEngine
        monkeypatch.setattr(analysis, "_engine_cls", ShimHVEngine)
    return analysis.hypervolume_history


def _reference(study, reference_point):
    from optuna.visualization._hypervolume_history import _get_hypervolume_history_info
    return _get_hypervolume_history_info(study, np.asarray(reference_point, dtype=np.float64))


def _changes(x: np.ndarray) -> np.ndarray:
    prev = np.concatenate([[0.0], x[:-1]])
    return np.flatnonzero(~((x == prev) | (np.isnan(x) & np.isnan(prev))))


def _assert_same(got, want) -> None:
    assert list(got.trial_numbers) == list(want.trial_numbers)
    a = np.asarray(got.values, dtype=np.float64)
    b = np.asarray(want.values, dtype=np.float64)
    assert a.shape == b.shape
    np.testing.assert_array_equal(_changes(a), _changes(b))
    for kind in (np.isnan, np.isposinf, np.isneginf):
        np.testing.assert_array_equal(kind(a), kind(b))
    fin = np.isfinite(b)
    if fin.any():
        tol = 1e-12 * np.max(np.abs(b[fin]))
        assert np.max(np.abs(a[fin] - b[fin])) <= tol, (np.max(np.abs(a[fin] - b[fin])), tol)


def _study(directions, rows, constraints=None, states=None):
    """rows[i]: objective values of trial i (None for a trial without values); constraints[i]: its constraint
    values (None: no attr); states[i]: its TrialState (default COMPLETE)."""
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


# sizes keep the reference's own exact hypervolume (WFG, exponential in the objectives) within seconds
@pytest.mark.parametrize("M,n", [(2, 600), (3, 400), (4, 200), (5, 60), (6, 30)])
def test_objectives(hvh, M, n):
    study = _study(["minimize"] * M, _converging(n, M, M))
    rp = [2.5] * M
    _assert_same(hvh(study, rp), _reference(study, rp))


@pytest.mark.parametrize("directions", [["maximize"] * 3, ["minimize", "maximize", "minimize"],
                                        ["maximize", "minimize"]])
def test_directions(hvh, directions):
    M = len(directions)
    signs = np.array([1.0 if d == "minimize" else -1.0 for d in directions])
    study = _study(directions, _converging(300, M, 7) * signs)
    rp = list(2.5 * signs)
    _assert_same(hvh(study, rp), _reference(study, rp))


def test_constraints(hvh):
    rs = np.random.RandomState(3)
    n = 300
    cons = []
    for i in range(n):
        k = rs.randint(3)
        cons.append(None if k == 0 else (list(rs.uniform(-1, 0, 2)) if k == 1 else [rs.uniform(-1, 0), 0.5]))
    study = _study(["minimize"] * 3, _converging(n, 3, 11), constraints=cons)
    _assert_same(hvh(study, [2.5] * 3), _reference(study, [2.5] * 3))


def test_pruned_failed_running_are_ignored(hvh):
    from optuna.trial import TrialState
    rs = np.random.RandomState(5)
    n = 200
    kinds = [TrialState.COMPLETE, TrialState.PRUNED, TrialState.FAIL, TrialState.RUNNING]
    states = [kinds[k] for k in rs.choice(4, n, p=[0.7, 0.1, 0.1, 0.1])]
    study = _study(["minimize"] * 2, _converging(n, 2, 13), states=states)
    got = hvh(study, [2.5, 2.5])
    _assert_same(got, _reference(study, [2.5, 2.5]))
    assert len(got.trial_numbers) == sum(s == TrialState.COMPLETE for s in states)


def test_outside_reference_box(hvh):
    study = _study(["minimize"] * 4, _converging(200, 4, 17))
    rp = [1.2, 1.0, 1.5, 0.9]
    _assert_same(hvh(study, rp), _reference(study, rp))


@pytest.mark.parametrize("M", [2, 3, 4])
def test_duplicate_vectors(hvh, M):
    rs = np.random.RandomState(19 + M)
    rows = rs.randint(0, 4, (250, M)).astype(float)
    study = _study(["minimize"] * M, rows)
    _assert_same(hvh(study, [4.0] * M), _reference(study, [4.0] * M))


@pytest.mark.parametrize("M", [2, 3, 4])
def test_infinite_values(hvh, M):
    rs = np.random.RandomState(23 + M)
    rows = _converging(120, M, 29 + M)
    rows[rs.rand(*rows.shape) < 0.03] = -np.inf
    rows[rs.rand(*rows.shape) < 0.03] = np.inf
    study = _study(["minimize"] * M, rows)
    _assert_same(hvh(study, [2.5] * M), _reference(study, [2.5] * M))


@pytest.mark.parametrize("M", [2, 3, 4])
def test_infinite_reference_coordinate(hvh, M):
    rows = _converging(120, M, 31 + M)
    rows[7, 0] = np.inf
    study = _study(["minimize"] * M, rows)
    rp = [math.inf] + [2.5] * (M - 1)
    _assert_same(hvh(study, rp), _reference(study, rp))


def test_empty_study_warns(hvh, caplog):
    study = _study(["minimize", "minimize"], [])
    optuna.logging.enable_propagation()
    try:
        with caplog.at_level(logging.WARNING):
            got = hvh(study, [1.0, 1.0])
    finally:
        optuna.logging.disable_propagation()
    _assert_same(got, _reference(study, [1.0, 1.0]))
    assert "Your study does not have any completed trials." in caplog.text
    assert "Your study does not have any feasible trials." in caplog.text


def test_no_feasible_trial_warns(hvh, caplog):
    rows = _converging(40, 3, 37)
    cons = [[1.0] if i % 2 else None for i in range(40)]
    study = _study(["minimize"] * 3, rows, constraints=cons)
    rp = [0.5, 0.5, 0.5]   # every point has a coordinate >= 1 / sqrt(3): all lie outside the box
    rows_ok = rows[[i for i in range(40) if i % 2 == 0]]
    assert (rows_ok > np.array(rp)).any(axis=1).all()
    optuna.logging.enable_propagation()
    try:
        with caplog.at_level(logging.WARNING):
            got = hvh(study, rp)
    finally:
        optuna.logging.disable_propagation()
    _assert_same(got, _reference(study, rp))
    assert "Your study does not have any completed trials." not in caplog.text
    assert "Your study does not have any feasible trials." in caplog.text


def test_errors(hvh):
    single = _study(["minimize"], [[1.0], [2.0]])
    with pytest.raises(ValueError, match="multi-objective"):
        hvh(single, [3.0])
    study = _study(["minimize"] * 3, _converging(10, 3, 41))
    with pytest.raises(ValueError, match="dimension of the reference point"):
        hvh(study, [2.5, 2.5])
    with pytest.raises(ValueError, match="NaN"):
        hvh(study, [2.5, math.nan, 2.5])


def test_plot_matches_optuna(monkeypatch):
    pytest.importorskip("plotly")
    from optuna_b200 import analysis
    from tests._hvhist_engine import ShimHVEngine
    monkeypatch.setattr(analysis, "_engine_cls", ShimHVEngine)
    study = _study(["minimize"] * 2, _converging(100, 2, 43))
    got = analysis.plot_hypervolume_history(study, [2.5, 2.5])
    want = optuna.visualization.plot_hypervolume_history(study, [2.5, 2.5])
    assert list(got.data[0].x) == list(want.data[0].x)
    np.testing.assert_allclose(got.data[0].y, want.data[0].y, rtol=1e-12)
    assert got.layout.title.text == want.layout.title.text


def test_lazy_exports():
    import optuna_b200
    from optuna_b200 import analysis
    assert optuna_b200.hypervolume_history is analysis.hypervolume_history
    assert optuna_b200.plot_hypervolume_history is analysis.plot_hypervolume_history


@pytest.mark.gpu
def test_full_size_20000x4(hvh):
    study = _study(["minimize"] * 4, _converging(20000, 4, 0))
    rp = [2.5] * 4
    _assert_same(hvh(study, rp), _reference(study, rp))


@pytest.mark.gpu
def test_engine_suggestion_unchanged_by_hypervolume_history():
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
        vals = _converging(3000, 4, 2)
        hv = eng.hypervolume_history(vals, None, np.full(4, 2.5))
        assert hv.shape == (3000,) and np.isfinite(hv).all() and hv[-1] > 0
        after = eng.suggest(list(range(P)), u, 1, **cfg)
        for a, b in zip(before, after):
            np.testing.assert_array_equal(a, b)
    finally:
        eng.close()
