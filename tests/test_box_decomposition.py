"""The device box decomposition of GPSampler's log-EHVI (``TPEEngine.box_decomposition``, tpe_boxdec.cuh) and the
sampler path that uses it, against the live reference: optuna's ``get_non_dominated_box_bounds``, ``LogEHVI`` and
``GPSampler``.  Runs on the NumPy restatement of the kernels (tests/_box_decomposition_engine.py) and, on the GPU, on
the CUDA library."""
from __future__ import annotations

import time
import warnings

import numpy as np
import pytest

optuna = pytest.importorskip("optuna")
torch = pytest.importorskip("torch")

import tests.test_gp_sampler as tgs  # noqa: E402
from tests.test_gp_sampler_ehvi import _capture_acqf, _dtlz2, _Stub, _values_mo  # noqa: E402


@pytest.fixture(params=[pytest.param("numpy", id="numpy-engine"),
                        pytest.param("cuda", id="cuda-engine", marks=pytest.mark.gpu)])
def engine_cls(request, monkeypatch):
    """The engine class behind optuna_b200.gp_sampler: the NumPy restatement or the CUDA library."""
    from optuna_b200 import TPEEngine, gp_sampler
    from tests._box_decomposition_engine import NumpyBoxDecompositionEngine
    cls = NumpyBoxDecompositionEngine if request.param == "numpy" else TPEEngine
    monkeypatch.setattr(gp_sampler, "_engine_cls", cls)
    return cls


def _reference(loss_vals, ref_point):
    from optuna._hypervolume import get_non_dominated_box_bounds
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return get_non_dominated_box_bounds(loss_vals, ref_point)


def _assert_bytes(want, got):
    for w, g in zip(want, got):
        assert g.shape == w.shape and g.dtype == w.dtype
        assert g.tobytes() == w.tobytes()


def _check(engine_cls, loss_vals, ref_point):
    want = _reference(loss_vals, ref_point)
    eng = engine_cls(0)
    try:
        _assert_bytes(want, eng.box_decomposition(loss_vals, ref_point))
    finally:
        eng.close()
    return want


def _dtlz2_front(M, n, seed=0, P=8):
    rs = np.random.RandomState(seed)
    F = _dtlz2(rs.uniform(0, 1, (n, P)), M)
    ref = np.max(F, axis=0)
    return F, np.nextafter(np.maximum(1.1 * ref, 0.9 * ref), np.inf)


# ---- against get_non_dominated_box_bounds ------------------------------------------------------------------------------

@pytest.mark.parametrize("M,n", [(2, 200), (3, 120), (4, 60), (5, 30), (6, 20), (7, 14), (8, 12)])
def test_dtlz2(engine_cls, M, n):
    want = _check(engine_cls, *_dtlz2_front(M, n, seed=M))
    assert want[0].shape[0] > 1


@pytest.mark.parametrize("M,n,levels,seed", [(2, 40, 5, 0), (3, 60, 4, 1), (4, 50, 3, 2), (5, 30, 3, 3)])
def test_integer_grid_ties(engine_cls, M, n, levels, seed):
    """Integer grids: ties in every coordinate, repeated and dominated rows, and (levels - 1) equal to the reference
    point in some coordinates."""
    rs = np.random.RandomState(seed)
    Y = rs.randint(0, levels, size=(n, M)).astype(float)
    _check(engine_cls, Y, np.full(M, levels - 1.0))
    _check(engine_cls, Y, np.full(M, float(levels)))


def test_repeated_and_dominated_rows(engine_cls):
    rs = np.random.RandomState(5)
    F, ref = _dtlz2_front(3, 40)
    Y = np.vstack([F, F[:10], F[5:15] + 0.25, F[::-1]])
    _check(engine_cls, Y[rs.permutation(len(Y))], ref)


def test_coordinate_at_reference_point(engine_cls):
    F, ref = _dtlz2_front(3, 30, seed=7)
    ref = ref.copy()
    ref[1] = F[:, 1].max()      # the row holding the maximum lies on the reference point in coordinate 1
    _check(engine_cls, F, ref)
    ref[0] = F[:, 0].min()      # only that coordinate's minimum row is not strictly below it
    _check(engine_cls, F, ref)


def test_single_point_and_no_box(engine_cls):
    want = _check(engine_cls, np.array([[1.0, 2.0, 3.0]]), np.array([2.0, 3.0, 4.0]))
    assert want[0].shape == (3, 3)   # one slab per objective
    # nothing lies strictly below the reference point: the one box below it
    want = _check(engine_cls, np.array([[1.0, 2.0], [0.5, 3.0]]), np.array([2.0, 2.0]))
    assert want[0].shape == (1, 2)
    # a reference point of -inf in a coordinate: every box is empty
    for ref in ([-np.inf, 5.0], [np.inf, -np.inf]):
        want = _check(engine_cls, np.array([[1.0, 2.0]]), np.array(ref))
        assert want[0].shape == (0, 2)
    want = _check(engine_cls, np.array([[1.0, 2.0, 3.0], [2.0, 1.0, 0.0]]), np.array([np.inf, np.inf, -np.inf]))
    assert want[0].shape == (0, 3)


def test_infinite_results(engine_cls):
    """Every box's lower bound is -inf in coordinate 0; an infinite reference point makes more infinite bounds."""
    F, ref = _dtlz2_front(3, 25, seed=9)
    want = _check(engine_cls, F, ref)
    assert np.all(np.isneginf(want[0][:, 0]))
    want = _check(engine_cls, F, np.array([np.inf, ref[1], np.inf]))
    assert np.isinf(want[1]).any()
    _check(engine_cls, F, np.array([ref[0], -np.inf, ref[2]]))


def test_signed_zeros(engine_cls):
    """np.unique(axis=0) compares rows with ==, so rows that differ only in the sign of a zero are one row, and which
    of them it keeps is numpy's choice.  The boxes are then compared with ==; rows without such twins byte-wise."""
    a = np.array([[0.0, 1.0], [-0.0, 1.0]])
    assert np.unique(a, axis=0).shape == (1, 2)   # numpy's behaviour this test rests on
    Y = np.array([[0.0, 1.0, 2.0], [-0.0, 1.0, 2.0], [1.0, -0.0, 1.0], [1.0, 0.0, 1.0], [2.0, 2.0, -0.0],
                  [0.5, 0.5, 0.5]])
    ref = np.array([3.0, 3.0, 3.0])
    want = _reference(Y, ref)
    eng = engine_cls(0)
    try:
        got = eng.box_decomposition(Y, ref)
    finally:
        eng.close()
    for w, g in zip(want, got):
        assert g.shape == w.shape and np.array_equal(g, w)


def test_same_bits(engine_cls):
    """Two calls, and calls of other sizes in between, on one engine return the same bytes."""
    F, ref = _dtlz2_front(4, 40, seed=3)
    F2, ref2 = _dtlz2_front(3, 80, seed=4)
    eng = engine_cls(0)
    try:
        first = eng.box_decomposition(F, ref)
        other = eng.box_decomposition(F2, ref2)
        _assert_bytes(first, eng.box_decomposition(F, ref))
        _assert_bytes(other, eng.box_decomposition(F2, ref2))
        _assert_bytes(_reference(F, ref), first)
    finally:
        eng.close()


@pytest.mark.parametrize("args,message", [
    ((np.zeros((3, 1)), np.ones(1)), "2 <= M <= 24 objectives, got 1"),
    ((np.zeros((3, 25)), np.ones(25)), "2 <= M <= 24 objectives, got 25"),
    ((np.zeros((0, 2)), np.ones(2)), "1 <= n"),
    ((np.array([[0.0, np.inf]]), np.ones(2)), "loss values must be finite"),
    ((np.array([[0.0, np.nan]]), np.ones(2)), "loss values must be finite"),
    ((np.zeros((2, 2)), np.array([1.0, np.nan])), "reference point holds a NaN"),
    ((np.zeros((2, 3)), np.ones(2)), "loss_vals must be"),
])
def test_invalid_inputs(engine_cls, args, message):
    eng = engine_cls(0)
    try:
        with pytest.raises(ValueError, match=message.replace("^", r"\^")):
            eng.box_decomposition(*args)
    finally:
        eng.close()


# ---- the sampler's acquisition ---------------------------------------------------------------------------------------

def _space(P):
    from optuna._gp import search_space as gp_search_space
    return gp_search_space.SearchSpace({f"x{j}": optuna.distributions.FloatDistribution(0, 1) for j in range(P)})


@pytest.mark.parametrize("M", [2, 3, 5])
def test_log_ehvi_state(engine_cls, M):
    """The ``LogEHVI`` the sampler builds with the device decomposition holds the bits of optuna's."""
    from optuna._gp import acqf
    from optuna_b200 import GPSampler
    rs = np.random.RandomState(M)
    Y = -_dtlz2(rs.uniform(0, 1, (30, 8)), M)
    Y = (Y - Y.mean(0)) / np.maximum(Y.std(0), 1e-12)
    space = _space(8)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        want = acqf.LogEHVI([_Stub(8)] * M, space, torch.from_numpy(Y), 128, 17)
        sampler = GPSampler(seed=0)
        sampler._device_ehvi = lambda a: a
        try:
            got = sampler._log_ehvi([_Stub(8)] * M, space, Y, 17)
        finally:
            sampler.close()
    assert type(got) is acqf.LogEHVI
    for name in ("_non_dominated_box_lower_bounds", "_non_dominated_box_intervals", "_fixed_samples"):
        w, g = getattr(want, name), getattr(got, name)
        assert g.shape == w.shape and g.numpy().tobytes() == w.numpy().tobytes(), name
    assert got.length_scales.tobytes() == want.length_scales.tobytes()
    assert got._stabilizing_noise == want._stabilizing_noise


@pytest.mark.parametrize("constrained", [False, True])
def test_sampler_acquisition_boxes(engine_cls, constrained):
    """One ask of the drop-in and of optuna's sampler on the same history: the acquisitions' boxes are the same
    bits (they depend on the standardised values only)."""
    from optuna_b200 import GPSampler
    d = tgs._dists("float")
    history = tgs._history(d, 14, 2, 3, constrained)
    cf = tgs._constraints_func if constrained else None
    got = []
    for cls in (GPSampler, optuna.samplers.GPSampler):
        sampler = cls(seed=1, constraints_func=cf)
        sampler._device_ehvi = lambda a: a
        seen = _capture_acqf(sampler)
        study = optuna.create_study(directions=["minimize"] * 2, sampler=sampler)
        study.add_trials(history)
        study.ask(d)
        if isinstance(sampler, GPSampler):
            sampler.close()
        got.append(seen[0]._acqf if constrained else seen[0])
    ours, ref = got
    for name in ("_non_dominated_box_lower_bounds", "_non_dominated_box_intervals", "_fixed_samples"):
        w, g = getattr(ref, name), getattr(ours, name)
        assert g.shape == w.shape and g.numpy().tobytes() == w.numpy().tobytes(), name


# ---- end-to-end replays -----------------------------------------------------------------------------------------------

def _pair_replay(monkeypatch, dists, history, steps, n_obj, constrained, seed):
    """The drop-in with and without the device decomposition, on the same history and seed: the suggestions are the
    same bits.  Each step the asked trials fail and the suggestion joins both histories as a complete trial."""
    from optuna_b200 import GPSampler, gp_sampler
    cf = tgs._constraints_func if constrained else None
    on, off = GPSampler(seed=seed, constraints_func=cf), GPSampler(seed=seed, constraints_func=cf)
    s_on = optuna.create_study(directions=["minimize"] * n_obj, sampler=on)
    s_off = optuna.create_study(directions=["minimize"] * n_obj, sampler=off)
    real = gp_sampler._answers_box_decomposition
    calls = []

    def counted(cls):
        calls.append(cls)
        return real(cls)
    try:
        for s in (s_on, s_off):
            s.add_trials(history)
        for _ in range(steps):
            monkeypatch.setattr(gp_sampler, "_answers_box_decomposition", counted)
            t_on = s_on.ask(dists)
            monkeypatch.setattr(gp_sampler, "_answers_box_decomposition", lambda cls: False)
            t_off = s_off.ask(dists)
            monkeypatch.setattr(gp_sampler, "_answers_box_decomposition", real)
            assert t_on.params == t_off.params
            for s, t in ((s_on, t_on), (s_off, t_off)):
                s.tell(t, state=optuna.trial.TrialState.FAIL)
                s.add_trial(tgs._frozen(t_on.params, dists, n_obj, constrained))
    finally:
        on.close()
        off.close()
    assert len(calls) == steps and real(calls[0])


@pytest.mark.parametrize("constrained", [False, True])
@pytest.mark.parametrize("n_obj", [2, 3, 4, 5])
def test_replay(engine_cls, monkeypatch, n_obj, constrained):
    """Suggestions bit-identical to the host-decomposition path, and within 1e-6 of optuna's ``GPSampler``."""
    d = tgs._dists("float")
    if n_obj > 2:
        monkeypatch.setattr(tgs, "_values", _values_mo)
    history = tgs._history(d, 14, n_obj, 40 + n_obj, constrained)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        _pair_replay(monkeypatch, d, history, 2, n_obj, constrained, seed=n_obj)
        tgs._replay(d, history, 2, n_obj=n_obj, constrained=constrained, seed=n_obj)


# ---- selection and the warning ----------------------------------------------------------------------------------------

def test_engine_without_box_decomposition(monkeypatch):
    """An engine class with the EHVI calls but without ``box_decomposition`` keeps optuna's host decomposition and
    still evaluates log-EHVI on the device."""
    from optuna._hypervolume import box_decomposition as bd_module
    from optuna_b200 import GPSampler, gp_sampler
    from optuna_b200.gp_sampler import _DeviceLogEHVI
    from tests._gp_sampler_ehvi_engine import NumpyEHVIEngine
    monkeypatch.setattr(gp_sampler, "_engine_cls", NumpyEHVIEngine)
    assert gp_sampler._answers_ehvi(NumpyEHVIEngine)
    assert not gp_sampler._answers_box_decomposition(NumpyEHVIEngine)
    host_calls = []
    real = bd_module._get_non_dominated_box_bounds
    monkeypatch.setattr(bd_module, "_get_non_dominated_box_bounds",
                        lambda *a: host_calls.append(1) or real(*a))
    d = tgs._dists("float")
    sampler = GPSampler(seed=0)
    seen = _capture_acqf(sampler)
    study = optuna.create_study(directions=["minimize"] * 2, sampler=sampler)
    study.add_trials(tgs._history(d, 12, 2, 5, False))
    try:
        study.ask(d)
    finally:
        sampler.close()
    assert isinstance(seen[0], _DeviceLogEHVI) and host_calls == [1]


def test_device_path_skips_host_decomposition(engine_cls, monkeypatch):
    from optuna._hypervolume import box_decomposition as bd_module
    from optuna_b200 import GPSampler

    def fail(*a):
        raise AssertionError("the host box decomposition ran")
    monkeypatch.setattr(bd_module, "_get_non_dominated_box_bounds", fail)
    d = tgs._dists("float")
    sampler = GPSampler(seed=0)
    _capture_acqf(sampler)
    study = optuna.create_study(directions=["minimize"] * 2, sampler=sampler)
    study.add_trials(tgs._history(d, 12, 2, 5, False))
    try:
        study.ask(d)
    finally:
        sampler.close()


def test_twenty_five_objectives_create_no_engine(engine_cls):
    from optuna._gp import acqf
    from optuna_b200 import GPSampler
    D = optuna.distributions
    dists = {"x0": D.FloatDistribution(0, 1), "x1": D.FloatDistribution(0, 1)}
    rs = np.random.RandomState(25)
    trials = [optuna.trial.create_trial(params={"x0": float(rs.uniform()), "x1": float(rs.uniform())},
                                        distributions=dists, values=list(float(i) + 0.01 * rs.uniform(0, 1, 25)))
              for i in range(6)]
    sampler = GPSampler(seed=0, n_startup_trials=2)
    seen = _capture_acqf(sampler)
    study = optuna.create_study(directions=["minimize"] * 25, sampler=sampler)
    study.add_trials(trials)
    try:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            study.ask(dists)
        assert type(seen[0]) is acqf.LogEHVI and sampler._ehvi_engine is None
    finally:
        sampler.close()


def _ask_warnings(cls, n_obj):
    d = tgs._dists("float")
    sampler = cls(seed=0)
    _capture_acqf(sampler)
    study = optuna.create_study(directions=["minimize"] * n_obj, sampler=sampler)
    study.add_trials(tgs._history(d, 12, n_obj, 7, False))
    try:
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            study.ask(d)
    finally:
        if hasattr(sampler, "close"):
            sampler.close()
    return [x for x in w if "Box decomposition" in str(x.message)]


@pytest.mark.parametrize("n_obj", [4, 5])
def test_warning(engine_cls, monkeypatch, n_obj):
    """More than four objectives: optuna's warning, as a ``UserWarning`` attributed to the same caller's line."""
    from optuna_b200 import GPSampler
    monkeypatch.setattr(tgs, "_values", _values_mo)
    ours, ref = _ask_warnings(GPSampler, n_obj), _ask_warnings(optuna.samplers.GPSampler, n_obj)
    assert len(ours) == len(ref) == (1 if n_obj > 4 else 0)
    for a, b in zip(ours, ref):
        assert a.category is b.category is UserWarning
        assert str(a.message) == str(b.message)
        assert a.filename == b.filename == __file__


# ---- GPU only ----------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("M,n", [(4, 1000), (5, 200)])
def test_large_against_reference(M, n):
    """DTLZ2 over 8 parameters, as the sampler sees it: the Pareto rows of the standardised values."""
    from optuna_b200 import TPEEngine
    F, ref = _dtlz2_front(M, n, seed=0)
    t0 = time.perf_counter()
    want = _reference(F, ref)
    t_ref = time.perf_counter() - t0
    eng = TPEEngine(0)
    try:
        t0 = time.perf_counter()
        got = eng.box_decomposition(F, ref)
        t_dev = time.perf_counter() - t0
        _assert_bytes(want, got)
        print(f"\n{M} x {n}: {want[0].shape[0]} boxes, stats {eng.last_box_stats}, host {t_ref:.3f} s, "
              f"device {t_dev:.3f} s (first call)")
    finally:
        eng.close()


@pytest.mark.gpu
def test_five_objectives_thousand_trials():
    """One ask of a five-objective DTLZ2 study of 1 000 trials over 8 parameters, which the host decomposition does
    not finish in reasonable time."""
    from optuna_b200 import GPSampler
    D = optuna.distributions
    P, M, n = 8, 5, 1000
    dists = {f"x{j}": D.FloatDistribution(0, 1) for j in range(P)}
    rs = np.random.RandomState(0)
    X = rs.uniform(0, 1, (n, P))
    F = _dtlz2(X, M)
    trials = [optuna.trial.create_trial(params={f"x{j}": float(x[j]) for j in range(P)}, distributions=dists,
                                        values=[float(v) for v in f]) for x, f in zip(X, F)]
    sampler = GPSampler(seed=0)
    study = optuna.create_study(directions=["minimize"] * M, sampler=sampler)
    study.add_trials(trials)
    try:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            t0 = time.perf_counter()
            t = study.ask(dists)
            dt = time.perf_counter() - t0
        stats = sampler._ehvi_engine.last_box_stats
    finally:
        sampler.close()
    print(f"\n5 x 1000 ask: {dt:.2f} s, box decomposition {stats}")
    assert set(t.params) == set(dists) and all(0.0 <= v <= 1.0 for v in t.params.values())
    assert dt < 300.0, dt
