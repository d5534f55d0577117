"""``optuna_b200.GPSampler`` against the live reference's ``optuna.samplers.GPSampler``
(optuna/samplers/_gp/sampler.py, optuna/_gp/gp.py, acqf.py, optim_mixed.py).

Every case runs twice: through ``NumpyGPSamplerEngine`` (tests/_gp_sampler_engine.py: the device algorithm in NumPy,
runs anywhere) and, with ``-m gpu``, through libtpe_b200.so.  Tolerances:
- ``gp_query`` against ``GPRegressor.posterior`` and its autograd gradient: mean and var within 1e-10 relative (with
  an absolute floor of 1e-10 times the largest magnitude of the batch), gradients within 1e-8 of their norm;
- acquisition values within 1e-9 relative (1e-9 absolute floor), their gradients within 1e-7 of their norm;
- replayed suggestions: normalised parameters within 1e-6 of the reference's.
"""
from __future__ import annotations

import json
import logging

import numpy as np
import pytest

optuna = pytest.importorskip("optuna")
torch = pytest.importorskip("torch")

from tests.test_terminator_gpu_gp import _gp_data  # noqa: E402


@pytest.fixture(params=[pytest.param("numpy", id="numpy-engine"),
                        pytest.param("cuda", id="cuda-engine", marks=pytest.mark.gpu)])
def engine_cls(request, monkeypatch):
    """The engine class behind optuna_b200.gp_sampler: the NumPy restatement or the CUDA library."""
    from optuna_b200 import TPEEngine, gp_sampler
    from tests._gp_sampler_engine import NumpyGPSamplerEngine
    cls = NumpyGPSamplerEngine if request.param == "numpy" else TPEEngine
    monkeypatch.setattr(gp_sampler, "_engine_cls", cls)
    return cls


def _params(P, seed, noise=None):
    rs = np.random.RandomState(seed)
    return np.concatenate([np.exp(rs.uniform(-1.0, 1.5, P)), [np.exp(rs.uniform(-0.5, 0.5))],
                           [1e-6 + np.exp(rs.uniform(-9, -3)) if noise is None else noise]])


def _ref_gp(X, y, cat, params):
    from optuna._gp.gp import GPRegressor
    P = X.shape[1]
    gpr = GPRegressor(torch.from_numpy(cat), torch.from_numpy(X), torch.from_numpy(y),
                      torch.from_numpy(params[:P].copy()), torch.tensor(params[P], dtype=torch.float64),
                      torch.tensor(params[P + 1], dtype=torch.float64))
    gpr._cache_matrix()
    return gpr


def _ref_query(gpr, xq):
    x = torch.from_numpy(xq).requires_grad_(True)
    mean, var = gpr.posterior(x)
    dmean, = torch.autograd.grad(mean.sum(), x, retain_graph=True)
    dvar, = torch.autograd.grad(var.sum(), x)
    return mean.detach().numpy(), var.detach().numpy(), dmean.numpy(), dvar.numpy()


def _device_gp(engine_cls, X, y, cat, params):
    from optuna_b200.gp_sampler import _DeviceGP
    eng = engine_cls(0)
    eng.gp_set_data(X, y, cat)
    return eng, _DeviceGP(eng, X, y, cat, params)


def _check_values(want, got):
    for w, g in zip(want, got):
        floor = 1e-10 * max(1.0, float(np.max(np.abs(w))))
        assert np.all(np.abs(g - w) <= 1e-10 * np.abs(w) + floor), np.max(np.abs(g - w))


def _check_grads(want, got):
    for w, g in zip(want, got):
        assert np.linalg.norm(g - w) <= 1e-8 * np.linalg.norm(w) + 1e-300, (np.linalg.norm(g - w), np.linalg.norm(w))


def _queries(X, m, seed):
    return np.random.RandomState(seed).uniform(0, 1, (m, X.shape[1]))


# ---- the query against GPRegressor.posterior -----------------------------------------------------------------------

@pytest.mark.parametrize("kind,n,m,dup", [
    ("mixed", 150, 1100, False),   # n not a multiple of 64, more than 1 024 value rows and 64 gradient rows
    ("mixed", 60, 130, True),      # duplicate training rows
    ("float", 70, 40, False),
    ("cat", 40, 30, False),        # every column categorical: zero gradients
    ("wide17", 130, 70, False),    # two passes of 16 gradient columns
    ("p1", 20, 10, False),
])
def test_query_against_reference(engine_cls, kind, n, m, dup):
    X, y, cat = _gp_data(kind, n, seed=n, duplicates=dup)
    params = _params(X.shape[1], n)
    xq = np.concatenate([_queries(X, m, 1), X[:5]])   # the last rows are training points
    if cat.any():   # categorical columns of a query hold one of the normalised choices
        xq[:, cat] = X[np.random.RandomState(2).randint(0, X.shape[0], xq.shape[0])][:, cat]
    want = _ref_query(_ref_gp(X, y, cat, params), xq)
    eng = engine_cls(0)
    try:
        eng.gp_set_data(X, y, cat)
        eng.gp_condition(params)
        got = eng.gp_query(xq, grad=True)
        values_only = eng.gp_query(xq)
        again = eng.gp_query(xq, grad=True)
    finally:
        eng.close()
    _check_values(want[:2], got[:2])
    _check_grads(want[2:], got[2:])
    assert np.all(got[2][:, cat] == 0.0) and np.all(got[3][:, cat] == 0.0)
    for a, b in zip(got[:2], values_only):   # values do not depend on the gradient request
        assert a.tobytes() == b.tobytes()
    for a, b in zip(got, again):
        assert a.tobytes() == b.tobytes()


def test_single_point(engine_cls):
    """A 1-D point gives scalars, as the reference does, at a random point and at a training point with the noise at
    its minimum, where the variance is near 0."""
    X, y, cat = _gp_data("mixed", 50, seed=4)
    params = _params(X.shape[1], 4, noise=1e-6)
    ref = _ref_gp(X, y, cat, params)
    eng, dev = _device_gp(engine_cls, X, y, cat, params)
    try:
        for x in (_queries(X, 1, 3)[0], X[7].copy()):
            xr = torch.from_numpy(x).requires_grad_(True)
            xd = torch.from_numpy(x.copy()).requires_grad_(True)
            (mr, vr), (md, vd) = ref.posterior(xr), dev.posterior(xd)
            assert md.shape == () and vd.shape == ()
            _check_values([mr.detach().numpy()[None], vr.detach().numpy()[None]],
                          [md.detach().numpy()[None], vd.detach().numpy()[None]])
            (mr + 0.5 * vr).backward()
            (md + 0.5 * vd).backward()
            _check_grads([xr.grad.numpy()], [xd.grad.numpy()])
    finally:
        eng.close()


def test_clamped_variance_has_no_variance_gradient(engine_cls):
    """A slightly negative noise (-1e-3, with lengthscales short enough that the covariance stays positive definite)
    makes the exact posterior variance negative, about -1e-3, at and next to the training points.  There the
    reference clamps it to 0 and torch's clamp_min_ passes no gradient; the unclamped variance's gradient is large.
    Away from the training points the variance is positive and both pass their gradients."""
    X, y, cat = _gp_data("float", 60, seed=11)
    P = X.shape[1]
    params = np.concatenate([np.full(P, 1000.0), [1.0, -1e-3]])
    xq = X[:20].copy()
    xq[:, 0] = np.clip(xq[:, 0] + 1e-4, 0.0, 1.0)
    xq = np.concatenate([xq, _queries(X, 10, 12)])
    ref = _ref_gp(X, y, cat, params)
    want = _ref_query(ref, xq)
    # the reference's raw variance (gp.py:232-248 without the clamp) and its gradient
    x = torch.from_numpy(xq).requires_grad_(True)
    K = ref.kernel(x, ref._X_all)
    chol = ref._cov_Y_Y_chol
    V = torch.linalg.solve_triangular(chol, torch.linalg.solve_triangular(chol.T, K, upper=True, left=False),
                                      upper=False, left=False)
    raw = ref.kernel_scale - torch.linalg.vecdot(K, V)
    raw_grad, = torch.autograd.grad(raw.sum(), x)
    clamped = raw.detach().numpy() < 0.0
    assert clamped[:20].all() and not clamped[20:].any()
    assert np.all(np.linalg.norm(raw_grad.numpy()[clamped], axis=1) > 1e-2)
    eng = engine_cls(0)
    try:
        eng.gp_set_data(X, y, cat)
        eng.gp_condition(params)
        mean, var, dmean, dvar = eng.gp_query(xq, grad=True)
    finally:
        eng.close()
    assert np.all(var[clamped] == 0.0) and np.all(want[1][clamped] == 0.0)
    assert np.all(dvar[clamped] == 0.0) and np.all(want[3][clamped] == 0.0)
    _check_values(want[:2], (mean, var))
    _check_grads(want[2:], (dmean, dvar))


def test_running_rows_appended(engine_cls):
    X, y, cat = _gp_data("mixed", 90, seed=5)
    params = _params(X.shape[1], 5)
    Xr = _queries(X, 4, 6)
    Xr[:, cat] = X[:4][:, cat]
    yr = torch.full((4,), float(y.max()), dtype=torch.float64)
    ref = _ref_gp(X, y, cat, params)
    ref.append_running_data(torch.from_numpy(Xr), yr)
    eng, dev = _device_gp(engine_cls, X, y, cat, params)
    try:
        dev.append_running_data(torch.from_numpy(Xr), yr)
        xq = np.concatenate([_queries(X, 20, 7), Xr])
        xq[:, cat] = X[:24][:, cat]
        got = eng.gp_query(xq, grad=True)
    finally:
        eng.close()
    want = _ref_query(ref, xq)
    _check_values(want[:2], got[:2])
    _check_grads(want[2:], got[2:])


def test_conditioning_state(engine_cls):
    X, y, cat = _gp_data("float", 30, seed=2)
    params = _params(X.shape[1], 2)
    eng = engine_cls(0)
    try:
        eng.gp_set_data(X, y, cat)
        with pytest.raises(RuntimeError):
            eng.gp_query(X[:2])
        eng.gp_condition(params)
        eng.gp_query(X[:2])
        eng.gp_loss(np.zeros(X.shape[1] + 2), 1e-6)   # overwrites the factor
        with pytest.raises(RuntimeError):
            eng.gp_query(X[:2])
        eng.gp_condition(params)
        eng.gp_posterior_moments(params, X[:3])
        with pytest.raises(RuntimeError):
            eng.gp_query(X[:2])
    finally:
        eng.close()


# ---- optuna's acquisition functions on both GPs --------------------------------------------------------------------

def _acqf_pair(engine_cls, which, X, y, cat, space):
    from optuna._gp import acqf
    engines = []

    def pair(k):
        params = _params(X.shape[1], 10 + k)
        yk = y if k == 0 else np.sin(3.0 * y + k)
        eng, dev = _device_gp(engine_cls, X, yk, cat, params)
        engines.append(eng)
        return _ref_gp(X, yk, cat, params), dev

    g0, g1, c0 = pair(0), pair(1), pair(2)
    Y2 = torch.from_numpy(np.stack([y, np.sin(3.0 * y + 1)], 1))
    running = X[:3] + 0.01 * (1 - 2 * (X[:3] > 0.5))
    running[:, cat] = X[:3][:, cat]
    out = []
    for side in (0, 1):
        if which == "logei":
            a = acqf.LogEI(g0[side], space, float(y.max()))
        elif which == "logei_running":
            a = acqf.LogEI(g0[side], space, float(y.max()), normalized_params_of_running_trials=running.copy())
        elif which == "logei_neginf":
            a = acqf.LogEI(g0[side], space, -np.inf)
        elif which == "constrained_logei":
            a = acqf.ConstrainedLogEI(g0[side], space, float(np.median(y)), [c0[side]], [0.1])
        elif which == "logehvi":
            a = acqf.LogEHVI([g0[side], g1[side]], space, Y2, 128, 7)
        else:
            a = acqf.ConstrainedLogEHVI([g0[side], g1[side]], space, Y2[:20], 128, 7, [c0[side]], [-0.2])
        out.append(a)
    return out, engines


@pytest.mark.parametrize("which", ["logei", "logei_running", "logei_neginf", "constrained_logei", "logehvi",
                                   "constrained_logehvi"])
def test_acquisition_functions(engine_cls, which):
    from optuna._gp import search_space as gp_search_space
    from optuna.search_space import intersection_search_space
    from tests.test_terminator_gpu_gp import _study
    trials = _study("mixed", 80, seed=3).trials
    space = gp_search_space.SearchSpace(intersection_search_space(trials))
    X = space.get_normalized_params(trials)
    y = np.array([t.value for t in trials])
    y = (y - y.mean()) / y.std()
    (ref, dev), engines = _acqf_pair(engine_cls, which, X, y, space.is_categorical, space)
    try:
        xs = space.sample_normalized_params(300, rng=np.random.RandomState(0))
        _check_acqf(ref.eval_acqf_no_grad(xs), dev.eval_acqf_no_grad(xs))
        # with a -inf threshold LogEI is the constant 0, which has no gradient in either
        for x in xs[:6] if which != "logei_neginf" else []:
            vr, gr = ref.eval_acqf_with_grad(x.copy())
            vd, gd = dev.eval_acqf_with_grad(x.copy())
            _check_acqf(np.array([vr]), np.array([vd]))
            assert np.linalg.norm(gd - gr) <= 1e-7 * np.linalg.norm(gr) + 1e-12, (gr, gd)
    finally:
        for e in engines:
            e.close()


def _check_acqf(want, got):
    assert np.all(np.abs(got - want) <= 1e-9 * np.abs(want) + 1e-9), np.max(np.abs(got - want))


# ---- end-to-end replay against optuna.samplers.GPSampler -----------------------------------------------------------

def _dists(kind):
    D = optuna.distributions
    if kind == "cat":
        return {"c": D.CategoricalDistribution([0, 1, 2, 3]), "d": D.CategoricalDistribution(["a", "b"])}
    if kind == "float":
        return {f"x{j}": D.FloatDistribution(-2, 2) for j in range(3)}
    return {"x": D.FloatDistribution(-3, 3), "y": D.FloatDistribution(1e-3, 10, log=True),
            "s": D.FloatDistribution(0, 1, step=0.1), "z": D.IntDistribution(-4, 9),
            "c": D.CategoricalDistribution([0, 1, 2])}


def _values(params, n_obj):
    v = sum((float(p) if not isinstance(p, str) else float(p == "a")) ** 2 * (1 + j)
            for j, p in enumerate(params.values()))
    return [v, -v + 3.0 * float(list(params.values())[0] if not isinstance(list(params.values())[0], str) else 1)][
        :n_obj]


def _constraint_values(params):
    vals = [float(p) if not isinstance(p, str) else float(p == "a") for p in params.values()]
    return [vals[0] - 0.5, 0.3 - abs(vals[-1])]


def _constraints_func(trial):
    """The replayed trials carry their constraint values in their system attributes (``_frozen``), and the asked
    trials are told FAIL, for which optuna does not evaluate constraints: this is never called."""
    raise AssertionError(f"constraints_func called on trial {trial.number}")


def _history(dists, n, n_obj, seed, constrained, running=0):
    """n complete trials (and ``running`` RUNNING ones) at random points of the space."""
    D = optuna.distributions
    rs = np.random.RandomState(seed)
    out = []
    for k in range(n + running):
        params = {}
        for name, d in dists.items():
            if isinstance(d, D.CategoricalDistribution):
                params[name] = d.choices[rs.randint(len(d.choices))]
            elif isinstance(d, D.IntDistribution):
                params[name] = int(rs.randint(d.low, d.high + 1))
            elif d.step is not None:
                params[name] = d.low + d.step * rs.randint(int(round((d.high - d.low) / d.step)) + 1)
            else:
                params[name] = float(rs.uniform(d.low, d.high))
        out.append(_frozen(params, dists, n_obj, constrained, running=k >= n))
    return out


def _frozen(params, dists, n_obj, constrained, running=False):
    attrs = {"constraints": _constraint_values(params)} if constrained else {}
    if running:
        return optuna.trial.create_trial(state=optuna.trial.TrialState.RUNNING, params=params, distributions=dists)
    vals = _values(params, n_obj)
    return optuna.trial.create_trial(params=params, distributions=dists, system_attrs=attrs,
                                     **({"value": vals[0]} if n_obj == 1 else {"values": vals}))


def _normalised(dists, params):
    from optuna._gp import search_space as gp_search_space
    t = optuna.trial.create_trial(params=params, distributions=dists, value=0.0)
    return gp_search_space.SearchSpace(dists).get_normalized_params([t])[0]


def _replay(dists, history, steps, n_obj=1, constrained=False, seed=0, extra=None, **kw):
    """Both samplers on the same history and seed; each step both ask, the asked trials fail, and the reference's
    suggestion joins both histories as a complete trial, so that differences do not compound."""
    from optuna_b200 import GPSampler
    directions = kw.pop("directions", ["minimize"] * n_obj)
    cf = _constraints_func if constrained else None
    ref = optuna.samplers.GPSampler(seed=seed, constraints_func=cf, **kw)
    ours = GPSampler(seed=seed, constraints_func=cf, **kw)
    sa = optuna.create_study(directions=directions, sampler=ref)
    sb = optuna.create_study(directions=directions, sampler=ours)
    for s in (sa, sb):
        s.add_trials(history)
    try:
        for k in range(steps):
            if extra is not None and k in extra:
                for s in (sa, sb):
                    s.add_trial(extra[k])
            ta, tb = sa.ask(dists), sb.ask(dists)
            assert ta.params.keys() == tb.params.keys()
            na, nb = _normalised(dists, ta.params), _normalised(dists, tb.params)
            assert np.max(np.abs(na - nb)) <= 1e-6, (k, ta.params, tb.params)
            ra = {key: v for key, v in sa._storage.get_trial_system_attrs(ta._trial_id).items()
                  if key.startswith("gp:relative_params")}
            rb = {key: v for key, v in sb._storage.get_trial_system_attrs(tb._trial_id).items()
                  if key.startswith("gp:relative_params")}
            assert ra.keys() == rb.keys()
            if ra:
                pa = json.loads("".join(ra[key] for key in sorted(ra)))
                pb = json.loads("".join(rb[key] for key in sorted(rb)))
                assert pa.keys() == pb.keys() and pb == {key: tb.params[key] for key in pb}
            for s, t in ((sa, ta), (sb, tb)):
                s.tell(t, state=optuna.trial.TrialState.FAIL)
                s.add_trial(_frozen(ta.params, dists, n_obj, constrained))
    finally:
        ours.close()


@pytest.mark.parametrize("direction", ["minimize", "maximize"])
def test_replay_single_objective(engine_cls, direction):
    d = _dists("mixed")
    _replay(d, _history(d, 14, 1, 0, False), 3, directions=[direction])


def test_replay_deterministic_objective(engine_cls):
    d = _dists("float")
    _replay(d, _history(d, 12, 1, 1, False), 3, deterministic_objective=True, seed=3)


def test_replay_constrained(engine_cls):
    d = _dists("mixed")
    _replay(d, _history(d, 14, 1, 2, True), 2, constrained=True, seed=1)


@pytest.mark.parametrize("constrained", [False, True])
def test_replay_two_objectives(engine_cls, constrained):
    d = _dists("float")
    _replay(d, _history(d, 14, 2, 3, constrained), 2, n_obj=2, constrained=constrained, seed=2)


def test_replay_running_trials(engine_cls):
    d = _dists("mixed")
    _replay(d, _history(d, 14, 1, 4, False, running=2), 2, seed=4)


def test_replay_startup_edge(engine_cls):
    """9 complete trials: the first ask samples independently; the second, with 10, uses the GP."""
    d = _dists("float")
    _replay(d, _history(d, 9, 1, 5, False), 2, seed=5)


def test_replay_search_space_change(engine_cls):
    """A trial without ``x2`` shrinks the intersection space: both samplers drop their cached GPs."""
    d = _dists("float")
    small = {k: v for k, v in d.items() if k != "x2"}
    extra = {1: optuna.trial.create_trial(params={"x0": 0.1, "x1": -0.4}, distributions=small, value=1.0)}
    _replay(d, _history(d, 12, 1, 6, False), 3, seed=6, extra=extra)


def test_replay_all_categorical(engine_cls):
    d = _dists("cat")
    _replay(d, _history(d, 12, 1, 7, False), 2, seed=7)


def test_parallel_trials(engine_cls):
    """``study.optimize(n_jobs=4)`` samples on four threads that share the sampler's engines: every trial completes
    and the GP-chosen ones have a complete parameter set."""
    from optuna_b200 import GPSampler

    def obj(t):
        return sum((t.suggest_float(f"x{j}", -2, 2) - 0.3 * j) ** 2 for j in range(3)) + t.suggest_int("z", 0, 5)

    sampler = GPSampler(seed=0, n_startup_trials=4)
    study = optuna.create_study(sampler=sampler)
    try:
        study.optimize(obj, n_trials=24, n_jobs=4)
    finally:
        sampler.close()
    assert [t.state for t in study.trials] == [optuna.trial.TrialState.COMPLETE] * 24
    assert all(len(t.params) == 4 for t in study.trials)


def test_fit_failure_falls_back(engine_cls, monkeypatch, caplog):
    """Every L-BFGS-B fit fails: both samplers warn and continue with the default kernel parameters."""
    import scipy.optimize
    real = scipy.optimize.minimize

    def failing(fun, x0, **kw):
        res = real(fun, x0, **kw)
        res.success = False
        res.message = "forced failure"
        return res

    monkeypatch.setattr(scipy.optimize, "minimize", failing)
    d = _dists("float")
    with caplog.at_level(logging.WARNING):
        _replay(d, _history(d, 11, 1, 8, False), 1, seed=8)
    msgs = [r.getMessage() for r in caplog.records if "optimization of kernel parameters failed" in r.getMessage()]
    assert len(msgs) == 2 and msgs[0] == msgs[1], msgs
    assert "forced failure" in msgs[0] and "default initial kernel parameters will be used" in msgs[0]


# ---- GPU only --------------------------------------------------------------------------------------------------------

def _large_history(n, P, seed=0):
    D = optuna.distributions
    dists = {f"x{j}": D.FloatDistribution(0, 1) for j in range(P)}
    rs = np.random.RandomState(seed)
    X = rs.uniform(0, 1, (n, P))
    vals = ((X - 0.3) ** 2 * np.arange(1, P + 1)).sum(1)
    return dists, [optuna.trial.create_trial(params={f"x{j}": float(x[j]) for j in range(P)}, distributions=dists,
                                             value=float(v)) for x, v in zip(X, vals)]


@pytest.mark.gpu
def test_large_study_against_reference():
    dists, hist = _large_history(3000, 8)
    _replay(dists, hist, 1, seed=0)


@pytest.mark.gpu
def test_same_seed_same_bits():
    from optuna_b200 import GPSampler
    dists, hist = _large_history(400, 8, seed=1)
    got = []
    for _ in range(2):
        s = GPSampler(seed=3)
        study = optuna.create_study(sampler=s)
        study.add_trials(hist)
        got.append(study.ask(dists).params)
        s.close()
    assert got[0] == got[1]


@pytest.mark.gpu
def test_tpe_suggestion_unchanged():
    from optuna_b200 import B200TPESampler, GPSampler
    dists, hist = _large_history(300, 4, seed=2)

    def tpe_params():
        s = B200TPESampler(seed=0, multivariate=True)
        study = optuna.create_study(sampler=s)
        study.add_trials(hist)
        p = study.ask(dists).params
        s.close()
        return p

    before = tpe_params()
    g = GPSampler(seed=0)
    study = optuna.create_study(sampler=g)
    study.add_trials(hist)
    study.ask(dists)
    after = tpe_params()
    g.close()
    assert before == after


@pytest.mark.gpu
def test_posterior_bits_unchanged_by_queries():
    """The posterior calls return the same bits before and after conditioning and gradient queries."""
    from optuna_b200 import TPEEngine
    X, y, cat = _gp_data("mixed", 200, seed=9)
    prm = np.concatenate([np.full(X.shape[1], 0.5), [1.1, 1e-4]])
    Xq = np.concatenate([X, np.random.RandomState(1).uniform(0, 1, (2048, X.shape[1]))])
    eng = TPEEngine(0)
    try:
        eng.gp_set_data(X, y, cat)
        before = eng.gp_posterior(prm, Xq, 2.5) + eng.gp_posterior_moments(prm, Xq, 3)
        eng.gp_condition(prm)
        q = eng.gp_query(Xq, grad=True)
        after = eng.gp_posterior(prm, Xq, 2.5) + eng.gp_posterior_moments(prm, Xq, 3)
        for a, b in zip(before, after):
            assert a.tobytes() == b.tobytes()
        # the conditioned query returns the moments' bits
        assert q[0].tobytes() == before[2].tobytes() and q[1].tobytes() == before[3].tobytes()
    finally:
        eng.close()
