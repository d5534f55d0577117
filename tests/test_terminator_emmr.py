"""``optuna_b200.EMMREvaluator`` against the live reference's ``optuna.terminator.EMMREvaluator``
(optuna/terminator/improvement/emmr.py, optuna/_gp/gp.py).

Every case runs twice: through ``NumpyEMMREngine`` (tests/_emmr_engine.py: the device algorithm in NumPy, runs
anywhere) and, with ``-m gpu``, through libtpe_b200.so.  Tolerances:
- the fixed-noise loss within 1e-10 relative and its gradient within 1e-8 of its norm (at the points of a replayed
  fit: of the larger of its norm and the size of its likelihood and prior parts, which cancel near the optimum);
- the posterior mean within 1e-8 (1 + |mean|), variance and covariance within 1e-12 ks;
- the criterion within 1e-6 relative (1e-9 absolute near 0) with the noise fitted, and 1e-5 relative with
  ``deterministic_objective=True``: there x_t's posterior variance (about 6e-7 at the fixed noise 1e-6) is
  multiplied by 1 / noise = 1e6 in the KL term.
"""
from __future__ import annotations

import logging
import math
import sys
import warnings

import numpy as np
import pytest

optuna = pytest.importorskip("optuna")
torch = pytest.importorskip("torch")

from tests.test_terminator_gpu_gp import _gp_data, _objective, _prior_grad, _random_raws, _study  # noqa: E402

MIN_NOISE = 1e-6
MIN = optuna.study.StudyDirection.MINIMIZE
MAX = optuna.study.StudyDirection.MAXIMIZE


@pytest.fixture(params=[pytest.param("numpy", id="numpy-engine"),
                        pytest.param("cuda", id="cuda-engine", marks=pytest.mark.gpu)])
def engine_cls(request, monkeypatch):
    """The engine class behind optuna_b200.terminator: the NumPy restatement or the CUDA library."""
    from optuna_b200 import TPEEngine, terminator
    from tests._emmr_engine import NumpyEMMREngine
    cls = NumpyEMMREngine if request.param == "numpy" else TPEEngine
    monkeypatch.setattr(terminator, "_engine_cls", cls)
    return cls


# ---- the fixed-noise loss -------------------------------------------------------------------------------------------

def _ref_loss_fixed(X, y, cat, raw):
    """loss_func of GPRegressor._fit_kernel_params with deterministic_objective=True (optuna/_gp/gp.py:312-327)."""
    from optuna._gp.gp import GPRegressor
    from optuna._gp.prior import default_log_prior
    P = X.shape[1]
    one = torch.tensor(1.0, dtype=torch.float64)
    gpr = GPRegressor(torch.from_numpy(cat), torch.from_numpy(X), torch.from_numpy(y),
                      torch.ones(P, dtype=torch.float64), one.clone(), one.clone())
    raw_t = torch.from_numpy(np.array(raw, dtype=np.float64)).requires_grad_(True)
    with torch.enable_grad():
        gpr.inverse_squared_lengthscales = torch.exp(raw_t[:P])
        gpr.kernel_scale = torch.exp(raw_t[P])
        gpr.noise_var = torch.tensor(MIN_NOISE, dtype=torch.float64)
        loss = -gpr.marginal_log_likelihood() - default_log_prior(gpr)
        loss.backward()
    return loss.item(), raw_t.grad.numpy()


def _our_loss_fixed(engine_cls, X, y, cat, raws):
    from optuna._gp.prior import default_log_prior
    from optuna_b200.terminator import _loss_and_grad
    eng = engine_cls(0)
    try:
        eng.gp_set_data(X, y, cat)
        return [_loss_and_grad(eng, np.asarray(r, dtype=np.float64), X.shape[1], default_log_prior, MIN_NOISE, True)
                for r in raws]
    finally:
        eng.close()


def _check_loss(want, got, scale=None):
    (lw, gw), (lg, gg) = want, got
    assert abs(lg - lw) <= 1e-10 * abs(lw), (lw, lg)
    ref = np.linalg.norm(gw) if scale is None else scale
    assert np.linalg.norm(gg - gw) <= 1e-8 * ref, (gw, gg, ref)
    assert gg[-1] == 0.0 and gw[-1] == 0.0


@pytest.mark.parametrize("kind,n,dup", [("mixed", 40, False), ("mixed", 30, True), ("float", 25, False),
                                        ("p1", 20, False), ("cat", 24, False), ("mixed", 2, False),
                                        # several 64-wide blocks, n not a multiple of 64; P = 17 and 33
                                        ("mixed", 150, True), ("mixed", 257, False), ("wide17", 130, True),
                                        ("wide33", 150, False)])
def test_fixed_noise_loss_known_answers(engine_cls, kind, n, dup):
    X, y, cat = _gp_data(kind, n, seed=n, duplicates=dup)
    # the raw noise entry is ignored: the loss must not move when it does
    raws = [np.concatenate([r[:-1], [v]]) for r in _random_raws(X.shape[1], n) for v in (r[-1], r[-1] + 3.0)]
    raws.append(np.zeros(X.shape[1] + 2))
    got = _our_loss_fixed(engine_cls, X, y, cat, raws)
    for raw, g in zip(raws, got):
        _check_loss(_ref_loss_fixed(X, y, cat, raw), g)
    for k in range(0, len(raws) - 1, 2):
        assert got[k][0] == got[k + 1][0] and got[k][1].tobytes() == got[k + 1][1].tobytes()


@pytest.mark.parametrize("kind,n", [("mixed", 60), ("float", 40), ("cat", 30), ("p1", 25), ("mixed", 257),
                                    ("wide17", 150), ("wide33", 200)])
def test_replay_of_reference_deterministic_fit(engine_cls, kind, n, monkeypatch):
    """Every raw-parameter vector at which the reference's loss_func is called during one deterministic fit."""
    import scipy.optimize
    from optuna._gp import gp
    from optuna._gp.prior import default_log_prior
    X, y, cat = _gp_data(kind, n, seed=3)
    seen = []
    real = scipy.optimize.minimize

    def recording(fun, x0, **kw):
        def wrapped(x):
            seen.append(np.array(x, dtype=np.float64))
            return fun(x)
        return real(wrapped, x0, **kw)

    monkeypatch.setattr(scipy.optimize, "minimize", recording)
    gp.fit_kernel_params(X, y, cat, default_log_prior, MIN_NOISE, True)
    monkeypatch.setattr(scipy.optimize, "minimize", real)
    assert len(seen) >= 2
    for raw, got in zip(seen, _our_loss_fixed(engine_cls, X, y, cat, seen)):
        want = _ref_loss_fixed(X, y, cat, raw)
        g_prior = _prior_grad(raw, X.shape[1])
        g_prior[-1] = 0.0   # the prior sees the fixed noise as a constant
        scale = max(np.linalg.norm(want[1]), np.linalg.norm(want[1] - g_prior) + np.linalg.norm(g_prior))
        _check_loss(want, got, scale)


# ---- posterior moments ----------------------------------------------------------------------------------------------

def _ref_gpr(X, y, cat, params):
    from optuna._gp.gp import GPRegressor
    P = X.shape[1]
    p = torch.from_numpy(np.array(params, dtype=np.float64))
    gpr = GPRegressor(torch.from_numpy(cat), torch.from_numpy(X), torch.from_numpy(y), p[:P].clone(), p[P].clone(),
                      p[P + 1].clone())
    gpr._cache_matrix()
    return gpr


def _fitted_params(X, y, cat, deterministic):
    from optuna._gp import gp
    from optuna._gp.prior import default_log_prior
    g = gp.fit_kernel_params(X, y, cat, default_log_prior, MIN_NOISE, deterministic)
    return np.concatenate([g.inverse_squared_lengthscales.numpy(), [g.kernel_scale.item(), g.noise_var.item()]])


@pytest.mark.parametrize("kind,n,deterministic", [("mixed", 60, False), ("mixed", 60, True), ("cat", 30, False),
                                                  ("p1", 25, True), ("float", 40, True), ("wide17", 150, False),
                                                  ("mixed", 257, True)])
def test_posterior_moments(engine_cls, kind, n, deterministic):
    X, y, cat = _gp_data(kind, n, seed=5)
    params = _fitted_params(X, y, cat, deterministic)
    ks = params[X.shape[1]]
    gpr = _ref_gpr(X, y, cat, params)
    rs = np.random.RandomState(n)
    Xr = rs.uniform(0, 1, (40, X.shape[1]))
    Xr[:, cat] = X[rs.randint(0, n, 40)][:, cat]
    # theta pairs: two training points, a duplicated point, a training point with a random one, then the rest
    Xq = np.concatenate([X[[3, n - 1]], X[[5, 5]], X[[7]], Xr[[0]], X, Xr])
    eng = engine_cls(0)
    try:
        eng.gp_set_data(X, y, cat)
        mean, var, cov0 = eng.gp_posterior_moments(params, Xq)
        assert cov0.shape == (0, 0)
        for j0, J in ((0, 2), (2, 2), (4, 2), (0, 6)):
            m2, v2, cov = eng.gp_posterior_moments(params, Xq[j0:], J)
            if engine_cls.__name__ == "TPEEngine":   # on the device a row's result does not depend on the others
                np.testing.assert_array_equal(m2, mean[j0:])
                np.testing.assert_array_equal(v2, var[j0:])
                assert np.array_equal(cov, cov.T)
            else:                                    # NumPy's matrix products block by shape
                np.testing.assert_allclose(m2, mean[j0:], rtol=1e-9, atol=1e-9)
                np.testing.assert_allclose(v2, var[j0:], rtol=0, atol=1e-13 * ks)
            _, want_cov = gpr.posterior(torch.from_numpy(Xq[j0:j0 + J]), joint=True)
            assert np.abs(cov - want_cov.numpy()).max() <= 1e-12 * ks, (cov, want_cov)
            assert np.all(np.diag(cov) >= 0.0)
    finally:
        eng.close()
    want_mean, want_var = (t.numpy() for t in gpr.posterior(torch.from_numpy(Xq)))
    assert np.all(np.abs(mean - want_mean) <= 1e-8 * (1.0 + np.abs(want_mean))), np.abs(mean - want_mean).max()
    assert np.abs(var - want_var).max() <= 1e-12 * ks
    assert np.all(var >= 0.0)


def test_posterior_moments_arguments(engine_cls):
    X, y, cat = _gp_data("mixed", 30, seed=2)
    eng = engine_cls(0)
    try:
        eng.gp_set_data(X, y, cat)
        prm = np.ones(X.shape[1] + 2)
        # n_joint is 0 or in [2, 64], and at most the number of points
        for Xq, bad in ((X, 1), (X, 31), (np.tile(X, (3, 1)), 65)):
            with pytest.raises(ValueError):
                eng.gp_posterior_moments(prm, Xq, bad)
        assert eng.gp_posterior_moments(prm, np.tile(X, (3, 1)), 64)[2].shape == (64, 64)
    finally:
        eng.close()


# ---- end to end ---------------------------------------------------------------------------------------------------

def _close(want, got, rel=1e-6):
    assert abs(got - want) <= max(rel * abs(want), 1e-9), (want, got)


def _compare(trials, direction=MIN, seed=0, **kw):
    import optuna_b200
    want = optuna.terminator.EMMREvaluator(seed=seed, **kw).evaluate(trials, direction)
    got = optuna_b200.EMMREvaluator(seed=seed, **kw).evaluate(trials, direction)
    _close(want, got, 1e-5 if kw.get("deterministic_objective") else 1e-6)
    return want, got


@pytest.mark.parametrize("kind", ["mixed", "float", "cat", "p1"])
@pytest.mark.parametrize("direction", ["minimize", "maximize"])
@pytest.mark.parametrize("seed", [0, 7])
@pytest.mark.parametrize("deterministic", [False, True])
def test_end_to_end(engine_cls, kind, direction, seed, deterministic):
    _compare(_study(kind, 40, seed=seed, direction=direction).trials, MIN if direction == "minimize" else MAX,
             seed=seed, deterministic_objective=deterministic)


@pytest.mark.parametrize("delta,deterministic", [(0.05, False), (0.3, True)])
def test_end_to_end_delta(engine_cls, delta, deterministic):
    _compare(_study("mixed", 50, seed=3).trials, seed=1, delta=delta, deterministic_objective=deterministic)


@pytest.mark.parametrize("kind,n", [("wide17", 130), ("mixed", 257)])
def test_end_to_end_blocked(engine_cls, kind, n):
    """GPs over several 64-wide blocks with P = 17 and 5."""
    _compare(_study(kind, n, seed=11).trials, seed=4)


@pytest.mark.parametrize("min_n,n", [(2, 2), (5, 5), (5, 4), (2, 1), (2, 0)])
def test_min_n_trials(engine_cls, min_n, n):
    want, got = _compare(_study("mixed", n, seed=2).trials, min_n_trials=min_n)
    if n < min_n:
        assert want == got == sys.float_info.max * 0.1


def _warned(fn):
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        value = fn()
    return value, [(x.category, str(x.message)) for x in w if not issubclass(x.category, optuna.exceptions.ExperimentalWarning)]


def test_empty_search_space(engine_cls):
    import optuna_b200
    study = optuna.create_study()
    study.optimize(lambda t: t.suggest_float("x", 0, 1) if t.number % 2 else t.suggest_float("y", 0, 1), n_trials=6)
    want, w_want = _warned(lambda: optuna.terminator.EMMREvaluator().evaluate(study.trials, MIN))
    got, w_got = _warned(lambda: optuna_b200.EMMREvaluator().evaluate(study.trials, MIN))
    assert want == got == sys.float_info.max * 0.1
    assert w_want == w_got and len(w_want) == 1 and "cannot consider any search space" in w_want[0][1]


def test_infinite_objective_value(engine_cls):
    import optuna_b200
    study = _study("mixed", 30, seed=4)
    t = study.trials[5]
    study.add_trial(optuna.trial.create_trial(params=t.params, distributions=t.distributions, value=float("inf")))
    study.optimize(_objective("mixed", 4), n_trials=5)
    want, w_want = _warned(lambda: optuna.terminator.EMMREvaluator(seed=2).evaluate(study.trials, MIN))
    got, w_got = _warned(lambda: optuna_b200.EMMREvaluator(seed=2).evaluate(study.trials, MIN))
    assert w_want == w_got and any("Clip non-finite values" in m for _, m in w_want)
    _close(want, got)


def test_other_trial_states(engine_cls):
    study = optuna.create_study(sampler=optuna.samplers.RandomSampler(seed=4))
    obj = _objective("mixed", 4)

    def objective(t):
        if t.number % 7 == 3:
            raise optuna.TrialPruned()
        if t.number % 11 == 5:
            raise RuntimeError("fail")
        return obj(t)

    study.optimize(objective, n_trials=50, catch=(RuntimeError,))
    running = study.ask()
    running.suggest_float("x", -3, 3)
    trials = study.get_trials(deepcopy=False)
    assert {t.state for t in trials} >= {optuna.trial.TrialState.PRUNED, optuna.trial.TrialState.FAIL,
                                         optuna.trial.TrialState.RUNNING}
    _compare(trials, seed=3)


def test_constant_objective(engine_cls):
    study = optuna.create_study(sampler=optuna.samplers.RandomSampler(seed=0))
    study.optimize(lambda t: 0.0 * t.suggest_float("x", 0, 1) + 1.5, n_trials=30)
    _compare(study.trials)


@pytest.mark.parametrize("last_is_best", [True, False])
def test_best_trial_last_or_earlier(engine_cls, last_is_best):
    """The best trial last: theta*_t is x_t and differs from theta*_{t-1} (the joint covariance); the best trial
    earlier: theta*_t = theta*_{t-1} (the variance)."""
    study = _study("float", 40, seed=6)
    t = study.trials[0]
    best = min(s.value for s in study.trials)
    params = {k: 0.3 for k in t.params} if last_is_best else {k: 1.9 for k in t.params}
    study.add_trial(optuna.trial.create_trial(params=params, distributions=t.distributions,
                                              value=_objective("float", 6)(optuna.trial.FixedTrial(params))))
    assert (study.trials[-1].value < best) == last_is_best
    for det in (False, True):
        _compare(study.trials, seed=5, deterministic_objective=det)


def test_fit_failure_falls_back(engine_cls, monkeypatch, caplog):
    """Both fits fail twice: each logs the warning and uses the default GP (noise_var 1.0, even deterministic)."""
    import scipy.optimize
    real = scipy.optimize.minimize

    def failing(*args, **kw):
        res = real(*args, **kw)
        res.success = False
        res.message = "patched failure"
        return res

    monkeypatch.setattr(scipy.optimize, "minimize", failing)
    trials = _study("mixed", 40, seed=5).trials
    optuna.logging.enable_propagation()
    try:
        for det in (False, True):
            caplog.clear()
            with caplog.at_level(logging.WARNING):
                import optuna_b200
                want = optuna.terminator.EMMREvaluator(seed=1, deterministic_objective=det).evaluate(trials, MIN)
                n_ref = len(caplog.records)
                got = optuna_b200.EMMREvaluator(seed=1, deterministic_objective=det).evaluate(trials, MIN)
            ref = [r.getMessage() for r in caplog.records[:n_ref] if r.name == "optuna._gp.gp"]
            ours = [r.getMessage() for r in caplog.records[n_ref:] if r.name == "optuna.terminator.optuna_b200"]
            # one warning per fit (caplog may hold each record twice, the same way for both)
            assert len(set(ref)) == 1 and len(ref) >= 2 and ref == ours, (ref, ours)
            assert "patched failure" in ref[0]
            _close(want, got, 1e-5 if det else 1e-6)
    finally:
        optuna.logging.disable_propagation()


def test_median_error_evaluator(engine_cls):
    import optuna_b200
    from optuna.terminator import MedianErrorEvaluator
    trials = _study("mixed", 40, seed=8).trials
    want = MedianErrorEvaluator(optuna.terminator.EMMREvaluator(seed=0)).evaluate(trials, MIN)
    got = MedianErrorEvaluator(optuna_b200.EMMREvaluator(seed=0)).evaluate(trials, MIN)
    _close(want, got)


def _terminated_at(improvement, error):
    # The reference stops this study after trial 56.  From trial 20 on, the criterion and the threshold differ by at
    # least 38 % of the threshold, far above the tolerance.
    from optuna.terminator import Terminator, TerminatorCallback
    study = optuna.create_study(sampler=optuna.samplers.TPESampler(seed=0))
    cb = TerminatorCallback(Terminator(improvement_evaluator=improvement, error_evaluator=error))
    study.optimize(_objective("mixed", 0), n_trials=80, callbacks=[cb])
    return len(study.trials)


def test_terminator_callback_stops_at_same_trial(engine_cls):
    import optuna_b200
    from optuna.terminator import MedianErrorEvaluator
    ref = optuna.terminator.EMMREvaluator(seed=0)
    want = _terminated_at(ref, MedianErrorEvaluator(ref))
    ours = optuna_b200.EMMREvaluator(seed=0)
    got = _terminated_at(ours, MedianErrorEvaluator(ours))
    assert want == got and want < 80, (want, got)


def test_improvement_info(engine_cls):
    import optuna_b200
    from optuna.terminator import MedianErrorEvaluator
    from optuna.visualization._terminator_improvement import _get_improvement_info
    study = _study("mixed", 34, seed=6)
    ref = optuna.terminator.EMMREvaluator(seed=0)
    want = _get_improvement_info(study, True, ref, MedianErrorEvaluator(ref))
    ours = optuna_b200.EMMREvaluator(seed=0)
    got = _get_improvement_info(study, True, ours, MedianErrorEvaluator(ours))
    assert want.trial_numbers == got.trial_numbers
    for a, b in zip(want.improvements, got.improvements):
        _close(a, b)
    for a, b in zip(want.errors, got.errors):
        _close(a, b)


def test_api():
    import optuna_b200
    from optuna_b200.terminator import EMMREvaluator
    assert optuna_b200.EMMREvaluator is EMMREvaluator
    assert issubclass(EMMREvaluator, optuna.terminator.EMMREvaluator)
    for bad in (1, 0, float("inf")):
        with pytest.raises(ValueError) as a:
            optuna.terminator.EMMREvaluator(min_n_trials=bad)
        with pytest.raises(ValueError) as b:
            EMMREvaluator(min_n_trials=bad)
        assert str(a.value) == str(b.value)
    with pytest.warns(optuna.exceptions.ExperimentalWarning):
        EMMREvaluator(device=0)


# ---- on the GPU only ------------------------------------------------------------------------------------------------

def _large_study(n, P, seed=0):
    rs = np.random.RandomState(seed)
    study = optuna.create_study()
    dists = {f"x{j}": optuna.distributions.FloatDistribution(0.0, 1.0) for j in range(P)}
    X = rs.uniform(0, 1, (n, P))
    v = ((X - 0.3) ** 2 * np.arange(1, P + 1)).sum(1) + 0.05 * rs.randn(n)
    study.add_trials([optuna.trial.create_trial(params={f"x{j}": X[i, j] for j in range(P)}, distributions=dists,
                                                value=float(v[i])) for i in range(n)])
    return study


@pytest.mark.gpu
def test_large_study_against_reference():
    """3 000 complete trials x 8 parameters: two GPs over 2 999 and 3 000 points."""
    import optuna_b200
    trials = _large_study(3000, 8).trials
    want = optuna.terminator.EMMREvaluator(seed=0).evaluate(trials, MIN)
    got = optuna_b200.EMMREvaluator(seed=0).evaluate(trials, MIN)
    _close(want, got)


@pytest.mark.gpu
def test_same_seed_same_bits():
    import optuna_b200
    from optuna_b200 import TPEEngine
    trials = _study("mixed", 300, seed=8).trials
    for det in (False, True):
        a = optuna_b200.EMMREvaluator(seed=5, deterministic_objective=det).evaluate(trials, MIN)
        b = optuna_b200.EMMREvaluator(seed=5, deterministic_objective=det).evaluate(trials, MIN)
        assert np.float64(a).tobytes() == np.float64(b).tobytes()
    X, y, cat = _gp_data("mixed", 300, seed=8)
    eng = TPEEngine(0)
    try:
        eng.gp_set_data(X, y, cat)
        prm = np.concatenate([np.full(X.shape[1], 0.7), [1.3, 1e-3]])
        Xq = np.concatenate([X[:40], np.random.RandomState(0).uniform(0, 1, (2100, X.shape[1]))])
        r1 = eng.gp_posterior_moments(prm, Xq, 40)
        r2 = eng.gp_posterior_moments(prm, Xq, 40)
        for a, b in zip(r1, r2):
            assert a.tobytes() == b.tobytes()
        l1, g1 = eng.gp_loss(_random_raws(X.shape[1], 1, 1)[0], MIN_NOISE, deterministic=True)
        l2, g2 = eng.gp_loss(_random_raws(X.shape[1], 1, 1)[0], MIN_NOISE, deterministic=True)
        assert l1 == l2 and g1.tobytes() == g2.tobytes()
    finally:
        eng.close()


@pytest.mark.gpu
def test_posterior_bounds_unchanged_by_moments():
    from optuna_b200 import TPEEngine
    X, y, cat = _gp_data("mixed", 200, seed=9)
    prm = np.concatenate([np.full(X.shape[1], 0.5), [1.1, 1e-4]])
    Xq = np.concatenate([X, np.random.RandomState(1).uniform(0, 1, (2048, X.shape[1]))])
    eng = TPEEngine(0)
    try:
        eng.gp_set_data(X, y, cat)
        before = eng.gp_posterior(prm, Xq, 2.5)
        mean, var, _ = eng.gp_posterior_moments(prm, Xq, 3)
        after = eng.gp_posterior(prm, Xq, 2.5)
        for a, b in zip(before, after):
            assert a.tobytes() == b.tobytes()
        # the bounds are the moments' mean +- sqrt(beta var)
        np.testing.assert_allclose(before[0], mean + np.sqrt(2.5 * var), rtol=0, atol=1e-14)
    finally:
        eng.close()


@pytest.mark.gpu
def test_engine_suggestion_unchanged_by_new_gp_calls():
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
        Xg, yg, cat = _gp_data("mixed", 200, seed=9)
        eng.gp_set_data(Xg, yg, cat)
        eng.gp_loss(np.zeros(Xg.shape[1] + 2), MIN_NOISE, deterministic=True)
        eng.gp_posterior_moments(np.ones(Xg.shape[1] + 2), Xg[:10], 2)
        after = eng.suggest(list(range(P)), u, 1, **cfg)
        for a, b in zip(before, after):
            np.testing.assert_array_equal(a, b)
    finally:
        eng.close()


def test_joint_cov_kernel_does_not_spill():
    """ptxas -v over the joint-covariance and finishing kernels: no spill stores or loads."""
    import os
    import re
    import shutil
    import subprocess
    import tempfile
    nvcc = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)
    if nvcc is None:
        pytest.skip("nvcc is not available")
    csrc = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "optuna_b200", "csrc")
    with tempfile.TemporaryDirectory() as tmp:
        src = os.path.join(tmp, "gp_only.cu")
        with open(src, "w") as f:
            f.write(f'#include "{csrc}/tpe_kernels.cuh"\n#include "{csrc}/tpe_gp.cuh"\n')
        out = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-c",
                              "-Xptxas", "-v", "-o", os.path.join(tmp, "gp.o"), src],
                             capture_output=True, text=True, check=True).stderr
    blocks = re.split(r"Compiling entry function", out)
    new = [b for b in blocks if re.search(r"k_gp_joint_cov|k_gp_post_finish", b.split("\n", 1)[0])]
    assert len(new) == 2, out
    for b in new:
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", b)
        assert m and m.group(1) == "0" and m.group(2) == "0", b
