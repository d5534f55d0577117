"""``optuna_b200.RegretBoundEvaluator`` against the live reference's ``optuna.terminator.RegretBoundEvaluator``
(optuna/terminator/improvement/evaluator.py, optuna/_gp/gp.py).

Every case runs twice: through ``NumpyGPEngine`` (tests/_gp_engine.py: the device algorithm in NumPy, runs anywhere)
and, with ``-m gpu``, through libtpe_b200.so.  Tolerances: the loss within 1e-10 relative and the gradient within
1e-8 of its norm against the reference's GPRegressor + default_log_prior + autograd (at the points of a replayed fit:
of the larger of its norm and the size of its likelihood and prior parts, which cancel near the optimum -- DESIGN.md
lists the measured ratios); the regret bound within 1e-6 relative (1e-9 absolute near 0).
"""
from __future__ import annotations

import logging
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

optuna = pytest.importorskip("optuna")
torch = pytest.importorskip("torch")

MIN_NOISE = 1e-6


@pytest.fixture(params=[pytest.param("numpy", id="numpy-engine"),
                        pytest.param("cuda", id="cuda-engine", marks=pytest.mark.gpu)])
def engine_cls(request, monkeypatch):
    """The engine class behind optuna_b200.terminator: the NumPy restatement or the CUDA library."""
    from optuna_b200 import TPEEngine, terminator
    from tests._gp_engine import NumpyGPEngine
    cls = NumpyGPEngine if request.param == "numpy" else TPEEngine
    monkeypatch.setattr(terminator, "_engine_cls", cls)
    return cls


def _objective(kind, seed=0):
    rs = np.random.RandomState(seed)
    w = rs.uniform(0.5, 2.0, 8)

    def obj(t):
        if kind == "float":
            return sum(w[j] * (t.suggest_float(f"x{j}", -2, 2) - 0.3) ** 2 for j in range(3))
        if kind == "p1":
            return (t.suggest_float("x", 0, 1) - 0.4) ** 2
        if kind in ("wide17", "wide33"):
            # 15 or 28 floats, then categoricals (and in wide33 an int, a log float and a stepped float): more than
            # 16 columns, so the gradient takes two or three passes of k_gp_grad
            nf = 15 if kind == "wide17" else 28
            v = sum((1.0 / (1 + j)) * (t.suggest_float(f"f{j}", -1, 1) - 0.2) ** 2 for j in range(nf))
            v += w[t.suggest_categorical("c", [0, 1, 2])] + 0.3 * w[int(t.suggest_categorical("d", ["a", "b"]) == "a")]
            if kind == "wide33":
                v += 0.05 * t.suggest_int("z", 0, 10) + 0.1 * math.log(t.suggest_float("g", 1e-3, 1, log=True))
                v += t.suggest_float("s", 0, 1, step=0.25)
            return v
        if kind == "cat":
            return w[t.suggest_categorical("c", [0, 1, 2, 3])] + 0.5 * w[int(t.suggest_categorical("d", ["a", "b"]) == "a")]
        x = t.suggest_float("x", -3, 3)
        y = t.suggest_float("y", 1e-3, 10, log=True)
        s = t.suggest_float("s", 0, 1, step=0.1)
        z = t.suggest_int("z", -4, 9)
        c = t.suggest_categorical("c", [0, 1, 2])
        return x * x + 0.3 * math.log(y) + s + 0.1 * z + w[c]
    return obj


def _study(kind, n, seed=0, direction="minimize"):
    study = optuna.create_study(direction=direction, sampler=optuna.samplers.RandomSampler(seed=seed))
    study.optimize(_objective(kind, seed), n_trials=n)
    return study


def _gp_data(kind, n, seed=0, duplicates=False):
    from optuna._gp import search_space as gp_search_space
    from optuna.search_space import intersection_search_space
    trials = _study(kind, n, seed).trials
    if duplicates:
        trials = trials + trials[: max(1, n // 3)]
    space = gp_search_space.SearchSpace(intersection_search_space(trials))
    X = space.get_normalized_params(trials)
    y = np.array([t.value for t in trials])
    y = (y - y.mean()) / max(1e-10, y.std())
    return X, y, space.is_categorical


def _ref_loss(X, y, cat, raw, min_noise=MIN_NOISE):
    """loss_func of GPRegressor._fit_kernel_params (optuna/_gp/gp.py:312-327)."""
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
        gpr.noise_var = torch.exp(raw_t[P + 1]) + min_noise
        loss = -gpr.marginal_log_likelihood() - default_log_prior(gpr)
        loss.backward()
    return loss.item(), raw_t.grad.numpy()


def _our_loss(engine_cls, X, y, cat, raws):
    from optuna._gp.prior import default_log_prior
    from optuna_b200.terminator import _loss_and_grad
    eng = engine_cls(0)
    try:
        eng.gp_set_data(X, y, cat)
        return [_loss_and_grad(eng, np.asarray(r, dtype=np.float64), X.shape[1], default_log_prior, MIN_NOISE)
                for r in raws]
    finally:
        eng.close()


def _check_loss(want, got, scale=None):
    """Loss within 1e-10 relative, gradient within 1e-8 of its norm -- or of ``scale``, the norm of the two parts
    it is the sum of, where they cancel (near the optimum of a fit)."""
    (lw, gw), (lg, gg) = want, got
    assert abs(lg - lw) <= 1e-10 * abs(lw), (lw, lg)
    ref = np.linalg.norm(gw) if scale is None else scale
    assert np.linalg.norm(gg - gw) <= 1e-8 * ref, (gw, gg, ref)


def _prior_grad(raw, P):
    from optuna._gp.prior import default_log_prior
    from optuna_b200.terminator import _KernelParams
    r = torch.from_numpy(np.array(raw, dtype=np.float64)).requires_grad_(True)
    with torch.enable_grad():
        (-default_log_prior(_KernelParams(torch.exp(r[:P]), torch.exp(r[P]), torch.exp(r[P + 1]) + MIN_NOISE))).backward()
    return r.grad.numpy()


def _random_raws(P, seed, k=3):
    rs = np.random.RandomState(seed)
    return [np.concatenate([rs.uniform(-2.0, 1.5, P), [rs.uniform(-1.0, 1.0), rs.uniform(-8.0, 0.0)]])
            for _ in range(k)]


@pytest.mark.parametrize("kind,n,dup", [("mixed", 40, False), ("mixed", 30, True), ("float", 25, False),
                                        ("p1", 20, False), ("cat", 24, False), ("mixed", 1, False),
                                        ("mixed", 2, False), ("p1", 2, True),
                                        # several 64-wide blocks, n not a multiple of 64 (150 + 50 duplicates,
                                        # 257, 130 + 43, 257 + 85), P = 5, 17 and 33
                                        ("mixed", 150, True), ("mixed", 257, False), ("wide17", 130, True),
                                        ("wide17", 257, False), ("wide33", 150, False), ("wide33", 257, True)])
def test_loss_and_gradient_known_answers(engine_cls, kind, n, dup):
    X, y, cat = _gp_data(kind, n, seed=n, duplicates=dup)
    assert X.shape[1] == {"mixed": 5, "float": 3, "p1": 1, "cat": 2, "wide17": 17, "wide33": 33}[kind]
    raws = _random_raws(X.shape[1], n) + [np.zeros(X.shape[1] + 2)]
    for raw, got in zip(raws, _our_loss(engine_cls, X, y, cat, raws)):
        _check_loss(_ref_loss(X, y, cat, raw), got)


@pytest.mark.parametrize("kind,n", [("mixed", 60), ("float", 40), ("mixed", 257), ("wide33", 200)])
def test_replay_of_reference_fit(engine_cls, kind, n, monkeypatch):
    """Every raw-parameter vector at which the reference's loss_func is called during one fit."""
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
    gp.fit_kernel_params(X, y, cat, default_log_prior, MIN_NOISE, False)
    monkeypatch.setattr(scipy.optimize, "minimize", real)
    assert len(seen) >= 2
    for raw, got in zip(seen, _our_loss(engine_cls, X, y, cat, seen)):
        want = _ref_loss(X, y, cat, raw)
        # near the optimum the likelihood and prior gradients cancel: measure against the size of the two parts
        g_prior = _prior_grad(raw, X.shape[1])
        scale = max(np.linalg.norm(want[1]), np.linalg.norm(want[1] - g_prior) + np.linalg.norm(g_prior))
        _check_loss(want, got, scale)


def _close(want, got):
    assert abs(got - want) <= max(1e-6 * abs(want), 1e-9), (want, got)


def _compare(trials, direction, seed=0, **kw):
    import optuna_b200
    d = optuna.study.StudyDirection.MINIMIZE if direction == "minimize" else optuna.study.StudyDirection.MAXIMIZE
    want = optuna.terminator.RegretBoundEvaluator(seed=seed, **kw).evaluate(trials, d)
    got = optuna_b200.RegretBoundEvaluator(seed=seed, **kw).evaluate(trials, d)
    _close(want, got)
    return got


@pytest.mark.parametrize("kind", ["mixed", "float", "cat", "p1"])
@pytest.mark.parametrize("direction", ["minimize", "maximize"])
@pytest.mark.parametrize("seed", [0, 7])
def test_end_to_end(engine_cls, kind, direction, seed):
    _compare(_study(kind, 60, seed=seed, direction=direction).trials, direction, seed=seed)


@pytest.mark.parametrize("ratio,min_n,n", [(0.3, 10, 80), (0.8, 5, 50), (0.5, 20, 12), (0.5, 30, 40)])
def test_end_to_end_top_trials(engine_cls, ratio, min_n, n):
    _compare(_study("mixed", n, seed=1).trials, "minimize", seed=2, top_trials_ratio=ratio, min_n_trials=min_n)


@pytest.mark.parametrize("kind,n", [("wide17", 300), ("wide33", 400), ("mixed", 514)])
def test_end_to_end_blocked(engine_cls, kind, n):
    """GPs over 150, 200 and 257 top trials (several 64-wide blocks) with P = 17, 33 and 5."""
    _compare(_study(kind, n, seed=11).trials, "minimize", seed=4)


def test_non_finite_raw_parameters_fail_like_cholesky(engine_cls):
    """A NaN or overflowing raw parameter raises the RuntimeError subclass the fit retries on, as torch's Cholesky
    raises LinAlgError (a RuntimeError) in the reference."""
    from optuna_b200.engine import GPCholeskyError
    X, y, cat = _gp_data("mixed", 30, seed=1)
    eng = engine_cls(0)
    try:
        eng.gp_set_data(X, y, cat)
        for bad in (np.nan, 1e4):
            raw = np.zeros(X.shape[1] + 2)
            raw[1] = bad
            with pytest.raises(GPCholeskyError):
                eng.gp_loss(raw, MIN_NOISE)
            with pytest.raises(RuntimeError):
                _ref_loss(X, y, cat, raw)
    finally:
        eng.close()


def test_constant_objective(engine_cls):
    study = optuna.create_study(sampler=optuna.samplers.RandomSampler(seed=0))
    study.optimize(lambda t: 0.0 * t.suggest_float("x", 0, 1) + 1.5, n_trials=30)
    _compare(study.trials, "minimize")


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
    _compare(trials, "minimize", seed=3)


def test_errors(engine_cls):
    import optuna_b200
    d = optuna.study.StudyDirection.MINIMIZE
    study = optuna.create_study()
    t = study.ask()
    t.suggest_float("x", 0, 1)
    for trials in ([], study.get_trials(deepcopy=False)):
        with pytest.raises(ValueError) as a:
            optuna.terminator.RegretBoundEvaluator().evaluate(trials, d)
        with pytest.raises(ValueError) as b:
            optuna_b200.RegretBoundEvaluator().evaluate(trials, d)
        assert str(a.value) == str(b.value)
    study = optuna.create_study()
    study.optimize(lambda t: t.suggest_float("x", 0, 1) if t.number % 2 else t.suggest_float("y", 0, 1), n_trials=4)
    with pytest.raises(ValueError) as a:
        optuna.terminator.RegretBoundEvaluator().evaluate(study.trials, d)
    with pytest.raises(ValueError) as b:
        optuna_b200.RegretBoundEvaluator().evaluate(study.trials, d)
    assert str(a.value) == str(b.value) and "intersection search space is empty" in str(a.value)


def test_fit_failure_falls_back(engine_cls, monkeypatch, caplog):
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
        with caplog.at_level(logging.WARNING):
            import optuna_b200
            d = optuna.study.StudyDirection.MINIMIZE
            want = optuna.terminator.RegretBoundEvaluator(seed=1).evaluate(trials, d)
            n_ref = len(caplog.records)
            assert n_ref >= 1
            got = optuna_b200.RegretBoundEvaluator(seed=1).evaluate(trials, d)
    finally:
        optuna.logging.disable_propagation()
    ref = {r.getMessage() for r in caplog.records[:n_ref] if r.name == "optuna._gp.gp"}
    ours = {r.getMessage() for r in caplog.records[n_ref:] if r.name == "optuna.terminator.optuna_b200"}
    assert len(ref) == 1 and ref == ours, (ref, ours)
    assert "patched failure" in next(iter(ref))
    _close(want, got)


def test_terminator_callback_stops_at_same_trial(engine_cls):
    import optuna_b200
    from optuna.terminator import StaticErrorEvaluator, Terminator, TerminatorCallback

    def run(improvement):
        study = optuna.create_study(sampler=optuna.samplers.RandomSampler(seed=2))
        cb = TerminatorCallback(Terminator(improvement_evaluator=improvement,
                                           error_evaluator=StaticErrorEvaluator(constant=4.5e-4), min_n_trials=20))
        study.optimize(_objective("p1", 2), n_trials=70, callbacks=[cb])
        return len(study.trials)

    want = run(optuna.terminator.RegretBoundEvaluator(seed=0))
    got = run(optuna_b200.RegretBoundEvaluator(seed=0))
    assert want == got and want < 70, (want, got)


def test_improvement_info(engine_cls):
    import optuna_b200
    from optuna.visualization._terminator_improvement import _get_improvement_info
    study = _study("mixed", 26, seed=6)
    want = _get_improvement_info(study, improvement_evaluator=optuna.terminator.RegretBoundEvaluator(seed=0))
    got = _get_improvement_info(study, improvement_evaluator=optuna_b200.RegretBoundEvaluator(seed=0))
    assert want.trial_numbers == got.trial_numbers
    for a, b in zip(want.improvements, got.improvements):
        _close(a, b)


def test_exported_lazily():
    import optuna_b200
    from optuna_b200.terminator import RegretBoundEvaluator
    assert optuna_b200.RegretBoundEvaluator is RegretBoundEvaluator
    assert issubclass(RegretBoundEvaluator, optuna.terminator.RegretBoundEvaluator)


def test_gp_kernels_do_not_spill():
    """ptxas -v over the GP kernels (tpe_gp.cuh): no spill stores or loads."""
    nvcc = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)
    if nvcc is None:
        pytest.skip("nvcc is not available")
    import tempfile
    csrc = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "optuna_b200", "csrc")
    with tempfile.TemporaryDirectory() as tmp:
        src = os.path.join(tmp, "gp_only.cu")
        with open(src, "w") as f:
            f.write(f'#include "{csrc}/tpe_kernels.cuh"\n#include "{csrc}/tpe_gp.cuh"\n'
                    "template __global__ void tpe::gp::k_gp_grad<tpe::gp::GRAD_DC>(const double*, const double*, "
                    "const uint8_t*, const double*, const double*, int, int, int, double*);\n"
                    "template __global__ void tpe::gp::k_gp_grad_finish<tpe::gp::GRAD_DC>(const double*, int, "
                    "const double*, int, int, double*);\n")
        out = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-c",
                              "-Xptxas", "-v", "-o", os.path.join(tmp, "gp.o"), src],
                             capture_output=True, text=True, check=True).stderr
    blocks = re.split(r"Compiling entry function", out)
    gp = [b for b in blocks if "k_gp_" in b.split("\n", 1)[0]]
    assert len(gp) >= 10, out
    for b in gp:
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", b)
        assert m and m.group(1) == "0" and m.group(2) == "0", b


# ---- on the GPU only ------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_large_study_against_reference():
    """4 000 complete trials x 8 parameters (the GP is fitted to the top 2 000)."""
    import optuna_b200
    rs = np.random.RandomState(0)
    study = optuna.create_study()
    dists = {f"x{j}": optuna.distributions.FloatDistribution(0.0, 1.0) for j in range(8)}
    X = rs.uniform(0, 1, (4000, 8))
    v = ((X - 0.3) ** 2 * np.arange(1, 9)).sum(1) + 0.05 * rs.randn(4000)
    study.add_trials([optuna.trial.create_trial(params={f"x{j}": X[i, j] for j in range(8)}, distributions=dists,
                                                value=float(v[i])) for i in range(4000)])
    d = optuna.study.StudyDirection.MINIMIZE
    want = optuna.terminator.RegretBoundEvaluator(seed=0).evaluate(study.trials, d)
    got = optuna_b200.RegretBoundEvaluator(seed=0).evaluate(study.trials, d)
    _close(want, got)


@pytest.mark.gpu
def test_same_seed_same_bits():
    import optuna_b200
    trials = _study("mixed", 300, seed=8).trials
    d = optuna.study.StudyDirection.MINIMIZE
    a = optuna_b200.RegretBoundEvaluator(seed=5).evaluate(trials, d)
    b = optuna_b200.RegretBoundEvaluator(seed=5).evaluate(trials, d)
    assert np.float64(a).tobytes() == np.float64(b).tobytes()
    from optuna_b200 import TPEEngine
    X, y, cat = _gp_data("mixed", 300, seed=8)
    eng = TPEEngine(0)
    try:
        eng.gp_set_data(X, y, cat)
        raw = _random_raws(X.shape[1], 1, 1)[0]
        l1, g1 = eng.gp_loss(raw, MIN_NOISE)
        l2, g2 = eng.gp_loss(raw, MIN_NOISE)
        assert l1 == l2 and g1.tobytes() == g2.tobytes()
    finally:
        eng.close()


@pytest.mark.gpu
def test_engine_suggestion_unchanged_by_gp():
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
        eng.gp_loss(np.zeros(Xg.shape[1] + 2), MIN_NOISE)
        eng.gp_posterior(np.ones(Xg.shape[1] + 2), Xg[:10], 2.0)
        after = eng.suggest(list(range(P)), u, 1, **cfg)
        for a, b in zip(before, after):
            np.testing.assert_array_equal(a, b)
    finally:
        eng.close()


@pytest.mark.gpu
def test_cuda_invalid_inputs():
    from optuna_b200 import TPEEngine
    eng = TPEEngine(0)
    try:
        with pytest.raises(ValueError):
            eng.gp_set_data(np.array([[np.nan]]), np.zeros(1), np.zeros(1, bool))
        with pytest.raises(ValueError):
            eng.gp_set_data(np.zeros((0, 2)), np.zeros(0), np.zeros(2, bool))
        with pytest.raises(ValueError, match="GB of device memory"):
            eng.gp_set_data(np.zeros((200_000, 1)), np.zeros(200_000), np.zeros(1, bool))
        # a set_data that failed leaves no GP data behind, not a half-allocated one
        with pytest.raises(RuntimeError, match="no GP data"):
            eng.gp_loss(np.zeros(3), MIN_NOISE)
    finally:
        eng.close()
