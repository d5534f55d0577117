"""``optuna_b200.terminator_improvement_history`` and ``plot_terminator_improvement`` against optuna's
``_get_improvement_info`` / ``plot_terminator_improvement``, and the batch calls behind them (tpe_gpbatch.cuh).

Every case runs on ``NumpyGPBatchEngine`` (tests/_gp_batch_engine.py, runs anywhere) and, with ``-m gpu``, on
libtpe_b200.so.  Improvements are compared with the bound of test_terminator_gpu_gp: within max(1e-6 |want|, 1e-9).
"""
from __future__ import annotations

import logging
import os
import re
import shutil
import subprocess
import threading

import numpy as np
import pytest

optuna = pytest.importorskip("optuna")
torch = pytest.importorskip("torch")

from tests.test_terminator_gpu_gp import MIN_NOISE, _check_loss, _close, _gp_data, _objective, _random_raws, _study  # noqa: E402


@pytest.fixture(params=[pytest.param("numpy", id="numpy-engine"),
                        pytest.param("cuda", id="cuda-engine", marks=pytest.mark.gpu)])
def engine_cls(request, monkeypatch):
    from optuna_b200 import TPEEngine, terminator
    from tests._gp_batch_engine import NumpyGPBatchEngine
    cls = NumpyGPBatchEngine if request.param == "numpy" else TPEEngine
    monkeypatch.setattr(terminator, "_engine_cls", cls)
    return cls


def _ref_info(study, seed, **kw):
    from optuna.visualization._terminator_improvement import _get_improvement_info
    ev = optuna.terminator.RegretBoundEvaluator(seed=seed, **kw)
    return _get_improvement_info(study, improvement_evaluator=ev), ev


def _ours(study, seed, **kw):
    import optuna_b200
    ev = optuna_b200.RegretBoundEvaluator(seed=seed, **kw)
    return optuna_b200.terminator_improvement_history(study, improvement_evaluator=ev), ev


def _compare(study, seed=0, **kw):
    want, ev_w = _ref_info(study, seed, **kw)
    got, ev_g = _ours(study, seed, **kw)
    assert want.trial_numbers == got.trial_numbers
    assert got.errors is None
    assert len(want.improvements) == len(got.improvements)
    for a, b in zip(want.improvements, got.improvements):
        _close(a, b)
    # the evaluator's stream is where the reference loop leaves it
    sw, sg = ev_w._rng.rng.get_state(), ev_g._rng.rng.get_state()
    assert sw[2] == sg[2] and np.array_equal(sw[1], sg[1])
    return got


@pytest.mark.parametrize("kind", ["mixed", "float", "cat", "p1"])
@pytest.mark.parametrize("direction", ["minimize", "maximize"])
@pytest.mark.parametrize("seed", [0, 7])
def test_against_reference(engine_cls, kind, direction, seed):
    _compare(_study(kind, 28, seed=seed, direction=direction), seed=seed)


@pytest.mark.parametrize("ratio,min_n,n", [(0.3, 10, 40), (0.8, 5, 30)])
def test_top_trials_options(engine_cls, ratio, min_n, n):
    _compare(_study("mixed", n, seed=1), seed=2, top_trials_ratio=ratio, min_n_trials=min_n)


def test_other_states_and_constant(engine_cls):
    study = optuna.create_study(sampler=optuna.samplers.RandomSampler(seed=4))
    obj = _objective("mixed", 4)

    def objective(t):
        if t.number % 7 == 3:
            raise optuna.TrialPruned()
        if t.number % 11 == 5:
            raise RuntimeError("fail")
        return obj(t)

    study.optimize(objective, n_trials=30, catch=(RuntimeError,))
    study.ask().suggest_float("x", -3, 3)
    study.optimize(objective, n_trials=4, catch=(RuntimeError,))
    states = {t.state for t in study.trials}
    assert {optuna.trial.TrialState.PRUNED, optuna.trial.TrialState.FAIL, optuna.trial.TrialState.RUNNING} <= states
    _compare(study, seed=3)
    const = optuna.create_study(sampler=optuna.samplers.RandomSampler(seed=0))
    const.optimize(lambda t: 0.0 * t.suggest_float("x", 0, 1) + 1.5, n_trials=15)
    _compare(const)


def test_search_space_changes(engine_cls):
    study = optuna.create_study(sampler=optuna.samplers.RandomSampler(seed=2))

    def obj(t):
        v = (t.suggest_float("x", 0, 1) - 0.3) ** 2
        if t.number >= 6:
            v += t.suggest_float("y", -1, 1) ** 2
        if t.number < 12:
            v += 0.1 * t.suggest_int("z", 0, 5)
        return v

    study.optimize(obj, n_trials=24)
    _compare(study, seed=1)


def test_random_stream_continues(engine_cls):
    study = _study("mixed", 22, seed=3)
    _, ev_w = _ref_info(study, 5)
    _, ev_g = _ours(study, 5)
    d = optuna.study.StudyDirection.MINIMIZE
    _close(ev_w.evaluate(study.trials, d), ev_g.evaluate(study.trials, d))


def test_same_bits_whatever_the_waves(engine_cls, monkeypatch):
    from optuna_b200 import terminator
    study = _study("mixed", 30, seed=9)
    a, _ = _ours(study, 1)
    b, _ = _ours(study, 1)
    monkeypatch.setattr(terminator, "_WAVE_BYTES", 1)
    c, _ = _ours(study, 1)
    assert np.array(a.improvements).tobytes() == np.array(b.improvements).tobytes()
    assert np.array(a.improvements).tobytes() == np.array(c.improvements).tobytes()


@pytest.mark.parametrize("n", [40, 150, 200])
def test_batched_loss_matches_single(engine_cls, n):
    """n on both sides of the shared-memory limit (160), two GPs of different sizes in one call, one job not PD."""
    X, y, cat = _gp_data("mixed", n, seed=n)
    X2, y2, _ = _gp_data("mixed", 23, seed=1)
    eng = engine_cls(0)
    single = engine_cls(0)
    try:
        eng.gp_batch_set([0, 23, 23 + n], np.concatenate([X2, X]), np.concatenate([y2, y]), cat)
        single.gp_set_data(X, y, cat)
        raws = _random_raws(X.shape[1], n) + [np.zeros(X.shape[1] + 2)]
        bad = np.zeros(X.shape[1] + 2)
        bad[1] = np.nan
        idx = [1] * len(raws) + [0, 1]
        loss, grad, status = eng.gp_batch_loss(idx, np.stack(raws + [raws[0], bad]), MIN_NOISE)
        assert list(status) == [0] * (len(raws) + 1) + [1]
        assert np.isnan(loss[-1])
        for b, raw in enumerate(raws):
            lw, gw = single.gp_loss(raw, MIN_NOISE)
            assert abs(loss[b] - lw) <= 1e-12 * abs(lw), (loss[b], lw)
            assert np.linalg.norm(grad[b] - gw) <= 1e-12 * np.linalg.norm(gw), (grad[b], gw)
    finally:
        eng.close()
        single.close()


def test_fit_failure_falls_back(engine_cls, monkeypatch, caplog):
    import scipy.optimize
    real = scipy.optimize.minimize

    def failing(*args, **kw):
        res = real(*args, **kw)
        res.success = False
        res.message = "patched failure"
        return res

    monkeypatch.setattr(scipy.optimize, "minimize", failing)
    study = _study("mixed", 12, seed=5)
    optuna.logging.enable_propagation()
    try:
        with caplog.at_level(logging.WARNING):
            want, _ = _ref_info(study, 1)
            n_ref = len(caplog.records)
            got, _ = _ours(study, 1)
    finally:
        optuna.logging.disable_propagation()
    ref = [r.getMessage() for r in caplog.records[:n_ref] if r.name == "optuna._gp.gp"]
    ours = [r.getMessage() for r in caplog.records[n_ref:] if r.name == "optuna.terminator.optuna_b200"]
    assert ref and set(ref) == set(ours) and len(ref) == len(ours)
    for a, b in zip(want.improvements, got.improvements):
        _close(a, b)


def test_routing_and_errors(engine_cls):
    import optuna_b200
    from optuna.terminator import (BestValueStagnationEvaluator, CrossValidationErrorEvaluator,
                                   StaticErrorEvaluator)
    from optuna.visualization._terminator_improvement import _get_improvement_info

    class Sub(optuna_b200.RegretBoundEvaluator):
        pass

    study = _study("mixed", 12, seed=2)
    for mk in (lambda: BestValueStagnationEvaluator(), lambda: Sub(seed=0),
               lambda: optuna.terminator.RegretBoundEvaluator(seed=0)):
        want = _get_improvement_info(study, improvement_evaluator=mk())
        got = optuna_b200.terminator_improvement_history(study, improvement_evaluator=mk())
        assert want == got
    err = StaticErrorEvaluator(constant=0.25)
    want = _get_improvement_info(study, True, optuna.terminator.RegretBoundEvaluator(seed=0), err)
    got = optuna_b200.terminator_improvement_history(study, optuna_b200.RegretBoundEvaluator(seed=0), err, True)
    assert want.trial_numbers == got.trial_numbers and want.errors == got.errors
    # without reported cross-validation scores both raise the same error
    with pytest.raises(ValueError) as a:
        _get_improvement_info(study, True, optuna.terminator.RegretBoundEvaluator(seed=0),
                              CrossValidationErrorEvaluator())
    with pytest.raises(ValueError) as b:
        optuna_b200.terminator_improvement_history(study, optuna_b200.RegretBoundEvaluator(seed=0),
                                                   CrossValidationErrorEvaluator(), True)
    assert str(a.value) == str(b.value)
    mo = optuna.create_study(directions=["minimize", "minimize"])
    with pytest.raises(ValueError, match="multi-objective"):
        optuna_b200.terminator_improvement_history(mo)
    empty = optuna.create_study()
    info = optuna_b200.terminator_improvement_history(empty, optuna_b200.RegretBoundEvaluator())
    assert info.trial_numbers == [] and info.improvements == [] and info.errors is None


def test_batch_call_validation(engine_cls):
    eng = engine_cls(0)
    try:
        with pytest.raises(ValueError):
            eng.gp_batch_set([0], np.zeros((0, 2)), np.zeros(0), np.zeros(2, bool))
        with pytest.raises(ValueError):
            eng.gp_batch_set([0, 0, 2], np.zeros((2, 2)), np.zeros(2), np.zeros(2, bool))
        with pytest.raises(ValueError):
            eng.gp_batch_set([0, 2], np.array([[0.0, np.nan], [1.0, 1.0]]), np.zeros(2), np.zeros(2, bool))
        eng.gp_batch_set([0, 2], np.array([[0.0, 0.5], [1.0, 1.0]]), np.array([-1.0, 1.0]), np.zeros(2, bool))
        with pytest.raises(ValueError, match="out of range"):
            eng.gp_batch_loss([3], np.zeros((1, 4)), MIN_NOISE)
    finally:
        eng.close()


def test_threaded_lbfgsb_iterates_equal_sequential():
    """scipy's L-BFGS-B gives the same iterates in threads, run together, as one after another."""
    import scipy.optimize

    def fun(c):
        def f(x):
            v = np.sum(c * (x - 0.3) ** 4) + np.sum(np.cos(x))
            return v, 4 * c * (x - 0.3) ** 3 - np.sin(x)
        return f

    cs = [np.linspace(1, 2 + k, 6) for k in range(8)]
    seq = [scipy.optimize.minimize(fun(c), np.zeros(6), jac=True, method="l-bfgs-b", options={"gtol": 1e-2}).x
           for c in cs]
    par = [None] * len(cs)
    barrier = threading.Barrier(len(cs))

    def run(k):
        barrier.wait()
        par[k] = scipy.optimize.minimize(fun(cs[k]), np.zeros(6), jac=True, method="l-bfgs-b",
                                         options={"gtol": 1e-2}).x

    ths = [threading.Thread(target=run, args=(k,)) for k in range(len(cs))]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    for a, b in zip(seq, par):
        assert a.tobytes() == b.tobytes()


def test_plot_matches_optuna(engine_cls):
    pytest.importorskip("plotly")
    import optuna_b200
    study = _study("mixed", 22, seed=1)
    want = optuna.visualization.plot_terminator_improvement(
        study, improvement_evaluator=optuna.terminator.RegretBoundEvaluator(seed=0))
    got = optuna_b200.plot_terminator_improvement(study, improvement_evaluator=optuna_b200.RegretBoundEvaluator(seed=0))
    assert len(want.data) == len(got.data)
    for a, b in zip(want.data, got.data):
        assert list(a.x) == list(b.x)
        for u, v in zip(a.y, b.y):
            _close(u, v)


def test_exported_lazily():
    import optuna_b200
    from optuna_b200 import analysis, terminator
    assert optuna_b200.terminator_improvement_history is terminator.terminator_improvement_history
    assert optuna_b200.plot_terminator_improvement is analysis.plot_terminator_improvement


def test_batch_kernels_do_not_spill():
    nvcc = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)
    if nvcc is None:
        pytest.skip("nvcc is not available")
    import tempfile
    csrc = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "optuna_b200", "csrc")
    with tempfile.TemporaryDirectory() as tmp:
        src = os.path.join(tmp, "gpb_only.cu")
        with open(src, "w") as f:
            f.write(f'#include "{csrc}/tpe_kernels.cuh"\n#include "{csrc}/tpe_gpbatch.cuh"\n')
        out = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-c",
                              "-Xptxas", "-v", "-o", os.path.join(tmp, "gpb.o"), src],
                             capture_output=True, text=True, check=True).stderr
    blocks = re.split(r"Compiling entry function", out)
    gpb = [b for b in blocks if "k_gpb_" in b.split("\n", 1)[0]]
    assert len(gpb) == 2, out
    for b in gpb:
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", b)
        assert m and m.group(1) == "0" and m.group(2) == "0", b


# ---- on the GPU only ------------------------------------------------------------------------------------------------

def _synthetic(n, P, seed=0):
    rs = np.random.RandomState(seed)
    study = optuna.create_study()
    dists = {f"x{j}": optuna.distributions.FloatDistribution(0.0, 1.0) for j in range(P)}
    X = rs.uniform(0, 1, (n, P))
    v = ((X - 0.3) ** 2 * np.arange(1, P + 1)).sum(1) + 0.05 * rs.randn(n)
    study.add_trials([optuna.trial.create_trial(params={f"x{j}": X[i, j] for j in range(P)}, distributions=dists,
                                                value=float(v[i])) for i in range(n)])
    return study


@pytest.mark.gpu
def test_gpu_100x8_against_reference():
    from optuna_b200 import TPEEngine, terminator
    assert terminator._engine_cls is TPEEngine
    _compare(_synthetic(100, 8), seed=0)


def _against_drop_in_loop(n, tol):
    import optuna_b200
    from optuna.visualization._terminator_improvement import _get_improvement_info
    study = _synthetic(n, 8, seed=1)
    want = _get_improvement_info(study, improvement_evaluator=optuna_b200.RegretBoundEvaluator(seed=0))
    got = optuna_b200.terminator_improvement_history(study, optuna_b200.RegretBoundEvaluator(seed=0))
    assert want.trial_numbers == got.trial_numbers
    for a, b in zip(want.improvements, got.improvements):
        assert abs(b - a) <= max(tol * abs(a), 1e-9), (a, b)


@pytest.mark.gpu
def test_gpu_300x8_against_drop_in_loop():
    _against_drop_in_loop(300, 1e-6)


@pytest.mark.gpu
def test_gpu_1000x8_against_drop_in_loop():
    """The batched and the single-GP loss agree to about 1e-14 relative, but over 1 000 fits of up to 500 rows a few
    L-BFGS-B runs take a different last step on that difference: the largest relative difference measured on an
    H100 was 1.1e-5, so this case is held to 1e-4."""
    _against_drop_in_loop(1000, 1e-4)
