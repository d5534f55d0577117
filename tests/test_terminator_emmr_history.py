"""``optuna_b200.terminator_improvement_history`` and ``plot_terminator_improvement`` with ``optuna_b200.EMMREvaluator``
against optuna's ``_get_improvement_info`` with optuna's ``EMMREvaluator``, and the batch calls behind them
(tpe_gpemmr.cuh, and the fixed-noise batched loss of tpe_gpbatch.cuh).

Every case runs on ``NumpyEMMRBatchEngine`` (tests/_emmr_batch_engine.py, runs anywhere) and, with ``-m gpu``, on
libtpe_b200.so.  Improvements are compared with the bounds of test_terminator_emmr: within 1e-6 relative (1e-9
absolute near 0) with the noise fitted, 1e-5 with it fixed.
"""
from __future__ import annotations

import logging
import os
import re
import shutil
import subprocess
import sys
import warnings

import numpy as np
import pytest

optuna = pytest.importorskip("optuna")
torch = pytest.importorskip("torch")

from tests.test_terminator_gpu_gp import _gp_data, _objective, _random_raws, _study  # noqa: E402
from tests.test_terminator_history import _synthetic  # noqa: E402

MIN_NOISE = 1e-6
CONST = sys.float_info.max * 0.1


@pytest.fixture(params=[pytest.param("numpy", id="numpy-engine"),
                        pytest.param("cuda", id="cuda-engine", marks=pytest.mark.gpu)])
def engine_cls(request, monkeypatch):
    from optuna_b200 import TPEEngine, terminator
    from tests._emmr_batch_engine import NumpyEMMRBatchEngine
    cls = NumpyEMMRBatchEngine if request.param == "numpy" else TPEEngine
    monkeypatch.setattr(terminator, "_engine_cls", cls)
    return cls


def _close(want, got, rel):
    assert abs(got - want) <= max(rel * abs(want), 1e-9), (want, got)


def _warned(fn):
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        value = fn()
    return value, [(x.category, str(x.message)) for x in w
                   if not issubclass(x.category, optuna.exceptions.ExperimentalWarning)]


def _ref_info(study, seed, **kw):
    from optuna.visualization._terminator_improvement import _get_improvement_info
    ev = optuna.terminator.EMMREvaluator(seed=seed, **kw)
    return _get_improvement_info(study, improvement_evaluator=ev), ev


def _ours(study, seed, **kw):
    import optuna_b200
    ev = optuna_b200.EMMREvaluator(seed=seed, **kw)
    return optuna_b200.terminator_improvement_history(study, improvement_evaluator=ev), ev


def _same_stream(a, b):
    sa, sb = a._rng.rng.get_state(), b._rng.rng.get_state()
    assert sa[2] == sb[2] and np.array_equal(sa[1], sb[1])


def _compare(study, seed=0, **kw):
    (want, ev_w), w_want = _warned(lambda: _ref_info(study, seed, **kw))
    (got, ev_g), w_got = _warned(lambda: _ours(study, seed, **kw))
    assert w_want == w_got
    assert want.trial_numbers == got.trial_numbers
    assert got.errors is None
    assert len(want.improvements) == len(got.improvements)
    rel = 1e-5 if kw.get("deterministic_objective") else 1e-6
    for a, b in zip(want.improvements, got.improvements):
        _close(a, b, rel)
    _same_stream(ev_w, ev_g)
    return got, w_got


def _reference_cases():
    """Every (kind, direction, seed, noise) case on the NumPy engine; on the library, every kind with the noise fitted
    and fixed, the direction and seed alternating.  Most of a case's time is optuna's own per-prefix fits on the host,
    the same for both engines, so the library runs the eight cases that cover its kernel paths rather than all 32."""
    cases = []
    for deterministic in (False, True):
        for seed in (0, 7):
            for direction in ("minimize", "maximize"):
                for i, kind in enumerate(("mixed", "float", "cat", "p1")):
                    args = (kind, direction, seed, deterministic)
                    cases.append(pytest.param("numpy", *args, id=f"numpy-engine-{kind}-{direction}-{seed}-{deterministic}"))
                    if (seed, direction) == ((0, "minimize"), (7, "maximize"))[i % 2]:
                        cases.append(pytest.param("cuda", *args, marks=pytest.mark.gpu,
                                                  id=f"cuda-engine-{kind}-{direction}-{seed}-{deterministic}"))
    return cases


@pytest.mark.parametrize("engine_cls,kind,direction,seed,deterministic", _reference_cases(), indirect=["engine_cls"])
def test_against_reference(engine_cls, kind, direction, seed, deterministic):
    _compare(_study(kind, 14, seed=seed, direction=direction), seed=seed, deterministic_objective=deterministic)


@pytest.mark.parametrize("delta,min_n,deterministic", [(0.05, 2, False), (0.3, 5, True), (0.1, 5, False)])
def test_options(engine_cls, delta, min_n, deterministic):
    got, _ = _compare(_study("mixed", 16, seed=1), seed=2, delta=delta, min_n_trials=min_n,
                      deterministic_objective=deterministic)
    assert got.improvements[: min_n - 1] == [CONST] * (min_n - 1)


def test_other_states_share_fits(engine_cls):
    study = optuna.create_study(sampler=optuna.samplers.RandomSampler(seed=4))
    obj = _objective("mixed", 4)

    def objective(t):
        if t.number % 7 == 3:
            raise optuna.TrialPruned()
        if t.number % 11 == 5:
            raise RuntimeError("fail")
        return obj(t)

    study.optimize(objective, n_trials=18, catch=(RuntimeError,))
    study.ask().suggest_float("x", -3, 3)
    study.optimize(objective, n_trials=3, catch=(RuntimeError,))
    states = {t.state for t in study.trials}
    assert {optuna.trial.TrialState.PRUNED, optuna.trial.TrialState.FAIL, optuna.trial.TrialState.RUNNING} <= states
    for det in (False, True):
        _compare(study, seed=3, deterministic_objective=det)


def test_search_space_changes(engine_cls):
    study = optuna.create_study(sampler=optuna.samplers.RandomSampler(seed=2))

    def obj(t):
        v = (t.suggest_float("x", 0, 1) - 0.3) ** 2
        if t.number >= 5:
            v += t.suggest_float("y", -1, 1) ** 2
        if t.number < 10:
            v += 0.1 * t.suggest_int("z", 0, 5)
        return v

    study.optimize(obj, n_trials=16)
    _compare(study, seed=1)


def test_constant_objective(engine_cls):
    study = optuna.create_study(sampler=optuna.samplers.RandomSampler(seed=0))
    study.optimize(lambda t: 0.0 * t.suggest_float("x", 0, 1) + 1.5, n_trials=12)
    _compare(study)


def test_infinite_values_warn_in_order(engine_cls):
    study = _study("mixed", 8, seed=4)
    t = study.trials[3]
    study.add_trial(optuna.trial.create_trial(params=t.params, distributions=t.distributions, value=float("inf")))
    study.optimize(_objective("mixed", 4), n_trials=3)
    study.add_trial(optuna.trial.create_trial(params=t.params, distributions=t.distributions, value=float("-inf")))
    study.optimize(_objective("mixed", 5), n_trials=2)
    _, w = _compare(study, seed=2)
    assert sum("Clip non-finite values" in m for _, m in w) >= 6


def test_empty_search_space(engine_cls):
    study = optuna.create_study(sampler=optuna.samplers.RandomSampler(seed=0))
    study.optimize(lambda t: t.suggest_float("x", 0, 1) if t.number % 2 else t.suggest_float("y", 0, 1), n_trials=6)
    got, w = _compare(study)
    assert got.improvements == [CONST] * 6
    assert sum("cannot consider any search space" in m for _, m in w) == 5


def test_same_bits_whatever_the_waves(engine_cls, monkeypatch):
    from optuna_b200 import terminator
    study = _study("mixed", 14, seed=9)
    for det in (False, True):
        a, _ = _ours(study, 1, deterministic_objective=det)
        b, _ = _ours(study, 1, deterministic_objective=det)
        monkeypatch.setattr(terminator, "_WAVE_BYTES", 1)
        c, _ = _ours(study, 1, deterministic_objective=det)
        monkeypatch.undo()
        monkeypatch.setattr(terminator, "_engine_cls", engine_cls)
        assert np.array(a.improvements).tobytes() == np.array(b.improvements).tobytes()
        assert np.array(a.improvements).tobytes() == np.array(c.improvements).tobytes()


@pytest.mark.parametrize("n", [1, 2, 40, 150, 161, 200])
def test_batched_moments_match_single(engine_cls, n):
    """n on both sides of the shared-memory limit (160) and n = 1; two GPs of different sizes in one call, one job
    not positive definite."""
    X, y, cat = _gp_data("mixed", n, seed=n, duplicates=n > 100)
    n = X.shape[0]
    X2, y2, _ = _gp_data("mixed", 23, seed=1)
    P = X.shape[1]
    eng, single = engine_cls(0), engine_cls(0)
    try:
        eng.gp_batch_set([0, 23, 23 + n], np.concatenate([X2, X]), np.concatenate([y2, y]), cat)
        single.gp_set_data(X, y, cat)
        rs = np.random.RandomState(n)
        prms = [np.concatenate([np.exp(r[:P + 1]), [np.exp(r[P + 1]) + MIN_NOISE]]) for r in _random_raws(P, n)]
        rows = [rs.randint(0, n, 3) for _ in prms] + [np.array([n - 1, 0, n // 2])]
        prms.append(np.concatenate([np.full(P, 0.8), [1.2, MIN_NOISE]]))
        bad = prms[0].copy()
        bad[P] = -1.0   # a negative kernel scale: not positive definite
        idx = [1] * len(prms) + [0, 1]
        allp = np.stack(prms + [np.ones(P + 2), bad])
        allr = np.stack(rows + [np.array([22, 0, 5]), rows[0]])
        mean, var, cov, status = eng.gp_batch_moments(idx, allp, allr, 2)
        assert list(status) == [0] * (len(prms) + 1) + [1]
        assert np.all(np.isnan(mean[-1]))
        for J in (0, 3):
            m2, v2, c2, st2 = eng.gp_batch_moments(idx[:-1], allp[:-1], allr[:-1], J)
            assert not st2.any() and c2.shape == (len(idx) - 1, J, J)
            np.testing.assert_allclose(m2, mean[:-1], rtol=1e-13, atol=1e-13)
        for b, (prm, r) in enumerate(zip(prms, rows)):
            ks = prm[P]
            mw, vw, cw = single.gp_posterior_moments(prm, X[r], 2)
            assert np.all(np.abs(mean[b] - mw) <= 1e-12 * (1.0 + np.abs(mw))), (mean[b], mw)
            assert np.abs(var[b] - vw).max() <= 1e-12 * ks and np.all(var[b] >= 0.0)
            assert np.abs(cov[b] - cw).max() <= 1e-12 * ks, (cov[b], cw)
            assert cov[b][0, 1] == cov[b][1, 0]
    finally:
        eng.close()
        single.close()


@pytest.mark.parametrize("n", [2, 40, 200])
def test_fixed_noise_batched_loss_matches_single(engine_cls, n):
    X, y, cat = _gp_data("mixed", n, seed=n)
    X2, y2, _ = _gp_data("mixed", 23, seed=1)
    eng, single = engine_cls(0), engine_cls(0)
    try:
        eng.gp_batch_set([0, 23, 23 + n], np.concatenate([X2, X]), np.concatenate([y2, y]), cat)
        single.gp_set_data(X, y, cat)
        raws = _random_raws(X.shape[1], n) + [np.zeros(X.shape[1] + 2)]
        moved = [np.concatenate([r[:-1], [r[-1] + 3.0]]) for r in raws]   # the raw noise is not read
        loss, grad, status = eng.gp_batch_loss([1] * (2 * len(raws)) + [0], np.stack(raws + moved + [raws[0]]),
                                               MIN_NOISE, deterministic=True)
        assert not status.any()
        for b, raw in enumerate(raws):
            lw, gw = single.gp_loss(raw, MIN_NOISE, deterministic=True)
            assert abs(loss[b] - lw) <= 1e-12 * abs(lw), (loss[b], lw)
            assert np.linalg.norm(grad[b] - gw) <= 1e-12 * np.linalg.norm(gw), (grad[b], gw)
            assert grad[b][-1] == 0.0 and gw[-1] == 0.0
            assert loss[b] == loss[len(raws) + b] and grad[b].tobytes() == grad[len(raws) + b].tobytes()
        # the fitted-noise call is unchanged beside it
        l2, _, _ = eng.gp_batch_loss([1], np.stack(raws[:1]), MIN_NOISE)
        assert abs(l2[0] - single.gp_loss(raws[0], MIN_NOISE)[0]) <= 1e-12 * abs(l2[0])
    finally:
        eng.close()
        single.close()


def test_batch_call_validation(engine_cls):
    eng = engine_cls(0)
    try:
        eng.gp_batch_set([0, 2, 5], np.random.RandomState(0).uniform(0, 1, (5, 2)), np.arange(5.0), np.zeros(2, bool))
        prm = np.ones((1, 4))
        for rows, J in (([[0, 2, 0]], 2), ([[-1, 0, 0]], 0), ([[0, 0, 0, 0]], 2), ([[0, 0]], 3), ([[0, 0]], 1)):
            with pytest.raises(ValueError):
                eng.gp_batch_moments([0], prm, np.array(rows), J)
        with pytest.raises(ValueError, match="out of range"):
            eng.gp_batch_moments([2], prm, np.array([[0, 0, 0]]), 2)
        with pytest.raises(ValueError, match="out of range"):
            eng.gp_batch_loss([3], np.zeros((1, 4)), MIN_NOISE, deterministic=True)
        mean, var, cov, status = eng.gp_batch_moments([1], prm, np.array([[2, 0, 1]]), 2)
        assert not status.any() and mean.shape == (1, 3) and cov.shape == (1, 2, 2)
    finally:
        eng.close()


def test_routing_unchanged(engine_cls):
    """optuna's EMMREvaluator, a subclass of the drop-in and RegretBoundEvaluator take their existing paths."""
    import optuna_b200
    from optuna.visualization._terminator_improvement import _get_improvement_info

    class Sub(optuna_b200.EMMREvaluator):
        pass

    study = _study("mixed", 10, seed=2)
    for mk in (lambda: optuna.terminator.EMMREvaluator(seed=0), lambda: Sub(seed=0)):
        want = _get_improvement_info(study, improvement_evaluator=mk())
        got = optuna_b200.terminator_improvement_history(study, improvement_evaluator=mk())
        assert want == got
    from optuna_b200 import terminator
    a = optuna_b200.terminator_improvement_history(study, optuna_b200.RegretBoundEvaluator(seed=0, min_n_trials=5))
    _, b = terminator._batched_improvements(optuna_b200.RegretBoundEvaluator(seed=0, min_n_trials=5), study)
    assert a.improvements == b


def test_get_error(engine_cls):
    import optuna_b200
    from optuna.terminator import CrossValidationErrorEvaluator, MedianErrorEvaluator, StaticErrorEvaluator
    from optuna.visualization._terminator_improvement import _get_improvement_info
    study = _study("mixed", 16, seed=6)
    err = StaticErrorEvaluator(constant=0.25)
    want = _get_improvement_info(study, True, optuna.terminator.EMMREvaluator(seed=0), err)
    got = optuna_b200.terminator_improvement_history(study, optuna_b200.EMMREvaluator(seed=0), err, True)
    assert want.trial_numbers == got.trial_numbers and want.errors == got.errors
    # a MedianErrorEvaluator paired with the same evaluator draws from its stream between prefixes
    ref = optuna.terminator.EMMREvaluator(seed=0)
    want = _get_improvement_info(study, True, ref, MedianErrorEvaluator(ref, warm_up_trials=2, n_initial_trials=4))
    ours = optuna_b200.EMMREvaluator(seed=0)
    got = optuna_b200.terminator_improvement_history(
        study, ours, MedianErrorEvaluator(ours, warm_up_trials=2, n_initial_trials=4), True)
    assert want.trial_numbers == got.trial_numbers
    for a, b in zip(want.improvements, got.improvements):
        _close(a, b, 1e-6)
    for a, b in zip(want.errors, got.errors):
        _close(a, b, 1e-6)
    _same_stream(ref, ours)
    with pytest.raises(ValueError) as a:
        _get_improvement_info(study, True, optuna.terminator.EMMREvaluator(seed=0), CrossValidationErrorEvaluator())
    with pytest.raises(ValueError) as b:
        optuna_b200.terminator_improvement_history(study, optuna_b200.EMMREvaluator(seed=0),
                                                   CrossValidationErrorEvaluator(), True)
    assert str(a.value) == str(b.value)
    empty = optuna.create_study()
    info = optuna_b200.terminator_improvement_history(empty, optuna_b200.EMMREvaluator(), get_error=True,
                                                      error_evaluator=err)
    assert info.trial_numbers == [] and info.improvements == [] and info.errors is None


def test_not_positive_definite_raises_with_the_stream(engine_cls, monkeypatch):
    """A final covariance that fails to factorise raises LinAlgError at the first failing prefix in trial order, and
    leaves the stream where the per-prefix loop with the drop-in leaves it."""
    import optuna_b200
    from optuna.visualization._terminator_improvement import _get_improvement_info
    study = _study("mixed", 12, seed=3)
    fail_at = 7   # complete trials: the moments of the second GP over 7 trials fail
    real_moments = engine_cls.gp_posterior_moments
    real_batch = engine_cls.gp_batch_moments
    from optuna_b200.engine import GPCholeskyError

    def moments(self, params, Xq, n_joint=0):
        if n_joint == 2 and self._gp_rows() == fail_at:
            raise GPCholeskyError("forced")
        return real_moments(self, params, Xq, n_joint)

    def batch(self, gp_idx, params, rows, n_joint=0):
        mean, var, cov, status = real_batch(self, gp_idx, params, rows, n_joint)
        status = status.copy()
        for b, g in enumerate(gp_idx):
            if g % 2 == 1 and self._batch_rows(int(g)) == fail_at:   # odd: the GP over all t trials
                status[b] = 1
        return mean, var, cov, status

    if engine_cls.__name__ == "TPEEngine":
        pytest.skip("the failure is injected through the host engine")
    monkeypatch.setattr(engine_cls, "_gp_rows", lambda self: self._X.shape[0], raising=False)
    monkeypatch.setattr(engine_cls, "_batch_rows", lambda self, g: self._gps[g]._X.shape[0], raising=False)
    monkeypatch.setattr(engine_cls, "gp_posterior_moments", moments)
    monkeypatch.setattr(engine_cls, "gp_batch_moments", batch)
    loop_ev, ours = optuna_b200.EMMREvaluator(seed=4), optuna_b200.EMMREvaluator(seed=4)
    with pytest.raises(np.linalg.LinAlgError):
        _get_improvement_info(study, improvement_evaluator=loop_ev)
    with pytest.raises(np.linalg.LinAlgError):
        optuna_b200.terminator_improvement_history(study, improvement_evaluator=ours)
    _same_stream(loop_ev, ours)


def test_fit_failure_falls_back(engine_cls, monkeypatch, caplog):
    import scipy.optimize
    real = scipy.optimize.minimize

    def failing(*args, **kw):
        res = real(*args, **kw)
        res.success = False
        res.message = "patched failure"
        return res

    monkeypatch.setattr(scipy.optimize, "minimize", failing)
    study = _study("mixed", 6, seed=5)
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
        _close(a, b, 1e-6)


def test_plot_matches_optuna(engine_cls):
    pytest.importorskip("plotly")
    import optuna_b200
    study = _study("mixed", 12, seed=1)
    want = optuna.visualization.plot_terminator_improvement(
        study, improvement_evaluator=optuna.terminator.EMMREvaluator(seed=0), min_n_trials=5)
    got = optuna_b200.plot_terminator_improvement(study, improvement_evaluator=optuna_b200.EMMREvaluator(seed=0),
                                                  min_n_trials=5)
    assert len(want.data) == len(got.data)
    for a, b in zip(want.data, got.data):
        assert list(a.x) == list(b.x)
        for u, v in zip(a.y, b.y):
            _close(u, v, 1e-6)


def test_moments_kernel_does_not_spill():
    nvcc = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)
    if nvcc is None:
        pytest.skip("nvcc is not available")
    import tempfile
    csrc = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "optuna_b200", "csrc")
    with tempfile.TemporaryDirectory() as tmp:
        src = os.path.join(tmp, "gpe_only.cu")
        with open(src, "w") as f:
            f.write(f'#include "{csrc}/tpe_kernels.cuh"\n#include "{csrc}/tpe_gpemmr.cuh"\n')
        out = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-c",
                              "-Xptxas", "-v", "-o", os.path.join(tmp, "gpe.o"), src],
                             capture_output=True, text=True, check=True).stderr
    blocks = re.split(r"Compiling entry function", out)
    gpe = [b for b in blocks if "k_gpe_" in b.split("\n", 1)[0]]
    assert len(gpe) == 1, out
    m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", gpe[0])
    assert m and m.group(1) == "0" and m.group(2) == "0", gpe[0]


# ---- on the GPU only ------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("deterministic", [False, True])
def test_gpu_60x8_against_reference(deterministic):
    """The library against optuna's own EMMREvaluator on a 60-trial study, with the noise fitted and fixed.  Optuna's
    two host fits per prefix take about 3 minutes per curve at 100 trials on the host of an H100 box; 60 trials keep
    each curve to a fraction of that.  Larger studies are checked against the drop-in per-prefix loop below."""
    from optuna_b200 import TPEEngine, terminator
    assert terminator._engine_cls is TPEEngine
    _compare(_synthetic(60, 8), seed=0, deterministic_objective=deterministic)


def _against_drop_in_loop(n, tol, deterministic=False):
    import optuna_b200
    from optuna.visualization._terminator_improvement import _get_improvement_info
    study = _synthetic(n, 8, seed=1)
    ev_w = optuna_b200.EMMREvaluator(seed=0, deterministic_objective=deterministic)
    want = _get_improvement_info(study, improvement_evaluator=ev_w)
    ev_g = optuna_b200.EMMREvaluator(seed=0, deterministic_objective=deterministic)
    got = optuna_b200.terminator_improvement_history(study, ev_g)
    assert want.trial_numbers == got.trial_numbers
    w, g = np.array(want.improvements), np.array(got.improvements)
    over = np.abs(g - w) > np.maximum(tol * np.abs(w), 1e-9)
    rel = np.abs(g - w) / np.maximum(np.abs(w), 1e-9)
    assert not over.any(), (f"{over.sum()} prefixes over {tol}, largest relative difference {rel.max():.3g} at "
                            f"prefix {int(rel.argmax())}")
    _same_stream(ev_w, ev_g)


@pytest.mark.gpu
@pytest.mark.parametrize("deterministic,tol", [(False, 1e-5), (True, 1e-5)])
def test_gpu_300x8_against_drop_in_loop(deterministic, tol):
    """With the noise fixed the batch agrees with the loop to 6.8e-8 relative on an H100.  With it fitted, one
    prefix of 300 (prefix 212) differs by 2.1e-6: the batched and single-GP losses agree to about 1e-14, but one
    L-BFGS-B run takes a different last step on that difference.  Both cases are held to 1e-5."""
    _against_drop_in_loop(300, tol, deterministic)


@pytest.mark.gpu
def test_gpu_1000x8_against_drop_in_loop():
    """The batched and the single-GP loss agree to about 1e-14 relative, but over 2 000 fits of up to 1 000 rows a
    few L-BFGS-B runs take a different last step on that difference, as with the regret bound's batch
    (test_terminator_history.test_gpu_1000x8_against_drop_in_loop).  The largest relative difference measured on an
    H100 was 6.0e-5, so this case is held to 1e-4."""
    _against_drop_in_loop(1000, 1e-4)
