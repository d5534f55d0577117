"""GPSampler's acquisition search in lock step (optuna_b200/_acqf_search.py) and the fused device acquisition
(``TPEEngine.acqf_set`` / ``acqf_eval``, csrc/tpe_acqf.cuh).

On any machine: the lock-step driver, given the acquisition objects optuna builds (LogEI with running trials,
ConstrainedLogEI, LogEHVI, ConstrainedLogEHVI with and without feasible trials), returns optuna's
``optimize_acqf_mixed`` bits and leaves the random stream where optuna leaves it, in continuous, integer (exhaustive and
line search), categorical and mixed spaces, with warm starts, a converged study and the non-convergence warning.  The
acquisition is evaluated row by row (``_RowWise``), so a row's value does not depend on its batch, as on the device.

On the GPU: ``acqf_eval`` against torch's acquisition over the same device GPs; a row's bits alone, inside 2 048 rows
and with or without gradients; the driver against optuna's own search over the device acquisition, bit for bit; the
drop-in against optuna's ``GPSampler``; and the error messages.
"""
from __future__ import annotations

import logging

import numpy as np
import pytest
import torch

from tests.conftest import HAVE_OPTUNA

pytestmark = pytest.mark.skipif(not HAVE_OPTUNA, reason="optuna (oracle/_ref) is not available")

if HAVE_OPTUNA:
    import optuna
    from optuna._gp import acqf as acqf_module
    from optuna._gp import gp as gp_module
    from optuna._gp import optim_mixed
    from optuna._gp import search_space as gp_search_space

    from optuna_b200 import _acqf_search

D = None if not HAVE_OPTUNA else optuna.distributions


def _space(kind: str):
    spaces = {
        "float": {"a": D.FloatDistribution(0, 1), "b": D.FloatDistribution(1e-3, 1, log=True),
                  "c": D.FloatDistribution(-2, 2)},
        "int_small": {"a": D.IntDistribution(0, 10), "b": D.IntDistribution(1, 7)},
        "int_large": {"a": D.IntDistribution(0, 100), "b": D.FloatDistribution(0, 1)},
        "cat": {"a": D.CategoricalDistribution(["x", "y", "z"]), "b": D.CategoricalDistribution([1, 2])},
        "mixed": {"a": D.FloatDistribution(0, 1), "b": D.IntDistribution(0, 9), "c": D.IntDistribution(0, 60, step=2),
                  "d": D.CategoricalDistribution(["x", "y", "z"])},
    }
    return gp_search_space.SearchSpace(spaces[kind])


def _gpr(ss, X, y, seed):
    rs = np.random.RandomState(seed)
    P = X.shape[1]
    gpr = gp_module.GPRegressor(torch.from_numpy(ss.is_categorical), torch.from_numpy(X), torch.from_numpy(y),
                                torch.from_numpy(rs.uniform(0.5, 8.0, P)), torch.tensor(rs.uniform(0.5, 2.0)),
                                torch.tensor(1e-4))
    gpr._cache_matrix()
    return gpr


def _rugged(X, seed):
    rs = np.random.RandomState(seed)
    w = rs.normal(size=(X.shape[1], 3)) * 6
    y = np.sin(X @ w).sum(1) + 0.3 * rs.normal(size=len(X))
    return (y - y.mean()) / y.std()


class _RowWise(acqf_module.BaseAcquisitionFunc):
    """``inner`` evaluated one row at a time: a row's value and gradient do not depend on its batch."""

    def __init__(self, inner) -> None:
        self._inner = inner
        super().__init__(inner.length_scales, inner.search_space)

    def eval_acqf(self, x: torch.Tensor) -> torch.Tensor:
        if x.ndim == 1:
            return self._inner.eval_acqf(x)
        return torch.stack([self._inner.eval_acqf(x[i]) for i in range(x.shape[0])])


def _evaluator(acqf, calls: list):
    def evaluate(x, grad):
        calls.append((len(x), grad))
        if not grad:
            return acqf.eval_acqf_no_grad(x)
        xt = torch.from_numpy(x).requires_grad_(True)
        f = acqf.eval_acqf(xt)
        f.sum().backward()
        return f.detach().numpy(), xt.grad.detach().numpy()
    return evaluate


def _acqf(kind: str, space: str, seed: int = 0, n: int = 24):
    ss = _space(space)
    rs = np.random.RandomState(seed)
    X = ss.sample_normalized_params(n, rs)
    y = _rugged(X, seed)
    gpr = _gpr(ss, X, y, seed)
    if kind == "logei":
        return acqf_module.LogEI(gpr, ss, float(y.max()))
    if kind == "logei_running":
        return acqf_module.LogEI(gpr, ss, float(y.max()), normalized_params_of_running_trials=X[:3] * 0.9 + 0.05)
    c = _gpr(ss, X, _rugged(X, seed + 7), seed + 1)
    if kind == "constrained_logei":
        return acqf_module.ConstrainedLogEI(gpr, ss, float(y.max()), [c], [0.3])
    if kind == "constrained_logei_infeasible":
        return acqf_module.ConstrainedLogEI(gpr, ss, -np.inf, [c], [0.3])
    y2 = _rugged(X, seed + 3)
    g2 = _gpr(ss, X, y2, seed + 2)
    Y = torch.from_numpy(np.stack([y, y2], 1))
    if kind == "logehvi":
        return acqf_module.LogEHVI([gpr, g2], ss, Y, 128, seed)
    if kind == "constrained_logehvi":
        return acqf_module.ConstrainedLogEHVI([gpr, g2], ss, Y[:12], 128, seed, [c], [0.1])
    if kind == "constrained_logehvi_infeasible":
        return acqf_module.ConstrainedLogEHVI([gpr, g2], ss, None, 128, seed, [c], [0.1])
    raise AssertionError(kind)


def _run_both(acqf, warm=None, **kw):
    rowwise = _RowWise(acqf)
    seq_calls: list = []

    class _Counted(_RowWise):
        def eval_acqf(self, x):
            seq_calls.append(x.shape[0] if x.ndim == 2 else 1)
            return super().eval_acqf(x)

    r1 = np.random.RandomState(5)
    x1, f1 = optim_mixed.optimize_acqf_mixed(_Counted(acqf), warmstart_normalized_params_array=warm, rng=r1, **kw)
    calls: list = []
    r2 = np.random.RandomState(5)
    x2, f2 = _acqf_search.optimize_acqf_mixed(rowwise, _evaluator(rowwise, calls),
                                              warmstart_normalized_params_array=warm, rng=r2, **kw)
    assert np.array_equal(x1, x2) and f1 == f2, (x1, x2, f1, f2)
    assert r1.randint(1 << 30) == r2.randint(1 << 30)
    return calls, seq_calls


_KINDS = ["logei", "logei_running", "constrained_logei", "constrained_logei_infeasible", "logehvi",
          "constrained_logehvi", "constrained_logehvi_infeasible"]


@pytest.mark.parametrize("kind", _KINDS)
@pytest.mark.parametrize("space", ["float", "int_small", "int_large", "cat", "mixed"])
def test_driver_matches_optuna(kind, space):
    if kind.endswith("logehvi") or "logehvi_" in kind:
        if space in ("int_small", "cat"):
            pytest.skip("covered by the single-objective kinds")
    calls, seq_calls = _run_both(_acqf(kind, space), n_preliminary_samples=256)
    # the same rows are evaluated, in fewer calls
    assert sum(n for n, _ in calls) == sum(seq_calls)
    assert len(calls) <= len(seq_calls)


def test_warm_start_and_round_count():
    """Warm starts join the start points; a round of k live L-BFGS-B searches is one call of k rows, not k calls."""
    acqf = _acqf("logei", "float", seed=3, n=40)
    warm = np.random.RandomState(9).uniform(0, 1, (2, 3))
    calls, seq_calls = _run_both(acqf, warm=warm, n_preliminary_samples=512)
    grad_calls = [n for n, g in calls if g]
    assert max(grad_calls) > 1
    assert len(grad_calls) < sum(grad_calls)
    assert len(calls) < len(seq_calls)


def _records(fn):
    records: list = []

    class _H(logging.Handler):
        def emit(self, record):
            records.append(record.getMessage())
    h = _H()
    optim_mixed._logger.addHandler(h)
    try:
        out = fn()
    finally:
        optim_mixed._logger.removeHandler(h)
    return out, records


def test_converged_study_warning():
    """Few preliminary samples with a non-zero roulette weight: fewer local searches, and optuna's warning."""
    acqf = _RowWise(_acqf("logei", "mixed", seed=1))
    (x1, f1), w1 = _records(lambda: optim_mixed.optimize_acqf_mixed(acqf, n_preliminary_samples=4,
                                                                     rng=np.random.RandomState(0)))
    (x2, f2), w2 = _records(lambda: _acqf_search.optimize_acqf_mixed(acqf, _evaluator(acqf, []),
                                                                      n_preliminary_samples=4,
                                                                      rng=np.random.RandomState(0)))
    assert np.array_equal(x1, x2) and f1 == f2
    assert w1 == w2 and "Study already converged, so the number of local search is reduced." in w1


def test_not_converged_warning():
    """``max_iter`` reached in a mixed space: the same points, values and warning as optuna's local search."""
    acqf = _RowWise(_acqf("constrained_logei", "mixed", seed=2))
    xs0 = acqf.search_space.sample_normalized_params(6, np.random.RandomState(4))
    (x1, f1), w1 = _records(lambda: optim_mixed.local_search_mixed_batched(acqf, xs0, max_iter=1))
    (x2, f2), w2 = _records(lambda: _acqf_search._local_search_mixed(acqf, _evaluator(acqf, []), xs0, max_iter=1))
    assert np.array_equal(x1, x2) and np.array_equal(f1, f2)
    assert w1 == w2 == ["local_search_mixed: Local search did not converge."]


def test_task_error_is_raised():
    """An exception inside a lock-step search is raised to the caller after every search has stopped."""
    acqf = _RowWise(_acqf("logei", "float"))

    def evaluate(x, grad):
        if grad:
            raise FloatingPointError("boom")
        return acqf.eval_acqf_no_grad(x)
    with pytest.raises(FloatingPointError, match="boom"):
        _acqf_search.optimize_acqf_mixed(acqf, evaluate, n_preliminary_samples=64, rng=np.random.RandomState(0))


def test_substitute_engine_keeps_optuna_search(monkeypatch):
    """An engine class without ``acqf_set`` / ``acqf_eval`` keeps optuna's search over the per-GP queries."""
    from optuna_b200 import gp_sampler
    from optuna_b200.gp_sampler import _answers_acqf
    from tests._gp_sampler_engine import NumpyGPSamplerEngine
    assert not _answers_acqf(NumpyGPSamplerEngine)
    from optuna_b200.engine import TPEEngine
    assert _answers_acqf(TPEEngine)
    monkeypatch.setattr(gp_sampler, "_engine_cls", NumpyGPSamplerEngine)
    sampler = gp_sampler.GPSampler(seed=0, n_startup_trials=3)
    study = optuna.create_study(sampler=sampler)
    study.optimize(lambda t: (t.suggest_float("x", 0, 1) - 0.3) ** 2, n_trials=5)
    assert sampler._acqf_engine is None and not hasattr(sampler, "last_acqf_calls")
    sampler.close()


# ---- on the GPU ----------------------------------------------------------------------------------------------------

def _device_pair(which, n=80):
    """optuna's acquisition ``which`` over device GPs (``_DeviceGP``) and its ``_DeviceAcqf`` on a fresh engine."""
    from optuna._gp import search_space as gp_search_space
    from optuna.search_space import intersection_search_space

    from optuna_b200 import TPEEngine
    from optuna_b200.gp_sampler import _DeviceAcqf, _DeviceLogEHVI
    from tests.test_gp_sampler import _acqf_pair
    from tests.test_terminator_gpu_gp import _study
    trials = _study("mixed", n, seed=3).trials
    space = gp_search_space.SearchSpace(intersection_search_space(trials))
    X = space.get_normalized_params(trials)
    y = np.array([t.value for t in trials])
    y = (y - y.mean()) / y.std()
    base = which.replace("_infeasible", "").replace("_far", "")
    (_, host), engines = _acqf_pair(TPEEngine, base, X, y, space.is_categorical, space)
    if which == "constrained_logehvi_infeasible":
        host._acqf = None
    if which == "logei_far":   # z < -25 everywhere away from the data
        host._threshold = float(y.max()) + 40.0
    acq = TPEEngine(0)
    engines.append(acq)
    ehvi = TPEEngine(0)
    engines.append(ehvi)
    dev_in = host
    if type(host) is acqf_module.LogEHVI:
        dev_in = _DeviceLogEHVI(host, ehvi)
    elif type(host) is acqf_module.ConstrainedLogEHVI and host._acqf is not None:
        dev_in = acqf_module.ConstrainedLogEHVI.__new__(acqf_module.ConstrainedLogEHVI)
        dev_in.__dict__.update(host.__dict__)
        dev_in._acqf = _DeviceLogEHVI(host._acqf, ehvi)
    dev = _DeviceAcqf.build(acq, dev_in)
    assert dev is not None
    return space, X, host, dev, engines


_DEVICE_KINDS = ["logei", "logei_running", "logei_neginf", "logei_far", "constrained_logei", "logehvi",
                 "constrained_logehvi", "constrained_logehvi_infeasible"]


def _close(engines):
    for e in engines:
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("which", _DEVICE_KINDS)
def test_acqf_eval_against_torch(which):
    """Values within 1e-13 relative (1e-13 absolute near 0) and gradients within 1e-12 of the norm of torch's
    acquisition over the same device posteriors; training points (variance at its clamp) included."""
    space, X, host, dev, engines = _device_pair(which)
    try:
        xs = np.concatenate([space.sample_normalized_params(200, rng=np.random.RandomState(0)), X[:4]])
        want = host.eval_acqf_no_grad(xs)
        got = dev.evaluate(xs, False)
        assert np.all(np.abs(got - want) <= 1e-13 * np.abs(want) + 1e-13), np.max(np.abs(got - want))
        if which == "logei_neginf":   # the reference's constant zeros: no gradient
            gw = np.zeros_like(xs)
        else:
            xt = torch.from_numpy(xs).requires_grad_(True)
            host.eval_acqf(xt).sum().backward()
            gw = xt.grad.numpy()
        v, g = dev.evaluate(xs, True)
        assert np.array_equal(v, got)
        assert np.array_equal(np.isnan(g), np.isnan(gw))
        ok = ~np.isnan(gw).any(axis=1)
        err = np.linalg.norm(g[ok] - gw[ok], axis=1)
        assert np.all(err <= 1e-12 * np.linalg.norm(gw[ok], axis=1) + 1e-300), np.max(err)
    finally:
        _close(engines)


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["logei", "constrained_logei", "constrained_logehvi"])
def test_row_bits_independent_of_batch(which):
    """A row's value is the same bits alone, inside 2 048 rows, with and without gradients, and on repeated calls;
    its gradient is the same bits alone and in the batch."""
    space, X, host, dev, engines = _device_pair(which)
    try:
        xs = space.sample_normalized_params(2048, rng=np.random.RandomState(1))
        v_all = dev.evaluate(xs, False)
        v_all_g, g_all = dev.evaluate(xs, True)
        assert np.array_equal(v_all, v_all_g) and np.array_equal(v_all, dev.evaluate(xs, False))
        for i in (0, 777, 2047):
            v1 = dev.evaluate(xs[i:i + 1], False)
            v1g, g1 = dev.evaluate(xs[i:i + 1], True)
            assert v1[0] == v_all[i] and v1g[0] == v_all[i] and np.array_equal(g1[0], g_all[i])
    finally:
        _close(engines)


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["logei", "constrained_logei", "logehvi", "constrained_logehvi_infeasible"])
def test_driver_bits_equal_optuna_search_on_device(which):
    """The lock-step search over the device acquisition returns the bits of optuna's own ``optimize_acqf_mixed``
    over the same acquisition, leaves the stream where it leaves it, and needs fewer device calls."""
    space, X, host, dev, engines = _device_pair(which)
    try:
        r1, r2 = np.random.RandomState(3), np.random.RandomState(3)
        warm = X[:1]
        n0 = dev.calls
        x1, f1 = optim_mixed.optimize_acqf_mixed(dev, warmstart_normalized_params_array=warm, rng=r1)
        seq = dev.calls - n0
        x2, f2 = _acqf_search.optimize_acqf_mixed(dev, dev.evaluate, warmstart_normalized_params_array=warm, rng=r2)
        assert np.array_equal(x1, x2) and f1 == f2
        assert r1.randint(1 << 30) == r2.randint(1 << 30)
        assert dev.calls - n0 - seq < seq
    finally:
        _close(engines)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["single", "constrained", "two", "two_constrained", "mixed_int"])
def test_end_to_end_against_optuna(case):
    """The drop-in with the device search against ``optuna.samplers.GPSampler``, at the replay tolerance of
    tests/test_gp_sampler.py."""
    from tests.test_gp_sampler import _dists, _history, _replay
    if case == "mixed_int":
        d = dict(_dists("mixed"), w=D.IntDistribution(0, 40))
        _replay(d, _history(d, 14, 1, 6, False), 2, seed=6)
        return
    n_obj = 2 if case.startswith("two") else 1
    constrained = case.endswith("constrained")
    d = _dists("float" if n_obj == 2 else "mixed")
    _replay(d, _history(d, 14, n_obj, 7, constrained), 2, n_obj=n_obj, constrained=constrained, seed=7)


@pytest.mark.gpu
def test_end_to_end_same_as_previous_path(monkeypatch):
    """Two-objective asks: log-EHVI's values are the previous path's bits (the same posterior and EHVI kernels, the
    same sqrt), so the suggestions match the per-GP path to within the gradient's rounding; counted calls drop."""
    from optuna_b200 import gp_sampler
    from tests.test_gp_sampler import _dists, _history
    d = _dists("float")
    hist = _history(d, 16, 2, 8, False)
    out = []
    for fused in (True, False):
        if not fused:
            monkeypatch.setattr(gp_sampler, "_answers_acqf", lambda cls: False)
        sampler = gp_sampler.GPSampler(seed=8)
        study = optuna.create_study(directions=["minimize"] * 2, sampler=sampler)
        study.add_trials(hist)
        try:
            t = study.ask(d)
            out.append(np.array([t.params[k] for k in d]))
        finally:
            sampler.close()
    assert np.max(np.abs(out[0] - out[1])) <= 1e-6, out


@pytest.mark.gpu
def test_errors():
    """Each refusal of tpe_acqf_set / tpe_acqf_eval is a message, not a fault."""
    from optuna_b200 import TPEEngine
    from tests.test_gp_sampler import _params
    rs = np.random.RandomState(0)
    X, y = rs.uniform(0, 1, (30, 3)), rs.normal(size=30)
    cat = np.zeros(3, dtype=bool)
    g1, g2, g3, acq = TPEEngine(0), TPEEngine(0), TPEEngine(0), TPEEngine(0)
    try:
        for g in (g1, g2):
            g.gp_set_data(X, y, cat)
        g3.gp_set_data(X[:, :2], y, cat[:2])
        with pytest.raises(RuntimeError, match="GP context 0 is not conditioned"):
            acq.acqf_set(TPEEngine.ACQF_LOGEI, [g1], 1, [0.0])
        g1.gp_condition(_params(3, 0))
        g2.gp_condition(_params(3, 1))
        g3.gp_condition(_params(2, 2))
        with pytest.raises(ValueError, match="GP context 1 has width 2, GP context 0 has width 3"):
            acq.acqf_set(TPEEngine.ACQF_LOGEI, [g1, g3], 1, [0.0, 0.1])
        with pytest.raises(ValueError, match="are the same context"):
            acq.acqf_set(TPEEngine.ACQF_LOGEI, [g1, g1], 1, [0.0, 0.1])
        with pytest.raises(ValueError, match="takes 1 objective GPs, got 2"):
            acq.acqf_set(TPEEngine.ACQF_LOGEI, [g1, g2], 2, [0.0, 0.1])
        acq.acqf_set(TPEEngine.ACQF_LOGEI, [g1, g2], 1, [0.0, 0.1])
        with pytest.raises(ValueError, match="Q 0"):
            acq.acqf_eval(np.empty((0, 3)))
        with pytest.raises(ValueError, match=r"X must be \[Q, 3\]"):
            acq.acqf_eval(np.zeros((2, 2)))
        acq.acqf_eval(rs.uniform(0, 1, (4, 3)), grad=True)
        # a NaN query point (an L-BFGS-B iterate after a NaN gradient) gives NaN, as torch does, not an error
        v, g = acq.acqf_eval(np.array([[np.nan, 0.5, 0.5], [0.5, 0.5, 0.5]]), grad=True)
        assert np.isnan(v[0]) and np.isnan(g[0]).all() and np.isfinite(v[1]) and np.isfinite(g[1]).all()
        g2.gp_condition(_params(3, 3))
        with pytest.raises(RuntimeError, match="GP context 1 was re-conditioned or changed since tpe_acqf_set"):
            acq.acqf_eval(rs.uniform(0, 1, (4, 3)))
        if torch.cuda.device_count() > 1:
            other = TPEEngine(1)
            try:
                other.gp_set_data(X, y, cat)
                other.gp_condition(_params(3, 0))
                with pytest.raises(ValueError, match="is on device 1, the acquisition context on device 0"):
                    acq.acqf_set(TPEEngine.ACQF_LOGEI, [other], 1, [0.0])
            finally:
                other.close()
    finally:
        for e in (g1, g2, g3, acq):
            e.close()


@pytest.mark.gpu
def test_short_of_memory_names_the_bytes():
    """An evaluation whose device buffers exceed the device (64 GPs, 27 M rows with gradients: about 83 GB on the
    device for 1.5 GB on the host) fails with a message naming the bytes."""
    from optuna_b200 import TPEEngine
    from tests.test_gp_sampler import _params
    rs = np.random.RandomState(0)
    X, y = rs.uniform(0, 1, (20, 3)), rs.normal(size=20)
    gps = [TPEEngine(0) for _ in range(64)]
    acq = TPEEngine(0)
    try:
        for k, g in enumerate(gps):
            g.gp_set_data(X, y, np.zeros(3, dtype=bool))
            g.gp_condition(_params(3, k))
        acq.acqf_set(TPEEngine.ACQF_LOGPI, gps, 0, np.zeros(64))
        with pytest.raises(ValueError, match=r"needs \d+ more bytes of device memory, device 0 has \d+ free"):
            acq.acqf_eval(np.full((27_000_000, 3), 0.5), grad=True)
    finally:
        for e in gps + [acq]:
            e.close()
