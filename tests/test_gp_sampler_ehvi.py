"""``GPSampler``'s multi-objective acquisition on the device (``TPEEngine.ehvi_set`` / ``ehvi``, tpe_ehvi.cuh, and
``gp_sampler._DeviceLogEHVI``) against the live reference's ``logehvi``, ``LogEHVI``, ``ConstrainedLogEHVI`` and
``optuna.samplers.GPSampler`` (optuna/_gp/acqf.py:45-62, 245-337).

Every case runs twice: through ``NumpyEHVIEngine`` (tests/_gp_sampler_ehvi_engine.py: the GP calls and the kernel's
algorithm in NumPy, runs anywhere) and, with ``-m gpu``, through libtpe_b200.so.  Tolerances:
- log-EHVI against ``logehvi`` on the same ``Y_post`` and its torch autograd gradient: values within 1e-12 relative (an
  absolute floor of 1e-12), gradients within 1e-10 of their norm;
- acquisition values within 1e-9 relative (1e-9 absolute floor), their gradients within 1e-7 of their norm;
- replayed suggestions: normalised parameters within 1e-6 of the reference's.
"""
from __future__ import annotations

import time

import numpy as np
import pytest

optuna = pytest.importorskip("optuna")
torch = pytest.importorskip("torch")

import tests.test_gp_sampler as tgs  # noqa: E402

_EPS = 1e-12


@pytest.fixture(params=[pytest.param("numpy", id="numpy-engine"),
                        pytest.param("cuda", id="cuda-engine", marks=pytest.mark.gpu)])
def engine_cls(request, monkeypatch):
    """The engine class behind optuna_b200.gp_sampler: the NumPy restatement or the CUDA library."""
    from optuna_b200 import TPEEngine, gp_sampler
    from tests._gp_sampler_ehvi_engine import NumpyEHVIEngine
    cls = NumpyEHVIEngine if request.param == "numpy" else TPEEngine
    monkeypatch.setattr(gp_sampler, "_engine_cls", cls)
    return cls


def _dtlz2(X, M):
    """DTLZ2 (Deb et al., 2005) over X in [0, 1]^P, P >= M: M objectives to minimise."""
    half = 0.5 * np.pi
    g = ((X[:, M - 1:] - 0.5) ** 2).sum(1)
    out = np.empty((X.shape[0], M))
    for m in range(M):
        f = 1.0 + g
        for i in range(M - 1 - m):
            f = f * np.cos(half * X[:, i])
        if m > 0:
            f = f * np.sin(half * X[:, M - 1 - m])
        out[:, m] = f
    return out


class _Stub:
    """What ``LogEHVI.__init__`` reads of a GP: its length scales."""

    def __init__(self, P):
        self.length_scales = np.ones(P)


def _log_ehvi_state(M, n, S=128, seed=0, P=8):
    """The boxes and samples optuna's ``LogEHVI`` builds for a seeded DTLZ2 study of n trials: (lower, intervals,
    samples) as torch tensors."""
    from optuna._gp import acqf
    from optuna._gp import search_space as gp_search_space
    rs = np.random.RandomState(seed)
    Y = -_dtlz2(rs.uniform(0, 1, (n, P)), M)
    Y = (Y - Y.mean(0)) / np.maximum(Y.std(0), 1e-12)
    space = gp_search_space.SearchSpace(
        {f"x{j}": optuna.distributions.FloatDistribution(0, 1) for j in range(P)})
    a = acqf.LogEHVI([_Stub(P)] * M, space, torch.from_numpy(Y), S, seed + 7)
    return a._non_dominated_box_lower_bounds, a._non_dominated_box_intervals, a._fixed_samples


def _rows(Q, M, seed):
    rs = np.random.RandomState(seed)
    return rs.normal(0.0, 1.0, (Q, M)), rs.uniform(0.05, 1.5, (Q, M))


def _reference(mean, sd, lb, iv, Z):
    """``logehvi`` on torch's ``Y_post`` (acqf.py:291) and its autograd gradients in mean and sd."""
    from optuna._gp import acqf
    m = torch.from_numpy(mean).requires_grad_(True)
    s = torch.from_numpy(sd).requires_grad_(True)
    Y = torch.stack([m[:, None, j] + s[:, None, j] * Z[..., j] for j in range(mean.shape[1])], dim=-1)
    v = acqf.logehvi(Y, lb, iv)
    v.sum().backward()
    return v.detach().numpy(), m.grad.numpy(), s.grad.numpy()


def _ours(engine_cls, lb, iv, Z, mean, sd):
    eng = engine_cls(0)
    try:
        eng.ehvi_set(np.asarray(lb), np.asarray(iv), np.asarray(Z))
        return eng.ehvi(mean, sd, grad=True), eng.ehvi(mean, sd)
    finally:
        eng.close()


def _check(want, got):
    v, dm, ds = want
    gv, gdm, gds = got
    assert np.all(np.abs(gv - v) <= 1e-12 * np.abs(v) + 1e-12), np.max(np.abs(gv - v))
    for w, g in ((dm, gdm), (ds, gds)):
        assert np.linalg.norm(g - w) <= 1e-10 * np.linalg.norm(w) + 1e-300, (np.linalg.norm(g - w), np.linalg.norm(w))


# ---- the kernel against logehvi and autograd -------------------------------------------------------------------------

@pytest.mark.parametrize("M,n,S,Q", [
    (2, 1, 128, 9),       # one trial: B = 2 boxes
    (2, 60, 128, 9),
    (3, 80, 37, 7),       # an odd S below one sample per thread
    (3, 300, 128, 5),     # B not a multiple of the chunk
    (4, 120, 300, 4),     # S over two samples per thread
    (6, 40, 128, 3),
    (4, 1000, 128, 2),    # B near 3 500 (DTLZ2, 4 x 1 000)
])
def test_kernel_against_logehvi(engine_cls, M, n, S, Q):
    lb, iv, Z = _log_ehvi_state(M, n, S, seed=n)
    if n == 1000:
        assert lb.shape[0] > 3000
    if M == 2 and n == 60:   # and one box alone
        lb, iv = lb[:1], iv[:1]
    mean, sd = _rows(Q, M, M + n)
    want = _reference(mean, sd, lb, iv, Z)
    got, values_only = _ours(engine_cls, lb, iv, Z, mean, sd)
    _check(want, got)
    assert values_only.tobytes() == got[0].tobytes()


def _compare_nan(want, got):
    for w, g in zip(want, got):
        assert np.array_equal(np.isnan(w), np.isnan(g)), (w, g)
        assert np.array_equal(np.isinf(w), np.isinf(g)), (w, g)
        ok = np.isfinite(w)
        assert np.allclose(g[ok], w[ok], rtol=1e-12, atol=1e-12), (w, g)


def test_edge_cases(engine_cls):
    """+inf intervals; differences exactly at EPS and at the interval, where the inclusive clamp mask passes the
    gradient; a box in which every sample is clamped below, which adds nothing to the gradient."""
    M = 3
    lb = torch.tensor([[0.0, 0.0, 0.0], [0.0, -1.0, 100.0], [-0.5, 0.2, -0.3]], dtype=torch.float64)
    iv = torch.tensor([[np.inf, 0.5, np.inf], [1.0, np.inf, 2.0], [0.7, np.inf, 0.4]], dtype=torch.float64)
    Z = torch.tensor([[0.0, 0.0, 0.0], [0.3, -1.2, 0.8], [-0.1, 0.5, 1.4]], dtype=torch.float64)
    # row 0: with z = 0, y = mean: y - lb = EPS exactly in objective 0 and = I = 0.5 in objective 1 for box 0
    mean = np.array([[_EPS, 0.5, 0.25], [0.4, 0.1, -0.2]])
    sd = np.array([[0.3, 0.2, 0.1], [0.5, 0.4, 0.6]])
    want = _reference(mean, sd, lb, iv, Z)
    got, values_only = _ours(engine_cls, lb, iv, Z, mean, sd)
    _check(want, got)
    assert values_only.tobytes() == got[0].tobytes()
    # box 1 alone: every sample is clamped below its lower bound of 100 in objective 2, whose gradients are then
    # exactly 0, as in torch
    want = _reference(mean, sd, lb[1:2], iv[1:2], Z)
    got, _ = _ours(engine_cls, lb[1:2], iv[1:2], Z, mean, sd)
    _check(want, got)
    for w, g in zip(want[1:], got[1:]):
        assert np.all(w[:, 2] == 0.0) and np.all(g[:, 2] == 0.0)


def test_infinite_sample_and_lower_bound(engine_cls):
    """A sample of -inf (erfinv(-1) of a Sobol point at 0) and an infinite lower bound: the values and the NaN and inf
    pattern of the gradients equal torch's."""
    lb = torch.tensor([[0.0, 0.0], [-0.5, 0.3], [1.0, -1.0]], dtype=torch.float64)
    iv = torch.tensor([[np.inf, 0.5], [0.7, np.inf], [np.inf, 2.0]], dtype=torch.float64)
    Z = torch.tensor([[-np.inf, 0.2], [0.3, -1.2], [0.5, -np.inf]], dtype=torch.float64)
    mean, sd = _rows(4, 2, 3)
    want = _reference(mean, sd, lb, iv, Z)
    assert np.isnan(want[2]).any() and np.isfinite(want[0]).all()
    got, _ = _ours(engine_cls, lb, iv, Z, mean, sd)
    _compare_nan(want, got)
    lb_inf = lb.clone()
    lb_inf[1, 0] = -np.inf
    iv_inf = iv.clone()
    iv_inf[1, 0] = np.inf
    Zf = torch.tensor([[-0.4, 0.2], [0.3, -1.2], [0.5, 0.1]], dtype=torch.float64)
    want = _reference(mean, sd, lb_inf, iv_inf, Zf)
    got, _ = _ours(engine_cls, lb_inf, iv_inf, Zf, mean, sd)
    _compare_nan(want, got)


# ---- the same bits -----------------------------------------------------------------------------------------------------

def test_same_bits(engine_cls):
    """A row's value is the same bits in a values-only call of 2 048 rows and in gradient calls of 1 and 10 rows,
    wherever it sits; repeats are bit-identical."""
    lb, iv, Z = _log_ehvi_state(3, 300, 128, seed=5)
    assert lb.shape[0] > 64
    mean, sd = _rows(2048, 3, 11)
    eng = engine_cls(0)
    try:
        eng.ehvi_set(lb.numpy(), iv.numpy(), Z.numpy())
        big = eng.ehvi(mean, sd)
        assert eng.ehvi(mean, sd).tobytes() == big.tobytes()
        for i in (0, 1000, 2047):
            one = eng.ehvi(mean[i:i + 1], sd[i:i + 1], grad=True)
            assert one[0].tobytes() == big[i:i + 1].tobytes()
        rows = np.array([5, 2047, 0, 999, 1500, 3, 1024, 64, 7, 1800])
        ten = eng.ehvi(mean[rows], sd[rows], grad=True)
        assert ten[0].tobytes() == big[rows].tobytes()
        again = eng.ehvi(mean[rows], sd[rows], grad=True)
        for a, b in zip(ten, again):
            assert a.tobytes() == b.tobytes()
        one = eng.ehvi(mean[1024:1025], sd[1024:1025], grad=True)
        assert one[1].tobytes() == ten[1][6:7].tobytes() and one[2].tobytes() == ten[2][6:7].tobytes()
    finally:
        eng.close()


# ---- the acquisition functions on both GPs ---------------------------------------------------------------------------

@pytest.mark.parametrize("which", ["logehvi", "constrained", "all_infeasible"])
@pytest.mark.parametrize("M", [2, 3, 4])
def test_acquisition_against_reference(engine_cls, which, M):
    """The wrapper over device GPs against optuna's ``LogEHVI`` / ``ConstrainedLogEHVI`` over ``GPRegressor``s."""
    from optuna._gp import acqf
    from optuna._gp import search_space as gp_search_space
    from optuna.search_space import intersection_search_space
    from optuna_b200.gp_sampler import _DeviceLogEHVI
    from tests.test_terminator_gpu_gp import _study
    trials = _study("mixed", 60, seed=M).trials
    space = gp_search_space.SearchSpace(intersection_search_space(trials))
    X = space.get_normalized_params(trials)
    cat = space.is_categorical
    y = np.array([t.value for t in trials])
    y = (y - y.mean()) / y.std()
    Y = np.stack([y] + [np.sin(3.0 * y + k) + 0.3 * X[:, k % X.shape[1]] for k in range(1, M)], 1)
    engines = []
    pairs = []
    for k in range(M + 1):
        params = tgs._params(X.shape[1], 20 + k)
        yk = Y[:, k] if k < M else np.cos(2.0 * y)
        eng, dev = tgs._device_gp(engine_cls, X, yk, cat, params)
        engines.append(eng)
        pairs.append((tgs._ref_gp(X, yk, cat, params), dev))
    ehvi_eng = engine_cls(0)
    engines.append(ehvi_eng)
    try:
        out = []
        for side in (0, 1):
            gprs = [p[side] for p in pairs[:M]]
            if which == "logehvi":
                a = acqf.LogEHVI(gprs, space, torch.from_numpy(Y), 128, 11)
            else:
                feasible = None if which == "all_infeasible" else torch.from_numpy(Y[:25])
                a = acqf.ConstrainedLogEHVI(gprs, space, feasible, 128, 11, [pairs[M][side]], [-0.2])
            if side == 1:
                if which == "logehvi":
                    a = _DeviceLogEHVI(a, ehvi_eng)
                elif a._acqf is not None:
                    a._acqf = _DeviceLogEHVI(a._acqf, ehvi_eng)
            out.append(a)
        ref, dev = out
        np.testing.assert_array_equal(ref.length_scales, dev.length_scales)
        xs = space.sample_normalized_params(300, rng=np.random.RandomState(M))
        tgs._check_acqf(ref.eval_acqf_no_grad(xs), dev.eval_acqf_no_grad(xs))
        for x in xs[:5]:
            vr, gr = ref.eval_acqf_with_grad(x.copy())
            vd, gd = dev.eval_acqf_with_grad(x.copy())
            tgs._check_acqf(np.array([vr]), np.array([vd]))
            assert np.linalg.norm(gd - gr) <= 1e-7 * np.linalg.norm(gr) + 1e-12, (gr, gd)
        # the batched shape of the local searches: [Q, P] with gradients
        xb = xs[5:9].copy()
        tr = torch.from_numpy(xb).requires_grad_(True)
        td = torch.from_numpy(xb.copy()).requires_grad_(True)
        ref.eval_acqf(tr).sum().backward()
        dev.eval_acqf(td).sum().backward()
        assert np.linalg.norm(td.grad.numpy() - tr.grad.numpy()) <= 1e-7 * np.linalg.norm(tr.grad.numpy()) + 1e-12
    finally:
        for e in engines:
            e.close()


# ---- end-to-end replay against optuna.samplers.GPSampler -------------------------------------------------------------

def _values_mo(params, n_obj):
    """n_obj conflicting objectives of the replay's float space."""
    x = np.array([float(p) for p in params.values()])
    out = [float(((x - 0.5 * j) ** 2).sum() + 0.3 * j * x[j % x.size]) for j in range(n_obj)]
    return out


@pytest.mark.parametrize("constrained", [False, True])
@pytest.mark.parametrize("n_obj", [2, 3, 4])
def test_replay_many_objectives(engine_cls, monkeypatch, n_obj, constrained):
    """Suggestions against optuna's; every ask's acquisition goes through the device log-EHVI.  Two objectives replay
    the history of ``test_gp_sampler.test_replay_two_objectives``."""
    from optuna_b200.gp_sampler import _DeviceLogEHVI
    built = []
    real_init = _DeviceLogEHVI.__init__

    def init(self, host, engine):
        built.append(engine)
        real_init(self, host, engine)
    monkeypatch.setattr(_DeviceLogEHVI, "__init__", init)
    d = tgs._dists("float")
    if n_obj == 2:
        tgs._replay(d, tgs._history(d, 14, 2, 3, constrained), 2, n_obj=2, constrained=constrained, seed=2)
    else:
        monkeypatch.setattr(tgs, "_values", _values_mo)
        tgs._replay(d, tgs._history(d, 14, n_obj, 40 + n_obj, constrained), 2, n_obj=n_obj, constrained=constrained,
                    seed=n_obj)
    assert len(built) == 2 and all(isinstance(e, engine_cls) for e in built)


def test_engine_without_ehvi_keeps_host_acquisition(monkeypatch):
    """An engine class that answers only the GP calls (``NumpyGPSamplerEngine``) leaves the acquisition to optuna's
    host ``LogEHVI`` and ``ConstrainedLogEHVI``, and no EHVI engine is created."""
    from optuna._gp import acqf
    from optuna_b200 import GPSampler, gp_sampler
    from tests._gp_sampler_engine import NumpyGPSamplerEngine
    monkeypatch.setattr(gp_sampler, "_engine_cls", NumpyGPSamplerEngine)
    assert not gp_sampler._answers_ehvi(NumpyGPSamplerEngine)
    d = tgs._dists("float")
    for constrained in (False, True):
        sampler = GPSampler(seed=0, constraints_func=tgs._constraints_func if constrained else None)
        seen = _capture_acqf(sampler)
        study = optuna.create_study(directions=["minimize"] * 2, sampler=sampler)
        study.add_trials(tgs._history(d, 12, 2, 5, constrained))
        try:
            study.ask(d)
        finally:
            sampler.close()
        inner = seen[0]._acqf if constrained else seen[0]
        assert type(inner) is acqf.LogEHVI and sampler._ehvi_engine is None


# ---- limits -------------------------------------------------------------------------------------------------------------

def _capture_acqf(sampler):
    seen = []

    def fake(acqf, best_params):
        seen.append(acqf)
        return np.full(len(acqf.length_scales), 0.5)
    sampler._optimize_acqf = fake
    return seen


@pytest.mark.parametrize("M", [24, 25])
def test_objective_limit(engine_cls, M):
    """Up to 24 objectives the sampler evaluates log-EHVI on the device; at 25 it keeps optuna's host ``LogEHVI``.
    One trial dominates the others, so the front is one point and there are few boxes."""
    from optuna._gp import acqf
    from optuna_b200 import GPSampler
    from optuna_b200.gp_sampler import _DeviceLogEHVI
    D = optuna.distributions
    dists = {"x0": D.FloatDistribution(0, 1), "x1": D.FloatDistribution(0, 1)}
    rs = np.random.RandomState(M)
    trials = []
    for i in range(6):
        v = float(i) + 0.01 * rs.uniform(0, 1, M)
        trials.append(optuna.trial.create_trial(params={"x0": float(rs.uniform()), "x1": float(rs.uniform())},
                                                distributions=dists, values=list(v)))
    sampler = GPSampler(seed=0, n_startup_trials=2)
    seen = _capture_acqf(sampler)
    study = optuna.create_study(directions=["minimize"] * M, sampler=sampler)
    study.add_trials(trials)
    try:
        study.ask(dists)
        assert len(seen) == 1
        if M == 25:
            assert type(seen[0]) is acqf.LogEHVI and sampler._ehvi_engine is None
        else:
            assert isinstance(seen[0], _DeviceLogEHVI) and sampler._ehvi_engine is not None
            # the same acquisition as optuna's host LogEHVI built by the same ask
            sampler2 = GPSampler(seed=0, n_startup_trials=2)
            seen2 = _capture_acqf(sampler2)
            sampler2._device_ehvi = lambda a: a
            study2 = optuna.create_study(directions=["minimize"] * M, sampler=sampler2)
            study2.add_trials(trials)
            try:
                study2.ask(dists)
                xs = np.random.RandomState(1).uniform(0, 1, (5, 2))
                tgs._check_acqf(seen2[0].eval_acqf_no_grad(xs), seen[0].eval_acqf_no_grad(xs))
            finally:
                sampler2.close()
    finally:
        sampler.close()
    assert sampler._ehvi_engine is None


@pytest.mark.parametrize("shape,change,message", [
    ((3, 1, 5), None, "EHVI needs 2 <= M <= 24 objectives, got 1"),
    ((3, 25, 5), None, "EHVI needs 2 <= M <= 24 objectives, got 25"),
    ((3, 2, 0), None, "EHVI needs 1 <= S <= 1024 samples, got 0"),
    ((3, 2, 1025), None, "EHVI needs 1 <= S <= 1024 samples, got 1025"),
    ((0, 2, 5), None, "EHVI needs 1 <= B <= 2^31 boxes, got 0"),
    ((3, 2, 5), 0, "EHVI box lower bounds hold a NaN"),
    ((3, 2, 5), 1, "EHVI box intervals hold a NaN"),
    ((3, 2, 5), 2, "EHVI samples hold a NaN"),
])
def test_invalid_inputs(engine_cls, shape, change, message):
    B, M, S = shape
    args = [np.zeros((B, M)), np.ones((B, M)), np.zeros((S, M))]
    if change is not None:
        args[change][-1, -1] = np.nan
    eng = engine_cls(0)
    try:
        with pytest.raises(ValueError, match=message.replace("^", r"\^")):
            eng.ehvi_set(*args)
        with pytest.raises(RuntimeError):   # a failed set leaves no state
            eng.ehvi(np.zeros((1, 2)), np.ones((1, 2)))
    finally:
        eng.close()


def test_ehvi_before_set(engine_cls):
    eng = engine_cls(0)
    try:
        with pytest.raises(RuntimeError, match="tpe_ehvi_set"):
            eng.ehvi(np.zeros((2, 3)), np.ones((2, 3)))
        eng.ehvi_set(np.zeros((1, 3)), np.ones((1, 3)), np.zeros((4, 3)))
        assert eng.ehvi(np.zeros((2, 3)), np.ones((2, 3))).shape == (2,)
    finally:
        eng.close()


# ---- GPU only ------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_four_objectives_thousand_trials():
    """One GP ask of a four-objective DTLZ2 study of 1 000 trials over 8 parameters, on the device: about 3 500 boxes,
    where optuna's host acquisition would need about 29 GB for each (2 048, 128, B, 4) intermediate tensor.  The test
    holds about 100 MB of device memory (four 1 000 x 1 000 GPs, the boxes and the partial sums of 2 048 rows) and
    takes seconds: the fits, the host box decomposition and the acquisition search."""
    from optuna_b200 import GPSampler
    D = optuna.distributions
    P, M, n = 8, 4, 1000
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
        t0 = time.perf_counter()
        t = study.ask(dists)
        dt = time.perf_counter() - t0
    finally:
        sampler.close()
    assert set(t.params) == set(dists) and all(0.0 <= v <= 1.0 for v in t.params.values())
    assert dt < 120.0, dt
