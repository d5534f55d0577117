"""MOTPE on every device path, 2 to 16 objectives (tests/_motpe_cases.py names the path each case reaches).

Yardstick: the live reference's own functions (oracle/_ref) -- `_split_trials` / `_split_complete_trials_multi_objective`
for the below set and `_calculate_weights_below_for_multi_objective` for its hypervolume weights.

Exact-tie cases (simplex lattices): contributions tie exactly, so the reference's greedy HSSP answer rests on two
choices it leaves to the platform.  (1) It visits candidates in `np.argsort(-bound)` order (hssp.py:80, numpy's
unstable sort).  (2) Its 3-D hypervolume ends in two BLAS products (wfg.py `_compute_3d`, `np.dot`), whose summation
order depends on the BLAS kernel the CPU dispatches to.  The device visits tied bounds by ascending index and sums the
3-D hypervolume row by row in index order.  A tie case whose reference answer changes when the reference is run with
a stable argsort and that row-by-row 3-D sum is compared with that run; every other case is compared with the
reference as it runs."""
import math
import types

import numpy as np
import pytest

from oracle import motpe as mo
from tests._motpe_cases import (split_cases, split_path, split_structure, weights_cases, weights_path,
                                weights_structure)

optuna = pytest.importorskip("optuna")
from optuna._hypervolume import hssp as ref_hssp  # noqa: E402
from optuna._hypervolume import wfg as ref_wfg  # noqa: E402
from optuna.samplers._base import _CONSTRAINTS_KEY  # noqa: E402
from optuna.samplers._tpe import sampler as ref_tpe  # noqa: E402
from optuna.study import StudyDirection  # noqa: E402
from optuna.trial import create_trial  # noqa: E402

SPLIT = {c.name: c for c in split_cases()}
WEIGHTS = {c.name: c for c in weights_cases()}
ALL = {**SPLIT, **WEIGHTS}
TIES = [n for n, c in SPLIT.items() if c.tie_order]


class _StableNumpy:
    """numpy with a stable argsort, swapped in as optuna._hypervolume.hssp's `np`."""

    def __getattr__(self, name):
        return getattr(np, name)

    @staticmethod
    def argsort(a, *args, **kw):
        return np.argsort(a, kind="stable")


def _compute_3d_rowwise(sorted_pareto_sols, reference_point):
    """wfg.py `_compute_3d` with its two BLAS products summed in index order (rows stably sorted by x, then the
    cumulative-max table walked in stable y order): the order the device's 3-D hypervolume (hv3_warp) uses."""
    s = sorted_pareto_sols[np.argsort(sorted_pareto_sols[:, 0], kind="stable")]
    n = s.shape[0]
    yo = np.argsort(s[:, 1], kind="stable")
    total = 0.0
    for i in range(n):
        dx = (s[i + 1, 0] if i + 1 < n else reference_point[0]) - s[i, 0]
        run = inner = 0.0
        for j in range(n):
            o = yo[j]
            if o <= i:
                run = max(run, reference_point[2] - s[o, 2])
            dy = (s[yo[j + 1], 1] if j + 1 < n else reference_point[1]) - s[o, 1]
            inner = inner + run * dy
        total = total + inner * dx
    return total


def _trials(case):
    feas = np.ones(len(case.v), bool) if case.feas is None else case.feas
    out = []
    for i, (row, f) in enumerate(zip(case.v, feas)):
        t = create_trial(values=[float(x) for x in row], system_attrs={_CONSTRAINTS_KEY: [-1.0 if f else 1.0]})
        t.number = i
        out.append(t)
    return out


def _study(M):
    return types.SimpleNamespace(directions=[StudyDirection.MINIMIZE] * M)


_cache: dict = {}


def ref_below(name, stable=False):
    """Trial positions of the reference's below set (COMPLETE trials split by rank + HSSP, then the infeasible
    trials by violation and trial order).  stable: with a stable argsort in hssp.py and the row-by-row 3-D sum."""
    key = ("below", name, stable)
    if key not in _cache:
        case = ALL[name]
        ref_tpe._solve_hssp_with_cache.cache_clear()
        saved = ref_hssp.np, ref_wfg._compute_3d
        if stable:
            ref_hssp.np, ref_wfg._compute_3d = _StableNumpy(), _compute_3d_rowwise
        try:
            below, _ = ref_tpe._split_trials(_study(case.v.shape[1]), _trials(case), case.nb, True)
        finally:
            ref_hssp.np, ref_wfg._compute_3d = saved
            ref_tpe._solve_hssp_with_cache.cache_clear()
        _cache[key] = np.array([t.number for t in below], np.int64)
    return _cache[key]


def ref_weights(name, below):
    key = ("w", name, tuple(below))
    if key not in _cache:
        case = ALL[name]
        trials = _trials(case)
        _cache[key] = ref_tpe._calculate_weights_below_for_multi_objective(
            _study(case.v.shape[1]), [trials[i] for i in below], lambda t: t.system_attrs[_CONSTRAINTS_KEY])
    return _cache[key]


def order_dependent(name):
    return not np.array_equal(ref_below(name), ref_below(name, stable=True))


# ------------------------------------------------------------------------------------------------------------------
# CPU: the cases are what they claim, and the oracle is the reference on every one of them
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(SPLIT))
def test_split_case_reaches_its_path(name):
    c = SPLIT[name]
    s = split_structure(c.v, c.nb)
    assert split_path(s) == c.path, s


@pytest.mark.parametrize("name", list(WEIGHTS))
def test_weights_case_reaches_its_path(name):
    c = WEIGHTS[name]
    assert weights_path(weights_structure(c.v, c.feas)) == c.wpath
    assert c.nb == len(c.v)   # the below set is every row


def test_cases_cover_every_path():
    assert {c.path for c in SPLIT.values()} >= {
        "hssp-2d", "hssp-contrib3-smem", "hssp-contrib3-arena", "hssp-contrib-nd", "hssp-contrib", "ref-not-finite",
        "fill-dups", "whole-ranks"}
    kernels = ("k_mo_weights-smem", "k_mo_weights-arena", "k_mo_weights3", "k_mo_weights_nd", "k_mow-le3", "k_mow-nd")
    got = {c.wpath for c in WEIGHTS.values()}
    assert set(kernels) <= got
    for edge in (":nf<=1", ":hv-inf", ":front-of-one"):
        assert {"k_mow" if k.startswith("k_mow") else "k_mo_weights" for k in got if k.endswith(edge)} == {
            "k_mo_weights", "k_mow"}, edge
    assert {c.v.shape[1] for c in SPLIT.values()} >= {2, 3, 4, 5, 6, 8, 12, 16}


@pytest.mark.parametrize("name", list(ALL))
def test_oracle_is_the_reference(name):
    c = ALL[name]
    feas = np.ones(len(c.v), bool) if c.feas is None else c.feas
    comp = np.flatnonzero(feas)
    want = comp[mo.split_complete_mo(c.v[comp], min(c.nb, comp.size))]
    below = np.sort(np.concatenate([want, np.flatnonzero(~feas)[: c.nb - want.size]]))
    assert np.array_equal(below, ref_below(name))
    w = mo.weights_below_mo(c.v[below], feas[below])
    r = ref_weights(name, below)
    assert np.array_equal(w, r) or np.allclose(w, r, rtol=0, atol=1e-15), np.max(np.abs(w - r))


def device_yardstick(name):
    """The below set the device must produce: the reference's, or for an order-dependent tie case the reference's
    run in the device's orders."""
    return ref_below(name, stable=ALL[name].tie_order and order_dependent(name))


@pytest.mark.parametrize("name", TIES)
def test_tie_cases_are_classified(name):
    """Both runs are valid greedy answers of the same size, and the argsort order alone (3-D sums as the reference
    computes them) reproduces the oracle with a stable argsort."""
    c = SPLIT[name]
    a, b = ref_below(name), ref_below(name, stable=True)
    assert a.size == b.size == c.nb
    saved = mo.np
    mo.np = _StableNumpy()
    try:
        got = mo.split_complete_mo(c.v, c.nb)
    finally:
        mo.np = saved
    if c.v.shape[1] != 3:   # the 3-D sum order only enters at three objectives
        assert np.array_equal(got, b)


def test_row_by_row_3d_sum_is_the_hypervolume():
    """The row-by-row 3-D sum agrees with the reference's BLAS products to rounding."""
    rs = np.random.RandomState(5)
    for n in (1, 2, 5, 17, 40):
        s = rs.dirichlet(np.ones(3), n)
        ref = mo.reference_point(s)
        s = s[np.argsort(s[:, 0])]
        np.testing.assert_allclose(_compute_3d_rowwise(s, ref), ref_wfg._compute_3d(s, ref), rtol=1e-14)


def test_the_fifteen_point_lattice():
    """{(i, j, l) * 0.1 / 4 : i + j + l = 4} in itertools.product order, n_below = 9: the reference picks positions
    [1, 3, 5, 6, 8, 10, 11, 12, 13].  With its 3-D hypervolumes summed row by row the exact contributions tie
    differently and it picks [1, 2, 3, 5, 6, 8, 11, 12, 13]: the case is order-dependent."""
    name = "lattice-M3-L4-s0.1-sorted-k9"
    assert list(ref_below(name)) == [1, 3, 5, 6, 8, 10, 11, 12, 13]
    assert list(ref_below(name, stable=True)) == [1, 2, 3, 5, 6, 8, 11, 12, 13]


# ------------------------------------------------------------------------------------------------------------------
# GPU: the device split and weights against the reference
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def eng():
    from optuna_b200 import TPEEngine
    e = TPEEngine(0)
    yield e
    e.close()


def _run(eng, c):
    from optuna_b200.engine import ParamSpec
    n = len(c.v)
    feas = np.ones(n, bool) if c.feas is None else c.feas
    eng.set_space([ParamSpec(kind=0, low=0.0, high=1.0) for _ in range(2)])
    eng.set_history(np.random.RandomState(n).uniform(0, 1, (n, 2)), np.where(feas, 0, 2).astype(np.int8),
                    np.zeros((n, 2)))
    eng.set_values(c.v, 0)
    info = eng.prepare([0, 1], n_below=c.nb, n_candidates=8, multivariate=True)
    below, _ = eng.get_split()
    assert info[0] == below.size
    w = None
    if below.size:
        eng.build()
        w = eng.get_mo_weights()
    return below, w


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(ALL))
def test_device_split_and_weights(eng, name):
    c = ALL[name]
    below, w = _run(eng, c)
    want = device_yardstick(name)
    assert np.array_equal(below, want), (list(below), list(want))
    if below.size:
        np.testing.assert_allclose(w, ref_weights(name, below), rtol=1e-9, atol=1e-15)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["M5-sphere-nb25", "M16-uniform-nb12", "w-M8-n65", "w-some-infeasible-M4-n70",
                                  "w-inf-value-M3-n20", "w-front-of-one-M2-n70"])
def test_device_mixture_weights(eng, name):
    """The below mixture's weights: the hypervolume weights of the below rows, then the prior, normalised."""
    c = ALL[name]
    below, w = _run(eng, c)
    raw = np.append(ref_weights(name, below), 1.0)
    np.testing.assert_allclose(eng.get_mixture(0)[0], raw / raw.sum(), rtol=1e-9, atol=1e-18)


@pytest.mark.gpu
def test_sixteen_objectives_accepted_seventeen_rejected(eng):
    from optuna_b200.engine import ParamSpec
    eng.set_space([ParamSpec(kind=0, low=0.0, high=1.0)])
    eng.set_history(np.zeros((4, 1)), np.zeros(4, np.int8), np.zeros((4, 2)))
    eng.set_values(np.random.RandomState(0).uniform(size=(4, 16)), 0)
    with pytest.raises(ValueError, match=r"\[1, 16\]"):
        eng.set_values(np.random.RandomState(0).uniform(size=(4, 17)), 0)


# ------------------------------------------------------------------------------------------------------------------
# Study level: many objectives through optuna's Study
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_obj", [5, 8])
def test_motpe_many_objectives_through_the_study(make_sampler, n_obj):
    from tests.test_plugin_optuna import run_both
    cs = np.linspace(0.1, 0.9, n_obj)
    dirs = ["maximize" if j % 3 == 1 else "minimize" for j in range(n_obj)]

    def obj(t):
        xs = [t.suggest_float(f"x{j}", 0, 1) for j in range(3)]
        return [math.fsum((x - c) ** 2 for x in xs) * (-1 if d == "maximize" else 1) for c, d in zip(cs, dirs)]

    for mv in (False, True):
        run_both(make_sampler, obj, 60, {"directions": dirs}, seed=11, multivariate=mv, n_startup_trials=10)
