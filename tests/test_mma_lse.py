"""The log-sum-exp of the tensor-core grid kernel (k_logpdf_mma, LseRef) on data that forces its rare paths: the
reference R moving (a candidate's largest terms lie far above the terms of the first tiles it sees), and the parked
near terms of one candidate filling its buffer again and again while the other candidates of its warp have none.
Both at P = 16 / 32 / 64, through the big (C = 4096) and the small (C = 24) path, against the oracle at 1e-12."""
from __future__ import annotations

import numpy as np
import pytest

from oracle import tpe_oracle as orc

pytestmark = pytest.mark.gpu

N_ABOVE = 4000


@pytest.fixture(scope="module")
def eng():
    from optuna_b200 import TPEEngine
    e = TPEEngine(0)
    yield e
    e.close()


def _above_logpdf(eng, X, pts, rs):
    """log g of `pts` under the above mixture of X (equal weights), from the engine and from the oracle."""
    from optuna_b200.engine import ParamSpec
    n, P = X.shape
    specs = [ParamSpec(kind=0, low=0.0, high=1.0) for _ in range(P)]
    params = [orc.Param("float", 0.0, 1.0) for _ in range(P)]
    # 25 best trials far from everything take the below slots; X is the above set, in trial order
    Xall = np.concatenate([rs.uniform(0.0, 0.02, (25, P)), X])
    key = np.stack([np.concatenate([np.full(25, -1.0), np.ones(n)]), np.zeros(n + 25)], 1)
    eng.set_space(specs)
    eng.set_history(Xall, np.zeros(n + 25, np.int8), key)
    eng.prepare(list(range(P)), n_below=25, n_candidates=pts.shape[0], multivariate=True)
    eng.build(None, np.ones(n))
    got = eng.logpdf(1, pts)
    assert eng.last_logpdf_kernel().startswith("k_logpdf_mma"), eng.last_logpdf_kernel()
    mix = orc.build_mixture(X, params, orc.Config(multivariate=True, weights=lambda k: np.ones(k)))
    return got, orc.mixture_log_pdf_chunked(mix, pts, 64)


def _close(got, want):
    assert np.isfinite(want).all()
    err = np.abs(got - want)
    assert err.max() <= 1e-12, f"max err {err.max()} at {np.argsort(err)[-5:].tolist()}"


@pytest.mark.parametrize("C", [4096, 24])
@pytest.mark.parametrize("P", [16, 32, 64])
def test_reference_moves_when_later_terms_lie_far_above_the_first(eng, P, C):
    """Kernels on spheres around x0 whose radius shrinks along the trial order (= the kernel order of the table): for a
    candidate near x0 the first tiles of every k-split hold terms 100-200 nats below the last ones, so each lane's
    reference, set from its first terms, has to move up several times."""
    rs = np.random.RandomState(P)
    x0 = np.full(P, 0.5)
    r = np.linspace(0.45, 0.0, N_ABOVE) * np.sqrt(P)
    X = x0 + rs.choice([-1.0, 1.0], size=(N_ABOVE, P)) * (r / np.sqrt(P))[:, None]
    pts = x0 + 0.01 * rs.standard_normal((C, P))
    pts[::7] = rs.uniform(0.0, 1.0, (len(pts[::7]), P))   # and some candidates anywhere
    got, want = _above_logpdf(eng, X, pts, rs)
    _close(got, want)


@pytest.mark.parametrize("C", [4096, 24])
@pytest.mark.parametrize("P", [16, 32, 64])
def test_near_terms_concentrated_in_one_candidate_of_a_warp(eng, P, C):
    """All kernels in a tight cluster: for the candidates placed on it every term is near (parked and folded
    exactly, the buffer fills every other step), for the other candidates of the same warp (16 candidates in the big
    path, 8 in the small one) every term but the prior's is dropped."""
    rs = np.random.RandomState(100 + P)
    x1 = rs.uniform(0.3, 0.7, P)
    X = np.clip(x1 + 1e-3 * rs.standard_normal((N_ABOVE, P)), 0.0, 1.0)
    pts = np.where(x1 < 0.5, 0.97, 0.03) + 0.01 * rs.uniform(-1.0, 1.0, (C, P))   # the far corner
    on = np.arange(C) % 16 == 5
    pts[on] = x1 + 1e-3 * rs.standard_normal((int(on.sum()), P))
    got, want = _above_logpdf(eng, X, pts, rs)
    _close(got, want)
