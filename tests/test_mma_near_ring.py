"""The near-term ring of the tensor-core grid kernel (k_logpdf_mma, LseRef): near terms parked in shared memory by a
predicated store and flushed after one warp vote, on data that drives the ring to its limits -- every term near (the
ring fills and flushes every few steps), one candidate of a warp near-heavy while the others have no near term, and the
reference R moving by more than kRefMove (48 nats) while terms are parked.  K is never a multiple of the tile and the
kernel axis is split over several CTAs.  P = 16 / 32 / 64 through the big (C = 4096) and the small (C = 24) path,
against the oracle at 1e-12 with the same argmax."""
from __future__ import annotations

import numpy as np
import pytest

from tests.test_mma_lse import _above_logpdf, _close

pytestmark = pytest.mark.gpu

PS = [16, 32, 64]
CS = [4096, 24]


@pytest.fixture(scope="module")
def eng():
    from optuna_b200 import TPEEngine
    e = TPEEngine(0)
    yield e
    e.close()


def _check(eng, X, pts, rs):
    got, want = _above_logpdf(eng, X, pts, rs)
    _close(got, want)
    assert int(np.argmax(got)) == int(np.argmax(want))


@pytest.mark.parametrize("C", CS)
@pytest.mark.parametrize("P", PS)
def test_every_term_near(eng, P, C):
    """Thousands of identical observations: every kernel of the above mixture but the prior's gives a candidate the
    same term, so every term is near and every lane's ring fills and is flushed again and again."""
    n = 4000
    rs = np.random.RandomState(200 + P)
    x1 = rs.uniform(0.3, 0.7, P)
    X = np.tile(x1, (n, 1))
    pts = rs.uniform(0.0, 1.0, (C, P))
    pts[::3] = x1 + 0.05 * rs.standard_normal((len(pts[::3]), P))
    _check(eng, X, pts, rs)


@pytest.mark.parametrize("C", CS)
@pytest.mark.parametrize("P", PS)
def test_one_lane_of_a_warp_near_heavy(eng, P, C):
    """A tight cluster of kernels and one candidate in 32 placed on it: that candidate's lanes park every term while the
    other lanes of the warp park none, so the warp flushes for one lane's ring alone."""
    rs = np.random.RandomState(300 + P)
    x1 = rs.uniform(0.3, 0.7, P)
    X = np.clip(x1 + 1e-3 * rs.standard_normal((4003, P)), 0.0, 1.0)
    pts = np.where(x1 < 0.5, 0.97, 0.03) + 0.01 * rs.uniform(-1.0, 1.0, (C, P))
    on = np.arange(C) % 32 == 9
    pts[on] = x1 + 1e-3 * rs.standard_normal((int(on.sum()), P))
    _check(eng, X, pts, rs)


@pytest.mark.parametrize("C", CS)
@pytest.mark.parametrize("P", PS)
def test_reference_moves_while_terms_are_parked(eng, P, C):
    """Kernels in a staircase along the kernel order: runs of 12 kernels whose terms for a candidate at x0 lie about
    110, 55 and 0 nats below the top, repeated.  A lane starting cold parks terms of a lower step and, before its ring
    is flushed, terms of the next one: the flush moves base and R by more than 48 nats above terms already parked."""
    rs = np.random.RandomState(400 + P)
    x0 = np.full(P, 0.5)
    sigma = 0.2 * 4002 ** (-1.0 / (P + 4))                  # multivariate bandwidth of the 4002-kernel above mixture
    d = sigma * np.sqrt(2.0 * np.array([110.0, 55.0, 0.0]) / P)   # per-coordinate offset of each step
    level = (np.arange(4001) // 12) % 3
    X = x0 + rs.choice([-1.0, 1.0], size=(4001, P)) * d[level][:, None]
    pts = x0 + 0.002 * rs.standard_normal((C, P))
    pts[::5] = rs.uniform(0.0, 1.0, (len(pts[::5]), P))
    _check(eng, X, pts, rs)
