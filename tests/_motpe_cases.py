"""Seeded MOTPE cases, each built to reach one path of the device split (`mo_select_complete`, tpe_capi.cu) or of the
hypervolume weights (`build_estimator`, tpe_capi.cu).  A case is loss vectors (every objective minimised), optional
feasibility, and n_below.  `split_path` / `weights_path` restate the host's choice of kernel from the case's
structure, so a case that drifts off its branch fails `test_motpe_paths.py` instead of silently testing nothing.

Structure used to reach the branches:
* points on a simplex (x / sum x) are mutually non-dominated: the tie rank is the whole set and the HSSP subset
  equals n_below;
* shifted copies of a front (front + k * shift) make one rank per copy.
"""
from __future__ import annotations

import itertools
import math
from dataclasses import dataclass

import numpy as np

from oracle import motpe as mo

MAX_SET = 64          # kMoMaxSet: one-CTA shared-memory kernels up to this many points
HV_FRAME_BYTES = 40   # sizeof(HvFrame): two pointers, two doubles, two ints


@dataclass
class Case:
    name: str
    v: np.ndarray                 # [n, M] losses
    nb: int                       # n_below
    path: str                     # split path (split_path) this case is built to reach
    wpath: str | None = None      # weights path (weights_path), when the case is built for one
    feas: np.ndarray | None = None
    tie_order: bool = False       # exact-tie lattice: may depend on the reference's argsort and 3-D sum orders


# ---- host arithmetic (tpe_capi.cu mo_select_complete / build_estimator, tpe_motpe*.cuh sizes) -------------------
def hv_arena_doubles(n: int, M: int) -> int:
    return (n * M + (n + 1) * (n + 2) // 2 * M + (n + 2) * ((2 * n + 7) // 8 + 2) + 4 * n + 64
            + ((n + 2) * HV_FRAME_BYTES + 7) // 8)


def hv_lane_doubles(n: int, M: int) -> int:
    return hv_arena_doubles(n, M) + n * M + 32


def hv_warp_scratch_doubles(n: int, M: int) -> int:
    return 3 * n * M + 2 * n + 16


def nd_warp_arena_bytes(nu: int, subset: int, M: int) -> int:
    """Global arena of k_hssp_contrib_nd: one warp per candidate, a WFG arena per lane."""
    return nu * (hv_warp_scratch_doubles(subset, M) + 32 * hv_lane_doubles(subset, M)) * 8


def mo_smem_stride(n: int, M: int) -> int:
    if M > 3:
        return 0
    stride = (2 * n * M + M + n + 9) | 1
    return stride if MAX_SET * stride * 8 <= 160 * 1024 else 0


def split_structure(v: np.ndarray, nb: int) -> dict:
    """What the host sees when it selects the below part of these COMPLETE trials."""
    n, M = v.shape
    m = min(nb, n)
    out = dict(n=n, M=M, m=m, subset=0, n_tie=0, nu=0, ref_finite=True, n_ranks=0)
    if m in (0, n):
        return out
    ranks = mo.nondomination_rank(v, n_below=m)
    uniq, counts = np.unique(ranks, return_counts=True)
    last = int(np.max(uniq[np.cumsum(counts) <= m], initial=-1))
    cum = int(np.count_nonzero(ranks <= last))
    tie = v[ranks == last + 1]
    out.update(subset=m - cum, n_tie=int(tie.shape[0]), n_ranks=int(uniq.size),
               nu=int(np.unique(tie, axis=0).shape[0]), ref_finite=bool(np.isfinite(mo.reference_point(tie)).all()))
    return out


def split_path(s: dict) -> str:
    M, subset, nu = s["M"], s["subset"], s["nu"]
    if s["m"] in (0, s["n"]):
        return "trivial"
    if subset == 0:
        return "whole-ranks"
    if not s["ref_finite"]:
        return "ref-not-finite"
    if nu <= subset:
        return "fill-dups" if nu < subset else "all-unique"
    if M == 2:
        return "hssp-2d"
    if M == 3:
        return "hssp-contrib3-smem" if subset + 1 <= MAX_SET + 1 else "hssp-contrib3-arena"
    return "hssp-contrib-nd" if nd_warp_arena_bytes(nu, subset, M) <= 8 << 30 else "hssp-contrib"


def weights_structure(v: np.ndarray, feas: np.ndarray | None) -> dict:
    n, M = v.shape
    f = np.ones(n, bool) if feas is None else np.asarray(feas, bool)
    out = dict(n=n, M=M, nf=int(f.sum()), np=0, hv_inf=False)
    if out["nf"] > 1:
        fv = v[f]
        ps = fv[mo.is_pareto_front(fv, assume_unique_lexsorted=False)]
        out["np"] = int(ps.shape[0])
        out["hv_inf"] = math.isinf(mo.hypervolume(ps, mo.reference_point(fv), assume_pareto=True))
    return out


def weights_path(s: dict) -> str:
    n, M = s["n"], s["M"]
    if n <= MAX_SET:
        k = ("k_mo_weights-smem" if mo_smem_stride(n + 1, M) else "k_mo_weights-arena") if M == 2 else \
            ("k_mo_weights3" if M == 3 else "k_mo_weights_nd")
    else:
        k = "k_mow-le3" if M <= 3 else "k_mow-nd"
    if s["nf"] <= 1:
        return k + ":nf<=1"
    if s["hv_inf"]:
        return k + ":hv-inf"
    if s["np"] == 1:
        return k + ":front-of-one"
    return k


# ---- value builders -------------------------------------------------------------------------------------------
def sphere(rs, n: int, M: int, P: int = 4) -> np.ndarray:
    """Squared distances of uniform points to M centres on the diagonal: small fronts."""
    X = rs.uniform(0, 1, (n, P))
    cs = np.linspace(0.1, 0.9, M)
    return ((X[:, None, :] - cs[None, :, None]) ** 2).sum(2)


def simplex(rs, n: int, M: int) -> np.ndarray:
    """Points on the probability simplex: mutually non-dominated."""
    return rs.dirichlet(np.ones(M), n)


def lattice(M: int, L: int, scale: float) -> np.ndarray:
    """{x in N^M : sum x = L} * scale / L in itertools.product order (all on the first front)."""
    return np.array([p for p in itertools.product(range(L + 1), repeat=M) if sum(p) == L], float) * scale / L


def nested(front: np.ndarray, copies: int, shift: float) -> np.ndarray:
    """`copies` shifted copies of a front, interleaved in trial order: one rank per copy."""
    out = np.concatenate([front + k * shift for k in range(copies)])
    return out[np.random.RandomState(copies).permutation(out.shape[0])]


# ---- the cases ------------------------------------------------------------------------------------------------
def split_cases() -> list[Case]:
    out = []
    # objective counts 2..16: sphere values (small fronts) and uniform values (large fronts), n_below = 25 and
    # ceil(0.1 n).  Uniform values at M >= 8 keep n small: the reference's exact weights grow fast with M.
    for M in (2, 3, 4, 5, 6, 8, 12, 16):
        for kind in ("sphere", "uniform"):
            rs = np.random.RandomState(100 * M + (kind == "uniform"))
            n = 300 if kind == "sphere" or M <= 4 else (120 if M <= 6 else 40)
            v = sphere(rs, n, M) if kind == "sphere" else rs.uniform(0, 1, (n, M))
            for nb in (25, math.ceil(0.1 * n)):
                if kind == "uniform" and M >= 8 and nb == 25:
                    nb = 12   # 25 points of a 12- or 16-objective front take the reference minutes to weigh
                s = split_structure(v, nb)
                out.append(Case(f"M{M}-{kind}-nb{nb}", v, nb, split_path(s)))
    # k_hssp_2d with more than 256 unique tie vectors: one CTA loops over them
    rs = np.random.RandomState(1)
    x = np.sort(rs.uniform(0, 1, 1000))
    out.append(Case("2d-1000-front-subset400", np.stack([x, 1 - x ** 0.5], 1)[rs.permutation(1000)], 400, "hssp-2d"))
    # M = 3: subset + 1 <= kMoMaxSet + 1 stages the hypervolume in shared memory, beyond it the global arena
    v = simplex(np.random.RandomState(2), 300, 3)
    for nb, p in ((64, "hssp-contrib3-smem"), (65, "hssp-contrib3-arena"), (66, "hssp-contrib3-arena")):
        out.append(Case(f"3d-300-front-subset{nb}", v, nb, p))
    # M > 3, one warp per candidate (arena nu * warp stride <= 8 GB)
    for M, n, nb in ((4, 80, 30), (5, 70, 25), (8, 50, 15), (16, 40, 10)):
        out.append(Case(f"nd-M{M}-front{n}-subset{nb}", simplex(np.random.RandomState(M), n, M), nb, "hssp-contrib-nd"))
    # M > 3 with the warp arena over 8 GB: one thread per candidate (k_hssp_contrib).  1100 unique tie vectors,
    # subset 140, M = 4: warp stride = 3*140*4 + 2*140 + 16 + 32 * (hv_arena_doubles(140, 4) + 140*4 + 32)
    # = 1976 + 32 * 47 939 = 1 536 024 doubles, times 1100 candidates times 8 bytes = 13.5 GB > 8 GB
    out.append(Case("nd-M4-front1100-subset140-thread", simplex(np.random.RandomState(7), 1100, 4), 140, "hssp-contrib"))
    # reference point not finite: the host takes the first `subset` unique tie vectors in lexicographic order (the
    # reference's np.unique order); trial order differs from it here
    f = simplex(np.random.RandomState(8), 30, 3)
    vi = np.concatenate([f, [[np.inf, -1.0, -1.0], [-1.0, np.inf, -2.0]]])
    out.append(Case("ref-inf-M3", vi, 12, "ref-not-finite"))
    vn = f.copy()
    vn[:, 0] = -np.inf          # -inf in every tie vector: the column's worst is -inf
    out.append(Case("ref-neg-inf-column-M3", vn, 12, "ref-not-finite"))
    vi4 = np.concatenate([simplex(np.random.RandomState(9), 30, 4), [[np.inf, -1.0, -1.0, -1.0]]])
    out.append(Case("ref-inf-M4", vi4, 9, "ref-not-finite"))
    # one -inf entry, finite reference point: that candidate's own box is infinite (incl = inf)
    vm = np.concatenate([f, [[-np.inf, 0.9, 0.9], [0.5, -np.inf, 0.7]]])
    out.append(Case("neg-inf-entry-M3", vm, 10, "hssp-contrib3-smem"))
    vm4 = np.concatenate([simplex(np.random.RandomState(10), 30, 4), [[-np.inf, 0.9, 0.9, 0.9]]])
    out.append(Case("neg-inf-entry-M4", vm4, 10, "hssp-contrib-nd"))
    # duplicates: fewer unique tie vectors than slots (k_mo_fill_dups)
    d = simplex(np.random.RandomState(11), 10, 3)
    vd = d[np.random.RandomState(12).randint(0, 10, 40)]
    vd[np.arange(10) * 4] = d   # every one of the 10 vectors occurs
    out.append(Case("dups-10-unique-40-rows", vd, 25, "fill-dups"))
    out.append(Case("dups-M5", np.repeat(simplex(np.random.RandomState(13), 6, 5), 3, 0), 10, "fill-dups"))
    # -0.0 / +0.0: vectors equal under == but with different bits (the rank hash folds -0.0, k_mo_lexrank
    # compares with <)
    z = lattice(3, 4, 1.0)
    zn = z.copy()
    zn[zn == 0] = -0.0
    vz = np.concatenate([z, zn])[np.random.RandomState(14).permutation(30)]
    out.append(Case("signed-zero-hssp", vz, 9, "hssp-contrib3-smem"))
    out.append(Case("signed-zero-fill-dups", vz, 20, "fill-dups"))
    z2 = lattice(2, 6, 1.0)
    zn2 = z2.copy()
    zn2[zn2 == 0] = -0.0
    out.append(Case("signed-zero-2d", np.concatenate([zn2, z2]), 5, "hssp-2d"))
    # many ranks: dozens of nested fronts, n_below cutting inside a late rank
    for M, shift in ((2, 0.02), (3, 0.03), (4, 0.05)):
        v = nested(simplex(np.random.RandomState(20 + M), 12, M), 40, shift)
        out.append(Case(f"nested-40-ranks-M{M}", v, 12 * 31 + 5, {2: "hssp-2d", 3: "hssp-contrib3-smem"}.get(M, "hssp-contrib-nd")))
    # rank peeling with > 256 alive points at M = 16: the 256-point sample removes almost nothing
    out.append(Case("peel-M16-600", np.random.RandomState(30).uniform(0, 1, (600, 16)), 8, "hssp-contrib-nd"))
    # exact ties: simplex lattices, unshuffled and shuffled, a range of subset sizes
    for M, L in ((3, 4), (3, 6), (4, 4)):
        for scale_name, scale in (("0.1", 0.1), ("1/3", 1 / 3), ("1", 1.0)):
            base = lattice(M, L, scale)
            for order in ("sorted", "shuffle1", "shuffle2"):
                v = base if order == "sorted" else base[np.random.RandomState(int(order[-1])).permutation(len(base))]
                for k in (3, 5, 7, 9, 11):
                    p = "hssp-contrib3-smem" if M == 3 else "hssp-contrib-nd"
                    out.append(Case(f"lattice-M{M}-L{L}-s{scale_name}-{order}-k{k}", v, k, p, tie_order=True))
    return out


def weights_cases() -> list[Case]:
    """Cases for the weights kernels: the split is the whole input (n_below = n), so the below set is every row."""
    out = []
    for M in (2, 3, 4, 5, 8):
        for nb in (60, 61, 64, 65):
            v = sphere(np.random.RandomState(40 + M), nb, M)
            s = weights_structure(v, None)
            out.append(Case(f"w-M{M}-n{nb}", v, nb, "trivial", weights_path(s)))
    # every row on the front (up to 64 points at M = 2 and 3; at M = 4 the WFG of a 64-point front is slow)
    for M, nb in ((2, 60), (2, 64), (3, 61), (3, 64), (2, 65), (3, 65), (4, 30), (5, 20)):
        v = simplex(np.random.RandomState(50 + M), nb, M)
        out.append(Case(f"w-front-M{M}-n{nb}", v, nb, "trivial", weights_path(weights_structure(v, None))))
    # edge cases: at most one feasible row, an infinite value (hv = inf: every weight 1), a front of one point
    for M in (2, 3, 4):
        for n in (20, 70):
            rs = np.random.RandomState(60 + M + n)
            v = sphere(rs, n, M)
            out.append(Case(f"w-none-feasible-M{M}-n{n}", v, n, "trivial", None, np.zeros(n, bool)))
            one = np.zeros(n, bool)
            one[n // 2] = True
            out.append(Case(f"w-one-feasible-M{M}-n{n}", v, n, "trivial", None, one))
            vi = v.copy()
            vi[3, 1] = np.inf
            out.append(Case(f"w-inf-value-M{M}-n{n}", vi, n, "trivial"))
            v1 = v.copy()
            v1[5] = -1.0          # dominates every other row
            out.append(Case(f"w-front-of-one-M{M}-n{n}", v1, n, "trivial"))
            feas = rs.uniform(size=n) < 0.7
            out.append(Case(f"w-some-infeasible-M{M}-n{n}", v, n, "trivial", None, feas))
    for c in out:
        if c.wpath is None:
            c.wpath = weights_path(weights_structure(c.v, c.feas))
    return out
