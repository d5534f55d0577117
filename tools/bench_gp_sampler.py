"""Time one ``sample_relative`` of ``optuna_b200.GPSampler`` against the reference's ``optuna.samplers.GPSampler``.

Each case is a seeded study built with ``add_trials``: n complete trials over P float parameters in [0, 1] with a
weighted sum of squares as the objective (a second objective, its negated sum of absolute offsets, for the two-objective
case; two constraints for the constrained case).  A fresh sampler with the same seed asks once, so that both fit from
the default kernel parameters.  The drop-in asks once to warm up (CUDA context, module load) and then twice timed;
the reference asks once.  Each row reports:
- the wall time of the ask, of the fits and of the acquisition search (``_optimize_acqf``) apart;
- the number of ``gp_query`` calls in the drop-in's search and their mean wall time (each ends in a stream synchronise);
- the largest difference between the two suggestions.
Also printed: whether ``greenlet`` is importable (it sets the L-BFGS batch size of the acquisition search in both
samplers) and the card's name and power limit.  Prints one JSON line.

    python tools/bench_gp_sampler.py [--cases 300x8,1000x8,3000x8,1000x32,c1000x8,mo1000x8] [--no-ref]
"""
from __future__ import annotations

import argparse
import importlib.util
import json
import os
import sys
import time
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.bench_hv_history import _gpu_info  # noqa: E402


def _case(spec: str):
    kind = "mo" if spec.startswith("mo") else "c" if spec.startswith("c") else "so"
    n, P = (int(v) for v in spec.lstrip("moc").split("x"))
    return kind, n, P


def _constraints(t):
    return [t.params["x0"] - 0.6, 0.2 - t.params["x1"]]


def _study_trials(kind, n, P, seed=0):
    import optuna
    dists = {f"x{j}": optuna.distributions.FloatDistribution(0.0, 1.0) for j in range(P)}
    rs = np.random.RandomState(seed)
    X = rs.uniform(0, 1, (n, P))
    w = np.arange(1, P + 1, dtype=np.float64)
    v0 = ((X - 0.3) ** 2 * w).sum(1)
    v1 = -np.abs(X - 0.7).sum(1)
    trials = []
    for x, a, b in zip(X, v0, v1):
        params = {f"x{j}": float(x[j]) for j in range(P)}
        attrs = {"constraints": [params["x0"] - 0.6, 0.2 - params["x1"]]} if kind == "c" else {}
        vals = {"values": [float(a), float(b)]} if kind == "mo" else {"value": float(a)}
        trials.append(optuna.trial.create_trial(params=params, distributions=dists, system_attrs=attrs, **vals))
    return dists, trials


def _ask(sampler_cls, kind, dists, trials, stats):
    """One ask on a fresh sampler over the study: (params, wall seconds); fit / search seconds added to stats."""
    import optuna
    sampler = sampler_cls(seed=0, constraints_func=_constraints if kind == "c" else None)
    if hasattr(sampler, "_fit_gp"):   # the drop-in; the reference's fits are timed by _ref_fit_timer
        real_fit = sampler._fit_gp

        def fit(*a, **kw):
            t0 = time.perf_counter()
            try:
                return real_fit(*a, **kw)
            finally:
                stats["fit"] += time.perf_counter() - t0
        sampler._fit_gp = fit
    real_opt = sampler._optimize_acqf

    def opt(*a, **kw):
        t0 = time.perf_counter()
        try:
            return real_opt(*a, **kw)
        finally:
            stats["search"] += time.perf_counter() - t0
    sampler._optimize_acqf = opt
    study = optuna.create_study(directions=["minimize"] * (2 if kind == "mo" else 1), sampler=sampler)
    study.add_trials(trials)
    t0 = time.perf_counter()
    t = study.ask(dists)
    dt = time.perf_counter() - t0
    if hasattr(sampler, "close"):
        sampler.close()
    return t.params, dt


def _ref_fit_timer(stats):
    """The reference's gp.fit_kernel_params with its wall time added to stats['fit']."""
    from optuna.samplers._gp import sampler as ref_sampler
    gp = ref_sampler.gp   # the sampler's lazy module: its first attribute read loads it, then it holds its own names
    real = gp.fit_kernel_params

    def fit(*a, **kw):
        t0 = time.perf_counter()
        try:
            return real(*a, **kw)
        finally:
            stats["fit"] += time.perf_counter() - t0
    gp.fit_kernel_params = fit
    return lambda: setattr(gp, "fit_kernel_params", real)


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--cases", default="300x8,1000x8,3000x8,1000x32,c1000x8,mo1000x8")
    ap.add_argument("--no-ref", action="store_true")
    args = ap.parse_args()

    from oracle import ref
    ref.enable()
    import optuna
    import optuna_b200
    from optuna_b200 import TPEEngine
    warnings.simplefilter("ignore")
    optuna.logging.set_verbosity(optuna.logging.ERROR)

    queries: list = []
    real_query = TPEEngine.gp_query

    def counted_query(self, Xq, grad=False):
        t0 = time.perf_counter()
        try:
            return real_query(self, Xq, grad)
        finally:
            queries.append(time.perf_counter() - t0)
    TPEEngine.gp_query = counted_query

    rows = []
    for spec in args.cases.split(","):
        kind, n, P = _case(spec)
        dists, trials = _study_trials(kind, n, P)
        _ask(optuna_b200.GPSampler, kind, dists, trials, {"fit": 0.0, "search": 0.0})   # warm-up
        row = {"case": spec, "n": n, "P": P, "kind": kind, "ours": []}
        for _ in range(2):
            stats = {"fit": 0.0, "search": 0.0}
            queries.clear()
            got, dt = _ask(optuna_b200.GPSampler, kind, dists, trials, stats)
            row["ours"].append({"total_s": dt, "fit_s": stats["fit"], "search_s": stats["search"],
                                "n_query": len(queries), "query_mean_ms": 1e3 * float(np.mean(queries))})
        if not args.no_ref:
            stats = {"fit": 0.0, "search": 0.0}
            undo = _ref_fit_timer(stats)
            try:
                want, dt = _ask(optuna.samplers.GPSampler, kind, dists, trials, stats)
            finally:
                undo()
            row["ref"] = {"total_s": dt, "fit_s": stats["fit"], "search_s": stats["search"]}
            row["max_param_diff"] = max(abs(got[k] - want[k]) for k in want)
            row["speedup"] = dt / min(r["total_s"] for r in row["ours"])
        rows.append(row)
        print(json.dumps(row), file=sys.stderr, flush=True)
    print(json.dumps({"gpu": _gpu_info(), "greenlet": importlib.util.find_spec("greenlet") is not None,
                      "rows": rows}))


if __name__ == "__main__":
    main()
