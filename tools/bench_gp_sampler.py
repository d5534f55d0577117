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

A case ``moK:nxP`` is a seeded DTLZ2 study with K objectives (``mo3:1000x8``, ``mo4:300x8``, ``mo4:1000x8``).  For it
the row reports, instead of a reference ask, the acquisition search on the drop-in's fitted GPs in two arms:
- the number of boxes B and the front size, and the wall time of the ask's `LogEHVI` build (the box decomposition on
  the device, the Pareto filter and the Sobol samples);
- the parent path (optuna's host ``LogEHVI`` over the device GPs) and the device log-EHVI, each running
  ``_optimize_acqf`` from the same random state, alternated twice, with the largest difference of their suggestions;
- the preliminary 2 048-point log-EHVI evaluation: its wall time in each arm, and the device kernels' time from
  ``torch.profiler`` in a separate call, with the fp64 rate from Q S B 4M operations and its ratio to
  ``tpe_probe_fp64_tflops``.
The parent arm runs only where its estimated host memory, 3 x 8 Q S B M bytes, fits in half the available memory;
otherwise the row says it cannot run and gives the estimate.

    python tools/bench_gp_sampler.py [--cases 300x8,1000x8,3000x8,1000x32,c1000x8,mo1000x8,mo3:1000x8,mo4:300x8,mo4:1000x8]
                                     [--no-ref]
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
    if ":" in spec:   # moK:nxP, a K-objective DTLZ2 study
        head, size = spec.split(":")
        n, P = (int(v) for v in size.split("x"))
        return f"dtlz{int(head[2:])}", n, P
    kind = "mo" if spec.startswith("mo") else "c" if spec.startswith("c") else "so"
    n, P = (int(v) for v in spec.lstrip("moc").split("x"))
    return kind, n, P


def _dtlz2(X, M):
    """DTLZ2 (Deb et al., 2005): M objectives to minimise over X in [0, 1]^P."""
    g = ((X[:, M - 1:] - 0.5) ** 2).sum(1)
    out = np.empty((X.shape[0], M))
    for m in range(M):
        f = 1.0 + g
        for i in range(M - 1 - m):
            f = f * np.cos(0.5 * np.pi * X[:, i])
        if m > 0:
            f = f * np.sin(0.5 * np.pi * X[:, M - 1 - m])
        out[:, m] = f
    return out


def _dtlz_trials(M, n, P, seed=0):
    import optuna
    dists = {f"x{j}": optuna.distributions.FloatDistribution(0.0, 1.0) for j in range(P)}
    X = np.random.RandomState(seed).uniform(0, 1, (n, P))
    F = _dtlz2(X, M)
    return dists, [optuna.trial.create_trial(params={f"x{j}": float(x[j]) for j in range(P)}, distributions=dists,
                                             values=[float(v) for v in f]) for x, f in zip(X, F)]


def _mem_available() -> float:
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return float(line.split()[1]) * 1024.0
    return 0.0


def _acq_arms(M, n, P):
    """One ask of the drop-in on a DTLZ2 study, with the acquisition search run afterwards in both arms on its GPs."""
    import optuna
    import optuna_b200
    dists, trials = _dtlz_trials(M, n, P)
    sampler = optuna_b200.GPSampler(seed=0)
    seen = {}
    real_dev = sampler._device_ehvi

    def device_ehvi(host):
        t0 = time.perf_counter()
        seen["decomp_s"] = t0 - seen["build_t0"]
        out = real_dev(host)
        seen["upload_s"] = time.perf_counter() - t0
        seen["host"], seen["dev"] = host, out
        return out
    sampler._device_ehvi = device_ehvi
    real_opt = sampler._optimize_acqf

    def opt(acqf, best_params):
        seen["best"], seen["rng"] = best_params, sampler._rng.rng.get_state()
        return real_opt(acqf, best_params)
    sampler._optimize_acqf = opt
    real_log_ehvi = sampler._log_ehvi

    def log_ehvi(*a, **kw):
        # the LogEHVI's build up to the EHVI upload: its box decomposition (the device's), Pareto filter and samples
        seen["build_t0"] = time.perf_counter()
        return real_log_ehvi(*a, **kw)
    sampler._log_ehvi = log_ehvi
    study = optuna.create_study(directions=["minimize"] * M, sampler=sampler)
    study.add_trials(trials)
    t0 = time.perf_counter()
    study.ask(dists)
    ask_s = time.perf_counter() - t0
    host, dev = seen["host"], seen["dev"]
    B = int(host._non_dominated_box_lower_bounds.shape[0])
    S = int(host._fixed_samples.shape[0])
    Q = 2048
    loss = -np.array([t.values for t in trials])
    from optuna.study._multi_objective import _is_pareto_front
    front = int(_is_pareto_front(-loss, assume_unique_lexsorted=False).sum())
    need = 3.0 * 8 * Q * S * B * M
    host_ok = need < 0.5 * _mem_available()
    row = {"case": f"mo{M}:{n}x{P}", "M": M, "n": n, "P": P, "front": front, "boxes": B,
           "box_decomposition_s": seen["decomp_s"], "ehvi_upload_s": seen["upload_s"], "ask_s": ask_s,
           "parent_host_bytes_est": need}
    xs = host.search_space.sample_normalized_params(Q, rng=np.random.RandomState(0))
    arms = {"device": dev} | ({"parent": host} if host_ok else {})
    row["search_s"] = {k: [] for k in arms}
    row["prelim_s"] = {k: [] for k in arms}
    suggestion = {}
    for _ in range(2):
        for name, a in arms.items():
            t0 = time.perf_counter()
            a.eval_acqf_no_grad(xs)
            row["prelim_s"][name].append(time.perf_counter() - t0)
            sampler._rng.rng.set_state(seen["rng"])
            t0 = time.perf_counter()
            suggestion[name] = real_opt(a, seen["best"])
            row["search_s"][name].append(time.perf_counter() - t0)
    if not host_ok:
        row["parent"] = f"cannot run: needs about {need / 1e9:.1f} GB of host memory"
    else:
        row["max_suggestion_diff"] = float(np.max(np.abs(suggestion["device"] - suggestion["parent"])))
        row["search_speedup"] = min(row["search_s"]["parent"]) / min(row["search_s"]["device"])
    # the device kernels of one preliminary evaluation are timed apart, by main, in one profiler session
    kernel_case = (host._non_dominated_box_lower_bounds.numpy(), host._non_dominated_box_intervals.numpy(),
                   host._fixed_samples.numpy())
    sampler.close()
    return row, kernel_case


def _kernel_times(cases, Q=2048):
    """Device time (ms) of the kernels of one values-only ``ehvi`` call of Q rows per case, from one
    ``torch.profiler`` session (a call of Q = 2 048 rows launches one chunk and one finish kernel)."""
    import torch
    from optuna_b200 import TPEEngine
    engines = []
    for lb, iv, Z in cases:
        eng = TPEEngine(0)
        eng.ehvi_set(lb, iv, Z)
        M = lb.shape[1]
        args = (np.random.RandomState(1).normal(0, 1, (Q, M)), np.random.RandomState(2).uniform(0.1, 1.0, (Q, M)))
        eng.ehvi(*args)   # warm-up
        engines.append((eng, args))
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for eng, args in engines:
            eng.ehvi(*args)
    for eng, _ in engines:
        eng.close()
    kernels = sorted((e for e in prof.events() if "k_ehvi" in e.name and e.device_time_total > 0),
                     key=lambda e: e.time_range.start)
    assert len(kernels) == 2 * len(cases), [e.name for e in kernels]
    return [(kernels[2 * i].device_time_total + kernels[2 * i + 1].device_time_total) / 1e3 for i in range(len(cases))]


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
    ap.add_argument("--cases", default="300x8,1000x8,3000x8,1000x32,c1000x8,mo1000x8,mo3:1000x8,mo4:300x8,mo4:1000x8")
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
    tflops = None
    kernel_cases = []
    for spec in args.cases.split(","):
        kind, n, P = _case(spec)
        if kind.startswith("dtlz"):
            if tflops is None:
                probe = TPEEngine(0)
                tflops = probe.probe_fp64_tflops()
                probe.close()
            row, kc = _acq_arms(int(kind[4:]), n, P)
            row["probe_fp64_tflops"] = tflops
            rows.append(row)
            kernel_cases.append((row, kc))
            print(json.dumps(row), file=sys.stderr, flush=True)
            continue
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
    if kernel_cases:
        for (row, kc), ms in zip(kernel_cases, _kernel_times([kc for _, kc in kernel_cases])):
            lb, _, Z = kc
            ops = 2048.0 * Z.shape[0] * lb.shape[0] * 4 * lb.shape[1]
            row["prelim_kernel_ms"] = ms
            row["fp64_tflops"] = ops / (ms * 1e-3) / 1e12
            row["fp64_of_probe"] = row["fp64_tflops"] / tflops
            print(json.dumps({k: row[k] for k in ("case", "prelim_kernel_ms", "fp64_tflops", "fp64_of_probe")}),
                  file=sys.stderr, flush=True)
    print(json.dumps({"gpu": _gpu_info(), "greenlet": importlib.util.find_spec("greenlet") is not None,
                      "rows": rows}))


if __name__ == "__main__":
    main()
