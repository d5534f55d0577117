"""GPSampler's acquisition search: the fused device acquisition with lock-step local searches against the per-GP
path (optuna's ``optimize_acqf_mixed`` over one device query per GP per evaluation) and optuna's own GPSampler.

Each case replays asks on a fixed history of random trials, so every arm sees the same study.  Per ask it reports the
time of the whole ask, of the acquisition search (``_optimize_acqf``) and of the rest (the fits), and the device
round trips of the search: ``acqf_eval`` calls on the fused path, ``gp_query`` plus ``ehvi`` calls on the per-GP
path.  The objectives are rugged (sums of sines of random projections), so the roulette keeps all ten local searches.

    python tools/bench_gp_search.py [--trials 300] [--asks 3] [--out results/bench_gp_search.json]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _objective(P: int, seed: int):
    rs = np.random.RandomState(seed)
    W = rs.normal(size=(P, 4)) * 4.0

    def f(x: np.ndarray) -> float:
        return float(np.sin(x @ W).sum() + 0.1 * (x ** 2).sum())
    return f


def _case(name: str):
    import optuna
    D = optuna.distributions
    if name in ("rugged8", "rugged32"):
        P = 8 if name == "rugged8" else 32
        return {f"x{j}": D.FloatDistribution(-3, 3) for j in range(P)}, 1, False
    if name == "mixed":
        d = {f"x{j}": D.FloatDistribution(-3, 3) for j in range(4)}
        d.update({"i": D.IntDistribution(-6, 6), "j": D.IntDistribution(0, 60), "c": D.CategoricalDistribution(
            ["a", "b", "c", "d"])})
        return d, 1, False
    if name == "two_obj_constrained":
        return {f"x{j}": D.FloatDistribution(-3, 3) for j in range(8)}, 2, True
    raise ValueError(name)


def _history(dists, n_obj, constrained, n, seed):
    import optuna
    D = optuna.distributions
    rs = np.random.RandomState(seed)
    fs = [_objective(len(dists), seed + k) for k in range(n_obj + 1)]
    out = []
    for _ in range(n):
        params, vec = {}, []
        for name, d in dists.items():
            if isinstance(d, D.CategoricalDistribution):
                params[name] = d.choices[rs.randint(len(d.choices))]
                vec.append(float(d.choices.index(params[name])))
            elif isinstance(d, D.IntDistribution):
                params[name] = int(rs.randint(d.low, d.high + 1))
                vec.append(params[name] / 10.0)
            else:
                params[name] = float(rs.uniform(d.low, d.high))
                vec.append(params[name])
        x = np.array(vec)
        vals = [fs[k](x) for k in range(n_obj)]
        attrs = {"constraints": [fs[-1](x)]} if constrained else {}
        out.append(optuna.trial.create_trial(params=params, distributions=dists, system_attrs=attrs,
                                             **({"value": vals[0]} if n_obj == 1 else {"values": vals})))
    return out


def _constraints_func(trial):   # the asked trials are failed, for which optuna evaluates no constraints
    raise AssertionError


def _run(arm: str, dists, n_obj, constrained, history, asks: int) -> dict:
    import optuna

    from optuna_b200 import TPEEngine, gp_sampler
    cf = _constraints_func if constrained else None
    counts = {"gp_query": 0, "ehvi": 0, "acqf_eval": 0}
    originals = {k: getattr(TPEEngine, k) for k in counts}

    def counted(name):
        fn = originals[name]

        def wrap(self, *a, **kw):
            counts[name] += 1
            return fn(self, *a, **kw)
        return wrap
    for k in counts:
        setattr(TPEEngine, k, counted(k))
    saved_gate = gp_sampler._answers_acqf
    if arm == "per_gp":
        gp_sampler._answers_acqf = lambda cls: False
    sampler = (optuna.samplers.GPSampler(seed=0, constraints_func=cf) if arm == "optuna"
               else gp_sampler.GPSampler(seed=0, constraints_func=cf))
    search = [0.0]
    opt = sampler._optimize_acqf

    def timed(acqf, best):
        t0 = time.perf_counter()
        try:
            return opt(acqf, best)
        finally:
            search[0] += time.perf_counter() - t0
    sampler._optimize_acqf = timed
    study = optuna.create_study(directions=["minimize"] * n_obj, sampler=sampler)
    study.add_trials(history)
    rows = []
    try:
        for k in range(asks + 1):   # the first ask warms up
            for c in counts:
                counts[c] = 0
            search[0] = 0.0
            t0 = time.perf_counter()
            t = study.ask(dists)
            total = time.perf_counter() - t0
            study.tell(t, state=optuna.trial.TrialState.FAIL)
            if k:
                trips = counts["acqf_eval"] if arm == "fused" else counts["gp_query"] + counts["ehvi"]
                rows.append((total, search[0], trips))
    finally:
        if arm != "optuna":
            sampler.close()
        gp_sampler._answers_acqf = saved_gate
        for k, fn in originals.items():
            setattr(TPEEngine, k, fn)
    a = np.array(rows)
    return {"ask_s": float(np.median(a[:, 0])), "search_s": float(np.median(a[:, 1])),
            "fit_s": float(np.median(a[:, 0] - a[:, 1])), "round_trips": int(np.median(a[:, 2]))}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--trials", type=int, default=300)
    ap.add_argument("--asks", type=int, default=3)
    ap.add_argument("--cases", default="rugged8,rugged32,mixed,two_obj_constrained")
    ap.add_argument("--arms", default="fused,per_gp,optuna")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from oracle import ref
    ref.enable()
    import optuna
    import torch
    optuna.logging.set_verbosity(optuna.logging.ERROR)
    gpu = torch.cuda.get_device_name(0) if torch.cuda.is_available() else "none"
    results = []
    for name in args.cases.split(","):
        dists, n_obj, constrained = _case(name)
        history = _history(dists, n_obj, constrained, args.trials, seed=1)
        for arm in args.arms.split(","):
            r = _run(arm, dists, n_obj, constrained, history, args.asks)
            r.update(case=name, arm=arm, trials=args.trials, gpu=gpu)
            results.append(r)
            print(json.dumps(r), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(results, fh, indent=1)


if __name__ == "__main__":
    main()
