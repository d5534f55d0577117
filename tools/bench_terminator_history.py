"""Times ``optuna_b200.terminator_improvement_history`` against optuna's ``_get_improvement_info`` with the drop-in
``optuna_b200.RegretBoundEvaluator`` (one fit per prefix) on synthetic studies of T trials x P float parameters.

    python tools/bench_terminator_history.py 100x8 300x8 1000x8 1000x32 [--reference 300]

Per size: wall time of both arms, the batched arm's rounds, device time per round (the loss launch and its copies)
and host time per round (the rest: priors, L-BFGS-B steps, thread hand-offs), and the largest relative difference.
``--reference N`` also runs optuna's own RegretBoundEvaluator up to N trials.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
import warnings

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("sizes", nargs="+")
    ap.add_argument("--reference", type=int, default=0)
    args = ap.parse_args()
    from oracle import ref
    ref.enable()
    import numpy as np
    import optuna
    from optuna.visualization._terminator_improvement import _get_improvement_info

    import optuna_b200
    from optuna_b200 import terminator
    warnings.simplefilter("ignore")
    optuna.logging.set_verbosity(optuna.logging.ERROR)
    for size in args.sizes:
        T, P = (int(v) for v in size.split("x"))
        rs = np.random.RandomState(0)
        study = optuna.create_study()
        dists = {f"x{j}": optuna.distributions.FloatDistribution(0.0, 1.0) for j in range(P)}
        X = rs.uniform(0, 1, (T, P))
        v = ((X - 0.3) ** 2 * np.arange(1, P + 1)).sum(1) + 0.05 * rs.randn(T)
        study.add_trials([optuna.trial.create_trial(params={f"x{j}": X[i, j] for j in range(P)}, distributions=dists,
                                                    value=float(v[i])) for i in range(T)])
        stats: dict = {}
        t0 = time.perf_counter()
        _, got = terminator._batched_improvements(optuna_b200.RegretBoundEvaluator(seed=0), study, stats)
        t_batch = time.perf_counter() - t0
        t0 = time.perf_counter()
        loop = _get_improvement_info(study, improvement_evaluator=optuna_b200.RegretBoundEvaluator(seed=0))
        t_loop = time.perf_counter() - t0
        got = np.array(got)
        rel = lambda w: float(np.max(np.abs(got - w) / np.maximum(np.abs(w), 1e-9)))
        row = {"size": size, "batched_s": round(t_batch, 3), "per_prefix_s": round(t_loop, 3),
               "rounds": stats["rounds"], "device_ms_per_round": round(1e3 * stats["device_seconds"] / stats["rounds"], 3),
               "host_ms_per_round": round(1e3 * (stats["wall_seconds"] - stats["device_seconds"]) / stats["rounds"], 3),
               "max_rel_vs_per_prefix": rel(np.array(loop.improvements))}
        if T <= args.reference:
            t0 = time.perf_counter()
            want = _get_improvement_info(study, improvement_evaluator=optuna.terminator.RegretBoundEvaluator(seed=0))
            row["reference_s"] = round(time.perf_counter() - t0, 3)
            row["max_rel_vs_reference"] = rel(np.array(want.improvements))
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
