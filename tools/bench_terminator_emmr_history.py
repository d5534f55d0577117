"""Times ``optuna_b200.terminator_improvement_history`` with ``optuna_b200.EMMREvaluator`` (both GPs of every prefix
fitted in lock step) against optuna's ``_get_improvement_info`` with the same drop-in evaluator (two fits per prefix,
one prefix after another), on the synthetic float studies of T trials x P parameters of tests/test_terminator_history
(seed 1, as the GPU tests of tests/test_terminator_emmr_history use them).

    python tools/bench_terminator_emmr_history.py 100x8 300x8 300x8d 1000x8 1000x32 [--reference 100]

A trailing ``d`` runs with ``deterministic_objective=True``.  Per size: wall time of both arms, the batched arm's
rounds, device time per round (the loss launch and its copies) and host time per round (the rest: pre-pass, priors,
L-BFGS-B steps, thread hand-offs, the bounds and moments launches), and the largest relative difference.
``--reference N`` also runs optuna's own EMMREvaluator up to N trials.  The first line names the card and its power
limit.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
import warnings

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _card() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, sm = (v.strip() for v in out.split(","))
        return {"card": name, "power_limit": power, "max_sm_clock": sm}
    except Exception as e:   # the numbers then carry no card
        return {"card": f"unknown ({e})"}


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
    from tests.test_terminator_history import _synthetic
    warnings.simplefilter("ignore")
    optuna.logging.set_verbosity(optuna.logging.ERROR)
    print(json.dumps(_card()), flush=True)
    for size in args.sizes:
        det = size.endswith("d")
        T, P = (int(v) for v in size.rstrip("d").split("x"))
        study = _synthetic(T, P, seed=1)   # the studies of the GPU tests against the per-prefix loop
        stats: dict = {}
        t0 = time.perf_counter()
        _, got, _ = terminator._batched_emmr(optuna_b200.EMMREvaluator(seed=0, deterministic_objective=det), study,
                                             stats=stats)
        t_batch = time.perf_counter() - t0
        t0 = time.perf_counter()
        loop = _get_improvement_info(study, improvement_evaluator=optuna_b200.EMMREvaluator(
            seed=0, deterministic_objective=det))
        t_loop = time.perf_counter() - t0
        got = np.array(got)
        rel = lambda w: float(np.max(np.abs(got - w) / np.maximum(np.abs(w), 1e-9)))
        row = {"size": size, "batched_s": round(t_batch, 3), "per_prefix_s": round(t_loop, 3),
               "rounds": stats["rounds"], "device_ms_per_round": round(1e3 * stats["device_seconds"] / stats["rounds"], 3),
               "host_ms_per_round": round(1e3 * (t_batch - stats["device_seconds"]) / stats["rounds"], 3),
               "max_rel_vs_per_prefix": rel(np.array(loop.improvements))}
        if T <= args.reference:
            t0 = time.perf_counter()
            want = _get_improvement_info(study, improvement_evaluator=optuna.terminator.EMMREvaluator(
                seed=0, deterministic_objective=det))
            row["reference_s"] = round(time.perf_counter() - t0, 3)
            row["max_rel_vs_reference"] = rel(np.array(want.improvements))
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
