"""Time ``optuna_b200.FanovaImportanceEvaluator`` against the reference's ``FanovaImportanceEvaluator``.

1. A seeded ``--trials`` x 8 study (an int, a log float, a 4-choice categorical and five floats, RandomSampler):
   ``get_param_importances`` with the reference evaluator and with the drop-in, same forest seed, end to end (the
   forest fit is in both).  The drop-in runs once to warm up (CUDA context, module load), then ``--repeat`` times.
   Every importance is compared.
2. A seeded ``--large-trials`` x 32 study (the same kinds of parameter), drop-in only: the scikit-learn fit and one
   ``tpe_fanova_variances`` call (``TPEEngine.fanova_variances``: copies in, kernels, copies out, ending in a stream
   synchronise) are timed separately, the call ``--repeat`` times after a warm-up.  The reference is not run at
   that size.
Prints one JSON line, with the card's name and power limit.

    python tools/bench_fanova.py [--trials 2000] [--large-trials 100000] [--repeat 3]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.bench_hv_history import _gpu_info  # noqa: E402


def _timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return time.perf_counter() - t0, out


def make_study(n_trials: int, n_params: int, seed: int):
    """Trials drawn uniformly (as RandomSampler draws them), added in one call; the objective weighs every parameter."""
    import optuna
    from optuna.distributions import CategoricalDistribution, FloatDistribution, IntDistribution

    rs = np.random.RandomState(seed)
    dists = {"i": IntDistribution(0, 20), "lf": FloatDistribution(1e-4, 1.0, log=True),
             "c": CategoricalDistribution(["a", "b", "c", "d"])}
    for j in range(n_params - 3):
        dists[f"x{j}"] = FloatDistribution(-1.0, 1.0)
    cw = {"a": 0.0, "b": 0.7, "c": -0.4, "d": 1.5}
    xw = 1.0 / (1.0 + np.arange(n_params - 3))
    trials = []
    for _ in range(n_trials):
        p = {"i": int(rs.randint(0, 21)), "lf": float(np.exp(rs.uniform(np.log(1e-4), 0.0))),
             "c": ["a", "b", "c", "d"][rs.randint(4)]}
        xs = rs.uniform(-1.0, 1.0, n_params - 3)
        p.update({f"x{j}": float(x) for j, x in enumerate(xs)})
        v = 0.05 * p["i"] + 0.2 * np.log(p["lf"]) + cw[p["c"]] + float((xw * xs * xs).sum()) + 0.05 * rs.randn()
        trials.append(optuna.trial.create_trial(params=p, distributions=dists, value=v))
    study = optuna.create_study(sampler=optuna.samplers.RandomSampler(seed=seed))
    study.add_trials(trials)
    return study


def _small(args) -> dict:
    import optuna

    import optuna_b200

    study = make_study(args.trials, 8, args.seed)
    optuna.importance.get_param_importances(study, evaluator=optuna_b200.FanovaImportanceEvaluator(seed=args.seed))
    times = []
    for _ in range(args.repeat):
        t, got = _timed(lambda: optuna.importance.get_param_importances(
            study, evaluator=optuna_b200.FanovaImportanceEvaluator(seed=args.seed)))
        times.append(t)
    t_ref, want = _timed(lambda: optuna.importance.get_param_importances(
        study, evaluator=optuna.importance.FanovaImportanceEvaluator(seed=args.seed)))
    err = max(abs(want[k] - got[k]) for k in want)
    t_gpu = float(np.median(times))
    return {"trials": args.trials, "params": 8, "gpu_s_median": round(t_gpu, 4),
            "gpu_s_all": [round(x, 4) for x in times], "reference_s": round(t_ref, 2),
            "speedup": round(t_ref / t_gpu, 1), "max_abs_diff": err, "same_order": list(want) == list(got),
            "importances": {k: round(v, 6) for k, v in got.items()}}


def _large(args) -> dict:
    from optuna._transform import _SearchSpaceTransform
    from optuna.importance._base import _get_distributions, _get_filtered_trials, _get_target_values, _get_trans_params

    from optuna_b200 import TPEEngine
    from optuna_b200.importance import _Fanova

    study = make_study(args.large_trials, 32, args.seed + 1)
    dists = _get_distributions(study, params=None)
    trials = _get_filtered_trials(study, params=list(dists), target=None)
    trans = _SearchSpaceTransform(dists, transform_log=False, transform_step=False)
    X, y = _get_trans_params(trials, trans), _get_target_values(trials, None)
    fa = _Fanova(n_trees=64, max_depth=64, seed=args.seed, device=0)
    t_fit, _ = _timed(lambda: fa._forest.fit(X, y))
    trees = [e.tree_ for e in fa._forest.estimators_]
    cols = trans.column_to_encoded_columns
    arrays = dict(node_offsets=np.concatenate([[0], np.cumsum([t.node_count for t in trees])]),
                  left=np.concatenate([t.children_left for t in trees]),
                  right=np.concatenate([t.children_right for t in trees]),
                  feature=np.concatenate([t.feature for t in trees]),
                  threshold=np.concatenate([t.threshold for t in trees]),
                  value=np.concatenate([t.value[:, 0, 0] for t in trees]), bounds=trans.bounds,
                  param_offsets=np.concatenate([[0], np.cumsum([len(c) for c in cols])]),
                  raw_features=np.concatenate(cols))
    eng = TPEEngine(0)
    try:
        eng.fanova_variances(**arrays)
        times = []
        outs = []
        for _ in range(args.repeat):
            t, out = _timed(lambda: eng.fanova_variances(**arrays))
            times.append(t)
            outs.append(out)
    finally:
        eng.close()
    tv, mv = outs[-1]
    keep = tv > 0
    imp = (np.clip(mv, 0, None)[:, keep] / tv[keep]).mean(1)
    spread = max(float(np.max(np.abs(o[1] - mv) / tv[None, :])) for o in outs)
    return {"trials": args.large_trials, "params": 32, "raw_features": int(X.shape[1]),
            "nodes": int(arrays["node_offsets"][-1]), "sklearn_fit_s": round(t_fit, 2),
            "device_call_s_median": round(float(np.median(times)), 4), "device_call_s_all": [round(x, 4) for x in times],
            "max_run_to_run_marginal_diff_over_tree_var": spread,
            "top_importances": {n: round(float(v), 5) for n, v in
                                sorted(zip(dists, imp), key=lambda kv: -kv[1])[:5]}}


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--trials", type=int, default=2000)
    ap.add_argument("--large-trials", type=int, default=100000)
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_fanova.py needs a CUDA device")
    from oracle import ref

    if not ref.enable():
        raise SystemExit("the reference optuna (oracle/_ref) is not available: run __graft_entry__.build()")
    import optuna

    optuna.logging.set_verbosity(optuna.logging.ERROR)
    small = _small(args)
    large = _large(args) if args.large_trials > 0 else None
    print(json.dumps({"workload": f"fANOVA importances, {args.trials} x 8 against the reference, "
                                  f"{args.large_trials} x 32 drop-in only, seed {args.seed}",
                      "small": small, "large": large, "gpu": _gpu_info()}))


if __name__ == "__main__":
    main()
