"""Time ``optuna_b200.best_trials`` and ``optuna_b200.pareto_front_info`` against the reference on seeded studies.

The studies are the DTLZ2-like ones of ``tools/bench_hv_history.py`` (converging fronts; at 100 000 trials the front
holds 20 to 43 % of the trials for 3 to 6 objectives).  For each number of objectives, ``best_trials`` is called once
to warm up and then ``--repeat`` times; the median is split into its three stages, each timed on its own with the
same steps ``best_trials`` takes: reading the COMPLETE trials and their values, creating the engine, the device
call (``TPEEngine.pareto_front``: copies in, kernels and copies out, ending in a stream synchronise) and the deep
copies of the front trials.  ``study.best_trials`` is timed once in the same run.  Then
``pareto_front_info(include_dominated_trials=True)`` is timed against ``_get_pareto_front_info`` on a
``--info-trials`` x 3 study.  Prints one JSON line, with the card's name and power limit.

    python tools/bench_pareto_front.py [--trials 100000] [--objectives 2 3 4 6] [--info-trials 20000] [--repeat 5]
"""
from __future__ import annotations

import argparse
import copy
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.bench_hv_history import _gpu_info, dtlz2_values, make_study  # noqa: E402


def _timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return time.perf_counter() - t0, out


def _read(study):
    from optuna.trial import TrialState

    trials = study.get_trials(deepcopy=False, states=(TrialState.COMPLETE,))
    return trials, np.asarray([x.values for x in trials], dtype=np.float64)


def _stages(study, repeat: int) -> dict:
    """Median seconds of the three stages of best_trials, each run on its own."""
    from optuna_b200 import TPEEngine

    read, ctx, dev, cp = [], [], [], []
    for _ in range(repeat):
        t, (trials, values) = _timed(lambda: _read(study))
        read.append(t)
        t, eng = _timed(lambda: TPEEngine(0))
        ctx.append(t)
        try:
            t, mask = _timed(lambda: eng.pareto_front(values))
        finally:
            eng.close()
        dev.append(t)
        front = [x for x, f in zip(trials, mask) if f]
        cp.append(_timed(lambda: copy.deepcopy(front))[0])
    med = {k: round(float(np.median(v)), 5) for k, v in
           (("read_s", read), ("engine_create_s", ctx), ("device_s", dev), ("deepcopy_s", cp))}
    return {**med, "device_s_all": [round(x, 5) for x in dev]}


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--trials", type=int, default=100000)
    ap.add_argument("--objectives", type=int, nargs="+", default=[2, 3, 4, 6])
    ap.add_argument("--info-trials", type=int, default=20000)
    ap.add_argument("--repeat", type=int, default=5)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_pareto_front.py needs a CUDA device")
    from oracle import ref

    if not ref.enable():
        raise SystemExit("the reference optuna (oracle/_ref) is not available: run __graft_entry__.build()")
    import optuna
    from optuna.visualization._pareto_front import _get_pareto_front_info

    import optuna_b200

    optuna.logging.set_verbosity(optuna.logging.ERROR)
    identical = True
    rows = []
    for M in args.objectives:
        study = make_study(dtlz2_values(args.trials, M, args.seed))
        optuna_b200.best_trials(study)   # warm-up: CUDA context, module load
        times = []
        for _ in range(args.repeat):
            t, got = _timed(lambda: optuna_b200.best_trials(study))
            times.append(t)
        t_ref, want = _timed(lambda: study.best_trials)
        same = got == want
        identical = identical and same
        t_gpu = float(np.median(times))
        rows.append({"trials": args.trials, "objectives": M, "front": len(want),
                     "gpu_s_median": round(t_gpu, 5), "gpu_s_all": [round(x, 5) for x in times],
                     **_stages(study, args.repeat),
                     "reference_s": round(t_ref, 3), "speedup": round(t_ref / t_gpu, 1), "identical": same})
        del study

    study = make_study(dtlz2_values(args.info_trials, 3, args.seed))
    optuna_b200.pareto_front_info(study)
    times = []
    for _ in range(args.repeat):
        t, got = _timed(lambda: optuna_b200.pareto_front_info(study, include_dominated_trials=True))
        times.append(t)
    t_ref, want = _timed(lambda: _get_pareto_front_info(study, include_dominated_trials=True))
    same = got == want
    identical = identical and same
    t_gpu = float(np.median(times))
    info = {"trials": args.info_trials, "objectives": 3, "front": len(want.best_trials_with_values),
            "gpu_s_median": round(t_gpu, 5), "gpu_s_all": [round(x, 5) for x in times],
            "reference_s": round(t_ref, 3), "speedup": round(t_ref / t_gpu, 1), "identical": same}

    print(json.dumps({"workload": f"best_trials {args.trials} trials, pareto_front_info {args.info_trials}x3, "
                                  f"seed {args.seed}",
                      "best_trials": rows, "pareto_front_info": info, "identical": identical,
                      "gpu": _gpu_info()}))


if __name__ == "__main__":
    main()
