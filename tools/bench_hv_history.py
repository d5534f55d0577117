"""Time ``optuna_b200.hypervolume_history`` against the reference's ``_get_hypervolume_history_info`` on one study.

The study is synthetic and seeded: DTLZ2-like fronts (points on the positive orthant of the unit sphere, pushed out
by a distance that shrinks over the trials), so the front converges as in a real run and thousands of trials change
the hypervolume.  The reference point is 2.5 in every coordinate.  Prints one JSON line: both wall times, the
largest difference of the two histories, and the card it ran on.

    python tools/bench_hv_history.py [--trials 20000] [--objectives 4] [--repeat 5]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

REFERENCE_POINT = 2.5


def dtlz2_values(n: int, n_objectives: int, seed: int = 0) -> np.ndarray:
    rs = np.random.RandomState(seed)
    d = np.abs(rs.normal(size=(n, n_objectives)))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    t = np.arange(n) / max(n, 1)
    return d * (1.0 + rs.uniform(size=(n, 1)) * (1.5 * (1.0 - t[:, None]) ** 2 + 0.02))


def make_study(values: np.ndarray):
    """An in-memory study of COMPLETE trials with these (minimised) objective values, in this order."""
    import optuna

    study = optuna.create_study(directions=["minimize"] * values.shape[1])
    study.add_trials([optuna.trial.create_trial(values=[float(x) for x in row]) for row in values])
    return study


def _gpu_info() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError, IndexError):
        return "unknown"


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--trials", type=int, default=20000)
    ap.add_argument("--objectives", type=int, default=4)
    ap.add_argument("--repeat", type=int, default=5)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_hv_history.py needs a CUDA device")
    from oracle import ref

    if not ref.enable():
        raise SystemExit("the reference optuna (oracle/_ref) is not available: run __graft_entry__.build()")
    import optuna
    from optuna.visualization._hypervolume_history import _get_hypervolume_history_info

    import optuna_b200

    optuna.logging.set_verbosity(optuna.logging.ERROR)
    values = dtlz2_values(args.trials, args.objectives, args.seed)
    study = make_study(values)
    rp = [REFERENCE_POINT] * args.objectives

    optuna_b200.hypervolume_history(study, rp)   # warm-up: CUDA context, module load, allocator
    times = []
    for _ in range(args.repeat):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        got = optuna_b200.hypervolume_history(study, rp)
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)

    t0 = time.perf_counter()
    want = _get_hypervolume_history_info(study, np.asarray(rp, dtype=np.float64))
    t_ref = time.perf_counter() - t0

    a, b = np.asarray(got.values), np.asarray(want.values)
    same_shape = got.trial_numbers == want.trial_numbers and a.shape == b.shape
    finite = np.isfinite(a) & np.isfinite(b)
    max_abs = float(np.max(np.abs(a[finite] - b[finite]), initial=0.0))
    scale = float(np.max(np.abs(b[finite]), initial=0.0))
    changes = int(np.count_nonzero(np.diff(b, prepend=0.0) != 0.0))
    t_gpu = float(np.median(times))
    print(json.dumps({
        "workload": f"hypervolume_history {args.trials}x{args.objectives} seed {args.seed}",
        "gpu_s_median": round(t_gpu, 5), "gpu_s_all": [round(t, 5) for t in times],
        "reference_s": round(t_ref, 3), "speedup": round(t_ref / t_gpu, 1),
        "max_abs_diff": max_abs, "max_rel_diff": max_abs / scale if scale else 0.0,
        "identical_trials_and_nonfinite": bool(same_shape and np.array_equal(np.isfinite(a), np.isfinite(b))),
        "trials_changing_hv": changes, "gpu": _gpu_info(),
    }))


if __name__ == "__main__":
    main()
