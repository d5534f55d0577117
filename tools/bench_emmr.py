"""Time ``optuna_b200.EMMREvaluator.evaluate`` against the reference's ``EMMREvaluator``.

1. Seeded studies of ``--sizes`` complete trials x P parameters (tools/bench_terminator.py's trials: floats, an int, a
   log float and a categorical): ``evaluate`` with both evaluators on the same trials and seed, the drop-in once to
   warm up (CUDA context, module load) and then ``--repeat`` times.  Both criteria are printed and compared.  The
   reference runs only for the sizes in ``--ref-sizes``.  Every drop-in row also reports how many loss evaluations
   its two fits made and their mean wall time (a host clock around ``TPEEngine.gp_loss``, which ends in a stream
   synchronise).
2. ``--callback N``: a ``TerminatorCallback(Terminator(EMMR, MedianErrorEvaluator(EMMR)))`` on an N-trial study
   (random sampler, 8 floats, a weighted sum of squares plus seeded noise), with each evaluator: the wall time spent
   in the callback, and the number of trials the study ran before the callback stopped it.  This is what a user of
   the terminator pays per study.
Prints one JSON line, with the card's name and power limit.

    python tools/bench_emmr.py [--sizes 1000x8,2000x8,2000x32,10000x8] [--ref-sizes 1000x8,2000x8,2000x32]
                               [--callback 300] [--repeat 2]
"""
from __future__ import annotations

import argparse
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
from tools.bench_terminator import _parse, _timed, make_trials  # noqa: E402


class _CountingEngine:
    """TPEEngine with the number and wall time of its gp_loss calls recorded."""
    calls: list = []

    def __init__(self, device):
        from optuna_b200 import TPEEngine
        self._e = TPEEngine(device)

    def __getattr__(self, name):
        return getattr(self._e, name)

    def gp_loss(self, raw, minimum_noise, deterministic=False):
        t0 = time.perf_counter()
        out = self._e.gp_loss(raw, minimum_noise, deterministic=deterministic)
        _CountingEngine.calls.append(time.perf_counter() - t0)
        return out


def _counted(fn):
    """Run fn with the drop-in's engine counting loss evaluations: (result, count, mean seconds per evaluation)."""
    from optuna_b200 import terminator
    saved = terminator._engine_cls
    terminator._engine_cls = _CountingEngine
    _CountingEngine.calls = []
    try:
        out = fn()
    finally:
        terminator._engine_cls = saved
    c = _CountingEngine.calls
    return out, len(c), (sum(c) / len(c) if c else 0.0)


def _callback_run(make_evaluator, n_trials: int) -> dict:
    import optuna
    from optuna.terminator import MedianErrorEvaluator, Terminator, TerminatorCallback
    w = 1.0 / (1.0 + np.arange(8))
    noise = np.random.RandomState(5).randn(n_trials)

    def objective(trial):
        x = np.array([trial.suggest_float(f"x{j}", -1.0, 1.0) for j in range(8)])
        return float((w * x * x).sum() + 0.05 * noise[trial.number])

    evaluator = make_evaluator()
    cb = TerminatorCallback(Terminator(improvement_evaluator=evaluator,
                                       error_evaluator=MedianErrorEvaluator(evaluator)))
    spent = [0.0]

    def timed_cb(study, trial):
        t0 = time.perf_counter()
        cb(study, trial)
        spent[0] += time.perf_counter() - t0
        if trial.number % 25 == 24:
            print(f"trial {trial.number + 1}: {spent[0]:.1f} s in the callback", file=sys.stderr, flush=True)

    study = optuna.create_study(sampler=optuna.samplers.RandomSampler(seed=0))
    study.optimize(objective, n_trials=n_trials, callbacks=[timed_cb])
    return {"callback_s": spent[0], "trials_run": len(study.trials)}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1000x8,2000x8,2000x32,10000x8")
    ap.add_argument("--ref-sizes", default="1000x8,2000x8,2000x32")
    ap.add_argument("--callback", type=int, default=300)
    ap.add_argument("--repeat", type=int, default=2)
    args = ap.parse_args()

    from oracle import ref
    if not ref.enable():
        raise SystemExit("optuna is not importable (build oracle/_ref first)")
    import optuna
    import optuna_b200
    optuna.logging.set_verbosity(optuna.logging.WARNING)
    warnings.simplefilter("ignore")
    d = optuna.study.StudyDirection.MINIMIZE
    out = {"gpu": _gpu_info(), "evaluate": [], "callback": None}
    ref_sizes = set(_parse(args.ref_sizes))
    for n, P in _parse(args.sizes):
        trials = make_trials(n, P, seed=n + P)
        optuna_b200.EMMREvaluator(seed=0).evaluate(trials[:200], d)   # warm-up: context, module load
        times = []
        for _ in range(args.repeat):
            t, got = _timed(lambda: optuna_b200.EMMREvaluator(seed=0).evaluate(trials, d))
            times.append(t)
        _, count, per = _counted(lambda: optuna_b200.EMMREvaluator(seed=0).evaluate(trials, d))
        row = {"n_complete": n, "P": P, "ours_s": times, "ours_value": got, "loss_evaluations": count,
               "s_per_loss_evaluation": per}
        if (n, P) in ref_sizes:
            t, want = _timed(lambda: optuna.terminator.EMMREvaluator(seed=0).evaluate(trials, d))
            row.update(ref_s=t, ref_value=want, speedup=t / min(times),
                       rel_diff=abs(got - want) / max(abs(want), 1e-300))
        out["evaluate"].append(row)
        print(json.dumps(row), file=sys.stderr, flush=True)
    if args.callback:
        out["callback"] = {"n_trials": args.callback}
        for name, cls in (("ours", optuna_b200.EMMREvaluator), ("ref", optuna.terminator.EMMREvaluator)):
            out["callback"][name] = _callback_run(lambda: cls(seed=0), args.callback)
            print(json.dumps({name: out["callback"][name]}), file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
