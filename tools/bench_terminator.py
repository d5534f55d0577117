"""Time ``optuna_b200.RegretBoundEvaluator.evaluate`` against the reference's ``RegretBoundEvaluator``.

1. Seeded studies of ``--sizes`` complete trials x P parameters (``n_complete x P``, floats, an int, a log float and
   a categorical): ``evaluate`` with both evaluators on the same trials and seed, the drop-in once to warm up (CUDA
   context, module load) and then ``--repeat`` times.  Both bounds are printed and compared.  The reference runs
   only for the sizes in ``--ref-sizes``.
2. ``--large`` (``n_complete x P``, default 60000 x 8, so the GP is fitted to n = 30 000 points): the drop-in only.
   Every drop-in ``evaluate`` also reports how many loss evaluations its fit made and their mean wall time (a host
   clock around ``TPEEngine.gp_loss``, which ends in a stream synchronise).
3. ``_get_improvement_info`` over a ``--prefix``-trial study (one ``evaluate`` per trial prefix), both evaluators.
4. ``--profile n_complete x P``: one ``evaluate`` under ``torch.profiler`` (CUDA activities), device time per kernel
   name; ``--flops`` turns the ``k_gp_gemm`` time into a rate with the GEMM flops of one loss evaluation (n^3: the
   Cholesky, the TRTRI and L^-T L^-1 at n^3 / 3 each), counted from the shapes.
5. ``--replay``: the raw parameters the reference's fit evaluates on a few seeded GP data sets (n up to 257, P up to
   33); at each, the device loss and gradient against the reference's: the largest loss difference (relative), and
   the largest gradient difference relative to the gradient's norm and to the size of its likelihood and prior parts.
Prints one JSON line, with the card's name and power limit.

    python tools/bench_terminator.py [--sizes 2000x8,10000x8,2000x32,10000x32] [--ref-sizes 2000x8,10000x8,2000x32]
                                     [--large 60000x8] [--prefix 300] [--repeat 2]
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


def make_trials(n_trials: int, n_params: int, seed: int):
    import optuna
    from optuna.distributions import CategoricalDistribution, FloatDistribution, IntDistribution

    rs = np.random.RandomState(seed)
    dists = {"i": IntDistribution(0, 20), "lf": FloatDistribution(1e-4, 1.0, log=True),
             "c": CategoricalDistribution(["a", "b", "c"])}
    for j in range(n_params - 3):
        dists[f"x{j}"] = FloatDistribution(-1.0, 1.0)
    cw = {"a": 0.0, "b": 0.7, "c": -0.4}
    xw = 1.0 / (1.0 + np.arange(n_params - 3))
    trials = []
    for _ in range(n_trials):
        p = {"i": int(rs.randint(0, 21)), "lf": float(np.exp(rs.uniform(np.log(1e-4), 0.0))),
             "c": ["a", "b", "c"][rs.randint(3)]}
        xs = rs.uniform(-1.0, 1.0, n_params - 3)
        p.update({f"x{j}": float(x) for j, x in enumerate(xs)})
        v = 0.05 * p["i"] + 0.2 * np.log(p["lf"]) + cw[p["c"]] + float((xw * xs * xs).sum()) + 0.05 * rs.randn()
        trials.append(optuna.trial.create_trial(params=p, distributions=dists, value=v))
    return trials


class _CountingEngine:
    """TPEEngine with the number and wall time of its gp_loss calls recorded."""
    calls: list = []

    def __init__(self, device):
        from optuna_b200 import TPEEngine
        self._e = TPEEngine(device)

    def __getattr__(self, name):
        return getattr(self._e, name)

    def gp_loss(self, raw, minimum_noise):
        t0 = time.perf_counter()
        out = self._e.gp_loss(raw, minimum_noise)
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


def _replay(cases, engine_cls=None):
    """Reference fit points on seeded GP data; device loss / gradient against the reference's at each (``engine_cls``:
    another implementation of the engine's GP methods to measure instead)."""
    import scipy.optimize
    import torch
    from optuna._gp import gp
    from optuna._gp.prior import default_log_prior
    from optuna_b200 import TPEEngine
    from optuna_b200.terminator import _KernelParams, _loss_and_grad
    from optuna._gp import search_space as gp_search_space
    from optuna.search_space import intersection_search_space
    rows = []
    for n, P in cases:
        trials = make_trials(n, P, seed=100 + n + P)
        space = gp_search_space.SearchSpace(intersection_search_space(trials))
        X = space.get_normalized_params(trials)
        y = np.array([t.value for t in trials])
        y = (y - y.mean()) / max(1e-10, y.std())
        cat = space.is_categorical
        seen = []
        real = scipy.optimize.minimize

        def recording(fun, x0, **kw):
            def wrapped(x):
                seen.append(np.array(x, dtype=np.float64))
                return fun(x)
            return real(wrapped, x0, **kw)

        scipy.optimize.minimize = recording
        try:
            gp.fit_kernel_params(X, y, cat, default_log_prior, 1e-6, False)
        finally:
            scipy.optimize.minimize = real
        eng = (engine_cls or TPEEngine)(0)
        eng.gp_set_data(X, y, cat)
        worst = {"loss_rel": 0.0, "grad_over_norm": 0.0, "grad_over_parts": 0.0, "at_point": None, "grad_norm": None}
        for k, raw in enumerate(seen):
            lg, gg = _loss_and_grad(eng, raw, P, default_log_prior, 1e-6)
            gpr = gp.GPRegressor(torch.from_numpy(cat), torch.from_numpy(X), torch.from_numpy(y),
                                 torch.ones(P, dtype=torch.float64), torch.tensor(1.0, dtype=torch.float64),
                                 torch.tensor(1.0, dtype=torch.float64))
            r = torch.from_numpy(raw).requires_grad_(True)
            with torch.enable_grad():
                gpr.inverse_squared_lengthscales = torch.exp(r[:P])
                gpr.kernel_scale = torch.exp(r[P])
                gpr.noise_var = torch.exp(r[P + 1]) + 1e-6
                loss = -gpr.marginal_log_likelihood() - default_log_prior(gpr)
                loss.backward()
            lw, gw = loss.item(), r.grad.numpy()
            r2 = torch.from_numpy(raw).requires_grad_(True)
            with torch.enable_grad():
                (-default_log_prior(_KernelParams(torch.exp(r2[:P]), torch.exp(r2[P]), torch.exp(r2[P + 1]) + 1e-6))).backward()
            gp_ = r2.grad.numpy()
            d = float(np.linalg.norm(gg - gw))
            over_norm = d / float(np.linalg.norm(gw))
            worst["loss_rel"] = max(worst["loss_rel"], abs(lg - lw) / abs(lw))
            worst["grad_over_parts"] = max(worst["grad_over_parts"],
                                           d / float(np.linalg.norm(gw - gp_) + np.linalg.norm(gp_)))
            if over_norm > worst["grad_over_norm"]:
                worst.update(grad_over_norm=over_norm, at_point=k, grad_norm=float(np.linalg.norm(gw)))
        eng.close()
        rows.append({"n": n, "P": P, "points": len(seen), **worst})
        print(json.dumps(rows[-1]), file=sys.stderr, flush=True)
    return rows


def _profile(n_complete, P, flops):
    import torch
    from torch.profiler import ProfilerActivity, profile
    import optuna
    import optuna_b200
    trials = make_trials(n_complete, P, seed=3)
    d = optuna.study.StudyDirection.MINIMIZE
    optuna_b200.RegretBoundEvaluator(seed=0).evaluate(trials[:200], d)   # warm-up: context, module load
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        (_, count, per) = _counted(lambda: optuna_b200.RegretBoundEvaluator(seed=0).evaluate(trials, d))
    torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if t > 0:
            kern[e.key] = {"ms": t / 1e3, "calls": e.count}
    total = sum(v["ms"] for v in kern.values())
    top = dict(sorted(kern.items(), key=lambda kv: -kv[1]["ms"])[:10])
    out = {"n_complete": n_complete, "P": P, "loss_evaluations": count, "kernel_ms_total": total, "kernels": top}
    if flops:
        n = n_complete // 2
        g = sum(v["ms"] for k, v in kern.items() if "k_gp_gemm" in k)
        # per loss evaluation n^3 GEMM flops; the posterior adds about 2 n^2 (n + 2048) / 2
        f = count * float(n) ** 3 + float(n) ** 2 * (n + 2048)
        out["k_gp_gemm_tflops"] = f / (g * 1e-3) / 1e12
    return out


def _timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return time.perf_counter() - t0, out


def _parse(s):
    return [tuple(int(v) for v in x.split("x")) for x in s.split(",") if x]


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="2000x8,10000x8,2000x32,10000x32")
    ap.add_argument("--ref-sizes", default="2000x8,10000x8,2000x32")
    ap.add_argument("--large", default="60000x8")
    ap.add_argument("--prefix", type=int, default=300)
    ap.add_argument("--repeat", type=int, default=2)
    ap.add_argument("--profile", default="")
    ap.add_argument("--flops", action="store_true")
    ap.add_argument("--replay", action="store_true")
    args = ap.parse_args()

    from oracle import ref
    if not ref.enable():
        raise SystemExit("optuna is not importable (build oracle/_ref first)")
    import optuna
    import optuna_b200
    optuna.logging.set_verbosity(optuna.logging.WARNING)
    warnings.simplefilter("ignore")
    d = optuna.study.StudyDirection.MINIMIZE
    out = {"gpu": _gpu_info(), "evaluate": [], "large": None, "prefix": None, "profile": None, "replay": None}
    if args.replay:
        out["replay"] = _replay([(300, 8), (514, 33), (400, 17)])
    if args.profile:
        (n, P), = _parse(args.profile)
        out["profile"] = _profile(n, P, args.flops)
        print(json.dumps(out["profile"]), file=sys.stderr, flush=True)
    ref_sizes = set(_parse(args.ref_sizes))
    for n, P in _parse(args.sizes):
        trials = make_trials(n, P, seed=n + P)
        ours = optuna_b200.RegretBoundEvaluator(seed=0)
        ours.evaluate(trials, d)
        times = []
        for _ in range(args.repeat):
            t, got = _timed(lambda: optuna_b200.RegretBoundEvaluator(seed=0).evaluate(trials, d))
            times.append(t)
        _, count, per = _counted(lambda: optuna_b200.RegretBoundEvaluator(seed=0).evaluate(trials, d))
        row = {"n_complete": n, "P": P, "ours_s": times, "ours_bound": got, "loss_evaluations": count,
               "s_per_loss_evaluation": per}
        if (n, P) in ref_sizes:
            t, want = _timed(lambda: optuna.terminator.RegretBoundEvaluator(seed=0).evaluate(trials, d))
            row.update(ref_s=t, ref_bound=want, speedup=t / min(times), rel_diff=abs(got - want) / max(abs(want), 1e-300))
        out["evaluate"].append(row)
        print(json.dumps(row), file=sys.stderr, flush=True)
    if args.large:
        (n, P), = _parse(args.large)
        trials = make_trials(n, P, seed=1)
        t, (got, count, per) = _timed(lambda: _counted(
            lambda: optuna_b200.RegretBoundEvaluator(seed=0).evaluate(trials, d)))
        out["large"] = {"n_complete": n, "P": P, "ours_s": t, "ours_bound": got, "loss_evaluations": count,
                        "s_per_loss_evaluation": per}
        print(json.dumps(out["large"]), file=sys.stderr, flush=True)
    if args.prefix:
        from optuna.visualization._terminator_improvement import _get_improvement_info
        study = optuna.create_study()
        study.add_trials(make_trials(args.prefix, 8, seed=2))
        t_ours, a = _timed(lambda: _get_improvement_info(study, improvement_evaluator=optuna_b200.RegretBoundEvaluator(seed=0)))
        t_ref, b = _timed(lambda: _get_improvement_info(study, improvement_evaluator=optuna.terminator.RegretBoundEvaluator(seed=0)))
        diff = max(abs(x - y) / max(abs(y), 1e-9) for x, y in zip(a.improvements, b.improvements))
        out["prefix"] = {"trials": args.prefix, "ours_s": t_ours, "ref_s": t_ref, "max_rel_diff": diff}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
