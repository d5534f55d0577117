"""Time the non-dominated box decomposition of GPSampler's log-EHVI: ``TPEEngine.box_decomposition`` (tpe_boxdec.cuh)
against optuna's ``get_non_dominated_box_bounds``.

Each case ``K:nxP`` is a seeded DTLZ2 study (the tests' ``_dtlz2``) of n trials over P parameters with K objectives,
decomposed as ``LogEHVI.__init__`` decomposes it (optuna/_gp/acqf.py:255-261): the Pareto rows of the standardised,
negated values and the reference point from their maxima.  Per case it reports:
- the front size, the steps of each pass (the front sizes they run over), the bounds each pass makes and the boxes;
- the host reference's wall time (one call; ``--no-ref`` skips it);
- the device's wall time: a host clock around the synchronous call, best and median of ``--repeat`` calls after one
  warm-up call;
- whether the device's arrays are the reference's bytes.
Also printed: the card's name and power limit, read in the same run.  Prints one JSON line.

    python tools/bench_box_decomposition.py [--cases 3:1000x8,4:300x8,4:1000x8,5:300x8,5:1000x8,6:300x8]
                                            [--no-ref] [--repeat 5]
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


def _inputs(M: int, n: int, P: int, seed: int = 0):
    from optuna.study._multi_objective import _is_pareto_front

    from tests.test_gp_sampler_ehvi import _dtlz2
    rs = np.random.RandomState(seed)
    Y = -_dtlz2(rs.uniform(0, 1, (n, P)), M)
    Y = (Y - Y.mean(0)) / np.maximum(Y.std(0), 1e-12)
    loss_vals = -Y
    pareto = loss_vals[_is_pareto_front(loss_vals, assume_unique_lexsorted=False)]
    ref = np.max(loss_vals, axis=0)
    return pareto, np.nextafter(np.maximum(1.1 * ref, 0.9 * ref), np.inf)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default="3:1000x8,4:300x8,4:1000x8,5:300x8,5:1000x8,6:300x8")
    ap.add_argument("--no-ref", action="store_true", help="skip optuna's host decomposition")
    ap.add_argument("--repeat", type=int, default=5)
    args = ap.parse_args()
    from oracle import ref as oracle_ref
    if not oracle_ref.enable():
        raise SystemExit("optuna (oracle/_ref) is not available")
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: the device timings need one")
    from optuna._hypervolume import get_non_dominated_box_bounds

    from optuna_b200 import TPEEngine
    rows = []
    eng = TPEEngine(0)
    try:
        for spec in args.cases.split(","):
            k, size = spec.split(":")
            M = int(k)
            n, P = (int(v) for v in size.split("x"))
            pareto, refp = _inputs(M, n, P)
            got = eng.box_decomposition(pareto, refp)   # warm-up (module load, pool growth)
            times = []
            for _ in range(args.repeat):
                t0 = time.perf_counter()
                out = eng.box_decomposition(pareto, refp)
                times.append(time.perf_counter() - t0)
                assert all(a.tobytes() == b.tobytes() for a, b in zip(out, got)), "device calls differ"
            row = {"case": spec, "front": len(pareto), **eng.last_box_stats, "boxes": int(got[0].shape[0]),
                   "device_best_s": min(times), "device_median_s": float(np.median(times))}
            if not args.no_ref:
                with warnings.catch_warnings():
                    warnings.simplefilter("ignore")
                    t0 = time.perf_counter()
                    want = get_non_dominated_box_bounds(pareto, refp)
                    row["host_s"] = time.perf_counter() - t0
                row["identical"] = all(a.shape == b.shape and a.tobytes() == b.tobytes() for a, b in zip(want, got))
                row["speedup"] = row["host_s"] / row["device_best_s"]
            rows.append(row)
            print(json.dumps(row), flush=True)
    finally:
        eng.close()
    print(json.dumps({"gpu": _gpu_info(), "rows": rows}))


if __name__ == "__main__":
    main()
