"""Tiling sweep of the fp64 tensor-core grid kernel (k_logpdf_mma) for every width, big and small path.

Needs the lab build (TPE_LAB=1, libtpe_b200_lab.so).  For each width P and candidate count C it times the
g(x) launch (CUDA events, stage `logpdf_above_main`) of the shipped tiling and of every lab tiling built for
that width (TPE_MMA_LAB=<index>, kMmaLab in tpe_capi.cu) on the same history and uniforms, and prints the
largest |log g| difference to the shipped tiling.  Usage:
    TPE_LAB=1 python tools/tune_mma.py [--widths 8,16,32,64] [--cands 4096,24] [--only 0,1,2]
"""
from __future__ import annotations

import argparse
import os
import re
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from optuna_b200 import ParamSpec, TPEEngine  # noqa: E402

CAPI = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "optuna_b200", "csrc", "tpe_capi.cu")


def lab_widths() -> list[int]:
    """Width (PB) of every kMmaLab entry, in index order, read from the table in tpe_capi.cu (the library ignores an
    index whose width does not match, so a stale list here would time the shipped tiling under a lab label)."""
    src = open(CAPI).read()
    m = re.search(r"const FastCfg kMmaLab\[\] = \{(.*?)\n\};", src, re.S)
    assert m, "kMmaLab not found in tpe_capi.cu"
    body = "\n".join(line.split("//")[0] for line in m.group(1).splitlines())
    widths = [int(v) for v in re.findall(r"MmaInst<\s*(\d+)\s*,", body)]
    assert widths, "kMmaLab is empty"
    return widths


def run(eng, P, C, steps, warm):
    rng = np.random.RandomState(1)
    ts = []
    lg0 = None
    for s in range(warm + steps):
        u = rng.random_sample(C * (1 + P))
        eng.suggest(list(range(P)), u, 1, n_below=25, n_candidates=C, multivariate=True)
        ms, _ = eng.last_timing()
        if s == 0:
            lg0 = eng.get_candidates()[2]
        if s >= warm:
            ts.append(ms[5])
    return np.array(ts), lg0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--widths", default="8,16,32,64")
    ap.add_argument("--cands", default="4096,24")
    ap.add_argument("--only", default="", help="comma-separated kMmaLab indices (default: all)")
    ap.add_argument("--n", type=int, default=100000)
    args = ap.parse_args()
    assert os.environ.get("TPE_LAB") == "1", "the lab tilings live in the lab build: run with TPE_LAB=1"
    lab_pb = lab_widths()
    only = [int(v) for v in args.only.split(",") if v] or list(range(len(lab_pb)))
    for P in [int(v) for v in args.widths.split(",")]:
        rs = np.random.RandomState(0)
        X = rs.uniform(0, 1, (args.n, P))
        key = np.stack([((X - 0.5) ** 2).sum(1), np.zeros(args.n)], 1)
        eng = TPEEngine(0)
        eng.set_space([ParamSpec(kind=0, low=0.0, high=1.0) for _ in range(P)])
        eng.set_history(X, np.zeros(args.n, np.int8), key)
        for C in [int(v) for v in args.cands.split(",")]:
            steps, warm = (10, 2) if C > 64 else (60, 5)
            os.environ.pop("TPE_MMA_LAB", None)
            t0, lg_ref = run(eng, P, C, steps, warm)
            print(f"P={P:3d} C={C:5d} shipped   {t0.mean():.4f} ms (min {t0.min():.4f} max {t0.max():.4f})", flush=True)
            for i in (i for i in only if lab_pb[i] == P):
                os.environ["TPE_MMA_LAB"] = str(i)
                t, lg = run(eng, P, C, steps, warm)
                d = np.abs(lg - lg_ref)
                print(f"P={P:3d} C={C:5d} lab {i:2d}    {t.mean():.4f} ms (min {t.min():.4f} max {t.max():.4f})"
                      f"  max|dlog g| {np.nanmax(d):.2e}", flush=True)
            os.environ.pop("TPE_MMA_LAB", None)
        eng.close()


if __name__ == "__main__":
    main()
