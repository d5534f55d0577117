"""Tiling sweep of the fp64 tensor-core grid kernel (k_logpdf_mma) for every width, big and small path.

Needs the lab build (TPE_LAB=1, libtpe_b200_lab.so).  For each width P and candidate count C it times the
g(x) launch (CUDA events, stage `logpdf_above_main`) of the shipped tiling and of every lab tiling built for
that width (TPE_MMA_LAB=<index>, kMmaLab in tpe_capi.cu) on the same history and uniforms, and prints the
largest |log g| difference to the shipped tiling.  The counting tilings (DBG = 5) instead print the near-term counters
of one suggestion: near and far terms per candidate (of the K kernels), flushes of the ring per warp and candidate group,
and the mean number of terms a lane had parked at a flush.  Usage:
    TPE_LAB=1 python tools/tune_mma.py [--widths 8,16,32,64] [--cands 4096,24] [--only 0,1,2]
"""
from __future__ import annotations

import argparse
import ctypes as C_
import os
import re
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from optuna_b200 import ParamSpec, TPEEngine  # noqa: E402

CAPI = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "optuna_b200", "csrc", "tpe_capi.cu")


def lab_entries() -> list[tuple[int, int]]:
    """(width PB, DBG) of every kMmaLab entry, in index order, read from the table in tpe_capi.cu (the library ignores
    an index whose width does not match, so a stale list here would time the shipped tiling under a lab label)."""
    src = open(CAPI).read()
    m = re.search(r"const FastCfg kMmaLab\[\] = \{(.*?)\n\};", src, re.S)
    assert m, "kMmaLab not found in tpe_capi.cu"
    body = "\n".join(line.split("//")[0] for line in m.group(1).splitlines())
    entries = [[int(v) for v in args.split(",")] for args in re.findall(r"MmaInst<([\d,\s]+)>", body)]
    assert entries, "kMmaLab is empty"
    return [(e[0], e[7] if len(e) > 7 else 0) for e in entries]


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


def counters(eng, P, C, K):
    """Near-term counters of one suggestion through the selected DBG = 5 tiling (tpe_lab_mma_counters), as shares of
    the C x K cells of the g(x) grid (the l(x) grid, 26 kernels, adds its few terms to the counts)."""
    fn = eng._lib.tpe_lab_mma_counters
    fn.restype, fn.argtypes = C_.c_int, [C_.c_void_p, C_.POINTER(C_.c_ulonglong)]
    out = (C_.c_ulonglong * 5)()
    assert fn(eng._h, out) == 0                    # clear
    u = np.random.RandomState(1).random_sample(C * (1 + P))
    eng.suggest(list(range(P)), u, 1, n_below=25, n_candidates=C, multivariate=True)
    assert fn(eng._h, out) == 0
    near, far, flushes, parked, walked = (int(v) for v in out)
    cells = C * K
    return (f"near {near / cells:.2%} far {far / cells:.2%} of {cells} terms, flushes {flushes}, "
            f"parked per lane at a flush {parked / max(flushes * 32, 1):.2f}, slots walked per flush "
            f"{walked / max(flushes, 1):.2f}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--widths", default="8,16,32,64")
    ap.add_argument("--cands", default="4096,24")
    ap.add_argument("--only", default="", help="comma-separated kMmaLab indices (default: all)")
    ap.add_argument("--n", type=int, default=100000)
    args = ap.parse_args()
    assert os.environ.get("TPE_LAB") == "1", "the lab tilings live in the lab build: run with TPE_LAB=1"
    lab = lab_entries()
    lab_pb = [pb for pb, _ in lab]
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
                if lab[i][1] == 5:
                    print(f"P={P:3d} C={C:5d} lab {i:2d}    {counters(eng, P, C, eng.split_info()[2] + 1)}", flush=True)
                    continue
                t, lg = run(eng, P, C, steps, warm)
                d = np.abs(lg - lg_ref)
                print(f"P={P:3d} C={C:5d} lab {i:2d}    {t.mean():.4f} ms (min {t.min():.4f} max {t.max():.4f})"
                      f"  max|dlog g| {np.nanmax(d):.2e}", flush=True)
            os.environ.pop("TPE_MMA_LAB", None)
        eng.close()


if __name__ == "__main__":
    main()
