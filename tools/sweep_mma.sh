#!/bin/bash
# A/B of the g(x) grid kernel variants at config 2: stage timings (CUDA events) + parity of the log-densities
# against the default variant (max |diff| of log g over the 4096 candidates of the same ask).
export TPE_LAB=1   # the variants live in the lab build (libtpe_b200_lab.so)
for v in ${VARIANTS:-default 0 1 2 3}; do
  if [ "$v" = default ]; then unset TPE_MMA_VARIANT; else export TPE_MMA_VARIANT=$v; fi
  echo "== variant $v"
  python - <<'PY'
import os, sys, numpy as np
sys.path.insert(0, os.getcwd())
from optuna_b200 import ParamSpec, TPEEngine
rs = np.random.RandomState(0); N, P, C = 100000, 32, 4096
X = rs.uniform(0, 1, (N, P)); key = np.stack([((X - 0.5) ** 2).sum(1), np.zeros(N)], 1)
eng = TPEEngine(0); eng.set_space([ParamSpec(kind=0, low=0.0, high=1.0) for _ in range(P)]); eng.set_history(X, np.zeros(N, np.int8), key)
rng = np.random.RandomState(1); tot = []
for s in range(12):
    u = rng.random_sample(C * (1 + P))
    x, acq, best = eng.suggest(list(range(P)), u, 1, n_below=25, n_candidates=C, multivariate=True)
    ms, nl = eng.last_timing()
    if s >= 2: tot.append(ms)
    if s == 0:
        smp, ll, lg = eng.get_candidates(); np.save("gpurun_out/lg_%s.npy" % os.environ.get("TPE_MMA_VARIANT", "default"), lg)
m = np.mean(tot, 0)
print("logpdf_above %.4f ms  span %.4f ms  (split %.3f build %.3f sample %.3f below %.3f fix %.3f select %.3f)" % (m[5], m[8], m[0], m[1], m[3], m[4], m[6], m[7]))
ref = "gpurun_out/lg_default.npy"
if os.path.exists(ref):
    print("max |log g - default| =", np.abs(np.load(ref) - lg).max() if False else np.abs(np.load(ref) - np.load("gpurun_out/lg_%s.npy" % os.environ.get("TPE_MMA_VARIANT", "default"))).max())
PY
done
