"""``NumpyEHVIEngine`` -- ``NumpyGPSamplerEngine`` (tests/_gp_sampler_engine.py) with the two engine calls of
``GPSampler``'s multi-objective acquisition: ``ehvi_set`` (tpe_ehvi_set) and ``ehvi`` (tpe_ehvi) (TEST
INFRASTRUCTURE).

The log-EHVI is tpe_ehvi.cuh's algorithm in its order: y = mean + sd z (a product, then a sum); for each chunk of 64
boxes, 128 "threads" each sum P = prod_j clamp(y_sj - lb_bj, EPS, I_bj) over their samples s = t, t + 128, ... and the
chunk's boxes in order; a thread's four values 32 apart are added in order, then a xor tree over 32 lanes; the chunks
are added in order and value = log(sum) - log S.  With gradients each thread also sums, per sample,
G_sj = sum_b (EPS <= d <= I ? P / c : 0) and adds G_sj and G_sj z_sj to its accumulators, reduced the same way.
"""
from __future__ import annotations

import numpy as np

from tests._gp_sampler_engine import NumpyGPSamplerEngine

_EHVI_EPS, _EHVI_CHUNK, _EHVI_THREADS = 1e-12, 64, 128


def _block_sum(r):
    """k_ehvi_chunk's block_sums over the last axis (128 threads)."""
    v = ((r[..., 0:32] + r[..., 32:64]) + r[..., 64:96]) + r[..., 96:128]
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = v + v[..., lanes ^ o]
    return v[..., 0]


class NumpyEHVIEngine(NumpyGPSamplerEngine):
    _ehvi_state = None

    def ehvi_set(self, lower, intervals, samples):
        lb, iv, z = (np.array(a, dtype=np.float64) for a in (lower, intervals, samples))
        if lb.ndim != 2 or iv.shape != lb.shape or z.ndim != 2 or z.shape[1] != lb.shape[1]:
            raise ValueError(f"EHVI inputs must be lower [B, M], intervals [B, M], samples [S, M]; got {lb.shape}, "
                             f"{iv.shape}, {z.shape}")
        self._ehvi_state = None
        B, (S, M) = lb.shape[0], z.shape
        if M < 2 or M > 24:
            raise ValueError(f"EHVI needs 2 <= M <= 24 objectives, got {M}")
        if S < 1 or S > 1024:
            raise ValueError(f"EHVI needs 1 <= S <= 1024 samples, got {S}")
        if B < 1:
            raise ValueError(f"EHVI needs 1 <= B <= 2^31 boxes, got {B}")
        for a, what in ((lb, "box lower bounds"), (iv, "box intervals"), (z, "samples")):
            if np.isnan(a).any():
                raise ValueError(f"EHVI {what} hold a NaN")
        self._ehvi_state = (lb, iv, z)

    def ehvi(self, mean, sd, grad=False):
        if self._ehvi_state is None:
            raise RuntimeError("no EHVI boxes and samples (tpe_ehvi_set)")
        lb, iv, z = self._ehvi_state
        m, s = np.asarray(mean, dtype=np.float64), np.asarray(sd, dtype=np.float64)
        if m.ndim != 2 or s.shape != m.shape or m.shape[1] != lb.shape[1]:
            raise ValueError(f"mean and sd must be [Q, {lb.shape[1]}], got shapes {m.shape}, {s.shape}")
        out = [self._ehvi_rows(m[r:r + 64], s[r:r + 64], grad) for r in range(0, m.shape[0], 64)]
        value = np.concatenate([o[0] for o in out])
        if not grad:
            return value
        return value, np.concatenate([o[1] for o in out]), np.concatenate([o[2] for o in out])

    def _ehvi_rows(self, m, s, grad):
        lb, iv, z = self._ehvi_state
        B, (S, M), Q, T = lb.shape[0], z.shape, m.shape[0], _EHVI_THREADS
        y = m[:, None, :] + s[:, None, :] * z[None]                       # [Q, S, M]
        tot = np.zeros(Q)
        gtot = np.zeros((Q, 2 * M))
        with np.errstate(all="ignore"):
            for b0 in range(0, B, _EHVI_CHUNK):
                acc = np.zeros((Q, T))
                gacc = np.zeros((Q, 2 * M, T))
                for g0 in range(0, S, T):
                    n = min(T, S - g0)
                    yg = y[:, g0:g0 + n]                                  # [Q, n, M]
                    G = np.zeros((Q, n, M))
                    for b in range(b0, min(b0 + _EHVI_CHUNK, B)):
                        d = yg - lb[b]
                        c = np.where(d < _EHVI_EPS, _EHVI_EPS, d)
                        c = np.where(c > iv[b], iv[b], c)
                        P = np.ones((Q, n))
                        for j in range(M):
                            P = P * c[..., j]
                        acc[:, :n] = acc[:, :n] + P
                        if grad:
                            G = G + np.where((d >= _EHVI_EPS) & (d <= iv[b]), P[..., None] / c, 0.0)
                    if grad:
                        gacc[:, :M, :n] = gacc[:, :M, :n] + G.transpose(0, 2, 1)
                        gacc[:, M:, :n] = gacc[:, M:, :n] + (G * z[g0:g0 + n]).transpose(0, 2, 1)
                tot = tot + _block_sum(acc)
                if grad:
                    gtot = gtot + _block_sum(gacc)
            value = np.log(tot) - np.log(S)
            if not grad:
                return (value,)
            return value, gtot[:, :M] / tot[:, None], gtot[:, M:] / tot[:, None]
