// Many independent Gaussian processes of one study at once: the fits behind plot_terminator_improvement, one per
// trial prefix (optuna/visualization/_terminator_improvement.py:83-132 calls RegretBoundEvaluator.evaluate once per
// trial).  Each GP has its own n_i rows of X / y (packed back to back, offsets off[]), all share P and the
// categorical flags.  One CTA per GP:
//   k_gpb_loss    -log p(y) and its gradient in the raw kernel parameters, as tpe_gp_loss returns them
//   k_gpb_bounds  max UCB over the train rows, max UCB over the sample rows and max LCB over the train rows
//                 (RegretBoundEvaluator.evaluate's three maxima, evaluator.py:50-84)
//
// The CTA keeps one n x n matrix M (lower triangle significant) and works on it in place: C, then L (column-by-column
// Cholesky), then L^-1 (column-by-column inversion, last column first), then C^-1 = L^-T L^-1 (row by row).  For
// n <= SMEM_N, M and the vectors live in shared memory (161 doubles per row: 160 x 161 x 8 B = 206 KB of the 227 KB a
// CTA may hold, with the three n-vectors beside it); above that, M and the vectors live in a per-GP global workspace
// and the same code runs on it.  The regime depends on n_i alone.
//
// Same bits: no atomics, every sum is in a fixed order that depends on n_i and P only (per thread ascending, then a
// fixed xor tree and the warps in order), so a GP's outputs do not depend on the other GPs of the launch, their
// positions or the wave.  Explicit _rn intrinsics where the compiler could contract.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "tpe_gp.cuh"

namespace tpe {
namespace gpb {

constexpr int THREADS = 256;
constexpr int WARPS = THREADS / 32;
constexpr int SMEM_N = 160;       // largest n whose matrix is kept in shared memory
constexpr int DC = 16;            // lengthscale gradients per pass over the lower triangle
constexpr int NQ = THREADS;       // queries per k_gpb_bounds step (one per thread)
constexpr double LOG_2PI = 1.8378770664093453;   // log(2 pi), correctly rounded

__host__ __device__ inline int64_t smem_ld(int n) { return n + 1; }
// shared-memory bytes of a GP in the shared-memory regime: M, then u, alpha, tmp; and the reduction scratch
__host__ __device__ inline size_t smem_bytes(int n, int P) {
  const size_t mat = n <= SMEM_N ? (size_t)n * smem_ld(n) + 3 * (size_t)n : 0;
  return 8 * (mat + (size_t)(P + 2) + (size_t)WARPS * (DC + 2) + 4);
}
// global workspace doubles of a GP in the global regime (M, u, alpha, tmp); 0 in the shared-memory regime
__host__ __device__ inline int64_t ws_doubles(int64_t n) { return n <= SMEM_N ? 0 : n * n + 3 * n; }

__device__ __forceinline__ double nanmax(double a, double b) {
  // np.max: NaN wins
  return (a != a || b != b) ? __longlong_as_double(0x7ff8000000000000LL) : fmax(a, b);
}

// Sum over the CTA of one value per thread: a xor tree in each warp, then the warps in order.  Every thread gets the
// result.  red holds WARPS doubles.
__device__ double cta_sum(double v, double* red) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o; o >>= 1) v = __dadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  double s = red[0];
  for (int k = 1; k < WARPS; ++k) s = __dadd_rn(s, red[k]);
  return s;
}

__device__ double cta_max(double v, double* red) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o; o >>= 1) v = nanmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  double s = red[0];
  for (int k = 1; k < WARPS; ++k) s = nanmax(s, red[k]);
  return s;
}

// C over the lower triangle: ks Matern52(r) off the diagonal, ks Matern52(0) + noise on it (k_gp_cov's values)
__device__ void cta_cov(const double* __restrict__ X, const uint8_t* __restrict__ cat, const double* prm, int P, int n,
                        double* M, int64_t ld) {
  const double ks = prm[P], noise = prm[P + 1];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int i = w; i < n; i += WARPS)
    for (int j = lane; j <= i; j += 32)
      M[i * ld + j] = i == j ? __dadd_rn(__dmul_rn(gp::matern52(0.0), ks), noise)
                             : __dmul_rn(gp::matern52(gp::gp_sqdist(X + (int64_t)i * P, X + (int64_t)j * P, cat, prm, P)),
                                         ks);
  __syncthreads();
}

// In-place Cholesky, column by column (right-looking).  Returns false, the same in every thread, when a pivot is
// <= 0 or NaN (LAPACK dpotrf's test).
__device__ bool cta_potrf(double* M, int64_t ld, int n) {
  const int t = threadIdx.x, lane = t & 31, w = t >> 5;
  for (int c = 0; c < n; ++c) {
    const double piv = M[c * ld + c];
    if (!(piv > 0.0)) return false;
    const double d = sqrt(piv);
    __syncthreads();   // every thread has read the pivot
    if (t == 0) M[c * ld + c] = d;
    for (int r = c + 1 + t; r < n; r += THREADS) M[r * ld + c] = __ddiv_rn(M[r * ld + c], d);
    __syncthreads();
    for (int r = c + 1 + w; r < n; r += WARPS) {
      const double lrc = M[r * ld + c];
      for (int s = c + 1 + lane; s <= r; s += 32)
        M[r * ld + s] = __dsub_rn(M[r * ld + s], __dmul_rn(lrc, M[s * ld + c]));
    }
    __syncthreads();
  }
  return true;
}

// L^-1 in place of L, last column first: L^-1[i][j] = -(sum_{k=j+1..i} L^-1[i][k] L[k][j]) / L[j][j] for i > j, the
// dot product one warp per row (lanes strided, then a xor tree).  tmp [n] holds the column of L being replaced.
__device__ void cta_trtri(double* M, int64_t ld, int n, double* tmp) {
  const int t = threadIdx.x, lane = t & 31, w = t >> 5;
  for (int j = n - 1; j >= 0; --j) {
    for (int i = j + 1 + t; i < n; i += THREADS) tmp[i] = M[i * ld + j];
    const double inv = __ddiv_rn(1.0, M[j * ld + j]);
    __syncthreads();
    for (int i = j + 1 + w; i < n; i += WARPS) {
      double s = 0.0;
      for (int k = j + 1 + lane; k <= i; k += 32) s = __fma_rn(M[i * ld + k], tmp[k], s);
#pragma unroll
      for (int o = 16; o; o >>= 1) s = __dadd_rn(s, __shfl_xor_sync(0xffffffffu, s, o));
      if (lane == 0) M[i * ld + j] = -__dmul_rn(s, inv);
    }
    if (t == 0) M[j * ld + j] = inv;
    __syncthreads();
  }
}

// C^-1 = L^-T L^-1 in place of L^-1 (lower triangle), row by row from the top: row i reads rows >= i only, which
// are still L^-1.  C^-1[i][j] = sum_{k >= i} L^-1[k][i] L^-1[k][j], one thread per j, k ascending.
__device__ void cta_lauum(double* M, int64_t ld, int n, double* tmp) {
  const int t = threadIdx.x;
  for (int i = 0; i < n; ++i) {
    for (int j = t; j <= i; j += THREADS) {
      double s = 0.0;
      for (int k = i; k < n; ++k) s = __fma_rn(M[k * ld + i], M[k * ld + j], s);
      tmp[j] = s;
    }
    __syncthreads();
    for (int j = t; j <= i; j += THREADS) M[i * ld + j] = tmp[j];
    __syncthreads();
  }
}

// u = L^-1 y (one warp per row), then alpha = L^-T u (one thread per column, rows ascending); M holds L^-1
__device__ void cta_alpha(const double* M, int64_t ld, int n, const double* __restrict__ y, double* u, double* alpha) {
  const int t = threadIdx.x, lane = t & 31, w = t >> 5;
  for (int i = w; i < n; i += WARPS) {
    double s = 0.0;
    for (int k = lane; k <= i; k += 32) s = __fma_rn(M[i * ld + k], y[k], s);
#pragma unroll
    for (int o = 16; o; o >>= 1) s = __dadd_rn(s, __shfl_xor_sync(0xffffffffu, s, o));
    if (lane == 0) u[i] = s;
  }
  __syncthreads();
  for (int j = t; j < n; j += THREADS) {
    double s = 0.0;
    for (int i = j; i < n; ++i) s = __fma_rn(M[i * ld + j], u[i], s);
    alpha[j] = s;
  }
  __syncthreads();
}

// Where a GP's matrix and vectors live: shared memory for n <= SMEM_N, else its global workspace
struct Frame {
  double *M, *u, *alpha, *tmp, *prm, *red;
  int64_t ld;
};
__device__ Frame frame(double* sm, int n, int P, double* ws) {
  Frame f;
  double* tail;
  if (n <= SMEM_N) {
    f.ld = smem_ld(n);
    f.M = sm;
    f.u = sm + (int64_t)n * f.ld;
    tail = f.u + 3 * n;
  } else {
    f.ld = n;
    f.M = ws;
    f.u = ws + (int64_t)n * n;
    tail = sm;
  }
  f.alpha = f.u + n;
  f.tmp = f.alpha + n;
  f.prm = tail;
  f.red = tail + P + 2;
  return f;
}

// prm [P + 2] into shared memory; true when every entry is finite (the same in every thread)
__device__ bool load_prm(const double* __restrict__ src, int P, double* prm) {
  for (int d = threadIdx.x; d < P + 2; d += THREADS) prm[d] = src[d];
  __syncthreads();
  bool ok = true;
  for (int d = 0; d < P + 2; ++d) ok = ok && isfinite(prm[d]);
  return ok;
}

// Job b: GP gp_idx[b] at prm[b] = [l_1 .. l_P, ks, noise_var] with noise_var = nexc[b] + minimum_noise.  Writes
// loss[b] = -log p(y), grad[b] [P + 2] in the raw parameters (as k_gp_grad_finish / k_gp_grad_tail form them) and
// status[b] = 0, or status 1 (loss and grad NaN) when the parameters are not finite or the covariance is not positive
// definite.  ws_off[b]: the job's workspace in ws (doubles).
__global__ void __launch_bounds__(THREADS) k_gpb_loss(const double* __restrict__ X, const double* __restrict__ Y,
                                                      const int64_t* __restrict__ off, const uint8_t* __restrict__ cat,
                                                      int P, const int32_t* __restrict__ gp_idx,
                                                      const double* __restrict__ prm_all,
                                                      const double* __restrict__ nexc, double* ws,
                                                      const int64_t* __restrict__ ws_off, double* __restrict__ loss,
                                                      double* __restrict__ grad, int32_t* __restrict__ status) {
  extern __shared__ double sm[];
  const int b = blockIdx.x, t = threadIdx.x;
  const int g = gp_idx[b];
  const int n = (int)(off[g + 1] - off[g]);
  const double* Xg = X + off[g] * P;
  const double* yg = Y + off[g];
  const Frame f = frame(sm, n, P, ws + ws_off[b]);
  double* gout = grad + (int64_t)b * (P + 2);
  const double qnan = __longlong_as_double(0x7ff8000000000000LL);
  bool ok = load_prm(prm_all + (int64_t)b * (P + 2), P, f.prm);
  if (ok) {
    cta_cov(Xg, cat, f.prm, P, n, f.M, f.ld);
    ok = cta_potrf(f.M, f.ld, n);
  }
  if (!ok) {
    for (int d = t; d < P + 2; d += THREADS) gout[d] = qnan;
    if (t == 0) {
      loss[b] = qnan;
      status[b] = 1;
    }
    return;
  }
  double a = 0.0;
  for (int i = t; i < n; i += THREADS) a = __dadd_rn(a, log(f.M[i * f.ld + i]));
  const double logdet = cta_sum(a, f.red);
  cta_trtri(f.M, f.ld, n, f.tmp);
  cta_alpha(f.M, f.ld, n, yg, f.u, f.alpha);
  a = 0.0;
  for (int i = t; i < n; i += THREADS) a = __fma_rn(f.u[i], f.u[i], a);
  const double uu = cta_sum(a, f.red);
  cta_lauum(f.M, f.ld, n, f.tmp);

  // one pass per DC lengthscales over the lower triangle with W = C^-1 - alpha alpha^T (k_gp_grad's sums); the
  // first pass also sums W_ij M(r_ij) below the diagonal and W_ii
  const int64_t total = (int64_t)n * (n + 1) / 2;
  const double ks = f.prm[P];
  double sval = 0.0, sdiag = 0.0;
  for (int d0 = 0; d0 < P; d0 += DC) {
    double acc[DC + 2];
#pragma unroll
    for (int s = 0; s < DC + 2; ++s) acc[s] = 0.0;
    const int dn = min(DC, P - d0);
    for (int64_t e = t; e < total; e += THREADS) {
      int i, j;
      gp::tri_index(e, i, j);
      const double wij = __dsub_rn(f.M[i * f.ld + j], __dmul_rn(f.alpha[i], f.alpha[j]));
      if (i == j) {
        acc[DC + 1] = __dadd_rn(acc[DC + 1], wij);
        continue;
      }
      const double* xi = Xg + (int64_t)i * P;
      const double* xj = Xg + (int64_t)j * P;
      double val, der;
      gp::matern52_both(gp::gp_sqdist(xi, xj, cat, f.prm, P), val, der);
      const double c = __dmul_rn(wij, der);
      acc[DC] = __fma_rn(wij, val, acc[DC]);
#pragma unroll
      for (int s = 0; s < DC; ++s) {
        if (s < dn) {
          const int d = d0 + s;
          const double q = __dsub_rn(xi[d], xj[d]);
          double sq = __dmul_rn(q, q);
          if (cat[d]) sq = sq > 0.0 ? 1.0 : 0.0;
          acc[s] = __fma_rn(c, sq, acc[s]);
        }
      }
    }
#pragma unroll
    for (int s = 0; s < DC + 2; ++s) {
      if (s < dn || (d0 == 0 && s >= DC)) {
        const double v = cta_sum(acc[s], f.red);
        if (s < DC) {
          if (t == 0) gout[d0 + s] = __dmul_rn(__dmul_rn(ks, f.prm[d0 + s]), v);
        } else if (s == DC) {
          sval = v;
        } else {
          sdiag = v;
        }
      }
    }
  }
  if (t == 0) {
    gout[P] = __dmul_rn(ks, __dadd_rn(sval, __dmul_rn(0.5, sdiag)));
    gout[P + 1] = __dmul_rn(__dmul_rn(0.5, nexc[b]), sdiag);
    // marginal_log_likelihood's order: (logdet_part + const) + quad_part, negated
    const double mll = __dadd_rn(__dsub_rn(-logdet, __dmul_rn(0.5 * (double)n, LOG_2PI)), __dmul_rn(-0.5, uu));
    loss[b] = -mll;
    status[b] = 0;
  }
}

// Job b: GP gp_idx[b] at params prm[b] = [l_1 .. l_P, ks, noise_var], queried at its own n train rows and at the S
// rows of Xs[b] [S, P]: mean +- sqrt(beta[b] var), var = ks - |L^-1 k*|^2 clamped at 0 (k_gp_post_finish's clamp).
// out[b] [3] = max UCB over the train rows, max UCB over the sample rows, max LCB over the train rows (NaN
// propagates as np.max propagates it); status as k_gpb_loss.  One thread per query row: k* into the job's kbuf
// [n x NQ] (column = thread, so a warp's loads are contiguous), then the triangular product against L^-1, i and k
// ascending.
__global__ void __launch_bounds__(THREADS) k_gpb_bounds(const double* __restrict__ X, const double* __restrict__ Y,
                                                        const int64_t* __restrict__ off,
                                                        const uint8_t* __restrict__ cat, int P,
                                                        const int32_t* __restrict__ gp_idx,
                                                        const double* __restrict__ prm_all,
                                                        const double* __restrict__ beta, const double* __restrict__ Xs,
                                                        int S, double* ws, const int64_t* __restrict__ ws_off,
                                                        double* __restrict__ out, int32_t* __restrict__ status) {
  extern __shared__ double sm[];
  const int b = blockIdx.x, t = threadIdx.x;
  const int g = gp_idx[b];
  const int n = (int)(off[g + 1] - off[g]);
  const double* Xg = X + off[g] * P;
  double* kbuf = ws + ws_off[b];
  const Frame f = frame(sm, n, P, kbuf + (int64_t)n * NQ);
  const double qnan = __longlong_as_double(0x7ff8000000000000LL);
  bool ok = load_prm(prm_all + (int64_t)b * (P + 2), P, f.prm);
  if (ok) {
    cta_cov(Xg, cat, f.prm, P, n, f.M, f.ld);
    ok = cta_potrf(f.M, f.ld, n);
  }
  if (!ok) {
    if (t == 0) {
      for (int s = 0; s < 3; ++s) out[(int64_t)b * 3 + s] = qnan;
      status[b] = 1;
    }
    return;
  }
  cta_trtri(f.M, f.ld, n, f.tmp);
  cta_alpha(f.M, f.ld, n, Y + off[g], f.u, f.alpha);
  const double ks = f.prm[P], bt = beta[b];
  const double ninf = -__longlong_as_double(0x7ff0000000000000LL);
  double ucb_train = ninf, ucb_samp = ninf, lcb_train = ninf;
  const int m = n + S;
  for (int q0 = 0; q0 < m; q0 += NQ) {
    const int q = q0 + t;
    if (q < m) {
      const double* xq = q < n ? Xg + (int64_t)q * P : Xs + ((int64_t)b * S + (q - n)) * P;
      double mean = 0.0;
      for (int k = 0; k < n; ++k) {
        const double kv = __dmul_rn(gp::matern52(gp::gp_sqdist(xq, Xg + (int64_t)k * P, cat, f.prm, P)), ks);
        kbuf[(int64_t)k * NQ + t] = kv;
        mean = __fma_rn(kv, f.alpha[k], mean);
      }
      double sq = 0.0;
      for (int i = 0; i < n; ++i) {
        double v = 0.0;
        for (int k = 0; k <= i; ++k) v = __fma_rn(f.M[i * f.ld + k], kbuf[(int64_t)k * NQ + t], v);
        sq = __fma_rn(v, v, sq);
      }
      double var = __dsub_rn(ks, sq);
      if (var < 0.0) var = 0.0;
      const double h = sqrt(__dmul_rn(bt, var));
      const double ucb = __dadd_rn(mean, h), lcb = __dsub_rn(mean, h);
      if (q < n) {
        ucb_train = nanmax(ucb_train, ucb);
        lcb_train = nanmax(lcb_train, lcb);
      } else {
        ucb_samp = nanmax(ucb_samp, ucb);
      }
    }
  }
  ucb_train = cta_max(ucb_train, f.red);
  ucb_samp = cta_max(ucb_samp, f.red);
  lcb_train = cta_max(lcb_train, f.red);
  if (t == 0) {
    out[(int64_t)b * 3 + 0] = ucb_train;
    out[(int64_t)b * 3 + 1] = ucb_samp;
    out[(int64_t)b * 3 + 2] = lcb_train;
    status[b] = 0;
  }
}

}  // namespace gpb
}  // namespace tpe
