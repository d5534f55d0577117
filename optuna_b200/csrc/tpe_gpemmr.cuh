// The posterior terms EMMREvaluator reads from its two Gaussian processes, for every trial prefix at once (the
// improvement curve of plot_terminator_improvement with EMMR, optuna/terminator/improvement/emmr.py:123-237).  The GPs
// are the batch of tpe_gpbatch.cuh (tpe_gp_batch_set); every query is one of the GP's own train rows, given by index:
//   k_gpe_moments  job b is GP gp_idx[b] at prm[b], queried at its rows rows[b][0 .. m-1] (m <= MQ): the posterior
//                  mean, the variance clamped at 0 and, with J > 0, the joint covariance of the first J rows
//
// One CTA per job, on tpe_gpbatch.cuh's frame: C, its Cholesky factor and L^-1 in shared memory for n <= SMEM_N, in
// the job's global workspace above that, then alpha = C^-1 y.  The m cross-covariance vectors k*_q live in the job's
// workspace after the matrix (m x n doubles).  v_q = L^-1 k*_q is formed one row i at a time by one warp (lanes
// strided over k <= i, then a xor tree); lane 0 of that warp keeps the row's products v_qi v_pi in row order, and the
// warps are added in order.  So, as in tpe_gpbatch.cuh, there are no atomics and every sum is in a fixed order that
// depends on n, m and P only: a job's outputs do not depend on the rest of the launch.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "tpe_gpbatch.cuh"

namespace tpe {
namespace gpe {

constexpr int MQ = 3;                        // query rows per job at most: theta*_t, theta*_{t-1}, x_t
constexpr int NPAIR = MQ * (MQ + 1) / 2;     // products v_q . v_p, q <= p
constexpr int THREADS = gpb::THREADS;
constexpr int WARPS = gpb::WARPS;

// workspace doubles of a job: tpe_gpbatch.cuh's matrix workspace (0 for n <= SMEM_N) and the MQ cross-covariance rows
__host__ __device__ inline int64_t ws_doubles(int64_t n) { return gpb::ws_doubles(n) + MQ * n; }

__device__ __forceinline__ int pair_index(int q, int p) { return q * MQ - q * (q - 1) / 2 + (p - q); }   // q <= p

// Job b: GP gp_idx[b] at prm[b] = [l_1 .. l_P, ks, noise_var], at its train rows rows[b * m + q], q < m.
// mean[b * m + q] = k*_q . alpha, var[b * m + q] = ks - |L^-1 k*_q|^2 clamped at 0 (k_gp_post_finish), and with J > 0
// cov[b * J * J + q * J + p] = ks Matern52(r(x_q, x_p)) - v_q . v_p for q, p < J, the diagonal clamped at 0
// (k_gp_joint_cov).  status[b] = 0, or 1 (outputs NaN) when the parameters are not finite or the covariance is not
// positive definite.  The host has checked the row indices.
__global__ void __launch_bounds__(THREADS) k_gpe_moments(const double* __restrict__ X, const double* __restrict__ Y,
                                                         const int64_t* __restrict__ off,
                                                         const uint8_t* __restrict__ cat, int P,
                                                         const int32_t* __restrict__ gp_idx,
                                                         const double* __restrict__ prm_all,
                                                         const int32_t* __restrict__ rows, int m, int J, double* ws,
                                                         const int64_t* __restrict__ ws_off,
                                                         double* __restrict__ mean_out, double* __restrict__ var_out,
                                                         double* __restrict__ cov_out,
                                                         int32_t* __restrict__ status) {
  extern __shared__ double sm[];
  const int b = blockIdx.x, t = threadIdx.x, lane = t & 31, w = t >> 5;
  const int g = gp_idx[b];
  const int n = (int)(off[g + 1] - off[g]);
  const double* Xg = X + off[g] * P;
  double* wsb = ws + ws_off[b];
  const gpb::Frame f = gpb::frame(sm, n, P, wsb);
  double* kq = wsb + gpb::ws_doubles(n);   // [m][n]
  const int32_t* rb = rows + (int64_t)b * m;
  const double qnan = __longlong_as_double(0x7ff8000000000000LL);
  bool ok = gpb::load_prm(prm_all + (int64_t)b * (P + 2), P, f.prm);
  if (ok) {
    gpb::cta_cov(Xg, cat, f.prm, P, n, f.M, f.ld);
    ok = gpb::cta_potrf(f.M, f.ld, n);
  }
  if (!ok) {
    if (t == 0) {
      for (int q = 0; q < m; ++q) mean_out[(int64_t)b * m + q] = var_out[(int64_t)b * m + q] = qnan;
      for (int e = 0; e < J * J; ++e) cov_out[(int64_t)b * J * J + e] = qnan;
      status[b] = 1;
    }
    return;
  }
  gpb::cta_trtri(f.M, f.ld, n, f.tmp);
  gpb::cta_alpha(f.M, f.ld, n, Y + off[g], f.u, f.alpha);
  const double ks = f.prm[P];
  // k*_q [k] = ks Matern52(r(x_q, x_k)) (no noise: the query is a point, not an observation), and k*_q . alpha
  double macc[MQ];
#pragma unroll
  for (int q = 0; q < MQ; ++q) macc[q] = 0.0;
  for (int k = t; k < n; k += THREADS) {
#pragma unroll
    for (int q = 0; q < MQ; ++q) {
      if (q < m) {
        const double kv = __dmul_rn(gp::matern52(gp::gp_sqdist(Xg + (int64_t)rb[q] * P, Xg + (int64_t)k * P, cat,
                                                               f.prm, P)), ks);
        kq[(int64_t)q * n + k] = kv;
        macc[q] = __fma_rn(kv, f.alpha[k], macc[q]);
      }
    }
  }
  __syncthreads();
  // v_qi = sum_{k <= i} L^-1[i][k] k*_q[k], one warp per row; lane 0 keeps the products of its rows
  double pacc[NPAIR];
#pragma unroll
  for (int e = 0; e < NPAIR; ++e) pacc[e] = 0.0;
  for (int i = w; i < n; i += WARPS) {
    double v[MQ];
#pragma unroll
    for (int q = 0; q < MQ; ++q) v[q] = 0.0;
    for (int k = lane; k <= i; k += 32) {
      const double lik = f.M[i * f.ld + k];
#pragma unroll
      for (int q = 0; q < MQ; ++q)
        if (q < m) v[q] = __fma_rn(lik, kq[(int64_t)q * n + k], v[q]);
    }
#pragma unroll
    for (int q = 0; q < MQ; ++q) {
#pragma unroll
      for (int o = 16; o; o >>= 1) v[q] = __dadd_rn(v[q], __shfl_xor_sync(0xffffffffu, v[q], o));
    }
    if (lane == 0) {
#pragma unroll
      for (int q = 0; q < MQ; ++q)
#pragma unroll
        for (int p = q; p < MQ; ++p)
          if (p < m) pacc[pair_index(q, p)] = __fma_rn(v[q], v[p], pacc[pair_index(q, p)]);
    }
  }
  double mq[MQ], pp[NPAIR];
#pragma unroll
  for (int q = 0; q < MQ; ++q) mq[q] = q < m ? gpb::cta_sum(macc[q], f.red) : 0.0;
#pragma unroll
  for (int q = 0; q < MQ; ++q)
#pragma unroll
    for (int p = q; p < MQ; ++p) pp[pair_index(q, p)] = p < m ? gpb::cta_sum(pacc[pair_index(q, p)], f.red) : 0.0;
  // every index below is a compile-time constant, so the arrays stay in registers
  if (t == 0) {
#pragma unroll
    for (int q = 0; q < MQ; ++q) {
      if (q < m) {
        double var = __dsub_rn(ks, pp[pair_index(q, q)]);
        if (var < 0.0) var = 0.0;
        mean_out[(int64_t)b * m + q] = mq[q];
        var_out[(int64_t)b * m + q] = var;
      }
    }
#pragma unroll
    for (int q = 0; q < MQ; ++q)
#pragma unroll
      for (int p = q; p < MQ; ++p) {
        if (p < J) {
          double cv = __dsub_rn(__dmul_rn(gp::matern52(gp::gp_sqdist(Xg + (int64_t)rb[q] * P,
                                                                     Xg + (int64_t)rb[p] * P, cat, f.prm, P)),
                                          ks),
                                pp[pair_index(q, p)]);
          if (q == p && cv < 0.0) cv = 0.0;
          cov_out[(int64_t)b * J * J + q * J + p] = cv;
          cov_out[(int64_t)b * J * J + p * J + q] = cv;
        }
      }
    status[b] = 0;
  }
}

}  // namespace gpe
}  // namespace tpe
