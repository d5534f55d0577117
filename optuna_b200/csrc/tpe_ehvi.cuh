// Log expected hypervolume improvement of GPSampler's multi-objective acquisition (optuna/_gp/acqf.py:45-62, logehvi,
// and :245-300, LogEHVI.eval_acqf), with its gradient in the posterior mean and standard deviation of every objective.
//
// For a query row q with posterior mean m_j and standard deviation sd_j, QMC sample s (z_sj) and box b of the
// non-dominated decomposition (lower bound lb_bj, interval I_bj):
//   y_sj  = m_j + sd_j z_sj                        (a rounded product, then a rounded sum: torch's Y_post)
//   c_sbj = min(max(y_sj - lb_bj, EPS), I_bj)      (torch's clamp, NaN propagating)
//   value = log(sum_{s,b} prod_j c_sbj) - log S
// which is the reference's logsumexp over (s, b) of sum_j log c_sbj without a transcendental per term.  Every factor is
// at least EPS = 1e-12, so with M <= 24 a product is at least 1e-288 and never subnormal.
// With P_sb = prod_j c_sbj and the clamp's inclusive mask m_sbj = (EPS <= y_sj - lb_bj <= I_bj),
//   G_sj = sum_b (m_sbj ? P_sb / c_sbj : 0),  dvalue/dm_j = sum_s G_sj / sum P,  dvalue/dsd_j = sum_s G_sj z_sj / sum P.
//
// k_ehvi_chunk: one CTA per (query row, chunk of CHUNK boxes), 128 threads; thread t owns the samples t, t + 128,
// ... and sums its boxes in order; the bounds of the chunk sit in shared memory.  Per CTA a fixed-order reduction
// gives the chunk's partials [sum P, sum_s G_s., sum_s G_s. z_s.].  k_ehvi_finish adds the chunks of a row in order.
// No atomics.  The chunk size is a constant, every sum of the value path is an explicit __dadd_rn / __dmul_rn (no
// contraction), and the value path is the same code with and without gradients: a row's value is the same bits
// whatever the batch, its position in it, or the gradient request.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace tpe {
namespace ehvi {

constexpr int MAX_M = 24;          // objectives at most (EPS^M stays a normal double)
constexpr int MAX_S = 1024;        // QMC samples at most
constexpr int THREADS = 128;
constexpr int CHUNK = 64;          // boxes per CTA
constexpr double EPS = 1e-12;      // optuna/_gp/acqf.py _EPS

// torch's clamp(d, min=EPS, max=I): NaN stays NaN
__device__ __forceinline__ double clamp_box(double d, double I) {
  double c = d < EPS ? EPS : d;
  return c > I ? I : c;
}

// Fixed-order sum of THREADS values red[k * THREADS + t] for k = 0 .. nk - 1 into out[k]: warp w takes k = w, w + 4,
// ...; each lane adds its four values in order, then a xor tree (every lane ends with the same bits).
__device__ __forceinline__ void block_sums(const double* red, int nk, double* out) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int k = warp; k < nk; k += THREADS / 32) {
    const double* r = red + k * THREADS;
    double v = __dadd_rn(__dadd_rn(__dadd_rn(r[lane], r[lane + 32]), r[lane + 64]), r[lane + 96]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = __dadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
    if (lane == 0) out[k] = v;
  }
}

// grid (chunks, rows).  lbI [B][M][2] = (lb, I) interleaved; Z [S][M]; mean, sd [rows][M] (the rows of this launch);
// part [rows][chunks][K] with K = 1 + 2M when GRAD, else 1.
// Shared memory: CHUNK * M * 2 doubles of bounds, then K * THREADS doubles of per-thread sums (ehvi::smem_bytes).
inline size_t smem_bytes(int M, bool grad) { return (size_t)(CHUNK * M * 2 + (grad ? 1 + 2 * M : 1) * THREADS) * 8; }

template <int MC, bool GRAD>
__global__ void __launch_bounds__(THREADS) k_ehvi_chunk(const double* __restrict__ lbI, int64_t B,
                                                       const double* __restrict__ Z, int S, int M,
                                                       const double* __restrict__ mean, const double* __restrict__ sd,
                                                       double* __restrict__ part) {
  extern __shared__ double sm[];
  const int chunk = blockIdx.x, nchunks = gridDim.x;
  const int64_t row = blockIdx.y;
  const int64_t b0 = (int64_t)chunk * CHUNK;
  const int nb = B - b0 < CHUNK ? (int)(B - b0) : CHUNK;
  const int K = GRAD ? 1 + 2 * M : 1;
  double* bnd = sm;                          // [nb][M][2]
  double* red = sm + CHUNK * M * 2;          // [K][THREADS]: sum P, then with GRAD sum_s G_sj and sum_s G_sj z_sj
  const double2* src = reinterpret_cast<const double2*>(lbI + b0 * M * 2);
  double2* dst = reinterpret_cast<double2*>(bnd);
  for (int i = threadIdx.x; i < nb * M; i += THREADS) dst[i] = src[i];
  const int t = threadIdx.x;
  if (GRAD)
    for (int k = 1; k < K; ++k) red[k * THREADS + t] = 0.0;
  __syncthreads();

  double acc = 0.0;   // sum of P over this thread's samples and the chunk's boxes, in order
  for (int s = t; s < S; s += THREADS) {
    double y[MC], G[MC];
#pragma unroll
    for (int j = 0; j < MC; ++j)
      if (j < M) {
        y[j] = __dadd_rn(mean[row * M + j], __dmul_rn(sd[row * M + j], Z[(int64_t)s * M + j]));
        G[j] = 0.0;
      }
    for (int b = 0; b < nb; ++b) {
      const double2* bb = dst + b * M;
      double P = 1.0;
#pragma unroll
      for (int j = 0; j < MC; ++j)
        if (j < M) {
          const double2 li = bb[j];
          P = __dmul_rn(P, clamp_box(__dadd_rn(y[j], -li.x), li.y));
        }
      acc = __dadd_rn(acc, P);
      if (GRAD) {
#pragma unroll
        for (int j = 0; j < MC; ++j)
          if (j < M) {
            const double2 li = bb[j];
            const double d = __dadd_rn(y[j], -li.x);
            const double c = clamp_box(d, li.y);
            if (d >= EPS && d <= li.y) G[j] = __dadd_rn(G[j], __ddiv_rn(P, c));
          }
      }
    }
    if (GRAD) {
#pragma unroll
      for (int j = 0; j < MC; ++j)
        if (j < M) {
          double* g = red + (1 + j) * THREADS + t;
          double* gz = red + (1 + M + j) * THREADS + t;
          *g = __dadd_rn(*g, G[j]);
          *gz = __dadd_rn(*gz, __dmul_rn(G[j], Z[(int64_t)s * M + j]));
        }
    }
  }
  red[t] = acc;
  __syncthreads();
  block_sums(red, K, part + (row * nchunks + chunk) * K);
}

// one thread per row: the chunks of the row in order.  value [rows]; with GRAD dmean, dsd [rows][M].
template <bool GRAD>
__global__ void k_ehvi_finish(const double* __restrict__ part, int64_t rows, int nchunks, int M, double log_s,
                              double* __restrict__ value, double* __restrict__ dmean, double* __restrict__ dsd) {
  const int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= rows) return;
  const int K = GRAD ? 1 + 2 * M : 1;
  const double* p = part + row * nchunks * K;
  double tot = 0.0;
  for (int c = 0; c < nchunks; ++c) tot = __dadd_rn(tot, p[c * K]);
  value[row] = __dadd_rn(log(tot), -log_s);
  if (!GRAD) return;
  for (int k = 0; k < 2 * M; ++k) {
    double g = 0.0;
    for (int c = 0; c < nchunks; ++c) g = __dadd_rn(g, p[c * K + 1 + k]);
    (k < M ? dmean[row * M + k] : dsd[row * M + k - M]) = __ddiv_rn(g, tot);
  }
}

}  // namespace ehvi
}  // namespace tpe
