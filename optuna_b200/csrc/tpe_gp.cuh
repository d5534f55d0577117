// Gaussian-process fit of the terminator's improvement evaluators (RegretBoundEvaluator, optuna/terminator/
// improvement/evaluator.py:142-177, and EMMREvaluator, emmr.py:123-237): the covariance, its Cholesky factor and
// inverse, the negative marginal log-likelihood with its gradient in the raw kernel parameters, and the posterior
// (mean and variance, confidence bounds, the joint covariance of a few points).  GPSampler (optuna/samplers/_gp/
// sampler.py) conditions once and then queries the posterior and its gradient in the query point many times against
// the kept L^-1 and alpha.  fp64 throughout.
//
// Storage: n x n row-major matrices, lower triangle significant.  Two of them:
//   A: C = ks Matern52(sum_d l_d sqd_d) + noise I (k_gp_cov), then L in place (right-looking blocked Cholesky), then
//      C^-1 = L^-T L^-1 (k_gp_gemm, lower triangle); during the posterior, the query-by-train cross covariance (and,
//      for gradients, C^-1 k* = L^-T L^-1 k* in rows 64 .. 127).
//   B: L^-1 (blocked TRTRI); upper triangle zero.
// Every O(n^3) step -- the trailing SYRK, the panel TRSM (against the inverted diagonal block), the TRMM of the
// TRTRI, the L^-T L^-1 product and L^-1 k* of the posterior -- is one k_gp_gemm: 64 x 64 tiles on mma.m16n8k8.f64.
// Every reduction is per-CTA partials summed in a fixed order: two calls on the same input return the same bits.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace tpe {
namespace gp {

constexpr int NB = 64;          // block size of the factorisation, tile edge of k_gp_gemm
constexpr int GK = 16;          // k depth of one k_gp_gemm stage
constexpr int GS = GK + 4;      // shared-memory row stride (doubles): conflict-free fragment reads
constexpr int GRAD_DC = 16;     // lengthscale gradients per k_gp_grad pass
constexpr int GRAD_THREADS = 256;

// optuna's Matern52Kernel forward and the derivative it saves for its backward (optuna/_gp/gp.py:63-90), in the
// same operation order.  The derivative is with respect to the squared distance and exact at 0.
__device__ __forceinline__ double matern52(double r) {
  const double s = sqrt(5.0 * r);
  const double e = exp(-s);
  return e * ((5.0 / 3.0) * r + s + 1.0);
}
__device__ __forceinline__ void matern52_both(double r, double& val, double& deriv) {
  const double s = sqrt(5.0 * r);
  const double e = exp(-s);
  val = e * ((5.0 / 3.0) * r + s + 1.0);
  deriv = (-5.0 / 6.0) * (s + 1.0) * e;
}

// sum_d l_d sqd_d with sqd = (a - b)^2, or [(a - b)^2 > 0] in a categorical column (gp.py:185-213)
__device__ __forceinline__ double gp_sqdist(const double* __restrict__ a, const double* __restrict__ b,
                                            const uint8_t* __restrict__ cat, const double* __restrict__ ell, int P) {
  double r = 0.0;
  for (int d = 0; d < P; ++d) {
    const double t = a[d] - b[d];
    double s = t * t;
    if (cat[d]) s = s > 0.0 ? 1.0 : 0.0;
    r += s * ell[d];
  }
  return r;
}

// prm = [l_1 .. l_P, ks, noise_var]
// C over the lower triangle: one thread per element of 32 x 32 tiles, upper tiles exit
__global__ void k_gp_cov(const double* __restrict__ X, const uint8_t* __restrict__ cat, const double* __restrict__ prm,
                         int P, int n, double* __restrict__ A) {
  if (blockIdx.x > blockIdx.y) return;
  const int i = blockIdx.y * 32 + threadIdx.y, j = blockIdx.x * 32 + threadIdx.x;
  if (i >= n || j > i) return;
  const double ks = prm[P], noise = prm[P + 1];
  double c;
  if (i == j) {
    c = matern52(0.0) * ks + noise;
  } else {
    c = matern52(gp_sqdist(X + (int64_t)i * P, X + (int64_t)j * P, cat, prm, P)) * ks;
  }
  A[(int64_t)i * n + j] = c;
}

// Kq[q][i] = ks Matern52(r(xq, X_i)) for q < Q, row stride n
__global__ void k_gp_cross(const double* __restrict__ Xq, const double* __restrict__ X, const uint8_t* __restrict__ cat,
                           const double* __restrict__ prm, int P, int n, int Q, double* __restrict__ K) {
  const int q = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= Q || i >= n) return;
  K[(int64_t)q * n + i] = matern52(gp_sqdist(Xq + (int64_t)q * P, X + (int64_t)i * P, cat, prm, P)) * prm[P];
}

// Unblocked Cholesky of the nb x nb diagonal block at (k0, k0) of A in shared memory, then its inverse by column
// forward substitution.  L goes back to A's lower triangle, L^-1 to the same block of B (upper part zero).  In shared
// memory L^-1[i][j] (i >= j) is kept transposed above L's diagonal, at a[j][i + 1].  A pivot that is <= 0 or NaN
// (LAPACK dpotrf's test) sets *fail; the factor is then meaningless and the caller reports it.
__global__ void __launch_bounds__(256) k_gp_potrf_diag(double* A, double* B, int n, int k0, int nb, int* fail) {
  __shared__ double a[NB][NB + 1];
  const int t = threadIdx.x;
  for (int e = t; e < NB * NB; e += blockDim.x) {
    const int r = e / NB, c = e % NB;
    a[r][c] = (r < nb && c <= r) ? A[(int64_t)(k0 + r) * n + k0 + c] : 0.0;
  }
  __syncthreads();
  for (int c = 0; c < nb; ++c) {
    const double piv = a[c][c];
    if (!(piv > 0.0)) {
      if (t == 0) atomicExch(fail, 1);
      return;   // uniform: every thread read the same pivot
    }
    const double d = sqrt(piv);
    __syncthreads();
    if (t == 0) a[c][c] = d;
    for (int r = c + 1 + t; r < nb; r += blockDim.x) a[r][c] /= d;
    __syncthreads();
    const int m = nb - c - 1;
    for (int e = t; e < m * m; e += blockDim.x) {
      const int r = c + 1 + e / m, s = c + 1 + e % m;
      if (s <= r) a[r][s] -= a[r][c] * a[s][c];
    }
    __syncthreads();
  }
  // L^-1 column by column: thread j solves L x = e_j into row j above the diagonal
  if (t < nb) {
    const int j = t;
    a[j][j + 1] = 1.0 / a[j][j];
    for (int i = j + 1; i < nb; ++i) {
      double s = 0.0;
      for (int k = j; k < i; ++k) s += a[i][k] * a[j][k + 1];
      a[j][i + 1] = -s / a[i][i];
    }
  }
  __syncthreads();
  for (int e = t; e < nb * nb; e += blockDim.x) {
    const int r = e / nb, c = e % nb;
    if (c <= r) A[(int64_t)(k0 + r) * n + k0 + c] = a[r][c];
    B[(int64_t)(k0 + r) * n + k0 + c] = c <= r ? a[c][r + 1] : 0.0;
  }
}

// k_gp_gemm flags
constexpr int GF_TA = 1;        // opA(i, k) = A[k * lda + i] (else A[i * lda + k])
constexpr int GF_TB = 2;        // opB(j, k) = B[k * ldb + j] (else B[j * ldb + k])
constexpr int GF_LOWER = 4;     // write only i >= j (tiles above the diagonal exit)
constexpr int GF_KLO_ROW = 8;   // k starts at the tile's first row (opA zero for k < i)
constexpr int GF_KHI_ROW = 16;  // k ends at the tile's last row (opA zero for k > i)
constexpr int GF_KHI_COL = 32;  // k ends at the tile's last column (opB zero for k > j)
constexpr int GF_SQSUM = 64;    // no store: part[i * gridDim.x + bx] = sum over the tile's columns of out(i, j)^2
constexpr int GF_ACCUM = 128;   // out = alpha * acc + out (else out = alpha * acc)
constexpr int GF_KLO_COL = 256; // k starts at the tile's first column (opB zero for k < j)

// out(i, j) = alpha sum_k opA(i, k) opB(j, k) over an M x N output in 64 x 64 tiles, 4 warps of 32 x 32, each warp
// 2 x 4 fragments of mma.m16n8k8.f64.  A CTA reads all its operand rows before it writes: out may alias the rows of
// A it alone reads (the in-place panel TRSM).
__global__ void __launch_bounds__(128) k_gp_gemm(const double* A, int64_t lda, const double* Bm, int64_t ldb,
                                                 double* out, int64_t ldc, int M, int N, int K, double alpha,
                                                 int flags) {
  const int bx = blockIdx.x, by = blockIdx.y;
  const int i0 = by * NB, j0 = bx * NB;
  if ((flags & GF_LOWER) && j0 > i0) return;
  __shared__ double As[NB][GS];
  __shared__ double Bs[NB][GS];
  __shared__ double red[2][NB];
  int kb = 0, ke = K;
  if (flags & GF_KLO_ROW) kb = i0;
  if (flags & GF_KLO_COL) kb = j0;
  if (flags & GF_KHI_ROW) ke = min(ke, i0 + NB);
  if (flags & GF_KHI_COL) ke = min(ke, j0 + NB);
  kb = (kb / GK) * GK;
  const int t = threadIdx.x, lane = t & 31, w = t >> 5;
  const int wr = (w >> 1) * 32, wc = (w & 1) * 32;
  const int g = lane >> 2, q = lane & 3;
  double acc[2][4][4];
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b)
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[a][b][c] = 0.0;
  const bool ta = flags & GF_TA, tb = flags & GF_TB;
  for (int k0 = kb; k0 < ke; k0 += GK) {
#pragma unroll
    for (int s = 0; s < NB * GK / 128; ++s) {
      const int e = t + 128 * s;
      int r, k;
      if (ta) { k = e / NB; r = e % NB; } else { r = e / GK; k = e % GK; }
      const int gi = i0 + r, gk = k0 + k;
      As[r][k] = (gi < M && gk < ke) ? (ta ? A[(int64_t)gk * lda + gi] : A[(int64_t)gi * lda + gk]) : 0.0;
      if (tb) { k = e / NB; r = e % NB; } else { r = e / GK; k = e % GK; }
      const int gj = j0 + r, gk2 = k0 + k;
      Bs[r][k] = (gj < N && gk2 < ke) ? (tb ? Bm[(int64_t)gk2 * ldb + gj] : Bm[(int64_t)gj * ldb + gk2]) : 0.0;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < GK; kk += 8) {
      double af[2][4], bf[4][2];
#pragma unroll
      for (int a = 0; a < 2; ++a) {
        const int r = wr + a * 16 + g;
        af[a][0] = As[r][kk + q];
        af[a][1] = As[r + 8][kk + q];
        af[a][2] = As[r][kk + q + 4];
        af[a][3] = As[r + 8][kk + q + 4];
      }
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        const int c = wc + b * 8 + g;
        bf[b][0] = Bs[c][kk + q];
        bf[b][1] = Bs[c][kk + q + 4];
      }
#pragma unroll
      for (int a = 0; a < 2; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b)
          tpe::dmma_16x8x8(acc[a][b][0], acc[a][b][1], acc[a][b][2], acc[a][b][3], af[a][0], af[a][1], af[a][2],
                           af[a][3], bf[b][0], bf[b][1]);
    }
    __syncthreads();
  }
  if (flags & GF_SQSUM) {
    // per row: the thread's 8 columns, then the 4 lanes of the row (xor tree), then the two column halves in order
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        double s = 0.0;
#pragma unroll
        for (int b = 0; b < 4; ++b) {
          const double x0 = alpha * acc[a][b][2 * h], x1 = alpha * acc[a][b][2 * h + 1];
          s += x0 * x0;
          s += x1 * x1;
        }
        s += __shfl_xor_sync(0xffffffffu, s, 1);
        s += __shfl_xor_sync(0xffffffffu, s, 2);
        if (q == 0) red[w & 1][wr + a * 16 + h * 8 + g] = s;
      }
    __syncthreads();
    if (t < NB && i0 + t < M) out[(int64_t)(i0 + t) * gridDim.x + bx] = red[0][t] + red[1][t];
    return;
  }
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b)
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int i = i0 + wr + a * 16 + g + (c >> 1) * 8;
        const int j = j0 + wc + b * 8 + 2 * q + (c & 1);
        if (i >= M || j >= N) continue;
        if ((flags & GF_LOWER) && j > i) continue;
        double* o = out + (int64_t)i * ldc + j;
        *o = (flags & GF_ACCUM) ? alpha * acc[a][b][c] + *o : alpha * acc[a][b][c];
      }
}

// u = L^-1 y: one warp per row, lanes strided over the row then a xor tree
__global__ void k_gp_trmv_lower(const double* __restrict__ B, const double* __restrict__ y, int n,
                                double* __restrict__ u) {
  const int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (i >= n) return;
  double s = 0.0;
  for (int k = lane; k <= i; k += 32) s += B[(int64_t)i * n + k] * y[k];
#pragma unroll
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) u[i] = s;
}

// alpha = L^-T u: a CTA of 8 warps takes 32 columns (lane = column), the warps stride over the rows, and the 8
// warp sums are added in warp order
__global__ void __launch_bounds__(256) k_gp_trmv_lower_t(const double* __restrict__ B, const double* __restrict__ u,
                                                         int n, double* __restrict__ alpha) {
  __shared__ double red[8][32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int j = blockIdx.x * 32 + lane;
  double s = 0.0;
  if (j < n)
    for (int i = j + w; i < n; i += 8) s += B[(int64_t)i * n + j] * u[i];
  red[w][lane] = s;
  __syncthreads();
  if (w == 0 && j < n) {
    double r = red[0][lane];
    for (int k = 1; k < 8; ++k) r += red[k][lane];
    alpha[j] = r;
  }
}

// out[0] = sum_i log L_ii, out[1] = u.u: one CTA, fixed strides then a fixed tree
__global__ void __launch_bounds__(256) k_gp_stats(const double* __restrict__ A, const double* __restrict__ u, int n,
                                                  double* __restrict__ out) {
  __shared__ double r0[256], r1[256];
  const int t = threadIdx.x;
  double a = 0.0, b = 0.0;
  for (int i = t; i < n; i += 256) {
    a += log(A[(int64_t)i * n + i]);
    b += u[i] * u[i];
  }
  r0[t] = a;
  r1[t] = b;
  __syncthreads();
  for (int s = 128; s; s >>= 1) {
    if (t < s) {
      r0[t] += r0[t + s];
      r1[t] += r1[t + s];
    }
    __syncthreads();
  }
  if (t == 0) {
    out[0] = r0[0];
    out[1] = r1[0];
  }
}

// (row, column) of the e-th element of the lower triangle in row order
__device__ __forceinline__ void tri_index(int64_t e, int& i, int& j) {
  int64_t r = (int64_t)((sqrt(8.0 * (double)e + 1.0) - 1.0) * 0.5);
  while (r * (r + 1) / 2 > e) --r;
  while ((r + 1) * (r + 2) / 2 <= e) ++r;
  i = (int)r;
  j = (int)(e - r * (r + 1) / 2);
}

// One pass over the lower triangle with W = C^-1 - alpha alpha^T (A holds C^-1).  Per CTA, slots:
//   [0, DC):  sum_{i > j} W_ij M'(r_ij) sqd_ij,d   for d = d0 + slot
//   DC:       sum_{i > j} W_ij M(r_ij)                (pass d0 = 0 only)
//   DC + 1:   sum_i W_ii                              (pass d0 = 0 only)
// part[blockIdx.x * (DC + 2) + slot]; the thread sums of a CTA go through a fixed xor tree and warp order.
template <int DC>
__global__ void __launch_bounds__(GRAD_THREADS) k_gp_grad(const double* __restrict__ A, const double* __restrict__ X,
                                                          const uint8_t* __restrict__ cat,
                                                          const double* __restrict__ prm,
                                                          const double* __restrict__ alpha, int P, int n, int d0,
                                                          double* __restrict__ part) {
  __shared__ double red[GRAD_THREADS / 32][DC + 2];
  double acc[DC + 2];
#pragma unroll
  for (int s = 0; s < DC + 2; ++s) acc[s] = 0.0;
  const int64_t total = (int64_t)n * (n + 1) / 2;
  const int64_t stride = (int64_t)gridDim.x * GRAD_THREADS;
  const int dn = min(DC, P - d0);
  for (int64_t e = (int64_t)blockIdx.x * GRAD_THREADS + threadIdx.x; e < total; e += stride) {
    int i, j;
    tri_index(e, i, j);
    const double w = A[(int64_t)i * n + j] - alpha[i] * alpha[j];
    if (i == j) {
      if (d0 == 0) acc[DC + 1] += w;
      continue;
    }
    const double* xi = X + (int64_t)i * P;
    const double* xj = X + (int64_t)j * P;
    double val, der;
    matern52_both(gp_sqdist(xi, xj, cat, prm, P), val, der);
    const double c = w * der;
    if (d0 == 0) acc[DC] += w * val;
#pragma unroll
    for (int s = 0; s < DC; ++s) {
      if (s < dn) {
        const int d = d0 + s;
        const double t = xi[d] - xj[d];
        double sq = t * t;
        if (cat[d]) sq = sq > 0.0 ? 1.0 : 0.0;
        acc[s] += c * sq;
      }
    }
  }
  const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
#pragma unroll
  for (int s = 0; s < DC + 2; ++s) {
    double v = acc[s];
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) red[wp][s] = v;
  }
  __syncthreads();
  if (threadIdx.x < DC + 2) {
    double v = red[0][threadIdx.x];
    for (int k = 1; k < GRAD_THREADS / 32; ++k) v += red[k][threadIdx.x];
    part[(int64_t)blockIdx.x * (DC + 2) + threadIdx.x] = v;
  }
}

// Sum the CTA partials of one k_gp_grad pass in CTA order and form the gradient of the negative marginal
// log-likelihood in the raw parameters (log l_d, log ks, log(noise - minimum_noise)):
//   d/d log l_d  = ks l_d sum_{i > j} W_ij M' sqd_d
//   d/d log ks   = ks (sum_{i > j} W_ij M + 1/2 sum_i W_ii)
//   d/d raw_noise = 1/2 exp(raw_noise) sum_i W_ii
// grad has P + 2 entries; this pass writes d0 .. d0 + DC - 1, and with d0 = 0 the two sums k_gp_grad_tail turns
// into the last two.
template <int DC>
__global__ void k_gp_grad_finish(const double* __restrict__ part, int nblk, const double* __restrict__ prm, int P,
                                 int d0, double* __restrict__ grad) {
  const int s = threadIdx.x;
  if (s >= DC + 2) return;
  double v = 0.0;
  for (int b = 0; b < nblk; ++b) v += part[(int64_t)b * (DC + 2) + s];
  const double ks = prm[P];
  if (s < DC) {
    if (d0 + s < P) grad[d0 + s] = ks * prm[d0 + s] * v;
  } else if (d0 == 0) {
    if (s == DC) grad[P] = v;   // combined with the diagonal below
    else grad[P + 1] = v;
  }
}

__global__ void k_gp_grad_tail(const double* __restrict__ prm, double noise_excess, int P, double* __restrict__ grad) {
  const double ks = prm[P];
  const double sdiag = grad[P + 1];
  grad[P] = ks * (grad[P] + 0.5 * sdiag);
  grad[P + 1] = 0.5 * noise_excess * sdiag;
}

// Per query: mean = k* . alpha (warp, fixed strides and xor tree); var = ks - sum over column tiles of the squared
// L^-1 k* partials, in tile order, clamped at 0 (gp.py:215-250).  moments: out0 = mean, out1 = var; else out0, out1 =
// mean +- sqrt(beta var) (acqf.py:185-214).
__global__ void k_gp_post_finish(const double* __restrict__ K, const double* __restrict__ alpha,
                                 const double* __restrict__ part, int ntiles, const double* __restrict__ prm, int P,
                                 int n, int Q, double beta, bool moments, double* __restrict__ out0,
                                 double* __restrict__ out1) {
  const int qi = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (qi >= Q) return;
  double m = 0.0;
  for (int i = lane; i < n; i += 32) m += K[(int64_t)qi * n + i] * alpha[i];
#pragma unroll
  for (int o = 16; o; o >>= 1) m += __shfl_xor_sync(0xffffffffu, m, o);
  if (lane == 0) {
    double s = 0.0;
    for (int b = 0; b < ntiles; ++b) s += part[(int64_t)qi * ntiles + b];
    double var = prm[P] - s;
    if (var < 0.0) var = 0.0;
    if (moments) {
      out0[qi] = m;
      out1[qi] = var;
    } else {
      const double h = sqrt(beta * var);
      out0[qi] = m + h;
      out1[qi] = m - h;
    }
  }
}

// Gradients of the posterior mean and variance in the query point (GPRegressor.posterior under autograd, gp.py:
// 215-250, with the Matern derivative saved by gp.py:63-90):
//   dmean/dx_d = 2 l_d ks sum_i alpha_i M'(r_i) (x_d - X_id)
//   dvar/dx_d  = -2 (2 l_d ks sum_i w_i M'(r_i) (x_d - X_id)),   w = C^-1 k* (row q of Wm, row stride n)
// Both are 0 in a categorical column (the reference's `> 0` passes no gradient), and dvar is 0 where the raw variance
// (ks minus the partials of part summed in k_gp_post_finish's order) was clamped.  One CTA per (query, DC columns):
// threads strided over the n training rows, then a xor tree and the warps in order; no atomics.
template <int DC>
__global__ void __launch_bounds__(GRAD_THREADS) k_gp_post_grad(const double* __restrict__ Xq,
                                                               const double* __restrict__ X,
                                                               const uint8_t* __restrict__ cat,
                                                               const double* __restrict__ prm,
                                                               const double* __restrict__ alpha,
                                                               const double* __restrict__ Wm,
                                                               const double* __restrict__ part, int ntiles, int P,
                                                               int n, double* __restrict__ dmean,
                                                               double* __restrict__ dvar) {
  __shared__ double red[GRAD_THREADS / 32][2 * DC];
  const int q = blockIdx.x, d0 = blockIdx.y * DC;
  const int dn = min(DC, P - d0);
  const double* xq = Xq + (int64_t)q * P;
  const double* wq = Wm + (int64_t)q * n;
  double am[DC], av[DC];
#pragma unroll
  for (int s = 0; s < DC; ++s) am[s] = av[s] = 0.0;
  for (int i = threadIdx.x; i < n; i += GRAD_THREADS) {
    const double* xi = X + (int64_t)i * P;
    double val, der;
    matern52_both(gp_sqdist(xq, xi, cat, prm, P), val, der);
    const double cm = alpha[i] * der, cv = wq[i] * der;
#pragma unroll
    for (int s = 0; s < DC; ++s) {
      if (s < dn) {
        const double t = xq[d0 + s] - xi[d0 + s];
        am[s] += cm * t;
        av[s] += cv * t;
      }
    }
  }
  const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
#pragma unroll
  for (int s = 0; s < DC; ++s) {
    double a = am[s], b = av[s];
#pragma unroll
    for (int o = 16; o; o >>= 1) {
      a += __shfl_xor_sync(0xffffffffu, a, o);
      b += __shfl_xor_sync(0xffffffffu, b, o);
    }
    if (lane == 0) {
      red[wp][s] = a;
      red[wp][DC + s] = b;
    }
  }
  __syncthreads();
  if (threadIdx.x < dn) {
    const int s = threadIdx.x, d = d0 + s;
    double vm = red[0][s], vv = red[0][DC + s];
    for (int k = 1; k < GRAD_THREADS / 32; ++k) {
      vm += red[k][s];
      vv += red[k][DC + s];
    }
    double sq = 0.0;
    for (int b = 0; b < ntiles; ++b) sq += part[(int64_t)q * ntiles + b];
    const bool clamped = prm[P] - sq < 0.0;
    const double l2 = 2.0 * prm[d] * prm[P];
    dmean[(int64_t)q * P + d] = cat[d] ? 0.0 : l2 * vm;
    dvar[(int64_t)q * P + d] = (cat[d] || clamped) ? 0.0 : -2.0 * (l2 * vv);
  }
}

// Joint posterior covariance of the first J query points (GPRegressor.posterior with joint=True, gp.py:240-245):
// cov[a][b] = ks Matern52(r(x_a, x_b)) - V_a . V_b with V = K L^-T (row stride n), the diagonal clamped at 0.  One
// warp per entry: lanes strided over n, then a xor tree.  V_a . V_b and V_b . V_a are summed in the same order, so
// the result is exactly symmetric.
__global__ void __launch_bounds__(256) k_gp_joint_cov(const double* __restrict__ Xq, const double* __restrict__ V,
                                                      const uint8_t* __restrict__ cat,
                                                      const double* __restrict__ prm, int P, int n, int J,
                                                      double* __restrict__ cov) {
  const int e = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (e >= J * J) return;
  const int a = e / J, b = e % J;
  const double* va = V + (int64_t)a * n;
  const double* vb = V + (int64_t)b * n;
  double s = 0.0;
  for (int k = lane; k < n; k += 32) s += va[k] * vb[k];
#pragma unroll
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) {
    double c = matern52(gp_sqdist(Xq + (int64_t)a * P, Xq + (int64_t)b * P, cat, prm, P)) * prm[P] - s;
    if (a == b && c < 0.0) c = 0.0;
    cov[e] = c;
  }
}

}  // namespace gp
}  // namespace tpe
