// GPSampler's acquisition functions over device posteriors (optuna/_gp/acqf.py), with their gradient in the query
// point.  The posteriors come from tpe_gp.cuh's kernels (k_gp_cross, k_gp_gemm, k_gp_post_finish, k_gp_post_grad),
// one GP after another on the acquisition context's stream, into mean / var [K][Q] and dmean / dvar [K][Q][P]; the
// log-EHVI part from tpe_ehvi.cuh.  Here:
//   k_acqf_ehvi_in   the objectives' means and standard deviations [Q][M] for k_ehvi_chunk, sd = sqrt(var + noise)
//                    (acqf.py:286), the same rounded operations torch makes;
//   k_acqf_combine   per row: the objective part (LogEI, or the log-EHVI value of k_ehvi_finish, or nothing), the
//                    LogPI terms of the constraints summed as Python's sum() does (0 + t_1 + t_2 ...), and per GP the
//                    coefficients of dmean and dvar that the autograd chain rule gives (coef [K][Q][2]);
//   k_acqf_grad      d value / dx_d = sum over GPs in order of c_mean dmean + c_var dvar, one thread per (row, d).
// Every row depends on its own posterior alone, no atomics and no cross-row sums: a row's value is the same bits
// whatever Q, the row's position and the gradient request.
//
// LogEI (acqf.py:65-92, 151-159), with v = var + noise, sigma = sqrt(v), z = (mean - f0) / sigma:
//   f = log(0.5 z erfc(-z / sqrt 2) + exp(-0.5 z z) / sqrt(2 pi)) + log sigma,   z >= -25
//   f = -0.5 z^2 - log sqrt(2 pi) + log(1 + sqrt(pi / 2) z erfcx(-z / sqrt 2)) + log sigma,   z < -25
// f0 = -inf gives 0 and no gradient.  The reference overwrites the first form where z < -25 by masked assignment, so
// autograd sends 0 / h into the first form's log: NaN where h underflowed to 0.  The gradient here does the same.
// LogPI (acqf.py:175-182): log_ndtr((mean - t) / sigma), torch's log_ndtr and its derivative
// exp(-(log_ndtr(z) + z^2 / 2)) / sqrt(2 pi).
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

namespace tpe {
namespace acqf {

constexpr double kSqrtHalf = 0.7071067811865476;      // math.sqrt(0.5)
constexpr double kInvSqrt2Pi = 0.3989422804014327;    // 1 / math.sqrt(2 * math.pi)
constexpr double kSqrtHalfPi = 1.2533141373155003;    // math.sqrt(0.5 * math.pi)
constexpr double kLogSqrt2Pi = 0.9189385332046727;    // math.log(math.sqrt(2 * math.pi))
constexpr double kSqrt2Pi = 2.5066282746310002;       // std::sqrt(2 * M_PI)
constexpr double kTwoInvSqrtPi = 1.1283791670955126;  // 2 / sqrt(pi), torch's erfc / erfcx derivative constant

// torch's calc_log_ndtr (aten/src/ATen/native/Math.h)
__device__ __forceinline__ double log_ndtr(double x) {
  const double t = __dmul_rn(x, kSqrtHalf);
  if (x < -1.0) return __dadd_rn(log(__dmul_rn(erfcx(-t), 0.5)), -__dmul_rn(t, t));
  return log1p(__dmul_rn(-erfc(t), 0.5));
}

// value and d value / dmean, d value / dvar of LogEI at (mean, var) for threshold f0 (finite)
__device__ __forceinline__ void logei(double mean, double var, double f0, double noise, double& f, double& gm,
                                      double& gv) {
  const double v = __dadd_rn(var, noise);
  const double sigma = sqrt(v);
  const double diff = __dadd_rn(mean, -f0);
  const double z = __ddiv_rn(diff, sigma);
  const double zh = __dmul_rn(0.5, z);
  const double E = erfc(__dmul_rn(-kSqrtHalf, z));
  const double ex = exp(__dmul_rn(-zh, z));
  const double h = __dadd_rn(__dmul_rn(zh, E), __dmul_rn(ex, kInvSqrt2Pi));
  double out, gz;
  if (z < -25.0) {
    const double w = __dmul_rn(-kSqrtHalf, z);
    const double cx = erfcx(w);
    const double a = __dmul_rn(__dmul_rn(kSqrtHalfPi, z), cx);
    const double u = __dadd_rn(1.0, a);
    out = __dadd_rn(__dadd_rn(__dmul_rn(-0.5, __dmul_rn(z, z)), -kLogSqrt2Pi), log(u));
    // d/dz of the second form: -z + (sqrt(pi/2) erfcx(w) + sqrt(pi/2) z erfcx'(w) dw/dz) / u
    const double dcx = __dadd_rn(__dmul_rn(__dmul_rn(2.0, w), cx), -kTwoInvSqrtPi);
    const double da = __dadd_rn(__dmul_rn(kSqrtHalfPi, cx), __dmul_rn(__dmul_rn(kSqrtHalfPi, z), __dmul_rn(dcx, -kSqrtHalf)));
    gz = __dadd_rn(-z, __ddiv_rn(da, u));
    if (h == 0.0) gz = __dadd_rn(gz, NAN);   // 0 / 0 through the overwritten first form
  } else {
    out = log(h);
    // d/dz of h through its operations: z_half E, then exp(-z_half z) / sqrt(2 pi)
    const double dE = __dmul_rn(__dmul_rn(kTwoInvSqrtPi, exp(-__dmul_rn(__dmul_rn(kSqrtHalf, z), __dmul_rn(kSqrtHalf, z)))),
                                kSqrtHalf);
    const double dh = __dadd_rn(__dadd_rn(__dmul_rn(0.5, E), __dmul_rn(zh, dE)), -__dmul_rn(__dmul_rn(ex, kInvSqrt2Pi), z));
    gz = __ddiv_rn(dh, h);
  }
  f = __dadd_rn(out, log(sigma));
  gm = __ddiv_rn(gz, sigma);
  // z = diff / sigma: d/dsigma = -gz diff / (sigma sigma), plus d log(sigma) = 1 / sigma; d sigma / dv = 1 / (2 sigma)
  const double gs = __dadd_rn(__ddiv_rn(__dmul_rn(-gz, diff), __dmul_rn(sigma, sigma)), __ddiv_rn(1.0, sigma));
  gv = __ddiv_rn(gs, __dmul_rn(2.0, sigma));
}

// value and d value / dmean, d value / dvar of LogPI at (mean, var) for threshold t
__device__ __forceinline__ void logpi(double mean, double var, double t, double noise, double& f, double& gm,
                                      double& gv) {
  const double sigma = sqrt(__dadd_rn(var, noise));
  const double diff = __dadd_rn(mean, -t);
  const double z = __ddiv_rn(diff, sigma);
  f = log_ndtr(z);
  const double gz = __dmul_rn(__ddiv_rn(1.0, kSqrt2Pi), exp(-__dadd_rn(f, __ddiv_rn(__dmul_rn(z, z), 2.0))));
  gm = __ddiv_rn(gz, sigma);
  const double gs = __ddiv_rn(__dmul_rn(-gz, diff), __dmul_rn(sigma, sigma));
  gv = __ddiv_rn(gs, __dmul_rn(2.0, sigma));
}

// the objectives' posteriors as k_ehvi_chunk reads them: mean_e, sd_e [Q][M] from mean, var [M][Q]
__global__ void k_acqf_ehvi_in(const double* __restrict__ mean, const double* __restrict__ var, int64_t Q, int M,
                               double noise, double* __restrict__ mean_e, double* __restrict__ sd_e) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= Q * M) return;
  const int64_t q = i / M;
  const int j = (int)(i - q * M);
  mean_e[i] = mean[(int64_t)j * Q + q];
  sd_e[i] = sqrt(__dadd_rn(var[(int64_t)j * Q + q], noise));
}

// kind: 0 LogEI (GP 0 the objective), 1 log-EHVI (GPs 0 .. n_obj - 1, ehvi_* from k_ehvi_finish), 2 no objective
// part.  GPs n_obj .. K - 1 are the constraints, with thresholds thr[n_obj ..].  coef [K][Q][2] when grad.
__global__ void k_acqf_combine(int kind, int K, int n_obj, const double* __restrict__ thr, double noise,
                               const double* __restrict__ mean, const double* __restrict__ var, int64_t Q,
                               const double* __restrict__ ehvi_v, const double* __restrict__ ehvi_dm,
                               const double* __restrict__ ehvi_ds, const double* __restrict__ sd_e,
                               double* __restrict__ value, double* __restrict__ coef) {
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= Q) return;
  const bool grad = coef != nullptr;
  double obj = 0.0;
  if (kind == 0) {
    double gm = 0.0, gv = 0.0;
    if (isinf(thr[0]) && thr[0] < 0.0) {
      obj = 0.0;   // torch.zeros: no gradient
    } else {
      logei(mean[q], var[q], thr[0], noise, obj, gm, gv);
    }
    if (grad) {
      coef[q * 2] = gm;
      coef[q * 2 + 1] = gv;
    }
  } else if (kind == 1) {
    obj = ehvi_v[q];
    if (grad)
      for (int j = 0; j < n_obj; ++j) {
        // sd = sqrt(var + noise): d sd / d var = 1 / (2 sd), torch's sqrt backward
        const double s = sd_e[q * n_obj + j];
        coef[((int64_t)j * Q + q) * 2] = ehvi_dm[q * n_obj + j];
        coef[((int64_t)j * Q + q) * 2 + 1] = __ddiv_rn(ehvi_ds[q * n_obj + j], __dmul_rn(2.0, s));
      }
  }
  double csum = 0.0;   // Python's sum(): 0 + t_1 + t_2 + ...
  for (int c = n_obj; c < K; ++c) {
    double f, gm, gv;
    logpi(mean[(int64_t)c * Q + q], var[(int64_t)c * Q + q], thr[c], noise, f, gm, gv);
    csum = __dadd_rn(csum, f);
    if (grad) {
      coef[((int64_t)c * Q + q) * 2] = gm;
      coef[((int64_t)c * Q + q) * 2 + 1] = gv;
    }
  }
  value[q] = K == n_obj ? obj : (kind == 2 ? csum : __dadd_rn(obj, csum));
}

// grad [Q][P]: one thread per (row, column), the GPs in order
__global__ void k_acqf_grad(int K, const double* __restrict__ coef, const double* __restrict__ dmean,
                            const double* __restrict__ dvar, int64_t Q, int P, double* __restrict__ grad) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= Q * P) return;
  const int64_t q = i / P;
  double acc = 0.0;
  for (int g = 0; g < K; ++g) {
    const double cm = coef[((int64_t)g * Q + q) * 2], cv = coef[((int64_t)g * Q + q) * 2 + 1];
    const int64_t o = (int64_t)g * Q * P + i;
    acc = __dadd_rn(acc, __dadd_rn(__dmul_rn(cm, dmean[o]), __dmul_rn(cv, dvar[o])));
  }
  grad[i] = acc;
}

}  // namespace acqf
}  // namespace tpe
