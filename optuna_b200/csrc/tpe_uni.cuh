// Univariate TPE (multivariate = 0, the reference's default): the 1-D mixture grid.
//
// One suggestion per parameter: log l(x) and log g(x) of C candidates under 1-D mixtures of K kernels
// (probability_distributions.py:154-223 with a single parameter).  At config 2 that is P = 32 grids of
// 4096 x 100 000 (candidate, kernel) pairs per trial -- as many pairs as the multivariate grid has cells, but now
// EVERY pair carries its own exponential.  What makes the 1-D case cheap again is that both axes can be sorted:
// with the kernels ordered by mu (the order the bandwidth computation needs anyway, parzen_estimator.py:196-218)
// and the candidates ordered by x,
//   * a warp owns 32 neighbouring candidates; a tile of 128 neighbouring kernels can be dismissed for all of them
//     with one comparison:  L <= max_tile(cst) - (dist / max_tile(sigma))^2 / 2,  dist = gap between the tile's mu
//     range and the warp's x range -- an upper bound that is exact arithmetic, no approximation;
//   * inside the tiles that remain, an fp32 evaluation with a rigorous rounding bound dismisses single pairs, and
//     the pairs that survive are evaluated in fp64 by lanes that mostly survive TOGETHER (neighbouring x);
//   * every warp walks ALL tiles itself (no k-split: the running max of a candidate is found in the tile under it,
//     first), so far tiles are dismissed against the true scale of the sum, not against a slice-local max.
// The log-sum-exp is the two-tier one of the multivariate kernels: terms within ln K + 17.5 of the running max in
// fp64 (uni_exp), terms down to ln K + 30 below it through MUFU.EX2 in fp32, the rest dropped; same bounds.
#pragma once
#include "tpe_kernels.cuh"

namespace tpe {

constexpr int kUniTile = 128;


struct UniTileMeta {
  double mu_lo, mu_hi;   // range of (mu - ctr) over the tile
  double smax, cmax;     // largest sigma, largest constant (ln w - ln sqrt(2 pi) - M(a, b) - ln sigma)
};

// Sorted tables of one estimator column: position j holds kernel order[j].
//   s32[j] = (m'' = (mu - ctr) / sigma, 1 / sigma, cst, w) in fp32, w = rounding bound of the fp32 z (see k_uni_grid)
//   smi[j] = (m'', 1 / sigma), sc[j] = cst in fp64 (the PAIR table of k_const / k_logpdf_fast, re-ordered)
// fgt != 0 (large estimators, see k_fgt_coeff): kernels whose bandwidth is the clip floor are summed by the fast
// Gauss transform; here they are muted in the screening table (cst = -inf: never pass) and left out of cmax, so
// k_uni_grid evaluates the others only.  bstart[q] = first sorted position whose box index is >= q.
struct FgtGeom {
  double klow, scale, bw;   // scale = sigma_floor * sqrt(2); box width bw = scale / 4
  double lo;                // sigma_floor
  int nb;
  __device__ __forceinline__ void init(const ColMeta& cm, int64_t n, bool magic_clip) {
    double hi;
    sigma_limits(cm, n, magic_clip, lo, hi);
    klow = cm.klow;
    scale = lo * 1.4142135623730951;
    bw = 0.25 * scale;
    const double q = ceil(hi / bw);
    nb = (q < 1.0) ? 1 : ((q > 287.0) ? 287 : (int)q);
  }
  __device__ __forceinline__ int box_of(double m) const {
    const double q = floor((m - klow) / bw);
    return (q < 0.0) ? 0 : ((q >= (double)nb) ? nb - 1 : (int)q);
  }
  __device__ __forceinline__ double centre(int b) const { return klow + ((double)b + 0.5) * bw; }
};
constexpr int kFgtMaxBoxes = 288;
constexpr int kFgtTerms = 24;          // Taylor terms per box (remainder <= 4e-14 of the box's own sum for |y| <= 9)
constexpr double kFgtYmax = 9.0;       // boxes further away (in units of sigma_floor * sqrt 2) are summed directly
constexpr int kFgtRow = 25;            // k_fgt_eval: padded coefficient row in shared memory
constexpr int kFgtCands = 128;         // k_fgt_eval: candidates per block
constexpr size_t kFgtEvalSmem = (64 + (size_t)kFgtMaxBoxes * kFgtRow) * 8 + (size_t)kFgtMaxBoxes * 16;

__device__ __forceinline__ void d_uni_tables(const int32_t* __restrict__ order, const double* __restrict__ mu, const double* __restrict__ sigma,
             const double* __restrict__ cst, const ColMeta* __restrict__ cols, int64_t K, float4* __restrict__ s32,
             double2* __restrict__ smi, double* __restrict__ sc, UniTileMeta* __restrict__ meta, int fgt,
             int magic_clip, int32_t* __restrict__ bstart) {
  __shared__ double r_lo[4], r_hi[4], r_s[4], r_c[4];
  const ColMeta cm = cols[0];
  const double ctr = TPE_MUL(0.5, TPE_ADD(cm.klow, cm.khigh));
  const double half = 0.5 * (cm.khigh - cm.klow);
  const int64_t pos = (int64_t)blockIdx.x * kUniTile + threadIdx.x;
  FgtGeom g;
  if (fgt) g.init(cm, K - 1, magic_clip != 0);
  double lo = INFINITY, hi = -INFINITY, sm = 0.0, cmx = -INFINITY;
  if (pos < K) {
    const int64_t k = order[pos];
    const double m = mu[k], s = sigma[k], c = cst[k];
    const double inv = TPE_DIV(1.0, s);
    const double mm = TPE_MUL(TPE_SUB(m, ctr), inv);
    smi[pos] = make_double2(mm, inv);
    sc[pos] = c;
    const bool regular = fgt && k != K - 1 && s == g.lo;
    // |z_fp32 - z| <= 2^-24 (2 |x'| inv + |m''| + |z|) <= 2^-22 Z with Z = (range / 2) inv >= |x' inv|, |m''|
    const float w = __double2float_ru(half * inv * 2.5e-7);
    s32[pos] = make_float4(__double2float_rn(mm), __double2float_rn(inv), regular ? -INFINITY : __double2float_rn(c), w);
    lo = hi = m - ctr;
    sm = s;
    cmx = regular ? -INFINITY : c;
    if (fgt) {
      const int b = g.box_of(m);
      const int bprev = pos > 0 ? g.box_of(mu[order[pos - 1]]) : -1;
      for (int q = bprev + 1; q <= b; ++q) bstart[q] = (int32_t)pos;
      if (pos == K - 1)
        for (int q = b + 1; q <= g.nb; ++q) bstart[q] = (int32_t)K;
    }
  } else {
    smi[pos] = make_double2(0.0, 0.0);
    sc[pos] = -INFINITY;
    s32[pos] = make_float4(0.0f, 0.0f, -INFINITY, 0.0f);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    lo = fmin(lo, __shfl_xor_sync(0xffffffffu, lo, o));
    hi = fmax(hi, __shfl_xor_sync(0xffffffffu, hi, o));
    sm = fmax(sm, __shfl_xor_sync(0xffffffffu, sm, o));
    cmx = fmax(cmx, __shfl_xor_sync(0xffffffffu, cmx, o));
  }
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) { r_lo[w] = lo; r_hi[w] = hi; r_s[w] = sm; r_c[w] = cmx; }
  __syncthreads();
  if (threadIdx.x == 0) {
    UniTileMeta t;
    t.mu_lo = fmin(fmin(r_lo[0], r_lo[1]), fmin(r_lo[2], r_lo[3]));
    t.mu_hi = fmax(fmax(r_hi[0], r_hi[1]), fmax(r_hi[2], r_hi[3]));
    t.smax = fmax(fmax(r_s[0], r_s[1]), fmax(r_s[2], r_s[3]));
    t.cmax = fmax(fmax(r_c[0], r_c[1]), fmax(r_c[2], r_c[3]));
    meta[blockIdx.x] = t;
  }
}
__global__ void __launch_bounds__(kUniTile)
k_uni_tables(const int32_t* __restrict__ order, const double* __restrict__ mu, const double* __restrict__ sigma,
             const double* __restrict__ cst, const ColMeta* __restrict__ cols, int64_t K, float4* __restrict__ s32,
             double2* __restrict__ smi, double* __restrict__ sc, UniTileMeta* __restrict__ meta, int fgt,
             int magic_clip, int32_t* __restrict__ bstart) { d_uni_tables(order, mu, sigma, cst, cols, K, s32, smi, sc, meta, fgt, magic_clip, bstart); }

// The tiles that hold a kernel k_uni_grid has to evaluate itself (cmax > -inf), ascending: with the fast Gauss transform
// on these are a handful (the prior, sparse regions), and the grid walks this list instead of all tiles.
// One block of 256 threads; list[0] = count, list[1 ..] = tile indices.
__device__ __forceinline__ void d_uni_tile_list(const UniTileMeta* __restrict__ meta, int ntiles, int32_t* __restrict__ list) {
  __shared__ int s_cnt[256];
  const int per = (ntiles + 255) / 256;
  const int t0 = threadIdx.x * per, t1 = min(ntiles, t0 + per);
  int cnt = 0;
  for (int t = t0; t < t1; ++t) cnt += meta[t].cmax > -INFINITY ? 1 : 0;
  s_cnt[threadIdx.x] = cnt;
  __syncthreads();
  if (threadIdx.x == 0) {
    int run = 0;
    for (int i = 0; i < 256; ++i) {
      const int v = s_cnt[i];
      s_cnt[i] = run;
      run += v;
    }
    list[0] = run;
  }
  __syncthreads();
  int at = s_cnt[threadIdx.x];
  for (int t = t0; t < t1; ++t)
    if (meta[t].cmax > -INFINITY) list[1 + at++] = t;
}
__global__ void __launch_bounds__(256)
k_uni_tile_list(const UniTileMeta* __restrict__ meta, int ntiles, int32_t* __restrict__ list) {
  d_uni_tile_list(meta, ntiles, list);
}

// ---- fast Gauss transform for the kernels at the bandwidth floor -------------------------------------------------
// With thousands of observations nearly every kernel of a 1-D estimator has sigma = sigma_floor = range / 100
// (parzen_estimator.py:220-228: the neighbour gaps are far smaller).  Their part of the mixture,
//     sum_j exp(c_j) exp(-(x - mu_j)^2 / (2 sigma^2)),
// is a Gauss transform with ONE bandwidth.  Boxes of width sigma sqrt(2) / 4 along the axis; for the sources of box B
// (centre c_B, t_j = (mu_j - c_B) / (sigma sqrt 2), |t_j| <= 1/8) and a target y = (x - c_B) / (sigma sqrt 2):
//     exp(-(y - t)^2) = exp(-y^2) sum_n H_n(y) t^n / n!          (generating function of the Hermite polynomials)
//     box sum         = exp(ref_B - y^2) sum_n A_n H_n(y),   A_n = sum_j exp(c_j - ref_B) t_j^n / n!
// so a candidate costs (boxes in reach) x kFgtTerms multiply-adds instead of one exponential per kernel in reach.
// Truncation after 24 terms: remainder <= |h_24(u)| |t|^24 / 24! with h_n = H_n exp(-u^2); by Cramer's bound
// (|h_n(u)| <= 1.09 2^(n/2) sqrt(n!) exp(-u^2 / 2)) that is <= 1e-18 of the box's own sum for |y| <= 7, and with
// |H_n(u)| <= (2u)^n beyond the last zero (u >= 7) it is <= (2 |y| / 8)^24 / 24! exp(|y| / 2) <= 4e-14 up to
// |y| = 9 (kFgtYmax); boxes further out that still matter (a candidate far from every observation) are summed
// directly.  A box is left out when its upper bound A_0 exp(ref - (|y| - 1/8)^2) lies 30 + ln(#boxes) below the
// largest lower bound A_0 exp(ref - (|y| + 1/8)^2) of any box or below the prior kernel's term: together <= 1e-13 of
// the sum, the truncation rule the pair kernels use.  Everything is summed in a fixed order.
struct FgtBox {
  double ref;     // largest c_j of the box's floor-bandwidth kernels (-inf: none)
  double lnw;     // ref + ln A_0
};

// grid = boxes, 128 threads
__device__ __forceinline__ void d_fgt_coeff(const int32_t* __restrict__ order, const double* __restrict__ mu, const double* __restrict__ sigma,
            const double* __restrict__ cst, const ColMeta* __restrict__ cols, int64_t K, int magic_clip,
            const int32_t* __restrict__ bstart, double* __restrict__ coef, FgtBox* __restrict__ box) {
  __shared__ double s_red[4][kFgtTerms];
  __shared__ double s_ref;
  FgtGeom g;
  g.init(cols[0], K - 1, magic_clip != 0);
  const int b = blockIdx.x;
  if (b >= g.nb) {
    if (threadIdx.x == 0) box[b] = FgtBox{-INFINITY, -INFINITY};
    return;
  }
  const int p0 = bstart[b], p1 = bstart[b + 1];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double ref = -INFINITY;
  for (int p = p0 + threadIdx.x; p < p1; p += 128) {
    const int k = order[p];
    if (k != K - 1 && sigma[k] == g.lo) ref = fmax(ref, cst[k]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ref = fmax(ref, __shfl_xor_sync(0xffffffffu, ref, o));
  if (lane == 0) s_red[warp][0] = ref;
  __syncthreads();
  if (threadIdx.x == 0) s_ref = fmax(fmax(s_red[0][0], s_red[1][0]), fmax(s_red[2][0], s_red[3][0]));
  __syncthreads();
  ref = s_ref;
  __syncthreads();
  double a[kFgtTerms];
#pragma unroll
  for (int n = 0; n < kFgtTerms; ++n) a[n] = 0.0;
  const double cb = g.centre(b), inv = 1.0 / g.scale;
  for (int p = p0 + threadIdx.x; p < p1; p += 128) {
    const int k = order[p];
    if (k == K - 1 || sigma[k] != g.lo) continue;
    const double t = (mu[k] - cb) * inv;
    double pw = exp(cst[k] - ref);
#pragma unroll
    for (int n = 0; n < kFgtTerms; ++n) {
      a[n] += pw;
      pw *= t * (1.0 / (double)(n + 1));
    }
  }
#pragma unroll
  for (int n = 0; n < kFgtTerms; ++n) {
    double v = a[n];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) s_red[warp][n] = v;
  }
  __syncthreads();
  if (threadIdx.x < kFgtTerms) {
    const int n = threadIdx.x;
    const double v = (s_red[0][n] + s_red[1][n]) + (s_red[2][n] + s_red[3][n]);
    coef[(size_t)b * kFgtRow + n] = v;
    if (n == 0) box[b] = FgtBox{ref, (ref > -INFINITY) ? ref + log(v) : -INFINITY};
  }
}
__global__ void __launch_bounds__(128)
k_fgt_coeff(const int32_t* __restrict__ order, const double* __restrict__ mu, const double* __restrict__ sigma,
            const double* __restrict__ cst, const ColMeta* __restrict__ cols, int64_t K, int magic_clip,
            const int32_t* __restrict__ bstart, double* __restrict__ coef, FgtBox* __restrict__ box) { d_fgt_coeff(order, mu, sigma, cst, cols, K, magic_clip, bstart, coef, box); }

// part[c] = (reference, sum) of the floor-bandwidth kernels for candidate c.  A block takes kFgtCands candidates of one
// column (one warp per candidate, eight at a time) and stages the column's coefficients and box table in shared memory
// first (rows padded to 25 doubles: a half-warp reading 16 consecutive boxes touches 16 different bank pairs).
//   xT [C] kernel-space coordinate of the candidates (log applied), in ask order
__device__ __forceinline__ void d_fgt_eval(const double* __restrict__ coef, const FgtBox* __restrict__ box, const int32_t* __restrict__ bstart,
           const float4* __restrict__ s32, const double2* __restrict__ smi, const double* __restrict__ sc,
           const double* __restrict__ mu,
           const double* __restrict__ sigma, const double* __restrict__ cst, const ColMeta* __restrict__ cols,
           int64_t K, int magic_clip, const double* __restrict__ xT, int C, double2* __restrict__ part) {
  extern __shared__ __align__(16) double s_fgt[];
  double* s_e64 = s_fgt;                                    // [64]
  double* s_coef = s_fgt + 64;                              // [nb][kFgtRow]
  const ColMeta cm = cols[0];
  FgtGeom g;
  g.init(cm, K - 1, magic_clip != 0);
  FgtBox* s_box = reinterpret_cast<FgtBox*>(s_coef + (size_t)kFgtMaxBoxes * kFgtRow);   // [nb]
  if (threadIdx.x < 64) s_e64[threadIdx.x] = exp2((double)threadIdx.x * 0.015625);
  for (int i = threadIdx.x; i < g.nb * kFgtRow; i += blockDim.x) s_coef[i] = coef[i];   // (rows padded to kFgtRow)
  for (int i = threadIdx.x; i < g.nb; i += blockDim.x) s_box[i] = box[i];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int c_end = min(C, (int)(blockIdx.x + 1) * kFgtCands);
  for (int c = blockIdx.x * kFgtCands + (threadIdx.x >> 5); c < c_end; c += (int)(blockDim.x >> 5)) {
  const double x = xT[c];
  const double inv = 1.0 / g.scale;
  // floor of the scale: the prior kernel's term (it is summed by k_uni_grid; here it only decides what is negligible)
  double best;
  {
    const double zp = (x - mu[K - 1]) / sigma[K - 1];
    best = cst[K - 1] - 0.5 * zp * zp;
    if (!(best > -INFINITY)) best = -INFINITY;
  }
  for (int b = lane; b < g.nb; b += 32) {
    const FgtBox bx = s_box[b];
    if (!(bx.lnw > -INFINITY)) continue;
    const double y = fabs((x - g.centre(b)) * inv) + 0.125;
    best = fmax(best, bx.lnw - y * y);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) best = fmax(best, __shfl_xor_sync(0xffffffffu, best, o));
  if (!(best > -INFINITY)) {                    // NaN candidate / no kernels at all
    if (lane == 0) part[c] = make_double2(-INFINITY, 0.0);
    continue;
  }
  const double drop = 30.0 + log((double)g.nb);
  const double ctr = TPE_MUL(0.5, TPE_ADD(cm.klow, cm.khigh));
  double sum = 0.0;
  for (int b = lane; b < g.nb; b += 32) {
    const FgtBox bx = s_box[b];
    if (!(bx.lnw > -INFINITY)) continue;
    const double y = (x - g.centre(b)) * inv;
    const double ay = fabs(y);
    const double near = fmax(ay - 0.125, 0.0);
    if (bx.lnw - near * near < best - drop) continue;
    if (ay <= kFgtYmax) {
      const double* __restrict__ a = s_coef + (size_t)b * kFgtRow;
      // sum_n A_n H_n(y):  H_0 = 1, H_1 = 2y, H_(n+1) = 2y H_n - 2n H_(n-1)
      const double y2 = 2.0 * y;
      double hm = 1.0, h = y2;
      double acc = fma(a[1], h, a[0]);
#pragma unroll
      for (int n = 1; n < kFgtTerms - 1; ++n) {
        const double hn = fma(y2, h, -2.0 * (double)n * hm);
        hm = h;
        h = hn;
        acc = fma(a[n + 1], h, acc);
      }
      sum += acc * uni_exp(fmax(bx.ref - y * y - best, -700.0), s_e64);
    } else {
      // a candidate far from this box that still counts (nothing nearer): its kernels one by one
      const int p0 = bstart[b], p1 = bstart[b + 1];
      const double xc = x - ctr;
      double part_sum = 0.0;
      for (int p = p0; p < p1; ++p) {
        if (s32[p].z > -INFINITY) continue;     // not at the floor: k_uni_grid has it
        const double2 mi = smi[p];
        const double tt = fma(xc, mi.y, -mi.x);
        part_sum += uni_exp(fmax(fma(-0.5 * tt, tt, sc[p]) - best, -700.0), s_e64);
      }
      sum += part_sum;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if (lane == 0) part[c] = (sum > 0.0) ? make_double2(best, sum) : make_double2(-INFINITY, 0.0);
  }
}
__global__ void __launch_bounds__(256)
k_fgt_eval(const double* __restrict__ coef, const FgtBox* __restrict__ box, const int32_t* __restrict__ bstart,
           const float4* __restrict__ s32, const double2* __restrict__ smi, const double* __restrict__ sc,
           const double* __restrict__ mu,
           const double* __restrict__ sigma, const double* __restrict__ cst, const ColMeta* __restrict__ cols,
           int64_t K, int magic_clip, const double* __restrict__ xT, int C, double2* __restrict__ part) { d_fgt_eval(coef, box, bstart, s32, smi, sc, mu, sigma, cst, cols, K, magic_clip, xT, C, part); }

// The candidates of one ask in ascending kernel-space order: xs[i] = x' = x - ctr of the i-th smallest,
// cidx[i] = its index.  One CTA of 1024 threads, bitonic sort in shared memory (C <= 4096), ties by index.
__device__ __forceinline__ void d_uni_sort_cands(const double* __restrict__ xT, int C, const ColMeta* __restrict__ cols, double* __restrict__ xs,
                 int32_t* __restrict__ cidx) {
  __shared__ double sv[4096];
  __shared__ int32_t si[4096];
  const ColMeta cm = cols[0];
  const double ctr = TPE_MUL(0.5, TPE_ADD(cm.klow, cm.khigh));
  int m2 = 32;
  while (m2 < C) m2 <<= 1;
  for (int i = threadIdx.x; i < m2; i += 1024) {
    sv[i] = (i < C) ? xT[i] - ctr : INFINITY;
    si[i] = (i < C) ? i : 0x7fffffff;
  }
  __syncthreads();
  for (int k = 2; k <= m2; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < m2; i += 1024) {
        const int l = i ^ j;
        if (l > i) {
          const double a = sv[i], b = sv[l];
          const int ia = si[i], ib = si[l];
          const bool a_gt_b = (a > b) || (a == b && ia > ib) || (a != a && b == b);
          const bool up = (i & k) == 0;
          if (up ? a_gt_b : !a_gt_b) {
            sv[i] = b; sv[l] = a;
            si[i] = ib; si[l] = ia;
          }
        }
      }
      __syncthreads();
    }
  }
  for (int i = threadIdx.x; i < m2; i += 1024) {
    if (i < ((C + 31) & ~31)) {
      xs[i] = (i < C) ? sv[i] : NAN;   // padding lanes of the last warp: never pass a test
      cidx[i] = (i < C) ? si[i] : -1;
    }
  }
}
__global__ void __launch_bounds__(1024, 1)
k_uni_sort_cands(const double* __restrict__ xT, int C, const ColMeta* __restrict__ cols, double* __restrict__ xs,
                 int32_t* __restrict__ cidx) { d_uni_sort_cands(xT, C, cols, xs, cidx); }

// part[cidx] = (reference, sum of e^(L - reference)) of the 1-D mixture for every candidate.
// CTA = 8 warps on the SAME 32 neighbouring candidates (lane = candidate): warp w takes the tiles at distance
// w, w + 8, ... on either side of the tile under the candidates.  Every lane sums e^(L - ref) against a FIXED
// reference (its largest term in the tile under it: within a few nats of its true max), so the exponentials of
// different kernels do not depend on each other: four kernels are evaluated at a time on four accumulators (the
// fp64 polynomial chains interleave), and the eight partial sums add up in a fixed order.  A term 600 nats above
// the reference moves it (exact, never seen on real data).  Every term within `skip` of the running max is
// evaluated in fp64 -- there is no fp32 tier here; pairs and whole tiles that cannot reach that window are
// dismissed by the two rigorous bounds described at the top of this file.
constexpr int kUniWarps = 8;
__device__ __forceinline__ void d_uni_grid(const float4* __restrict__ s32, const double2* __restrict__ smi, const double* __restrict__ sc,
           const UniTileMeta* __restrict__ meta, int64_t K, const double* __restrict__ xs,
           const int32_t* __restrict__ cidx, int C, double lse_skip, double2* __restrict__ part,
           const int32_t* __restrict__ tlist) {
  __shared__ double s_ref[kUniWarps][32];
  __shared__ double s_sum[kUniWarps][32];
  // one staged tile per warp: the three table slices are fetched with 10 independent coalesced loads per lane
  // (the latency is paid once per tile, not once per kernel) and then read back as broadcasts
  __shared__ __align__(16) float4 t_32[kUniWarps][kUniTile];
  __shared__ __align__(16) double2 t_mi[kUniWarps][kUniTile];
  __shared__ double t_c[kUniWarps][kUniTile];
  __shared__ double s_e64[64];
  if (threadIdx.x < 64) s_e64[threadIdx.x] = exp2((double)threadIdx.x * 0.015625);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int i = blockIdx.x * 32 + lane;      // sorted position of this lane's candidate
  const double x = xs[i];                    // NaN for the padding lanes of the last group
  const bool live = x == x;
  const float xf = __double2float_rn(x);
  const int ntiles = (int)((K + kUniTile - 1) / kUniTile);
  const unsigned valid = __ballot_sync(0xffffffffu, live);
  const double xlo = __shfl_sync(0xffffffffu, x, __ffs(valid) - 1);
  const double xhi = __shfl_sync(0xffffffffu, x, 31 - __clz(valid));
  const double skip = lse_skip;
  // the tile under the candidates
  int tstart = 0;
  {
    int lo = 0, hi = ntiles - 1;             // first tile whose mu range does not lie entirely below xlo
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (meta[mid].mu_hi < xlo) lo = mid + 1; else hi = mid;
    }
    tstart = lo;
  }
  // reference: the largest term of that tile (all 8 warps: 16 kernels each)
  {
    double mx = -INFINITY;
    const int64_t j0 = (int64_t)tstart * kUniTile + warp * (kUniTile / kUniWarps);
    for (int q = 0; q < kUniTile / kUniWarps; ++q) {
      const double2 mi = __ldg(smi + j0 + q);
      const double tt = fma(x, mi.y, -mi.x);
      const double L = fma(-0.5 * tt, tt, __ldg(sc + j0 + q));
      mx = (L > mx) ? L : mx;
    }
    s_ref[warp][lane] = mx;
  }
  __syncthreads();
  double ref = s_ref[0][lane];
#pragma unroll
  for (int w = 1; w < kUniWarps; ++w) ref = fmax(ref, s_ref[w][lane]);
  __syncthreads();                           // s_ref is written again at the end (a warp without tiles gets there at once)
  if (!(ref > -INFINITY)) ref = -INFINITY;   // an all-padding tile cannot happen for tstart; NaN x stays dead
  double mrun = ref;                         // lower bound of the candidate's max (it IS one of its terms)
  float thrf = __double2float_rd(mrun - skip);
  double acc[4] = {0.0, 0.0, 0.0, 0.0};

  auto do_tile = [&](int t) {
    const int64_t j0 = (int64_t)t * kUniTile;
    __syncwarp();                            // the previous tile has been consumed
#pragma unroll
    for (int q = lane; q < kUniTile; q += 32) {
      t_32[warp][q] = __ldg(s32 + j0 + q);
      t_mi[warp][q] = __ldg(smi + j0 + q);
      t_c[warp][q] = __ldg(sc + j0 + q);
    }
    __syncwarp();
    for (int q = 0; q < kUniTile; q += 4) {
      bool pass[4];
      bool any = false;
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const float4 v = t_32[warp][q + u];
        const float tf = fmaf(xf, v.y, -v.x);
        const float Lf = fmaf(-0.5f * tf, tf, v.z);
        const float ub = fmaf(fabsf(tf) + 1.0f, v.w, Lf) + 2.5e-7f * (fabsf(v.z) + fabsf(Lf));
        pass[u] = !(ub < thrf) && live && v.z > -INFINITY;   // cannot be dismissed in fp32 (-inf: muted / padding)
        any = any || pass[u];
      }
      if (!__any_sync(0xffffffffu, any)) continue;
      double L[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const double2 mi = t_mi[warp][q + u];
        const double tt = fma(x, mi.y, -mi.x);
        L[u] = fma(-0.5 * tt, tt, t_c[warp][q + u]);
      }
      double big = fmax(fmax(L[0], L[1]), fmax(L[2], L[3]));
      big = live ? big : -INFINITY;
      if (__any_sync(0xffffffffu, big > ref + 600.0)) {   // never on real data: keep the sums finite
        if (big > ref + 600.0) {
          const double sc2 = uni_exp(fmax(ref - big, -700.0), s_e64);
#pragma unroll
          for (int u = 0; u < 4; ++u) acc[u] *= sc2;
          ref = big;
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const double d = L[u] - mrun;
        const bool take = pass[u] && d > -skip;            // L = -inf (padding), NaN: compare false
        // a term taken against the OLD running max may lie far below a reference this very group has just moved
        const double e = uni_exp(take ? fmax(L[u] - ref, -700.0) : 0.0, s_e64);
        acc[u] += take ? e : 0.0;
      }
      if (big > mrun) {
        mrun = big;
        thrf = __double2float_rd(mrun - skip);
      }
    }
  };
  // tlist != nullptr: only the listed tiles hold kernels this kernel evaluates (ascending; the tile under the
  // candidates comes first in any case: the running maxima start there)
  const int nlist = tlist != nullptr ? tlist[0] : 0;
  const int nwalk = tlist != nullptr ? nlist + 1 : ntiles;
  for (int dt = warp; dt < nwalk; dt += kUniWarps) {
    for (int side = 0; side < (tlist != nullptr ? 1 : 2); ++side) {
      int t;
      if (tlist != nullptr) {
        t = dt == 0 ? tstart : tlist[dt];
        if (dt != 0 && t == tstart) continue;
      } else {
        t = side == 0 ? tstart + dt : tstart - 1 - dt;
      }
      if (t < 0 || t >= ntiles) continue;
      if (t != tstart) {
        const UniTileMeta tm = meta[t];
        // L <= cmax - (dist / smax)^2 / 2 for every kernel of the tile and every candidate of the warp
        const double dist = fmax(fmax(tm.mu_lo - xhi, xlo - tm.mu_hi), 0.0) * (1.0 - 1e-12);
        const double z = dist / tm.smax;
        const double ub = tm.cmax - 0.5 * z * z + 1e-9;
        double thr = live ? mrun - skip : INFINITY;   // against the LOWEST threshold of the warp
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) thr = fmin(thr, __shfl_xor_sync(0xffffffffu, thr, o));
        if (ub < thr) continue;
      }
      do_tile(t);
    }
  }
  // the eight partial sums refer to (possibly) different references only if one was moved: bring them to the largest
  s_ref[warp][lane] = ref;
  s_sum[warp][lane] = (acc[0] + acc[1]) + (acc[2] + acc[3]);
  __syncthreads();
  if (warp == 0 && live) {
    double r = s_ref[0][lane];
#pragma unroll
    for (int w = 1; w < kUniWarps; ++w) r = fmax(r, s_ref[w][lane]);
    double tot = 0.0;
#pragma unroll
    for (int w = 0; w < kUniWarps; ++w) {
      const double rw = s_ref[w][lane];
      tot += (rw == r) ? s_sum[w][lane] : s_sum[w][lane] * uni_exp(fmax(rw - r, -700.0), s_e64);
    }
    part[cidx[i]] = (r > -INFINITY) ? make_double2(r, tot) : make_double2(-INFINITY, 0.0);
  }
}
__global__ void __launch_bounds__(kUniWarps * 32)
k_uni_grid(const float4* __restrict__ s32, const double2* __restrict__ smi, const double* __restrict__ sc,
           const UniTileMeta* __restrict__ meta, int64_t K, const double* __restrict__ xs,
           const int32_t* __restrict__ cidx, int C, double lse_skip, double2* __restrict__ part,
           const int32_t* __restrict__ tlist) { d_uni_grid(s32, smi, sc, meta, K, xs, cidx, C, lse_skip, part, tlist); }

}  // namespace tpe
