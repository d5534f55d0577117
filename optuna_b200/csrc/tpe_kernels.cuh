// CUDA kernels of the TPE suggestion path (sm_90a).  Host orchestration lives in tpe_capi.cu.
//
// Stage map (reference file:line each kernel replaces):
//   k_rowok / k_split_coop   optuna/samplers/_tpe/sampler.py:511-521, :686-722, :735-742, :782-821
//   k_build_mv / k_mu / k_sigma_* / k_const / k_wraw..k_wnorm / k_cat_tables
//                            optuna/samplers/_tpe/parzen_estimator.py:39-78, :132-251
//   k_sample                 optuna/samplers/_tpe/probability_distributions.py:86-152
//   k_logpdf_mma (fp64 tensor-core grid, multivariate) / k_logpdf_fast (DFMA grid) /
//   k_logpdf_pairs + k_disc_tables (mixed spaces) / k_logpdf_generic / k_logpdf_prior_fix
//                            optuna/samplers/_tpe/probability_distributions.py:154-223,
//                            optuna/samplers/_tpe/_truncnorm.py:286-297
//   k_mt19937_uniform        numpy RandomState.random_sample as drawn in probability_distributions.py:87,100,138-144
//   k_select                 optuna/samplers/_tpe/sampler.py:591-618
#pragma once
#include <cooperative_groups.h>

#include <type_traits>

#include "tpe_common.cuh"
#include "tpe_math.cuh"
#include "mt_jump_table.inc"

namespace tpe {

// ================================================================================================
// split
// ================================================================================================
__global__ void k_rowok(const double* __restrict__ X, int64_t n, int32_t pall, const ColMeta* __restrict__ cols,
                        int32_t pc, uint8_t* __restrict__ ok) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    bool good = true;
    for (int j = 0; j < pc; ++j) {
      const double v = X[i * pall + cols[j].src];
      good = good && (v == v);
    }
    ok[i] = good ? 1 : 0;
  }
}

// counts written by the split: [0] |below| before the row filter, [1] below observations, [2] above observations
// ------------------------------------------------------------------------------------------------
// Multi-CTA split (cooperative launch): the same selection as k_split, spread over the whole GPU.
// No candidate lists: every radix pass re-scans the (tiny: 17 B/trial) key arrays with all CTAs and
// histograms the next byte of the trials that still match the 128-bit prefix; grid.sync() between
// passes.  Ordered (stable) outputs come from per-CTA contiguous chunks + a prefix over CTA counts.
// ------------------------------------------------------------------------------------------------
struct SplitWork {        // global scratch, zeroed by the host before the launch
  int cat_count[4];       // trials per category
  int hist[16][256];      // one histogram per radix pass
  int cta_tie[1024];      // per-CTA number of boundary ties
  int cta_cnt[1024][3];   // per-CTA (below_all, below_ok, above_ok)
};

__device__ __forceinline__ void key_u128(const double* __restrict__ key, int i, uint64_t& hi, uint64_t& lo) {
  hi = order_bits(key[2 * (int64_t)i]);
  lo = order_bits(key[2 * (int64_t)i + 1]);
}
// keep the top `nb` bytes of a 128-bit value
__device__ __forceinline__ void top_bytes(int nb, uint64_t& hi, uint64_t& lo) {
  if (nb <= 0) { hi = 0; lo = 0; }
  else if (nb < 8) { hi &= ~0ull << (8 * (8 - nb)); lo = 0; }
  else if (nb == 8) { lo = 0; }
  else if (nb < 16) { lo &= ~0ull << (8 * (16 - nb)); }
}

__global__ void __launch_bounds__(512, 1)
k_split_coop(int n, const int8_t* __restrict__ cat, const double* __restrict__ key, int64_t n_below,
             const uint8_t* __restrict__ row_ok, const uint8_t* __restrict__ pre_member, SplitWork* __restrict__ wk,
             int64_t* __restrict__ below_rows,
             int64_t* __restrict__ below_pos, int64_t* __restrict__ above_rows, int64_t* __restrict__ counts,
             int64_t* __restrict__ below_all_rows /* every below trial, also those lacking a selected parameter
                                                    (the multi-objective weights are computed over all of them) */) {
  cooperative_groups::grid_group grid = cooperative_groups::this_grid();
  __shared__ int s_hist[256];
  __shared__ int s_pick[3];
  __shared__ int s_warp[32];
  __shared__ int s_base[4];
  const int tid = threadIdx.x;
  const int G = gridDim.x, b = blockIdx.x;
  const int chunk = (n + G - 1) / G;
  const int lo_i = min(n, b * chunk), hi_i = min(n, lo_i + chunk);

  // ---- category sizes ---------------------------------------------------------------------------
  if (tid < 4) s_base[tid] = 0;
  __syncthreads();
  for (int i = lo_i + tid; i < hi_i; i += blockDim.x) {
    const int c = cat[i];
    if (c >= 0 && c <= 3) atomicAdd(&s_base[c], 1);  // TPE_CAT_EXCLUDED rows belong to neither set
  }
  __syncthreads();
  if (tid < 4 && s_base[tid]) atomicAdd(&wk->cat_count[tid], s_base[tid]);
  grid.sync();

  // which category holds the cut?  (earlier ones are entirely below, later ones entirely above)
  // pre_member != nullptr: the COMPLETE group was selected elsewhere (multi-objective split); n_below
  // is what is left for the PRUNED / infeasible groups.
  int64_t remaining = n_below < 0 ? 0 : n_below;
  int thr_cat = 3, need = 0;
  for (int c = (pre_member != nullptr ? 1 : 0); c < 3; ++c) {
    const int cnt = wk->cat_count[c];
    if (remaining >= cnt) { remaining -= cnt; continue; }
    thr_cat = c;
    need = (int)remaining;
    break;
  }
  // categories < thr_cat: all below; == thr_cat: the `need` smallest keys; > thr_cat: above.
  uint64_t p_hi = 0, p_lo = 0;  // selected key prefix
  int nb = 0;                   // number of leading bytes of the prefix that are fixed
  bool take_all_eq = false;     // every trial equal to the prefix on `nb` bytes is below
  if (thr_cat < 3 && need > 0) {
    for (int d = 15; d >= 0; --d) {
      for (int t = tid; t < 256; t += blockDim.x) s_hist[t] = 0;
      __syncthreads();
      for (int i = lo_i + tid; i < hi_i + ((32 - ((hi_i - lo_i) & 31)) & 31); i += blockDim.x) {
        bool v = i < hi_i && cat[i] == thr_cat;
        int dg = -1 - (tid & 31);
        if (v) {
          uint64_t h, l, mh, ml;
          key_u128(key, i, h, l);
          mh = h; ml = l;
          top_bytes(15 - d, mh, ml);
          v = (mh == p_hi && ml == p_lo);
          if (v) dg = (int)(((d >= 8 ? h : l) >> ((d & 7) * 8)) & 0xffull);
        }
        const unsigned peers = __match_any_sync(0xffffffffu, dg);
        if (v && (__ffs(peers) - 1) == (tid & 31)) atomicAdd(&s_hist[dg], __popc(peers));
      }
      __syncthreads();
      for (int t = tid; t < 256; t += blockDim.x)
        if (s_hist[t]) atomicAdd(&wk->hist[d][t], s_hist[t]);
      grid.sync();
      if (tid == 0) {
        int cum = 0, q = 0;
        for (; q < 256; ++q) {
          const int hq = wk->hist[d][q];
          if (cum + hq >= need) break;
          cum += hq;
        }
        s_pick[0] = q;
        s_pick[1] = cum;
        s_pick[2] = wk->hist[d][q];
      }
      __syncthreads();
      const int D = s_pick[0], less = s_pick[1], eq = s_pick[2];
      __syncthreads();
      if (d >= 8) p_hi |= (uint64_t)D << ((d & 7) * 8);
      else p_lo |= (uint64_t)D << ((d & 7) * 8);
      nb = 16 - d;
      need -= less;
      if (need == eq) { take_all_eq = true; break; }
    }
  }
  // classification of trial i: 2 = below, 1 = boundary tie (identical 128-bit key), 0 = above
  auto classify = [&](int i) -> int {
    const int c = cat[i];
    if (c == 0 && pre_member != nullptr) return pre_member[i] ? 2 : 0;
    if (c >= 3 || c < 0 || c > thr_cat) return 0;
    if (c < thr_cat) return 2;
    if (need <= 0 && !take_all_eq) return 0;
    uint64_t h, l;
    key_u128(key, i, h, l);
    top_bytes(nb, h, l);
    if (h < p_hi || (h == p_hi && l < p_lo)) return 2;
    if (h == p_hi && l == p_lo) return take_all_eq ? 2 : 1;
    return 0;
  };
  const bool have_ties = (thr_cat < 3) && !take_all_eq && need > 0;  // nb == 16 here

  // ---- ordered partition ------------------------------------------------------------------------------
  // pass A: boundary ties per CTA (earliest trials win, sampler.py stable sort)
  int tie_before = 0;
  if (have_ties) {
    int mine = 0;
    for (int i = lo_i + tid; i < hi_i; i += blockDim.x) mine += classify(i) == 1;
    for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
    if ((tid & 31) == 0) s_warp[tid >> 5] = mine;
    __syncthreads();
    if (tid == 0) {
      int t = 0;
      for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += s_warp[w];
      wk->cta_tie[b] = t;
    }
    grid.sync();
    for (int q = 0; q < b; ++q) tie_before += wk->cta_tie[q];
  }
  // pass B: per-CTA counts with tie membership resolved; pass C: write.  Both walk the chunk in
  // tiles of blockDim with an ordered block scan.
  auto walk = [&](bool write, int base_all, int base_b, int base_a) {
    int tie_seen = tie_before, nb_all = base_all, nbo = base_b, nao = base_a;
    for (int t0 = lo_i; t0 < hi_i; t0 += blockDim.x) {
      const int i = t0 + tid;
      const bool v = i < hi_i;
      const int cls = v ? classify(i) : 0;
      const bool ok = v && (row_ok == nullptr || row_ok[i] != 0) && (unsigned)cat[i] <= 3u;
      // ordered rank helpers (512 threads = 16 warps)
      auto rank = [&](bool f, int& total) -> int {
        const unsigned m = __ballot_sync(0xffffffffu, f);
        const int lane = tid & 31, w = tid >> 5;
        const int wpos = __popc(m & ((1u << lane) - 1u));
        __syncthreads();
        if (lane == 0) s_warp[w] = __popc(m);
        __syncthreads();
        int vv = (lane < (int)(blockDim.x >> 5)) ? s_warp[lane] : 0, incl = vv;
        for (int o = 1; o < 32; o <<= 1) {
          const int t = __shfl_up_sync(0xffffffffu, incl, o);
          if (lane >= o) incl += t;
        }
        total = __shfl_sync(0xffffffffu, incl, 31);
        return __shfl_sync(0xffffffffu, incl - vv, w) + wpos;
      };
      int tot_t = 0, tot_all = 0, tot_b = 0, tot_a = 0;
      bool isb = cls == 2;
      if (have_ties) {
        const int tr = rank(cls == 1, tot_t);
        if (cls == 1 && tie_seen + tr < need) isb = true;
        tie_seen += tot_t;
      }
      const int r_all = rank(isb, tot_all);
      const int r_b = rank(isb && ok, tot_b);
      const int r_a = rank(v && !isb && ok, tot_a);
      if (write) {
        if (isb && below_all_rows != nullptr) below_all_rows[nb_all + r_all] = i;
        if (isb && ok) {
          below_rows[nbo + r_b] = i;
          below_pos[nbo + r_b] = nb_all + r_all;
        }
        if (v && !isb && ok) above_rows[nao + r_a] = i;
      }
      nb_all += tot_all;
      nbo += tot_b;
      nao += tot_a;
    }
    if (!write && tid == 0) {
      wk->cta_cnt[b][0] = nb_all;
      wk->cta_cnt[b][1] = nbo;
      wk->cta_cnt[b][2] = nao;
    }
  };
  walk(false, 0, 0, 0);
  grid.sync();
  int base[3] = {0, 0, 0};
  for (int q = 0; q < b; ++q)
    for (int e = 0; e < 3; ++e) base[e] += wk->cta_cnt[q][e];
  walk(true, base[0], base[1], base[2]);
  if (b == G - 1 && tid == 0) {
    counts[0] = base[0] + wk->cta_cnt[b][0];
    counts[1] = base[1] + wk->cta_cnt[b][1];
    counts[2] = base[2] + wk->cta_cnt[b][2];
  }
}

// ================================================================================================
// Parzen-estimator build
// ================================================================================================
// mu[k][j] for the n observation kernels and the prior kernel (k = n).  Categorical columns store
// the observed choice index (prior: nch).
__device__ __forceinline__ void d_mu(const double* __restrict__ X, int32_t pall, const int64_t* __restrict__ rows, int64_t n,
                     const ColMeta* __restrict__ cols, int32_t pc, double* __restrict__ mu) {
  const int64_t total = (n + 1) * pc;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t k = t / pc;
    const int j = (int)(t - k * pc);
    const ColMeta cm = cols[j];
    double v;
    if (k < n) {
      v = X[rows[k] * pall + cm.src];
      if (cm.cls != COL_CAT && cm.log) v = log(v);
    } else {
      v = (cm.cls == COL_CAT) ? (double)cm.nch : TPE_MUL(0.5, TPE_ADD(cm.klow, cm.khigh));
    }
    mu[t] = v;
  }
}
__global__ void
k_mu(const double* __restrict__ X, int32_t pall, const int64_t* __restrict__ rows, int64_t n,
                     const ColMeta* __restrict__ cols, int32_t pc, double* __restrict__ mu) { d_mu(X, pall, rows, n, cols, pc, mu); }

// Bandwidth limits of parzen_estimator.py:220-228.
__device__ __forceinline__ void sigma_limits(const ColMeta& cm, int64_t n, bool magic_clip, double& lo, double& hi) {
  hi = TPE_SUB(cm.khigh, cm.klow);
  if (magic_clip) {
    const double kk = 1.0 + (double)(n + 1);
    lo = TPE_DIV(hi, kk < 100.0 ? kk : 100.0);
  } else {
    lo = 1e-12;
  }
}

// multivariate: sigma = 0.2 * max(n,1)^(-1/(d+4)) * (high-low), clipped; prior: high-low.
__global__ void k_sigma_mv(const ColMeta* __restrict__ cols, int32_t pc, int64_t n, int magic_clip,
                           double* __restrict__ sigma) {
  const int64_t total = (n + 1) * pc;
  // the bandwidth factor is the same for every cell: one pow() per thread, not per cell
  const double e = TPE_DIV(-1.0, (double)(pc + 4));
  const double factor = TPE_MUL(0.2, pow((double)(n > 1 ? n : 1), e));
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t k = t / pc;
    const int j = (int)(t - k * pc);
    const ColMeta cm = cols[j];
    if (cm.cls == COL_CAT) {
      sigma[t] = 0.0;
      continue;
    }
    double lo, hi;
    sigma_limits(cm, n, magic_clip != 0, lo, hi);
    sigma[t] = (k == n) ? hi : fmin(fmax(TPE_MUL(factor, hi), lo), hi);
  }
}

// univariate: neighbour gaps in the sorted order of mu U {prior mu} (parzen_estimator.py:196-218).
// order[j] = index (0..n, n = prior) of the j-th smallest value of column `j_col`.
__device__ __forceinline__ void d_sigma_uni(const double* __restrict__ mu, const int32_t* __restrict__ order,
                            const ColMeta* __restrict__ cols, int32_t pc, int j_col, int64_t n, int magic_clip,
                            int endpoints, double* __restrict__ sigma) {
  const ColMeta cm = cols[j_col];
  double lo, hi;
  sigma_limits(cm, n, magic_clip != 0, lo, hi);
  const int64_t m = n + 1;  // sorted length
  for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j < m; j += (int64_t)gridDim.x * blockDim.x) {
    const int64_t me = order[j];
    const double v = mu[me * pc + j_col];
    const double left = j == 0 ? cm.klow : mu[(int64_t)order[j - 1] * pc + j_col];
    const double right = j == m - 1 ? cm.khigh : mu[(int64_t)order[j + 1] * pc + j_col];
    double g = fmax(TPE_SUB(v, left), TPE_SUB(right, v));
    if (!endpoints && m >= 2) {
      if (j == 0) g = TPE_SUB(right, v);
      if (j == m - 1) g = TPE_SUB(v, left);
    }
    g = fmin(fmax(g, lo), hi);
    sigma[me * pc + j_col] = (me == n) ? hi : g;
  }
}
__global__ void
k_sigma_uni(const double* __restrict__ mu, const int32_t* __restrict__ order,
                            const ColMeta* __restrict__ cols, int32_t pc, int j_col, int64_t n, int magic_clip,
                            int endpoints, double* __restrict__ sigma) { d_sigma_uni(mu, order, cols, pc, j_col, n, magic_clip, endpoints, sigma); }

// Stable LSD radix sort of one estimator column (cooperative launch, 8 passes of 8 bits) for the
// univariate bandwidths: order[j] = index of the j-th smallest (value, index).  Each CTA owns a
// contiguous chunk; per pass: chunk histogram -> grid.sync -> global digit offsets (digit-major,
// CTA-minor) -> stable scatter by warp match + per-warp digit counts.  Ping-pong buffers.
struct SortWork {
  int hist[256][160];  // [digit][cta]
};
__device__ __forceinline__ void d_radix_sort_coop(const double* __restrict__ mu, int32_t pc, int j_col, int n, uint64_t* __restrict__ key_a,
                  uint64_t* __restrict__ key_b, int32_t* __restrict__ idx_a, int32_t* __restrict__ idx_b,
                  SortWork* __restrict__ wk, int32_t* __restrict__ order, const int* __restrict__ run_flag,
                  const int32_t* __restrict__ perm = nullptr) {
  // run_flag != nullptr: the order may already have been brought up to date incrementally (k_order_update);
  // every CTA reads the same word before the first grid.sync
  if (run_flag != nullptr && *run_flag < 2) return;
  cooperative_groups::grid_group grid = cooperative_groups::this_grid();
  __shared__ int s_hist[256];
  __shared__ int s_base[256];
  __shared__ int s_wcnt[16][256];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int G = gridDim.x, b = blockIdx.x;
  const int chunk = (n + G - 1) / G;
  const int lo = min(n, b * chunk), hi = min(n, lo + chunk);
  // perm != nullptr: sort the rows perm[0, n) (stable in that order), so that sorts by successive columns chain into
  // a lexicographic order
  for (int i = lo + tid; i < hi; i += blockDim.x) {
    const int32_t r = perm != nullptr ? perm[i] : i;
    key_a[i] = order_bits(mu[(int64_t)r * pc + j_col]);
    idx_a[i] = r;
  }
  uint64_t* kin = key_a;
  uint64_t* kout = key_b;
  int32_t* iin = idx_a;
  int32_t* iout = idx_b;
  for (int pass = 0; pass < 8; ++pass) {
    const int shift = pass * 8;
    for (int t = tid; t < 256; t += blockDim.x) s_hist[t] = 0;
    __syncthreads();
    for (int i = lo + tid; i < hi; i += blockDim.x) atomicAdd(&s_hist[(int)((kin[i] >> shift) & 0xff)], 1);
    __syncthreads();
    for (int t = tid; t < 256; t += blockDim.x) wk->hist[t][b] = s_hist[t];
    grid.sync();
    // global offset of this CTA's first element of every digit
    if (tid < 256) {
      int tot = 0, pre = 0;
      for (int c = 0; c < G; ++c) {
        const int v = wk->hist[tid][c];
        if (c < b) pre += v;
        tot += v;
      }
      s_hist[tid] = tot;
      s_base[tid] = pre;
    }
    __syncthreads();
    if (tid == 0) {
      int run = 0;
      for (int d = 0; d < 256; ++d) {
        const int t = s_hist[d];
        s_hist[d] = run;
        run += t;
      }
    }
    __syncthreads();
    if (tid < 256) s_base[tid] += s_hist[tid];
    __syncthreads();
    // stable scatter, 512 elements at a time
    for (int t0 = lo; t0 < hi; t0 += blockDim.x) {
      const int i = t0 + tid;
      const bool v = i < hi;
      for (int t = tid; t < 16 * 256; t += blockDim.x) (&s_wcnt[0][0])[t] = 0;
      __syncthreads();
      const uint64_t kv = v ? kin[i] : 0;
      const int d = v ? (int)((kv >> shift) & 0xff) : -1 - lane;
      const unsigned peers = __match_any_sync(0xffffffffu, d);
      const int rank_w = __popc(peers & ((1u << lane) - 1u));
      if (v && rank_w == 0) s_wcnt[warp][d] = __popc(peers);
      __syncthreads();
      int off = 0;
      if (v) {
        for (int w = 0; w < warp; ++w) off += s_wcnt[w][d];
        const int pos = s_base[d] + off + rank_w;
        kout[pos] = kv;
        iout[pos] = iin[i];
      }
      __syncthreads();
      if (tid < 256) {
        int tot = 0;
        for (int w = 0; w < 16; ++w) tot += s_wcnt[w][tid];
        s_base[tid] += tot;
      }
      __syncthreads();
    }
    grid.sync();
    uint64_t* tk = kin; kin = kout; kout = tk;
    int32_t* ti = iin; iin = iout; iout = ti;
  }
  for (int i = lo + tid; i < hi; i += blockDim.x) order[i] = iin[i];
}
__global__ void __launch_bounds__(512, 1)
k_radix_sort_coop(const double* __restrict__ mu, int32_t pc, int j_col, int n, uint64_t* __restrict__ key_a,
                  uint64_t* __restrict__ key_b, int32_t* __restrict__ idx_a, int32_t* __restrict__ idx_b,
                  SortWork* __restrict__ wk, int32_t* __restrict__ order, const int* __restrict__ run_flag) { d_radix_sort_coop(mu, pc, j_col, n, key_a, key_b, idx_a, idx_b, wk, order, run_flag); }
__global__ void __launch_bounds__(512, 1)
k_radix_sort_coop_perm(const double* __restrict__ mu, int32_t pc, int j_col, int n, uint64_t* __restrict__ key_a,
                       uint64_t* __restrict__ key_b, int32_t* __restrict__ idx_a, int32_t* __restrict__ idx_b,
                       SortWork* __restrict__ wk, int32_t* __restrict__ order, const int32_t* __restrict__ perm) { d_radix_sort_coop(mu, pc, j_col, n, key_a, key_b, idx_a, idx_b, wk, order, nullptr, perm); }

// Incremental maintenance of a column's sorted order between two suggestions (univariate TPE): the above set of the
// next trial is almost always the previous one plus the trial that has just finished.
//   k_rows_delta : mode = 0 rows identical, 1 exactly one row appended at the end, >= 2 anything else (sort again)
//   k_order_update: mode 0 copies the order; mode 1 inserts the new observation (index n_old; the prior kernel moves
//                   from index n_old to n_old + 1) at its place -- every old element shifts by one iff the new key is
//                   smaller (ties by index, like the stable radix sort), the new element lands behind the elements
//                   that did not shift.
__global__ void k_rows_delta(const int64_t* __restrict__ rows_new, const int64_t* __restrict__ rows_old, int64_t n_old,
                             int cand, int* __restrict__ mode /* zeroed */) {
  if (blockIdx.x == 0 && threadIdx.x == 0 && cand) atomicOr(mode, cand);
  if (cand == 2) return;
  bool diff = false;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n_old; i += (int64_t)gridDim.x * blockDim.x)
    diff |= rows_new[i] != rows_old[i];
  if (diff) atomicOr(mode, 2);   // mode >= 2: sort
}
__device__ __forceinline__ void d_order_update(const int* __restrict__ mode, const int32_t* __restrict__ old_order, int K_old, int K_new,
               const double* __restrict__ mu, int32_t* __restrict__ out, int* __restrict__ work) {
  const int m = *mode;
  if (m >= 2) return;
  if (m == 0) {
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < K_old; p += gridDim.x * blockDim.x) out[p] = old_order[p];
    return;
  }
  __shared__ int s_cnt;
  __shared__ bool s_last;
  if (threadIdx.x == 0) s_cnt = 0;
  __syncthreads();
  const int n_old = K_old - 1;                       // index of the new observation (and the prior's old index)
  const uint64_t v = order_bits(mu[n_old]);
  int mine = 0;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < K_old; p += gridDim.x * blockDim.x) {
    const int e = old_order[p];
    const int ne = (e == n_old) ? n_old + 1 : e;
    const uint64_t key = order_bits(mu[ne]);
    const bool shift = (v < key) || (v == key && n_old < ne);
    out[p + (shift ? 1 : 0)] = ne;
    mine += shift ? 0 : 1;
  }
  for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
  if ((threadIdx.x & 31) == 0 && mine) atomicAdd(&s_cnt, mine);
  __syncthreads();
  if (threadIdx.x == 0) {
    if (s_cnt) atomicAdd(&work[0], s_cnt);
    __threadfence();
    s_last = atomicAdd(&work[1], 1) == (int)gridDim.x - 1;
  }
  __syncthreads();
  if (s_last && threadIdx.x == 0) {
    __threadfence();
    out[*reinterpret_cast<volatile int*>(&work[0])] = n_old;
  }
  (void)K_new;
}
__global__ void __launch_bounds__(256)
k_order_update(const int* __restrict__ mode, const int32_t* __restrict__ old_order, int K_old, int K_new,
               const double* __restrict__ mu, int32_t* __restrict__ out, int* __restrict__ work) { d_order_update(mode, old_order, K_old, K_new, mu, out, work); }

// Whole bitonic sort in shared memory for m2 <= 4096 (one CTA of 1024 threads).
__device__ __forceinline__ void d_sort_small(const double* __restrict__ mu, int32_t pc, int j_col, int m, int m2, int32_t* __restrict__ order) {
  __shared__ double sv[4096];
  __shared__ int32_t si[4096];
  for (int i = threadIdx.x; i < m2; i += 1024) {
    if (i < m) {
      double v = mu[(int64_t)i * pc + j_col];
      if (v == 0.0) v = 0.0;
      sv[i] = v;
      si[i] = i;
    } else {
      sv[i] = INFINITY;
      si[i] = 0x7fffffff;
    }
  }
  __syncthreads();
  for (int k = 2; k <= m2; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < m2; i += 1024) {
        const int l = i ^ j;
        if (l > i) {
          const double a = sv[i], b = sv[l];
          const int ia = si[i], ib = si[l];
          const bool a_gt_b = (a > b) || (a == b && ia > ib);
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
  for (int i = threadIdx.x; i < m; i += 1024) order[i] = si[i];
}
__global__ void __launch_bounds__(1024, 1)
k_sort_small(const double* __restrict__ mu, int32_t pc, int j_col, int m, int m2, int32_t* __restrict__ order) { d_sort_small(mu, pc, j_col, m, m2, order); }

// Per-(kernel, column) constants.  One warp per kernel; lanes stride over columns.
//   continuous: c = ln sqrt(2 pi) + M(a, b) + ln sigma      (a, b = normalised support)
//   discrete  : c = M(a, b) over the half-step-extended support
//   cst_part[k] = -sum_j c
// Fast-kernel tables, in coordinates centred on the column midpoint c_p (so that magnitudes are
// bounded by range / sigma and the scaled difference keeps ~1e-15 absolute accuracy, DESIGN.md):
//   mode 1 (PAIR,  sigma varies per kernel): tabp[k][slot] = ((mu - c_p) / sigma_kp, 1 / sigma_kp)
//   mode 2 (CONST, sigma_p shared by all observation kernels -- multivariate TPE):
//                                            tabc[k][slot] = (mu - c_p) / sigma_p   for k < K - 1
//   colprm[slot] = (c_p, 1 / sigma_p) (CONST) or (c_p, 1) (PAIR); padded slots are zero.
__global__ void k_const(const double* __restrict__ mu, const double* __restrict__ sigma,
                        const ColMeta* __restrict__ cols, int32_t pc, int64_t K, int32_t pb, int mode,
                        double2* __restrict__ tabp, double* __restrict__ tabc, double2* __restrict__ colprm,
                        double* __restrict__ cst_part) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t k = warp; k < K; k += nwarps) {
    double acc = 0.0;
    for (int j = lane; j < pc; j += 32) {
      const ColMeta cm = cols[j];
      if (cm.cls == COL_CAT) continue;
      const double m = mu[k * pc + j], s = sigma[k * pc + j];
      const double a = TPE_DIV(TPE_SUB(cm.klow, m), s);
      const double b = TPE_DIV(TPE_SUB(cm.khigh, m), s);
      const double mass = log_gauss_mass_fast(a, b);
      if (cm.cls == COL_CONT) {
        acc += kLogSqrt2Pi + mass + log(s);
        if (mode != 0) {
          const double ctr = TPE_MUL(0.5, TPE_ADD(cm.klow, cm.khigh));
          const double inv = TPE_DIV(1.0, s);
          if (mode == 1) {
            tabp[k * pb + cm.slot] = make_double2(TPE_MUL(TPE_SUB(m, ctr), inv), inv);
            if (k == 0) colprm[cm.slot] = make_double2(ctr, 1.0);
          } else {
            if (k < K - 1) tabc[k * pb + cm.slot] = TPE_MUL(TPE_SUB(m, ctr), inv);
            if (k == 0) colprm[cm.slot] = make_double2(ctr, inv);
          }
        }
      } else {
        acc += mass;
      }
    }
    acc = warp_sum(acc);
    if (lane == 0) cst_part[k] = -acc;
  }
}
// zero the padded slots [ncont, pb) of the fast tables
__global__ void k_tab_pad(double2* __restrict__ tabp, double* __restrict__ tabc, double2* __restrict__ colprm,
                          int64_t rows, int32_t pb, int32_t ncont) {
  const int w = pb - ncont;
  const int64_t total = rows * w;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t k = t / w;
    const int sl = ncont + (int)(t - k * w);
    if (tabp) tabp[k * pb + sl] = make_double2(0.0, 0.0);
    if (tabc) tabc[k * pb + sl] = 0.0;
  }
  if (blockIdx.x == 0)
    for (int sl = ncont + threadIdx.x; sl < pb; sl += blockDim.x) colprm[sl] = make_double2(0.0, 0.0);
}

// Fragment-major layout of the CONST table for the tensor-core kernel (k_logpdf_mma): kernels in
// groups of 8, inside a group the order in which the 32 lanes of a warp read their B fragments of
// mma.m8n8k4 (lane = 4 * (k % 8) + slot % 4 holds B[row = slot % 4][col = k % 8] of k-step slot / 4),
// two k-steps interleaved so that one LDS.128 per lane fetches both.  The pair is also exactly the B fragment
// {b0, b1} of one mma.m16n8k8 over the 8 slots of both k-steps.
__host__ __device__ __forceinline__ int64_t mma_tab_index(int64_t k, int slot, int pb) {
  const int i = slot >> 2;
  const int lane = (int)(k & 7) * 4 + (slot & 3);
  return (k >> 3) * (8 * (int64_t)pb) + ((int64_t)(i >> 1) * 32 + lane) * 2 + (i & 1);
}

// Fused multivariate build: k_mu + k_sigma_mv + k_const in one pass (one warp per kernel, lanes over
// columns).  mode / tables as in k_const.
__global__ void k_build_mv(const double* __restrict__ X, int32_t pall, const int64_t* __restrict__ rows, int64_t n,
                           const ColMeta* __restrict__ cols, int32_t pc, int magic_clip, int32_t pb, int mode,
                           double* __restrict__ mu, double* __restrict__ sigma, double2* __restrict__ tabp,
                           double* __restrict__ tabc, double2* __restrict__ colprm, double* __restrict__ cst_part,
                           int32_t* __restrict__ cls, int* __restrict__ offgrid, double* __restrict__ tabm,
                           double* __restrict__ hb) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t K = n + 1;
  const double e = TPE_DIV(-1.0, (double)(pc + 4));
  const double factor = TPE_MUL(0.2, pow((double)(n > 1 ? n : 1), e));
  for (int64_t k = warp; k < K; k += nwarps) {
    const int64_t row = (k < n) ? rows[k] : 0;
    double acc = 0.0, sq = 0.0;
    for (int j = lane; j < pc; j += 32) {
      const ColMeta cm = cols[j];
      if (cm.cls == COL_CAT) {
        mu[k * pc + j] = (k < n) ? X[row * pall + cm.src] : (double)cm.nch;
        sigma[k * pc + j] = 0.0;
        continue;
      }
      double lo, hi;
      sigma_limits(cm, n, magic_clip != 0, lo, hi);
      const double ctr = TPE_MUL(0.5, TPE_ADD(cm.klow, cm.khigh));
      double m, s;
      if (k < n) {
        m = X[row * pall + cm.src];
        if (cm.grid > 0 && cls != nullptr) {
          // kernel class of a tabulated discrete column = grid index of the observation; the table is
          // only valid if the observation sits on the grid exactly
          const double g = rint(TPE_DIV(TPE_SUB(m, cm.low), cm.step));
          const bool on = g >= 0.0 && g < (double)cm.grid && TPE_ADD(cm.low, TPE_MUL(g, cm.step)) == m;
          cls[k * pc + j] = on ? (int32_t)g : 0;
          if (!on) atomicOr(offgrid, 1);
        }
        if (cm.log) m = log(m);
        s = fmin(fmax(TPE_MUL(factor, hi), lo), hi);
      } else {
        m = ctr;
        s = hi;
      }
      mu[k * pc + j] = m;
      sigma[k * pc + j] = s;
      const double a = TPE_DIV(TPE_SUB(cm.klow, m), s);
      const double b = TPE_DIV(TPE_SUB(cm.khigh, m), s);
      const double mass = log_gauss_mass_fast(a, b);
      if (cm.cls == COL_CONT) {
        acc += kLogSqrt2Pi + mass + log(s);
        if (mode != 0) {
          const double inv = TPE_DIV(1.0, s);
          if (mode == 1) {
            tabp[k * pb + cm.slot] = make_double2(TPE_MUL(TPE_SUB(m, ctr), inv), inv);
            if (k == 0) colprm[cm.slot] = make_double2(ctr, 1.0);
          } else {
            const double t = TPE_MUL(TPE_SUB(m, ctr), inv);
            if (k < K - 1) {
              tabc[k * pb + cm.slot] = t;
              if (tabm != nullptr) {
                tabm[mma_tab_index(k, cm.slot, pb)] = t;
                sq = fma(t, t, sq);
              }
            }
            if (k == 0) colprm[cm.slot] = make_double2(ctr, inv);
          }
        }
      } else {
        acc += mass;
      }
    }
    acc = warp_sum(acc);
    if (lane == 0) cst_part[k] = -acc;
    if (hb != nullptr) {
      sq = warp_sum(sq);
      if (lane == 0) hb[k] = 0.5 * sq;
    }
  }
}

// Mixture weights (parzen_estimator.py:59-69, sampler.py:61-69): raw weights (default ramp computed
// here, or host-evaluated) + per-block partial sums, then normalisation, log-weights, cst and the
// sequential cumulative sum used by rng.choice.
// Partial sums are combined in a fixed order, so the result is deterministic.
__device__ __forceinline__ double raw_weight(const double* __restrict__ w_in, const int64_t* __restrict__ pos,
                                             int64_t n, int64_t k, double prior_weight) {
  if (n == 0) return 1.0;
  if (k == n) return prior_weight;
  if (w_in != nullptr) return w_in[pos != nullptr ? pos[k] : k];
  const int64_t nramp = n - 25;
  if (n < 25 || k >= nramp) return 1.0;
  if (k == nramp - 1 && nramp > 1) return 1.0;
  const double start = TPE_DIV(1.0, (double)n);
  const double step = nramp > 1 ? TPE_DIV(TPE_SUB(1.0, start), (double)(nramp - 1)) : 0.0;
  return TPE_ADD(TPE_MUL((double)k, step), start);
}
__global__ void __launch_bounds__(256)
k_wraw(const double* __restrict__ w_in, const int64_t* __restrict__ pos, int64_t n, double prior_weight,
       double* __restrict__ w, double* __restrict__ part) {
  __shared__ double s_red[8];
  const int64_t K = n + 1;
  const int64_t chunk = (K + gridDim.x - 1) / gridDim.x;
  const int64_t lo = blockIdx.x * chunk, hi = (lo + chunk < K) ? lo + chunk : K;
  double acc = 0.0;
  for (int64_t k = lo + threadIdx.x; k < hi; k += blockDim.x) {
    const double r = raw_weight(w_in, pos, n, k, prior_weight);
    w[k] = r;
    acc += r;
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int i = 0; i < 8; ++i) t += s_red[i];
    part[blockIdx.x] = t;
  }
}
__global__ void __launch_bounds__(256)
k_wfinal(const double* __restrict__ part, int nparts, int64_t n, double* __restrict__ w, double* __restrict__ logw,
         const double* __restrict__ cst_part, double* __restrict__ cst, double* __restrict__ cdf, int64_t k_alloc,
         const double* __restrict__ hb, double* __restrict__ ckk) {
  __shared__ double s_total;
  const int64_t K = n + 1;
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int i = 0; i < nparts; ++i) t += part[i];
    s_total = t;
  }
  __syncthreads();
  const double total = s_total;
  if (cdf != nullptr && blockIdx.x == 0 && threadIdx.x == 0) {
    // cumsum(w / total) / last, sequential like numpy.cumsum (rng.choice, probability_distributions.py:87)
    double run = 0.0;
    for (int64_t k = 0; k < K; ++k) {
      run = TPE_ADD(run, TPE_DIV(w[k], total));
      cdf[k] = run;
    }
    const double last = run;
    for (int64_t k = 0; k < K; ++k) cdf[k] = TPE_DIV(cdf[k], last);
  }
  __syncthreads();
  for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < k_alloc; k += (int64_t)gridDim.x * blockDim.x) {
    if (k < K) {
      if (cdf != nullptr && blockIdx.x == 0) {
        // block 0 normalises its own elements only after thread 0 has read the raw values (sync above)
      }
      const double v = TPE_DIV(w[k], total);
      const double lw = log(v);
      logw[k] = lw;
      const double c = cst_part[k] + lw;
      cst[k] = c;
      // tensor-core kernel: constant of the expanded square, cst - |mu''|^2 / 2 (prior kernel excluded)
      if (ckk != nullptr) ckk[k] = (k < K - 1) ? c - hb[k] : -INFINITY;
    } else {
      cst[k] = -INFINITY;  // padding read by the bulk copies
      if (ckk != nullptr) ckk[k] = -INFINITY;
    }
  }
}
// w is kept raw by k_wfinal (other blocks may still read it); this pass stores the normalised values.
__global__ void k_wnorm(const double* __restrict__ part, int nparts, int64_t K, double* __restrict__ w) {
  __shared__ double s_total;
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int i = 0; i < nparts; ++i) t += part[i];
    s_total = t;
  }
  __syncthreads();
  const double total = s_total;
  for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < K; k += (int64_t)gridDim.x * blockDim.x)
    w[k] = TPE_DIV(w[k], total);
}

// Categorical kernel rows (parzen_estimator.py:132-166): the row of kernel k depends only on its
// observed choice, so a column needs (nch + 1) distinct rows (last = prior kernel).
// tab layout per column: W[(nch+1) x nch] followed by lnW[(nch+1) x nch].
__global__ void k_cat_tables(const ColMeta* __restrict__ cols, int32_t pc, int64_t n, double prior_weight,
                             const double* __restrict__ cat_dist, double* __restrict__ tab) {
  const int j = blockIdx.x;
  const ColMeta cm = cols[j];
  if (cm.cls != COL_CAT) return;
  const int c = cm.nch;
  double* W = tab + cm.tab_off;
  double* LW = W + (int64_t)(c + 1) * c;
  const double K = (double)(n + 1);
  for (int r = threadIdx.x; r <= c; r += blockDim.x) {
    double* row = W + (int64_t)r * c;
    if (n == 0) {
      for (int i = 0; i < c; ++i) row[i] = TPE_DIV(1.0, (double)c);
    } else {
      const double base = TPE_DIV(prior_weight, K);
      if (r < c && cm.dist_off >= 0) {
        const double* d = cat_dist + cm.dist_off + (int64_t)r * c;
        double dmax = d[0];
        for (int i = 1; i < c; ++i) dmax = fmax(dmax, d[i]);
        const double coef = TPE_DIV(TPE_MUL(log(TPE_DIV(K, prior_weight)), log((double)c)), log(6.0));
        for (int i = 0; i < c; ++i) {
          const double q = TPE_DIV(d[i], dmax);
          row[i] = exp(TPE_MUL(-TPE_MUL(q, q), coef));
        }
      } else {
        for (int i = 0; i < c; ++i) row[i] = (i == r) ? TPE_ADD(base, 1.0) : base;
      }
      double tot = np_pairwise_sum(row, c);
      if (tot == 0.0) tot = 1.0;
      for (int i = 0; i < c; ++i) row[i] = TPE_DIV(row[i], tot);
    }
    for (int i = 0; i < c; ++i) LW[(int64_t)r * c + i] = log(row[i]);
  }
}

// ================================================================================================
// candidate sampling from l(x)
// ================================================================================================
// One thread per (candidate, column).  S[ct][j] = sampled value (internal representation),
// xT[slot][ct] = kernel-space value of continuous columns (ln x for log columns) for the fast
// log-density kernel, oob[ct] = 1 if a continuous value left [low, high] through rounding.
__device__ __forceinline__ void d_sample(const double* __restrict__ U, int64_t n_asks, int32_t C, const ColMeta* __restrict__ cols,
                         int32_t pc, int32_t ncat, int32_t nnum, const double* __restrict__ cdf, int64_t Kb,
                         const double* __restrict__ mu, const double* __restrict__ sigma,
                         const double* __restrict__ tab, double* __restrict__ S, double* __restrict__ xT,
                         int64_t ct_stride, uint8_t* __restrict__ oob) {
  const int64_t total = n_asks * C * pc;
  const int64_t per_ask = (int64_t)C * (1 + ncat + nnum);
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t ct = t / pc;
    const int j = (int)(t - ct * pc);
    const int64_t ask = ct / C;
    const int c = (int)(ct - ask * C);
    const double* Ua = U + ask * per_ask;
    // active kernel: cdf.searchsorted(u, side="right")
    const double u0 = Ua[c];
    int64_t lo = 0, hi = Kb;
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      if (u0 < cdf[mid]) hi = mid; else lo = mid + 1;
    }
    const int64_t k = lo < Kb ? lo : Kb - 1;
    const ColMeta cm = cols[j];
    double out;
    if (cm.cls == COL_CAT) {
      const double u = Ua[(int64_t)C * (1 + cm.cat_rank) + c];
      const int nch = cm.nch;
      const int row = (k == Kb - 1) ? nch : (int)mu[k * pc + j];
      const double* w = tab + cm.tab_off + (int64_t)row * nch;
      double run = 0.0;
      int cnt = 0;
      for (int i = 0; i < nch; ++i) {
        run = TPE_ADD(run, w[i]);
        const double cp = (i == nch - 1) ? 1.0 : run;
        cnt += (cp < u) ? 1 : 0;
      }
      out = (double)cnt;
    } else {
      const double u = Ua[(int64_t)C * (1 + ncat) + (int64_t)cm.num_rank * C + c];
      const double m = mu[k * pc + j], s = sigma[k * pc + j];
      const double a = TPE_DIV(TPE_SUB(cm.klow, m), s);
      const double b = TPE_DIV(TPE_SUB(cm.khigh, m), s);
      double x = TPE_ADD(TPE_MUL(trunc_ppf(u, a, b), s), m);
      if (cm.log) x = exp(x);
      if (cm.cls == COL_DISC) {
        x = TPE_ADD(cm.low, TPE_MUL(rint(TPE_DIV(TPE_SUB(x, cm.low), cm.step)), cm.step));
        x = fmin(fmax(x, cm.low), cm.high);
      } else {
        if (xT != nullptr) xT[(int64_t)cm.slot * ct_stride + ct] = cm.log ? log(x) : x;
        if (!(x >= cm.low && x <= cm.high)) oob[ct] = 1;
      }
      out = x;
    }
    S[ct * pc + j] = out;
  }
}
__global__ void
k_sample(const double* __restrict__ U, int64_t n_asks, int32_t C, const ColMeta* __restrict__ cols,
                         int32_t pc, int32_t ncat, int32_t nnum, const double* __restrict__ cdf, int64_t Kb,
                         const double* __restrict__ mu, const double* __restrict__ sigma,
                         const double* __restrict__ tab, double* __restrict__ S, double* __restrict__ xT,
                         int64_t ct_stride, uint8_t* __restrict__ oob) { d_sample(U, n_asks, C, cols, pc, ncat, nnum, cdf, Kb, mu, sigma, tab, S, xT, ct_stride, oob); }

// For tpe_logpdf on caller-supplied points: fill xT / oob from S.
__global__ void k_prep_points(const double* __restrict__ S, int64_t n, const ColMeta* __restrict__ cols, int32_t pc,
                              double* __restrict__ xT, int64_t ct_stride, uint8_t* __restrict__ oob) {
  const int64_t total = n * pc;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t ct = t / pc;
    const int j = (int)(t - ct * pc);
    const ColMeta cm = cols[j];
    if (cm.cls != COL_CONT) continue;
    const double x = S[t];
    if (xT != nullptr) xT[(int64_t)cm.slot * ct_stride + ct] = cm.log ? log(x) : x;
    if (!(x >= cm.low && x <= cm.high)) oob[ct] = 1;
  }
}

// ================================================================================================
// log-density grid
// ================================================================================================
// Cell-mass tables of the tabulated discrete columns (multivariate TPE: one sigma per column):
//   T[r][g] = M((x_r -+ step/2 - mu_g) / sigma_g),  g = grid index of the kernel's observation (g = G: prior).
// Rows: with fewer candidates than grid values (Ct < G) row r is candidate r (any x, on the grid or
// not); otherwise row r is grid value low + r * step.  One candidate reads one contiguous row of
// G + 1 doubles.  Same expression as the direct evaluation, so identical values.
// grid = (chunks, pc); a block exits at once for a column that is not tabulated.
__global__ void k_disc_tables(const ColMeta* __restrict__ cols, int32_t pc, const double* __restrict__ mu,
                              const double* __restrict__ sigma, int64_t K, const double* __restrict__ S, int64_t Ct,
                              double* __restrict__ dtab) {
  const int j = blockIdx.y;
  const ColMeta cm = cols[j];
  if (cm.cls != COL_DISC || cm.grid <= 0) return;
  const int G = cm.grid;
  const bool by_cand = Ct < G;
  const int64_t total = (by_cand ? Ct : (int64_t)G) * (G + 1);
  const double sg_obs = sigma[j];  // kernel 0 (any observation kernel; unused when K == 1)
  const double mu_prior = mu[(K - 1) * pc + j], sg_prior = sigma[(K - 1) * pc + j];
  const double half = TPE_DIV(cm.step, 2.0);
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = t / (G + 1);
    const int g = (int)(t - r * (G + 1));
    double m, s;
    if (g < G) {
      m = TPE_ADD(cm.low, TPE_MUL((double)g, cm.step));
      if (cm.log) m = log(m);
      s = sg_obs;
    } else {
      m = mu_prior;
      s = sg_prior;
    }
    const double x = by_cand ? S[r * pc + j] : TPE_ADD(cm.low, TPE_MUL((double)r, cm.step));
    double lo = TPE_SUB(x, half), hi = TPE_ADD(x, half);
    if (cm.log) { lo = log(lo); hi = log(hi); }
    dtab[cm.dtab_off + t] = log_gauss_mass(TPE_DIV(TPE_SUB(lo, m), s), TPE_DIV(TPE_SUB(hi, m), s));
  }
}

// Exact, any-kind evaluation of one (candidate, kernel) cell sum -- follows the reference's
// operation order (division by sigma, support test on normalised coordinates).
__device__ __forceinline__ double cell_one_exact(const ColMeta& cm, double x, double m, double s, bool is_prior,
                                                 const double* __restrict__ tab) {
  if (cm.cls == COL_CAT) {
    const int nch = cm.nch;
    const int row = is_prior ? nch : (int)m;
    const double* LW = tab + cm.tab_off + (int64_t)(nch + 1) * nch;
    return LW[(int64_t)row * nch + (int)x];
  }
  if (cm.cls == COL_CONT) {
    const double xv = cm.log ? log(x) : x;
    const double z = TPE_DIV(TPE_SUB(xv, m), s);
    const double a = TPE_DIV(TPE_SUB(cm.klow, m), s);
    const double b = TPE_DIV(TPE_SUB(cm.khigh, m), s);
    if (a == b) return NAN;
    if (z < a || z > b) return -INFINITY;
    return TPE_DIV(-TPE_MUL(z, z), 2.0);
  }
  const double h = TPE_DIV(cm.step, 2.0);
  double lo = TPE_SUB(x, h), hi = TPE_ADD(x, h);
  if (cm.log) { lo = log(lo); hi = log(hi); }
  return log_gauss_mass(TPE_DIV(TPE_SUB(lo, m), s), TPE_DIV(TPE_SUB(hi, m), s));
}
__device__ __forceinline__ double cell_sum_exact(const double* __restrict__ xrow, const double* __restrict__ mu_k,
                                                 const double* __restrict__ sg_k, const ColMeta* __restrict__ cols,
                                                 int32_t pc, bool is_prior, const double* __restrict__ tab) {
  double acc = 0.0;
  for (int j = 0; j < pc; ++j) acc += cell_one_exact(cols[j], xrow[j], mu_k[j], sg_k[j], is_prior, tab);
  return acc;
}

// Generic path: one thread per candidate, kernels [k0, k1) of split blockIdx.y.
// only_flagged != nullptr restricts the work to candidates with only_flagged[ct] != 0 (fix-up pass).
__global__ void k_logpdf_generic(const double* __restrict__ S, int64_t Ct, const ColMeta* __restrict__ cols, int32_t pc,
                                 const double* __restrict__ mu, const double* __restrict__ sigma,
                                 const double* __restrict__ cst, int64_t K, int64_t k_begin, int64_t kps,
                                 const double* __restrict__ tab, const uint8_t* __restrict__ only_flagged,
                                 double2* __restrict__ part, int64_t ct_stride) {
  const int64_t ct = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (ct >= Ct) return;
  double m = -INFINITY, s = 0.0;
  if (only_flagged == nullptr || only_flagged[ct] != 0) {
    const int64_t k0 = k_begin + blockIdx.y * kps;
    const int64_t k1 = (k0 + kps < K) ? k0 + kps : K;
    const double* xrow = S + ct * pc;
    for (int64_t k = k0; k < k1; ++k) {
      const double L = cst[k] + cell_sum_exact(xrow, mu + k * pc, sigma + k * pc, cols, pc, k == K - 1, tab);
      lse_push(L, m, s);
    }
  }
  part[blockIdx.y * ct_stride + ct] = make_double2(m, s);
}

// One warp per candidate, after the grid kernel:
//  * the prior kernel alone (CONST tables leave it out: its sigma differs), lanes over the columns,
//    same cell formula as the generic path, summed by a shuffle tree -> one more partial row;
//  * fix-up: a candidate outside [low, high] (rounding of ppf * sigma + mu; flagged by k_sample) is
//    re-evaluated exactly against every kernel, lanes over the kernels.
__device__ __forceinline__ void d_logpdf_prior_fix(const double* __restrict__ S, int64_t Ct, const ColMeta* __restrict__ cols,
                                   int32_t pc, const double* __restrict__ mu, const double* __restrict__ sigma,
                                   const double* __restrict__ cst, int64_t K, const double* __restrict__ tab,
                                   double2* __restrict__ part_prior, const uint8_t* __restrict__ oob,
                                   double2* __restrict__ fix, int do_fix = 1) {
  const int lane = threadIdx.x & 31;
  const int64_t ct = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  if (ct >= Ct) return;
  if (part_prior != nullptr) {
    const int64_t k = K - 1;
    double acc = 0.0;
    for (int j = lane; j < pc; j += 32)
      acc += cell_one_exact(cols[j], S[ct * pc + j], mu[k * pc + j], sigma[k * pc + j], true, tab);
    acc = warp_sum(acc);
    if (lane == 0) part_prior[ct] = make_double2(cst[k] + acc, 1.0);
  }
  if (do_fix && oob[ct] != 0) {
    double m = -INFINITY, s = 0.0;
    const double* xrow = S + ct * pc;
    for (int64_t k = lane; k < K; k += 32) {
      const double L = cst[k] + cell_sum_exact(xrow, mu + k * pc, sigma + k * pc, cols, pc, k == K - 1, tab);
      lse_push(L, m, s);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double m2 = __shfl_xor_sync(0xffffffffu, m, o), s2 = __shfl_xor_sync(0xffffffffu, s, o);
      lse_merge(m2, s2, m, s);
    }
    if (lane == 0) fix[ct] = make_double2(m, s);
  }
}
__global__ void
k_logpdf_prior_fix(const double* __restrict__ S, int64_t Ct, const ColMeta* __restrict__ cols,
                                   int32_t pc, const double* __restrict__ mu, const double* __restrict__ sigma,
                                   const double* __restrict__ cst, int64_t K, const double* __restrict__ tab,
                                   double2* __restrict__ part_prior, const uint8_t* __restrict__ oob,
                                   double2* __restrict__ fix, int do_fix = 1) { d_logpdf_prior_fix(S, Ct, cols, pc, mu, sigma, cst, K, tab, part_prior, oob, fix, do_fix); }

// Mixture weights of a small estimator (K <= 2048, i.e. the below set) in ONE launch: the bodies of
// k_wraw, k_wfinal and k_wnorm with a single CTA (same summation order as their one-part case).
__global__ void __launch_bounds__(256)
k_weights_one(const double* __restrict__ w_in, const int64_t* __restrict__ pos, int64_t n, double prior_weight,
              double* __restrict__ w, double* __restrict__ logw, const double* __restrict__ cst_part,
              double* __restrict__ cst, double* __restrict__ cdf, int64_t k_alloc, const double* __restrict__ hb,
              double* __restrict__ ckk) {
  __shared__ double s_red[8];
  __shared__ double s_total;
  const int64_t K = n + 1;
  double acc = 0.0;
  for (int64_t k = threadIdx.x; k < K; k += 256) {
    const double r = raw_weight(w_in, pos, n, k, prior_weight);
    w[k] = r;
    acc += r;
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int i = 0; i < 8; ++i) t += s_red[i];
    s_total = 0.0 + t;  // k_wfinal adds the (single) part to 0.0
  }
  __syncthreads();
  const double total = s_total;
  if (cdf != nullptr && threadIdx.x == 0) {
    double run = 0.0;
    for (int64_t k = 0; k < K; ++k) {
      run = TPE_ADD(run, TPE_DIV(w[k], total));
      cdf[k] = run;
    }
    const double last = run;
    for (int64_t k = 0; k < K; ++k) cdf[k] = TPE_DIV(cdf[k], last);
  }
  __syncthreads();
  for (int64_t k = threadIdx.x; k < k_alloc; k += 256) {
    if (k < K) {
      const double v = TPE_DIV(w[k], total);
      const double lw = log(v);
      logw[k] = lw;
      const double c = cst_part[k] + lw;
      cst[k] = c;
      if (ckk != nullptr) ckk[k] = (k < K - 1) ? c - hb[k] : -INFINITY;
      w[k] = v;
    } else {
      cst[k] = -INFINITY;
      if (ckk != nullptr) ckk[k] = -INFINITY;
    }
  }
}

// Generic path, pair-parallel: one CTA = one candidate x (256 * kpt) kernels, one thread evaluates
// whole (candidate, kernel) cell sums with the reference's operation order, block-level log-sum-exp.
// Used for spaces with discrete / categorical columns (every thread of a warp walks the same column
// kinds, so the special-function branches are the only divergence).
// Pair-parallel evaluation for spaces the fast kernel does not take (discrete / categorical columns,
// wide spaces): block = one candidate x one chunk of kernels, thread = one (candidate, kernel) cell sum.
// The candidate's columns are decoded once per block into shared descriptors:
//   kind 0  continuous, candidate inside [low, high]: -z^2/2 (the support test cannot fire)
//   kind 1  tabulated discrete: one load from the candidate's row of the cell-mass table
//   kind 3  categorical: one load from the log-weight table (row = the kernel's observed choice)
//   kind 2  anything else: the direct formula
struct PairCol {
  int kind, stride, gprior, pad;
  double xv;
  const double* base;
};
// CB candidates per CTA: mu / sigma / class of a kernel are loaded once for all of them (CB = 8 for
// large estimators, CB = 1 for the handful of kernels of l(x), where parallelism matters more)
template <int CB>
__global__ void __launch_bounds__(256, 2)
k_logpdf_pairs(const double* __restrict__ S, int64_t Ct, const ColMeta* __restrict__ cols, int32_t pc,
               const double* __restrict__ mu, const double* __restrict__ sigma, const double* __restrict__ cst,
               int64_t K, int kpt, const double* __restrict__ tab, const int32_t* __restrict__ cls,
               const double* __restrict__ dtab, const int* __restrict__ offgrid, const uint8_t* __restrict__ oob,
               double2* __restrict__ part, int64_t ct_stride) {
  extern __shared__ double s_dyn[];  // CB * pc PairCol descriptors, then pc flag bytes
  __shared__ double s_m[8][CB], s_s[8][CB];
  PairCol* s_col = reinterpret_cast<PairCol*>(s_dyn);
  uint8_t* s_need = reinterpret_cast<uint8_t*>(s_col + (size_t)CB * pc);  // 1: mu, 2: sigma, 4: class
  const int64_t ct0 = (int64_t)blockIdx.x * CB;
  const int64_t k0 = (int64_t)blockIdx.y * 256 * kpt;
  const bool tables_ok = dtab != nullptr && offgrid != nullptr && *offgrid == 0;
  for (int j = threadIdx.x; j < pc; j += 256) s_need[j] = 0;
  __syncthreads();
  for (int t = threadIdx.x; t < CB * pc; t += 256) {
    const int c = t / pc, j = t - c * pc;
    const int64_t ct = ct0 + c;
    PairCol pcj;
    pcj.kind = 4; pcj.stride = 0; pcj.gprior = 0; pcj.pad = 0; pcj.xv = 0.0; pcj.base = nullptr;  // 4: no candidate
    if (ct < Ct) {
      const bool in_support = oob != nullptr && oob[ct] == 0;
      const double x = S[ct * pc + j];
      const ColMeta cm = cols[j];
      pcj.kind = 2;
      pcj.xv = x;
      if (cm.cls == COL_CAT) {
        pcj.kind = 3;
        pcj.stride = cm.nch;
        pcj.gprior = cm.nch;
        pcj.base = tab + cm.tab_off + (int64_t)(cm.nch + 1) * cm.nch + (int)x;
      } else if (cm.cls == COL_CONT) {
        if (in_support && cm.klow < cm.khigh) {
          pcj.kind = 0;
          pcj.xv = cm.log ? log(x) : x;
        }
      } else if (cm.grid > 0 && tables_ok) {
        int64_t row = -1;
        if (Ct < cm.grid) {
          row = ct;  // candidate-indexed table
        } else {
          const double h = rint(TPE_DIV(TPE_SUB(x, cm.low), cm.step));
          if (h >= 0.0 && h < (double)cm.grid && TPE_ADD(cm.low, TPE_MUL(h, cm.step)) == x) row = (int64_t)h;
        }
        if (row >= 0) {
          pcj.kind = 1;
          pcj.stride = 1;
          pcj.gprior = cm.grid;
          pcj.base = dtab + cm.dtab_off + row * (cm.grid + 1);
        }
      }
      const int need = (pcj.kind == 1) ? 4 : ((pcj.kind == 3) ? 1 : 3);
      atomicOr(reinterpret_cast<unsigned int*>(s_need) + (j >> 2), (unsigned int)need << (8 * (j & 3)));
    }
    s_col[t] = pcj;
  }
  __syncthreads();
  double m[CB], s[CB];
#pragma unroll
  for (int c = 0; c < CB; ++c) {
    m[c] = -INFINITY;
    s[c] = 0.0;
  }
  for (int q = 0; q < kpt; ++q) {
    const int64_t k = k0 + (int64_t)q * 256 + threadIdx.x;
    if (k < K) {
      const bool is_prior = k == K - 1;
      const double* mu_k = mu + k * pc;
      const double* sg_k = sigma + k * pc;
      double acc[CB];
#pragma unroll
      for (int c = 0; c < CB; ++c) acc[c] = 0.0;
      for (int j = 0; j < pc; ++j) {
        const int need = s_need[j];
        const double mk = (need & 1) ? mu_k[j] : 0.0;
        const double sk = (need & 2) ? sg_k[j] : 1.0;
        const int ck = (need & 4) ? cls[k * pc + j] : 0;
#pragma unroll
        for (int c = 0; c < CB; ++c) {
          const PairCol d = s_col[c * pc + j];
          if (d.kind == 0) {
            const double z = TPE_DIV(TPE_SUB(d.xv, mk), sk);
            acc[c] += TPE_DIV(-TPE_MUL(z, z), 2.0);
          } else if (d.kind == 1) {
            acc[c] += d.base[is_prior ? d.gprior : ck];
          } else if (d.kind == 3) {
            acc[c] += d.base[(int64_t)(is_prior ? d.gprior : (int)mk) * d.stride];
          } else if (d.kind == 2) {
            acc[c] += cell_one_exact(cols[j], d.xv, mk, sk, is_prior, tab);
          }
        }
      }
      const double ck0 = cst[k];
#pragma unroll
      for (int c = 0; c < CB; ++c) lse_push(ck0 + acc[c], m[c], s[c]);
    }
  }
#pragma unroll
  for (int c = 0; c < CB; ++c) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double m2 = __shfl_xor_sync(0xffffffffu, m[c], o), s2 = __shfl_xor_sync(0xffffffffu, s[c], o);
      lse_merge(m2, s2, m[c], s[c]);
    }
    if ((threadIdx.x & 31) == 0) {
      s_m[threadIdx.x >> 5][c] = m[c];
      s_s[threadIdx.x >> 5][c] = s[c];
    }
  }
  __syncthreads();
  if (threadIdx.x < CB && ct0 + threadIdx.x < Ct) {
    const int c = threadIdx.x;
    double mm = s_m[0][c], ss = s_s[0][c];
    for (int w = 1; w < 8; ++w) lse_merge(s_m[w][c], s_s[w][c], mm, ss);
    part[(int64_t)blockIdx.y * ct_stride + ct0 + c] = make_double2(mm, ss);
  }
}

// Fast path: every selected column continuous.  Kernels are streamed through shared memory by TMA
// bulk copies (mbarrier completion); candidates live in registers; online log-sum-exp per candidate.
// Two fp64 instructions per (candidate, kernel, param) cell:
//   PAIR : t = fma(x', s_kp, -mu_s)      CONST: t = x'' - mu_s       then acc = fma(t, t, acc)
// with x' = x - c_p, x'' = (x - c_p) / sigma_p prepared once per candidate in the prologue.
//
// Register tiling.  Every table element fetched from shared memory (the LDS return path moves
// 128 B/clk/SM, broadcast or not) must feed enough fp64 work, so a thread owns RC candidates; for
// wide spaces the P axis is additionally split over PS adjacent lanes (PL = PB / PS params per lane)
// and the per-kernel partial sums are reduce-scattered with shuffles: lane h of a group ends up
// with the full sums of candidates [h * RC / PS, (h + 1) * RC / PS) and runs their log-sum-exp.
//
// Deferred exp.  Only terms within kLseSkip of the running max matter; they are rare (~1 %) but a
// warp diverges if any lane has one.  Such terms are parked in a 4-deep per-candidate register
// buffer and folded in at tile boundaries (or when a buffer fills), where all lanes do it together.
//
//   tab  [Kf][PB]  double2 (PAIR) or double (CONST), zero padded;  cst [Kf(+pad)]
//   xT   [PB][ct_stride] kernel-space candidate coordinates (zero padded)
//   part [gridDim.y][ct_stride] (running max, running sum)
struct LseAcc {
  double m, s, thr, b0, b1, b2, b3;
  double gm;  // best running max any CTA has published for this candidate (a lower bound of the true max)
  int cnt;
  __device__ __forceinline__ void init() {
    m = -INFINITY; s = 0.0; thr = -INFINITY; b0 = b1 = b2 = b3 = 0.0; cnt = 0; gm = -INFINITY;
  }
  // Truncation against the max over ALL kernels seen so far by any CTA / lane working on this
  // candidate, not just this lane's slice: the k-splits and the lanes of a candidate publish their
  // running max in `slot` (ordered-integer atomicMax) and read the others'.  Any published value is
  // some kernel's L, hence <= the true max: thresholds derived from it only drop terms that the
  // final log-sum-exp could drop as well.
  __device__ __forceinline__ void sync_global(unsigned long long* slot) {
    if (m > gm) atomicMax(slot, static_cast<unsigned long long>(order_bits(m)));
    const double seen = from_order_bits(*reinterpret_cast<volatile unsigned long long*>(slot));
    gm = fmax(gm, seen);
    thr = fmax(m, gm) - skip();
  }
  static __device__ __forceinline__ double& skip() {
    static __shared__ double s_skip;  // per-launch truncation distance (see k_logpdf_fast)
    return s_skip;
  }
  // branch-free fold of one parked term (valid == false leaves the accumulator untouched)
  __device__ __forceinline__ void fold(double L, bool valid) {
    const double d = L - m;
    const double e = exp(-fabs(d));  // m = -inf, L finite: d = +inf -> e = 0 -> s = 1
    const bool bigger = valid && (d > 0.0);
    const double grown = fma(s, e, 1.0);
    const double added = s + e;
    s = bigger ? grown : ((valid && d == d) ? added : s);
    m = bigger ? L : m;
  }
  // executed by the whole warp together (see push_sync)
  __device__ __forceinline__ void flush() {
    fold(b0, cnt > 0);
    fold(b1, cnt > 1);
    fold(b2, cnt > 2);
    fold(b3, cnt > 3);
    cnt = 0;
    thr = fmax(m, gm) - skip();
  }
  // Park L if it is within kLseSkip of the (possibly stale, i.e. lower) running max; when any lane's
  // buffer is full every lane folds its parked terms -- one converged pass instead of 32 diverged ones.
  __device__ __forceinline__ void push_sync(double L) {
    const bool hit = L > thr;
    b3 = hit ? b2 : b3;
    b2 = hit ? b1 : b2;
    b1 = hit ? b0 : b1;
    b0 = hit ? L : b0;
    cnt += hit ? 1 : 0;
    if (__any_sync(0xffffffffu, cnt == 4)) flush();
  }
};

template <int PB, int PS, int RC, int NT, int TK, int ST, bool PAIR, int MINB>
__global__ void __launch_bounds__(NT, MINB)
k_logpdf_fast(const void* __restrict__ tab_v, const double* __restrict__ cst, int64_t Kf,
              const double2* __restrict__ colprm, const double* __restrict__ xT, int64_t ct_stride, int64_t kps,
              double lse_skip, double2* __restrict__ part) {
  static_assert(PB % PS == 0 && RC % PS == 0, "bad tiling");
  static_assert(!PAIR || PS == 1, "PAIR tables are not split over lanes");
  constexpr int PL = PB / PS;   // params per lane
  constexpr int RL = RC / PS;   // candidates whose log-sum-exp this lane owns
  constexpr int GW = 32 / PS;   // candidate groups per warp
  constexpr int CW = GW * RC;   // candidates per warp
  using Elem = typename std::conditional<PAIR, double2, double>::type;
  constexpr int ES = PAIR ? 16 : 8;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  Elem* tiles = reinterpret_cast<Elem*>(smem_raw);                                 // ST * TK * PB
  double* csts = reinterpret_cast<double*>(smem_raw + (size_t)ST * TK * PB * ES);  // ST * TK
  uint64_t* full = reinterpret_cast<uint64_t*>(csts + (size_t)ST * TK);            // ST
  const Elem* tab = reinterpret_cast<const Elem*>(tab_v);
  const int tid = threadIdx.x;
  const int lane = tid & 31;
  const int h = lane % PS;      // which slice of the params
  const int g = lane / PS;      // candidate group inside the warp
  const int64_t k0 = blockIdx.y * kps;
  const int64_t k1 = (k0 + kps < Kf) ? k0 + kps : Kf;
  const int ntiles = (k1 > k0) ? (int)((k1 - k0 + TK - 1) / TK) : 0;
  // candidate r of this lane's group: wbase + r * GW + g
  const int64_t wbase = (int64_t)blockIdx.x * ((NT / 32) * CW) + (int64_t)(tid >> 5) * CW;

  if (tid == 0) {
    for (int s = 0; s < ST; ++s) mbar_init(&full[s], 1);
    mbar_fence_init();
    LseAcc::skip() = lse_skip;
  }
  __syncthreads();

  auto issue = [&](int t) {
    const int st = t % ST;
    const int64_t ks = k0 + (int64_t)t * TK;
    const int tk = (int)((k1 - ks < TK) ? (k1 - ks) : TK);
    const uint32_t b_tile = (uint32_t)(((size_t)tk * PB * ES + 15) & ~(size_t)15);
    const uint32_t b_cst = (uint32_t)(((tk + 1) & ~1) * 8);
    fence_proxy_async();
    mbar_expect_tx(&full[st], b_tile + b_cst);
    bulk_g2s(tiles + (size_t)st * TK * PB, tab + ks * PB, b_tile, &full[st]);
    bulk_g2s(csts + (size_t)st * TK, cst + ks, b_cst, &full[st]);
  };
  if (tid == 0) {
    for (int t = 0; t < ST - 1 && t < ntiles; ++t) issue(t);
  }

  double x[RC][PL];
  // lane h of a group owns the 16-byte slot pairs (q * PS + h): adjacent lanes read adjacent
  // shared-memory chunks (no bank conflicts); the sum over params does not care about the order
#pragma unroll
  for (int p = 0; p < PL; ++p) {
    const int slot = (PL == 1) ? h : 2 * ((p >> 1) * PS + h) + (p & 1);
    const double2 cp = colprm[slot];
#pragma unroll
    for (int r = 0; r < RC; ++r) {
      const int64_t ct = wbase + (int64_t)r * GW + g;
      x[r][p] = (xT[(int64_t)slot * ct_stride + ct] - cp.x) * cp.y;
    }
  }
  LseAcc acc[RL];
#pragma unroll
  for (int r = 0; r < RL; ++r) acc[r].init();

  for (int t = 0; t < ntiles; ++t) {
    const int st = t % ST;
    if (tid == 0 && t + ST - 1 < ntiles) issue(t + ST - 1);
    mbar_wait(&full[st], (uint32_t)((t / ST) & 1));
    const int64_t ks = k0 + (int64_t)t * TK;
    const int tk = (int)((k1 - ks < TK) ? (k1 - ks) : TK);
    const Elem* tile = tiles + (size_t)st * TK * PB;
    const double* ctile = csts + (size_t)st * TK;
    for (int kk = 0; kk < tk; ++kk) {
      double a0[RC], a1[RC];
#pragma unroll
      for (int r = 0; r < RC; ++r) {
        a0[r] = 0.0;
        a1[r] = 0.0;
      }
      if constexpr (PAIR) {
        const double2* row = reinterpret_cast<const double2*>(tile) + (size_t)kk * PB;
#pragma unroll
        for (int p = 0; p < PL; ++p) {
          const double2 v = row[p];
#pragma unroll
          for (int r = 0; r < RC; ++r) {
            const double d = fma(x[r][p], v.y, -v.x);
            if (p & 1) a1[r] = fma(d, d, a1[r]);
            else a0[r] = fma(d, d, a0[r]);
          }
        }
      } else if constexpr (PL == 1) {
        const double v = reinterpret_cast<const double*>(tile)[(size_t)kk * PB + h];
#pragma unroll
        for (int r = 0; r < RC; ++r) {
          const double d = x[r][0] - v;
          a0[r] = d * d;
        }
      } else {
        const double2* row =
            reinterpret_cast<const double2*>(reinterpret_cast<const double*>(tile) + (size_t)kk * PB) + h;
#pragma unroll
        for (int q = 0; q < PL / 2; ++q) {
          const double2 v = row[q * PS];
#pragma unroll
          for (int r = 0; r < RC; ++r) {
            const double d0 = x[r][2 * q] - v.x;
            const double d1 = x[r][2 * q + 1] - v.y;
            a0[r] = fma(d0, d0, a0[r]);
            a1[r] = fma(d1, d1, a1[r]);
          }
        }
      }
      double sum[RC];
#pragma unroll
      for (int r = 0; r < RC; ++r) sum[r] = a0[r] + a1[r];
      // reduce-scatter over the PS lanes of the group
      if constexpr (PS == 2) {
#pragma unroll
        for (int r = 0; r < RL; ++r) {
          const double mine = h ? sum[RL + r] : sum[r];
          const double send = h ? sum[r] : sum[RL + r];
          sum[r] = mine + __shfl_xor_sync(0xffffffffu, send, 1);
        }
      } else if constexpr (PS == 4) {
        // step 1 (xor 2): keep the half of the candidates selected by bit 1 of h
        double half[RC / 2];
#pragma unroll
        for (int r = 0; r < RC / 2; ++r) {
          const double mine = (h & 2) ? sum[RC / 2 + r] : sum[r];
          const double send = (h & 2) ? sum[r] : sum[RC / 2 + r];
          half[r] = mine + __shfl_xor_sync(0xffffffffu, send, 2);
        }
        // step 2 (xor 1): keep the quarter selected by bit 0 of h
#pragma unroll
        for (int r = 0; r < RL; ++r) {
          const double mine = (h & 1) ? half[RL + r] : half[r];
          const double send = (h & 1) ? half[r] : half[RL + r];
          sum[r] = mine + __shfl_xor_sync(0xffffffffu, send, 1);
        }
      }
      const double c = ctile[kk];
#pragma unroll
      for (int r = 0; r < RL; ++r) acc[r].push_sync(fma(-0.5, sum[r], c));
    }
    __syncthreads();  // stage `st` may be refilled by the next iteration's issue()
  }
#pragma unroll
  for (int r = 0; r < RL; ++r) acc[r].flush();
  // lane h owns candidates r = h * RL + r' of its group
#pragma unroll
  for (int r = 0; r < RL; ++r) {
    const int64_t ct = wbase + (int64_t)(h * RL + r) * GW + g;
    part[blockIdx.y * ct_stride + ct] = make_double2(acc[r].m, acc[r].s);
  }
}

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// e^x for -700 <= x <= 700 in ~17 instructions: x = (64 n + j) ln2 / 64 + r, |r| <= ln2 / 128;
// e^x = 2^n * 2^(j/64) * P5(r) with a 64-entry table in shared memory (filled by the CTA: exp2(j / 64), 1 ulp) and a
// degree-5 Taylor polynomial (truncation 3.5e-17).  The two-term Cody-Waite reduction is exact for |x| < 700
// (ln2_hi / 64 keeps 21 trailing zero bits).  Relative error <= 3e-16.
__device__ __forceinline__ double uni_exp(double x, const double* __restrict__ tab64) {
  const double t = fma(x, 92.332482616893656768, 6755399441055744.0);
  const int ni = __double2loint(t);
  const double nf = t - 6755399441055744.0;
  double r = fma(nf, -1.08304246932675596327e-02, x);
  r = fma(nf, -2.98158582698529328128e-12, r);
  double p = 8.33333333333333333333e-03;
  p = fma(p, r, 4.16666666666666666667e-02);
  p = fma(p, r, 1.66666666666666666667e-01);
  p = fma(p, r, 0.5);
  p = fma(p, r, 1.0);
  p = fma(p, r, 1.0);
  const double y = tab64[ni & 63] * p;
  return __hiloint2double(__double2hiint(y) + ((ni >> 6) << 20), __double2loint(y));
}

// Two-tier log-sum-exp of the tensor-core kernel, summed against a fixed reference R.  Terms are classified against
// `base`, a lower bound of the candidate's true max (the largest term this lane has folded, or a larger one published
// by another lane / CTA):
//   near  L - base > -tnear           parked, then e^(L - R) in fp64 (uni_exp) by the whole warp at once
//   far   -skip < L - base <= -tnear  e^(L - R) at once on the fp32 SFU path (MUFU.EX2), summed in fp32:
//                                     no parking, no fp64 work, branch-free
//   else  dropped
// With tnear = ln K + 17.5 and skip = ln K + 30 the result stays inside the fp64-parity budget whatever the data:
// each far term is <= e^-tnear of the max term, there are <= K of them and each carries <= 7.5e-6 relative error
// (fp32 rounding of L - R: 1.9e-6 for |L - R| < 64; rounding of the product with log2 e and of that constant:
// 3.2e-6; ex2.approx: 2.4e-7; fp32 runs of <= 32 terms: 1.9e-6), so the far tier adds <= 7.5e-6 * K * e^-tnear =
// 1.9e-13 relative to the sum; dropped terms add <= 1e-13.  The thresholds are compared in fp32 (against
// fl(base - R) - tnear), which moves them by < 1e-5 nats: a factor e^1e-5 on these bounds.
// R is the first value base takes and moves (to base, with one rescale of the sum) only when base climbs more than
// kRefMove above it, so R <= base <= R + kRefMove at all times.  Hence a far term has -skip < L - R <= kRefMove -
// tnear (|L - R| < 64 for any K <= e^34), a near term e^(L - R) <= e^kRefMove, and the exact terms need no running
// max: they are independent exponentials, and a rise of base costs no rescale.
// Near terms are parked as raw L in a per-(lane, candidate group) ring of D slots in shared memory, slot i at
// ring[i * RS] (slot-major, so a warp's store or load is conflict-free whatever each lane's count): a near term is
// stored with a predicated store and no branch, and one warp vote per step decides whether to flush (MmaSmem).
constexpr double kRefMove = 48.0;
__device__ __forceinline__ unsigned long long ld_relaxed_gpu(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p));
  return v;
}
struct LseRef {
  double R, s, base;     // reference, sum of e^(L - R), classification base
  float ffar;            // current fp32 run of far terms, relative to R
  float thn;             // near threshold on fl(L - R): fl(base - R) - tnear (far: - skip)
  unsigned wp;           // shared-memory address of the next free ring slot: slot0 + (parked terms) * RS * 8
  __device__ __forceinline__ void init(unsigned slot0) {
    R = -INFINITY; s = 0.0; base = -INFINITY;
    ffar = 0.0f; thn = -INFINITY; wp = slot0;   // cold: every finite term is near
  }
  // base := nb (>= base); R follows when nb is more than kRefMove above it (also the cold start, R = -inf: s and the
  // far run are 0 then).  Executed by the whole warp together.
  __device__ __forceinline__ void rebase(double nb, float tnear, const double* e64) {
    if (__any_sync(0xffffffffu, nb > R + kRefMove)) {
      const bool mv = nb > R + kRefMove;
      const double f = uni_exp(fmax(R - nb, -700.0), e64);
      s = mv ? (s + (double)ffar) * f : s;
      ffar = mv ? 0.0f : ffar;
      R = mv ? nb : R;
    }
    base = nb;
    const float d = __double2float_rn(base - R);   // R = -inf only while base = -inf: stay cold
    thn = (R == -INFINITY) ? -INFINITY : d - tnear;
  }
  // fold the parked terms (executed by the whole warp together): base first (to the largest parked term, so that
  // e^(L - R) <= e^kRefMove), then independent exps over the slots any lane of the warp has filled
  template <int RS>
  __device__ __forceinline__ void flush(const double* ring, float tnear, const double* e64) {
    const unsigned slot0 = (unsigned)__cvta_generic_to_shared(ring);
    const int cnt = parked<RS>(slot0);
    const int n = __reduce_max_sync(0xffffffffu, cnt);
    double nb = base;
    for (int i = 0; i < n; ++i) {
      const double v = ring[i * RS];
      nb = (i < cnt && v > nb) ? v : nb;
    }
    rebase(nb, tnear, e64);
    double sum = 0.0;
    for (int i = 0; i < n; ++i) {   // slots >= cnt may hold anything: selected away, never multiplied
      const double e = uni_exp(fmax(ring[i * RS] - R, -700.0), e64);
      sum += (i < cnt) ? e : 0.0;
    }
    s += sum;
    wp = slot0;
  }
  // park L in the next free slot if it is near: a predicated store (written in PTX: the compiler turns `if (near)`
  // into a branch), no vote
  template <int RS>
  __device__ __forceinline__ void park(double L, bool near) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %2, 0;\n\t@p st.shared.f64 [%0], %1;\n\t}"
                 :: "r"(wp), "d"(L), "r"((unsigned)near) : "memory");
    wp += near ? RS * 8 : 0;
  }
  // terms parked in the ring starting at slot0
  template <int RS>
  __device__ __forceinline__ int parked(unsigned slot0) const { return (int)((wp - slot0) / (RS * 8)); }
  __device__ __forceinline__ void roll() {  // bounds the length of the fp32 runs (once per tile)
    s += (double)ffar;
    ffar = 0.0f;
  }
  // Publish base in `slot` (ordered-integer atomicMax) and adopt a larger one published by the k-splits and lanes
  // that share the candidate.  Any published value is some kernel's L, hence <= the true max.  `pend` holds the
  // slot as read at the previous exchange; the read for the next one is issued here, so its L2 round trip overlaps
  // the tile instead of stalling the warp.
  __device__ __forceinline__ void sync_global(unsigned long long* slot, unsigned long long& pend, float tnear,
                                              const double* e64) {
    const double seen = from_order_bits(pend);
    pend = ld_relaxed_gpu(slot);
    if (base > seen) atomicMax(slot, static_cast<unsigned long long>(order_bits(base)));
    if (__any_sync(0xffffffffu, seen > base)) rebase(fmax(base, seen), tnear, e64);
  }
  // One term's classification, independent of every other term's (so the kernel interleaves it with the mma chain
  // of the next step): adds a far term to `add` (the caller folds it into ffar), counts it in `nfar` (lab counters)
  // and says whether the term is near.  gap = skip - tnear.
  __device__ __forceinline__ bool classify(double L, float gap, float& add, int& nfar) const {
    const float df = __double2float_rn(L - R);  // cold (R = -inf): +inf -> near; L = -inf or NaN: dropped
    const bool near = df > thn;
    const bool far = !near && df > thn - gap;
    const float e = ex2_approx(df * 1.44269504f);
    add += far ? e : 0.0f;
    nfar += far ? 1 : 0;
    return near;
  }
  // the lane's (max, sum) pair for lse_merge, relative to base (s e^(R - base); R = base = -inf: (-inf, 0))
  __device__ __forceinline__ double2 result(const double* e64) const {
    return make_double2(base, s * uni_exp(fmax(R - base, -700.0), e64));
  }
};

// ================================================================================================
// Tensor-core variant of the CONST kernel (multivariate TPE, continuous columns).
//
// With one sigma per column the cell sum is a squared distance in scaled coordinates
//   a_cp = (x_cp - ctr_p) / sigma_p,  b_kp = (mu_kp - ctr_p) / sigma_p,
//   L[c,k] = cst_k - |a_c - b_k|^2 / 2 = (cst_k - |b_k|^2 / 2) + a_c . b_k - |a_c|^2 / 2,
// i.e. ONE fma per cell instead of two, and the a . b part is a [C x P] x [P x K] fp64 GEMM: it runs
// on the fp64 tensor-core path with the operands shared in registers, so neither the issue slots nor the
// shared-memory pipe limit it.  With M even a warp owns pairs of candidate groups and issues mma.sync
// m16n8k8 (SASS DMMA.16x8x8, 1024 fma per warp instruction, twice the DFMA rate on H100); with M = 1 it
// issues m8n8k4 (DMMA.8x8x4, 256 fma, the DFMA rate on H100), which still wins for a single small ask.
// Both read the same registers and table: one m16n8k8 does the work of four m8n8k4 (two k-steps x two
// candidate groups), only the order of the roundings inside one k8 step differs.  The accumulator fragment is initialised with
// cst_k - |b_k|^2 / 2 (host side of the build), so L - ha_c falls out of the mma chain directly and
// -|a_c|^2 / 2 is added once per candidate after the log-sum-exp (shift invariance).
// Rounding: |a|, |b| <= rho = range / (2 sigma); the expanded form loses ~P * rho^2 * 2^-52 absolute
// (8e-14 at config 2); the host falls back to k_logpdf_fast when that bound exceeds 5e-13.
//
//   rows of A = candidates (8 per group, M groups per warp), columns of B = kernels (8 per mma);
//   lane (g = lane / 4, q = lane % 4) holds C[candidate g][kernels 2q, 2q + 1]: it owns one
//   log-sum-exp state per candidate group and the 4 lanes of a candidate are merged at the end.
//   tabm: fragment-major table (mma_tab_index), ckk: per-kernel constants (-inf padded to 8).
// ================================================================================================
__device__ __forceinline__ void dmma_8x8x4(double& d0, double& d1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
               : "+d"(d0), "+d"(d1)
               : "d"(a), "d"(b));
}
// m16n8k8 (SASS DMMA.16x8x8, twice the DFMA rate on H100): rows g and g + 8 of A are two candidate groups,
// a0..a3 = A[g][q], A[g + 8][q], A[g][q + 4], A[g + 8][q + 4]; b0, b1 = B[q][g], B[q + 4][g];
// {d0, d1} = C[g][2q, 2q + 1], {d2, d3} = C[g + 8][2q, 2q + 1] -- the m8n8k4 fragments of two k-steps and
// two candidate groups, so the table and the A registers are the same as for m8n8k4.
__device__ __forceinline__ void dmma_16x8x8(double& d0, double& d1, double& d2, double& d3, double a0, double a1,
                                            double a2, double a3, double b0, double b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+d"(d0), "+d"(d1), "+d"(d2), "+d"(d3)
               : "d"(a0), "d"(a1), "d"(a2), "d"(a3), "d"(b0), "d"(b1));
}
// Dynamic shared memory of one k_logpdf_mma CTA: the TMA stages (table tiles, constants, full / empty barriers),
// then the near-term ring.  The ring takes D slots per (warp, candidate group, lane), 8 B each, laid out
// [slot][warp][group][lane].  D is as deep as the memory the stages leave allows at the CTAs per SM they allow (at
// most MINB; 228 KB per SM, 1 KB reserved and the 512 B uni_exp table per CTA), capped at max(8, 2 NVG), and must
// hold at least the NVG values one step can park: a warp flushes once a lane has more than D - NVG terms parked.
template <int PB, int M, int KG, int NT, int TK, int ST, int MINB>
struct MmaSmem {
  static constexpr size_t stages = (size_t)ST * TK * PB * 8 + (size_t)ST * TK * 8 + (size_t)ST * 16;
  static constexpr int NVG = 2 * KG;                                // values per lane, candidate group and step
  static constexpr int RS = (NT / 32) * M * 32;                     // doubles between two slots of a lane's ring
  static constexpr size_t kSm = 228 * 1024, kCta = 1024 + 64 * 8;
  static constexpr size_t ctas_ = kSm / (stages + kCta);
  static constexpr size_t ctas = ctas_ < (size_t)MINB ? ctas_ : (size_t)MINB;
  static constexpr size_t fit = (kSm / ctas - kCta - stages) / (RS * 8);
  static constexpr int cap = (2 * NVG > 8) ? 2 * NVG : 8;
  static constexpr int D = (fit < (size_t)cap) ? (int)fit : cap;
  static_assert(D >= NVG, "the near-term ring does not fit beside the TMA stages: fewer stages or a shorter tile");
  static constexpr size_t bytes = stages + (size_t)D * RS * 8;
};

#ifdef TPE_LAB
// lab counters of k_logpdf_mma<..., DBG = 5> (summed over launches until read by tpe_lab_mma_counters): near terms,
// far terms, flushes by the vote (per warp and candidate group), terms parked at those flushes, ring slots they walked
__device__ unsigned long long g_mma_lab_count[5];
#endif

// KG kernel groups (8 kernels each) per step of a warp: KG * M independent m8n8k4 chains (M = 1), or KG * M / 2
// m16n8k8 chains (M even, two candidate groups per instruction).  The steps are software-pipelined: a warp issues
// the chains of step s + 1 before it classifies the sums of step s, so the DMMA latency of one step hides behind
// the log-sum-exp of the previous one (two accumulator sets live at once).
template <int PB, int M, int KG, int NT, int TK, int ST, int MINB, int DBG = 0>
__global__ void __launch_bounds__(NT, MINB)
k_logpdf_mma(const double* __restrict__ tabm, const double* __restrict__ ckk, int64_t Kfp,
             const double2* __restrict__ colprm, const double* __restrict__ xT, int64_t ct_stride, int64_t kps,
             double lse_skip, double2* __restrict__ part, unsigned long long* __restrict__ gmax,
             double lse_near) {
  static_assert(PB % 8 == 0 && TK % (8 * KG) == 0 && (M == 1 || M % 2 == 0), "bad tiling");
  constexpr int NI = PB / 4;        // k-steps of the mma chain
  constexpr int CW = 8 * M;         // candidates per warp
  extern __shared__ __align__(128) unsigned char smem_raw[];
  __shared__ double s_e64[64];                                                     // uni_exp table
  double* tiles = reinterpret_cast<double*>(smem_raw);                             // ST * TK * PB
  double* csts = tiles + (size_t)ST * TK * PB;                                     // ST * TK
  uint64_t* full = reinterpret_cast<uint64_t*>(csts + (size_t)ST * TK);            // ST
  uint64_t* empty = full + ST;                                                     // ST
  using SM = MmaSmem<PB, M, KG, NT, TK, ST, MINB>;
  double* ring = reinterpret_cast<double*>(empty + ST) + (threadIdx.x >> 5) * M * 32 + (threadIdx.x & 31);
  const int tid = threadIdx.x;
  const int lane = tid & 31;
  const int g = lane >> 2, q = lane & 3;
  const int64_t k0 = blockIdx.y * kps;
  const int64_t k1 = (k0 + kps < Kfp) ? k0 + kps : Kfp;   // Kfp, kps: multiples of 8 * KG
  const int ntiles = (k1 > k0) ? (int)((k1 - k0 + TK - 1) / TK) : 0;
  const int nsteps = (k1 > k0) ? (int)((k1 - k0) / (8 * KG)) : 0;
  const int64_t wbase = (int64_t)blockIdx.x * ((NT / 32) * CW) + (int64_t)(tid >> 5) * CW;

  if (tid < 64) s_e64[tid] = exp2((double)tid * 0.015625);
  if (tid == 0) {
    for (int s = 0; s < ST; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], NT / 32);
    }
    mbar_fence_init();
  }
  __syncthreads();
  auto issue = [&](int t) {
    const int st = t % ST;
    const int64_t ks = k0 + (int64_t)t * TK;
    const int tk = (int)((k1 - ks < TK) ? (k1 - ks) : TK);
    const uint32_t b_tile = (uint32_t)((size_t)tk * PB * 8);
    const uint32_t b_cst = (uint32_t)(tk * 8);
    fence_proxy_async();
    mbar_expect_tx(&full[st], b_tile + b_cst);
    bulk_g2s(tiles + (size_t)st * TK * PB, tabm + ks * PB, b_tile, &full[st]);
    bulk_g2s(csts + (size_t)st * TK, ckk + ks, b_cst, &full[st]);
  };
  if (tid == 0) {
    for (int t = 0; t < ST - 1 && t < ntiles; ++t) issue(t);
  }
  // make tile t readable; the stage being refilled held tile t - 1: first wait until every warp has released it
  auto enter = [&](int t) {
    if (tid == 0 && t + ST - 1 < ntiles) {
      if (t > 0) mbar_wait(&empty[(t - 1) % ST], (uint32_t)(((t - 1) / ST) & 1));
      issue(t + ST - 1);
    }
    mbar_wait(&full[t % ST], (uint32_t)((t / ST) & 1));
  };
  auto groups_in = [&](int t) {  // kernel groups of tile t
    const int64_t ks = k0 + (int64_t)t * TK;
    return (int)((k1 - ks < TK) ? (k1 - ks) : TK) / 8;
  };

  // A fragments: a[m][i] = A[row g][col q] of k-step i = scaled coordinate 4 i + q of candidate 8 m + g
  double a[M][NI];
  double ha[M];
#pragma unroll
  for (int m = 0; m < M; ++m) ha[m] = 0.0;
#pragma unroll
  for (int i = 0; i < NI; ++i) {
    const int slot = 4 * i + q;
    const double2 cp = colprm[slot];
#pragma unroll
    for (int m = 0; m < M; ++m) {
      const int64_t ct = wbase + 8 * m + g;
      const double v = (xT[(int64_t)slot * ct_stride + ct] - cp.x) * cp.y;
      a[m][i] = v;
      ha[m] = fma(v, v, ha[m]);
    }
  }
#pragma unroll
  for (int m = 0; m < M; ++m) {
    ha[m] += __shfl_xor_sync(0xffffffffu, ha[m], 1);
    ha[m] += __shfl_xor_sync(0xffffffffu, ha[m], 2);
    ha[m] *= -0.5;
  }

  // The mma chains of kernel groups kg .. kg + KG - 1 of tile t: d[u][m] = C[candidate 8 m + g][kernels 2q, 2q + 1].
  // work(i) runs after the DMMAs of dependent level i (NL levels): the warp issues in order, so independent work placed
  // there fills the DMMA latency instead of a stall before the next level.
  constexpr int NL = (M % 2 == 0) ? NI / 2 : NI;
  auto chain = [&](int t, int kg, double (&d)[KG][M][2], auto&& work) {
    const double* tile = tiles + (size_t)(t % ST) * TK * PB;
    const double* ctile = csts + (size_t)(t % ST) * TK;
    const double2* fb = reinterpret_cast<const double2*>(tile + (size_t)kg * 8 * PB) + lane;
#pragma unroll
    for (int u = 0; u < KG; ++u) {
      const double2 cc = reinterpret_cast<const double2*>(ctile + (kg + u) * 8)[q];
#pragma unroll
      for (int m = 0; m < M; ++m) {
        d[u][m][0] = cc.x;
        d[u][m][1] = cc.y;
      }
    }
    double2 v[2][KG];
#pragma unroll
    for (int u = 0; u < KG; ++u) v[0][u] = fb[u * (4 * PB)];   // one kernel group = 8 * PB doubles
#pragma unroll
    for (int i2 = 0; i2 < NI / 2; ++i2) {
      if (i2 + 1 < NI / 2) {
#pragma unroll
        for (int u = 0; u < KG; ++u) v[(i2 + 1) & 1][u] = fb[u * (4 * PB) + (i2 + 1) * 32];
      }
      if constexpr (M % 2 == 0) {
#pragma unroll
        for (int u = 0; u < KG; ++u)
#pragma unroll
          for (int m = 0; m < M; m += 2)
            dmma_16x8x8(d[u][m][0], d[u][m][1], d[u][m + 1][0], d[u][m + 1][1], a[m][2 * i2], a[m + 1][2 * i2],
                        a[m][2 * i2 + 1], a[m + 1][2 * i2 + 1], v[i2 & 1][u].x, v[i2 & 1][u].y);
        work(i2);
      } else {
#pragma unroll
        for (int u = 0; u < KG; ++u) dmma_8x8x4(d[u][0][0], d[u][0][1], a[0][2 * i2], v[i2 & 1][u].x);
        work(2 * i2);
#pragma unroll
        for (int u = 0; u < KG; ++u) dmma_8x8x4(d[u][0][0], d[u][0][1], a[0][2 * i2 + 1], v[i2 & 1][u].y);
        work(2 * i2 + 1);
      }
    }
  };

  LseRef acc[M];
  unsigned long long gpend[M];   // gmax slot as read for the next exchange of maxima
#pragma unroll
  for (int m = 0; m < M; ++m) {
    acc[m].init((unsigned)__cvta_generic_to_shared(ring + m * 32));
    gpend[m] = ld_relaxed_gpu(gmax + wbase + 8 * m + g);
  }
  const float lim_near = (float)lse_near, lim_gap = (float)(lse_skip - lse_near);
  int lab_far = 0;                                   // lab counters (DBG = 5)
  unsigned lab_near = 0, lab_flush = 0, lab_occ = 0, lab_walk = 0;

  constexpr int NV = 2 * KG * M;   // sums per lane and step: value j = (m, u, h) = (j / 2KG, j % 2KG / 2, j % 2)
  double cur[KG][M][2], nxt[KG][M][2];
  int tc = 0, kc = 0;            // tile and first kernel group of the step in `cur`
  int ngc = 0;                   // kernel groups of tile tc
  auto none = [](int) {};
  if (nsteps > 0) {
    enter(0);
    ngc = groups_in(0);
    chain(0, 0, cur, none);
  }
  for (int s = 0; s < nsteps; ++s) {
    if constexpr (DBG != 4) {
      if (kc == 0 || tc == 0) {  // every tile, and every step of the CTA's first tile (cold start)
#pragma unroll
        for (int m = 0; m < M; ++m) {
          acc[m].roll();
          acc[m].sync_global(gmax + wbase + 8 * m + g, gpend[m], lim_near, s_e64);
        }
      } else if ((kc & 15) == 0) {  // long tiles (small PB): keep the fp32 runs at <= 32 terms
#pragma unroll
        for (int m = 0; m < M; ++m) acc[m].roll();
      }
    }
    // classification of value j (far terms summed at once, near ones flagged); DBG = 1 / 4: plain sums
    bool nr[M][2 * KG];
    float add[M];
#pragma unroll
    for (int m = 0; m < M; ++m) add[m] = 0.0f;
    auto cls = [&](int j) {
      const int m = j / (2 * KG), u = (j % (2 * KG)) / 2, h = j & 1;
      if constexpr (DBG == 1 || DBG == 4) acc[m].s += cur[u][m][h];
      else nr[m][j % (2 * KG)] = acc[m].classify(cur[u][m][h], lim_gap, add[m], lab_far);
    };
    // level i of the next chain is followed by the values j with j * NL / NV == i
    auto work = [&](int i) {
#pragma unroll
      for (int j = 0; j < NV; ++j)
        if (j * NL / NV == i) cls(j);
    };

    // position of step s + 1; at the end of a tile release its stage (its last chain has read the table)
    int tn = tc, kn = kc + KG, ngn = ngc;
    if (kn == ngc) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[tc % ST]);
      tn = tc + 1;
      kn = 0;
      if (tn < ntiles) {
        enter(tn);
        ngn = groups_in(tn);
      }
    }
    if (s + 1 < nsteps) {
      chain(tn, kn, nxt, work);
    } else {
#pragma unroll
      for (int j = 0; j < NV; ++j) cls(j);
    }

    if constexpr (DBG != 1 && DBG != 4) {
#pragma unroll
      for (int m = 0; m < M; ++m) {
        acc[m].ffar += add[m];
        if constexpr (DBG == 0 || DBG == 5) {
          // terms classified far against the old base stay far (exact enough by construction) even if the flush
          // raises base
#pragma unroll
          for (int i = 0; i < 2 * KG; ++i) {
            acc[m].template park<SM::RS>(cur[i / 2][m][i % 2], nr[m][i]);
            if constexpr (DBG == 5) lab_near += nr[m][i] ? 1 : 0;
          }
          const unsigned slot0 = (unsigned)__cvta_generic_to_shared(ring + m * 32);
          if (__any_sync(0xffffffffu, acc[m].wp > slot0 + (SM::D - SM::NVG) * SM::RS * 8)) {
            if constexpr (DBG == 5) {
              const int cnt = acc[m].template parked<SM::RS>(slot0);
              lab_flush += 1;
              lab_occ += cnt;
              lab_walk += __reduce_max_sync(0xffffffffu, cnt);
            }
            acc[m].template flush<SM::RS>(ring + m * 32, lim_near, s_e64);
          }
        }
      }
    }
#pragma unroll
    for (int u = 0; u < KG; ++u)
#pragma unroll
      for (int m = 0; m < M; ++m) {
        cur[u][m][0] = nxt[u][m][0];
        cur[u][m][1] = nxt[u][m][1];
      }
    tc = tn;
    kc = kn;
    ngc = ngn;
  }
#pragma unroll
  for (int m = 0; m < M; ++m) {
    acc[m].template flush<SM::RS>(ring + m * 32, lim_near, s_e64);
    acc[m].roll();
    const double2 r = acc[m].result(s_e64);
    double mm = r.x, ss = r.y;
#pragma unroll
    for (int o = 1; o <= 2; o <<= 1) {
      const double m2 = __shfl_xor_sync(0xffffffffu, mm, o), s2 = __shfl_xor_sync(0xffffffffu, ss, o);
      lse_merge(m2, s2, mm, ss);
    }
    if (q == 0) part[blockIdx.y * ct_stride + wbase + 8 * m + g] = make_double2(mm + ha[m], ss);
  }
#ifdef TPE_LAB
  if constexpr (DBG == 5) {
    const unsigned nn = __reduce_add_sync(0xffffffffu, lab_near);
    const unsigned nf = __reduce_add_sync(0xffffffffu, (unsigned)lab_far);
    const unsigned no = __reduce_add_sync(0xffffffffu, lab_occ);
    if (lane == 0) {
      atomicAdd(&g_mma_lab_count[0], (unsigned long long)nn);
      atomicAdd(&g_mma_lab_count[1], (unsigned long long)nf);
      atomicAdd(&g_mma_lab_count[2], (unsigned long long)lab_flush);
      atomicAdd(&g_mma_lab_count[3], (unsigned long long)no);
      atomicAdd(&g_mma_lab_count[4], (unsigned long long)lab_walk);
    }
  }
#endif
}

// ================================================================================================
// acquisition + argmax
// ================================================================================================
// Grid-wide pass: logl/logg = merge of the k-split partials (or the fix-up value for
// out-of-support candidates), written for every candidate.  One warp per candidate: lanes stride
// over the partial rows (a single small ask has > 1000 of them), then a shuffle merge.
__device__ __forceinline__ void d_acq(const double2* __restrict__ part_l, int nsl, const double2* __restrict__ part_g, int nsg,
                      int64_t ct_stride, const uint8_t* __restrict__ oob, const double2* __restrict__ fix_l,
                      const double2* __restrict__ fix_g, int64_t Ct, double* __restrict__ logl,
                      double* __restrict__ logg) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t ct = warp; ct < Ct; ct += nwarps) {
    double ml = -INFINITY, sl = 0.0, mg = -INFINITY, sg = 0.0;
    if (oob != nullptr && oob[ct]) {
      ml = fix_l[ct].x; sl = fix_l[ct].y;
      mg = fix_g[ct].x; sg = fix_g[ct].y;
    } else {
      for (int s = lane; s < nsl; s += 32) {
        const double2 v = part_l[(int64_t)s * ct_stride + ct];
        lse_merge(v.x, v.y, ml, sl);
      }
      for (int s = lane; s < nsg; s += 32) {
        const double2 v = part_g[(int64_t)s * ct_stride + ct];
        lse_merge(v.x, v.y, mg, sg);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const double m2 = __shfl_xor_sync(0xffffffffu, ml, o), s2 = __shfl_xor_sync(0xffffffffu, sl, o);
        lse_merge(m2, s2, ml, sl);
        const double m3 = __shfl_xor_sync(0xffffffffu, mg, o), s3 = __shfl_xor_sync(0xffffffffu, sg, o);
        lse_merge(m3, s3, mg, sg);
      }
    }
    if (lane == 0) {
      // np.log(sum exp(L - max)) + max, with max := 0 when it is -inf
      logl[ct] = (ml == -INFINITY) ? -INFINITY : log(sl) + ml;
      logg[ct] = (mg == -INFINITY) ? -INFINITY : log(sg) + mg;
    }
  }
}
__global__ void
k_acq(const double2* __restrict__ part_l, int nsl, const double2* __restrict__ part_g, int nsg,
                      int64_t ct_stride, const uint8_t* __restrict__ oob, const double2* __restrict__ fix_l,
                      const double2* __restrict__ fix_g, int64_t Ct, double* __restrict__ logl,
                      double* __restrict__ logg) { d_acq(part_l, nsl, part_g, nsg, ct_stride, oob, fix_l, fix_g, Ct, logl, logg); }

// (max, sum) per candidate over the k-split partials of ONE estimator, merged in slice order (what a rank of a
// kernel-sharded suggestion contributes: tpe_sample_and_partial)
__global__ void k_reduce_parts(const double2* __restrict__ part, int ns, int64_t ct_stride, int64_t Ct,
                               double2* __restrict__ out) {
  for (int64_t ct = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; ct < Ct; ct += (int64_t)gridDim.x * blockDim.x) {
    double m = -INFINITY, s = 0.0;
    for (int i = 0; i < ns; ++i) {
      const double2 v = part[(int64_t)i * ct_stride + ct];
      lse_merge(v.x, v.y, m, s);
    }
    out[ct] = make_double2(m, s);
  }
}

// One CTA per ask: acq = logl - logg, best = first maximum (NaN wins, like np.argmax).
__device__ __forceinline__ void d_select(const double* __restrict__ logl, const double* __restrict__ logg, int32_t C, const double* __restrict__ S,
         int32_t pc, double* __restrict__ out_x, double* __restrict__ out_acq, int64_t* __restrict__ out_best) {
  __shared__ double s_val[256];
  __shared__ int s_idx[256];
  const int64_t ask = blockIdx.x;
  const int tid = threadIdx.x;
  double best = 0.0;
  int besti = -1;
  bool best_nan = false;
  for (int c = tid; c < C; c += 256) {
    const int64_t ct = ask * C + c;
    const double a = logl[ct] - logg[ct];
    const bool a_nan = a != a;
    if (besti < 0 || (!best_nan && (a_nan || a > best))) {
      best = a;
      besti = c;
      best_nan = a_nan;
    }
  }
  s_val[tid] = best;
  s_idx[tid] = besti;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (tid < o) {
      const double a = s_val[tid], b = s_val[tid + o];
      const int ia = s_idx[tid], ib = s_idx[tid + o];
      bool take_b;
      if (ib < 0) take_b = false;
      else if (ia < 0) take_b = true;
      else {
        const bool an = a != a, bn = b != b;
        if (an && bn) take_b = ib < ia;
        else if (an) take_b = false;
        else if (bn) take_b = true;
        else take_b = (b > a) || (b == a && ib < ia);
      }
      if (take_b) {
        s_val[tid] = b;
        s_idx[tid] = ib;
      }
    }
    __syncthreads();
  }
  const int bi = s_idx[0];
  if (tid == 0) {
    if (out_best) out_best[ask] = bi;
    if (out_acq) out_acq[ask] = s_val[0];
  }
  for (int j = tid; j < pc; j += 256) out_x[ask * pc + j] = S[(ask * C + bi) * pc + j];
}
__global__ void __launch_bounds__(256)
k_select(const double* __restrict__ logl, const double* __restrict__ logg, int32_t C, const double* __restrict__ S,
         int32_t pc, double* __restrict__ out_x, double* __restrict__ out_acq, int64_t* __restrict__ out_best) { d_select(logl, logg, C, S, pc, out_x, out_acq, out_best); }

// Merge k-split partials into final log-densities (tpe_logpdf entry point).
__global__ void k_finish_logpdf(const double2* __restrict__ part, int ns, int64_t ct_stride,
                                const uint8_t* __restrict__ oob, const double2* __restrict__ fix, int64_t n,
                                double* __restrict__ out) {
  for (int64_t ct = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; ct < n; ct += (int64_t)gridDim.x * blockDim.x) {
    double m = -INFINITY, s = 0.0;
    if (oob != nullptr && oob[ct]) {
      m = fix[ct].x;
      s = fix[ct].y;
    } else {
      for (int i = 0; i < ns; ++i) {
        const double2 v = part[(int64_t)i * ct_stride + ct];
        lse_merge(v.x, v.y, m, s);
      }
    }
    out[ct] = (m == -INFINITY) ? -INFINITY : log(s) + m;
  }
}

// ================================================================================================
// MT19937 on the device: the exact stream of numpy.random.RandomState.random_sample
// (numpy/random/_mt19937.pyx + legacy double: (a >> 5, b >> 6) -> (a * 2^26 + b) / 2^53), so that
// the uniforms of an ask never exist on the host (reference: self._rng.rng draws in
// probability_distributions.py:87,100,138-144).  One CTA: the 624-word state is regenerated block by
// block (the twist of one block is three data-parallel phases of 227 / 227 / 170 words), tempered in
// parallel and converted to doubles; the first `skip` doubles are generated and dropped (a rank that
// owns a later slice of a batch of asks), the next `count` are written.  ~80 ns per block of 312
// doubles; the final state goes back to the host generator.
//   key [624] state words (in/out), pos_io: index of the next unused word of the state (624 = exhausted)
// ================================================================================================
__device__ __forceinline__ uint32_t mt_temper(uint32_t y) {
  y ^= y >> 11;
  y ^= (y << 7) & 0x9d2c5680u;
  y ^= (y << 15) & 0xefc60000u;
  y ^= y >> 18;
  return y;
}
__device__ __forceinline__ uint32_t mt_twist(uint32_t cur, uint32_t nxt, uint32_t far) {
  const uint32_t y = (cur & 0x80000000u) | (nxt & 0x7fffffffu);
  return far ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
}
// Two state buffers (ping-pong) and two warp groups: warps 0-7 regenerate block b + 1 from block b in
// three phases (one 256-thread named barrier each: every "old" read goes to the other buffer) while
// warps 8-23 temper block b and write its doubles; one CTA-wide barrier per block.
constexpr int kMtThreads = 768;
__device__ __forceinline__ void mt_gen_barrier() { asm volatile("bar.sync 1, 256;" ::: "memory"); }
__global__ void __launch_bounds__(kMtThreads, 1)
k_mt19937_uniform(uint32_t* __restrict__ key, int* __restrict__ pos_io, int64_t skip, int64_t count,
                  double* __restrict__ out) {
  __shared__ uint32_t buf[2][624];
  __shared__ uint32_t carry;  // a >> 5 of a double whose second word is the first word of the next block
  const int tid = threadIdx.x;
  const bool gen = tid < 256;
  const int wt = tid - 256;     // writer index 0..511
  for (int i = tid; i < 624; i += kMtThreads) buf[0][i] = key[i];
  int cur = 0;                  // buffer holding the block the outputs are taken from
  int start = *pos_io;          // first unused word of that block
  int64_t gw = 0;               // words consumed before that block's [start, 624) range
  const int64_t total_words = 2 * (skip + count);
  int end_pos = start;
  __syncthreads();
  // blocks that lie entirely inside the dropped prefix: the generator warps alone walk the recurrence
  // (three named barriers per block), the writers rejoin at the first block that is needed
  {
    const int64_t drop_words = 2 * skip;
    int blocks = 0;
    if (gw + (624 - start) <= drop_words && gw + (624 - start) < total_words) {
      blocks = 1 + (int)((drop_words - (gw + (624 - start))) / 624);
      // the block reached after `blocks` regenerations must still be needed
      while (blocks > 0 && gw + (624 - start) + (int64_t)(blocks - 1) * 624 >= total_words) --blocks;
    }
    if (blocks > 0) {
      if (gen) {
        for (int bl = 0; bl < blocks; ++bl) {
          const uint32_t* A = buf[(cur + bl) & 1];
          uint32_t* B = buf[(cur + bl + 1) & 1];
          if (tid < 227) B[tid] = mt_twist(A[tid], A[tid + 1], A[tid + 397]);
          mt_gen_barrier();
          if (tid < 227) B[227 + tid] = mt_twist(A[227 + tid], A[228 + tid], B[tid]);
          mt_gen_barrier();
          if (tid < 170) {
            const int j = 454 + tid;
            B[j] = mt_twist(A[j], (j == 623) ? B[0] : A[j + 1], B[j - 227]);
          }
          mt_gen_barrier();
        }
      }
      gw += (624 - start) + (int64_t)(blocks - 1) * 624;
      cur = (cur + blocks) & 1;
      start = 0;
      end_pos = 0;
      __syncthreads();
    }
  }
  while (gw < total_words) {
    const int64_t avail = 624 - start;
    const int take = (int)((total_words - gw < avail) ? (total_words - gw) : avail);
    const bool more = gw + take < total_words;
    const uint32_t* A = buf[cur];
    uint32_t* B = buf[cur ^ 1];
    if (gen) {
      if (more) {
        if (tid < 227) B[tid] = mt_twist(A[tid], A[tid + 1], A[tid + 397]);
        mt_gen_barrier();
        if (tid < 227) B[227 + tid] = mt_twist(A[227 + tid], A[228 + tid], B[tid]);
        mt_gen_barrier();
        if (tid < 170) {
          const int j = 454 + tid;
          B[j] = mt_twist(A[j], (j == 623) ? B[0] : A[j + 1], B[j - 227]);
        }
      }
    } else {
      // words [start, start + take) of A are global words [gw, gw + take); a double = words (2d, 2d + 1)
      const int odd = (int)(gw & 1);               // the first word completes the previous block's double
      if (odd && wt == 0 && take > 0) {
        const int64_t d = gw >> 1;
        const uint32_t a = carry, b2 = mt_temper(A[start]) >> 6;
        if (d >= skip) out[d - skip] = ((double)a * 67108864.0 + (double)b2) / 9007199254740992.0;
      }
      const int pairs = (take - odd) / 2;           // whole doubles inside this block
      for (int p = wt; p < pairs; p += 512) {
        const int j = start + odd + 2 * p;
        const int64_t d = (gw + odd) / 2 + p;
        const uint32_t a = mt_temper(A[j]) >> 5, b2 = mt_temper(A[j + 1]) >> 6;
        if (d >= skip) out[d - skip] = ((double)a * 67108864.0 + (double)b2) / 9007199254740992.0;
      }
    }
    __syncthreads();
    // a trailing first-half word is published after the barrier (its reader, wt == 0 above, is done)
    if (tid == 256 && take > 0 && ((take - (int)(gw & 1)) & 1)) carry = mt_temper(A[start + take - 1]) >> 5;
    gw += take;
    if (more) {
      cur ^= 1;
      start = 0;
      end_pos = 0;
    } else {
      end_pos = start + take;
    }
    // no second barrier: `carry` is written and read by the same thread (tid 256), and the next block's
    // writes go to the buffer whose readers all passed the barrier above
  }
  __syncthreads();
  for (int i = tid; i < 624; i += kMtThreads) key[i] = buf[cur][i];
  if (tid == 0) *pos_io = end_pos;
}

// ================================================================================================
// Multi-CTA MT19937: jump-ahead.  The state transition is linear over GF(2) with a primitive characteristic
// polynomial phi (degree 19937), so advancing by J words is multiplication by g_J = x^J mod phi, and in terms of
// the word sequence the generator emits:  x_{J+j} = XOR_{i : g_J[i] = 1} x_{i+j}  for every j >= 1 (Haramoto et
// al. 2008; derivation and the table generator: tools/gen_mt_jump.py).  The table holds g = x^(2^k - 1) mod phi,
// so one application moves a 624-word key by exactly 2^k words:  new[j'] = XOR_i g_i W[i + j' + 1].
//
// k_mt19937_uniform_mc: CTA c produces doubles [c * chunk, (c + 1) * chunk) of the requested stretch.  It jumps
// from the caller's state to the 512-word boundary below its first word (one table polynomial per set bit of the
// distance) and then runs the same block generator as the single-CTA kernel.  A rank that owns a later slice of a
// batch (`skip`) no longer walks the prefix: the 6.5 M uniforms of 8192 asks on one CTA become ~15 jumps
// plus 1/G of the stream.
//
// One jump = (a) 32 more blocks generated into a 33 x 624-word shared buffer (W[0..623] = key), (b) the GF(2)
// convolution with the lanes on the output axis: lane l owns outputs 20 l .. 20 l + 19 in registers, warp w walks
// the polynomial words w, w + 24, ...; per polynomial word a 51-word window of W is loaded once (13 x LDS.128,
// conflict-free at a 20-word lane stride) and every set bit costs 20 register XORs; (c) XOR-reduction over the
// 24 warps.
// ================================================================================================
constexpr int kMtJumpWords = 33 * 624;          // W[0 .. 20591]: needs up to W[19936 + 624]
constexpr int kMtJumpPad = 64;                  // windows of the last lane / last polynomial word run past the end
constexpr int kMtJumpOut = 20;                  // outputs per lane
constexpr size_t kMtJumpSmem = (size_t)(4 + kMtJumpWords + kMtJumpPad) * 4 + (size_t)24 * 640 * 4 + 2 * 624 * 4 + 16;

// generator warps only (tid < 256): block `A + 624` from block `A`
__device__ __forceinline__ void mt_next_block(const uint32_t* A, uint32_t* B, int tid) {
  if (tid < 227) B[tid] = mt_twist(A[tid], A[tid + 1], A[tid + 397]);
  mt_gen_barrier();
  if (tid < 227) B[227 + tid] = mt_twist(A[227 + tid], A[228 + tid], B[tid]);
  mt_gen_barrier();
  if (tid < 170) {
    const int j = 454 + tid;
    B[j] = mt_twist(A[j], (j == 623) ? B[0] : A[j + 1], B[j - 227]);
  }
  mt_gen_barrier();
}

// W: shared, W[0..623] holds the key on entry and the key advanced by 2^k words on exit (all 768 threads call).
// `red`: 24 x 640 words of shared scratch.  W must be 16-byte aligned at W + 1 (see the caller's layout).
__device__ __forceinline__ void mt_jump_apply(uint32_t* W, uint32_t* red, const uint32_t* __restrict__ g) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid < 256)
    for (int b = 1; b < 33; ++b) mt_next_block(W + 624 * (b - 1), W + 624 * b, tid);
  __syncthreads();
  uint32_t acc[kMtJumpOut];
#pragma unroll
  for (int q = 0; q < kMtJumpOut; ++q) acc[q] = 0u;
  for (int ib = warp; ib < 624; ib += 24) {
    const uint32_t G = __ldg(g + ib);
    if (G == 0u) continue;
    // window: W[32 ib + 20 lane + 1 + (0 .. 51)]
    uint32_t win[52];
    const uint4* src = reinterpret_cast<const uint4*>(W + 1 + 32 * ib + kMtJumpOut * lane);
#pragma unroll
    for (int v = 0; v < 13; ++v) {
      const uint4 x = src[v];
      win[4 * v] = x.x; win[4 * v + 1] = x.y; win[4 * v + 2] = x.z; win[4 * v + 3] = x.w;
    }
#pragma unroll
    for (int t = 0; t < 32; ++t) {
      if ((G >> t) & 1u) {   // uniform over the warp
#pragma unroll
        for (int q = 0; q < kMtJumpOut; ++q) acc[q] ^= win[t + q];
      }
    }
  }
#pragma unroll
  for (int q = 0; q < kMtJumpOut; ++q) red[warp * 640 + kMtJumpOut * lane + q] = acc[q];
  __syncthreads();
  if (tid < 624) {
    uint32_t v = 0u;
#pragma unroll
    for (int w = 0; w < 24; ++w) v ^= red[w * 640 + tid];
    W[tid] = v;
  }
  __syncthreads();
}

// The block generator of k_mt19937_uniform on caller-provided shared buffers (buf[2][624], carry); all 768 threads.
// Produces doubles [0, count) from the state (buf[0], start); returns the buffer index and position of the end state.
__device__ __forceinline__ void mt_emit(uint32_t (*buf)[624], uint32_t* carry, int start, int64_t count,
                                        double* __restrict__ out, int& cur_out, int& end_out) {
  const int tid = threadIdx.x;
  const bool gen = tid < 256;
  const int wt = tid - 256;
  int cur = 0, end_pos = start;
  int64_t gw = 0;
  const int64_t total_words = 2 * count;
  while (gw < total_words) {
    const int64_t avail = 624 - start;
    const int take = (int)((total_words - gw < avail) ? (total_words - gw) : avail);
    const bool more = gw + take < total_words;
    const uint32_t* A = buf[cur];
    uint32_t* B = buf[cur ^ 1];
    if (gen) {
      if (more) {
        if (tid < 227) B[tid] = mt_twist(A[tid], A[tid + 1], A[tid + 397]);
        mt_gen_barrier();
        if (tid < 227) B[227 + tid] = mt_twist(A[227 + tid], A[228 + tid], B[tid]);
        mt_gen_barrier();
        if (tid < 170) {
          const int j = 454 + tid;
          B[j] = mt_twist(A[j], (j == 623) ? B[0] : A[j + 1], B[j - 227]);
        }
      }
    } else {
      const int odd = (int)(gw & 1);
      if (odd && wt == 0 && take > 0) {
        const int64_t d = gw >> 1;
        const uint32_t a = *carry, b2 = mt_temper(A[start]) >> 6;
        out[d] = ((double)a * 67108864.0 + (double)b2) / 9007199254740992.0;
      }
      const int pairs = (take - odd) / 2;
      for (int p = wt; p < pairs; p += 512) {
        const int j = start + odd + 2 * p;
        const int64_t d = (gw + odd) / 2 + p;
        const uint32_t a = mt_temper(A[j]) >> 5, b2 = mt_temper(A[j + 1]) >> 6;
        out[d] = ((double)a * 67108864.0 + (double)b2) / 9007199254740992.0;
      }
    }
    __syncthreads();
    if (tid == 256 && take > 0 && ((take - (int)(gw & 1)) & 1)) *carry = mt_temper(A[start + take - 1]) >> 5;
    gw += take;
    if (more) {
      cur ^= 1;
      start = 0;
      end_pos = 0;
    } else {
      end_pos = start + take;
    }
  }
  __syncthreads();
  cur_out = cur;
  end_out = end_pos;
}

// key_in[625] = 624 state words + position (read-only: every CTA starts from it); key_out[625] = the state after
// the (skip + count) draws, written by the CTA that produces the last double.  jump_table: kMtJumpTable on the device.
__global__ void __launch_bounds__(kMtThreads, 1)
k_mt19937_uniform_mc(const uint32_t* __restrict__ key_in, int64_t skip, int64_t count, int64_t chunk,
                     const uint32_t* __restrict__ jump_table, int kmin, int kmax, double* __restrict__ out,
                     uint32_t* __restrict__ key_out) {
  extern __shared__ __align__(16) uint32_t mt_smem[];
  uint32_t* W = mt_smem + 3;                               // W + 1 is 16-byte aligned
  uint32_t* red = mt_smem + 4 + kMtJumpWords + kMtJumpPad;
  uint32_t (*buf)[624] = reinterpret_cast<uint32_t (*)[624]>(red + 24 * 640);
  uint32_t* carry = red + 24 * 640 + 2 * 624;
  const int tid = threadIdx.x;
  const int64_t first = (int64_t)blockIdx.x * chunk;
  const int64_t mine = (count - first < chunk) ? (count - first) : chunk;
  if (mine <= 0) return;
  for (int i = tid; i < 624; i += kMtThreads) W[i] = key_in[i];
  for (int i = tid; i < kMtJumpPad; i += kMtThreads) W[kMtJumpWords + i] = 0u;
  // numpy regenerates its 624-word state block by block from the seed, and key_in is such a block: the CTA first
  // jumps to the largest multiple of 512 below the block that holds its first word (one polynomial per set bit),
  // then slides the window forward to that block -- so the walk that follows, and the end state, sit on numpy's
  // own block grid (the state handed back to RandomState.set_state is the one numpy itself would hold)
  const int64_t w0 = (int64_t)key_in[624] + 2 * (skip + first);   // first word of this CTA, relative to key[0]
  const int64_t blk = (w0 >= 624) ? ((w0 - 1) / 624) * 624 : 0;   // numpy: a block is replaced only when a word beyond it is needed
  const int64_t dist = blk & ~(int64_t)511;
  const int shift = (int)(blk - dist);                            // 0..511
  const int start = (int)(w0 - blk);                              // 0..624
  __syncthreads();
  for (int k = kmin; k <= kmax; ++k)
    if ((dist >> k) & 1) mt_jump_apply(W, red, jump_table + (size_t)(k - kmin) * 624);
  if (shift > 0) {
    if (tid < 256) mt_next_block(W, W + 624, tid);
    __syncthreads();
  }
  for (int i = tid; i < 624; i += kMtThreads) buf[0][i] = W[shift + i];
  __syncthreads();
  int cur, end_pos;
  mt_emit(buf, carry, start, mine, out + first, cur, end_pos);
  if (first + mine >= count) {
    for (int i = tid; i < 624; i += kMtThreads) key_out[i] = buf[cur][i];
    if (tid == 0) key_out[624] = (uint32_t)end_pos;
  }
}

// ================================================================================================
// fp64 FMA peak probe (roofline denominator for the compute-bound grid kernel)
// ================================================================================================
__global__ void k_fp64_probe(double* out, int iters) {
  double a0 = threadIdx.x * 1e-9, a1 = a0 + 1, a2 = a0 + 2, a3 = a0 + 3, a4 = a0 + 4, a5 = a0 + 5, a6 = a0 + 6,
         a7 = a0 + 7;
  const double m = 1.0000001, c = 1e-9;
  for (int i = 0; i < iters; ++i) {
    a0 = fma(a0, m, c); a1 = fma(a1, m, c); a2 = fma(a2, m, c); a3 = fma(a3, m, c);
    a4 = fma(a4, m, c); a5 = fma(a5, m, c); a6 = fma(a6, m, c); a7 = fma(a7, m, c);
  }
  out[blockIdx.x * blockDim.x + threadIdx.x] = a0 + a1 + a2 + a3 + a4 + a5 + a6 + a7;
}

}  // namespace tpe
