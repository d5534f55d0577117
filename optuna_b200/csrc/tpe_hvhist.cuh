// Hypervolume history of a multi-objective study (optuna/visualization/_hypervolume_history.py:83-138,
// _get_hypervolume_history_info), restated so that the expensive part runs in parallel.
//
// v: [n, M] sign-normalised objective values in trial order, r: the sign-normalised reference point.
//   eligible_i  feasible and no coordinate of v_i is > r
//   added_i     eligible_i and no eligible j < i has v_j <= v_i in every coordinate   (k_hh_added)
//   death_j     first added k > j with v_k <= v_j (n if none)                          (k_hh_death)
//   front_i     {added j < i : death_j >= i}: the reference's front when it reaches trial i, before it drops
//               the members that i dominates
//   history     at every added i: hv = hv + prod(r - v_i), then (unless i is the first added trial)
//               hv = hv - HV(max(front_i, v_i)); every other trial repeats the previous value    (k_hh_scan)
// Only the per-trial HV(max(front_i, v_i)) are expensive, and they are independent.  compute_hypervolume first
// applies np.unique and a Pareto filter, so its result depends on the unique non-dominated part of the clipped set
// only: k_hh_front gathers, clips and filters (one warp per added trial), k_hh_hv evaluates the survivors with the
// exact MOTPE hypervolume code (hv_2d / hv3_warp / hv_nd_warp, bit-identical to hypervolume()).
//
// The per-point predicates are `__host__ __device__` so that tests/csrc/hvhist_shim.cu runs the same gather / clip /
// filter / order on the host; TPE_HVHIST_HOST_ONLY leaves the kernels out of that build.
#pragma once
#include "tpe_motpe.cuh"

namespace tpe {

// a <= b in every coordinate
TPE_HD bool hh_le(const double* a, const double* b, int M) {
  for (int j = 0; j < M; ++j)
    if (!(a[j] <= b[j])) return false;
  return true;
}

// row q of the clipped front: max(front member, v_i) (np.maximum; values hold no NaN)
TPE_HD void hh_clip_row(const double* member, const double* vi, int M, double* out) {
  for (int j = 0; j < M; ++j) out[j] = member[j] > vi[j] ? member[j] : vi[j];
}

// Is row k of the clipped set C [c, M] dropped by np.unique + the Pareto filter?  Yes when another row is <= it
// everywhere and differs from it, or equals it and comes first (the first copy of a vector stands for all copies).
TPE_HD bool hh_dropped(const double* C, int c, int k, int M) {
  const double* me = C + (size_t)k * M;
  for (int q = 0; q < c; ++q) {
    if (q == k) continue;
    const double* o = C + (size_t)q * M;
    if (!hh_le(o, me, M)) continue;
    if (q < k || lex_cmp(o, me, M) != 0) return true;
  }
  return false;
}

// position of kept row k among the kept rows in lexicographic order (kept rows are unique)
TPE_HD int hh_lexrank(const double* C, const uint8_t* keep, int c, int k, int M) {
  const double* me = C + (size_t)k * M;
  int r = 0;
  for (int q = 0; q < c; ++q) r += (keep[q] && lex_cmp(C + (size_t)q * M, me, M) < 0) ? 1 : 0;
  return r;
}

}  // namespace tpe

#if !defined(TPE_HVHIST_HOST_ONLY)
#include "tpe_motpe_kernels.cuh"

namespace tpe {

// threads per CTA of the tiled kernels (one trial each) = rows per tile.  The kernels declare a minimum of 4 CTAs
// per SM: that lets ptxas use up to 128 registers, where without it it kept them at 32 and spilled.
constexpr int kHhThreads = 128;

// doubles of k_hh_hv scratch for a front of m points
inline size_t hh_hv_scratch_doubles(int m, int M) {
  if (M == 2) return 0;                                   // hv_2d runs on the survivors in place
  if (M == 3) return (size_t)5 * m + 8;                   // hv3_warp: sorted rows 3m, terms m, ranks m ints
  return hv_warp_scratch_doubles(m, M) + (size_t)32 * hv_lane_doubles(m, M);
}

__global__ void k_hh_eligible(const double* __restrict__ v, const uint8_t* __restrict__ feasible, int n, int M,
                              const double* __restrict__ ref, uint8_t* __restrict__ elig) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  bool e = feasible ? feasible[i] != 0 : true;
  for (int j = 0; j < M; ++j) e = e && !(v[(size_t)i * M + j] > ref[j]);
  elig[i] = e;
}

// added_i: one thread per trial, earlier trials streamed through shared memory in tiles of kHhThreads rows;
// the CTA stops as soon as every one of its trials has met an earlier eligible trial that is <= it.
// Dynamic shared memory: hh_added_smem(M).
__host__ __device__ inline size_t hh_added_smem(int M) { return (size_t)2 * M * kHhThreads * 8 + kHhThreads; }
__global__ void __launch_bounds__(kHhThreads, 4)
k_hh_added(const double* __restrict__ v, int n, int M, const uint8_t* __restrict__ elig, uint8_t* __restrict__ added) {
  extern __shared__ double hh_sm[];
  double* s_me = hh_sm;                              // [M][kHhThreads]: this thread's row, column-major
  double* s_t = hh_sm + (size_t)M * kHhThreads;      // [kHhThreads][M]: tile of earlier rows
  uint8_t* s_e = reinterpret_cast<uint8_t*>(s_t + (size_t)M * kHhThreads);
  const int t = threadIdx.x;
  const int i0 = blockIdx.x * kHhThreads, i = i0 + t;
  const bool live = i < n && elig[i];
  for (int j = 0; j < M; ++j) s_me[j * kHhThreads + t] = live ? v[(size_t)i * M + j] : 0.0;
  bool covered = !live;
  const int jend = min(n, i0 + kHhThreads);
  for (int j0 = 0; j0 < jend; j0 += kHhThreads) {
    if (__syncthreads_and(covered)) break;           // also keeps the previous tile until every thread is done
    const int rows = min(kHhThreads, n - j0);
    for (int q = t; q < rows * M; q += kHhThreads) s_t[q] = v[(size_t)j0 * M + q];
    if (t < rows) s_e[t] = elig[j0 + t];
    __syncthreads();
    if (!covered) {
      const int rmax = min(rows, i - j0);
      for (int r = 0; r < rmax; ++r) {
        if (!s_e[r]) continue;
        bool le = true;
        for (int j = 0; j < M && le; ++j) le = s_t[r * M + j] <= s_me[j * kHhThreads + t];
        if (le) { covered = true; break; }
      }
    }
  }
  if (i < n) added[i] = live && !covered;
}

// Order-preserving compaction of the added trials (one CTA of 1024 threads): list[0..K) ascending trial indices,
// rank[i] = added trials in [0, i], *K_out = K.
__global__ void __launch_bounds__(1024)
k_hh_compact(const uint8_t* __restrict__ added, int n, int32_t* __restrict__ list, int32_t* __restrict__ rank,
             int32_t* __restrict__ K_out) {
  __shared__ int s_w[32];
  const int t = threadIdx.x, lane = t & 31, w = t >> 5;
  int base = 0;
  for (int c0 = 0; c0 < n; c0 += 1024) {
    const int i = c0 + t;
    const int f = (i < n && added[i]) ? 1 : 0;
    int x = f;
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) s_w[w] = x;
    __syncthreads();
    if (w == 0) {
      int s = s_w[lane];
      for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, s, o);
        if (lane >= o) s += y;
      }
      s_w[lane] = s;
    }
    __syncthreads();
    const int incl = base + x + (w ? s_w[w - 1] : 0);
    if (i < n) {
      rank[i] = incl;
      if (f) list[incl - 1] = i;
    }
    base += s_w[31];
    __syncthreads();
  }
  if (t == 0) *K_out = base;
}

// death over the list of added trials (one thread per added trial, later added rows in shared-memory tiles),
// and incl[p] = prod(r - v) of the trial, multiplied from the first coordinate on as np.prod does.
__global__ void __launch_bounds__(kHhThreads, 4)
k_hh_death(const double* __restrict__ v, int n, int M, const int32_t* __restrict__ list, int K,
           const double* __restrict__ ref, int32_t* __restrict__ death, double* __restrict__ incl) {
  extern __shared__ double hh_sm[];
  double* s_me = hh_sm;
  double* s_t = hh_sm + (size_t)M * kHhThreads;
  const int t = threadIdx.x;
  const int p0 = blockIdx.x * kHhThreads, p = p0 + t;
  const bool live = p < K;
  const int ip = live ? list[p] : 0;
  double pr = 1.0;
  for (int j = 0; j < M; ++j) {
    const double x = live ? v[(size_t)ip * M + j] : 0.0;
    s_me[j * kHhThreads + t] = x;
    const double d = TPE_SUB(ref[j], x);
    pr = j == 0 ? d : TPE_MUL(pr, d);
  }
  int found = live ? -1 : 0;
  for (int q0 = p0 + 1; q0 < K; q0 += kHhThreads) {
    if (__syncthreads_and(found >= 0)) break;
    const int rows = min(kHhThreads, K - q0);
    for (int e = t; e < rows * M; e += kHhThreads) {
      const int r = e / M;
      s_t[e] = v[(size_t)list[q0 + r] * M + (e - r * M)];
    }
    __syncthreads();
    if (found < 0) {
      for (int r = max(0, p + 1 - q0); r < rows; ++r) {
        bool le = true;
        for (int j = 0; j < M && le; ++j) le = s_t[r * M + j] <= s_me[j * kHhThreads + t];
        if (le) { found = list[q0 + r]; break; }
      }
    }
  }
  if (live) {
    death[p] = found >= 0 ? found : n;
    incl[p] = pr;
  }
}

// |front_i| of every added trial: the earlier added trials still alive when it arrives
__global__ void k_hh_count(const int32_t* __restrict__ list, const int32_t* __restrict__ death, int K,
                           int32_t* __restrict__ cnt) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= K) return;
  const int ip = list[p];
  int c = 0;
  for (int q = 0; q < p; ++q) c += __ldg(death + q) >= ip ? 1 : 0;
  cnt[p] = c;
}

// One warp per added trial p in [pa, pb): gather front_i, clip it by v_i, keep its unique non-dominated rows and
// write them lexicographically sorted to surv (np.unique(axis=0) + _is_pareto_front order).  The rows of trial p
// start at row off[p] - off[pa] of clip / surv / keep (off: prefix sum of cnt).  m[p] = rows kept.
__global__ void __launch_bounds__(kHhThreads, 4)
k_hh_front(const double* __restrict__ v, int M, const int32_t* __restrict__ list, const int32_t* __restrict__ death,
           const int32_t* __restrict__ cnt, const int64_t* __restrict__ off, int pa, int pb, double* __restrict__ clip,
           uint8_t* __restrict__ keep, double* __restrict__ surv, int32_t* __restrict__ m_out) {
  const int lane = threadIdx.x & 31;
  const int p = pa + blockIdx.x * (kHhThreads / 32) + (threadIdx.x >> 5);
  if (p >= pb) return;
  const int c = cnt[p];
  if (c == 0) {   // the first added trial
    if (lane == 0) m_out[p] = 0;
    return;
  }
  const int64_t row0 = off[p] - off[pa];
  double* C = clip + row0 * M;
  uint8_t* kp = keep + row0;
  double* S = surv + row0 * M;
  const int ip = list[p];
  const double* vi = v + (size_t)ip * M;
  int w = 0;
  for (int q0 = 0; q0 < p; q0 += 32) {
    const int q = q0 + lane;
    const bool in = q < p && death[q] >= ip;
    const unsigned b = __ballot_sync(0xffffffffu, in);
    if (in) hh_clip_row(v + (size_t)list[q] * M, vi, M, C + (size_t)(w + __popc(b & ((1u << lane) - 1))) * M);
    w += __popc(b);
  }
  __syncwarp();
  for (int k = lane; k < c; k += 32) kp[k] = !hh_dropped(C, c, k, M);
  __syncwarp();
  int kept = 0;
  for (int k = lane; k < c; k += 32) {
    if (!kp[k]) continue;
    const int r = hh_lexrank(C, kp, c, k, M);
    for (int j = 0; j < M; ++j) S[(size_t)r * M + j] = C[(size_t)k * M + j];
    ++kept;
  }
  for (int o = 16; o; o >>= 1) kept += __shfl_xor_sync(0xffffffffu, kept, o);
  if (lane == 0) m_out[p] = kept;
}

// One warp per added trial p in [pa, pb) (p > 0): hv[p] = HV of its m[p] sorted survivors, with the exact
// hypervolume code of MOTPE.  The survivors are those k_hh_front wrote for the chunk starting at p_base; the
// scratch of trial p is arena + soff[p - p_base], hh_hv_scratch_doubles(m[p], M) doubles.
__global__ void __launch_bounds__(kHhThreads, 4)
k_hh_hv(int M, const int32_t* __restrict__ cnt, const int64_t* __restrict__ off, int p_base, int pa, int pb,
        const double* __restrict__ surv, const int32_t* __restrict__ m_in, const double* __restrict__ ref,
        const int64_t* __restrict__ soff, double* __restrict__ arena, double* __restrict__ hv) {
  const int lane = threadIdx.x & 31;
  const int p = pa + blockIdx.x * (kHhThreads / 32) + (threadIdx.x >> 5);
  if (p >= pb) return;
  if (cnt[p] == 0) {
    if (lane == 0) hv[p] = 0.0;
    return;
  }
  const int m = m_in[p];
  const double* S = surv + (off[p] - off[p_base]) * M;
  double* ws = arena + soff[p - p_base];
  double h;
  if (M == 2) {
    h = 0.0;
    if (lane == 0) {
      h = (isfinite(ref[0]) && isfinite(ref[1])) ? hv_2d(S, m, ref) : INFINITY;
      h = isfinite(h) ? h : INFINITY;
    }
  } else if (M == 3) {
    // the survivors are lexsorted: hv3_warp's stable order by x keeps it, as hypervolume()'s hv_3d input is
    h = hv3_warp(S, m, ref, ws, ws + (size_t)3 * m, reinterpret_cast<int*>(ws + (size_t)4 * m));
  } else {
    // already unique, non-dominated and lexsorted: assume_pareto's stable sort by coordinate 0 keeps that order
    double* lanes = ws + hv_warp_scratch_doubles(m, M);
    h = hv_nd_warp(S, m, M, ref, true, ws, lanes + (size_t)lane * hv_lane_doubles(m, M));
  }
  if (lane == 0) hv[p] = h;
}

// The history in trial order, by one thread: exactly the reference's two fp64 operations per added trial.
__global__ void k_hh_scan(int K, const double* __restrict__ incl, const double* __restrict__ hv,
                          double* __restrict__ cum) {
  double h = 0.0;
  for (int p = 0; p < K; ++p) {
    h = TPE_ADD(h, incl[p]);
    if (p > 0) h = TPE_SUB(h, hv[p]);
    cum[p] = h;
  }
}

__global__ void k_hh_fill(const int32_t* __restrict__ rank, int n, const double* __restrict__ cum,
                          double* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int r = rank[i];
  out[i] = r ? cum[r - 1] : 0.0;
}

}  // namespace tpe
#endif
