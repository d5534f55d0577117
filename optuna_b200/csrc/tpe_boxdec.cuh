// Non-dominated box decomposition of GPSampler's log-EHVI (optuna/_hypervolume/box_decomposition.py:30-157,
// get_non_dominated_box_bounds), bit for bit and in the reference's row order.  The algorithm does no arithmetic: only
// comparisons, copies, negations and maxima.
//
//   1. the input rows in np.unique(axis=0) order (lexicographic by ==, so -0.0 ties with +0.0; repeats dropped), then
//      their Pareto front: M stable radix passes (k_radix_sort_coop_perm, last column first), k_bd_unique, the Pareto
//      filter of tpe_pareto.cuh;
//   2. pass 1, _get_upper_bound_set (Lacour et al. 2017, Alg. 2): k_bd_pass over that front and the reference point;
//   3. the pass's upper bounds negated, again in unique-lexsorted order and filtered to their Pareto front;
//   4. pass 2: k_bd_pass over that front with a reference point of +inf;
//   5. _get_box_bounds: k_bd_boxes, a running maximum of the defining points and the non-empty test, then the kept
//      rows in order, negated and swapped.
//
// k_bd_pass is one persistent CTA that runs every step of a pass.  Its state is an append-only pool of bounds (upper
// bound [M] and defining points [M][M]) with a live flag:
//   - order: the reference rebuilds the set each step as vstack([survivors in order, children]), the children ordered
//     by their parent's position, then by dimension j.  The step appends its children in (parent pool index, j) order
//     and clears the parents' live flags, so the live rows read in pool order are the reference's array;
//   - retirement: the points of a pass come in ascending coordinate 0, so a bound with u_0 <= z_0 never again meets
//     the strict test z < u.  Such a bound stays live but leaves the active list the steps scan; the child made in
//     dimension 0 (u_0 = z_0) is born retired.  The active list is kept in pool order, so the dominated bounds come
//     out of the scan in pool order;
//   - overflow: a step whose children do not fit the pool stops the pass and reports it; the host grows the pool and
//     runs the pass again.  Nothing is truncated.
// Every ordered write goes through a block-wide exclusive scan; no atomics.
#pragma once
#include "tpe_common.cuh"

namespace tpe {
namespace boxdec {

constexpr int THREADS = 1024;
constexpr int MAX_M = 24;   // one lane per objective in a warp

// block-wide exclusive scan of a 64-bit value (blockDim.x == 1024): {prefix, total}.  s: 32 long longs of shared memory.
__device__ __forceinline__ longlong2 block_scan_1024(long long v, long long* s) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  long long incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const long long u = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += u;
  }
  __syncthreads();   // the previous call's readers are done with s
  if (lane == 31) s[warp] = incl;
  __syncthreads();
  const long long w = s[lane];
  long long winc = w;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const long long u = __shfl_up_sync(0xffffffffu, winc, o);
    if (lane >= o) winc += u;
  }
  const long long total = __shfl_sync(0xffffffffu, winc, 31);
  const long long wbase = __shfl_sync(0xffffffffu, winc - w, warp);
  return make_longlong2(wbase + incl - v, total);
}

// keep[p] = 1 unless sorted row p compares == to sorted row p - 1 in every column (np.unique's duplicate mask)
__global__ void k_bd_unique(const double* __restrict__ rows, const int32_t* __restrict__ order, int n, int M,
                            uint8_t* __restrict__ keep) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  bool differs = p == 0;
  if (!differs) {
    const double* a = rows + (size_t)order[p] * M;
    const double* b = rows + (size_t)order[p - 1] * M;
    for (int j = 0; j < M && !differs; ++j) differs = a[j] != b[j];
  }
  keep[p] = differs ? 1 : 0;
}

// sel[0, *count) = the positions p < n with keep[p], ascending.  One CTA of 1024 threads, a contiguous range each.
__global__ void __launch_bounds__(THREADS, 1)
k_bd_select(const uint8_t* __restrict__ keep, int n, int32_t* __restrict__ sel, int* __restrict__ count) {
  __shared__ long long s_scan[32];
  const int per = (n + THREADS - 1) / THREADS;
  const int lo = min(n, (int)threadIdx.x * per), hi = min(n, lo + per);
  int c = 0;
  for (int p = lo; p < hi; ++p) c += keep[p];
  const longlong2 r = block_scan_1024(c, s_scan);
  int q = (int)r.x;
  for (int p = lo; p < hi; ++p)
    if (keep[p]) sel[q++] = p;
  if (threadIdx.x == 0) *count = (int)r.y;
}

// dst[r, :] = (neg ? -1 : 1) * src[i1[i2[r]], :], an absent index array being the identity
__global__ void k_bd_gather(const double* __restrict__ src, const int32_t* __restrict__ i1,
                            const int32_t* __restrict__ i2, int n, int M, bool neg, double* __restrict__ dst) {
  const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (e >= (int64_t)n * M) return;
  const int r = (int)(e / M), j = (int)(e - (int64_t)r * M);
  int p = i2 ? i2[r] : r;
  if (i1) p = i1[p];
  const double x = src[(size_t)p * M + j];
  dst[e] = neg ? -x : x;
}

// One pass of _get_upper_bound_set (box_decomposition.py:30-93) over the sorted front [nf, M] from the reference point
// ref [M].  Pool of cap bounds: ub [cap, M], dp [cap, M, M] (dp[i, k] = z^k(u_i)), live [cap].  act_a / act_b: the
// active list, double-buffered; dlist, dmask, doff: a step's dominated bounds, their update masks and child offsets
// ([cap] each).  stat[0] = bounds in the pool at the end, stat[1] = 1 + the step that overflowed the pool, or 0.
__global__ void __launch_bounds__(THREADS, 1)
k_bd_pass(const double* __restrict__ front, int nf, int M, const double* __restrict__ ref, double* __restrict__ ub,
          double* __restrict__ dp, uint8_t* __restrict__ live, int32_t* __restrict__ act_a, int32_t* __restrict__ act_b,
          int32_t* __restrict__ dlist, uint32_t* __restrict__ dmask, int32_t* __restrict__ doff, int cap,
          int* __restrict__ stat) {
  __shared__ double z[MAX_M];
  __shared__ long long s_scan[32];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int MM = M * M;
  // Line 1 of Alg. 2: the reference point, its defining points -inf but z^k_k = ref_k
  if (t < M) ub[t] = ref[t];
  for (int e = t; e < MM; e += THREADS) dp[e] = (e / M == e % M) ? ref[e % M] : -INFINITY;
  if (t == 0) {
    live[0] = 1;
    act_a[0] = 0;
  }
  int n_act = 1, pool = 1, overflow = 0;
  int32_t* act = act_a;
  int32_t* nxt = act_b;
  for (int s = 0; s < nf; ++s) {
    if (t < M) z[t] = front[(size_t)s * M + t];
    __syncthreads();   // z, and every write of the previous step
    const double z0 = z[0];
    // A. the active bounds, in pool order: dominated (z < u everywhere), kept (u_0 > z_0) or retired
    const int per = (n_act + THREADS - 1) / THREADS;
    const int lo = min(n_act, t * per), hi = min(n_act, lo + per);
    int nk = 0, nd = 0;
    for (int p = lo; p < hi; ++p) {
      const double* u = ub + (size_t)act[p] * M;
      bool dom = true;
      for (int j = 0; j < M && dom; ++j) dom = z[j] < u[j];
      nd += dom;
      nk += !dom && u[0] > z0;
    }
    const longlong2 sc = block_scan_1024(((long long)nk << 32) | nd, s_scan);
    int qk = (int)(sc.x >> 32), qd = (int)(sc.x & 0xffffffff);
    const int n_keep = (int)(sc.y >> 32), n_dom = (int)(sc.y & 0xffffffff);
    for (int p = lo; p < hi; ++p) {
      const int a = act[p];
      const double* u = ub + (size_t)a * M;
      bool dom = true;
      for (int j = 0; j < M && dom; ++j) dom = z[j] < u[j];
      if (dom) {
        dlist[qd++] = a;
        live[a] = 0;
      } else if (u[0] > z0) {
        nxt[qk++] = a;
      }
    }
    if (n_dom > 0) {
      __syncthreads();   // dlist
      // B1. update mask of each dominated bound (box_decomposition.py:71): j = 0 always, j >= 1 when
      //     z_j >= max_{k != j} z^k_j(u); lane j of the bound's warp decides dimension j
      for (int r = warp; r < n_dom; r += THREADS / 32) {
        const double* d = dp + (size_t)dlist[r] * MM;
        bool upd = false;
        if (lane < M) {
          upd = true;
          if (lane > 0) {
            double m = -INFINITY;
            for (int k = 0; k < M; ++k)
              if (k != lane) m = fmax(m, d[k * M + lane]);
            upd = z[lane] >= m;
          }
        }
        const unsigned mask = __ballot_sync(0xffffffffu, upd);
        if (lane == 0) dmask[r] = mask;
      }
      __syncthreads();
      // B2. child offsets: a bound's children follow those of the dominated bounds before it
      const int per2 = (n_dom + THREADS - 1) / THREADS;
      const int lo2 = min(n_dom, t * per2), hi2 = min(n_dom, lo2 + per2);
      int c = 0;
      for (int r = lo2; r < hi2; ++r) c += __popc(dmask[r]);
      const longlong2 so = block_scan_1024(c, s_scan);
      int q = (int)so.x;
      for (int r = lo2; r < hi2; ++r) {
        doff[r] = q;
        q += __popc(dmask[r]);
      }
      const int n_child = (int)so.y;
      if ((long long)pool + n_child > cap) {
        overflow = s + 1;
        break;
      }
      __syncthreads();   // doff
      // B3. the children, bound r's at pool + doff[r] in ascending j: (z_j, u_-j) with z^j = z (Alg. 2, Lines 2-3);
      //     all but the dimension-0 child join the active list after the kept bounds
      for (int r = warp; r < n_dom; r += THREADS / 32) {
        const int a = dlist[r];
        unsigned mask = dmask[r];
        const int base = pool + doff[r];
        const double* pu = ub + (size_t)a * M;
        const double* pd = dp + (size_t)a * MM;
        for (int c2 = 0; mask; ++c2, mask &= mask - 1) {
          const int j = __ffs(mask) - 1;
          const int idx = base + c2;
          double* cu = ub + (size_t)idx * M;
          double* cd = dp + (size_t)idx * MM;
          for (int l = lane; l < M; l += 32) cu[l] = l == j ? z[l] : pu[l];
          for (int e = lane; e < MM; e += 32) cd[e] = e / M == j ? z[e - j * M] : pd[e];
          if (lane == 0) {
            live[idx] = 1;
            if (c2 > 0) nxt[n_keep + doff[r] - r + c2 - 1] = idx;
          }
        }
      }
      n_act = n_keep + n_child - n_dom;
      pool += n_child;
    } else {
      n_act = n_keep;
    }
    int32_t* tmp = act;
    act = nxt;
    nxt = tmp;
    __syncthreads();   // every reader of z and of the old active list is done
  }
  if (t == 0) {
    stat[0] = pool;
    stat[1] = overflow;
  }
}

// _get_box_bounds (box_decomposition.py:96-109) of the final pass-2 bounds sel[0, L) of the pool, negated and swapped
// as _get_non_dominated_box_bounds returns them: lo[r] = -upper, hi[r] = -lower, where lower_0 = z^0_0, upper_0 =
// +inf, lower_c = max_{k < c} z^k_c (np.maximum.accumulate, in order), upper_c = u_c; keep[r] = no upper_c <= lower_c.
__global__ void k_bd_boxes(const double* __restrict__ ub, const double* __restrict__ dp, const int32_t* __restrict__ sel,
                           int L, int M, double* __restrict__ lo, double* __restrict__ hi, uint8_t* __restrict__ keep) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= L) return;
  const size_t a = (size_t)sel[r];
  const double* u = ub + a * M;
  const double* d = dp + a * M * M;
  bool empty = false;
  const double l0 = d[0];
  empty = INFINITY <= l0;
  lo[(size_t)r * M] = -INFINITY;
  hi[(size_t)r * M] = -l0;
  for (int c = 1; c < M; ++c) {
    double acc = d[c];
    for (int k = 1; k < c; ++k) {
      const double x = d[k * M + c];
      acc = acc >= x ? acc : x;   // numpy's maximum: the first operand unless the second is larger
    }
    empty = empty || u[c] <= acc;
    lo[(size_t)r * M + c] = -u[c];
    hi[(size_t)r * M + c] = -acc;
  }
  keep[r] = empty ? 0 : 1;
}

}  // namespace boxdec
}  // namespace tpe
