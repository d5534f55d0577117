// MOTPE kernels: non-domination ranks, greedy hypervolume subset selection, hypervolume weights.
//   k_mo_peel / k_mo_commit      optuna/study/_multi_objective.py:187-219 (_calculate_nondomination_rank)
//   k_mo_refpoint                optuna/samplers/_tpe/sampler.py:679-683 (_get_reference_point)
//   k_mo_lexrank / k_hssp_*      optuna/_hypervolume/hssp.py:10-176 (_solve_hssp)
//   k_mo_weights                 optuna/samplers/_tpe/sampler.py:824-863
// vals: [N, M] sign-normalised objective values of the whole history; lists index into it.
#pragma once
#include "tpe_common.cuh"
#include "tpe_motpe.cuh"

namespace tpe {

constexpr int kMoMaxM = 16;      // objectives (shared-memory staging of the small-set kernels; exact WFG beyond ~8 is slow anyway)
constexpr int kMoMaxSet = 64;    // "small set": points staged in shared memory by the one-CTA kernels; larger sets take
                                 // the global-memory kernels at the end of this file (no limit but memory)

struct MoCounters {
  int covered_unique, covered_all, n_unique, pad;
};

// does a dominate b (a <= b everywhere, a != b)?
__device__ __forceinline__ bool dominates(const double* a, const double* b, int M) {
  bool le = true, lt = false;
  for (int j = 0; j < M; ++j) {
    le = le && (a[j] <= b[j]);
    lt = lt || (a[j] < b[j]);
  }
  return le && lt;
}

// ---- duplicates (np.unique semantics: identical vectors share a rank and count once) ---------------
// is_first[i] = no earlier trial has the identical objective vector.  Open-addressing table of trial
// positions keyed by a hash of the vector (-0.0 folded onto +0.0 like ==); a slot keeps the smallest
// position among the identical vectors that landed in it.
constexpr int kMoEmpty = 0x7f7f7f7f;  // cudaMemset(0x7f)
__device__ __forceinline__ uint64_t mo_hash(const double* v, int M) {
  uint64_t h = 0x9e3779b97f4a7c15ull;
  for (int j = 0; j < M; ++j) {
    double x = v[j];
    if (x == 0.0) x = 0.0;
    uint64_t z = static_cast<uint64_t>(__double_as_longlong(x)) + h;
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    h = z ^ (z >> 31);
  }
  return h;
}
__device__ __forceinline__ bool mo_same(const double* a, const double* b, int M) {
  bool eq = true;
  for (int j = 0; j < M; ++j) eq = eq && (a[j] == b[j]);
  return eq;
}
__global__ void k_mo_first_insert(const double* __restrict__ vals, int M, const int64_t* __restrict__ list, int nc,
                                  int* __restrict__ table, uint32_t mask) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nc) return;
  const double* me = vals + list[i] * M;
  uint32_t slot = (uint32_t)mo_hash(me, M) & mask;
  for (;;) {
    int cur = *reinterpret_cast<volatile int*>(table + slot);
    if (cur == kMoEmpty) {
      const int old = atomicCAS(table + slot, kMoEmpty, i);
      if (old == kMoEmpty) return;
      cur = old;
    }
    if (mo_same(vals + list[cur] * M, me, M)) {
      atomicMin(table + slot, i);
      return;
    }
    slot = (slot + 1) & mask;
  }
}
__global__ void k_mo_first_lookup(const double* __restrict__ vals, int M, const int64_t* __restrict__ list, int nc,
                                  const int* __restrict__ table, uint32_t mask, uint8_t* __restrict__ is_first,
                                  MoCounters* __restrict__ ctr) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  bool first = false;
  if (i < nc) {
    const double* me = vals + list[i] * M;
    uint32_t slot = (uint32_t)mo_hash(me, M) & mask;
    for (;;) {
      const int cur = table[slot];
      if (cur == i || cur == kMoEmpty) {  // own entry (also the only match of a vector holding a NaN) / not found
        first = true;
        break;
      }
      if (mo_same(vals + list[cur] * M, me, M)) {
        first = false;  // an identical vector with a smaller position owns the slot
        break;
      }
      slot = (slot + 1) & mask;
    }
    is_first[i] = first ? 1 : 0;
  }
  const unsigned b = __ballot_sync(0xffffffffu, first);
  if ((threadIdx.x & 31) == 0 && b) atomicAdd(&ctr->n_unique, __popc(b));
}

// ---- one peel of the non-domination ranking ---------------------------------------------------------
// dominated[i] = some alive j dominates i.  All-pairs is O(n^2); instead every alive point is first
// tested against a sample of <= 256 alive points (a point dominated by the sample is dominated,
// whoever does it), and only the survivors -- a few per cent for 2-4 objectives -- are tested
// against every alive point.
__global__ void __launch_bounds__(1024, 1)
k_mo_sample(int nc, const uint8_t* __restrict__ alive, int32_t* __restrict__ sample, int* __restrict__ n_sample,
            int* __restrict__ n_surv) {
  __shared__ int s_warp[32];
  int base = 0;
  for (int t0 = 0; t0 < nc && base < 256; t0 += 1024) {
    const int i = t0 + threadIdx.x;
    const bool f = i < nc && alive[i];
    const int2 rk = block_rank_1024(f, s_warp);
    if (f && base + rk.x < 256) sample[base + rk.x] = i;
    base += rk.y;
  }
  if (threadIdx.x == 0) {
    *n_sample = base < 256 ? base : 256;
    *n_surv = 0;
  }
}
__global__ void k_mo_peel_a(const double* __restrict__ vals, int M, const int64_t* __restrict__ list, int nc,
                            const uint8_t* __restrict__ alive, const int32_t* __restrict__ sample,
                            const int* __restrict__ n_sample, uint8_t* __restrict__ dominated,
                            int32_t* __restrict__ surv, int* __restrict__ n_surv) {
  extern __shared__ double s_tile[];  // 256 * M
  const int ns = *n_sample;
  if (threadIdx.x < ns)
    for (int j = 0; j < M; ++j) s_tile[threadIdx.x * M + j] = vals[list[sample[threadIdx.x]] * M + j];
  __syncthreads();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nc) return;
  bool dom = false;
  if (alive[i]) {
    double me[kMoMaxM];
    for (int j = 0; j < M; ++j) me[j] = vals[list[i] * M + j];
    for (int r = 0; r < ns && !dom; ++r) dom = dominates(s_tile + r * M, me, M);
    if (!dom) surv[atomicAdd(n_surv, 1)] = i;
  }
  dominated[i] = dom ? 1 : 0;
}
__global__ void __launch_bounds__(256)
k_mo_peel_b(const double* __restrict__ vals, int M, const int64_t* __restrict__ list, int nc,
            const uint8_t* __restrict__ alive, const int32_t* __restrict__ surv, const int* __restrict__ n_surv,
            uint8_t* __restrict__ dominated) {
  const int ns = *n_surv;
  for (int s = blockIdx.x; s < ns; s += gridDim.x) {
    const int i = surv[s];
    double me[kMoMaxM];
    for (int j = 0; j < M; ++j) me[j] = vals[list[i] * M + j];
    bool dom = false;
    for (int q = threadIdx.x; q < nc && !dom; q += 256)
      if (alive[q]) dom = dominates(vals + list[q] * M, me, M);
    if (__syncthreads_or(dom) && threadIdx.x == 0) dominated[i] = 1;
  }
}
// front = alive & !dominated gets rank r
__global__ void k_mo_commit(int nc, uint8_t* __restrict__ alive, const uint8_t* __restrict__ dominated,
                            const uint8_t* __restrict__ is_first, int32_t* __restrict__ rank, int r,
                            MoCounters* __restrict__ ctr) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nc || !alive[i] || dominated[i]) return;
  rank[i] = r;
  alive[i] = 0;
  atomicAdd(&ctr->covered_all, 1);
  if (is_first[i]) atomicAdd(&ctr->covered_unique, 1);
}
__global__ void k_mo_fill_rank(int nc, const uint8_t* __restrict__ alive, int32_t* __restrict__ rank, int r) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < nc && alive[i]) rank[i] = r;
}

// Ordered list of the positions with rank == r (single CTA of 1024 threads) and the membership
// flags of ranks <= last.
__global__ void __launch_bounds__(1024, 1)
k_mo_gather_rank(int nc, const int32_t* __restrict__ rank, int last, const int64_t* __restrict__ list,
                 uint8_t* __restrict__ member /*[N] by history row*/, int32_t* __restrict__ tie_pos, int* n_tie) {
  __shared__ int s_warp[32];
  int cnt = 0;
  for (int base = 0; base < nc; base += 1024) {
    const int i = base + threadIdx.x;
    const bool v = i < nc;
    if (v && rank[i] <= last) member[list[i]] = 1;
    const bool f = v && rank[i] == last + 1;
    const int2 rr = block_rank_1024(f, s_warp);
    if (f) tie_pos[cnt + rr.x] = i;
    cnt += rr.y;
  }
  if (threadIdx.x == 0) *n_tie = cnt;
}

// reference point of a point list: max(1.1 w, 0.9 w), 0 -> EPS
__global__ void __launch_bounds__(256)
k_mo_refpoint(const double* __restrict__ vals, int M, const int64_t* __restrict__ list, const int32_t* __restrict__ sub,
              int n, double* __restrict__ ref) {
  __shared__ double s_red[256];
  for (int j = 0; j < M; ++j) {
    double w = -INFINITY;
    for (int i = threadIdx.x; i < n; i += 256) {
      const double v = vals[list[sub ? sub[i] : i] * M + j];
      w = (v > w || v != v) ? v : w;
    }
    s_red[threadIdx.x] = w;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
      if (threadIdx.x < o) {
        const double a = s_red[threadIdx.x], b = s_red[threadIdx.x + o];
        s_red[threadIdx.x] = (b > a || b != b) ? b : a;
      }
      __syncthreads();
    }
    if (threadIdx.x == 0) {
      const double worst = s_red[0];
      double r = fmax(TPE_MUL(1.1, worst), TPE_MUL(0.9, worst));
      if (r == 0.0) r = 1e-12;
      ref[j] = r;
    }
    __syncthreads();
  }
}

// Lexicographic position of every tie point among the tie points (duplicates ordered by original
// position) + duplicate flag (an identical vector occurs earlier).  O(n^2), n = |tie rank|.
__global__ void k_mo_lexrank(const double* __restrict__ vals, int M, const int64_t* __restrict__ list,
                             const int32_t* __restrict__ tie_pos, int n, int32_t* __restrict__ lexpos,
                             uint8_t* __restrict__ is_dup) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double me[kMoMaxM];
  for (int j = 0; j < M; ++j) me[j] = vals[list[tie_pos[i]] * M + j];
  int before = 0;
  bool dup = false;
  for (int q = 0; q < n; ++q) {
    const double* o = vals + list[tie_pos[q]] * M;
    const int c = lex_cmp(o, me, M);
    if (c < 0 || (c == 0 && q < i)) ++before;
    if (c == 0 && q < i) dup = true;
  }
  lexpos[i] = before;
  is_dup[i] = dup ? 1 : 0;
}
// sorted[lexpos[i]] = i ; then the unique list in lexicographic order (single CTA)
__global__ void __launch_bounds__(1024, 1)
k_mo_unique(int n, const int32_t* __restrict__ lexpos, const uint8_t* __restrict__ is_dup,
            int32_t* __restrict__ sorted, int32_t* __restrict__ uniq /*tie-local index of first occurrences*/,
            int* n_unique) {
  __shared__ int s_warp[32];
  for (int i = threadIdx.x; i < n; i += 1024) sorted[lexpos[i]] = i;
  __syncthreads();
  int cnt = 0;
  for (int base = 0; base < n; base += 1024) {
    const int p = base + threadIdx.x;
    const bool f = p < n && !is_dup[sorted[p]];
    const int2 rr = block_rank_1024(f, s_warp);
    if (f) uniq[cnt + rr.x] = sorted[p];
    cnt += rr.y;
  }
  if (threadIdx.x == 0) *n_unique = cnt;
}

// Greedy-selection state in global memory: header, then sel[cap * M] (selected vectors, pick order), then
// pick[cap] (tie-local index of the picks).  cap = subset size of this call.
struct HsspState {
  double hv;            // hypervolume of the selected set (running sum of picked contributions)
  int n_sel;
  int cap;
};
__host__ __device__ inline double* hssp_sel(HsspState* s) { return reinterpret_cast<double*>(s + 1); }
__host__ __device__ inline const double* hssp_sel(const HsspState* s) { return reinterpret_cast<const double*>(s + 1); }
__host__ __device__ inline int32_t* hssp_pick(HsspState* s, int M) {
  return reinterpret_cast<int32_t*>(hssp_sel(s) + (size_t)s->cap * M);
}
__host__ __device__ inline size_t hssp_bytes(int cap, int M) {
  return sizeof(HsspState) + (size_t)cap * M * 8 + (size_t)cap * 4 + 8;
}

// The reference's lazily updated upper bound of a candidate's contribution (hssp.py:68-77), one per unique
// candidate, kept across rounds: the first round's bound is the candidate's own box incl; later rounds cap the
// previous value (what the last scan left: exact, bound or inf) by the contribution to the newest pick alone,
// incl - |box(max(me, last pick))|; every bound is inf once the selected hypervolume is (hssp.py:68-70).
// np.minimum propagates NaN (inf - inf when both boxes are infinite).
__device__ __forceinline__ double hssp_bound(const double* me, int M, const double* ref, const HsspState* st,
                                             double incl, double prev) {
  const int t = st->n_sel;
  if (t == 0) return incl;
  if (isinf(st->hv)) return INFINITY;
  const double* last = hssp_sel(st) + (size_t)(t - 1) * M;
  double cap = 1.0;
  for (int j = 0; j < M; ++j) cap = TPE_MUL(cap, TPE_SUB(ref[j], me[j] > last[j] ? me[j] : last[j]));
  const double b = TPE_SUB(incl, cap);
  return (prev != prev || b != b) ? NAN : (b < prev ? b : prev);
}

// Warp-cooperative exact 3-D hypervolume of n <= kMoMaxSet + 1 mutually non-dominated points
// (the assume_pareto branch of hypervolume()), bit-identical to it: the two stable insertion sorts
// become ranks by counting, every row's inner sum is evaluated by one lane exactly as hv_3d does,
// and the row terms are added in row order by lane 0.
//   pts [n,3]; scratch: s [n,3] (rows sorted by x), term [n], ord [n]
__device__ double hv3_warp(const double* pts, int n, const double* ref, double* s, double* term, int* ord) {
  const int lane = threadIdx.x & 31;
  if (!isfinite(ref[0]) || !isfinite(ref[1]) || !isfinite(ref[2])) return INFINITY;
  if (n == 0) return 0.0;
  for (int i = lane; i < n; i += 32) {
    const double x = pts[i * 3];
    int r = 0;
    for (int j = 0; j < n; ++j) {
      const double xj = pts[j * 3];
      r += (xj < x || (xj == x && j < i)) ? 1 : 0;
    }
    s[r * 3] = x;
    s[r * 3 + 1] = pts[i * 3 + 1];
    s[r * 3 + 2] = pts[i * 3 + 2];
  }
  __syncwarp();
  for (int i = lane; i < n; i += 32) {
    const double y = s[i * 3 + 1];
    int r = 0;
    for (int j = 0; j < n; ++j) {
      const double yj = s[j * 3 + 1];
      r += (yj < y || (yj == y && j < i)) ? 1 : 0;
    }
    ord[r] = i;
  }
  __syncwarp();
  for (int i = lane; i < n; i += 32) {
    const double dx = TPE_SUB(i + 1 < n ? s[(i + 1) * 3] : ref[0], s[i * 3]);
    double run = 0.0, inner = 0.0;
    for (int j = 0; j < n; ++j) {
      const int o = ord[j];
      if (o <= i) {
        const double z = TPE_SUB(ref[2], s[o * 3 + 2]);
        run = z > run ? z : run;
      }
      const double dy = TPE_SUB(j + 1 < n ? s[ord[j + 1] * 3 + 1] : ref[1], s[o * 3 + 1]);
      inner = TPE_ADD(inner, TPE_MUL(run, dy));
    }
    term[i] = TPE_MUL(inner, dx);
  }
  __syncwarp();
  double total = 0.0;
  if (lane == 0)
    for (int i = 0; i < n; ++i) total = TPE_ADD(total, term[i]);
  total = __shfl_sync(0xffffffffu, total, 0);
  __syncwarp();
  return isfinite(total) ? total : INFINITY;
}
constexpr int kHv3Scratch = (kMoMaxSet + 1) * 8;  // doubles per warp: pts 3n + s 3n + term n + ord n/2 (+ slack)

// k_hssp_contrib for three objectives: one warp per remaining candidate.
__global__ void __launch_bounds__(128)
k_hssp_contrib3(const double* __restrict__ vals, const int64_t* __restrict__ list,
                const int32_t* __restrict__ tie_pos, const int32_t* __restrict__ uniq, int nu,
                const uint8_t* __restrict__ removed, const double* __restrict__ ref,
                const HsspState* __restrict__ st, double* __restrict__ contrib, double* __restrict__ bound,
                double* __restrict__ arena, size_t arena_stride) {
  __shared__ double s_scr[4][kHv3Scratch];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int u = blockIdx.x * 4 + w;
  if (u >= nu) return;
  if (removed[u]) {
    if (lane == 0) contrib[u] = -INFINITY;
    return;
  }
  const double* me = vals + list[tie_pos[uniq[u]]] * 3;
  double incl = 1.0;
  for (int j = 0; j < 3; ++j) incl = TPE_MUL(incl, TPE_SUB(ref[j], me[j]));
  if (lane == 0) { bound[u] = hssp_bound(me, 3, ref, st, incl, bound[u]); bound[nu + u] = incl; }
  const int t = st->n_sel;
  if (t == 0 || isinf(incl)) {
    if (lane == 0) contrib[u] = incl;
    return;
  }
  if (isinf(st->hv)) {
    if (lane == 0) contrib[u] = INFINITY;
    return;
  }
  double* pts = (t + 1 <= kMoMaxSet + 1) ? s_scr[w] : arena + (size_t)u * arena_stride;
  double* srt = pts + (t + 1) * 3;
  double* term = srt + (t + 1) * 3;
  int* ord = reinterpret_cast<int*>(term + (t + 1));
  for (int q = lane; q < t * 3; q += 32) pts[q] = hssp_sel(st)[q];
  if (lane < 3) pts[t * 3 + lane] = me[lane];
  __syncwarp();
  const double hv = hv3_warp(pts, t + 1, ref, srt, term, ord);
  if (lane == 0) contrib[u] = TPE_SUB(hv, st->hv);
}

// Warp-cooperative exact N-D (M > 3) hypervolume of n <= kMoMaxSet + 1 points, bit-identical to
// hypervolume(): the lexicographic insertion sort + duplicate removal become ranks by counting, the
// sequential front sweep becomes "no earlier point is <= in coordinates 1..M-1" (equivalent by
// transitivity), and the top level of the WFG recursion
//     HV(S) = incl(last) + sum_i [ incl(i) - HV(front(limit(S_{>i}, i))) ]
// gives every lane one i: its exclusive part is evaluated by the sequential hv_nd() in a private
// arena, and lane 0 adds the terms in index order, as the frame loop of hv_nd() does.
//   pts [n, M] input (not modified); ws: warp scratch, >= 2 n M + 2 n doubles;
//   lane_arena: private arena of this lane, >= hv_lane_doubles(n, M)
__host__ __device__ inline size_t hv_lane_doubles(int n, int M) { return hv_arena_doubles(n, M) + (size_t)n * M + 32; }
__device__ double hv_nd_warp(const double* pts, int n, int M, const double* ref, bool assume_pareto, double* ws,
                             double* lane_arena) {
  const int lane = threadIdx.x & 31;
  for (int j = 0; j < M; ++j)
    if (!isfinite(ref[j])) return INFINITY;
  if (n == 0) return 0.0;
  double* srt = ws;                       // n * M, sorted rows
  double* s = ws + (size_t)n * M;         // n * M, compacted rows
  int* flag = reinterpret_cast<int*>(s + (size_t)n * M);   // n ints
  int* cntp = flag + n;                   // 1 int
  // stable sort: by all coordinates (+ duplicates flagged) or by coordinate 0 only (assume_pareto)
  for (int i = lane; i < n; i += 32) {
    const double* me = pts + (size_t)i * M;
    int r = 0;
    bool dup = false;
    for (int q = 0; q < n; ++q) {
      const double* o = pts + (size_t)q * M;
      int c;
      if (assume_pareto) c = (o[0] < me[0]) ? -1 : ((o[0] > me[0]) ? 1 : 0);
      else c = lex_cmp(o, me, M);
      r += (c < 0 || (c == 0 && q < i)) ? 1 : 0;
      dup = dup || (!assume_pareto && c == 0 && q < i);
    }
    for (int j = 0; j < M; ++j) srt[(size_t)r * M + j] = me[j];
    flag[r] = dup ? 0 : 1;   // keep flag
  }
  __syncwarp();
  int m;
  if (!assume_pareto) {
    // front filter on the unique rows: row i survives unless an earlier kept row is <= in coords 1..M-1
    for (int i = lane; i < n; i += 32) {
      if (!flag[i]) continue;
      const double* me = srt + (size_t)i * M;
      bool killed = false;
      for (int h = 0; h < i && !killed; ++h) {
        if (!flag[h]) continue;   // duplicates of an earlier row: the earlier row decides
        const double* o = srt + (size_t)h * M;
        bool better = false;
        for (int j = 1; j < M; ++j) better = better || (me[j] < o[j]);
        killed = !better;
      }
      if (killed) flag[i] = 2;   // dominated (2 keeps the duplicate test of later rows intact)
    }
    __syncwarp();
    if (lane == 0) {
      int w = 0;
      for (int i = 0; i < n; ++i) {
        if (flag[i] != 1) continue;
        for (int j = 0; j < M; ++j) s[(size_t)w * M + j] = srt[(size_t)i * M + j];
        ++w;
      }
      *cntp = w;
    }
    __syncwarp();
    m = *cntp;
  } else {
    for (int q = lane; q < n * M; q += 32) s[q] = srt[q];
    __syncwarp();
    m = n;
  }
  double total;
  if (m <= 2) {
    total = 0.0;
    if (lane == 0) total = hv_nd(s, m, M, ref, lane_arena);
    total = __shfl_sync(0xffffffffu, total, 0);
  } else {
    double* term = srt;   // reuse: m doubles
    for (int i = lane; i < m - 1; i += 32) {
      double incl = 1.0;
      for (int j = 0; j < M; ++j) incl = TPE_MUL(incl, TPE_SUB(ref[j], s[(size_t)i * M + j]));
      double* lim = lane_arena;
      int cnt = m - 1 - i;
      for (int r = 0; r < cnt; ++r)
        for (int j = 0; j < M; ++j) {
          const double a = s[(size_t)i * M + j], b = s[(size_t)(i + 1 + r) * M + j];
          lim[r * M + j] = a > b ? a : b;
        }
      uint8_t* fl = reinterpret_cast<uint8_t*>(lim + (size_t)(m - 1) * M);
      if (cnt > 3) {
        uint8_t* mask = fl;
        uint8_t* alive = fl + m;
        front_sorted(lim, cnt, M, mask, alive);
        int w = 0;
        for (int r = 0; r < cnt; ++r) {
          if (!mask[r]) continue;
          if (w != r)
            for (int j = 0; j < M; ++j) lim[w * M + j] = lim[r * M + j];
          ++w;
        }
        cnt = w;
      }
      double* sub = lim + (size_t)(m - 1) * M + (2 * m + 7) / 8 + 1;
      const double child = hv_nd(lim, cnt, M, ref, sub);
      term[i] = TPE_SUB(incl, child);
    }
    __syncwarp();
    total = 0.0;
    if (lane == 0) {
      double sum = 0.0;
      for (int i = 0; i < m - 1; ++i) sum = TPE_ADD(sum, term[i]);
      double last = 1.0;
      for (int j = 0; j < M; ++j) last = TPE_MUL(last, TPE_SUB(ref[j], s[(size_t)(m - 1) * M + j]));
      total = TPE_ADD(last, sum);
    }
    total = __shfl_sync(0xffffffffu, total, 0);
  }
  __syncwarp();
  return isfinite(total) ? total : INFINITY;
}
// scratch doubles per warp for hv_nd_warp incl. the caller's point list
__host__ __device__ inline size_t hv_warp_scratch_doubles(int n, int M) { return (size_t)3 * n * M + 2 * n + 16; }

// k_hssp_contrib for more than three objectives: one warp per remaining candidate
// (H({i}) - H(S limited by i), hssp.py:45-97).
__global__ void __launch_bounds__(128)
k_hssp_contrib_nd(const double* __restrict__ vals, int M, const int64_t* __restrict__ list,
                  const int32_t* __restrict__ tie_pos, const int32_t* __restrict__ uniq, int nu,
                  const uint8_t* __restrict__ removed, const double* __restrict__ ref,
                  const HsspState* __restrict__ st, double* __restrict__ contrib, double* __restrict__ bound,
                  double* __restrict__ arena, size_t warp_stride, size_t lane_stride) {
  const int lane = threadIdx.x & 31;
  const int u = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (u >= nu) return;
  if (removed[u]) {
    if (lane == 0) contrib[u] = -INFINITY;
    return;
  }
  const double* me = vals + list[tie_pos[uniq[u]]] * M;
  double incl = 1.0;
  for (int j = 0; j < M; ++j) incl = TPE_MUL(incl, TPE_SUB(ref[j], me[j]));
  if (lane == 0) { bound[u] = hssp_bound(me, M, ref, st, incl, bound[u]); bound[nu + u] = incl; }
  const int t = st->n_sel;
  if (t == 0 || isinf(incl)) {
    if (lane == 0) contrib[u] = incl;
    return;
  }
  if (isinf(st->hv)) {
    if (lane == 0) contrib[u] = INFINITY;
    return;
  }
  double* wsb = arena + (size_t)u * warp_stride;
  double* pts = wsb;                         // t * M
  double* ws = wsb + (size_t)t * M;
  double* lanes = wsb + hv_warp_scratch_doubles(t, M);
  for (int q = lane; q < t * M; q += 32) {
    const int j = q % M;
    const double b = hssp_sel(st)[q];
    pts[q] = me[j] > b ? me[j] : b;
  }
  __syncwarp();
  const double hv = hv_nd_warp(pts, t, M, ref, false, ws, lanes + (size_t)lane * lane_stride);
  if (lane == 0) contrib[u] = TPE_SUB(incl, hv);
}

// Exact contribution of every remaining unique candidate given the selected set (hssp.py:87-95) and its lazy
// bound (hssp_bound), and its own box incl in bound[nu + u]; k_hssp_pick decides which the reference's scan keeps.
__global__ void k_hssp_contrib(const double* __restrict__ vals, int M, const int64_t* __restrict__ list,
                               const int32_t* __restrict__ tie_pos, const int32_t* __restrict__ uniq, int nu,
                               const uint8_t* __restrict__ removed, const double* __restrict__ ref,
                               const HsspState* __restrict__ st, double* __restrict__ contrib, double* __restrict__ bound,
                               double* __restrict__ arena, size_t arena_stride, int smem_stride) {
  // smem_stride != 0 (M <= 3, where the scratch is a few hundred doubles per thread): the scratch
  // lives in shared memory instead of the global arena
  extern __shared__ double s_arena[];
  const int u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= nu) return;
  if (removed[u]) {
    contrib[u] = -INFINITY;
    return;
  }
  const double* me = vals + list[tie_pos[uniq[u]]] * M;
  double incl = 1.0;
  for (int j = 0; j < M; ++j) incl = TPE_MUL(incl, TPE_SUB(ref[j], me[j]));
  bound[u] = hssp_bound(me, M, ref, st, incl, bound[u]);
  bound[nu + u] = incl;
  const int t = st->n_sel;
  if (t == 0 || isinf(incl)) {
    contrib[u] = incl;
    return;
  }
  if (isinf(st->hv)) {
    contrib[u] = INFINITY;
    return;
  }
  double* a = smem_stride ? s_arena + (size_t)threadIdx.x * smem_stride : arena + (size_t)u * arena_stride;
  double* pts = a;  // (t + 1) * M
  double* rest = a + (size_t)(t + 1) * M;
  if (M <= 3) {
    // H(S + {i}) - H(S), assume_pareto (points of one non-domination rank are mutually non-dominated)
    for (int s = 0; s < t; ++s)
      for (int j = 0; j < M; ++j) pts[s * M + j] = hssp_sel(st)[s * M + j];
    for (int j = 0; j < M; ++j) pts[t * M + j] = me[j];
    contrib[u] = TPE_SUB(hypervolume(pts, t + 1, M, ref, true, rest), st->hv);
  } else {
    // H({i}) - H(S limited by i)
    for (int s = 0; s < t; ++s)
      for (int j = 0; j < M; ++j) {
        const double b = hssp_sel(st)[s * M + j];
        pts[s * M + j] = me[j] > b ? me[j] : b;
      }
    contrib[u] = TPE_SUB(incl, hypervolume(pts, t, M, ref, false, rest));
  }
}
// First argmax over a 256-thread block of one (value, index) candidate per thread (index < 0: none): np.argmax
// semantics, the first NaN wins, ties go to the smaller index.  Result in s_val[0] / s_idx[0].
__device__ void block_first_argmax256(double best, int bi, double* s_val, int* s_idx) {
  s_val[threadIdx.x] = best;
  s_idx[threadIdx.x] = bi;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      const double a = s_val[threadIdx.x], b = s_val[threadIdx.x + o];
      const int ia = s_idx[threadIdx.x], ib = s_idx[threadIdx.x + o];
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
      if (take_b) { s_val[threadIdx.x] = b; s_idx[threadIdx.x] = ib; }
    }
    __syncthreads();
  }
}
__device__ __forceinline__ void argmax_step(double c, int u, double& best, int& bi, bool& bnan) {
  const bool cn = c != c;
  if (bi < 0 || (!bnan && (cn || c > best))) { best = c; bi = u; bnan = cn; }
}

constexpr int kPickStage = 1024;   // candidates whose bounds and exact values k_hssp_pick stages in shared memory

// The value the reference's scan leaves for remaining candidate u (see k_hssp_pick): inf for an infinite own box;
// its bound b when b < 0 or a candidate visited earlier (larger bound, or equal bound and smaller index) has an
// exact value above b; else its exact value.  A removed candidate has exact value -inf and never decides.
// js >= 0: a candidate with the largest exact value ejs and bound bjs, tried first.
__device__ __forceinline__ double hssp_scan_value(int u, int nu, double incl, const double* B, const double* E, int js,
                                                  double ejs, double bjs) {
  if (isinf(incl)) return INFINITY;
  const double b = B[u];
  bool keep = !(b >= 0.0);
  if (!keep && js >= 0 && js != u && (bjs > b || (bjs == b && js < u)) && ejs > b) keep = true;
  for (int q = 0; q < nu && !keep; ++q) {
    const double bq = B[q];
    keep = q != u && (bq > b || (bq == b && q < u)) && E[q] > b;
  }
  return keep ? b : E[u];
}

// One round of the reference's greedy pick (hssp.py:78-97, then :123): the lazy scan over the remaining unique
// candidates, then the first argmax of what it leaves, appended to the selected set.
// The scan visits candidates in descending bound order, ties by ascending index (a stable argsort; numpy's is not
// stable, so where bounds tie the reference's own visiting order is unspecified).  A candidate whose own box is
// infinite becomes inf; one whose bound is below the best exact value seen so far keeps its bound; any other takes
// its exact value.  As bounds only fall along the visiting order and the best only rises, a candidate keeps its bound
// exactly when its bound is < 0 or a candidate visited before it has an exact value above that bound, which every
// thread decides for its own candidates without a sequential pass.
//   contrib: exact contributions (k_hssp_contrib*; -inf for removed candidates);
//   bound: [0, nu) lazy bounds in, the scan's values out; [nu, 2 nu) each candidate's incl in, scratch
__global__ void __launch_bounds__(256)
k_hssp_pick(const double* __restrict__ vals, int M, const int64_t* __restrict__ list,
            const int32_t* __restrict__ tie_pos, const int32_t* __restrict__ uniq, int nu,
            uint8_t* __restrict__ removed, const double* __restrict__ contrib, double* __restrict__ bound,
            HsspState* __restrict__ st) {
  __shared__ double s_val[256];
  __shared__ int s_idx[256];
  __shared__ double s_b[kPickStage], s_e[kPickStage];
  double* scan = bound + nu;
  const int t = st->n_sel;
  double best = -INFINITY;
  int bi = -1;
  bool bnan = false;
  if (t == 0 || isinf(st->hv)) {   // first round: bound = exact = incl; inf hypervolume: every value is inf
    for (int u = threadIdx.x; u < nu; u += 256)
      if (!removed[u]) argmax_step(bound[u], u, best, bi, bnan);
  } else if (nu <= kPickStage) {
    // every thread keeps the values of its (at most four) candidates in registers
    double mine[kPickStage / 256], incl[kPickStage / 256];
#pragma unroll
    for (int k = 0; k < kPickStage / 256; ++k) {
      const int u = threadIdx.x + k * 256;
      if (u < nu) { s_b[u] = bound[u]; s_e[u] = contrib[u]; incl[k] = scan[u]; }
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kPickStage / 256; ++k) {
      const int u = threadIdx.x + k * 256;
      if (u < nu) mine[k] = hssp_scan_value(u, nu, incl[k], s_b, s_e, -1, 0.0, 0.0);
    }
#pragma unroll
    for (int k = 0; k < kPickStage / 256; ++k) {
      const int u = threadIdx.x + k * 256;
      if (u < nu && !removed[u]) {
        bound[u] = mine[k];
        argmax_step(mine[k], u, best, bi, bnan);
      }
    }
  } else {
    // the best exact value: usually visited early, it decides most candidates at once
    for (int u = threadIdx.x; u < nu; u += 256)
      if (!removed[u]) argmax_step(contrib[u], u, best, bi, bnan);
    block_first_argmax256(best, bi, s_val, s_idx);
    const int js = s_idx[0];
    const double ejs = s_val[0], bjs = bound[js];
    for (int u = threadIdx.x; u < nu; u += 256)
      if (!removed[u]) scan[u] = hssp_scan_value(u, nu, scan[u], bound, contrib, js, ejs, bjs);
    __syncthreads();
    best = -INFINITY;
    bi = -1;
    bnan = false;
    for (int u = threadIdx.x; u < nu; u += 256)
      if (!removed[u]) {
        bound[u] = scan[u];
        argmax_step(scan[u], u, best, bi, bnan);
      }
  }
  block_first_argmax256(best, bi, s_val, s_idx);
  if (threadIdx.x == 0) {
    const int u = s_idx[0];
    st->hv = TPE_ADD(st->hv, s_val[0]);
    hssp_pick(st, M)[t] = uniq[u];
    const double* me = vals + list[tie_pos[uniq[u]]] * M;
    for (int j = 0; j < M; ++j) hssp_sel(st)[t * M + j] = me[j];
    st->n_sel = t + 1;
    removed[u] = 1;
  }
}
// 2-objective greedy (_solve_hssp_2d, hssp.py:10-42): one CTA, the unique list is lexsorted.
__global__ void __launch_bounds__(256)
k_hssp_2d(const double* __restrict__ vals, const int64_t* __restrict__ list, const int32_t* __restrict__ tie_pos,
          const int32_t* __restrict__ uniq, int nu, int k, const double* __restrict__ ref,
          double* __restrict__ diag /*[nu, 2] scratch*/, uint8_t* __restrict__ removed, HsspState* __restrict__ st) {
  __shared__ double s_val[256];
  __shared__ int s_idx[256];
  for (int u = threadIdx.x; u < nu; u += 256) {
    diag[2 * u] = ref[0];
    diag[2 * u + 1] = ref[1];
    removed[u] = 0;
  }
  __syncthreads();
  for (int t = 0; t < k; ++t) {
    double best = -INFINITY;
    int bi = -1;
    bool bnan = false;
    for (int u = threadIdx.x; u < nu; u += 256) {
      if (removed[u]) continue;
      const double* p = vals + list[tie_pos[uniq[u]]] * 2;
      const double c = TPE_MUL(TPE_SUB(diag[2 * u], p[0]), TPE_SUB(diag[2 * u + 1], p[1]));
      const bool cn = c != c;
      if (bi < 0 || (!bnan && (cn || c > best))) { best = c; bi = u; bnan = cn; }
    }
    s_val[threadIdx.x] = best;
    s_idx[threadIdx.x] = bi;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
      if (threadIdx.x < o) {
        const double a = s_val[threadIdx.x], b = s_val[threadIdx.x + o];
        const int ia = s_idx[threadIdx.x], ib = s_idx[threadIdx.x + o];
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
        if (take_b) { s_val[threadIdx.x] = b; s_idx[threadIdx.x] = ib; }
      }
      __syncthreads();
    }
    const int j = s_idx[0];
    const double* pj = vals + list[tie_pos[uniq[j]]] * 2;
    const double px = pj[0], py = pj[1];
    __syncthreads();
    if (threadIdx.x == 0) {
      hssp_pick(st, 2)[t] = uniq[j];
      st->n_sel = t + 1;
      removed[j] = 1;
    }
    // rows before j (lexicographically): clip x; rows after: clip y
    for (int u = threadIdx.x; u < nu; u += 256) {
      if (u == j || removed[u]) continue;
      if (u < j) diag[2 * u] = fmin(px, diag[2 * u]);
      else diag[2 * u + 1] = fmin(py, diag[2 * u + 1]);
    }
    __syncthreads();
  }
}
// mark the selected tie points (and, when there are fewer unique vectors than slots, the first
// duplicates in trial order) in the membership array
__global__ void k_mo_mark(const int64_t* __restrict__ list, const int32_t* __restrict__ tie_pos,
                          const int32_t* __restrict__ chosen, int n, uint8_t* __restrict__ member) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) member[list[tie_pos[chosen[i]]]] = 1;
}
__global__ void __launch_bounds__(1024, 1)
k_mo_fill_dups(int n, const uint8_t* __restrict__ is_dup, int want, int32_t* __restrict__ chosen, int at) {
  __shared__ int s_warp[32];
  int cnt = 0;
  for (int base = 0; base < n; base += 1024) {
    const int i = base + threadIdx.x;
    const bool f = i < n && is_dup[i];
    const int2 rr = block_rank_1024(f, s_warp);
    if (f && cnt + rr.x < want) chosen[at + cnt + rr.x] = i;
    cnt += rr.y;
  }
}

// Hypervolume weights of the below set (sampler.py:824-863).  One CTA; thread p evaluates the
// leave-one-out term of below point p.  rows: history rows of the below trials (trial order),
// cat: category per history row (INFEASIBLE -> EPS weight).
__global__ void __launch_bounds__(kMoMaxSet)
k_mo_weights(const double* __restrict__ vals, int M, const int64_t* __restrict__ rows, int n,
             const int8_t* __restrict__ cat, double* __restrict__ w, double* __restrict__ arena, size_t arena_stride,
             int smem_stride) {
  extern __shared__ double s_arena[];           // per-thread scratch when smem_stride != 0 (M <= 3)
  __shared__ double s_v[kMoMaxSet * kMoMaxM];   // feasible points, trial order
  __shared__ double s_ps[kMoMaxSet * kMoMaxM];  // Pareto points, trial order
  __shared__ double s_ref[kMoMaxM];
  __shared__ double s_contrib[kMoMaxSet];
  __shared__ int s_map[kMoMaxSet];      // feasible index -> below index
  __shared__ int s_front[kMoMaxSet];    // front index -> feasible index
  __shared__ int s_nf, s_np;
  __shared__ double s_hv, s_max;
  const int tid = threadIdx.x;
  if (tid == 0) {
    int nf = 0;
    for (int i = 0; i < n; ++i) {
      const bool feas = cat[rows[i]] != 2;
      w[i] = feas ? 1.0 : 1e-12;
      if (feas) {
        for (int j = 0; j < M; ++j) s_v[nf * M + j] = vals[rows[i] * M + j];
        s_map[nf++] = i;
      }
    }
    s_nf = nf;
    if (nf > 1) {
      for (int j = 0; j < M; ++j) {
        double worst = s_v[j];
        for (int i = 1; i < nf; ++i) {
          const double v = s_v[i * M + j];
          worst = (v > worst || v != v) ? v : worst;
        }
        double r = fmax(TPE_MUL(1.1, worst), TPE_MUL(0.9, worst));
        if (r == 0.0) r = 1e-12;
        s_ref[j] = r;
      }
      int np = 0;
      for (int i = 0; i < nf; ++i) {
        bool dom = false;
        for (int q = 0; q < nf && !dom; ++q) dom = (q != i) && dominates(s_v + q * M, s_v + i * M, M);
        if (!dom) {
          for (int j = 0; j < M; ++j) s_ps[np * M + j] = s_v[i * M + j];
          s_front[np++] = i;
        }
      }
      s_np = np;
      s_hv = hypervolume(s_ps, np, M, s_ref, true, smem_stride ? s_arena : arena);
    }
  }
  __syncthreads();
  const int nf = s_nf;
  if (nf <= 1) return;
  const int np = s_np;
  const double hv = s_hv;
  if (isinf(hv)) return;
  if (tid < nf) s_contrib[tid] = 0.0;
  __syncthreads();
  if (tid < np) {
    double* a = smem_stride ? s_arena + (size_t)tid * smem_stride : arena + (size_t)tid * arena_stride;
    double* pts = a;
    double* rest = a + (size_t)np * M;
    int c = 0;
    double val;
    if (M <= 3) {
      for (int q = 0; q < np; ++q) {
        if (q == tid) continue;
        for (int j = 0; j < M; ++j) pts[c * M + j] = s_ps[q * M + j];
        ++c;
      }
      val = TPE_SUB(hv, hypervolume(pts, c, M, s_ref, true, rest));
    } else {
      double incl = 1.0;
      for (int j = 0; j < M; ++j) incl = TPE_MUL(incl, TPE_SUB(s_ref[j], s_ps[tid * M + j]));
      for (int q = 0; q < np; ++q) {
        if (q == tid) continue;
        for (int j = 0; j < M; ++j) {
          const double x = s_ps[q * M + j], y = s_ps[tid * M + j];
          pts[c * M + j] = x > y ? x : y;
        }
        ++c;
      }
      val = TPE_SUB(incl, hypervolume(pts, c, M, s_ref, false, rest));
    }
    s_contrib[s_front[tid]] = val;
  }
  __syncthreads();
  if (tid == 0) {
    double mx = s_contrib[0];
    for (int i = 1; i < nf; ++i) mx = (s_contrib[i] > mx || s_contrib[i] != s_contrib[i]) ? s_contrib[i] : mx;
    s_max = fmax(mx, 1e-12);
  }
  __syncthreads();
  if (tid < nf) w[s_map[tid]] = fmax(TPE_DIV(s_contrib[tid], s_max), 1e-12);
}

// k_mo_weights for three objectives: same result, the Pareto filter is evaluated by one thread per
// point and every hypervolume by one warp (32 warps: the front's, then the leave-one-out terms).
__global__ void __launch_bounds__(1024, 1)
k_mo_weights3(const double* __restrict__ vals, const int64_t* __restrict__ rows, int n,
              const int8_t* __restrict__ cat, double* __restrict__ w) {
  constexpr int M = 3;
  __shared__ double s_v[kMoMaxSet * M];   // feasible points, trial order
  __shared__ double s_ps[kMoMaxSet * M];  // Pareto points, trial order
  __shared__ double s_ref[M];
  __shared__ double s_contrib[kMoMaxSet];
  __shared__ int s_map[kMoMaxSet];        // feasible index -> below index
  __shared__ int s_front[kMoMaxSet];      // front index -> feasible index
  __shared__ uint8_t s_nd[kMoMaxSet];
  __shared__ int s_nf, s_np;
  __shared__ double s_hv, s_max;
  extern __shared__ double s_scr_dyn[];  // 32 warps x kHv3Scratch doubles
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0) {
    int nf = 0;
    for (int i = 0; i < n; ++i) {
      const bool feas = cat[rows[i]] != 2;
      w[i] = feas ? 1.0 : 1e-12;
      if (feas) {
        for (int j = 0; j < M; ++j) s_v[nf * M + j] = vals[rows[i] * M + j];
        s_map[nf++] = i;
      }
    }
    s_nf = nf;
    if (nf > 1) {
      for (int j = 0; j < M; ++j) {
        double worst = s_v[j];
        for (int i = 1; i < nf; ++i) {
          const double v = s_v[i * M + j];
          worst = (v > worst || v != v) ? v : worst;
        }
        double r = fmax(TPE_MUL(1.1, worst), TPE_MUL(0.9, worst));
        if (r == 0.0) r = 1e-12;
        s_ref[j] = r;
      }
    }
  }
  __syncthreads();
  const int nf = s_nf;
  if (nf <= 1) return;
  if (tid < nf) {
    bool dom = false;
    for (int q = 0; q < nf && !dom; ++q) dom = (q != tid) && dominates(s_v + q * M, s_v + tid * M, M);
    s_nd[tid] = dom ? 0 : 1;
  }
  __syncthreads();
  if (tid == 0) {
    int np = 0;
    for (int i = 0; i < nf; ++i)
      if (s_nd[i]) {
        for (int j = 0; j < M; ++j) s_ps[np * M + j] = s_v[i * M + j];
        s_front[np++] = i;
      }
    s_np = np;
  }
  if (tid < nf) s_contrib[tid] = 0.0;
  __syncthreads();
  const int np = s_np;
  {
    double* scr = s_scr_dyn + (size_t)wid * kHv3Scratch;
    if (wid == 0) {
      const double hv = hv3_warp(s_ps, np, s_ref, scr, scr + np * 3, reinterpret_cast<int*>(scr + np * 4));
      if (lane == 0) s_hv = hv;
    }
  }
  __syncthreads();
  const double hv = s_hv;
  if (isinf(hv)) return;
  for (int p = wid; p < np; p += 32) {
    double* pts = s_scr_dyn + (size_t)wid * kHv3Scratch;
    const int c = np - 1;
    for (int q = lane; q < np; q += 32) {
      if (q == p) continue;
      const int d = q < p ? q : q - 1;
      for (int j = 0; j < M; ++j) pts[d * M + j] = s_ps[q * M + j];
    }
    __syncwarp();
    double* srt = pts + c * 3;
    double* term = srt + c * 3;
    const double h = hv3_warp(pts, c, s_ref, srt, term, reinterpret_cast<int*>(term + c));
    if (lane == 0) s_contrib[s_front[p]] = TPE_SUB(hv, h);
    __syncwarp();
  }
  __syncthreads();
  if (tid == 0) {
    double mx = s_contrib[0];
    for (int i = 1; i < nf; ++i) mx = (s_contrib[i] > mx || s_contrib[i] != s_contrib[i]) ? s_contrib[i] : mx;
    s_max = fmax(mx, 1e-12);
  }
  __syncthreads();
  if (tid < nf) w[s_map[tid]] = fmax(TPE_DIV(s_contrib[tid], s_max), 1e-12);
}

// k_mo_weights for more than three objectives: Pareto filter by one thread per point, every
// hypervolume by one warp (hv_nd_warp); scratch in the global arena (per warp: warp_stride doubles).
__global__ void __launch_bounds__(1024, 1)
k_mo_weights_nd(const double* __restrict__ vals, int M, const int64_t* __restrict__ rows, int n,
                const int8_t* __restrict__ cat, double* __restrict__ w, double* __restrict__ arena,
                size_t warp_stride, size_t lane_stride) {
  __shared__ double s_v[kMoMaxSet * kMoMaxM];   // feasible points, trial order
  __shared__ double s_ps[kMoMaxSet * kMoMaxM];  // Pareto points, trial order
  __shared__ double s_ref[kMoMaxM];
  __shared__ double s_contrib[kMoMaxSet];
  __shared__ int s_map[kMoMaxSet];
  __shared__ int s_front[kMoMaxSet];
  __shared__ uint8_t s_nd[kMoMaxSet];
  __shared__ int s_nf, s_np;
  __shared__ double s_hv, s_max;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0) {
    int nf = 0;
    for (int i = 0; i < n; ++i) {
      const bool feas = cat[rows[i]] != 2;
      w[i] = feas ? 1.0 : 1e-12;
      if (feas) {
        for (int j = 0; j < M; ++j) s_v[nf * M + j] = vals[rows[i] * M + j];
        s_map[nf++] = i;
      }
    }
    s_nf = nf;
    if (nf > 1) {
      for (int j = 0; j < M; ++j) {
        double worst = s_v[j];
        for (int i = 1; i < nf; ++i) {
          const double v = s_v[i * M + j];
          worst = (v > worst || v != v) ? v : worst;
        }
        double r = fmax(TPE_MUL(1.1, worst), TPE_MUL(0.9, worst));
        if (r == 0.0) r = 1e-12;
        s_ref[j] = r;
      }
    }
  }
  __syncthreads();
  const int nf = s_nf;
  if (nf <= 1) return;
  if (tid < nf) {
    bool dom = false;
    for (int q = 0; q < nf && !dom; ++q) dom = (q != tid) && dominates(s_v + q * M, s_v + tid * M, M);
    s_nd[tid] = dom ? 0 : 1;
  }
  __syncthreads();
  if (tid == 0) {
    int np = 0;
    for (int i = 0; i < nf; ++i)
      if (s_nd[i]) {
        for (int j = 0; j < M; ++j) s_ps[np * M + j] = s_v[i * M + j];
        s_front[np++] = i;
      }
    s_np = np;
  }
  if (tid < nf) s_contrib[tid] = 0.0;
  __syncthreads();
  const int np = s_np;
  double* wsb = arena + (size_t)wid * warp_stride;
  double* pts = wsb;
  double* ws = wsb + (size_t)np * M;
  double* lanes = wsb + hv_warp_scratch_doubles(np, M);
  if (wid == 0) {
    const double hv = hv_nd_warp(s_ps, np, M, s_ref, true, ws, lanes + (size_t)lane * lane_stride);
    if (lane == 0) s_hv = hv;
  }
  __syncthreads();
  const double hv = s_hv;
  if (isinf(hv)) return;
  for (int p = wid; p < np; p += 32) {
    double incl = 1.0;
    for (int j = 0; j < M; ++j) incl = TPE_MUL(incl, TPE_SUB(s_ref[j], s_ps[p * M + j]));
    const int c = np - 1;
    for (int q = lane; q < np; q += 32) {
      if (q == p) continue;
      const int d = q < p ? q : q - 1;
      for (int j = 0; j < M; ++j) {
        const double x = s_ps[q * M + j], y = s_ps[p * M + j];
        pts[d * M + j] = x > y ? x : y;
      }
    }
    __syncwarp();
    const double h = hv_nd_warp(pts, c, M, s_ref, false, ws, lanes + (size_t)lane * lane_stride);
    if (lane == 0) s_contrib[s_front[p]] = TPE_SUB(incl, h);
    __syncwarp();
  }
  __syncthreads();
  if (tid == 0) {
    double mx = s_contrib[0];
    for (int i = 1; i < nf; ++i) mx = (s_contrib[i] > mx || s_contrib[i] != s_contrib[i]) ? s_contrib[i] : mx;
    s_max = fmax(mx, 1e-12);
  }
  __syncthreads();
  if (tid < nf) w[s_map[tid]] = fmax(TPE_DIV(s_contrib[tid], s_max), 1e-12);
}

// ================================================================================================
// Hypervolume weights of a below set of ANY size (sampler.py:824-863) -- global-memory version of k_mo_weights*.
// Only the Pareto front of the feasible below trials enters a hypervolume (everything else gets contribution 0,
// i.e. weight EPS), so the exact work is bounded by the size of that front, not by n_below: with gamma = 0.1 n at
// 20 000 four-objective trials the below set has 2000 trials and its front 34 points.
//   k_mow_prep   one CTA: feasibility, reference point, Pareto flags (thread per point), ordered compaction
//   k_mow_hv     one warp per leave-one-out term (index np = nothing left out: the front's own hypervolume)
//   k_mow_norm   weights = max(contrib / max(contrib), EPS)
// ================================================================================================
struct MowHead {
  int nf, np;
  double hv;
  double ref[kMoMaxM];
};

__global__ void __launch_bounds__(1024, 1)
k_mow_prep(const double* __restrict__ vals, int M, const int64_t* __restrict__ rows, int n, const int8_t* __restrict__ cat,
           double* __restrict__ w, double* __restrict__ fv, int32_t* __restrict__ map, double* __restrict__ ps,
           int32_t* __restrict__ front, double* __restrict__ contrib, MowHead* __restrict__ head) {
  __shared__ int s_warp[32];
  __shared__ double s_red[32];
  __shared__ int s_nan;
  const int tid = threadIdx.x;
  // feasible points in trial order
  int nf = 0;
  for (int base = 0; base < n; base += 1024) {
    const int i = base + tid;
    const bool feas = i < n && cat[rows[i]] != 2;
    if (i < n) w[i] = feas ? 1.0 : 1e-12;
    const int2 rr = block_rank_1024(feas, s_warp);
    if (feas) {
      for (int j = 0; j < M; ++j) fv[(size_t)(nf + rr.x) * M + j] = vals[rows[i] * M + j];
      map[nf + rr.x] = i;
    }
    nf += rr.y;
  }
  __syncthreads();
  if (tid == 0) { head->nf = nf; head->np = 0; head->hv = 0.0; }
  if (nf <= 1) return;
  // reference point: np.max per objective (NaN wins), 1.1 / 0.9 rule, 0 -> EPS (sampler.py:679-683)
  for (int j = 0; j < M; ++j) {
    if (tid == 0) s_nan = 0;
    __syncthreads();
    double mx = -INFINITY;
    for (int i = tid; i < nf; i += 1024) {
      const double v = fv[(size_t)i * M + j];
      if (v != v) s_nan = 1;
      else mx = v > mx ? v : mx;
    }
    for (int o = 16; o > 0; o >>= 1) { const double t = __shfl_xor_sync(0xffffffffu, mx, o); mx = t > mx ? t : mx; }
    if ((tid & 31) == 0) s_red[tid >> 5] = mx;
    __syncthreads();
    if (tid == 0) {
      double worst = s_red[0];
      for (int q = 1; q < 32; ++q) worst = s_red[q] > worst ? s_red[q] : worst;
      if (s_nan) worst = NAN;
      double r = fmax(TPE_MUL(1.1, worst), TPE_MUL(0.9, worst));
      if (r == 0.0) r = 1e-12;
      head->ref[j] = r;
    }
    __syncthreads();
  }
  // Pareto front of the feasible points, trial order
  int np = 0;
  for (int base = 0; base < nf; base += 1024) {
    const int i = base + tid;
    bool keep = false;
    if (i < nf) {
      bool dom = false;
      for (int q = 0; q < nf && !dom; ++q) dom = (q != i) && dominates(fv + (size_t)q * M, fv + (size_t)i * M, M);
      keep = !dom;
      contrib[i] = 0.0;
    }
    const int2 rr = block_rank_1024(keep, s_warp);
    if (keep) {
      for (int j = 0; j < M; ++j) ps[(size_t)(np + rr.x) * M + j] = fv[(size_t)i * M + j];
      front[np + rr.x] = i;
    }
    np += rr.y;
  }
  if (tid == 0) head->np = np;
}

// warp w of the grid evaluates terms p = first + w, first + w + nwarps, ...  (p == np: the whole front -> head->hv).
// The other terms need head->hv: launch once with [np, np] and then with [0, np - 1].
__global__ void __launch_bounds__(128)
k_mow_hv(const double* __restrict__ ps, const int32_t* __restrict__ front, int M, MowHead* __restrict__ head,
         int first, int last, double* __restrict__ contrib, double* __restrict__ arena, size_t warp_stride,
         size_t lane_stride) {
  const int lane = threadIdx.x & 31;
  const int gw = blockIdx.x * 4 + (threadIdx.x >> 5), nw = gridDim.x * 4;
  const int np = head->np;
  const double* ref = head->ref;
  double* wsb = arena + (size_t)gw * warp_stride;
  for (int p = first + gw; p <= last && p <= np; p += nw) {
    const bool whole = p == np;
    if (!whole && isinf(head->hv)) return;   // weights stay at 1 / EPS (sampler.py:846-849)
    const int c = whole ? np : np - 1;
    double* pts = wsb;
    double val;
    if (M <= 3) {
      for (int q = lane; q < np; q += 32) {
        if (q == p) continue;
        const int d = (whole || q < p) ? q : q - 1;
        for (int j = 0; j < M; ++j) pts[(size_t)d * M + j] = ps[(size_t)q * M + j];
      }
      __syncwarp();
      double h;
      if (M == 3) {
        double* srt = pts + (size_t)c * 3;
        double* term = srt + (size_t)c * 3;
        h = hv3_warp(pts, c, ref, srt, term, reinterpret_cast<int*>(term + c));
      } else {
        h = 0.0;
        if (lane == 0) h = hypervolume(pts, c, M, ref, true, pts + (size_t)c * M);
        h = __shfl_sync(0xffffffffu, h, 0);
      }
      val = whole ? h : TPE_SUB(head->hv, h);
    } else {
      double* ws = wsb + (size_t)np * M;
      double* lanes = wsb + (size_t)np * M + hv_warp_scratch_doubles(np, M);
      if (whole) {
        val = hv_nd_warp(ps, np, M, ref, true, ws, lanes + (size_t)lane * lane_stride);
      } else {
        double incl = 1.0;
        for (int j = 0; j < M; ++j) incl = TPE_MUL(incl, TPE_SUB(ref[j], ps[(size_t)p * M + j]));
        for (int q = lane; q < np; q += 32) {
          if (q == p) continue;
          const int d = q < p ? q : q - 1;
          for (int j = 0; j < M; ++j) {
            const double x = ps[(size_t)q * M + j], y = ps[(size_t)p * M + j];
            pts[(size_t)d * M + j] = x > y ? x : y;
          }
        }
        __syncwarp();
        const double h = hv_nd_warp(pts, c, M, ref, false, ws, lanes + (size_t)lane * lane_stride);
        val = TPE_SUB(incl, h);
      }
    }
    if (lane == 0) {
      if (whole) head->hv = val;
      else contrib[front[p]] = val;
    }
    __syncwarp();
  }
}

__global__ void __launch_bounds__(1024, 1)
k_mow_norm(const MowHead* __restrict__ head, const double* __restrict__ contrib, const int32_t* __restrict__ map,
           double* __restrict__ w) {
  __shared__ double s_max;
  const int nf = head->nf;
  if (nf <= 1 || isinf(head->hv)) return;
  if (threadIdx.x == 0) {  // np.max: NaN wins; then max(., EPS)
    double mx = contrib[0];
    for (int i = 1; i < nf; ++i) mx = (contrib[i] > mx || contrib[i] != contrib[i]) ? contrib[i] : mx;
    s_max = fmax(mx, 1e-12);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < nf; i += 1024) w[map[i]] = fmax(TPE_DIV(contrib[i], s_max), 1e-12);
}

}  // namespace tpe
