// Pareto front of a set of objective vectors (optuna/study/_multi_objective.py:171-184, _is_pareto_front), by
// sorting on the first objective and filtering the sorted rows chunk by chunk.
//
// v: [n, M] sign-normalised values (every objective minimised).  on_front_i = no row j has v_j <= v_i in every
// coordinate and v_j < v_i in at least one; identical rows never dominate each other.
//   1. order the rows by coordinate 0 (k_radix_sort_coop, stable) and gather them in that order (k_pf_gather);
//   2. cut the sorted rows into chunks of about kPfChunk rows.  A cut never falls inside a tie run, a run of rows whose
//      coordinates 0 compare == (the host places the cuts from the sorted column, k_pf_gather's s0);
//   3. chunk by chunk, in order: every row of the chunk is tested against the front found so far and against every row
//      of its own chunk (k_pf_filter); the rows nothing dominated are appended to the front (k_pf_append).
// Why this is exact: a dominator of row i has coordinate 0 <= v_i[0], so it lies in an earlier chunk or in i's own.
// One in an earlier chunk, j, is either on the front or dominated by a row k that is (dominance is transitive and
// irreflexive, so some dominator of j is dominated by nothing).  k[0] <= j[0], and ties stay in one chunk, so k lies
// in j's chunk or an earlier one and was appended; k dominates i too.  So i meets a dominator iff it has one.
// Every front row of an earlier chunk is strictly below the current chunk in coordinate 0, so k_pf_filter compares
// front rows from coordinate 1 on.
// -0.0 == +0.0: order_bits folds -0.0 onto +0.0, and the cuts compare the doubles with ==, so a +0.0 row that
// dominates a -0.0 row (or the reverse) is always in that row's chunk and meets the full test.
#pragma once
#include "tpe_common.cuh"

namespace tpe {

constexpr int kPfThreads = 128;   // rows of the chunk per CTA of k_pf_filter = source rows per shared-memory tile
constexpr int kPfSlice = 1024;    // source rows one k_pf_filter CTA tests its rows against (8 tiles)
constexpr int kPfChunk = 4096;    // rows per chunk before a cut is moved to the end of its tie run

// s[p, :] = v[order[p], :]; s0[p] = s[p, 0] (the sorted first coordinate, which the host cuts on)
__global__ void k_pf_gather(const double* __restrict__ v, const int32_t* __restrict__ order, int n, int M,
                            double* __restrict__ s, double* __restrict__ s0) {
  const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (e >= (int64_t)n * M) return;
  const int p = (int)(e / M), j = (int)(e - (int64_t)p * M);
  const double x = v[(int64_t)order[p] * M + j];
  s[e] = x;
  if (j == 0) s0[p] = x;
}

// dom[i] = 1 for each row i of the chunk [c0, c1) of the sorted rows s that a front row (fv[0, *n_front)) or a row of
// the chunk dominates.  blockIdx.x picks kPfThreads rows of the chunk, one per thread.  Source slices of kPfSlice rows
// are spread over blockIdx.y (grid-stride): the first n_fslices cover the front (the host sizes them for the largest
// front the chunk can meet, slices past *n_front are empty), the rest cover the chunk.  A CTA stops as soon as all of
// its rows are dominated, and skips rows another CTA has already flagged.  Dynamic shared memory: pf_filter_smem(M).
__host__ __device__ inline size_t pf_filter_smem(int M) { return (size_t)2 * M * kPfThreads * 8; }
__global__ void __launch_bounds__(kPfThreads, 4)
k_pf_filter(const double* __restrict__ s, int c0, int c1, int M, const double* __restrict__ fv,
            const int* __restrict__ n_front, int n_fslices, uint8_t* __restrict__ dom) {
  extern __shared__ double pf_sm[];
  double* s_me = pf_sm;                            // [M][kPfThreads]: this thread's row, column-major
  double* s_t = pf_sm + (size_t)M * kPfThreads;    // [kPfThreads][M]: tile of source rows
  const int t = threadIdx.x;
  const int i0 = c0 + blockIdx.x * kPfThreads, i = i0 + t;
  const bool live = i < c1;
  for (int j = 0; j < M; ++j) s_me[j * kPfThreads + t] = live ? s[(size_t)i * M + j] : 0.0;
  bool covered = !live || __ldcg(dom + i) != 0;
  // chunk rows above this CTA's largest coordinate 0 dominate none of its rows (s is sorted)
  const double top0 = s[(size_t)(min(c1, i0 + kPfThreads) - 1) * M];
  const int nf = *n_front;
  const int n_slices = n_fslices + (c1 - c0 + kPfSlice - 1) / kPfSlice;
  bool done = false;
  for (int y = blockIdx.y; y < n_slices && !done; y += gridDim.y) {
    const bool front = y < n_fslices;
    const double* src = front ? fv : s;
    const int a = front ? y * kPfSlice : c0 + (y - n_fslices) * kPfSlice;
    const int b = front ? min(nf, a + kPfSlice) : min(c1, a + kPfSlice);
    for (int r0 = a; r0 < b; r0 += kPfThreads) {
      if (!front && src[(size_t)r0 * M] > top0) break;
      // (the barrier also keeps the previous tile until every thread is done with it)
      if (__syncthreads_and(covered)) {
        done = true;
        break;
      }
      const int rows = min(kPfThreads, b - r0);
      for (int q = t; q < rows * M; q += kPfThreads) s_t[q] = src[(size_t)r0 * M + q];
      __syncthreads();
      for (int r = 0; r < rows && !covered; ++r) {
        const double* o = s_t + r * M;
        bool le = true, lt = front;
        for (int j = front ? 1 : 0; j < M; ++j) {
          const double x = o[j], me = s_me[j * kPfThreads + t];
          if (!(x <= me)) {
            le = false;
            break;
          }
          lt = lt || x < me;
        }
        covered = le && lt;
      }
    }
  }
  if (live && covered) dom[i] = 1;
}

// Appends the rows of the chunk [c0, c1) that k_pf_filter left unflagged to the front fv, in sorted order, advances
// *n_front, and sets on_front at their input positions (order).  One CTA of 1024 threads.
__global__ void __launch_bounds__(1024, 1)
k_pf_append(const double* __restrict__ s, const int32_t* __restrict__ order, int c0, int c1, int M,
            const uint8_t* __restrict__ dom, double* __restrict__ fv, int* __restrict__ n_front,
            uint8_t* __restrict__ on_front) {
  __shared__ int s_warp[32];
  int nf = *n_front;   // every thread reads it before the first barrier of block_rank_1024 (c1 > c0)
  for (int p0 = c0; p0 < c1; p0 += 1024) {
    const int i = p0 + threadIdx.x;
    const bool keep = i < c1 && !dom[i];
    const int2 rk = block_rank_1024(keep, s_warp);
    if (keep) {
      for (int j = 0; j < M; ++j) fv[(size_t)(nf + rk.x) * M + j] = s[(size_t)i * M + j];
      on_front[order[i]] = 1;
    }
    nf += rk.y;
  }
  if (threadIdx.x == 0) *n_front = nf;
}

}  // namespace tpe
