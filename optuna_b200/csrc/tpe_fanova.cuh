// fANOVA variances of a fitted random forest (optuna/importance/_fanova/_tree.py): per tree the variance of the
// forest's prediction over the search space, and per (tree, parameter) the variance of the marginal prediction.
//
// Trees are processed in chunks (the host sizes a chunk so that its per-node boxes, nodes x F x 16 bytes, stay
// bounded).  Node indices are global over the concatenated forest; left / right / parent were made global by the
// host, which also validated the arrays (children > parent, each non-root node has one parent).
//   1. boxes, top-down by depth level (k_fa_down): a child's box is its parent's with one bound replaced by the
//      parent's threshold (_get_subspaces, _tree.py:314 -- replacement, not intersection);
//   2. leaves (k_fa_leaf): (value, weight = prod of the box widths); internal nodes, bottom-up by level (k_fa_up):
//      (v_l w_l + v_r w_r) / (w_l + w_r), w_l + w_r (_tree.py:144-181), and the set of parameters split on in the
//      subtree (a bit mask, _precompute_subtree_active_features mapped to parameters);
//   3. the tree variance over the leaves (k_fa_tree_var, _tree.py:33-45);
//   4. split midpoints and sizes per (tree, feature): the thresholds are put in (tree, feature, threshold) order by two
//      passes of the stable cooperative radix sort (threshold, then segment), and k_fa_midpoints keeps the first of
//      every run of == values and forms the edges [low, unique thresholds..., high] (_tree.py:183-222);
//   5. the marginal variance of every (tree, parameter) in one CTA (k_fa_marginal).  For parameter A (its raw feature
//      columns) the reference walks the tree once per grid cell; a node is on some walk iff it is the root or its
//      parent's subtree splits on A, and it ends a walk (a terminal) iff in addition its own subtree does not split
//      on A.  A midpoint x reaches a terminal iff x lies in the terminal's A-box, lo < x <= hi per column (x <=
//      threshold goes left; a tree's thresholds on one feature nest, so the box is the path condition).  Each
//      terminal adds (w / prod_A width, v w / prod_A width) to every cell it covers: through the canonical ranges of a
//      segment tree over the midpoint index for one column, cell by cell for several (a categorical's one-hot
//      columns, at most kFaMaxCells cells).  Only additions: a cell's sums never come from a difference.
//      Then the weighted mean and variance over the cells, with cell weight sum_w * prod(sizes) (_tree.py:47-78).
#pragma once
#include "tpe_common.cuh"

namespace tpe {

constexpr int kFaMaxCells = 1 << 20;   // grid cells of one (tree, parameter); more is TPE_E_INVALID
constexpr int kFaMaxSplitCols = 20;    // columns with >= 2 midpoints in such a grid (2^20 cells)
constexpr int kFaThreads = 256;

__device__ __forceinline__ bool fa_has(const uint64_t* __restrict__ mask, int64_t n, int n_words, int p) {
  return (mask[n * n_words + (p >> 6)] >> (p & 63)) & 1ull;
}

// first index j in [0, K) with mp[j] > x (K if none); mp is non-decreasing
__device__ __forceinline__ int fa_upper(const double* __restrict__ mp, int K, double x) {
  int a = 0, b = K;
  while (a < b) {
    const int m = (a + b) >> 1;
    if (mp[m] > x) b = m; else a = m + 1;
  }
  return a;
}

// box[(n - base) * F + f] for the nodes n of one depth level
__global__ void k_fa_down(const int32_t* __restrict__ lvl, int n_lvl, int64_t base, const int32_t* __restrict__ parent,
                          const int32_t* __restrict__ left, const int32_t* __restrict__ feature,
                          const double* __restrict__ thr, const double2* __restrict__ bounds, int F,
                          double2* __restrict__ box) {
  const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (e >= (int64_t)n_lvl * F) return;
  const int j = (int)(e / F), f = (int)(e - (int64_t)j * F);
  const int n = lvl[j], p = parent[n];
  double2 b;
  if (p < 0) {
    b = bounds[f];
  } else {
    b = box[(p - base) * F + f];
    if (feature[p] == f) {
      if (left[p] == n) b.y = thr[p]; else b.x = thr[p];
    }
  }
  box[(n - base) * F + f] = b;
}

// leaves of the chunk [base, base + cnt): stat = (value, prod of box widths in feature order); mask = 0
__global__ void k_fa_leaf(int64_t base, int cnt, const int32_t* __restrict__ feature, const double* __restrict__ value,
                          const double2* __restrict__ box, int F, int n_words, double2* __restrict__ stat,
                          uint64_t* __restrict__ mask) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= cnt) return;
  const int64_t n = base + i;
  if (feature[n] >= 0) return;
  const double2* b = box + (int64_t)i * F;
  double w = __dsub_rn(b[0].y, b[0].x);
  for (int f = 1; f < F; ++f) w = __dmul_rn(w, __dsub_rn(b[f].y, b[f].x));
  stat[n] = make_double2(value[n], w);
  for (int k = 0; k < n_words; ++k) mask[n * n_words + k] = 0ull;
}

// internal nodes of one depth level (every deeper level done): weighted mean of the children, summed weight, and
// the parameters split on in the subtree (feat_param[f] = parameter of raw feature f, -1 for none)
__global__ void k_fa_up(const int32_t* __restrict__ lvl, int n_lvl, const int32_t* __restrict__ left,
                        const int32_t* __restrict__ right, const int32_t* __restrict__ feature,
                        const int32_t* __restrict__ feat_param, int n_words, double2* __restrict__ stat,
                        uint64_t* __restrict__ mask) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n_lvl) return;
  const int n = lvl[j], f = feature[n];
  if (f < 0) return;
  const int l = left[n], r = right[n];
  const double2 a = stat[l], b = stat[r];
  const double w = __dadd_rn(a.y, b.y);
  stat[n] = make_double2(__ddiv_rn(__dadd_rn(__dmul_rn(a.x, a.y), __dmul_rn(b.x, b.y)), w), w);
  const int p = feat_param[f];
  for (int k = 0; k < n_words; ++k) {
    uint64_t m = mask[(int64_t)l * n_words + k] | mask[(int64_t)r * n_words + k];
    if (p >= 0 && (p >> 6) == k) m |= 1ull << (p & 63);
    mask[(int64_t)n * n_words + k] = m;
  }
}

// sum over the CTA (kFaThreads threads); every thread gets the total
__device__ __forceinline__ double fa_block_sum(double v, double* s_red) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) s_red[warp] = v;
  __syncthreads();
  double t = 0.0;
  for (int k = 0; k < kFaThreads / 32; ++k) t += s_red[k];
  return t;
}

// weighted variance of the leaves of tree t0 + blockIdx.x
__global__ void __launch_bounds__(kFaThreads)
k_fa_tree_var(const int64_t* __restrict__ off, int t0, const int32_t* __restrict__ feature,
              const double2* __restrict__ stat, double* __restrict__ tree_var) {
  __shared__ double s_red[kFaThreads / 32];
  const int t = t0 + blockIdx.x;
  const int64_t a = off[t], b = off[t + 1];
  double sw = 0.0, svw = 0.0;
  for (int64_t n = a + threadIdx.x; n < b; n += kFaThreads)
    if (feature[n] < 0) {
      const double2 s = stat[n];
      sw += s.y;
      svw += s.x * s.y;
    }
  sw = fa_block_sum(sw, s_red);
  svw = fa_block_sum(svw, s_red);
  const double mean = svw / sw;
  double s2 = 0.0;
  for (int64_t n = a + threadIdx.x; n < b; n += kFaThreads)
    if (feature[n] < 0) {
      const double2 s = stat[n];
      const double d = s.x - mean;
      s2 += s.y * d * d;
    }
  s2 = fa_block_sum(s2, s_red);
  if (threadIdx.x == 0) tree_var[t] = s2 / sw;
}

// sort keys of the chunk's nodes: key1 = threshold, key2 = segment (tree - t0) * F + feature; leaves sort last
__global__ void k_fa_keys(int64_t base, int cnt, int t0, int n_seg, const int32_t* __restrict__ tree_of,
                          const int32_t* __restrict__ feature, const double* __restrict__ thr, int F,
                          double* __restrict__ key1, double* __restrict__ key2) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= cnt) return;
  const int64_t n = base + i;
  const int f = feature[n];
  key1[i] = f >= 0 ? thr[n] : INFINITY;
  key2[i] = f >= 0 ? (double)((tree_of[n] - t0) * F + f) : (double)n_seg;
}

__global__ void k_fa_gather(const int32_t* __restrict__ order, int cnt, const double* __restrict__ key,
                            double* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < cnt) out[i] = key[order[i]];
}

// One CTA (1024 threads) per segment s = (tree, feature) of the chunk.  Its thresholds are the sorted positions
// [so[s], so[s + 1]) (node base + order1[order2[p]]).  Edges e = [low, unique thresholds..., high] at e_buf[so[s] + 2s],
// midpoints 0.5 (e_j + e_{j+1}) and sizes e_{j+1} - e_j at mp / sz[so[s] + s]; K[s] = number of midpoints.
__global__ void __launch_bounds__(1024, 1)
k_fa_midpoints(int64_t base, const int32_t* __restrict__ order1, const int32_t* __restrict__ order2,
               const int64_t* __restrict__ so, const double* __restrict__ thr, const double2* __restrict__ bounds,
               int F, double* __restrict__ e_buf, double* __restrict__ mp, double* __restrict__ sz,
               int32_t* __restrict__ K) {
  __shared__ int s_warp[32];
  const int s = blockIdx.x;
  const int64_t a = so[s], b = so[s + 1];
  double* e = e_buf + a + 2 * s;
  int k = 0;
  for (int64_t p0 = a; p0 < b; p0 += 1024) {
    const int64_t p = p0 + threadIdx.x;
    double th = 0.0;
    bool first = false;
    if (p < b) {
      th = thr[base + order1[order2[p]]];
      first = p == a || thr[base + order1[order2[p - 1]]] != th;
    }
    const int2 rk = block_rank_1024(first, s_warp);
    if (first) e[1 + k + rk.x] = th;
    k += rk.y;
  }
  const double2 bd = bounds[s % F];
  if (threadIdx.x == 0) {
    e[0] = bd.x;
    e[k + 1] = bd.y;
    K[s] = k + 1;
  }
  __syncthreads();
  for (int j = threadIdx.x; j <= k; j += 1024) {
    mp[a + s + j] = 0.5 * __dadd_rn(e[j + 1], e[j]);
    sz[a + s + j] = __dsub_rn(e[j + 1], e[j]);
  }
}

// Marginal variance of parameter p = blockIdx.x in tree t = t0 + blockIdx.y.  cols = raw_features[po[p], po[p + 1]).
// acc (zeroed, at acc_off[(t - t0) * n_params + p]): a segment tree of 2 P (sum_w, sum_vw) for one column (leaf i at
// P + i), else one (sum_w, sum_vw) per cell (mixed radix over cols, the last column fastest, as itertools.product).
__global__ void __launch_bounds__(kFaThreads)
k_fa_marginal(const int64_t* __restrict__ off, int t0, int64_t base, int n_params, const int32_t* __restrict__ po,
              const int32_t* __restrict__ cols, const int32_t* __restrict__ parent, const double2* __restrict__ stat,
              const uint64_t* __restrict__ mask, int n_words, const double2* __restrict__ box, int F,
              const int64_t* __restrict__ so, const double* __restrict__ mp, const double* __restrict__ sz,
              const int32_t* __restrict__ K, const int64_t* __restrict__ acc_off, double2* __restrict__ acc_buf,
              double* __restrict__ marginal_var, int n_trees) {
  __shared__ double s_red[kFaThreads / 32];
  const int p = blockIdx.x, tl = blockIdx.y, t = t0 + tl;
  const int c0 = po[p], nc = po[p + 1] - c0;
  double2* acc = acc_buf + acc_off[(int64_t)tl * n_params + p];
  // seg_of(c) = tl * F + c; its midpoints start at so[seg] + seg
  int cells = 1, P = 1;
  for (int j = 0; j < nc; ++j) cells *= K[tl * F + cols[c0 + j]];
  if (cells == 1) {
    if (threadIdx.x == 0) marginal_var[(int64_t)p * n_trees + t] = 0.0;
    return;
  }
  if (nc == 1) while (P < cells) P <<= 1;
  // 1. terminals
  const int64_t a = off[t], b = off[t + 1];
  for (int64_t n = a + threadIdx.x; n < b; n += kFaThreads) {
    const int q = parent[n];
    if ((q >= 0 && !fa_has(mask, q, n_words, p)) || fa_has(mask, n, n_words, p)) continue;
    const double2* bx = box + (n - base) * F;
    double card = 1.0;
    for (int j = 0; j < nc; ++j) {
      const double2 c = bx[cols[c0 + j]];
      card = __dmul_rn(card, __dsub_rn(c.y, c.x));
    }
    const double2 st = stat[n];
    const double W = __ddiv_rn(st.y, card), V = __dmul_rn(st.x, W);
    if (nc == 1) {
      const int sg = tl * F + cols[c0];
      const double* m = mp + so[sg] + sg;
      const double2 c = bx[cols[c0]];
      int l = P + fa_upper(m, cells, c.x), r = P + fa_upper(m, cells, c.y);
      for (; l < r; l >>= 1, r >>= 1) {
        if (l & 1) { atomicAdd(&acc[l].x, W); atomicAdd(&acc[l].y, V); ++l; }
        if (r & 1) { --r; atomicAdd(&acc[r].x, W); atomicAdd(&acc[r].y, V); }
      }
      continue;
    }
    // several columns: the index range of each column with >= 2 midpoints (a column the tree never splits on is
    // never tested by the walk), then every covered cell
    int lo[kFaMaxSplitCols], hi[kFaMaxSplitCols], stride[kFaMaxSplitCols];
    int ns = 0, cell0 = 0, str = 1;
    bool empty = false;
    for (int j = nc - 1; j >= 0 && !empty; --j) {
      const int sg = tl * F + cols[c0 + j];
      const int Kc = K[sg];
      if (Kc >= 2) {
        const double* m = mp + so[sg] + sg;
        const double2 c = bx[cols[c0 + j]];
        const int u = fa_upper(m, Kc, c.x), v = fa_upper(m, Kc, c.y);
        empty = u >= v;
        lo[ns] = u; hi[ns] = v; stride[ns] = str;
        cell0 += u * str;
        ++ns;
      }
      str *= Kc;
    }
    if (empty) continue;
    int idx[kFaMaxSplitCols];
    for (int j = 0; j < ns; ++j) idx[j] = lo[j];
    int cell = cell0;
    while (true) {
      atomicAdd(&acc[cell].x, W);
      atomicAdd(&acc[cell].y, V);
      int j = 0;
      for (; j < ns; ++j) {
        if (++idx[j] < hi[j]) { cell += stride[j]; break; }
        cell -= (idx[j] - 1 - lo[j]) * stride[j];
        idx[j] = lo[j];
      }
      if (j == ns) break;
    }
  }
  __syncthreads();
  // 2. per cell: value = sum_vw / sum_w, weight = sum_w * prod(sizes); weighted mean, then variance
  double sw = 0.0, svw = 0.0;
  for (int pass = 0; pass < 2; ++pass) {
    const double mean = pass ? svw / sw : 0.0;
    double r0 = 0.0, r1 = 0.0;
    for (int i = threadIdx.x; i < cells; i += kFaThreads) {
      double W = 0.0, V = 0.0, size = 1.0;
      if (nc == 1) {
        for (int j = P + i; j >= 1; j >>= 1) {
          const double2 x = __ldcg(&acc[j]);
          W += x.x;
          V += x.y;
        }
        const int sg = tl * F + cols[c0];
        size = sz[so[sg] + sg + i];
      } else {
        const double2 x = __ldcg(&acc[i]);
        W = x.x;
        V = x.y;
        int rest = i, str = cells;
        for (int j = 0; j < nc; ++j) {
          const int sg = tl * F + cols[c0 + j];
          str /= K[sg];
          const int ij = rest / str;
          rest -= ij * str;
          size = __dmul_rn(size, sz[so[sg] + sg + ij]);
        }
      }
      const double v = V / W, w = W * size;
      if (pass == 0) {
        r0 += w;
        r1 += v * w;
      } else {
        const double d = v - mean;
        r0 += w * d * d;
      }
    }
    r0 = fa_block_sum(r0, s_red);
    if (pass == 0) {
      r1 = fa_block_sum(r1, s_red);
      sw = r0;
      svw = r1;
    } else if (threadIdx.x == 0) {
      marginal_var[(int64_t)p * n_trees + t] = r0 / sw;
    }
  }
}

}  // namespace tpe
