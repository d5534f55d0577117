// TEST-ONLY host instantiation of the per-trial part of optuna_b200/csrc/tpe_hvhist.cuh (the product never links
// this).  Lets `pytest -m "not gpu"` check the hypervolume-history arithmetic against the reference without a GPU
// (tests/_hvhist_engine.py).
#include "../../optuna_b200/csrc/tpe_motpe.cuh"
#define TPE_HVHIST_HOST_ONLY
#include "../../optuna_b200/csrc/tpe_hvhist.cuh"
#include <vector>

extern "C" {
// HV(max(front_p, v_i)) of added trial p (i = list[p]) as k_hh_front + k_hh_hv compute it: gather the added trials
// q < p with death[q] >= i, clip them by v_i, keep the unique non-dominated rows in lexicographic order, and
// evaluate them with hypervolume() (whose paths hv_2d / hv3_warp / hv_nd_warp reproduce bit for bit).
// v [n, m]; list [K] added trials ascending; death [K].  *kept = rows that reached the hypervolume.
double shim_hvhist_trial(const double* v, const int* list, const int* death, int p, int m, const double* ref,
                         int* kept) {
  const int ip = list[p];
  std::vector<double> C;
  for (int q = 0; q < p; ++q) {
    if (death[q] < ip) continue;
    C.resize(C.size() + m);
    tpe::hh_clip_row(v + (size_t)list[q] * m, v + (size_t)ip * m, m, C.data() + C.size() - m);
  }
  const int c = (int)(C.size() / m);
  std::vector<uint8_t> keep(c);
  for (int k = 0; k < c; ++k) keep[k] = !tpe::hh_dropped(C.data(), c, k, m);
  int w = 0;
  for (int k = 0; k < c; ++k) w += keep[k];
  std::vector<double> S((size_t)w * m);
  for (int k = 0; k < c; ++k)
    if (keep[k]) {
      const int r = tpe::hh_lexrank(C.data(), keep.data(), c, k, m);
      for (int j = 0; j < m; ++j) S[(size_t)r * m + j] = C[(size_t)k * m + j];
    }
  *kept = w;
  std::vector<double> arena(tpe::hv_arena_doubles(w, m) + 16);
  memset(arena.data(), 0xFF, arena.size() * 8);
  return tpe::hypervolume(S.data(), w, m, ref, true, arena.data());
}
}
