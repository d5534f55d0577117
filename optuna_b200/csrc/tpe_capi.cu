// C ABI of libtpe_b200.so (see include/optuna_b200_tpe.h) -- host orchestration of the kernels in
// tpe_kernels.cuh.  No torch types, no Python: plain pointers and sizes.
#include <cuda_runtime.h>
#include <math.h>
#include <stdarg.h>
#include <stddef.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <mutex>
#include <thread>
#include <set>
#include <string>
#include <vector>

#include "../../include/optuna_b200_tpe.h"
#include "tpe_kernels.cuh"
#include "tpe_motpe_kernels.cuh"
#include "tpe_hvhist.cuh"
#include "tpe_pareto.cuh"
#include "tpe_fanova.cuh"
#include "tpe_gp.cuh"
#include "tpe_gpbatch.cuh"
#include "tpe_gpemmr.cuh"
#include "tpe_ehvi.cuh"
#include "tpe_acqf.cuh"
#include "tpe_boxdec.cuh"
#include "tpe_uni.cuh"
#include "tpe_mixed.cuh"
#include "tpe_tcscreen.cuh"
#include "tpe_unib.cuh"
// Lab build (-DTPE_LAB): the experimental grid kernels and the timing-attribution variants, selectable by
// environment variables.  Some of them switch parts of the
// log-sum-exp off (wrong results by design).  The product library contains none of them.
#ifdef TPE_LAB
#include "tpe_screen.cuh"
#endif

using namespace tpe;

namespace {

struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  bool owned = true;   // false: a view of another context's buffer (batched univariate sub-contexts)
  void alias(void* q, size_t bytes) {
    if (owned && p) cudaFree(p);
    p = q;
    cap = bytes;
    owned = false;
  }
  cudaError_t ensure(size_t bytes) {
    if (!owned) { p = nullptr; cap = 0; owned = true; }
    if (bytes <= cap) return cudaSuccess;
    // 12 % headroom: a study grows by one trial per suggestion, and a cudaFree + cudaMalloc of a 50 MB table in the
    // middle of an ask costs milliseconds (and synchronises the device)
    size_t want = std::max(bytes + bytes / 8, cap + cap / 2);
    want = (want + 255) & ~(size_t)255;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    cudaError_t e = cudaMalloc(&p, want);
    if (e == cudaSuccess) cap = want;
    return e;
  }
  // grow while keeping the first `keep` bytes
  cudaError_t grow(size_t bytes, size_t keep, cudaStream_t st) {
    if (bytes <= cap) return cudaSuccess;
    size_t want = std::max(bytes, cap * 2);
    want = (want + 255) & ~(size_t)255;
    void* q = nullptr;
    cudaError_t e = cudaMalloc(&q, want);
    if (e != cudaSuccess) return e;
    if (p && keep) e = cudaMemcpyAsync(q, p, keep, cudaMemcpyDeviceToDevice, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (p) cudaFree(p);
    p = q;
    cap = want;
    return e;
  }
  template <class T>
  T* as() const { return reinterpret_cast<T*>(p); }
  void release() {
    if (p && owned) cudaFree(p);
    p = nullptr;
    cap = 0;
    owned = true;
  }
};

struct Estimator {
  int64_t n = 0, K = 0;
  DevBuf rows, pos, wstage, wpart, w, logw, cdf, mu, sigma, cst_part, cst, tabp, tabc, colprm, tab, part, fix;
  DevBuf tab32, tab64p, d32;   // fp32-screening copies (tpe_screen.cuh)
  DevBuf cls, dtab, offgrid;   // tabulated discrete columns (multivariate)
  DevBuf tabm, hb, ckk;        // tensor-core kernel: fragment-major table, |mu''|^2 / 2, cst - |mu''|^2 / 2
  DevBuf uord, us32, usmi, usc, umeta;  // univariate 1-D grid (tpe_uni.cuh): sorted order and sorted tables
  DevBuf ucoef, ubox, ubstart, utlist;  // ... and the fast Gauss transform of the floor-bandwidth kernels
  bool fgt = false;
  DevBuf tcs_h, tcs_ak, tcs_ak64;       // bf16 tensor-core screen of the multivariate grid (tpe_tcscreen.cuh)
  bool tcs = false;
  int64_t tcs_kpad = 0;
  DevBuf mxc, mxd;                      // mixed spaces, many candidates (tpe_mixed.cuh): kernel-minor tables
  bool mixed = false;
  int64_t mix_kstride = 0;
  bool uni_ready = false;
  bool mma = false;            // tables above are valid for this build
  bool screen_ready = false;
  int nsplit = 0;
  void release() {
    for (DevBuf* b : {&uord, &us32, &usmi, &usc, &umeta, &ucoef, &ubox, &ubstart, &utlist, &mxc, &mxd, &tcs_h, &tcs_ak, &tcs_ak64, &tabm, &hb, &ckk, &cls, &dtab, &offgrid, &tab32, &tab64p, &d32, &rows, &pos, &wstage, &wpart, &w, &logw, &cdf, &mu, &sigma, &cst_part, &cst, &tabp, &tabc, &colprm, &tab,
                      &part, &fix})
      b->release();
  }
};

// Gaussian process of the terminator's regret bound (tpe_gp_*, tpe_gp.cuh): the data of tpe_gp_set_data and the
// exact-size buffers -- two n x n matrices (A holds at least 1024 rows of n for the posterior's cross covariance)
struct GpState {
  int64_t n = 0;
  int32_t P = 0;
  double *X = nullptr, *y = nullptr, *A = nullptr, *B = nullptr, *W = nullptr, *u = nullptr, *alpha = nullptr;
  double *prm = nullptr, *part = nullptr, *scal = nullptr, *grad = nullptr, *Xq = nullptr, *ucb = nullptr,
         *lcb = nullptr, *dmean = nullptr, *dvar = nullptr;
  uint8_t* cat = nullptr;
  int* fail = nullptr;
  int64_t part_cap = 0, xq_cap = 0;
  bool ready = false;         // tpe_gp_set_data completed: every buffer above is allocated
  bool conditioned = false;   // B, alpha and prm hold the factor of tpe_gp_condition: tpe_gp_query may read them
  void release() {
    for (void* p : {(void*)X, (void*)y, (void*)A, (void*)B, (void*)W, (void*)u, (void*)alpha, (void*)prm, (void*)part,
                    (void*)scal, (void*)grad, (void*)Xq, (void*)ucb, (void*)lcb, (void*)dmean, (void*)dvar,
                    (void*)cat, (void*)fail})
      if (p) cudaFree(p);
    *this = GpState();
  }
};

// Many Gaussian processes of one study at once (tpe_gp_batch_*, tpe_gpbatch.cuh): the packed data of
// tpe_gp_batch_set, and the per-call buffers (jobs, per-job workspace, outputs) of the loss and bounds calls
struct GpBatchState {
  int32_t n_gp = 0, P = 0;
  std::vector<int64_t> off;   // host copy of the row offsets [n_gp + 1]
  DevBuf X, y, doff, cat, idx, prm, nexc, ws, wsoff, loss, grad, status, beta, Xs, out, rows;
  bool ready = false;
  void release() {
    for (DevBuf* b : {&X, &y, &doff, &cat, &idx, &prm, &nexc, &ws, &wsoff, &loss, &grad, &status, &beta, &Xs, &out,
                      &rows})
      b->release();
    *this = GpBatchState();
  }
};

// log-EHVI of GPSampler's multi-objective acquisition (tpe_ehvi_*, tpe_ehvi.cuh): the box decomposition and the QMC
// samples of tpe_ehvi_set, and the per-call buffers of tpe_ehvi
struct EhviState {
  int64_t B = 0;
  int32_t S = 0, M = 0;
  DevBuf lbI, Z, mean, sd, part, value, dmean, dsd;
  bool ready = false;
  void release() {
    for (DevBuf* b : {&lbI, &Z, &mean, &sd, &part, &value, &dmean, &dsd}) b->release();
    *this = EhviState();
  }
};

// GPSampler's acquisition function (tpe_acqf_*, tpe_acqf.cuh): the GP contexts of tpe_acqf_set with the conditioning
// generation each had then, one event per GP context, the thresholds, and the per-call buffers of tpe_acqf_eval.  The
// log-EHVI boxes and samples live in the context's EhviState.
struct AcqfState {
  int32_t kind = 0, n_obj = 0, P = 0;
  double noise = 0.0;
  std::vector<tpe_ctx*> gps;
  std::vector<uint64_t> gen;
  std::vector<cudaEvent_t> ev;
  DevBuf thr, X, mean, var, dmean, dvar, coef, value, grad;
  bool ready = false;
  void release() {
    for (DevBuf* b : {&thr, &X, &mean, &var, &dmean, &dvar, &coef, &value, &grad}) b->release();
    for (cudaEvent_t e : ev) cudaEventDestroy(e);
    *this = AcqfState();
  }
};

// non-dominated box decomposition (tpe_box_decomposition, tpe_boxdec.cuh): the pool of k_bd_pass (cap bounds, kept
// across calls), the sorting and selection scratch, and the result of the last call on the host
struct BoxDecState {
  int64_t cap = 0;
  DevBuf ub, dp, live, act, dlist, dmask, doff, stat;
  DevBuf rows, ref, sorted, front, key, idx, work, keep, sel, cnt, lo, hi;
  std::vector<double> lower, upper;
  int64_t stats[6] = {0, 0, 0, 0, 0, 0};
  bool ready = false;
  void release() {
    for (DevBuf* b : {&ub, &dp, &live, &act, &dlist, &dmask, &doff, &stat, &rows, &ref, &sorted, &front, &key, &idx,
                      &work, &keep, &sel, &cnt, &lo, &hi})
      b->release();
    *this = BoxDecState();
  }
};

}  // namespace

struct tpe_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  // the above-set estimator is built on a second stream while the main stream builds l(x), samples
  // the candidates and evaluates them under l(x); joined before the first consumer of est[1]
  cudaStream_t stream2 = nullptr;
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  bool above_pending = false;
  // tpe_suggest uploads the uniforms on a third stream before the split starts
  cudaStream_t stream3 = nullptr;
  cudaEvent_t ev_u = nullptr;
  const double* u_staged = nullptr;
  int64_t u_staged_count = 0;
  bool u_device_rng = false;     // U was filled by k_mt19937_uniform (tpe_stage_uniforms_mt19937)
  DevBuf mt_state;               // 624 state words + pos: generator state after the staged uniforms
  // Speculation: while an ask is evaluated, the uniforms of the NEXT ask (same count) are generated from
  // the end state into U2 / mt_spec.  The next tpe_stage_uniforms_mt19937 adopts them if the caller's
  // generator is exactly in that state (mt_host, as returned by tpe_rng_state); otherwise they are dropped.
  DevBuf U2, mt_spec;
  DevBuf mt_jump, mt_tmp;        // jump-ahead polynomials (kMtJumpTable) / end state of the multi-CTA generator
  bool mt_jump_ready = false;
  cudaEvent_t ev_spec = nullptr;
  bool spec_pending = false, mt_host_valid = false;
  int64_t spec_count = 0;
  uint32_t* mt_host = nullptr;   // page-locked host copy of mt_state (625 words), read back with the results of the ask
                                 // (page-locked: a copy into pageable memory would make the asynchronous entry points wait)
  cudaEvent_t ev[9] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  std::mutex mu;
  std::string err;
  int sm_count = 132;   // H100 SXM; replaced by the device's count at context creation

  // search space
  std::vector<tpe_param_desc> space;
  std::vector<double> cat_dist_h;
  std::vector<int64_t> cat_dist_off;
  DevBuf cat_dist;

  // history
  DevBuf X, cat, key, vals;
  int32_t M = 1;                 // objectives (>= 2: MOTPE)
  std::vector<int8_t> cat_h;     // host mirror of the categories (MOTPE list building)
  int64_t cat_cnt[5] = {0, 0, 0, 0, 0};  // trials per category incl. TPE_CAT_EXCLUDED (sizes of the split without a read-back)
  // the split depends on the history and n_below only (not on the selected columns, unless rows lack
  // parameters): consecutive tpe_prepare calls on the same history -- the P sample_independent calls of a
  // univariate trial -- reuse it
  uint64_t hist_version = 0, split_version = 0;
  int64_t split_n_below = -1;
  bool split_valid = false;
  int64_t N = 0;
  // MOTPE scratch
  DevBuf mo_list, mo_alive, mo_dom, mo_first, mo_rank, mo_ctr, mo_tie, mo_ntie, mo_lexpos, mo_isdup, mo_sorted,
      mo_uniq, mo_nuniq, mo_ref, mo_removed, mo_contrib, mo_bound, mo_state, mo_arena, mo_chosen, mo_diag, mo_w, mo_table,
      mo_sample, mo_surv, mo_nsurv, mo_fv, mo_ps, mo_map, mo_front, mo_head;
  bool mo_weights_ready = false;
  std::vector<uint8_t> col_missing, col_oor, col_offgrid;   // col_offgrid: a step column holds a value off its grid
  bool history_set = false;

  // current call
  bool prepared = false, built = false, sampled = false;
  tpe_cfg cfg{};
  std::vector<ColMeta> cols_h;
  DevBuf cols;
  int32_t pc = 0, ncont = 0, ndisc = 0, ncat = 0, nnum = 0, pb = 0;
  int64_t tab_doubles = 0;
  int64_t dtab_doubles = 0;  // cell-mass tables of tabulated discrete columns
  bool fast = false;
  bool uni_fast = false;   // one continuous column, univariate: the sorted 1-D grid kernel (tpe_uni.cuh)
  bool cands_sorted = false;
  DevBuf uxs, ucidx;
  int fast_mode = 0;  // 0 generic, 1 PAIR (sigma per kernel), 2 CONST (sigma per column)
  tpe_split_info info{};
  DevBuf row_ok, member, counts, split_work, below_all;
  Estimator est[2];
  DevBuf sort_val, sort_idx, sort_work;

  // candidates
  int64_t n_asks = 0, Ct = 0, ct_stride = 0;
  DevBuf U, S, xT, oob, logl, logg, out_x, out_acq, out_best, x64s, x32s, e32s, gmax, lse_gmax;
  bool screen_attr_set = false;
  float ms[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  int32_t launches = 0;
  const char* last_kernel = "none";
  int32_t launch_counter = 0;
  std::set<const void*> prepared_cfgs;
  // batched univariate suggestions (tpe_suggest_univariate_batch): one light sub-context per column -- own streams,
  // own estimator / candidate buffers, views of this context's history and split
  std::vector<tpe_ctx*> uni_sub;
  cudaEvent_t ev_uni = nullptr;
  bool is_sub = false;
  // staged univariate batch (tpe_unib.cuh): one arena carved per call + the sorted orders kept between calls
  DevBuf ub_arena, ub_ord_a, ub_ord_b, ub_wstage;
  int ub_ord_cur = 0;                  // which of ub_ord_a / ub_ord_b holds the latest above orders
  uint64_t ub_ord_seq = 0, ub_ord_lineage = 0;
  int64_t ub_ord_K = -1, ub_ord_ks = 0;
  std::vector<int32_t> ub_ord_cols;
  int ub_sort_g = 0;
  bool mixed_ok = false;         // the selected columns suit k_logpdf_mixed (setup_columns)
  std::vector<MixCol> mixcols_h;
  DevBuf mixcols;
  int mix_ncont = 0, mix_nd = 0, mix_tabd = 0;
  bool user_points = false;      // the resident candidates came through tpe_logpdf, not from k_sample
  static constexpr size_t kUpSlot = 8192;     // page-locked staging of small history uploads (upload_history)
  static constexpr int kUpSlots = 16;
  void* up_host = nullptr;
  cudaEvent_t up_ev[kUpSlots] = {};
  bool up_used[kUpSlots] = {};
  int up_next = 0;
  // one suggestion over several GPUs: this context evaluates g(x) over its slice of the above kernels only
  // (tpe_set_kernel_shard, tpe_sample_and_partial, tpe_finish_from_partials)
  int32_t kshard_rank = 0, kshard_world = 1;
  DevBuf kpart;
  bool partial_ready = false;
  bool deferred = false;         // tpe_sample_and_select_async issued, tpe_collect not yet called
  int64_t deferred_uni = 0;      // tpe_suggest_univariate_batch_async issued (columns), not yet collected
  bool deferred_uni_rng = false;
  bool issued_dev_rng = false;
  void* res_host = nullptr;      // page-locked staging of deferred results
  size_t res_host_cap = 0;
  int sort_cta_cap = 0;          // sub-contexts: CTAs of a cooperative sort (several sorts share the GPU)
  // incremental sorted orders (univariate batch): the parent compares the above rows of this call with the previous
  // call's; every column context then updates its order instead of sorting (k_rows_delta / k_order_update)
  uint64_t hist_lineage = 0;     // changes whenever rows the estimators can see are replaced (not on appends)
  DevBuf uni_prev_rows, uni_mode, uni_work;
  int64_t uni_prev_n = -1;
  uint64_t uni_prev_lineage = 0;
  const int* uni_mode_ptr = nullptr;   // sub-contexts: the parent's mode word, or nullptr (always sort)
  uint64_t uni_seq = 0;                // batch calls so far (sub-contexts: the running call's number)
  uint64_t uni_ord_seq = 0;            // sub-contexts: the call that left the cached order of est[1] ...
  uint64_t uni_ord_lineage = 0;        // ... and what else it belongs to
  int32_t uni_ord_col = -1;
  int64_t uni_ord_K = -1;
  GpState gp;
  uint64_t gp_generation = 0;   // successful tpe_gp_condition calls: an acquisition context checks it is unchanged
  GpBatchState gpb;
  EhviState ehvi;
  BoxDecState boxdec;
  AcqfState acqf;
};

namespace {

int fail(tpe_ctx* c, int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  if (c) c->err = buf;
  return code;
}

#define CU(call)                                                                                   \
  do {                                                                                             \
    cudaError_t e_ = (call);                                                                       \
    if (e_ != cudaSuccess)                                                                         \
      return fail(ctx, e_ == cudaErrorMemoryAllocation ? TPE_E_NOMEM : TPE_E_CUDA, "%s failed: %s (%s:%d)", \
                  #call, cudaGetErrorString(e_), __FILE__, __LINE__);                              \
  } while (0)

// slot of a history category in cat_cnt: anything outside 0..3 is TPE_CAT_EXCLUDED
inline int cat_slot(int8_t c) { return (c >= 0 && c <= 3) ? c : 4; }

inline int grid_for(int64_t work, int threads, int cap) {
  int64_t g = (work + threads - 1) / threads;
  if (g < 1) g = 1;
  if (g > cap) g = cap;
  return (int)g;
}

template <class T>
constexpr T round_up(T v, T m) { return (v + m - 1) / m * m; }

// ---- fast-kernel configuration table ------------------------------------------------------------
struct FastCfg {
  int pb, cands_per_cta, nt, tk, st, minb;
  size_t smem;
  void (*launch)(dim3, size_t, cudaStream_t, const void*, const double*, int64_t, const double2*, const double*,
                 int64_t, int64_t, double, double2*, unsigned long long*);
  cudaError_t (*prepare)();
};

template <int PB, int PS, int RC, int NT, int TK, int ST, bool PAIR, int MINB>
struct FastInst {
  static constexpr size_t smem = (size_t)ST * TK * PB * (PAIR ? 16 : 8) + (size_t)ST * TK * 8 + (size_t)ST * 8;
  static void launch(dim3 grid, size_t sm, cudaStream_t st, const void* tab, const double* cst, int64_t Kf,
                     const double2* colprm, const double* xT, int64_t ct_stride, int64_t kps, double skip,
                     double2* part, unsigned long long*) {
    k_logpdf_fast<PB, PS, RC, NT, TK, ST, PAIR, MINB>
        <<<grid, NT, sm, st>>>(tab, cst, Kf, colprm, xT, ct_stride, kps, skip, part);
  }
  static cudaError_t prepare() {
    return cudaFuncSetAttribute(k_logpdf_fast<PB, PS, RC, NT, TK, ST, PAIR, MINB>,
                                cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  }
  static FastCfg cfg() { return FastCfg{PB, (NT / 32) * (32 / PS) * RC, NT, TK, ST, MINB, smem, &launch, &prepare}; }
};

// Tensor-core (DMMA) instances of the CONST kernel: same launch signature (tab = fragment-major table,
// cst = ckk, Kf = kernels rounded up to 8).
constexpr int kMmaKPad = 32;  // kernels are padded to 8 * KG (KG <= 4)
template <int PB, int M, int KG, int NT, int TK, int ST, int MINB, int DBG = 0>
struct MmaInst {
  static constexpr size_t smem = MmaSmem<PB, M, KG, NT, TK, ST, MINB>::bytes;   // TMA stages + near-term ring
  static void launch(dim3 grid, size_t sm, cudaStream_t st, const void* tab, const double* cst, int64_t Kf,
                     const double2* colprm, const double* xT, int64_t ct_stride, int64_t kps, double skip,
                     double2* part, unsigned long long* gmax) {
    // near tier: within ln K + 17.5 of the reference max (see LseRef); TPE_TNEAR_DELTA shrinks it for
    // timing experiments only (the accuracy bound no longer holds)
#ifdef TPE_LAB
    static const double delta = [] { const char* v = getenv("TPE_TNEAR_DELTA"); return v ? atof(v) : 0.0; }();
#else
    constexpr double delta = 0.0;
#endif
    k_logpdf_mma<PB, M, KG, NT, TK, ST, MINB, DBG><<<grid, NT, sm, st>>>(static_cast<const double*>(tab), cst, Kf, colprm,
                                                                        xT, ct_stride, kps, skip, part, gmax,
                                                                        skip - 12.5 - delta);
  }
  static cudaError_t prepare() {
    return cudaFuncSetAttribute(k_logpdf_mma<PB, M, KG, NT, TK, ST, MINB, DBG>,
                                cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  }
  static FastCfg cfg() { return FastCfg{PB, (NT / 32) * 8 * M, NT, TK, ST, MINB, smem, &launch, &prepare}; }
};
#ifdef TPE_LAB
#endif  // TPE_LAB
// Tilings measured on an H100 SXM (400 W power limit, 1980 MHz max SM clock), CUDA events around the g(x)
// launch, 100k kernels (tools/tune_mma.py).  M = 2 issues mma.m16n8k8 (twice the m8n8k4 rate on H100), M = 1
// issues m8n8k4.  With two candidate groups per warp a thread needs 120-200 registers, so the big path runs
// 16 warps per SM (8 for P = 64); the probe (tools/probe_dmma2.cu) shows that 8 warps with one m16n8k8 chain
// each already saturate the pipe.  4096 candidates:
//   P = 16: 1.18 ms (m8n8k4: 1.27)   P = 32: 1.14 ms (m8n8k4: 1.41)   P = 64: 1.77 ms (m8n8k4: 2.15)
//   P = 8: m8n8k4 stays faster: 1.151-1.154 ms against 1.190 ms for the best m16n8k8 tiling in three alternated
//   pairs of runs (the means of one tiling spread by 0.003 ms, the gap is 0.037 ms).
// Small path (one ask of 24 candidates): m8n8k4 stays at P <= 32 (14-30 % faster there).  At P = 64 m16n8k8 wins
// since the steps are software-pipelined: 0.061 against 0.065 ms (H100 SXM, 400 W).
// The big path at P = 8 and 16 runs 2 TMA stages of the same tile instead of 3, so that the near-term ring
// (MmaSmem) fits beside them at 2 CTAs per SM.
//                                   PB M KG  NT   TK ST MINB
const FastCfg kMmaBig[] = {
    MmaInst<8, 1, 4, 256, 512, 2, 2>::cfg(), MmaInst<16, 2, 2, 256, 256, 2, 2>::cfg(),
    MmaInst<32, 2, 1, 256, 128, 2, 2>::cfg(), MmaInst<64, 2, 2, 256, 64, 3, 1>::cfg(),
};
const FastCfg kMmaSmall[] = {
    MmaInst<8, 1, 4, 64, 512, 3, 4>::cfg(), MmaInst<16, 1, 4, 64, 256, 3, 4>::cfg(),
    MmaInst<32, 1, 4, 64, 128, 3, 4>::cfg(), MmaInst<64, 2, 2, 64, 64, 3, 3>::cfg(),
};
#ifdef TPE_LAB
// Tilings for every width, big and small path, selected by TPE_MMA_LAB=<index> when the width matches
// (tools/tune_mma.py); DBG = 1 / 2 time the mma + TMA floor and the classification + far tier alone, DBG = 4 the mma +
// TMA floor without the per-tile exchange of maxima (sync_global), DBG = 5 is the full kernel with the near-term
// counters (g_mma_lab_count, read by tpe_lab_mma_counters).
//                                   PB M KG  NT   TK ST MINB DBG
const FastCfg kMmaLab[] = {
    MmaInst<32, 1, 2, 256, 128, 2, 3, 1>::cfg(),  //  0
    MmaInst<32, 1, 2, 256, 128, 2, 3, 2>::cfg(),  //  1
    MmaInst<32, 2, 1, 256, 128, 2, 2>::cfg(),     //  2
    MmaInst<32, 2, 2, 256, 128, 2, 2>::cfg(),     //  3
    MmaInst<32, 2, 1, 256, 128, 2, 3>::cfg(),     //  4
    MmaInst<32, 2, 2, 256, 128, 2, 2, 1>::cfg(),  //  5
    MmaInst<32, 2, 2, 256, 128, 2, 2, 2>::cfg(),  //  6
    MmaInst<32, 2, 1, 256, 128, 2, 2, 1>::cfg(),  //  7
    MmaInst<32, 2, 1, 256, 128, 2, 2, 2>::cfg(),  //  8
    MmaInst<32, 2, 1, 512, 128, 3, 1>::cfg(),     //  9
    MmaInst<32, 2, 2, 512, 128, 2, 1>::cfg(),     // 10
    MmaInst<32, 2, 1, 128, 128, 2, 4>::cfg(),     // 11
    MmaInst<32, 2, 2, 64, 128, 3, 4>::cfg(),      // 12  small
    MmaInst<32, 2, 1, 64, 128, 3, 4>::cfg(),      // 13  small
    MmaInst<32, 2, 4, 64, 128, 3, 2>::cfg(),      // 14  small
    MmaInst<8, 2, 2, 256, 512, 2, 2>::cfg(),      // 15
    MmaInst<8, 2, 4, 256, 512, 2, 2>::cfg(),      // 16
    MmaInst<8, 1, 4, 256, 256, 3, 2>::cfg(),      // 17
    MmaInst<8, 2, 2, 64, 512, 3, 4>::cfg(),       // 18  small
    MmaInst<8, 2, 4, 64, 256, 2, 4>::cfg(),       // 19  small
    MmaInst<16, 2, 2, 256, 128, 3, 2>::cfg(),     // 20
    MmaInst<16, 2, 4, 256, 256, 2, 2>::cfg(),     // 21
    MmaInst<16, 2, 2, 256, 128, 2, 3>::cfg(),     // 22
    MmaInst<16, 2, 2, 64, 256, 3, 4>::cfg(),      // 23  small
    MmaInst<16, 2, 4, 64, 256, 3, 4>::cfg(),      // 24  small
    MmaInst<64, 2, 1, 256, 64, 3, 1>::cfg(),      // 25
    MmaInst<64, 2, 2, 256, 64, 3, 1>::cfg(),      // 26
    MmaInst<64, 2, 1, 256, 64, 2, 2>::cfg(),      // 27
    MmaInst<64, 2, 1, 64, 64, 3, 3>::cfg(),       // 28  small
    MmaInst<64, 2, 2, 64, 64, 3, 3>::cfg(),       // 29  small
    MmaInst<32, 2, 1, 256, 128, 2, 2, 4>::cfg(),  // 30  as 7, without the per-tile exchange of maxima
    MmaInst<16, 2, 2, 256, 256, 2, 2, 5>::cfg(),  // 31  shipped tilings with the near-term counters
    MmaInst<16, 1, 4, 64, 256, 3, 4, 5>::cfg(),   // 32  small
    MmaInst<32, 2, 1, 256, 128, 2, 2, 5>::cfg(),  // 33
    MmaInst<32, 1, 4, 64, 128, 3, 4, 5>::cfg(),   // 34  small
    MmaInst<64, 2, 2, 256, 64, 3, 1, 5>::cfg(),   // 35
    MmaInst<64, 2, 2, 64, 64, 3, 3, 5>::cfg(),    // 36  small
};
constexpr int kMmaLabN = sizeof(kMmaLab) / sizeof(kMmaLab[0]);
#endif  // TPE_LAB

const FastCfg* pick_mma(int pb, int64_t Ct) {
  const bool small = Ct <= 64;
#ifdef TPE_LAB
  if (const char* v = getenv("TPE_MMA_LAB")) {
    const int i = atoi(v);
    if (i >= 0 && i < kMmaLabN && kMmaLab[i].pb == pb) return &kMmaLab[i];
  }
#endif
  const FastCfg* tabs = small ? kMmaSmall : kMmaBig;
  for (int i = 0; i < 4; ++i)
    if (tabs[i].pb == pb) return &tabs[i];
  return nullptr;
}

// "big": many candidates (c-tiles of `cands_per_cta`, kernels split over blockIdx.y);
// "small": a single ask with few candidates -- one warp per CTA, the grid splits the kernel axis.
// CONST = one sigma per column (multivariate TPE), PAIR = sigma per kernel (univariate TPE).
//                 PB PS RC  NT    TK ST  PAIR MINB
// One candidate per lane: the log-sum-exp over kernels needs no cross-lane traffic, where the lane-split
// tilings pay a shuffle on the shared pipe per term; the 2-candidate tiling leaves too few warps per SM to
// hide the DADD->DFMA latency.  (These tilings were chosen on another GPU and not re-tuned for H100.)
const FastCfg kConstBig[] = {
    FastInst<1, 1, 4, 256, 2048, 3, false, 2>::cfg(), FastInst<2, 1, 4, 256, 1024, 3, false, 2>::cfg(),
    FastInst<4, 1, 4, 256, 1024, 3, false, 2>::cfg(), FastInst<8, 1, 4, 256, 512, 3, false, 1>::cfg(),
    FastInst<16, 1, 2, 256, 256, 3, false, 2>::cfg(), FastInst<32, 1, 1, 512, 128, 3, false, 1>::cfg(),
    FastInst<64, 1, 1, 256, 64, 3, false, 1>::cfg(),
};
const FastCfg kPairBig[] = {
    FastInst<1, 1, 4, 256, 1024, 3, true, 2>::cfg(), FastInst<2, 1, 4, 256, 1024, 3, true, 1>::cfg(),
    FastInst<4, 1, 4, 256, 512, 3, true, 1>::cfg(),  FastInst<8, 1, 4, 256, 256, 3, true, 1>::cfg(),
    FastInst<16, 1, 4, 256, 128, 3, true, 1>::cfg(), FastInst<32, 1, 2, 256, 64, 3, true, 1>::cfg(),
    FastInst<64, 1, 1, 256, 32, 3, true, 1>::cfg(),
};
const FastCfg kConstSmall[] = {
    FastInst<1, 1, 1, 32, 1024, 2, false, 1>::cfg(), FastInst<2, 1, 1, 32, 512, 2, false, 1>::cfg(),
    FastInst<4, 1, 1, 32, 256, 2, false, 1>::cfg(),  FastInst<8, 1, 1, 32, 128, 2, false, 1>::cfg(),
    FastInst<16, 1, 1, 32, 64, 2, false, 1>::cfg(),  FastInst<32, 1, 1, 32, 32, 2, false, 1>::cfg(),
    FastInst<64, 1, 1, 32, 16, 2, false, 1>::cfg(),
};
const FastCfg kPairSmall[] = {
    FastInst<1, 1, 1, 32, 512, 2, true, 1>::cfg(), FastInst<2, 1, 1, 32, 256, 2, true, 1>::cfg(),
    FastInst<4, 1, 1, 32, 128, 2, true, 1>::cfg(), FastInst<8, 1, 1, 32, 64, 2, true, 1>::cfg(),
    FastInst<16, 1, 1, 32, 32, 2, true, 1>::cfg(), FastInst<32, 1, 1, 32, 16, 2, true, 1>::cfg(),
    FastInst<64, 1, 1, 32, 8, 2, true, 1>::cfg(),
};
#ifdef TPE_LAB
// tuning variants of the P = 32 CONST kernel, selectable with TPE_FAST_VARIANT=0..3 (experiments)
const FastCfg kConst32Variants[] = {
    FastInst<32, 1, 1, 256, 128, 3, false, 2>::cfg(),  // 0: 1 candidate / lane, 16 warps / SM
    FastInst<32, 1, 2, 256, 128, 3, false, 1>::cfg(),  // 1: 2 candidates / lane, 8 warps / SM
    FastInst<32, 2, 4, 256, 128, 3, false, 1>::cfg(),  // 2: params split over 2 lanes, 4 candidates
    FastInst<32, 4, 4, 256, 128, 3, false, 2>::cfg(),  // 3: params split over 4 lanes, 4 candidates
    FastInst<32, 1, 2, 320, 128, 3, false, 1>::cfg(),  // 4: 2 candidates / lane, 10 warps / SM
    FastInst<32, 1, 2, 384, 128, 3, false, 1>::cfg(),  // 5: 2 candidates / lane, 12 warps / SM
    FastInst<32, 1, 2, 128, 64, 3, false, 2>::cfg(),   // 6: 2 candidates / lane, 2 CTAs x 4 warps
    FastInst<32, 1, 1, 128, 64, 3, false, 4>::cfg(),   // 7: 4 CTAs x 4 warps
    FastInst<32, 1, 1, 256, 128, 2, false, 2>::cfg(),  // 8: 2 stages
    FastInst<32, 1, 1, 512, 128, 3, false, 1>::cfg(),  // 9: 1 CTA x 16 warps
};
#endif  // TPE_LAB
constexpr int kMaxFastP = 64;

int pick_pb(int ncont) {
  for (int pb : {1, 2, 4, 8, 16, 32, 64})
    if (ncont <= pb) return pb;
  return 0;
}
const FastCfg* pick_fast(int mode, int pb, int64_t Ct) {
  const bool small = Ct <= 128;
#ifdef TPE_LAB
  if (mode == 2 && pb == 32 && !small) {
    const char* v = getenv("TPE_FAST_VARIANT");
    if (v && v[0] >= '0' && v[0] <= '9') return &kConst32Variants[v[0] - '0'];
  }
#endif
  const FastCfg* tabs = (mode == 2) ? (small ? kConstSmall : kConstBig) : (small ? kPairSmall : kPairBig);
  for (int i = 0; i < 7; ++i)
    if (tabs[i].pb == pb) return &tabs[i];
  return nullptr;
}

// `count` outputs of the MT19937 stream after dropping `skip`, from the 625-word device state `state` (updated in
// place to the state after the draws).  Short stretches: one CTA walks the recurrence (k_mt19937_uniform).  Long
// ones (a batch of asks, or a rank's slice far into the batch): every CTA jumps to its own chunk
// (k_mt19937_uniform_mc) -- no serial prefix walk.
int launch_mt(tpe_ctx* ctx, cudaStream_t st, uint32_t* state, int64_t skip, int64_t count, double* out) {
  static const int64_t mc_min = [] { const char* v = getenv("TPE_MT_MC_MIN"); return v ? atoll(v) : (int64_t)400000; }();
  if (skip + count < mc_min) {
    k_mt19937_uniform<<<1, kMtThreads, 0, st>>>(state, reinterpret_cast<int*>(state + 624), skip, count, out);
    ctx->launch_counter++;
    CU(cudaGetLastError());
    return TPE_OK;
  }
  if (!ctx->mt_jump_ready) {
    CU(ctx->mt_jump.ensure(sizeof(kMtJumpTable)));
    CU(ctx->mt_tmp.ensure(625 * 4));
    CU(cudaMemcpyAsync(ctx->mt_jump.p, kMtJumpTable, sizeof(kMtJumpTable), cudaMemcpyHostToDevice, st));
    CU(cudaFuncSetAttribute(k_mt19937_uniform_mc, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMtJumpSmem));
    ctx->mt_jump_ready = true;
  }
  const int64_t G = std::max<int64_t>(1, std::min<int64_t>(ctx->sm_count, (count + 16383) / 16384));
  const int64_t chunk = round_up<int64_t>((count + G - 1) / G, 256);
  const int64_t grid = (count + chunk - 1) / chunk;
  k_mt19937_uniform_mc<<<(unsigned)grid, kMtThreads, kMtJumpSmem, st>>>(state, skip, count, chunk, ctx->mt_jump.as<uint32_t>(),
                                                                       kMtJumpKMin, kMtJumpKMax, out,
                                                                       ctx->mt_tmp.as<uint32_t>());
  ctx->launch_counter++;
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(state, ctx->mt_tmp.p, 625 * 4, cudaMemcpyDeviceToDevice, st));
  return TPE_OK;
}

int join_above(tpe_ctx* ctx) {
  if (ctx->above_pending) {
    CU(cudaStreamWaitEvent(ctx->stream, ctx->ev_join, 0));
    ctx->above_pending = false;
  }
  return TPE_OK;
}
int set_device(tpe_ctx* ctx, bool join = true) {
  CU(cudaSetDevice(ctx->device));
  if (join) return join_above(ctx);
  return TPE_OK;
}

// A few rows from the host (the per-trial case) go through a slot of page-locked staging memory, without waiting: a
// copy from pageable memory would first wait for everything queued on the stream, i.e. for a suggestion that was
// queued ahead of time (tpe_sample_and_select_async) and must keep running while the caller goes on.
bool rows_fit_staging(const tpe_ctx* ctx, int64_t n) {
  return (size_t)n * ((size_t)ctx->space.size() * 8 + 16 + 1) + 64 <= tpe_ctx::kUpSlot;
}
int stage_rows(tpe_ctx* ctx, const double* X, const int8_t* category, const double* key, int64_t n, int64_t at) {
  const int64_t P = (int64_t)ctx->space.size();
  if (!ctx->up_host) {
    CU(cudaHostAlloc(&ctx->up_host, tpe_ctx::kUpSlot * tpe_ctx::kUpSlots, cudaHostAllocDefault));
    for (auto& e : ctx->up_ev) CU(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  }
  const int slot = ctx->up_next;
  ctx->up_next = (slot + 1) % tpe_ctx::kUpSlots;
  if (ctx->up_used[slot]) CU(cudaEventSynchronize(ctx->up_ev[slot]));   // (its copies of kUpSlots uploads ago)
  char* h = static_cast<char*>(ctx->up_host) + (size_t)slot * tpe_ctx::kUpSlot;
  const size_t xb = (size_t)n * P * 8, kb = (size_t)n * 16;
  memcpy(h, X, xb);
  memcpy(h + xb, key, kb);
  memcpy(h + xb + kb, category, (size_t)n);
  CU(cudaMemcpyAsync(ctx->X.as<double>() + at * P, h, xb, cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaMemcpyAsync(ctx->key.as<double>() + at * 2, h + xb, kb, cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaMemcpyAsync(ctx->cat.as<int8_t>() + at, h + xb + kb, (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaEventRecord(ctx->up_ev[slot], ctx->stream));
  ctx->up_used[slot] = true;
  return TPE_OK;
}

int upload_history(tpe_ctx* ctx, const double* X, const int8_t* category, const double* key, int64_t n,
                   int64_t at, bool device_src) {
  const int64_t P = (int64_t)ctx->space.size();
  const int64_t total = at + n;
  CU(ctx->X.grow((size_t)std::max<int64_t>(total, 1) * P * 8, (size_t)at * P * 8, ctx->stream));
  CU(ctx->cat.grow((size_t)std::max<int64_t>(total, 1), (size_t)at, ctx->stream));
  CU(ctx->key.grow((size_t)std::max<int64_t>(total, 1) * 16, (size_t)at * 16, ctx->stream));
  const cudaMemcpyKind kind = device_src ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
  if (n > 0 && !device_src && rows_fit_staging(ctx, n)) {
    if (int rc = stage_rows(ctx, X, category, key, n, at)) return rc;
  } else if (n > 0) {
    CU(cudaMemcpyAsync(ctx->X.as<double>() + at * P, X, (size_t)n * P * 8, kind, ctx->stream));
    CU(cudaMemcpyAsync(ctx->cat.as<int8_t>() + at, category, (size_t)n, kind, ctx->stream));
    CU(cudaMemcpyAsync(ctx->key.as<double>() + at * 2, key, (size_t)n * 16, kind, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
  }
  ctx->cat_h.resize((size_t)total);
  if (n > 0) {
    if (device_src) CU(cudaMemcpy(ctx->cat_h.data() + at, category, (size_t)n, cudaMemcpyDeviceToHost));
    else memcpy(ctx->cat_h.data() + at, category, (size_t)n);
  }
  if (at == 0) ctx->cat_cnt[0] = ctx->cat_cnt[1] = ctx->cat_cnt[2] = ctx->cat_cnt[3] = ctx->cat_cnt[4] = 0;
  for (int64_t i = at; i < total; ++i) ctx->cat_cnt[cat_slot(ctx->cat_h[(size_t)i])]++;
  if (at == 0) ctx->M = 1;  // a fresh history is single-objective until values are supplied
  ctx->N = total;
  ctx->history_set = true;
  ctx->prepared = ctx->built = ctx->sampled = false;
  ctx->hist_version++;
  return TPE_OK;
}

// ---- MOTPE: selection of the below part of the COMPLETE group (sampler.py:745-779) ----------------
// Fills ctx->member (u8 per history row) and returns how many COMPLETE trials went below.
// Per-thread scratch (doubles, odd so that the threads spread over the banks) of an M <= 3
// hypervolume of up to n points held in shared memory: caller's point list + hypervolume()'s copy,
// tmp row and order / mask words.  0 = does not fit (or M > 3, where hv_nd needs the O(n^2) arena).
int mo_smem_stride(int n, int M) {
  if (M > 3) return 0;
  const int stride = (2 * n * M + M + n + 9) | 1;
  return ((size_t)kMoMaxSet * stride * 8 <= 160 * 1024) ? stride : 0;
}

int mo_select_complete(tpe_ctx* ctx, int64_t n_below, int64_t* taken) {
  cudaStream_t st = ctx->stream;
  const int M = ctx->M;
  const int64_t N = ctx->N;
  std::vector<int64_t> list;
  for (int64_t i = 0; i < N; ++i)
    if (ctx->cat_h[i] == TPE_CAT_COMPLETE) list.push_back(i);
  const int nc = (int)list.size();
  const int64_t m = std::min<int64_t>(std::max<int64_t>(n_below, 0), nc);
  *taken = m;
  CU(ctx->member.ensure((size_t)std::max<int64_t>(N, 1)));
  CU(cudaMemsetAsync(ctx->member.p, 0, (size_t)std::max<int64_t>(N, 1), st));
  if (m == 0) return TPE_OK;
  if (m == nc) {
    std::vector<uint8_t> mem((size_t)N, 0);
    for (int64_t r : list) mem[(size_t)r] = 1;
    CU(cudaMemcpyAsync(ctx->member.p, mem.data(), (size_t)N, cudaMemcpyHostToDevice, st));
    CU(cudaStreamSynchronize(st));
    return TPE_OK;
  }
  CU(ctx->mo_list.ensure((size_t)nc * 8));
  CU(cudaMemcpyAsync(ctx->mo_list.p, list.data(), (size_t)nc * 8, cudaMemcpyHostToDevice, st));
  for (DevBuf* b : {&ctx->mo_alive, &ctx->mo_dom, &ctx->mo_first, &ctx->mo_isdup, &ctx->mo_removed})
    CU(b->ensure((size_t)nc));
  for (DevBuf* b : {&ctx->mo_rank, &ctx->mo_tie, &ctx->mo_lexpos, &ctx->mo_sorted, &ctx->mo_uniq, &ctx->mo_chosen})
    CU(b->ensure((size_t)nc * 4));
  CU(ctx->mo_ctr.ensure(sizeof(MoCounters)));
  CU(ctx->mo_ntie.ensure(16));
  CU(ctx->mo_nuniq.ensure(16));
  CU(ctx->mo_ref.ensure(kMoMaxM * 8));
  CU(ctx->mo_contrib.ensure((size_t)nc * 8));
  CU(ctx->mo_diag.ensure((size_t)nc * 16));
  CU(ctx->mo_sample.ensure(256 * 4));
  CU(ctx->mo_surv.ensure((size_t)nc * 4));
  CU(ctx->mo_nsurv.ensure(16));
  CU(cudaMemsetAsync(ctx->mo_alive.p, 1, (size_t)nc, st));
  CU(cudaMemsetAsync(ctx->mo_rank.p, 0, (size_t)nc * 4, st));
  CU(cudaMemsetAsync(ctx->mo_ctr.p, 0, sizeof(MoCounters), st));
  const double* vals = ctx->vals.as<double>();
  const int64_t* dlist = ctx->mo_list.as<int64_t>();
  const int gb = (nc + 255) / 256;
  // peel Pareto fronts until n_below unique vectors are ranked
  std::vector<int64_t> rank_count;
  MoCounters ctr{};
  int r = 0;
  int64_t prev_all = 0;
  for (;;) {
    if (r == 0) {  // duplicates of the whole complete set, once
      uint32_t tsize = 1024;
      while (tsize < 2u * (uint32_t)nc) tsize <<= 1;
      CU(ctx->mo_table.ensure((size_t)tsize * 4));
      CU(cudaMemsetAsync(ctx->mo_table.p, 0x7f, (size_t)tsize * 4, st));
      k_mo_first_insert<<<gb, 256, 0, st>>>(vals, M, dlist, nc, ctx->mo_table.as<int>(), tsize - 1);
      k_mo_first_lookup<<<gb, 256, 0, st>>>(vals, M, dlist, nc, ctx->mo_table.as<int>(), tsize - 1,
                                            ctx->mo_first.as<uint8_t>(), ctx->mo_ctr.as<MoCounters>());
      ctx->launch_counter += 2;
    }
    k_mo_sample<<<1, 1024, 0, st>>>(nc, ctx->mo_alive.as<uint8_t>(), ctx->mo_sample.as<int32_t>(),
                                    ctx->mo_nsurv.as<int>(), ctx->mo_nsurv.as<int>() + 1);
    k_mo_peel_a<<<gb, 256, 256 * M * 8, st>>>(vals, M, dlist, nc, ctx->mo_alive.as<uint8_t>(),
                                               ctx->mo_sample.as<int32_t>(), ctx->mo_nsurv.as<int>(),
                                               ctx->mo_dom.as<uint8_t>(), ctx->mo_surv.as<int32_t>(),
                                               ctx->mo_nsurv.as<int>() + 1);
    k_mo_peel_b<<<std::min(nc, ctx->sm_count * 8), 256, 0, st>>>(vals, M, dlist, nc, ctx->mo_alive.as<uint8_t>(),
                                                                  ctx->mo_surv.as<int32_t>(), ctx->mo_nsurv.as<int>() + 1,
                                                                  ctx->mo_dom.as<uint8_t>());
    ctx->launch_counter += 1;
    k_mo_commit<<<gb, 256, 0, st>>>(nc, ctx->mo_alive.as<uint8_t>(), ctx->mo_dom.as<uint8_t>(),
                                     ctx->mo_first.as<uint8_t>(), ctx->mo_rank.as<int32_t>(), r,
                                     ctx->mo_ctr.as<MoCounters>());
    ctx->launch_counter += 2;
    CU(cudaMemcpyAsync(&ctr, ctx->mo_ctr.p, sizeof(ctr), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    rank_count.push_back(ctr.covered_all - prev_all);
    prev_all = ctr.covered_all;
    ++r;
    const int64_t goal = std::min<int64_t>(m, ctr.n_unique);
    if (ctr.covered_unique >= goal || ctr.covered_all >= nc) break;
    if (rank_count.back() == 0) return fail(ctx, TPE_E_INVALID, "MOTPE rank peeling made no progress (NaN objective values?)");
  }
  if (ctr.covered_all < nc) {
    k_mo_fill_rank<<<gb, 256, 0, st>>>(nc, ctx->mo_alive.as<uint8_t>(), ctx->mo_rank.as<int32_t>(), r);
    ctx->launch_counter++;
    rank_count.push_back(nc - ctr.covered_all);
  }
  // whole ranks that fit
  int64_t cum = 0;
  int last = -1;
  for (size_t q = 0; q < rank_count.size(); ++q) {
    if (cum + rank_count[q] > m) break;
    cum += rank_count[q];
    last = (int)q;
  }
  k_mo_gather_rank<<<1, 1024, 0, st>>>(nc, ctx->mo_rank.as<int32_t>(), last, dlist, ctx->member.as<uint8_t>(),
                                       ctx->mo_tie.as<int32_t>(), ctx->mo_ntie.as<int>());
  ctx->launch_counter++;
  const int subset = (int)(m - cum);
  if (subset > 0) {
    int n_tie = 0;
    CU(cudaMemcpyAsync(&n_tie, ctx->mo_ntie.p, 4, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    k_mo_refpoint<<<1, 256, 0, st>>>(vals, M, dlist, ctx->mo_tie.as<int32_t>(), n_tie, ctx->mo_ref.as<double>());
    double ref[kMoMaxM];
    CU(cudaMemcpyAsync(ref, ctx->mo_ref.p, (size_t)M * 8, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    ctx->launch_counter += 1;
    bool finite = true;
    for (int j = 0; j < M; ++j) finite = finite && std::isfinite(ref[j]);
    const int n_chosen = subset;
    {
      k_mo_lexrank<<<(n_tie + 127) / 128, 128, 0, st>>>(vals, M, dlist, ctx->mo_tie.as<int32_t>(), n_tie,
                                                         ctx->mo_lexpos.as<int32_t>(), ctx->mo_isdup.as<uint8_t>());
      k_mo_unique<<<1, 1024, 0, st>>>(n_tie, ctx->mo_lexpos.as<int32_t>(), ctx->mo_isdup.as<uint8_t>(),
                                      ctx->mo_sorted.as<int32_t>(), ctx->mo_uniq.as<int32_t>(), ctx->mo_nuniq.as<int>());
      ctx->launch_counter += 2;
      int nu = 0;
      CU(cudaMemcpyAsync(&nu, ctx->mo_nuniq.p, 4, cudaMemcpyDeviceToHost, st));
      CU(cudaStreamSynchronize(st));
      if (nu <= subset) {
        // every unique vector, then the first duplicates in trial order (hssp.py:162-171)
        CU(cudaMemcpyAsync(ctx->mo_chosen.p, ctx->mo_uniq.p, (size_t)nu * 4, cudaMemcpyDeviceToDevice, st));
        if (nu < subset) {
          k_mo_fill_dups<<<1, 1024, 0, st>>>(n_tie, ctx->mo_isdup.as<uint8_t>(), subset - nu,
                                             ctx->mo_chosen.as<int32_t>(), nu);
          ctx->launch_counter++;
        }
      } else if (!finite) {
        // the first `subset` unique vectors in lexicographic order (hssp.py:106-107 sees np.unique's output)
        CU(cudaMemcpyAsync(ctx->mo_chosen.p, ctx->mo_uniq.p, (size_t)subset * 4, cudaMemcpyDeviceToDevice, st));
      } else {
        CU(ctx->mo_state.ensure(hssp_bytes(subset, M)));
        CU(cudaMemsetAsync(ctx->mo_state.p, 0, hssp_bytes(subset, M), st));
        {
          HsspState head{0.0, 0, subset};
          CU(cudaMemcpyAsync(ctx->mo_state.p, &head, sizeof(head), cudaMemcpyHostToDevice, st));
          CU(cudaStreamSynchronize(st));  // `head` is a stack object
        }
        CU(cudaMemsetAsync(ctx->mo_removed.p, 0, (size_t)nc, st));
        if (M == 2) {
          k_hssp_2d<<<1, 256, 0, st>>>(vals, dlist, ctx->mo_tie.as<int32_t>(), ctx->mo_uniq.as<int32_t>(), nu, subset,
                                       ctx->mo_ref.as<double>(), ctx->mo_diag.as<double>(),
                                       ctx->mo_removed.as<uint8_t>(), ctx->mo_state.as<HsspState>());
          ctx->launch_counter++;
        } else {
          const size_t stride = (size_t)(subset + 2) * M + hv_arena_doubles(subset + 1, M);
          const int sstride = mo_smem_stride(subset + 1, M);
          const int cthreads = sstride ? 32 : 64;
          const size_t csmem = sstride ? (size_t)cthreads * sstride * 8 : 0;
          // more than three objectives: one warp per candidate, a private WFG arena per lane (global memory);
          // falls back to one thread per candidate when that would need more than 8 GB
          const size_t nd_lane_stride = hv_lane_doubles(subset, M);
          const size_t nd_warp_stride = hv_warp_scratch_doubles(subset, M) + 32 * nd_lane_stride;
          const bool nd_warp = M > 3 && (size_t)nu * nd_warp_stride * 8 <= ((size_t)8 << 30);
          const size_t stride3 = (size_t)(subset + 1) * 8 + 16;  // hv3_warp scratch per candidate beyond the shared-memory size
          const bool big3 = M == 3 && subset + 1 > kMoMaxSet + 1;
          if (!nd_warp && M > 3 && (size_t)nu * stride * 8 > ((size_t)32 << 30))
            return fail(ctx, TPE_E_NOMEM, "MOTPE subset selection: %d candidates x %d picks in %d objectives need %zu GB of "
                        "hypervolume scratch", nu, subset, M, ((size_t)nu * stride * 8) >> 30);
          CU(ctx->mo_bound.ensure((size_t)nu * 16));   // lazy bounds + k_hssp_pick's scratch
          if (nd_warp) CU(ctx->mo_arena.ensure((size_t)nu * nd_warp_stride * 8));
          else if (big3) CU(ctx->mo_arena.ensure((size_t)nu * stride3 * 8));
          else if (!sstride && M != 3) CU(ctx->mo_arena.ensure((size_t)nu * stride * 8));
          if (csmem > 48 * 1024)
            CU(cudaFuncSetAttribute(k_hssp_contrib, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)csmem));
          for (int t = 0; t < subset; ++t) {
            if (M == 3) {
              k_hssp_contrib3<<<(nu + 3) / 4, 128, 0, st>>>(vals, dlist, ctx->mo_tie.as<int32_t>(),
                                                            ctx->mo_uniq.as<int32_t>(), nu,
                                                            ctx->mo_removed.as<uint8_t>(), ctx->mo_ref.as<double>(),
                                                            ctx->mo_state.as<HsspState>(), ctx->mo_contrib.as<double>(),
                                                            ctx->mo_bound.as<double>(), ctx->mo_arena.as<double>(), stride3);
            } else if (nd_warp) {
              k_hssp_contrib_nd<<<(nu + 3) / 4, 128, 0, st>>>(
                  vals, M, dlist, ctx->mo_tie.as<int32_t>(), ctx->mo_uniq.as<int32_t>(), nu,
                  ctx->mo_removed.as<uint8_t>(), ctx->mo_ref.as<double>(), ctx->mo_state.as<HsspState>(),
                  ctx->mo_contrib.as<double>(), ctx->mo_bound.as<double>(), ctx->mo_arena.as<double>(), nd_warp_stride,
                  nd_lane_stride);
            } else {
              k_hssp_contrib<<<(nu + cthreads - 1) / cthreads, cthreads, csmem, st>>>(
                  vals, M, dlist, ctx->mo_tie.as<int32_t>(), ctx->mo_uniq.as<int32_t>(), nu,
                  ctx->mo_removed.as<uint8_t>(), ctx->mo_ref.as<double>(), ctx->mo_state.as<HsspState>(),
                  ctx->mo_contrib.as<double>(), ctx->mo_bound.as<double>(), ctx->mo_arena.as<double>(), stride, sstride);
            }
            k_hssp_pick<<<1, 256, 0, st>>>(vals, M, dlist, ctx->mo_tie.as<int32_t>(), ctx->mo_uniq.as<int32_t>(), nu,
                                           ctx->mo_removed.as<uint8_t>(), ctx->mo_contrib.as<double>(),
                                           ctx->mo_bound.as<double>(), ctx->mo_state.as<HsspState>());
            ctx->launch_counter += 2;
          }
        }
        CU(cudaMemcpyAsync(ctx->mo_chosen.p, (char*)ctx->mo_state.p + sizeof(HsspState) + (size_t)subset * M * 8,
                           (size_t)subset * 4, cudaMemcpyDeviceToDevice, st));
      }
    }
    k_mo_mark<<<(n_chosen + 127) / 128, 128, 0, st>>>(dlist, ctx->mo_tie.as<int32_t>(), ctx->mo_chosen.as<int32_t>(),
                                                      n_chosen, ctx->member.as<uint8_t>());
    ctx->launch_counter++;
    CU(cudaStreamSynchronize(st));
  }
  CU(cudaGetLastError());
  return TPE_OK;
}

// Host scan of uploaded rows: which columns have absent values (the split then needs the row filter) and which
// hold observations outside the column's current [low, high] (legal: optuna lets a range change between trials;
// the a-priori rounding bound of the tensor-core grid kernel assumes |mu''| <= range / (2 sigma), so such columns
// take the elementwise kernel).  TPE_CAT_EXCLUDED placeholders are in no estimator and do not count.
void scan_missing(tpe_ctx* ctx, const double* X, const int8_t* category, int64_t n) {
  const int64_t P = (int64_t)ctx->space.size();
  for (int64_t i = 0; i < n; ++i) {
    if (category && cat_slot(category[i]) == 4) continue;
    for (int64_t j = 0; j < P; ++j) {
      const double v = X[i * P + j];
      if (v != v) { ctx->col_missing[j] = 1; continue; }
      const tpe_param_desc& d = ctx->space[j];
      if (d.kind != TPE_KIND_CAT && (v < d.low || v > d.high)) ctx->col_oor[j] = 1;
      if (d.kind != TPE_KIND_CAT && d.has_step) {   // the test k_build_mv applies to tabulated columns
        const double gsz = floor((d.high - d.low) / d.step + 0.5) + 1.0;
        const double g = rint((v - d.low) / d.step);
        if (!(g >= 0.0 && g < gsz && d.low + g * d.step == v)) ctx->col_offgrid[j] = 1;
      }
    }
  }
}

bool mma_enabled() {
  static const bool on = [] { const char* v = getenv("TPE_MMA"); return !(v && v[0] == '0'); }();
  return on;
}

int build_estimator(tpe_ctx* ctx, int which, const double* w_host, cudaStream_t st) {
  Estimator& e = ctx->est[which];
  e.screen_ready = false;
  const int64_t n = e.n, K = n + 1;
  const int32_t pc = ctx->pc;
  const int cap = ctx->sm_count * 8;
  e.K = K;
  const int64_t k_alloc = round_up<int64_t>(K + 32, 32);  // >= round_up(K - 1, kMmaKPad), bulk-copy padding
  CU(e.mu.ensure((size_t)K * pc * 8));
  CU(e.sigma.ensure((size_t)K * pc * 8));
  CU(e.cst_part.ensure((size_t)K * 8));
  CU(e.cst.ensure((size_t)(k_alloc + kTcsTile) * 8));   // (+ one tile: k_tcs copies whole tiles)
  CU(e.w.ensure((size_t)K * 8));
  CU(e.logw.ensure((size_t)K * 8));
  CU(e.cdf.ensure((size_t)K * 8));
  if (ctx->fast_mode == 1) CU(e.tabp.ensure((size_t)K * ctx->pb * 16 + 16));
  if (ctx->fast_mode == 2) CU(e.tabc.ensure((size_t)(K + kTcsTile) * ctx->pb * 8 + 16));
  if (ctx->fast) CU(e.colprm.ensure((size_t)ctx->pb * 16));
  bool in_range = true;  // every selected column's observations lie inside its current [low, high]
  for (const ColMeta& cm : ctx->cols_h) in_range = in_range && !ctx->col_oor[cm.src];
  e.mma = ctx->fast_mode == 2 && ctx->pb >= 8 && in_range && mma_enabled();
  if (e.mma) {
    CU(e.tabm.ensure((size_t)k_alloc * ctx->pb * 8));
    CU(e.hb.ensure((size_t)k_alloc * 8));
    CU(e.ckk.ensure((size_t)k_alloc * 8));
    CU(cudaMemsetAsync(e.tabm.p, 0, (size_t)k_alloc * ctx->pb * 8, st));  // padded slots, last group, prior row
  }
  if (ctx->tab_doubles) CU(e.tab.ensure((size_t)ctx->tab_doubles * 8));
  if (ctx->dtab_doubles) {
    CU(e.dtab.ensure((size_t)ctx->dtab_doubles * 8));
    CU(e.cls.ensure((size_t)K * pc * 4));
    CU(e.offgrid.ensure(16));
    CU(cudaMemsetAsync(e.offgrid.p, 0, 16, st));
  }

  if (ctx->fast && ctx->pb > ctx->ncont) {
    k_tab_pad<<<grid_for(K * (ctx->pb - ctx->ncont), 256, cap), 256, 0, st>>>(
        ctx->fast_mode == 1 ? e.tabp.as<double2>() : nullptr, ctx->fast_mode == 2 ? e.tabc.as<double>() : nullptr,
        e.colprm.as<double2>(), ctx->fast_mode == 2 ? K - 1 : K, ctx->pb, ctx->ncont);
    ctx->launch_counter++;
  }
  if (ctx->cfg.multivariate) {
    k_build_mv<<<grid_for(K * 32, 256, cap), 256, 0, st>>>(
        ctx->X.as<double>(), (int32_t)ctx->space.size(), e.rows.as<int64_t>(), n, ctx->cols.as<ColMeta>(), pc,
        ctx->cfg.magic_clip, ctx->pb, ctx->fast_mode, e.mu.as<double>(), e.sigma.as<double>(), e.tabp.as<double2>(),
        e.tabc.as<double>(), e.colprm.as<double2>(), e.cst_part.as<double>(),
        ctx->dtab_doubles ? e.cls.as<int32_t>() : nullptr, ctx->dtab_doubles ? e.offgrid.as<int>() : nullptr,
        e.mma ? e.tabm.as<double>() : nullptr, e.mma ? e.hb.as<double>() : nullptr);
    ctx->launch_counter++;
    e.mixed = ctx->mixed_ok && K - 1 >= 2048;
    if (e.mixed) {
      const int ncp = (ctx->mix_ncont + 1) / 2, nd4 = (ctx->mix_nd + 3) / 4;
      e.mix_kstride = round_up<int64_t>(K - 1, 32);
      CU(e.mxc.ensure((size_t)std::max(ncp, 1) * e.mix_kstride * 16));
      CU(e.mxd.ensure((size_t)std::max(nd4, 1) * e.mix_kstride * 8));
      k_mixed_tables<<<grid_for(e.mix_kstride, 256, 1 << 20), 256, 0, st>>>(
          ctx->mixcols.as<MixCol>(), ctx->mix_ncont, ctx->mix_nd, ctx->cols.as<ColMeta>(), pc, e.mu.as<double>(),
          e.sigma.as<double>(), ctx->dtab_doubles ? e.cls.as<int32_t>() : nullptr, K - 1, e.mix_kstride,
          e.mxc.as<double2>(), e.mxd.as<ushort4>());
      ctx->launch_counter++;
    }
  } else {
    k_mu<<<grid_for(K * pc, 256, cap), 256, 0, st>>>(ctx->X.as<double>(), (int32_t)ctx->space.size(),
                                                     e.rows.as<int64_t>(), n, ctx->cols.as<ColMeta>(), pc,
                                                     e.mu.as<double>());
    ctx->launch_counter++;
    // categorical columns: sigma unused; numeric columns: sort-based neighbour gaps
    CU(cudaMemsetAsync(e.sigma.p, 0, (size_t)K * pc * 8, st));
    int64_t m2 = 1;
    while (m2 < K) m2 <<= 1;
    CU(ctx->sort_idx.ensure((size_t)std::max<int64_t>(m2, K * 3) * 4));
    for (int j = 0; j < pc; ++j) {
      if (ctx->cols_h[j].cls == COL_CAT) continue;
      if (m2 <= 4096) {
        k_sort_small<<<1, 1024, 0, st>>>(e.mu.as<double>(), pc, j, (int)K, (int)m2, ctx->sort_idx.as<int32_t>());
        ctx->launch_counter++;
      } else {
        // cooperative stable radix sort (one launch instead of ~150 bitonic steps)
        CU(ctx->sort_val.ensure((size_t)K * 8 * 2));
        CU(ctx->sort_idx.ensure((size_t)K * 4 * 3));
        CU(ctx->sort_work.ensure(sizeof(SortWork)));
        const double* d_mu = e.mu.as<double>();
        int32_t pc_i = pc;
        int j_i = j, n_i = (int)K;
        uint64_t* ka = ctx->sort_val.as<uint64_t>();
        uint64_t* kb = ka + K;
        int32_t* order = ctx->sort_idx.as<int32_t>();
        int32_t* ia = order + K;
        int32_t* ib = ia + K;
        SortWork* wk = ctx->sort_work.as<SortWork>();
        // column contexts of a univariate batch: the previous trial's order, if it belongs to this column of this
        // history and the set has the same size or one observation more, is updated instead (the sort then returns
        // at once unless the parent found the rows changed otherwise)
        const int* run_flag = nullptr;
        if (which == 1 && ctx->uni_fast && ctx->uni_mode_ptr != nullptr && ctx->uni_ord_seq + 1 == ctx->uni_seq &&
            ctx->uni_ord_lineage == ctx->hist_lineage &&
            ctx->uni_ord_col == ctx->cols_h[0].src && (ctx->uni_ord_K == K || ctx->uni_ord_K == K - 1) &&
            e.uord.cap >= (size_t)ctx->uni_ord_K * 4) {
          run_flag = ctx->uni_mode_ptr;
          CU(ctx->uni_work.ensure(16));
          CU(cudaMemsetAsync(ctx->uni_work.p, 0, 16, st));
          k_order_update<<<grid_for(ctx->uni_ord_K, 256, ctx->sm_count), 256, 0, st>>>(
              run_flag, e.uord.as<int32_t>(), (int)ctx->uni_ord_K, (int)K, e.mu.as<double>(), order, ctx->uni_work.as<int>());
          ctx->launch_counter++;
        }
        void* args[] = {&d_mu, &pc_i, &j_i, &n_i, &ka, &kb, &ia, &ib, &wk, &order, &run_flag};
        int G = (int)std::max<int64_t>(1, std::min<int64_t>(std::min(ctx->sm_count, 160), (K + 1023) / 1024));
        if (ctx->sort_cta_cap > 0) G = std::min(G, ctx->sort_cta_cap);
        CU(cudaLaunchCooperativeKernel((const void*)k_radix_sort_coop, dim3(G), dim3(512), args, 0, st));
        ctx->launch_counter++;
      }
      k_sigma_uni<<<grid_for(K, 256, cap), 256, 0, st>>>(e.mu.as<double>(), ctx->sort_idx.as<int32_t>(),
                                                         ctx->cols.as<ColMeta>(), pc, j, n, ctx->cfg.magic_clip,
                                                         ctx->cfg.endpoints, e.sigma.as<double>());
      ctx->launch_counter++;
      if (ctx->uni_fast) {   // the 1-D grid walks the kernels in this order
        CU(e.uord.ensure((size_t)(K + 1024) * 4));   // room to grow without a reallocation (the old order is read above)
        CU(cudaMemcpyAsync(e.uord.p, ctx->sort_idx.p, (size_t)K * 4, cudaMemcpyDeviceToDevice, st));
        if (which == 1) {
          ctx->uni_ord_seq = ctx->uni_seq;
          ctx->uni_ord_lineage = ctx->hist_lineage;
          ctx->uni_ord_col = ctx->cols_h[0].src;
          ctx->uni_ord_K = K;
        }
      }
    }
    k_const<<<grid_for(K * 32, 256, cap), 256, 0, st>>>(e.mu.as<double>(), e.sigma.as<double>(),
                                                        ctx->cols.as<ColMeta>(), pc, K, ctx->pb, ctx->fast_mode,
                                                        e.tabp.as<double2>(), e.tabc.as<double>(),
                                                        e.colprm.as<double2>(), e.cst_part.as<double>());
    ctx->launch_counter++;
  }
  const double* w_dev = nullptr;
  const int64_t* w_pos = nullptr;
  if (w_host != nullptr && n > 0) {
    CU(e.wstage.ensure((size_t)n * 8));
    CU(cudaMemcpyAsync(e.wstage.p, w_host, (size_t)n * 8, cudaMemcpyHostToDevice, st));
    w_dev = e.wstage.as<double>();
  } else if (which == 0 && ctx->M >= 2 && n > 0) {
    // MOTPE: hypervolume weights of ALL below trials, then the rows holding every selected param
    // pick theirs through `pos` (weights_below[param_mask_below], sampler.py:570-576)
    const int nba = (int)ctx->info.n_below_all;
    const int M = ctx->M;
    const int64_t* brows = ctx->below_all.as<int64_t>();   // every below trial, trial order (k_split_coop)
    CU(ctx->mo_w.ensure((size_t)std::max(nba, 1) * 8));
    if (nba <= kMoMaxSet) {
      // small below set (the default gamma caps it at 25): one CTA, everything staged in shared memory
      const size_t stride = (size_t)(nba + 2) * M + hv_arena_doubles(nba + 1, M);
      const int sstride = mo_smem_stride(nba + 1, M);
      const size_t wsmem = sstride ? (size_t)kMoMaxSet * sstride * 8 : 0;
      if (!sstride) CU(ctx->mo_arena.ensure((size_t)(nba + 1) * stride * 8));
      if (wsmem > 32 * 1024)
        CU(cudaFuncSetAttribute(k_mo_weights, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)wsmem));
      if (M == 3) {
        static const size_t w3smem = (size_t)32 * kHv3Scratch * 8;
        CU(cudaFuncSetAttribute(k_mo_weights3, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)w3smem));
        k_mo_weights3<<<1, 1024, w3smem, st>>>(ctx->vals.as<double>(), brows, nba, ctx->cat.as<int8_t>(),
                                               ctx->mo_w.as<double>());
      } else if (M > 3) {
        const size_t lane_stride = hv_lane_doubles(nba + 1, M);
        const size_t warp_stride = hv_warp_scratch_doubles(nba + 1, M) + 32 * lane_stride;
        CU(ctx->mo_arena.ensure((size_t)32 * warp_stride * 8));
        k_mo_weights_nd<<<1, 1024, 0, st>>>(ctx->vals.as<double>(), M, brows, nba, ctx->cat.as<int8_t>(),
                                            ctx->mo_w.as<double>(), ctx->mo_arena.as<double>(), warp_stride, lane_stride);
      } else {
        k_mo_weights<<<1, kMoMaxSet, wsmem, st>>>(ctx->vals.as<double>(), M, brows, nba, ctx->cat.as<int8_t>(),
                                                  ctx->mo_w.as<double>(), ctx->mo_arena.as<double>(), stride, sstride);
      }
    } else {
      // any size: global-memory kernels; the exact hypervolumes run over the Pareto front of the below set only
      CU(ctx->mo_fv.ensure((size_t)nba * M * 8));
      CU(ctx->mo_ps.ensure((size_t)nba * M * 8));
      CU(ctx->mo_map.ensure((size_t)nba * 4));
      CU(ctx->mo_front.ensure((size_t)nba * 4));
      CU(ctx->mo_contrib.ensure((size_t)nba * 8));
      CU(ctx->mo_head.ensure(sizeof(MowHead)));
      k_mow_prep<<<1, 1024, 0, st>>>(ctx->vals.as<double>(), M, brows, nba, ctx->cat.as<int8_t>(), ctx->mo_w.as<double>(),
                                     ctx->mo_fv.as<double>(), ctx->mo_map.as<int32_t>(), ctx->mo_ps.as<double>(),
                                     ctx->mo_front.as<int32_t>(), ctx->mo_contrib.as<double>(), ctx->mo_head.as<MowHead>());
      MowHead head{};
      CU(cudaMemcpyAsync(&head, ctx->mo_head.p, sizeof(head), cudaMemcpyDeviceToHost, st));
      CU(cudaStreamSynchronize(st));
      ctx->launch_counter++;
      const int np = head.np;
      if (head.nf > 1 && np > 0) {
        size_t lane_stride = 0, warp_stride;
        if (M > 3) {
          lane_stride = hv_lane_doubles(np, M);
          warp_stride = (size_t)np * M + hv_warp_scratch_doubles(np, M) + 32 * lane_stride;
        } else {
          warp_stride = (size_t)np * M + hv_arena_doubles(np, M) + (size_t)np * 8 + 64;
        }
        const size_t budget = (size_t)16 << 30;
        int64_t warps = std::min<int64_t>(np, (int64_t)ctx->sm_count * 16);
        warps = std::min<int64_t>(warps, (int64_t)(budget / (warp_stride * 8)));
        if (warps < 1)
          return fail(ctx, TPE_E_NOMEM, "MOTPE weights: a Pareto front of %d points in %d objectives needs %zu GB of exact-"
                      "hypervolume scratch per warp", np, M, (warp_stride * 8) >> 30);
        const int blocks = (int)((warps + 3) / 4);
        CU(ctx->mo_arena.ensure((size_t)blocks * 4 * warp_stride * 8));
        k_mow_hv<<<1, 128, 0, st>>>(ctx->mo_ps.as<double>(), ctx->mo_front.as<int32_t>(), M, ctx->mo_head.as<MowHead>(), np,
                                    np, ctx->mo_contrib.as<double>(), ctx->mo_arena.as<double>(), warp_stride, lane_stride);
        k_mow_hv<<<blocks, 128, 0, st>>>(ctx->mo_ps.as<double>(), ctx->mo_front.as<int32_t>(), M,
                                         ctx->mo_head.as<MowHead>(), 0, np - 1, ctx->mo_contrib.as<double>(),
                                         ctx->mo_arena.as<double>(), warp_stride, lane_stride);
        k_mow_norm<<<1, 1024, 0, st>>>(ctx->mo_head.as<MowHead>(), ctx->mo_contrib.as<double>(), ctx->mo_map.as<int32_t>(),
                                       ctx->mo_w.as<double>());
        ctx->launch_counter += 3;
      }
    }
    w_pos = e.pos.as<int64_t>();   // an observation row picks the weight of its position among ALL below trials
                                   // (weights_below[param_mask_below], sampler.py:570-576)
    ctx->launch_counter++;
    ctx->mo_weights_ready = true;
    w_dev = ctx->mo_w.as<double>();
  }
  {
    const int nparts = grid_for(K, 2048, ctx->sm_count * 2);
    if (nparts == 1) {
      k_weights_one<<<1, 256, 0, st>>>(w_dev, w_pos, n, ctx->cfg.prior_weight, e.w.as<double>(), e.logw.as<double>(),
                                       e.cst_part.as<double>(), e.cst.as<double>(),
                                       which == 0 ? e.cdf.as<double>() : nullptr, k_alloc,
                                       e.mma ? e.hb.as<double>() : nullptr, e.mma ? e.ckk.as<double>() : nullptr);
      ctx->launch_counter += 1;
    } else {
      CU(e.wpart.ensure((size_t)nparts * 8));
      k_wraw<<<nparts, 256, 0, st>>>(w_dev, w_pos, n, ctx->cfg.prior_weight, e.w.as<double>(), e.wpart.as<double>());
      k_wfinal<<<grid_for(k_alloc, 256, ctx->sm_count * 4), 256, 0, st>>>(
          e.wpart.as<double>(), nparts, n, e.w.as<double>(), e.logw.as<double>(), e.cst_part.as<double>(),
          e.cst.as<double>(), which == 0 ? e.cdf.as<double>() : nullptr, k_alloc,
          e.mma ? e.hb.as<double>() : nullptr, e.mma ? e.ckk.as<double>() : nullptr);
      k_wnorm<<<grid_for(K, 256, ctx->sm_count * 4), 256, 0, st>>>(e.wpart.as<double>(), nparts, K, e.w.as<double>());
      ctx->launch_counter += 3;
    }
  }
  if (ctx->ncat) {
    k_cat_tables<<<pc, 64, 0, st>>>(ctx->cols.as<ColMeta>(), pc, n, ctx->cfg.prior_weight,
                                    ctx->cat_dist.as<double>(), e.tab.as<double>());
    ctx->launch_counter++;
  }
  // Experimental and OFF by default (TPE_TCS=1): correct (same parity tests) but slower than k_logpdf_mma at
  // config 2 -- the bf16 screen itself is cheap, the exact evaluation of the 8.9 % survivors on the CUDA cores is not
  static const bool tcs_on = [] { const char* v = getenv("TPE_TCS"); return v && v[0] == '1'; }();
  e.tcs = tcs_on && e.mma && K - 1 >= 1024 && (ctx->pb == 16 || ctx->pb == 32 || ctx->pb == 64);
  if (e.tcs) {
    e.tcs_kpad = round_up<int64_t>(K - 1, kTcsTile);
    CU(e.tcs_h.ensure((size_t)e.tcs_kpad * (ctx->pb + 8) * 2));
    CU(e.tcs_ak.ensure((size_t)e.tcs_kpad * 4));
    CU(e.tcs_ak64.ensure((size_t)e.tcs_kpad * 8));
    k_tcs_tables<<<grid_for(e.tcs_kpad, 256, 1 << 20), 256, 0, st>>>(
        e.tabc.as<double>(), e.cst.as<double>(), K - 1, e.tcs_kpad, ctx->pb,
        reinterpret_cast<__nv_bfloat16*>(e.tcs_h.p), e.tcs_ak.as<float>(), e.tcs_ak64.as<double>());
    ctx->launch_counter++;
  }
  e.uni_ready = false;
  if (ctx->uni_fast) {
    const int64_t ntiles = (K + kUniTile - 1) / kUniTile;
    CU(e.us32.ensure((size_t)ntiles * kUniTile * 16));
    CU(e.usmi.ensure((size_t)ntiles * kUniTile * 16));
    CU(e.usc.ensure((size_t)ntiles * kUniTile * 8));
    CU(e.umeta.ensure((size_t)ntiles * sizeof(UniTileMeta)));
    // large estimators: the kernels at the bandwidth floor go through the fast Gauss transform (k_fgt_*)
    static const int64_t fgt_min = [] { const char* v = getenv("TPE_FGT_MIN_K"); return v ? atoll(v) : 1024ll; }();
    e.fgt = ctx->cfg.magic_clip && K >= fgt_min;
    if (e.fgt) {
      CU(e.ucoef.ensure((size_t)kFgtMaxBoxes * kFgtRow * 8));
      CU(e.ubox.ensure((size_t)kFgtMaxBoxes * sizeof(FgtBox)));
      CU(e.ubstart.ensure((size_t)(kFgtMaxBoxes + 1) * 4));
    }
    k_uni_tables<<<(unsigned)ntiles, kUniTile, 0, st>>>(e.uord.as<int32_t>(), e.mu.as<double>(), e.sigma.as<double>(),
                                                        e.cst.as<double>(), ctx->cols.as<ColMeta>(), K, e.us32.as<float4>(),
                                                        e.usmi.as<double2>(), e.usc.as<double>(), e.umeta.as<UniTileMeta>(),
                                                        e.fgt ? 1 : 0, ctx->cfg.magic_clip, e.ubstart.as<int32_t>());
    ctx->launch_counter++;
    if (e.fgt) {
      k_fgt_coeff<<<kFgtMaxBoxes, 128, 0, st>>>(e.uord.as<int32_t>(), e.mu.as<double>(), e.sigma.as<double>(),
                                                e.cst.as<double>(), ctx->cols.as<ColMeta>(), K, ctx->cfg.magic_clip,
                                                e.ubstart.as<int32_t>(), e.ucoef.as<double>(), e.ubox.as<FgtBox>());
      CU(e.utlist.ensure((size_t)(ntiles + 1) * 4));
      k_uni_tile_list<<<1, 256, 0, st>>>(e.umeta.as<UniTileMeta>(), (int)ntiles, e.utlist.as<int32_t>());
      ctx->launch_counter += 2;
    }
    e.uni_ready = true;
  }
  CU(cudaGetLastError());
  return TPE_OK;
}

// k_logpdf_mixed: candidates per CTA that fit the shared memory (0: none do), and the bytes they take
size_t mixed_smem(const tpe_ctx* ctx, int CB) {
  const int ncp = (ctx->mix_ncont + 1) / 2, nd4 = (ctx->mix_nd + 3) / 4;
  return (size_t)CB * (2 * ncp + ctx->mix_tabd + 1) * 8 + (size_t)nd4 * 16 + 16;
}
int mixed_cb(const tpe_ctx* ctx) {
  for (int CB : {8, 4, 2})
    if (mixed_smem(ctx, CB) <= 200 * 1024) return CB;
  return 0;
}

// log-density of the Ct resident candidates under estimator `which`: fills e.part (k-split
// partials) and, for out-of-support candidates, e.fix.
int run_logpdf(tpe_ctx* ctx, int which, int64_t Ct, cudaEvent_t after_main = nullptr) {
  Estimator& e = ctx->est[which];
  cudaStream_t st = ctx->stream;
  if (which == 1 && join_above(ctx)) return TPE_E_CUDA;
  const int64_t K = e.K;
  if (which == 1 && ctx->kshard_world > 1 && !(ctx->fast && ctx->fast_mode == 2))
    return fail(ctx, TPE_E_STATE, "kernel sharding is for multivariate all-continuous suggestions");
  if (ctx->uni_fast && e.uni_ready && Ct <= 4096) {
    // one continuous column, univariate: sorted candidates x sorted kernels (tpe_uni.cuh)
    const int C = (int)Ct;
    if (!ctx->cands_sorted) {
      CU(ctx->uxs.ensure((size_t)round_up<int64_t>(C, 32) * 8));
      CU(ctx->ucidx.ensure((size_t)round_up<int64_t>(C, 32) * 4));
      k_uni_sort_cands<<<1, 1024, 0, st>>>(ctx->xT.as<double>(), C, ctx->cols.as<ColMeta>(), ctx->uxs.as<double>(),
                                           ctx->ucidx.as<int32_t>());
      ctx->launch_counter++;
      ctx->cands_sorted = true;
    }
    CU(e.part.ensure((size_t)2 * ctx->ct_stride * 16));
    const double skip = std::min(46.0, log((double)std::max<int64_t>(K, 1)) + 30.0);
    k_uni_grid<<<(unsigned)((C + 31) / 32), kUniWarps * 32, 0, st>>>(e.us32.as<float4>(), e.usmi.as<double2>(),
                                                                     e.usc.as<double>(), e.umeta.as<UniTileMeta>(), K,
                                                                     ctx->uxs.as<double>(), ctx->ucidx.as<int32_t>(), C, skip,
                                                                     e.part.as<double2>(), e.fgt ? e.utlist.as<int32_t>() : nullptr);
    ctx->launch_counter++;
    if (e.fgt) {
      static bool fgt_attr = false;
      if (!fgt_attr) {
        CU(cudaFuncSetAttribute(k_fgt_eval, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFgtEvalSmem));
        fgt_attr = true;
      }
      k_fgt_eval<<<(unsigned)((C + kFgtCands - 1) / kFgtCands), 256, kFgtEvalSmem, st>>>(
          e.ucoef.as<double>(), e.ubox.as<FgtBox>(), e.ubstart.as<int32_t>(), e.us32.as<float4>(), e.usmi.as<double2>(),
          e.usc.as<double>(), e.mu.as<double>(), e.sigma.as<double>(), e.cst.as<double>(), ctx->cols.as<ColMeta>(), K,
          ctx->cfg.magic_clip, ctx->xT.as<double>(), C, e.part.as<double2>() + ctx->ct_stride);
      ctx->launch_counter++;
    }
    ctx->last_kernel = e.fgt ? "k_uni_grid<sorted 1-D> + k_fgt_eval" : "k_uni_grid<sorted 1-D>";
    if (after_main) CU(cudaEventRecord(after_main, st));
    CU(e.fix.ensure((size_t)ctx->ct_stride * 16));
    k_logpdf_prior_fix<<<(unsigned)((Ct * 32 + 255) / 256), 256, 0, st>>>(
        ctx->S.as<double>(), Ct, ctx->cols.as<ColMeta>(), ctx->pc, e.mu.as<double>(), e.sigma.as<double>(),
        e.cst.as<double>(), K, e.tab.as<double>(), nullptr, ctx->oob.as<uint8_t>(), e.fix.as<double2>());
    ctx->launch_counter++;
    e.nsplit = e.fgt ? 2 : 1;
    CU(cudaGetLastError());
    return TPE_OK;
  }
  if (ctx->fast) {
    const bool cst_mode = ctx->fast_mode == 2;
    // tensor-core kernel unless the expanded square would lose more than 5e-13 (see k_logpdf_mma)
    bool use_mma = false;
    if (e.mma && K > 1) {
      const double nobs = (double)std::max<int64_t>(e.n, 1);
      double fac = 0.2 * pow(nobs, -1.0 / (ctx->pc + 4));
      if (ctx->cfg.magic_clip) fac = std::max(fac, 1.0 / std::min(100.0, 1.0 + (double)K));
      fac = std::min(std::max(fac, 1e-9), 1.0);
      const double rho = 0.5 / fac;
      use_mma = ctx->pb * rho * rho * 2.3e-16 <= 5e-13 && pick_mma(ctx->pb, Ct) != nullptr;
    }
    const FastCfg* fc = use_mma ? pick_mma(ctx->pb, Ct) : pick_fast(ctx->fast_mode, ctx->pb, Ct);
    // CONST tables exclude the prior kernel (its sigma differs); the mma table is padded to groups of 8
    int64_t Kf = use_mma ? round_up<int64_t>(K - 1, kMmaKPad) : (cst_mode ? K - 1 : K);
    // kernel sharding (g(x) only): this context takes the tiles [k_lo, k_hi) of the table; the prior kernel's slice
    // belongs to rank 0
    int64_t k_lo = 0;
    const bool sharded = which == 1 && ctx->kshard_world > 1;
    if (sharded) {
      if (!cst_mode) return fail(ctx, TPE_E_STATE, "kernel sharding is for multivariate all-continuous suggestions");
      const int64_t chunk = round_up<int64_t>((Kf + ctx->kshard_world - 1) / ctx->kshard_world, fc->tk);
      k_lo = std::min(Kf, chunk * ctx->kshard_rank);
      Kf = std::min(Kf, k_lo + chunk) - k_lo;
    }
    const int tc = fc->cands_per_cta;
    const int64_t ctiles = (Ct + tc - 1) / tc;
    // k-splits: two full waves of resident CTAs for the big configurations
    const int64_t ktiles = (Kf + fc->tk - 1) / fc->tk;
    const int64_t target = (fc->nt >= 256) ? (int64_t)ctx->sm_count * fc->minb * 2 : (int64_t)ctx->sm_count * 8;
    int64_t nsplit = 0, kps = fc->tk;
    if (ktiles > 0) {
      nsplit = std::max<int64_t>(1, std::min<int64_t>(ktiles, target / ctiles));
      const int64_t tiles_per = (ktiles + nsplit - 1) / nsplit;
      nsplit = (ktiles + tiles_per - 1) / tiles_per;
      kps = tiles_per * fc->tk;
    }
    // bf16 tensor-core screen + exact survivors (tpe_tcscreen.cuh): many candidates, rounding bound small enough
    bool use_tcs = false;
    if (e.tcs && cst_mode && Ct >= 256 && !sharded) {
      const double nobs = (double)std::max<int64_t>(e.n, 1);
      double fac = 0.2 * pow(nobs, -1.0 / (ctx->pc + 4));
      if (ctx->cfg.magic_clip) fac = std::max(fac, 1.0 / std::min(100.0, 1.0 + (double)K));
      fac = std::min(std::max(fac, 1e-9), 1.0);
      const double rho = 0.5 / fac, pr2 = ctx->pb * rho * rho;
      const double delta = pr2 * (1.0 / 256 + 1.0 / 65536 + (ctx->pb + 2) * 5.97e-8) * 1.02 + 2e-3;
      if (delta <= 6.0 && pr2 * 2.3e-16 <= 5e-13) {   // (the second: conditioning of the expanded square, as for k_logpdf_mma)
        use_tcs = true;
        const int pb = ctx->pb;
        const size_t smem_sum = pb == 16 ? sizeof(TcsSmem<16>) : pb == 32 ? sizeof(TcsSmem<32>) : sizeof(TcsSmem<64>);
        const size_t smem_max = pb == 16 ? offsetof(TcsSmem<16>, b64) : pb == 32 ? offsetof(TcsSmem<32>, b64) : offsetof(TcsSmem<64>, b64);
        const int64_t tctiles = (Ct + kTcsRows - 1) / kTcsRows, tktiles = e.tcs_kpad / kTcsTile;
        const int64_t slots = (int64_t)ctx->sm_count * (smem_sum <= 113 * 1024 ? 2 : 1);
        int64_t tns = std::max<int64_t>(1, std::min<int64_t>(tktiles, slots / tctiles));
        const int64_t tiles_per = (tktiles + tns - 1) / tns;
        tns = (tktiles + tiles_per - 1) / tiles_per;
        const int64_t tkps = tiles_per * kTcsTile;
        CU(e.part.ensure((size_t)(tns + 1) * ctx->ct_stride * 16));
        CU(ctx->x64s.ensure((size_t)ctx->ct_stride * pb * 8));
        CU(ctx->e32s.ensure((size_t)ctx->ct_stride * 4));
        CU(ctx->x32s.ensure((size_t)ctx->ct_stride * 8));   // (-|x''|^2 / 2 in fp64)
        CU(ctx->gmax.ensure((size_t)ctx->ct_stride * 4));
        k_tcs_xprep<<<grid_for(ctx->ct_stride, 256, 1 << 20), 256, 0, st>>>(
            ctx->xT.as<double>(), e.colprm.as<double2>(), ctx->ct_stride, pb, ctx->x64s.as<double>(),
            ctx->e32s.as<float>(), ctx->x32s.as<double>(), ctx->gmax.as<int>());
        const double skip_t = std::min(46.0, log((double)std::max<int64_t>(K, 1)) + 30.0);
        const float window = (float)(skip_t + 2.0 * delta);
        // TPE_TCS_STATS=1 (diagnostics): count the survivors of every launch and print them
        static const bool tcs_stats_on = [] { const char* v = getenv("TPE_TCS_STATS"); return v && v[0] == '1'; }();
        unsigned long long* tcs_stats = nullptr;
        if (tcs_stats_on) {
          CU(ctx->lse_gmax.ensure(64));
          CU(cudaMemsetAsync(ctx->lse_gmax.p, 0, 8, st));
          tcs_stats = ctx->lse_gmax.as<unsigned long long>();
        }
#define TPE_TCS_LAUNCH(PBV)                                                                                            \
        do {                                                                                                           \
          static bool attr_done = false;                                                                               \
          if (!attr_done) {                                                                                            \
            CU(cudaFuncSetAttribute(k_tcs<PBV, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_max));   \
            CU(cudaFuncSetAttribute(k_tcs<PBV, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_sum));    \
            attr_done = true;                                                                                          \
          }                                                                                                            \
          k_tcs<PBV, false><<<dim3((unsigned)tctiles, (unsigned)tns), kTcsNT, smem_max, st>>>(                         \
              reinterpret_cast<const __nv_bfloat16*>(e.tcs_h.p), e.tcs_ak.as<float>(), e.tabc.as<double>(),            \
              e.tcs_ak64.as<double>(), e.tcs_kpad, tkps, ctx->x64s.as<double>(), ctx->e32s.as<float>(),               \
              ctx->x32s.as<double>(), ctx->gmax.as<int>(), Ct, ctx->ct_stride, window, e.part.as<double2>(), tcs_stats);                                                       \
          k_tcs<PBV, true><<<dim3((unsigned)tctiles, (unsigned)tns), kTcsNT, smem_sum, st>>>(                          \
              reinterpret_cast<const __nv_bfloat16*>(e.tcs_h.p), e.tcs_ak.as<float>(), e.tabc.as<double>(),            \
              e.tcs_ak64.as<double>(), e.tcs_kpad, tkps, ctx->x64s.as<double>(), ctx->e32s.as<float>(),               \
              ctx->x32s.as<double>(), ctx->gmax.as<int>(), Ct, ctx->ct_stride, window, e.part.as<double2>(), tcs_stats);                                                       \
        } while (0)
        if (pb == 16) TPE_TCS_LAUNCH(16);
        else if (pb == 32) TPE_TCS_LAUNCH(32);
        else TPE_TCS_LAUNCH(64);
#undef TPE_TCS_LAUNCH
        ctx->launch_counter += 3;
        if (tcs_stats_on) {
          unsigned long long hs = 0;
          CU(cudaMemcpyAsync(&hs, tcs_stats, 8, cudaMemcpyDeviceToHost, st));
          CU(cudaStreamSynchronize(st));
          fprintf(stderr, "[tpe] k_tcs: %llu survivors of %lld x %lld cells (%.2f %%), window %.2f\n", hs, (long long)Ct,
                  (long long)(K - 1), 100.0 * (double)hs / ((double)Ct * (double)(K - 1)), (double)window);
        }
        nsplit = tns;
        ctx->last_kernel = "k_tcs<bf16 screen + exact survivors>";
      }
    }
#ifdef TPE_LAB
    // fp32-screened variant (tpe_screen.cuh): multivariate, 17..32 continuous columns, many candidates
    // Experimental and OFF by default: correct (same parity tests) but slower than the exact kernel at
    // config 2.  TPE_SCREEN=1 enables it.
    static const bool screen_on = [] { const char* v = getenv("TPE_SCREEN"); return v && v[0] == '1'; }();
    const bool use_screen = !use_tcs && cst_mode && !use_mma && ctx->pb == kScrP && Ct > 128 && Kf > 0 && screen_on;
    if (use_screen) {
      const int64_t sctiles = (Ct + kScrCands - 1) / kScrCands;
      const int64_t sktiles = (Kf + kScrTK - 1) / kScrTK;
      int64_t sns = std::max<int64_t>(1, std::min<int64_t>(sktiles, (int64_t)ctx->sm_count * 2 / sctiles));
      const int64_t tiles_per = (sktiles + sns - 1) / sns;
      sns = (sktiles + tiles_per - 1) / tiles_per;
      const int64_t skps = tiles_per * kScrTK;
      CU(e.part.ensure((size_t)(sns + 1) * ctx->ct_stride * 16));
      if (!e.screen_ready) {
        CU(e.tab32.ensure((size_t)Kf * kScrP * 4 + 64));
        CU(e.tab64p.ensure((size_t)Kf * kScrStride * 8 + 64));
        CU(e.d32.ensure((size_t)Kf * 4 + 64));
        k_screen_tabprep<<<grid_for(Kf * 32, 256, ctx->sm_count * 8), 256, 0, st>>>(
            e.tabc.as<double>(), e.cst.as<double>(), Kf, e.tab32.as<float>(), e.tab64p.as<double>(), e.d32.as<float>());
        ctx->launch_counter++;
        e.screen_ready = true;
      }
      CU(ctx->x64s.ensure((size_t)ctx->ct_stride * kScrP * 8));
      CU(ctx->x32s.ensure((size_t)ctx->ct_stride * kScrP * 4));
      CU(ctx->e32s.ensure((size_t)ctx->ct_stride * 4));
      CU(ctx->gmax.ensure((size_t)ctx->ct_stride * 4));
      k_screen_xprep<<<grid_for(ctx->ct_stride, 256, 1 << 20), 256, 0, st>>>(
          ctx->xT.as<double>(), e.colprm.as<double2>(), ctx->ct_stride, ctx->x64s.as<double>(), ctx->x32s.as<float>(),
          ctx->e32s.as<float>(), ctx->gmax.as<float>());
      ctx->launch_counter++;
      if (!ctx->screen_attr_set) {
        CU(cudaFuncSetAttribute(k_logpdf_screen, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(ScreenSmem)));
        ctx->screen_attr_set = true;
      }
      // fp32 error bound of the screening value: dot product of P terms + input rounding, over
      // |x''|, |mu''| <= rho = (range / 2) / sigma (identical for every column of a multivariate estimator)
      const double nobs = (double)std::max<int64_t>(e.n, 1);
      double fac = 0.2 * pow(nobs, -1.0 / (ctx->pc + 4));
      if (ctx->cfg.magic_clip) fac = std::max(fac, 1.0 / std::min(100.0, 1.0 + (double)K));
      fac = std::min(std::max(fac, 1e-9), 1.0);
      const double rho = 0.5 / fac;
      const float margin = (float)(0.5 + 8e-6 * kScrP * rho * rho);
      k_logpdf_screen<<<dim3((unsigned)sctiles, (unsigned)sns), kScrNT, sizeof(ScreenSmem), st>>>(
          e.tab32.as<float>(), e.tab64p.as<double>(), e.cst.as<double>(), e.d32.as<float>(), Kf,
          ctx->x64s.as<double>(), ctx->x32s.as<float>(), ctx->e32s.as<float>(), ctx->gmax.as<float>(),
          ctx->ct_stride, skps,
          std::min(46.0, log((double)std::max<int64_t>(K, 1)) + 30.0), margin, e.part.as<double2>());
      ctx->launch_counter++;
      nsplit = sns;
      ctx->last_kernel = "k_logpdf_screen<fp32 screen + fp64 exact>";
    }
#else
    constexpr bool use_screen = false;
#endif
    if (!use_screen && !use_tcs) CU(e.part.ensure((size_t)(nsplit + 1) * ctx->ct_stride * 16));
    if (nsplit > 0 && !use_screen && !use_tcs) {
      if (!ctx->prepared_cfgs.count(fc)) {
        CU(fc->prepare());
        ctx->prepared_cfgs.insert(fc);
      }
      if (use_mma) {
        CU(ctx->lse_gmax.ensure((size_t)ctx->ct_stride * 8));
        CU(cudaMemsetAsync(ctx->lse_gmax.p, 0, (size_t)ctx->ct_stride * 8, st));
      }
      // (both CONST tables are blocked by whole kernels -- the fragment-major one in groups of 8 -- so a slice that
      // starts at a multiple of the tile is a plain offset)
      fc->launch(dim3((unsigned)ctiles, (unsigned)nsplit), fc->smem, st,
                 use_mma ? (const void*)(e.tabm.as<double>() + k_lo * ctx->pb)
                         : (cst_mode ? (const void*)(e.tabc.as<double>() + k_lo * ctx->pb) : (const void*)e.tabp.p),
                 (use_mma ? e.ckk.as<double>() : e.cst.as<double>()) + k_lo, Kf,
                 e.colprm.as<double2>(), ctx->xT.as<double>(), ctx->ct_stride, kps,
                 std::min(46.0, log((double)std::max<int64_t>(K, 1)) + 30.0), e.part.as<double2>(),
                 use_mma ? ctx->lse_gmax.as<unsigned long long>() : nullptr);
      ctx->launch_counter++;
    }
    if (use_tcs) {
    } else if (use_mma && !use_screen)
      ctx->last_kernel = (fc->nt >= 256) ? "k_logpdf_mma<big>" : "k_logpdf_mma<small>";
    else if (!use_screen)
      ctx->last_kernel = cst_mode ? ((fc->nt >= 256) ? "k_logpdf_fast<const,big>" : "k_logpdf_fast<const,small>")
                                  : ((fc->nt >= 256) ? "k_logpdf_fast<pair,big>" : "k_logpdf_fast<pair,small>");
    if (after_main) CU(cudaEventRecord(after_main, st));
    // the prior kernel of CONST tables (one more partial row) and the exact fix-up of the candidates
    // outside [low, high], one launch
    CU(e.fix.ensure((size_t)ctx->ct_stride * 16));
    k_logpdf_prior_fix<<<(unsigned)((Ct * 32 + 255) / 256), 256, 0, st>>>(
        ctx->S.as<double>(), Ct, ctx->cols.as<ColMeta>(), ctx->pc, e.mu.as<double>(), e.sigma.as<double>(),
        e.cst.as<double>(), K, e.tab.as<double>(),
        (cst_mode && !(sharded && ctx->kshard_rank != 0)) ? e.part.as<double2>() + nsplit * ctx->ct_stride : nullptr,
        ctx->oob.as<uint8_t>(), e.fix.as<double2>());
    ctx->launch_counter++;
    if (cst_mode && !(sharded && ctx->kshard_rank != 0)) nsplit += 1;
    e.nsplit = (int)nsplit;
  } else if (e.mixed && !ctx->user_points && Ct >= 64 && mixed_cb(ctx) > 0) {
    // mixed space, many candidates: kernel-minor tables, the candidates' table rows in shared memory (tpe_mixed.cuh)
    if (ctx->dtab_doubles) {
      int64_t rows_max = 1;
      for (const ColMeta& cm : ctx->cols_h)
        if (cm.grid > 0) rows_max = std::max<int64_t>(rows_max, (int64_t)std::min<int64_t>(Ct, cm.grid) * (cm.grid + 1));
      const unsigned gx = (unsigned)std::min<int64_t>((rows_max + 255) / 256, ctx->sm_count * 4);
      k_disc_tables<<<dim3(gx, (unsigned)ctx->pc), 256, 0, st>>>(ctx->cols.as<ColMeta>(), ctx->pc, e.mu.as<double>(),
                                                                 e.sigma.as<double>(), K, ctx->S.as<double>(), Ct,
                                                                 e.dtab.as<double>());
      ctx->launch_counter++;
    }
    const int CB = mixed_cb(ctx);
    const int64_t nx = (Ct + CB - 1) / CB;
    int64_t nsplit = std::max<int64_t>(1, std::min<int64_t>(32, (2ll * ctx->sm_count + nx - 1) / nx));
    const int64_t kps = round_up<int64_t>((K - 1 + nsplit - 1) / nsplit, 512);
    nsplit = (K - 1 + kps - 1) / kps;
    CU(e.part.ensure((size_t)(nsplit + 1) * ctx->ct_stride * 16));
    CU(e.fix.ensure((size_t)ctx->ct_stride * 16));
    const size_t smem = mixed_smem(ctx, CB);
    const double skip = std::min(46.0, log((double)std::max<int64_t>(K, 1)) + 30.0);
#define TPE_MIXED_LAUNCH(CBV)                                                                                          \
    do {                                                                                                               \
      static bool attr_done = false;                                                                                   \
      if (!attr_done) {                                                                                                \
        CU(cudaFuncSetAttribute(k_logpdf_mixed<CBV>, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));        \
        attr_done = true;                                                                                              \
      }                                                                                                                \
      k_logpdf_mixed<CBV><<<dim3((unsigned)nx, (unsigned)nsplit), 512, smem, st>>>(                                    \
          ctx->S.as<double>(), Ct, ctx->cols.as<ColMeta>(), ctx->pc, ctx->mixcols.as<MixCol>(), ctx->mix_ncont,        \
          ctx->mix_nd, ctx->mix_tabd, e.sigma.as<double>(), e.cst.as<double>(), K - 1, e.mix_kstride, kps,             \
          e.mxc.as<double2>(), e.mxd.as<ushort4>(), e.tab.as<double>(), e.dtab.as<double>(), ctx->oob.as<uint8_t>(),   \
          skip, e.part.as<double2>(), ctx->ct_stride);                                                                 \
    } while (0)
    if (CB == 8) TPE_MIXED_LAUNCH(8);
    else if (CB == 4) TPE_MIXED_LAUNCH(4);
    else TPE_MIXED_LAUNCH(2);
#undef TPE_MIXED_LAUNCH
    ctx->launch_counter++;
    ctx->last_kernel = "k_logpdf_mixed";
    if (after_main) CU(cudaEventRecord(after_main, st));
    k_logpdf_prior_fix<<<(unsigned)((Ct * 32 + 255) / 256), 256, 0, st>>>(
        ctx->S.as<double>(), Ct, ctx->cols.as<ColMeta>(), ctx->pc, e.mu.as<double>(), e.sigma.as<double>(),
        e.cst.as<double>(), K, e.tab.as<double>(), e.part.as<double2>() + nsplit * ctx->ct_stride, ctx->oob.as<uint8_t>(),
        e.fix.as<double2>(), 0);
    ctx->launch_counter++;
    e.nsplit = (int)nsplit + 1;
  } else {
    // pair-parallel generic kernel: grid = (candidates, kernel chunks of 256 * kpt)
    int kpt = 1;
    while ((K + 256ll * kpt - 1) / (256ll * kpt) > 65535 ||
           ((K + 256ll * kpt - 1) / (256ll * kpt)) * Ct > (1ll << 22) * 4)
      kpt *= 2;  // keep the partial table (nsplit x Ct) and the grid within bounds
    const int64_t nsplit = (K + 256ll * kpt - 1) / (256ll * kpt);
    CU(e.part.ensure((size_t)nsplit * ctx->ct_stride * 16));
    e.nsplit = (int)nsplit;
    if (ctx->dtab_doubles) {
      int64_t rows_max = 1;
      for (const ColMeta& cm : ctx->cols_h)
        if (cm.grid > 0) rows_max = std::max<int64_t>(rows_max, (int64_t)std::min<int64_t>(Ct, cm.grid) * (cm.grid + 1));
      const unsigned gx = (unsigned)std::min<int64_t>((rows_max + 255) / 256, ctx->sm_count * 4);
      k_disc_tables<<<dim3(gx, (unsigned)ctx->pc), 256, 0, st>>>(ctx->cols.as<ColMeta>(), ctx->pc, e.mu.as<double>(),
                                                                 e.sigma.as<double>(), K, ctx->S.as<double>(), Ct,
                                                                 e.dtab.as<double>());
      ctx->launch_counter++;
    }
    if (K >= 4096) {
      constexpr int CB = 8;
      k_logpdf_pairs<CB><<<dim3((unsigned)((Ct + CB - 1) / CB), (unsigned)nsplit), 256,
                           (size_t)CB * ctx->pc * sizeof(PairCol) + (((size_t)ctx->pc + 7) & ~(size_t)7), st>>>(
          ctx->S.as<double>(), Ct, ctx->cols.as<ColMeta>(), ctx->pc, e.mu.as<double>(), e.sigma.as<double>(),
          e.cst.as<double>(), K, kpt, e.tab.as<double>(), ctx->dtab_doubles ? e.cls.as<int32_t>() : nullptr,
          ctx->dtab_doubles ? e.dtab.as<double>() : nullptr, ctx->dtab_doubles ? e.offgrid.as<int>() : nullptr,
          ctx->oob.as<uint8_t>(), e.part.as<double2>(), ctx->ct_stride);
    } else {
      constexpr int CB = 1;
      k_logpdf_pairs<CB><<<dim3((unsigned)((Ct + CB - 1) / CB), (unsigned)nsplit), 256,
                           (size_t)CB * ctx->pc * sizeof(PairCol) + (((size_t)ctx->pc + 7) & ~(size_t)7), st>>>(
          ctx->S.as<double>(), Ct, ctx->cols.as<ColMeta>(), ctx->pc, e.mu.as<double>(), e.sigma.as<double>(),
          e.cst.as<double>(), K, kpt, e.tab.as<double>(), ctx->dtab_doubles ? e.cls.as<int32_t>() : nullptr,
          ctx->dtab_doubles ? e.dtab.as<double>() : nullptr, ctx->dtab_doubles ? e.offgrid.as<int>() : nullptr,
          ctx->oob.as<uint8_t>(), e.part.as<double2>(), ctx->ct_stride);
    }
    ctx->launch_counter++;
    ctx->last_kernel = "k_logpdf_pairs";
    if (after_main) CU(cudaEventRecord(after_main, st));
  }
  CU(cudaGetLastError());
  return TPE_OK;
}

int ensure_candidate_buffers(tpe_ctx* ctx, int64_t Ct) {
  ctx->Ct = Ct;
  ctx->cands_sorted = false;
  ctx->ct_stride = round_up<int64_t>(Ct, 1024);
  CU(ctx->S.ensure((size_t)ctx->ct_stride * ctx->pc * 8));
  CU(ctx->oob.ensure((size_t)ctx->ct_stride));
  CU(ctx->logl.ensure((size_t)ctx->ct_stride * 8));
  CU(ctx->logg.ensure((size_t)ctx->ct_stride * 8));
  CU(cudaMemsetAsync(ctx->oob.p, 0, (size_t)ctx->ct_stride, ctx->stream));
  if (ctx->fast) {
    CU(ctx->xT.ensure((size_t)ctx->ct_stride * ctx->pb * 8));
    CU(cudaMemsetAsync(ctx->xT.p, 0, (size_t)ctx->ct_stride * ctx->pb * 8, ctx->stream));
  }
  return TPE_OK;
}

}  // namespace


// ---- univariate batch, stage by stage over all columns (tpe_unib.cuh) ---------------------------------------------------
struct Carver {
  char* base = nullptr;
  size_t off = 0;
  template <class T>
  T* take(size_t count) {
    off = (off + 255) & ~(size_t)255;
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off += count * sizeof(T);
    return p;
  }
};
struct UbPtrs {
  double *mu[2], *sigma[2], *cstp[2], *cst[2], *w[2], *logw[2], *cdf, *wpart, *zero, *cstscr, *sc[2], *coef;
  int32_t *ord0, *bstart, *cidx, *sidx, *tlist;
  float4* s32[2];
  double2 *smi[2], *part[2], *fix[2];
  UniTileMeta* meta[2];
  FgtBox* box;
  double *S, *xT, *xs, *logl, *logg;
  uint8_t* oob;
  uint64_t* skeys;
  SortWork* swk;
  int* work;
  ColMeta* cols;
};
static void ub_carve(Carver& c, UbPtrs& p, int P, const int64_t ks[2], int64_t cs, bool big_sort) {
  for (int w = 0; w < 2; ++w) {
    p.mu[w] = c.take<double>((size_t)P * ks[w]);
    p.sigma[w] = c.take<double>((size_t)P * ks[w]);
    p.cstp[w] = c.take<double>((size_t)P * ks[w]);
    p.cst[w] = c.take<double>((size_t)P * ks[w]);
    p.w[w] = c.take<double>((size_t)ks[w]);
    p.logw[w] = c.take<double>((size_t)ks[w]);
    p.s32[w] = c.take<float4>((size_t)P * ks[w]);
    p.smi[w] = c.take<double2>((size_t)P * ks[w]);
    p.sc[w] = c.take<double>((size_t)P * ks[w]);
    p.meta[w] = c.take<UniTileMeta>((size_t)P * (ks[w] / kUniTile));
    p.part[w] = c.take<double2>((size_t)P * 2 * cs);
    p.fix[w] = c.take<double2>((size_t)P * cs);
  }
  p.cdf = c.take<double>((size_t)ks[0]);
  p.wpart = c.take<double>(1024);
  p.zero = c.take<double>((size_t)ks[1]);
  p.cstscr = c.take<double>((size_t)ks[1]);
  p.ord0 = c.take<int32_t>((size_t)P * ks[0]);
  p.bstart = c.take<int32_t>((size_t)P * (kFgtMaxBoxes + 1));
  p.tlist = c.take<int32_t>((size_t)P * (ks[1] / kUniTile + 1));
  p.coef = c.take<double>((size_t)P * kFgtMaxBoxes * kFgtRow);
  p.box = c.take<FgtBox>((size_t)P * kFgtMaxBoxes);
  p.S = c.take<double>((size_t)P * cs);
  p.xT = c.take<double>((size_t)P * cs);
  p.xs = c.take<double>((size_t)P * cs);
  p.cidx = c.take<int32_t>((size_t)P * cs);
  p.logl = c.take<double>((size_t)P * cs);
  p.logg = c.take<double>((size_t)P * cs);
  p.oob = c.take<uint8_t>((size_t)P * cs);
  p.work = c.take<int>((size_t)P * 4);
  p.cols = c.take<ColMeta>((size_t)P);
  if (big_sort) {
    p.skeys = c.take<uint64_t>((size_t)P * 2 * ks[1]);
    p.sidx = c.take<int32_t>((size_t)P * 2 * ks[1]);
    p.swk = c.take<SortWork>((size_t)P);
  } else {
    p.skeys = nullptr;
    p.sidx = nullptr;
    p.swk = nullptr;
  }
}

// The caller (tpe_suggest_univariate_batch) has run the split, checked the weights and compared the above rows with
// the previous call's (ctx->uni_mode); U holds the uniforms [n_cols][2 C] (ctx->ev_u).  Results into ctx->out_*.
static int uni_batch_staged(tpe_ctx* ctx, const tpe_cfg* cfg, const int32_t* cols, int32_t P, const double* w_below,
                            const double* w_above) {
  cudaStream_t st = ctx->stream;
  const int32_t C = cfg->n_candidates;
  const int64_t n[2] = {ctx->est[0].n, ctx->est[1].n};
  const int64_t K[2] = {n[0] + 1, n[1] + 1};
  const int64_t ks[2] = {round_up<int64_t>(K[0] + 160, 1024), round_up<int64_t>(K[1] + 160, 1024)};
  const int64_t cs = round_up<int64_t>(C, 1024);
  const bool big_sort = K[1] > 4096 || K[0] > 4096;
  Carver c0;
  UbPtrs p{};
  ub_carve(c0, p, P, ks, cs, big_sort);
  CU(ctx->ub_arena.ensure(c0.off + 4096));
  Carver c;
  c.base = static_cast<char*>(ctx->ub_arena.p);
  ub_carve(c, p, P, ks, cs, big_sort);
  UbDims d[2];
  for (int w = 0; w < 2; ++w) {
    d[w].ks = ks[w];
    d[w].cs = cs;
    d[w].pall = (int32_t)ctx->space.size();
  }
  kb_cols<<<(P + 63) / 64, 64, 0, st>>>(ctx->cols.as<ColMeta>(), P, p.cols);   // (on the device: a copy from pageable
                                                                               // host memory would wait for the split)
  const ColMeta* dcols = p.cols;
  const int cap = ctx->sm_count * 8;
  const unsigned Pu = (unsigned)P;
  CU(cudaMemsetAsync(p.zero, 0, (size_t)ks[1] * 8, st));
  CU(cudaMemsetAsync(p.oob, 0, (size_t)P * cs, st));
  CU(cudaMemsetAsync(p.work, 0, (size_t)P * 16, st));
  // the above orders of the previous call, if they belong to this one
  DevBuf& ord_new_buf = ctx->ub_ord_cur == 0 ? ctx->ub_ord_b : ctx->ub_ord_a;
  DevBuf& ord_old_buf = ctx->ub_ord_cur == 0 ? ctx->ub_ord_a : ctx->ub_ord_b;
  CU(ord_new_buf.ensure((size_t)P * ks[1] * 4));
  const bool inc = K[1] > 4096 && ctx->ub_ord_seq + 1 == ctx->uni_seq && ctx->ub_ord_lineage == ctx->hist_lineage &&
                   (ctx->ub_ord_K == K[1] || ctx->ub_ord_K == K[1] - 1) && ctx->ub_ord_ks == ks[1] &&
                   ord_old_buf.cap >= (size_t)P * ks[1] * 4 && ctx->ub_ord_cols.size() == (size_t)P &&
                   std::equal(cols, cols + P, ctx->ub_ord_cols.begin());
  int32_t* ord[2] = {p.ord0, ord_new_buf.as<int32_t>()};
  for (int w = 0; w < 2; ++w) {
    const double* wh = w == 0 ? w_below : w_above;
    kb_mu<<<dim3((unsigned)grid_for(K[w], 256, cap), Pu), 256, 0, st>>>(ctx->X.as<double>(), d[w],
                                                                        ctx->est[w].rows.as<int64_t>(), n[w], dcols, p.mu[w]);
    int64_t m2 = 1;
    while (m2 < K[w]) m2 <<= 1;
    if (m2 <= 4096) {
      kb_sort_small<<<dim3(1, Pu), 1024, 0, st>>>(p.mu[w], d[w], (int)K[w], (int)m2, ord[w]);
    } else {
      const int* run_flag = nullptr;
      if (w == 1 && inc) {
        run_flag = ctx->uni_mode.as<int>();
        kb_order_update<<<dim3((unsigned)grid_for(ctx->ub_ord_K, 256, ctx->sm_count), Pu), 256, 0, st>>>(
            run_flag, ord_old_buf.as<int32_t>(), d[1], (int)ctx->ub_ord_K, (int)K[1], p.mu[1], ord[1], p.work);
        ctx->launch_counter++;
      }
      if (ctx->ub_sort_g == 0) {
        int occ = 0;
        CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kb_radix_sort, 512, 0));
        ctx->ub_sort_g = std::max(1, occ) * ctx->sm_count;
      }
      const int G = (int)std::max<int64_t>(1, std::min<int64_t>(std::min<int64_t>(160, ctx->ub_sort_g / P), (K[w] + 1023) / 1024));
      if (G * P > ctx->ub_sort_g) return fail(ctx, TPE_E_STATE, "not batchable: %d columns exceed the cooperative sort", P);
      const double* a_mu = p.mu[w];
      UbDims a_d = d[w];
      int a_n = (int)K[w];
      uint64_t* a_keys = p.skeys;
      int32_t* a_idx = p.sidx;
      SortWork* a_wk = p.swk;
      int32_t* a_order = ord[w];
      void* args[] = {&a_mu, &a_d, &a_n, &a_keys, &a_idx, &a_wk, &a_order, &run_flag};
      CU(cudaLaunchCooperativeKernel((const void*)kb_radix_sort, dim3((unsigned)G, Pu), dim3(512), args, 0, st));
    }
    kb_sigma_uni<<<dim3((unsigned)grid_for(K[w], 256, cap), Pu), 256, 0, st>>>(
        p.mu[w], ord[w], d[w], dcols, n[w], cfg->magic_clip, cfg->endpoints, p.sigma[w]);
    kb_const<<<dim3((unsigned)grid_for(K[w], 256, cap), Pu), 256, 0, st>>>(p.mu[w], p.sigma[w], d[w], dcols, K[w], p.cstp[w]);
    // mixture weights: the same for every column
    const double* w_dev = nullptr;
    if (wh != nullptr && n[w] > 0) {
      CU(ctx->ub_wstage.ensure((size_t)(n[0] + n[1] + 2) * 8));
      double* dst = ctx->ub_wstage.as<double>() + (w == 0 ? 0 : n[0] + 1);
      CU(cudaMemcpyAsync(dst, wh, (size_t)n[w] * 8, cudaMemcpyHostToDevice, st));
      w_dev = dst;
    }
    const int64_t k_alloc = round_up<int64_t>(K[w] + 32, 32);
    const int nparts = grid_for(K[w], 2048, ctx->sm_count * 2);
    if (nparts == 1) {
      k_weights_one<<<1, 256, 0, st>>>(w_dev, nullptr, n[w], cfg->prior_weight, p.w[w], p.logw[w], p.zero, p.cstscr,
                                       w == 0 ? p.cdf : nullptr, k_alloc, nullptr, nullptr);
      ctx->launch_counter += 1;
    } else {
      k_wraw<<<nparts, 256, 0, st>>>(w_dev, nullptr, n[w], cfg->prior_weight, p.w[w], p.wpart);
      k_wfinal<<<grid_for(k_alloc, 256, ctx->sm_count * 4), 256, 0, st>>>(p.wpart, nparts, n[w], p.w[w], p.logw[w], p.zero,
                                                                          p.cstscr, w == 0 ? p.cdf : nullptr, k_alloc,
                                                                          nullptr, nullptr);
      k_wnorm<<<grid_for(K[w], 256, ctx->sm_count * 4), 256, 0, st>>>(p.wpart, nparts, K[w], p.w[w]);
      ctx->launch_counter += 3;
    }
    kb_cst<<<dim3((unsigned)grid_for(ks[w], 256, cap), Pu), 256, 0, st>>>(p.cstp[w], p.logw[w], d[w], K[w], p.cst[w]);
    static const int64_t fgt_min = [] { const char* v = getenv("TPE_FGT_MIN_K"); return v ? atoll(v) : 1024ll; }();
    const bool fgt = cfg->magic_clip && K[w] >= fgt_min;
    const unsigned ntiles = (unsigned)((K[w] + kUniTile - 1) / kUniTile);
    kb_uni_tables<<<dim3(ntiles, Pu), kUniTile, 0, st>>>(ord[w], p.mu[w], p.sigma[w], p.cst[w], d[w], dcols, K[w], p.s32[w],
                                                         p.smi[w], p.sc[w], p.meta[w], fgt ? 1 : 0, cfg->magic_clip, p.bstart);
    if (fgt) {
      if (w == 0) return fail(ctx, TPE_E_STATE, "not batchable: a below set of %lld trials", (long long)n[0]);
      kb_fgt_coeff<<<dim3(kFgtMaxBoxes, Pu), 128, 0, st>>>(ord[w], p.mu[w], p.sigma[w], p.cst[w], d[w], dcols, K[w],
                                                           cfg->magic_clip, p.bstart, p.coef, p.box);
      kb_uni_tile_list<<<dim3(1, Pu), 256, 0, st>>>(p.meta[w], d[w], (int)ntiles, p.tlist);
      ctx->launch_counter += 2;
    }
    ctx->launch_counter += 6;
  }
  // candidates of every column from its l(x), both log-densities, the argmax
  CU(cudaStreamWaitEvent(st, ctx->ev_u, 0));
  kb_sample<<<dim3((unsigned)grid_for((int64_t)C, 128, ctx->sm_count * 16), Pu), 128, 0, st>>>(
      ctx->U.as<double>(), C, d[0], dcols, p.cdf, K[0], p.mu[0], p.sigma[0], p.S, p.xT, p.oob);
  kb_uni_sort_cands<<<dim3(1, Pu), 1024, 0, st>>>(p.xT, C, d[0], dcols, p.xs, p.cidx);
  const unsigned ngrp = (unsigned)((C + 31) / 32);
  static const int64_t fgt_min2 = [] { const char* v = getenv("TPE_FGT_MIN_K"); return v ? atoll(v) : 1024ll; }();
  int nsl[2] = {1, 1};
  for (int w = 0; w < 2; ++w) {
    const double skip = std::min(46.0, log((double)std::max<int64_t>(K[w], 1)) + 30.0);
    const bool fgt_w = cfg->magic_clip && K[w] >= fgt_min2;
    kb_uni_grid<<<dim3(ngrp, Pu), kUniWarps * 32, 0, st>>>(p.s32[w], p.smi[w], p.sc[w], p.meta[w], d[w], K[w], p.xs, p.cidx, C,
                                                           skip, p.part[w], fgt_w ? p.tlist : nullptr);
    if (fgt_w) {
      static bool fgt_attr = false;
      if (!fgt_attr) {
        CU(cudaFuncSetAttribute(kb_fgt_eval, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFgtEvalSmem));
        fgt_attr = true;
      }
      kb_fgt_eval<<<dim3((unsigned)((C + kFgtCands - 1) / kFgtCands), Pu), 256, kFgtEvalSmem, st>>>(
          p.coef, p.box, p.bstart, p.s32[w], p.smi[w], p.sc[w], p.mu[w], p.sigma[w], p.cst[w], d[w], dcols, K[w],
          cfg->magic_clip, p.xT, C, p.part[w]);
      nsl[w] = 2;
      ctx->launch_counter++;
    }
    kb_prior_fix<<<dim3((unsigned)(((int64_t)C * 32 + 255) / 256), Pu), 256, 0, st>>>(p.S, C, d[w], dcols, p.mu[w], p.sigma[w],
                                                                                     p.cst[w], K[w], p.oob, p.fix[w]);
    ctx->launch_counter += 2;
  }
  kb_acq2<<<dim3((unsigned)((C + 255) / 256), Pu), 256, 0, st>>>(
      p.part[0], nsl[0], p.part[1], nsl[1], d[0], p.oob, p.fix[0], p.fix[1], C, p.logl, p.logg);
  kb_select<<<dim3(1, Pu), 256, 0, st>>>(p.logl, p.logg, C, d[0], p.S, ctx->out_x.as<double>(), ctx->out_acq.as<double>(),
                                         ctx->out_best.as<int64_t>());
  ctx->launch_counter += 4;
  CU(cudaGetLastError());
  // what the next call may start from
  ctx->ub_ord_cur ^= 1;
  ctx->ub_ord_seq = ctx->uni_seq;
  ctx->ub_ord_lineage = ctx->hist_lineage;
  ctx->ub_ord_K = K[1];
  ctx->ub_ord_ks = ks[1];
  ctx->ub_ord_cols.assign(cols, cols + P);
  ctx->last_kernel = (cfg->magic_clip && K[1] >= fgt_min2) ? "k_uni_grid<sorted 1-D> + k_fgt_eval (staged)"
                                                           : "k_uni_grid<sorted 1-D> (staged)";
  return TPE_OK;
}

// ---- hypervolume history (tpe_hvhist.cuh) -------------------------------------------------------
// Device memory of one tpe_hypervolume_history call, released when it returns: nothing a suggestion reads is touched.
struct HhScratch {
  DevBuf v, feas, ref, elig, added, list, rank, K, death, incl, cnt, off, clip, keep, surv, m, soff, arena, hv, cum, out;
  ~HhScratch() {
    for (DevBuf* b : {&v, &feas, &ref, &elig, &added, &list, &rank, &K, &death, &incl, &cnt, &off, &clip, &keep, &surv, &m,
                      &soff, &arena, &hv, &cum, &out})
      b->release();
  }
};
// Memory bounds per pass: the clipped fronts of one chunk of added trials (clip and surv each) and the hypervolume
// scratch of one launch.  A single trial that needs more gets a chunk of its own, sized for it.
constexpr size_t kHhClipDoubles = (size_t)1 << 25;
constexpr size_t kHhHvDoubles = (size_t)1 << 26;

int hv_history_run(tpe_ctx* ctx, const double* values, const uint8_t* feasible, int n, int M, const double* ref,
                   double* out) {
  cudaStream_t st = ctx->stream;
  HhScratch s;
  const size_t vb = (size_t)n * M * 8;
  CU(s.v.ensure(vb));
  CU(s.ref.ensure((size_t)M * 8));
  CU(cudaMemcpyAsync(s.v.p, values, vb, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(s.ref.p, ref, (size_t)M * 8, cudaMemcpyHostToDevice, st));
  if (feasible) {
    CU(s.feas.ensure((size_t)n));
    CU(cudaMemcpyAsync(s.feas.p, feasible, (size_t)n, cudaMemcpyHostToDevice, st));
  }
  for (DevBuf* b : {&s.elig, &s.added}) CU(b->ensure((size_t)n));
  for (DevBuf* b : {&s.list, &s.rank}) CU(b->ensure((size_t)n * 4));
  CU(s.K.ensure(4));
  const double* v = s.v.as<double>();
  const double* dref = s.ref.as<double>();
  const int nb = (n + kHhThreads - 1) / kHhThreads;
  k_hh_eligible<<<nb, kHhThreads, 0, st>>>(v, feasible ? s.feas.as<uint8_t>() : nullptr, n, M, dref,
                                           s.elig.as<uint8_t>());
  k_hh_added<<<nb, kHhThreads, hh_added_smem(M), st>>>(v, n, M, s.elig.as<uint8_t>(), s.added.as<uint8_t>());
  k_hh_compact<<<1, 1024, 0, st>>>(s.added.as<uint8_t>(), n, s.list.as<int32_t>(), s.rank.as<int32_t>(),
                                   s.K.as<int32_t>());
  CU(cudaGetLastError());
  int K = 0;
  CU(cudaMemcpyAsync(&K, s.K.p, 4, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  if (K > 0) {
    const int kb = (K + kHhThreads - 1) / kHhThreads;
    for (DevBuf* b : {&s.death, &s.cnt, &s.m}) CU(b->ensure((size_t)K * 4));
    for (DevBuf* b : {&s.incl, &s.hv, &s.cum}) CU(b->ensure((size_t)K * 8));
    k_hh_death<<<kb, kHhThreads, hh_added_smem(M), st>>>(v, n, M, s.list.as<int32_t>(), K, dref,
                                                          s.death.as<int32_t>(), s.incl.as<double>());
    k_hh_count<<<kb, kHhThreads, 0, st>>>(s.list.as<int32_t>(), s.death.as<int32_t>(), K, s.cnt.as<int32_t>());
    CU(cudaGetLastError());
    std::vector<int32_t> cnt((size_t)K), m((size_t)K);
    CU(cudaMemcpyAsync(cnt.data(), s.cnt.p, (size_t)K * 4, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    std::vector<int64_t> off((size_t)K + 1, 0), soff((size_t)K);
    for (int p = 0; p < K; ++p) off[p + 1] = off[p] + cnt[p];
    CU(s.off.ensure((size_t)(K + 1) * 8));
    CU(s.soff.ensure((size_t)K * 8));
    CU(cudaMemcpyAsync(s.off.p, off.data(), (size_t)(K + 1) * 8, cudaMemcpyHostToDevice, st));
    // chunks [pa, pb) of added trials whose clipped fronts fit the bound, sized before any kernel reads them
    std::vector<int> cuts{0};
    size_t rows_max = 1;
    while (cuts.back() < K) {
      const int pa = cuts.back();
      int pb = pa + 1;
      while (pb < K && (size_t)(off[pb + 1] - off[pa]) * M <= kHhClipDoubles) ++pb;
      rows_max = std::max(rows_max, (size_t)(off[pb] - off[pa]));
      cuts.push_back(pb);
    }
    CU(s.clip.ensure(rows_max * M * 8));
    CU(s.surv.ensure(rows_max * M * 8));
    CU(s.keep.ensure(rows_max));
    for (size_t c = 0; c + 1 < cuts.size(); ++c) {
      const int pa = cuts[c], pb = cuts[c + 1];
      k_hh_front<<<(pb - pa + 3) / 4, kHhThreads, 0, st>>>(v, M, s.list.as<int32_t>(), s.death.as<int32_t>(),
                                                           s.cnt.as<int32_t>(), s.off.as<int64_t>(), pa, pb,
                                                           s.clip.as<double>(), s.keep.as<uint8_t>(),
                                                           s.surv.as<double>(), s.m.as<int32_t>());
      CU(cudaGetLastError());
      // (this wait also ends the previous chunk's hypervolume launches, so the arena may be reallocated below)
      CU(cudaMemcpyAsync(m.data() + pa, s.m.as<int32_t>() + pa, (size_t)(pb - pa) * 4, cudaMemcpyDeviceToHost, st));
      CU(cudaStreamSynchronize(st));
      // launches [qa, qb) of this chunk whose hypervolume scratch fits the bound; soff is relative to each launch
      std::vector<std::pair<int, int>> launches;
      size_t need = 0, arena = 1;
      int qa = pa;
      for (int p = pa; p < pb; ++p) {
        const size_t d = (hh_hv_scratch_doubles(m[p], M) + 1) & ~(size_t)1;
        if (p > qa && need + d > kHhHvDoubles) {
          launches.push_back({qa, p});
          qa = p;
          need = 0;
        }
        soff[p] = (int64_t)need;
        need += d;
        arena = std::max(arena, need);
      }
      launches.push_back({qa, pb});
      CU(s.arena.ensure(arena * 8));
      CU(cudaMemcpyAsync(s.soff.as<int64_t>() + pa, soff.data() + pa, (size_t)(pb - pa) * 8, cudaMemcpyHostToDevice, st));
      for (auto& q : launches)
        k_hh_hv<<<(q.second - q.first + 3) / 4, kHhThreads, 0, st>>>(
            M, s.cnt.as<int32_t>(), s.off.as<int64_t>(), pa, q.first, q.second, s.surv.as<double>(),
            s.m.as<int32_t>(), dref, s.soff.as<int64_t>() + pa, s.arena.as<double>(), s.hv.as<double>());
      CU(cudaGetLastError());
    }
    k_hh_scan<<<1, 1, 0, st>>>(K, s.incl.as<double>(), s.hv.as<double>(), s.cum.as<double>());
  }
  CU(s.out.ensure((size_t)n * 8));
  k_hh_fill<<<nb, kHhThreads, 0, st>>>(s.rank.as<int32_t>(), n, K > 0 ? s.cum.as<double>() : nullptr,
                                       s.out.as<double>());
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(out, s.out.p, (size_t)n * 8, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  return TPE_OK;
}

// ---- Pareto front (tpe_pareto.cuh) ---------------------------------------------------------------
// Device memory of one tpe_pareto_front call, released when it returns: nothing a suggestion reads is touched.
struct PfScratch {
  DevBuf v, s, s0, fv, key, idx, work, dom, nf, flags;
  ~PfScratch() {
    for (DevBuf* b : {&v, &s, &s0, &fv, &key, &idx, &work, &dom, &nf, &flags}) b->release();
  }
};

// Pareto-front flags of the device rows d_v [n, M] into b.flags (n >= 1); b's other buffers are sized here
int pareto_front_device(tpe_ctx* ctx, PfScratch& b, const double* d_v, int n, int M) {
  cudaStream_t st = ctx->stream;
  const size_t vb = (size_t)n * M * 8;
  for (DevBuf* x : {&b.s, &b.fv}) CU(x->ensure(vb));
  CU(b.s0.ensure((size_t)n * 8));
  CU(b.key.ensure((size_t)n * 16));
  CU(b.idx.ensure((size_t)n * 12));
  CU(b.work.ensure(sizeof(SortWork)));
  for (DevBuf* x : {&b.dom, &b.flags}) CU(x->ensure((size_t)n));
  CU(b.nf.ensure(4));
  for (DevBuf* x : {&b.dom, &b.flags}) CU(cudaMemsetAsync(x->p, 0, (size_t)n, st));
  CU(cudaMemsetAsync(b.nf.p, 0, 4, st));
  // 1. stable order by coordinate 0
  int32_t pc = M;
  int j_col = 0, n_i = n;
  uint64_t* ka = b.key.as<uint64_t>();
  uint64_t* kb = ka + n;
  int32_t* order = b.idx.as<int32_t>();
  int32_t* ia = order + n;
  int32_t* ib = ia + n;
  SortWork* wk = b.work.as<SortWork>();
  const int* run_flag = nullptr;
  void* args[] = {&d_v, &pc, &j_col, &n_i, &ka, &kb, &ia, &ib, &wk, &order, &run_flag};
  int G = std::max(1, std::min(std::min(ctx->sm_count, 160), (n + 1023) / 1024));
  if (ctx->sort_cta_cap > 0) G = std::min(G, ctx->sort_cta_cap);
  CU(cudaLaunchCooperativeKernel((const void*)k_radix_sort_coop, dim3(G), dim3(512), args, 0, st));
  const int64_t nm = (int64_t)n * M;
  k_pf_gather<<<(unsigned)((nm + 255) / 256), 256, 0, st>>>(d_v, order, n, M, b.s.as<double>(), b.s0.as<double>());
  CU(cudaGetLastError());
  // 2. chunks [cuts[c], cuts[c + 1]) of about kPfChunk sorted rows; a tie run of coordinate 0 (==, so -0.0 ties
  //    with +0.0) is never split
  std::vector<double> s0((size_t)n);
  CU(cudaMemcpyAsync(s0.data(), b.s0.p, (size_t)n * 8, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  std::vector<int> cuts{0};
  while (cuts.back() < n) {
    int c = std::min(n, cuts.back() + kPfChunk);
    while (c < n && s0[c] == s0[c - 1]) ++c;
    cuts.push_back(c);
  }
  // 3. filter and append, chunk by chunk; no host round trip (the front size stays on the device)
  for (size_t c = 0; c + 1 < cuts.size(); ++c) {
    const int c0 = cuts[c], c1 = cuts[c + 1];
    const int n_fslices = (c0 + kPfSlice - 1) / kPfSlice;   // the front holds at most c0 rows
    const int n_slices = n_fslices + (c1 - c0 + kPfSlice - 1) / kPfSlice;
    const dim3 grid((unsigned)((c1 - c0 + kPfThreads - 1) / kPfThreads), (unsigned)std::min(n_slices, 65535));
    k_pf_filter<<<grid, kPfThreads, pf_filter_smem(M), st>>>(b.s.as<double>(), c0, c1, M, b.fv.as<double>(),
                                                             b.nf.as<int>(), n_fslices, b.dom.as<uint8_t>());
    k_pf_append<<<1, 1024, 0, st>>>(b.s.as<double>(), order, c0, c1, M, b.dom.as<uint8_t>(), b.fv.as<double>(),
                                    b.nf.as<int>(), b.flags.as<uint8_t>());
    CU(cudaGetLastError());
  }
  return TPE_OK;
}

int pareto_front_run(tpe_ctx* ctx, const double* values, int n, int M, uint8_t* on_front) {
  cudaStream_t st = ctx->stream;
  PfScratch b;
  const size_t vb = (size_t)n * M * 8;
  CU(b.v.ensure(vb));
  CU(cudaMemcpyAsync(b.v.p, values, vb, cudaMemcpyHostToDevice, st));
  const int rc = pareto_front_device(ctx, b, b.v.as<double>(), n, M);
  if (rc != TPE_OK) return rc;
  CU(cudaMemcpyAsync(on_front, b.flags.p, (size_t)n, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  return TPE_OK;
}

// ---- non-dominated box decomposition (tpe_boxdec.cuh) -------------------------------------------
// bytes of the pool per bound: upper bound, defining points, live flag, and the active list (two), dominated list,
// masks and offsets of k_bd_pass
static size_t bd_bytes_per_bound(int M) { return (size_t)8 * M * (M + 1) + 1 + 5 * 4; }

static int bd_oom(tpe_ctx* ctx, int64_t bounds, int M) {
  cudaGetLastError();   // an allocation failure is not sticky; clear it
  size_t free_b = 0, total_b = 0;
  cudaMemGetInfo(&free_b, &total_b);
  return fail(ctx, TPE_E_INVALID, "box decomposition: a pool of %lld bounds in %d objectives needs %zu bytes of device "
              "memory (%zu free)", (long long)bounds, M, (size_t)bounds * bd_bytes_per_bound(M), free_b);
}

#define BD_ALLOC(buf, bytes, bounds)                                          \
  do {                                                                        \
    cudaError_t e_ = (buf).ensure(bytes);                                     \
    if (e_ == cudaErrorMemoryAllocation) return bd_oom(ctx, (bounds), M);     \
    CU(e_);                                                                   \
  } while (0)

// *count = number of keep[0, n) set, sel[0, *count) their positions (k_bd_select); synchronises
static int bd_select(tpe_ctx* ctx, const uint8_t* keep, int n, int32_t* sel, int* count) {
  BoxDecState& d = ctx->boxdec;
  cudaStream_t st = ctx->stream;
  boxdec::k_bd_select<<<1, boxdec::THREADS, 0, st>>>(keep, n, sel, d.cnt.as<int>());
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(count, d.cnt.p, 4, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  return TPE_OK;
}

// d.front [*nf, M] = the Pareto front of the rows d_rows [n, M] in np.unique(axis=0) order (box_decomposition.py:
// 143-146 and 120-129): a lexicographic order by M stable radix passes, last column first; the rows that differ from
// their predecessor; the Pareto filter of tpe_pareto.cuh over those.  Uses d.sorted, d.key, d.idx, d.work, d.keep,
// d.sel.
static int bd_sorted_front(tpe_ctx* ctx, const double* d_rows, int n, int M, int* nf) {
  BoxDecState& d = ctx->boxdec;
  cudaStream_t st = ctx->stream;
  BD_ALLOC(d.key, (size_t)n * 16, n);
  BD_ALLOC(d.idx, (size_t)n * 20, n);
  BD_ALLOC(d.work, sizeof(SortWork), n);
  BD_ALLOC(d.keep, (size_t)n, n);
  BD_ALLOC(d.sel, (size_t)n * 4, n);
  BD_ALLOC(d.sorted, (size_t)n * M * 8, n);
  uint64_t* ka = d.key.as<uint64_t>();
  uint64_t* kb = ka + n;
  int32_t* ia = d.idx.as<int32_t>();
  int32_t* ib = ia + n;
  int32_t* ord[2] = {ib + n, ib + 2 * n};
  SortWork* wk = d.work.as<SortWork>();
  int G = std::max(1, std::min(std::min(ctx->sm_count, 160), (n + 1023) / 1024));
  if (ctx->sort_cta_cap > 0) G = std::min(G, ctx->sort_cta_cap);
  int32_t pc = M, n_i = n;
  const int32_t* perm = nullptr;
  int32_t* out = nullptr;
  for (int j = M - 1; j >= 0; --j) {
    out = ord[j & 1];
    int j_col = j;
    void* args[] = {&d_rows, &pc, &j_col, &n_i, &ka, &kb, &ia, &ib, &wk, &out, &perm};
    CU(cudaLaunchCooperativeKernel((const void*)k_radix_sort_coop_perm, dim3(G), dim3(512), args, 0, st));
    perm = out;
  }
  const int32_t* order = out;
  boxdec::k_bd_unique<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_rows, order, n, M, d.keep.as<uint8_t>());
  CU(cudaGetLastError());
  int nu = 0;
  int rc = bd_select(ctx, d.keep.as<uint8_t>(), n, d.sel.as<int32_t>(), &nu);
  if (rc != TPE_OK) return rc;
  const int64_t nm = (int64_t)nu * M;
  boxdec::k_bd_gather<<<(unsigned)((nm + 255) / 256), 256, 0, st>>>(d_rows, order, d.sel.as<int32_t>(), nu, M, false,
                                                                    d.sorted.as<double>());
  CU(cudaGetLastError());
  PfScratch pf;
  rc = pareto_front_device(ctx, pf, d.sorted.as<double>(), nu, M);
  if (rc != TPE_OK) return rc;
  rc = bd_select(ctx, pf.flags.as<uint8_t>(), nu, d.sel.as<int32_t>(), nf);
  if (rc != TPE_OK) return rc;
  BD_ALLOC(d.front, (size_t)*nf * M * 8, n);
  const int64_t fm = (int64_t)*nf * M;
  boxdec::k_bd_gather<<<(unsigned)((fm + 255) / 256), 256, 0, st>>>(d.sorted.as<double>(), nullptr, d.sel.as<int32_t>(),
                                                                    *nf, M, false, d.front.as<double>());
  CU(cudaGetLastError());
  return TPE_OK;
}

// one _get_upper_bound_set pass over d.front [nf, M] from d.ref: the pool's first *pool bounds, *live_n of them live
// and listed in d.sel.  A pass that overflows the pool is run again on a pool four times larger.
static int bd_pass(tpe_ctx* ctx, int nf, int M, int* pool, int* live_n) {
  BoxDecState& d = ctx->boxdec;
  cudaStream_t st = ctx->stream;
  if (d.cap == 0) d.cap = 4096;
  for (;;) {
    const int64_t cap = d.cap;
    BD_ALLOC(d.ub, (size_t)cap * M * 8, cap);
    BD_ALLOC(d.dp, (size_t)cap * M * M * 8, cap);
    BD_ALLOC(d.live, (size_t)cap, cap);
    BD_ALLOC(d.act, (size_t)cap * 8, cap);
    BD_ALLOC(d.dlist, (size_t)cap * 4, cap);
    BD_ALLOC(d.dmask, (size_t)cap * 4, cap);
    BD_ALLOC(d.doff, (size_t)cap * 4, cap);
    BD_ALLOC(d.sel, (size_t)cap * 4, cap);
    BD_ALLOC(d.keep, (size_t)cap, cap);
    int32_t* act = d.act.as<int32_t>();
    boxdec::k_bd_pass<<<1, boxdec::THREADS, 0, st>>>(d.front.as<double>(), nf, M, d.ref.as<double>(), d.ub.as<double>(),
                                                     d.dp.as<double>(), d.live.as<uint8_t>(), act, act + cap,
                                                     d.dlist.as<int32_t>(), d.dmask.as<uint32_t>(),
                                                     d.doff.as<int32_t>(), (int)cap, d.stat.as<int>());
    CU(cudaGetLastError());
    int stat[2];
    CU(cudaMemcpyAsync(stat, d.stat.p, 8, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    if (stat[1] == 0) {
      *pool = stat[0];
      return bd_select(ctx, d.live.as<uint8_t>(), stat[0], d.sel.as<int32_t>(), live_n);
    }
    if (cap >= INT32_MAX / 4) return bd_oom(ctx, cap * 4, M);
    d.cap = cap * 4;
  }
}

// get_non_dominated_box_bounds (box_decomposition.py:138-157) of d.rows [n, M] against ref [M]: d.lower, d.upper
static int bd_run(tpe_ctx* ctx, int n, int M, const double* ref) {
  BoxDecState& d = ctx->boxdec;
  cudaStream_t st = ctx->stream;
  CU(d.ref.ensure((size_t)M * 8));
  CU(d.cnt.ensure(4));
  CU(d.stat.ensure(8));
  // 1. the front of the unique-lexsorted rows; 2. pass 1
  int nf1 = 0, pool1 = 0, live1 = 0;
  int rc = bd_sorted_front(ctx, d.rows.as<double>(), n, M, &nf1);
  if (rc != TPE_OK) return rc;
  CU(cudaMemcpyAsync(d.ref.p, ref, (size_t)M * 8, cudaMemcpyHostToDevice, st));
  rc = bd_pass(ctx, nf1, M, &pool1, &live1);
  if (rc != TPE_OK) return rc;
  // 3. the negated upper bounds, their unique-lexsorted front; 4. pass 2 from +inf
  BD_ALLOC(d.rows, (size_t)live1 * M * 8, live1);
  const int64_t lm = (int64_t)live1 * M;
  boxdec::k_bd_gather<<<(unsigned)((lm + 255) / 256), 256, 0, st>>>(d.ub.as<double>(), nullptr, d.sel.as<int32_t>(),
                                                                    live1, M, true, d.rows.as<double>());
  CU(cudaGetLastError());
  int nf2 = 0, pool2 = 0, live2 = 0;
  rc = bd_sorted_front(ctx, d.rows.as<double>(), live1, M, &nf2);
  if (rc != TPE_OK) return rc;
  const std::vector<double> inf((size_t)M, INFINITY);
  CU(cudaMemcpyAsync(d.ref.p, inf.data(), (size_t)M * 8, cudaMemcpyHostToDevice, st));
  rc = bd_pass(ctx, nf2, M, &pool2, &live2);
  if (rc != TPE_OK) return rc;
  // 5. the boxes of the final bounds, the empty ones dropped
  // (lo and hi hold the boxes of every final bound, then the kept ones behind them)
  BD_ALLOC(d.lo, (size_t)live2 * M * 16, live2);
  BD_ALLOC(d.hi, (size_t)live2 * M * 16, live2);
  double* lo = d.lo.as<double>();
  double* hi = d.hi.as<double>();
  boxdec::k_bd_boxes<<<(unsigned)((live2 + 255) / 256), 256, 0, st>>>(d.ub.as<double>(), d.dp.as<double>(),
                                                                      d.sel.as<int32_t>(), live2, M, lo, hi,
                                                                      d.keep.as<uint8_t>());
  CU(cudaGetLastError());
  int B = 0;
  rc = bd_select(ctx, d.keep.as<uint8_t>(), live2, d.sel.as<int32_t>(), &B);
  if (rc != TPE_OK) return rc;
  d.lower.assign((size_t)B * M, 0.0);
  d.upper.assign((size_t)B * M, 0.0);
  if (B > 0) {
    const int64_t bm = (int64_t)B * M;
    const unsigned g = (unsigned)((bm + 255) / 256);
    double* lo_kept = lo + (size_t)live2 * M;
    double* hi_kept = hi + (size_t)live2 * M;
    boxdec::k_bd_gather<<<g, 256, 0, st>>>(lo, nullptr, d.sel.as<int32_t>(), B, M, false, lo_kept);
    boxdec::k_bd_gather<<<g, 256, 0, st>>>(hi, nullptr, d.sel.as<int32_t>(), B, M, false, hi_kept);
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(d.lower.data(), lo_kept, (size_t)bm * 8, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(d.upper.data(), hi_kept, (size_t)bm * 8, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
  }
  const int64_t stats[6] = {nf1, pool1 - 1, live1, nf2, pool2 - 1, live2};
  std::copy(stats, stats + 6, d.stats);
  return TPE_OK;
}

// ---- fANOVA variances (tpe_fanova.cuh) -----------------------------------------------------------
// Device memory of one tpe_fanova_variances call, released when it returns: nothing a suggestion reads is touched.
struct FaScratch {
  DevBuf off, left, right, feat, thr, val, parent, tree_of, bounds, fparam, po, cols, stat, mask, tvar, mvar;
  DevBuf box, lvl, key1, key2, k2s, key, idx, work, so, ebuf, mp, sz, K, acc_off, acc;
  ~FaScratch() {
    for (DevBuf* b : {&off, &left, &right, &feat, &thr, &val, &parent, &tree_of, &bounds, &fparam, &po, &cols, &stat,
                      &mask, &tvar, &mvar, &box, &lvl, &key1, &key2, &k2s, &key, &idx, &work, &so, &ebuf, &mp, &sz,
                      &K, &acc_off, &acc})
      b->release();
  }
};

constexpr size_t kFaBoxBudget = (size_t)1 << 30;   // bytes of per-node boxes (nodes x F x 16) per chunk of trees

// The validated forest: global child / parent indices (-1: none), the tree and depth of every node.
struct FaForest {
  std::vector<int32_t> left, right, parent, tree_of, depth;
};

// The host checks of tpe_fanova_variances; fills fo.  Returns TPE_OK or TPE_E_INVALID (message in ctx).
int fanova_validate(tpe_ctx* ctx, int T, const int64_t* off, const int32_t* left, const int32_t* right,
                    const int32_t* feature, const double* thr, int F, const double* bounds, int n_params,
                    const int32_t* po, const int32_t* cols, FaForest& fo) {
  if (off[0] != 0) return fail(ctx, TPE_E_INVALID, "node_offsets[0] must be 0");
  for (int t = 0; t < T; ++t)
    if (off[t + 1] <= off[t]) return fail(ctx, TPE_E_INVALID, "tree %d has no nodes", t);
  const int64_t N = off[T];
  if (N >= (1ll << 31) - 1) return fail(ctx, TPE_E_INVALID, "too many nodes (%lld)", (long long)N);
  for (int f = 0; f < F; ++f)
    if (!(bounds[2 * f] <= bounds[2 * f + 1])) return fail(ctx, TPE_E_INVALID, "bad bounds of feature %d", f);
  if (po[0] != 0) return fail(ctx, TPE_E_INVALID, "param_offsets[0] must be 0");
  std::vector<uint8_t> used((size_t)F, 0);
  for (int p = 0; p < n_params; ++p) {
    if (po[p + 1] <= po[p]) return fail(ctx, TPE_E_INVALID, "parameter %d has no raw features", p);
    for (int j = po[p]; j < po[p + 1]; ++j) {
      if (cols[j] < 0 || cols[j] >= F || used[cols[j]])
        return fail(ctx, TPE_E_INVALID, "raw feature %d of parameter %d is out of range or repeated", cols[j], p);
      used[cols[j]] = 1;
    }
  }
  fo.left.assign((size_t)N, -1);
  fo.right.assign((size_t)N, -1);
  fo.parent.assign((size_t)N, -1);
  fo.tree_of.resize((size_t)N);
  fo.depth.assign((size_t)N, 0);
  for (int t = 0; t < T; ++t) {
    const int64_t a = off[t], n_t = off[t + 1] - a;
    for (int64_t i = 0; i < n_t; ++i) {
      const int64_t g = a + i;
      fo.tree_of[g] = t;
      const int f = feature[g];
      if (f < 0) continue;
      if (f >= F) return fail(ctx, TPE_E_INVALID, "tree %d node %lld splits on feature %d >= %d", t, (long long)i, f, F);
      const double th = thr[g];
      if (std::isnan(th) || th < bounds[2 * f] || th > bounds[2 * f + 1])
        return fail(ctx, TPE_E_INVALID, "tree %d node %lld: threshold is NaN or outside its feature's bounds", t,
                    (long long)i);
      for (int32_t c : {left[g], right[g]}) {
        if (c <= i || c >= n_t)
          return fail(ctx, TPE_E_INVALID, "tree %d node %lld: child %d is not in (%lld, %lld)", t, (long long)i, c,
                      (long long)i, (long long)n_t);
        if (fo.parent[a + c] >= 0)
          return fail(ctx, TPE_E_INVALID, "tree %d node %d has two parents", t, c);
        fo.parent[a + c] = (int32_t)g;
        fo.depth[a + c] = fo.depth[g] + 1;
      }
      if (left[g] == right[g]) return fail(ctx, TPE_E_INVALID, "tree %d node %lld: equal children", t, (long long)i);
      fo.left[g] = (int32_t)(a + left[g]);
      fo.right[g] = (int32_t)(a + right[g]);
    }
    for (int64_t i = 1; i < n_t; ++i)
      if (fo.parent[a + i] < 0) return fail(ctx, TPE_E_INVALID, "tree %d node %lld has no parent", t, (long long)i);
  }
  return TPE_OK;
}

int fanova_run(tpe_ctx* ctx, int T, const int64_t* off, const FaForest& fo, const int32_t* feature, const double* thr,
               const double* value, int F, const double* bounds, int n_params, const int32_t* po,
               const int32_t* cols, double* tree_var, double* marginal_var) {
  cudaStream_t st = ctx->stream;
  FaScratch b;
  const int64_t N = off[T];
  const int n_cols = po[n_params];
  const int n_words = std::max(1, (n_params + 63) / 64);
  std::vector<int32_t> fparam((size_t)F, -1);
  for (int p = 0; p < n_params; ++p)
    for (int j = po[p]; j < po[p + 1]; ++j) fparam[cols[j]] = p;
  auto up = [&](DevBuf& d, const void* h, size_t bytes) -> cudaError_t {
    cudaError_t e = d.ensure(std::max<size_t>(bytes, 8));
    if (e == cudaSuccess && bytes) e = cudaMemcpyAsync(d.p, h, bytes, cudaMemcpyHostToDevice, st);
    return e;
  };
  CU(up(b.off, off, (size_t)(T + 1) * 8));
  CU(up(b.left, fo.left.data(), (size_t)N * 4));
  CU(up(b.right, fo.right.data(), (size_t)N * 4));
  CU(up(b.parent, fo.parent.data(), (size_t)N * 4));
  CU(up(b.tree_of, fo.tree_of.data(), (size_t)N * 4));
  CU(up(b.feat, feature, (size_t)N * 4));
  CU(up(b.thr, thr, (size_t)N * 8));
  CU(up(b.val, value, (size_t)N * 8));
  CU(up(b.bounds, bounds, (size_t)F * 16));
  CU(up(b.fparam, fparam.data(), (size_t)F * 4));
  CU(up(b.po, po, (size_t)(n_params + 1) * 4));
  CU(up(b.cols, cols, (size_t)n_cols * 4));
  CU(b.stat.ensure((size_t)N * 16));
  CU(b.mask.ensure((size_t)N * n_words * 8));
  CU(b.tvar.ensure((size_t)T * 8));
  CU(b.mvar.ensure((size_t)std::max(1, n_params) * T * 8));
  CU(b.work.ensure(sizeof(SortWork)));
  const int32_t* d_feat = b.feat.as<int32_t>();
  const double* d_thr = b.thr.as<double>();
  const double2* d_bounds = b.bounds.as<double2>();
  std::vector<int32_t> lvl;
  std::vector<int64_t> lvl_off, so;
  std::vector<int32_t> Kh;
  std::vector<int64_t> acc_off;
  for (int t0 = 0; t0 < T;) {
    // 0. a chunk [t0, t1) of trees whose boxes fit kFaBoxBudget (at least one tree)
    int t1 = t0 + 1;
    while (t1 < T && (size_t)(off[t1 + 1] - off[t0]) * F * 16 <= kFaBoxBudget) ++t1;
    const int Tc = t1 - t0, n_seg = Tc * F;
    const int64_t base = off[t0];
    const int cnt = (int)(off[t1] - base);
    // nodes by depth (counting sort) and internal nodes per (tree, feature) segment
    int max_d = 0;
    for (int i = 0; i < cnt; ++i) max_d = std::max(max_d, fo.depth[base + i]);
    lvl_off.assign((size_t)max_d + 2, 0);
    so.assign((size_t)n_seg + 1, 0);
    for (int i = 0; i < cnt; ++i) {
      ++lvl_off[fo.depth[base + i] + 1];
      if (feature[base + i] >= 0) ++so[(size_t)(fo.tree_of[base + i] - t0) * F + feature[base + i] + 1];
    }
    for (int d = 0; d <= max_d; ++d) lvl_off[d + 1] += lvl_off[d];
    for (int s = 0; s < n_seg; ++s) so[s + 1] += so[s];
    lvl.resize((size_t)cnt);
    {
      std::vector<int64_t> at(lvl_off.begin(), lvl_off.end() - 1);
      for (int i = 0; i < cnt; ++i) lvl[at[fo.depth[base + i]]++] = (int32_t)(base + i);
    }
    CU(up(b.lvl, lvl.data(), (size_t)cnt * 4));
    CU(up(b.so, so.data(), (size_t)(n_seg + 1) * 8));
    CU(b.box.ensure((size_t)cnt * F * 16));
    // 1-2. boxes top-down, leaves, statistics and subtree parameter masks bottom-up
    for (int d = 0; d <= max_d; ++d) {
      const int n_l = (int)(lvl_off[d + 1] - lvl_off[d]);
      const int64_t work = (int64_t)n_l * F;
      k_fa_down<<<(unsigned)((work + 255) / 256), 256, 0, st>>>(b.lvl.as<int32_t>() + lvl_off[d], n_l, base,
                                                               b.parent.as<int32_t>(), b.left.as<int32_t>(), d_feat,
                                                               d_thr, d_bounds, F, b.box.as<double2>());
    }
    k_fa_leaf<<<(cnt + 255) / 256, 256, 0, st>>>(base, cnt, d_feat, b.val.as<double>(), b.box.as<double2>(), F, n_words,
                                                  b.stat.as<double2>(), b.mask.as<uint64_t>());
    for (int d = max_d; d >= 0; --d) {
      const int n_l = (int)(lvl_off[d + 1] - lvl_off[d]);
      k_fa_up<<<(n_l + 255) / 256, 256, 0, st>>>(b.lvl.as<int32_t>() + lvl_off[d], n_l, b.left.as<int32_t>(),
                                                 b.right.as<int32_t>(), d_feat, b.fparam.as<int32_t>(), n_words,
                                                 b.stat.as<double2>(), b.mask.as<uint64_t>());
    }
    CU(cudaGetLastError());
    // 3. tree variances
    k_fa_tree_var<<<Tc, kFaThreads, 0, st>>>(b.off.as<int64_t>(), t0, d_feat, b.stat.as<double2>(),
                                             b.tvar.as<double>());
    // 4. (tree, feature, threshold) order by two stable radix sorts, then the midpoints of every segment
    for (DevBuf* x : {&b.key1, &b.key2, &b.k2s}) CU(x->ensure((size_t)cnt * 8));
    CU(b.key.ensure((size_t)cnt * 16));
    CU(b.idx.ensure((size_t)cnt * 16));
    k_fa_keys<<<(cnt + 255) / 256, 256, 0, st>>>(base, cnt, t0, n_seg, b.tree_of.as<int32_t>(), d_feat, d_thr, F,
                                                  b.key1.as<double>(), b.key2.as<double>());
    CU(cudaGetLastError());
    int32_t* order1 = b.idx.as<int32_t>();
    int32_t* order2 = order1 + cnt;
    auto sort = [&](const double* keys, int32_t* order) -> cudaError_t {
      int32_t pc = 1;
      int j_col = 0, n_i = cnt;
      uint64_t* ka = b.key.as<uint64_t>();
      uint64_t* kb = ka + cnt;
      int32_t* ia = order2 + cnt;
      int32_t* ib = ia + cnt;
      SortWork* wk = b.work.as<SortWork>();
      const int* run_flag = nullptr;
      void* args[] = {&keys, &pc, &j_col, &n_i, &ka, &kb, &ia, &ib, &wk, &order, &run_flag};
      int G = std::max(1, std::min(std::min(ctx->sm_count, 160), (cnt + 1023) / 1024));
      if (ctx->sort_cta_cap > 0) G = std::min(G, ctx->sort_cta_cap);
      return cudaLaunchCooperativeKernel((const void*)k_radix_sort_coop, dim3(G), dim3(512), args, 0, st);
    };
    CU(sort(b.key1.as<double>(), order1));
    k_fa_gather<<<(cnt + 255) / 256, 256, 0, st>>>(order1, cnt, b.key2.as<double>(), b.k2s.as<double>());
    CU(sort(b.k2s.as<double>(), order2));
    const int64_t n_int = so[n_seg];
    CU(b.ebuf.ensure((size_t)(n_int + 2 * n_seg) * 8));
    CU(b.mp.ensure((size_t)(n_int + n_seg) * 8));
    CU(b.sz.ensure((size_t)(n_int + n_seg) * 8));
    CU(b.K.ensure((size_t)n_seg * 4));
    k_fa_midpoints<<<n_seg, 1024, 0, st>>>(base, order1, order2, b.so.as<int64_t>(), d_thr, d_bounds, F,
                                           b.ebuf.as<double>(), b.mp.as<double>(), b.sz.as<double>(),
                                           b.K.as<int32_t>());
    CU(cudaGetLastError());
    Kh.resize((size_t)n_seg);
    CU(cudaMemcpyAsync(Kh.data(), b.K.p, (size_t)n_seg * 4, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    if (n_params == 0) {
      t0 = t1;
      continue;
    }
    // 5. accumulator of every (tree, parameter): a segment tree for one column, the grid for several
    acc_off.assign((size_t)Tc * n_params + 1, 0);
    for (int tl = 0; tl < Tc; ++tl)
      for (int p = 0; p < n_params; ++p) {
        int64_t cells = 1;
        for (int j = po[p]; j < po[p + 1] && cells <= kFaMaxCells; ++j) cells *= Kh[(size_t)tl * F + cols[j]];
        if (cells > kFaMaxCells)
          return fail(ctx, TPE_E_INVALID,
                      "parameter %d: tree %d splits its %d raw features into more than 2^20 grid cells", p, t0 + tl,
                      po[p + 1] - po[p]);
        int64_t sz_acc = cells;
        if (po[p + 1] - po[p] == 1) {
          int64_t P = 1;
          while (P < cells) P <<= 1;
          sz_acc = 2 * P;
        }
        acc_off[(size_t)tl * n_params + p + 1] = acc_off[(size_t)tl * n_params + p] + sz_acc;
      }
    CU(up(b.acc_off, acc_off.data(), acc_off.size() * 8));
    CU(b.acc.ensure((size_t)acc_off.back() * 16));
    CU(cudaMemsetAsync(b.acc.p, 0, (size_t)acc_off.back() * 16, st));
    k_fa_marginal<<<dim3((unsigned)n_params, (unsigned)Tc), kFaThreads, 0, st>>>(
        b.off.as<int64_t>(), t0, base, n_params, b.po.as<int32_t>(), b.cols.as<int32_t>(), b.parent.as<int32_t>(),
        b.stat.as<double2>(), b.mask.as<uint64_t>(), n_words, b.box.as<double2>(), F, b.so.as<int64_t>(),
        b.mp.as<double>(), b.sz.as<double>(), b.K.as<int32_t>(), b.acc_off.as<int64_t>(), b.acc.as<double2>(),
        b.mvar.as<double>(), T);
    CU(cudaGetLastError());
    // the next chunk overwrites the host vectors the pending copies read
    CU(cudaStreamSynchronize(st));
    t0 = t1;
  }
  CU(cudaMemcpyAsync(tree_var, b.tvar.p, (size_t)T * 8, cudaMemcpyDeviceToHost, st));
  if (n_params > 0)
    CU(cudaMemcpyAsync(marginal_var, b.mvar.p, (size_t)n_params * T * 8, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  return TPE_OK;
}


// =================================================================================================
extern "C" {

int tpe_abi_version(void) { return TPE_ABI_VERSION; }

int tpe_ctx_create(int device, tpe_ctx** out) {
  if (!out) return TPE_E_INVALID;
  *out = nullptr;
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || device < 0 || device >= count) return TPE_E_CUDA;
  tpe_ctx* ctx = new tpe_ctx();
  ctx->device = device;
  if (cudaSetDevice(device) != cudaSuccess ||
      cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess ||
      cudaStreamCreateWithFlags(&ctx->stream2, cudaStreamNonBlocking) != cudaSuccess ||
      cudaStreamCreateWithFlags(&ctx->stream3, cudaStreamNonBlocking) != cudaSuccess) {
    delete ctx;
    return TPE_E_CUDA;
  }
  for (auto& e : ctx->ev) cudaEventCreate(&e);
  cudaEventCreateWithFlags(&ctx->ev_fork, cudaEventDisableTiming);
  cudaEventCreateWithFlags(&ctx->ev_join, cudaEventDisableTiming);
  cudaEventCreateWithFlags(&ctx->ev_u, cudaEventDisableTiming);
  cudaEventCreateWithFlags(&ctx->ev_spec, cudaEventDisableTiming);
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) ctx->sm_count = prop.multiProcessorCount;
  void* mh = nullptr;
  if (cudaHostAlloc(&mh, 625 * 4, cudaHostAllocDefault) != cudaSuccess) {
    tpe_ctx_destroy(ctx);
    return TPE_E_NOMEM;
  }
  memset(mh, 0, 625 * 4);
  ctx->mt_host = static_cast<uint32_t*>(mh);
  *out = ctx;
  return TPE_OK;
}

void tpe_ctx_destroy(tpe_ctx* ctx) {
  if (!ctx) return;
  for (tpe_ctx* c : ctx->uni_sub) tpe_ctx_destroy(c);
  ctx->uni_sub.clear();
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  if (ctx->stream2) cudaStreamSynchronize(ctx->stream2);
  if (ctx->stream3) cudaStreamSynchronize(ctx->stream3);
  for (DevBuf* b : {&ctx->cat_dist, &ctx->X, &ctx->cat, &ctx->key, &ctx->vals, &ctx->mo_list, &ctx->mo_alive, &ctx->mo_dom,
                    &ctx->mo_first, &ctx->mo_rank, &ctx->mo_ctr, &ctx->mo_tie, &ctx->mo_ntie, &ctx->mo_lexpos,
                    &ctx->mo_isdup, &ctx->mo_sorted, &ctx->mo_uniq, &ctx->mo_nuniq, &ctx->mo_ref, &ctx->mo_removed, &ctx->mo_table,
                    &ctx->mo_sample, &ctx->mo_surv, &ctx->mo_nsurv, &ctx->mo_fv, &ctx->mo_ps, &ctx->mo_map, &ctx->mo_front, &ctx->mo_head,
                    &ctx->mo_contrib, &ctx->mo_bound, &ctx->mo_state, &ctx->mo_arena, &ctx->mo_chosen, &ctx->mo_diag, &ctx->mo_w, &ctx->cols, &ctx->row_ok, &ctx->member,
                    &ctx->counts, &ctx->split_work, &ctx->below_all, &ctx->kpart, &ctx->mixcols, &ctx->ub_arena, &ctx->ub_ord_a, &ctx->ub_ord_b, &ctx->ub_wstage, &ctx->uxs, &ctx->ucidx, &ctx->uni_prev_rows, &ctx->uni_mode, &ctx->uni_work, &ctx->sort_val, &ctx->sort_idx, &ctx->sort_work, &ctx->U, &ctx->S,
                    &ctx->xT, &ctx->x64s, &ctx->x32s, &ctx->e32s, &ctx->gmax, &ctx->lse_gmax, &ctx->mt_state, &ctx->U2, &ctx->mt_spec, &ctx->mt_jump, &ctx->mt_tmp, &ctx->oob, &ctx->logl, &ctx->logg, &ctx->out_x, &ctx->out_acq, &ctx->out_best})
    b->release();
  ctx->est[0].release();
  ctx->est[1].release();
  ctx->gp.release();
  ctx->gpb.release();
  ctx->ehvi.release();
  ctx->acqf.release();
  ctx->boxdec.release();
  if (ctx->res_host) cudaFreeHost(ctx->res_host);
  if (ctx->mt_host) cudaFreeHost(ctx->mt_host);
  if (ctx->up_host) cudaFreeHost(ctx->up_host);
  for (auto& e : ctx->up_ev)
    if (e) cudaEventDestroy(e);
  for (auto& e : ctx->ev)
    if (e) cudaEventDestroy(e);
  if (ctx->ev_fork) cudaEventDestroy(ctx->ev_fork);
  if (ctx->ev_join) cudaEventDestroy(ctx->ev_join);
  if (ctx->ev_u) cudaEventDestroy(ctx->ev_u);
  if (ctx->ev_spec) cudaEventDestroy(ctx->ev_spec);
  if (ctx->ev_uni) cudaEventDestroy(ctx->ev_uni);
  if (ctx->stream2) cudaStreamDestroy(ctx->stream2);
  if (ctx->stream3) cudaStreamDestroy(ctx->stream3);
  cudaStreamDestroy(ctx->stream);
  delete ctx;
}

const char* tpe_last_error(tpe_ctx* ctx) { return ctx ? ctx->err.c_str() : "null context"; }

int tpe_space_set(tpe_ctx* ctx, const tpe_param_desc* params, int32_t n_params, const double* cat_dist,
                  const int64_t* cat_dist_offset) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (!params || n_params <= 0) return fail(ctx, TPE_E_INVALID, "space must hold at least one parameter");
  if (set_device(ctx)) return TPE_E_CUDA;
  for (int i = 0; i < n_params; ++i) {
    const tpe_param_desc& d = params[i];
    if (d.kind == TPE_KIND_CAT) {
      if (d.n_choices < 1) return fail(ctx, TPE_E_INVALID, "param %d: categorical needs n_choices >= 1", i);
    } else if (d.kind == TPE_KIND_FLOAT || d.kind == TPE_KIND_INT) {
      if (!(d.low <= d.high)) return fail(ctx, TPE_E_INVALID, "param %d: low <= high must hold", i);
      if (d.kind == TPE_KIND_INT && !d.has_step) return fail(ctx, TPE_E_INVALID, "param %d: int needs a step", i);
      if (d.has_step && !(d.step > 0)) return fail(ctx, TPE_E_INVALID, "param %d: step > 0 must hold", i);
      if (d.log && d.kind == TPE_KIND_FLOAT && d.has_step)
        return fail(ctx, TPE_E_INVALID, "param %d: step is not supported when log is true", i);
      if (d.log && !(d.low - (d.has_step ? d.step / 2 : 0.0) > 0))
        return fail(ctx, TPE_E_INVALID, "param %d: low > 0 must hold for log", i);
    } else {
      return fail(ctx, TPE_E_INVALID, "param %d: unknown kind %d", i, d.kind);
    }
  }
  ctx->space.assign(params, params + n_params);
  ctx->cat_dist_off.assign(n_params, -1);
  ctx->cat_dist_h.clear();
  if (cat_dist && cat_dist_offset) {
    int64_t end = 0;
    for (int i = 0; i < n_params; ++i) {
      ctx->cat_dist_off[i] = cat_dist_offset[i];
      if (cat_dist_offset[i] >= 0)
        end = std::max<int64_t>(end, cat_dist_offset[i] + (int64_t)params[i].n_choices * params[i].n_choices);
    }
    ctx->cat_dist_h.assign(cat_dist, cat_dist + end);
    CU(ctx->cat_dist.ensure((size_t)std::max<int64_t>(end, 1) * 8));
    if (end) CU(cudaMemcpy(ctx->cat_dist.p, cat_dist, (size_t)end * 8, cudaMemcpyHostToDevice));
  }
  ctx->col_missing.assign(n_params, 0);
  ctx->col_oor.assign(n_params, 0);
  ctx->col_offgrid.assign(n_params, 0);
  ctx->hist_lineage++;
  ctx->N = 0;
  ctx->history_set = false;
  ctx->prepared = ctx->built = ctx->sampled = false;
  ctx->hist_version++;
  return TPE_OK;
}

int tpe_history_set(tpe_ctx* ctx, const double* X, const int8_t* category, const double* key, int64_t n) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (ctx->space.empty()) return fail(ctx, TPE_E_STATE, "tpe_space_set must precede tpe_history_set");
  if (n < 0 || (n > 0 && (!X || !category || !key))) return fail(ctx, TPE_E_INVALID, "bad history arguments");
  if (n >= (1ll << 31) - 4096) return fail(ctx, TPE_E_INVALID, "history too long");
  if (set_device(ctx)) return TPE_E_CUDA;
  std::fill(ctx->col_missing.begin(), ctx->col_missing.end(), 0);
  std::fill(ctx->col_oor.begin(), ctx->col_oor.end(), 0);
  std::fill(ctx->col_offgrid.begin(), ctx->col_offgrid.end(), 0);
  ctx->hist_lineage++;
  scan_missing(ctx, X, category, n);
  return upload_history(ctx, X, category, key, n, 0, false);
}

int tpe_history_append(tpe_ctx* ctx, const double* X, const int8_t* category, const double* key, int64_t n) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (ctx->space.empty()) return fail(ctx, TPE_E_STATE, "tpe_space_set must precede tpe_history_append");
  if (n < 0 || (n > 0 && (!X || !category || !key))) return fail(ctx, TPE_E_INVALID, "bad history arguments");
  if (ctx->N + n >= (1ll << 31) - 4096) return fail(ctx, TPE_E_INVALID, "history too long");
  if (set_device(ctx)) return TPE_E_CUDA;
  scan_missing(ctx, X, category, n);
  return upload_history(ctx, X, category, key, n, ctx->N, false);
}

int tpe_history_update(tpe_ctx* ctx, const double* X, const int8_t* category, const double* key, int64_t n,
                       int64_t at_row) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (!ctx->history_set) return fail(ctx, TPE_E_STATE, "tpe_history_set must precede tpe_history_update");
  if (n < 0 || at_row < 0 || at_row > ctx->N || (n > 0 && (!X || !category || !key)))
    return fail(ctx, TPE_E_INVALID, "tpe_history_update: rows [%lld, %lld) do not continue the history of %lld rows",
                (long long)at_row, (long long)(at_row + n), (long long)ctx->N);
  if (n == 0) return TPE_OK;
  if (at_row + n >= (1ll << 31) - 4096) return fail(ctx, TPE_E_INVALID, "history too long");
  if (set_device(ctx)) return TPE_E_CUDA;
  if ((int64_t)ctx->cat_h.size() != ctx->N)
    return fail(ctx, TPE_E_STATE, "tpe_history_update needs a host-uploaded history");
  scan_missing(ctx, X, category, n);
  const int64_t P = (int64_t)ctx->space.size();
  const int64_t total = std::max(ctx->N, at_row + n);
  if (total > ctx->N) {  // the write runs past the end: the history grows (rows [at_row, N) are overwritten)
    CU(ctx->X.grow((size_t)total * P * 8, (size_t)ctx->N * P * 8, ctx->stream));
    CU(ctx->cat.grow((size_t)total, (size_t)ctx->N, ctx->stream));
    CU(ctx->key.grow((size_t)total * 16, (size_t)ctx->N * 16, ctx->stream));
    if (ctx->M >= 2)
      CU(ctx->vals.grow((size_t)total * ctx->M * 8, (size_t)ctx->N * ctx->M * 8, ctx->stream));
  }
  if (rows_fit_staging(ctx, n)) {
    if (int rc = stage_rows(ctx, X, category, key, n, at_row)) return rc;
  } else {
    CU(cudaMemcpyAsync(ctx->X.as<double>() + at_row * P, X, (size_t)n * P * 8, cudaMemcpyHostToDevice, ctx->stream));
    CU(cudaMemcpyAsync(ctx->cat.as<int8_t>() + at_row, category, (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
    CU(cudaMemcpyAsync(ctx->key.as<double>() + at_row * 2, key, (size_t)n * 16, cudaMemcpyHostToDevice, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
  }
  ctx->cat_h.resize((size_t)total, (int8_t)TPE_CAT_EXCLUDED);
  for (int64_t i = 0; i < n; ++i) {
    const int64_t r = at_row + i;
    if (r < ctx->N) {
      if (cat_slot(ctx->cat_h[(size_t)r]) != 4) ctx->hist_lineage++;   // a row the estimators could see is replaced
      ctx->cat_cnt[cat_slot(ctx->cat_h[(size_t)r])]--;
    }
    ctx->cat_h[(size_t)r] = category[i];
    ctx->cat_cnt[cat_slot(category[i])]++;
  }
  ctx->N = total;
  ctx->prepared = ctx->built = ctx->sampled = false;
  ctx->hist_version++;
  return TPE_OK;
}

int tpe_history_set_device(tpe_ctx* ctx, const double* dX, const int8_t* dcategory, const double* dkey, int64_t n,
                           const uint8_t* col_has_missing) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (ctx->space.empty()) return fail(ctx, TPE_E_STATE, "tpe_space_set must precede tpe_history_set_device");
  if (n < 0 || (n > 0 && (!dX || !dcategory || !dkey))) return fail(ctx, TPE_E_INVALID, "bad history arguments");
  if (set_device(ctx)) return TPE_E_CUDA;
  ctx->hist_lineage++;
  for (size_t j = 0; j < ctx->col_missing.size(); ++j) ctx->col_missing[j] = col_has_missing ? col_has_missing[j] : 1;
  // a history adopted from device memory is not scanned on the host: treat every column as possibly out of range
  // unless the caller vouches for it through col_has_missing (the broadcast path of optuna_b200/dist.py does)
  std::fill(ctx->col_oor.begin(), ctx->col_oor.end(), col_has_missing ? 0 : 1);
  std::fill(ctx->col_offgrid.begin(), ctx->col_offgrid.end(), col_has_missing ? 0 : 1);
  return upload_history(ctx, dX, dcategory, dkey, n, 0, true);
}

int tpe_history_set_values(tpe_ctx* ctx, const double* values, int64_t n, int32_t n_objectives, int64_t at_row) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (!ctx->history_set) return fail(ctx, TPE_E_STATE, "tpe_history_set must precede tpe_history_set_values");
  if (n_objectives < 1 || n_objectives > kMoMaxM)
    return fail(ctx, TPE_E_INVALID, "n_objectives must be in [1, %d]", kMoMaxM);
  if (n < 0 || at_row < 0 || at_row + n > ctx->N || (n > 0 && !values))
    return fail(ctx, TPE_E_INVALID, "bad values range");
  if (at_row > 0 && n_objectives != ctx->M) return fail(ctx, TPE_E_INVALID, "n_objectives changed");
  ctx->hist_lineage++;
  if (set_device(ctx)) return TPE_E_CUDA;
  // a partial write keeps every row already there (rows after the written range included)
  const size_t keep = (n_objectives == ctx->M && at_row > 0)
                          ? std::min(ctx->vals.cap, (size_t)ctx->N * n_objectives * 8) : 0;
  CU(ctx->vals.grow((size_t)std::max<int64_t>(ctx->N, 1) * n_objectives * 8, keep, ctx->stream));
  if (n > 0)
    CU(cudaMemcpyAsync(ctx->vals.as<double>() + at_row * n_objectives, values, (size_t)n * n_objectives * 8,
                       cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  ctx->M = n_objectives;
  ctx->prepared = ctx->built = ctx->sampled = false;
  ctx->hist_version++;
  return TPE_OK;
}

int tpe_get_mo_weights(tpe_ctx* ctx, double* weights) {
  if (!ctx || !weights) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (!ctx->built || !ctx->mo_weights_ready) return fail(ctx, TPE_E_STATE, "no MOTPE weights available");
  if (set_device(ctx)) return TPE_E_CUDA;
  CU(cudaMemcpyAsync(weights, ctx->mo_w.p, (size_t)ctx->info.n_below_all * 8, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return TPE_OK;
}

int tpe_hypervolume_history(tpe_ctx* ctx, const double* values, const uint8_t* feasible, int64_t n,
                            int32_t n_objectives, const double* ref, double* out) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  const int M = n_objectives;
  if (M < 2 || M > kMoMaxM) return fail(ctx, TPE_E_INVALID, "n_objectives must be in [2, %d]", kMoMaxM);
  if (n < 0 || n >= (1ll << 31) - 4096) return fail(ctx, TPE_E_INVALID, "bad number of trials %lld", (long long)n);
  if (!ref || (n > 0 && (!values || !out))) return fail(ctx, TPE_E_INVALID, "bad hypervolume history arguments");
  for (int j = 0; j < M; ++j)
    if (std::isnan(ref[j])) return fail(ctx, TPE_E_INVALID, "the reference point holds NaN");
  for (int64_t q = 0; q < n * M; ++q)
    if (std::isnan(values[q])) return fail(ctx, TPE_E_INVALID, "objective values hold NaN (trial %lld)", (long long)(q / M));
  if (n == 0) return TPE_OK;
  if (set_device(ctx, false)) return TPE_E_CUDA;
  return hv_history_run(ctx, values, feasible, (int)n, M, ref, out);
}

int tpe_pareto_front(tpe_ctx* ctx, const double* values, int64_t n, int32_t n_objectives, uint8_t* on_front) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  const int M = n_objectives;
  if (M < 1 || M > kMoMaxM) return fail(ctx, TPE_E_INVALID, "n_objectives must be in [1, %d]", kMoMaxM);
  if (n < 0 || n >= (1ll << 31) - 4096) return fail(ctx, TPE_E_INVALID, "bad number of rows %lld", (long long)n);
  if (n > 0 && (!values || !on_front)) return fail(ctx, TPE_E_INVALID, "bad Pareto front arguments");
  for (int64_t q = 0; q < n * M; ++q)
    if (std::isnan(values[q])) return fail(ctx, TPE_E_INVALID, "objective values hold NaN (row %lld)", (long long)(q / M));
  if (n == 0) return TPE_OK;
  if (set_device(ctx, false)) return TPE_E_CUDA;
  return pareto_front_run(ctx, values, (int)n, M, on_front);
}

int tpe_fanova_variances(tpe_ctx* ctx, int32_t n_trees, const int64_t* node_offsets, const int32_t* left,
                         const int32_t* right, const int32_t* feature, const double* threshold, const double* value,
                         int32_t n_features, const double* bounds, int32_t n_params, const int32_t* param_offsets,
                         const int32_t* raw_features, double* tree_variance, double* marginal_variance) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (n_trees < 1 || n_features < 1 || n_params < 0)
    return fail(ctx, TPE_E_INVALID, "bad sizes (n_trees %d, n_features %d, n_params %d)", n_trees, n_features,
                n_params);
  if (!node_offsets || !left || !right || !feature || !threshold || !value || !bounds || !param_offsets ||
      (n_params > 0 && (!raw_features || !marginal_variance)) || !tree_variance)
    return fail(ctx, TPE_E_INVALID, "bad fANOVA arguments");
  FaForest fo;
  const int rc = fanova_validate(ctx, n_trees, node_offsets, left, right, feature, threshold, n_features, bounds,
                                 n_params, param_offsets, raw_features, fo);
  if (rc != TPE_OK) return rc;
  if (set_device(ctx, false)) return TPE_E_CUDA;
  return fanova_run(ctx, n_trees, node_offsets, fo, feature, threshold, value, n_features, bounds, n_params,
                    param_offsets, raw_features, tree_variance, marginal_variance);
}

int64_t tpe_history_size(tpe_ctx* ctx) { return ctx ? ctx->N : -1; }

int tpe_history_device_ptrs(tpe_ctx* ctx, double** dX, int8_t** dcategory, double** dkey) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (!ctx->history_set) return fail(ctx, TPE_E_STATE, "no history");
  if (dX) *dX = ctx->X.as<double>();
  if (dcategory) *dcategory = ctx->cat.as<int8_t>();
  if (dkey) *dkey = ctx->key.as<double>();
  return TPE_OK;
}

// The selected columns of a call: kinds, kernel-space bounds, table offsets, which grid kernel family applies;
// uploads the ColMeta array.  Returns (through need_rowok) whether any selected column has absent values.
static int setup_columns(tpe_ctx* ctx, const tpe_cfg* cfg, const int32_t* cols, int32_t n_cols, bool* need_rowok_out) {
  const int P = (int)ctx->space.size();
  ctx->cols_h.clear();
  ctx->ncont = ctx->ndisc = ctx->ncat = ctx->nnum = 0;
  int64_t tab = 0, dtab = 0;
  bool need_rowok = false;
  for (int j = 0; j < n_cols; ++j) {
    const int src = cols[j];
    if (src < 0 || src >= P) return fail(ctx, TPE_E_INVALID, "column %d out of range", src);
    const tpe_param_desc& d = ctx->space[src];
    ColMeta cm{};
    cm.src = src;
    cm.log = d.log;
    cm.nch = d.n_choices;
    cm.low = d.low;
    cm.high = d.high;
    cm.step = d.has_step ? d.step : 0.0;
    cm.num_rank = cm.cat_rank = -1;
    cm.dist_off = -1;
    if (d.kind == TPE_KIND_CAT) {
      cm.cls = COL_CAT;
      cm.cat_rank = ctx->ncat++;
      cm.slot = cm.cat_rank;
      cm.tab_off = (int32_t)tab;
      tab += 2ll * (d.n_choices + 1) * d.n_choices;
      cm.dist_off = (int32_t)ctx->cat_dist_off[src];
    } else {
      cm.num_rank = ctx->nnum++;
      double lo = d.low, hi = d.high;
      if (d.has_step) {
        lo -= d.step / 2;
        hi += d.step / 2;
      }
      if (d.log) {
        lo = log(lo);
        hi = log(hi);
      }
      cm.klow = lo;
      cm.khigh = hi;
      if (d.has_step) {
        cm.cls = COL_DISC;
        cm.slot = ctx->ndisc++;
        const double gsz = floor((d.high - d.low) / d.step + 0.5) + 1.0;
        if (cfg->multivariate && gsz >= 1.0 && gsz <= 4096.0 && dtab + (int64_t)(gsz + 1) * (int64_t)gsz <= (1ll << 24)) {
          cm.grid = (int32_t)gsz;
          cm.dtab_off = dtab;
          dtab += (int64_t)(gsz + 1) * (int64_t)gsz;
        }
      } else {
        cm.cls = COL_CONT;
        cm.slot = ctx->ncont++;
      }
    }
    need_rowok = need_rowok || ctx->col_missing[src];
    ctx->cols_h.push_back(cm);
  }
  ctx->pc = n_cols;
  ctx->tab_doubles = tab;
  ctx->dtab_doubles = dtab;
  ctx->fast = (ctx->ndisc == 0 && ctx->ncat == 0 && ctx->ncont <= kMaxFastP);
  ctx->pb = ctx->fast ? pick_pb(ctx->ncont) : 0;
  ctx->fast_mode = ctx->fast ? (cfg->multivariate ? 2 : 1) : 0;
  static const bool uni_on = [] { const char* v = getenv("TPE_UNI_FAST"); return !(v && v[0] == '0'); }();
  ctx->uni_fast = uni_on && !cfg->multivariate && n_cols == 1 && ctx->ncont == 1;
  // mixed spaces with many candidates: kernel-minor tables + per-candidate table rows in shared memory
  static const bool mixed_on = [] { const char* v = getenv("TPE_MIXED"); return !(v && v[0] == '0'); }();
  ctx->mixed_ok = mixed_on && cfg->multivariate && !ctx->fast && ctx->ndisc + ctx->ncat > 0 && ctx->ncont <= 128 &&
                  ctx->ndisc + ctx->ncat <= 128;
  ctx->mixcols_h.clear();
  if (ctx->mixed_ok) {
    int off = 0;
    std::vector<MixCol> tail;
    for (int j = 0; j < n_cols && ctx->mixed_ok; ++j) {
      const ColMeta& cm = ctx->cols_h[j];
      if (cm.cls == COL_CONT) {
        ctx->mixcols_h.push_back(MixCol{j, 0, 0, 0});
      } else if (cm.cls == COL_DISC) {
        if (cm.grid <= 0 || cm.grid > 65535 || ctx->col_offgrid[cm.src]) ctx->mixed_ok = false;
        tail.push_back(MixCol{j, 1, cm.grid, off});
        off += cm.grid;
      } else {
        tail.push_back(MixCol{j, 2, cm.nch, off});
        off += cm.nch;
      }
    }
    ctx->mix_ncont = (int)ctx->mixcols_h.size();
    ctx->mix_nd = (int)tail.size();
    ctx->mix_tabd = off;
    ctx->mixcols_h.insert(ctx->mixcols_h.end(), tail.begin(), tail.end());
    if (ctx->mixed_ok) {
      CU(ctx->mixcols.ensure(sizeof(MixCol) * ctx->mixcols_h.size()));
      CU(cudaMemcpyAsync(ctx->mixcols.p, ctx->mixcols_h.data(), sizeof(MixCol) * ctx->mixcols_h.size(),
                         cudaMemcpyHostToDevice, ctx->stream));
    }
  }
  CU(ctx->cols.ensure(sizeof(ColMeta) * n_cols));
  CU(cudaMemcpyAsync(ctx->cols.p, ctx->cols_h.data(), sizeof(ColMeta) * n_cols, cudaMemcpyHostToDevice, ctx->stream));

  *need_rowok_out = need_rowok;
  return TPE_OK;
}

static int prepare_locked(tpe_ctx* ctx, const tpe_cfg* cfg, const int32_t* cols, int32_t n_cols,
                          tpe_split_info* info) {
  if (!ctx->history_set) return fail(ctx, TPE_E_STATE, "tpe_history_set must precede tpe_prepare");
  if (!cfg || !cols || n_cols <= 0) return fail(ctx, TPE_E_INVALID, "bad prepare arguments");
  if (cfg->prior_weight < 0)
    return fail(ctx, TPE_E_INVALID, "A non-negative value must be specified for prior_weight, but got %g.",
                cfg->prior_weight);
  if (cfg->n_candidates <= 0) return fail(ctx, TPE_E_INVALID, "n_candidates must be positive");
  if (set_device(ctx)) return TPE_E_CUDA;
  ctx->cfg = *cfg;
  ctx->launch_counter = 0;
  ctx->deferred = false;   // a new sequence abandons results nobody collected
  ctx->deferred_uni = 0;
  CU(cudaEventRecord(ctx->ev[0], ctx->stream));
  bool need_rowok = false;
  if (int rc0 = setup_columns(ctx, cfg, cols, n_cols, &need_rowok)) return rc0;
  const int P = (int)ctx->space.size();
  const int64_t N = ctx->N;
  const int64_t nal = std::max<int64_t>(N, 1);
  CU(ctx->counts.ensure(64));
  for (int w = 0; w < 2; ++w) {
    CU(ctx->est[w].rows.ensure((size_t)nal * 8));
  }
  CU(ctx->est[0].pos.ensure((size_t)nal * 8));
  const uint8_t* rowok = nullptr;
  if (need_rowok && N > 0) {
    CU(ctx->row_ok.ensure((size_t)nal));
    k_rowok<<<grid_for(N, 256, ctx->sm_count * 8), 256, 0, ctx->stream>>>(
        ctx->X.as<double>(), N, P, ctx->cols.as<ColMeta>(), n_cols, ctx->row_ok.as<uint8_t>());
    ctx->launch_counter++;
    rowok = ctx->row_ok.as<uint8_t>();
  }
  const uint8_t* pre_member = nullptr;
  int64_t nb_rest = cfg->n_below;
  ctx->mo_weights_ready = false;
  if (ctx->M >= 2) {
    int64_t taken = 0;
    int rc = mo_select_complete(ctx, cfg->n_below, &taken);
    if (rc) return rc;
    pre_member = ctx->member.as<uint8_t>();
    nb_rest = std::max<int64_t>(0, cfg->n_below - taken);
  }
  const bool plain = !need_rowok && ctx->M < 2;
  // univariate only: a multivariate suggestion prepares once per trial anyway, and a benchmark that asks
  // repeatedly against a frozen history must pay for its split every time
  const bool reuse_split = plain && !cfg->multivariate && ctx->split_valid &&
                           ctx->split_version == ctx->hist_version && ctx->split_n_below == (int64_t)cfg->n_below;
  if (!reuse_split) {
    CU(ctx->split_work.ensure(sizeof(SplitWork)));
    CU(cudaMemsetAsync(ctx->split_work.p, 0, sizeof(SplitWork), ctx->stream));
    int n_i = (int)N;
    int64_t nb = nb_rest;
    const int8_t* d_cat = ctx->cat.as<int8_t>();
    const double* d_key = ctx->key.as<double>();
    SplitWork* d_wk = ctx->split_work.as<SplitWork>();
    int64_t* d_b = ctx->est[0].rows.as<int64_t>();
    int64_t* d_p = ctx->est[0].pos.as<int64_t>();
    int64_t* d_a = ctx->est[1].rows.as<int64_t>();
    int64_t* d_c = ctx->counts.as<int64_t>();
    int64_t* d_ball = nullptr;
    if (ctx->M >= 2) {
      CU(ctx->below_all.ensure((size_t)nal * 8));
      d_ball = ctx->below_all.as<int64_t>();
    }
    void* args[] = {&n_i, &d_cat, &d_key, &nb, &rowok, &pre_member, &d_wk, &d_b, &d_p, &d_a, &d_c, &d_ball};
    const int G = (int)std::max<int64_t>(1, std::min<int64_t>(ctx->sm_count, (N + 1023) / 1024));
    CU(cudaLaunchCooperativeKernel((const void*)k_split_coop, dim3(G), dim3(512), args, 0, ctx->stream));
    ctx->launch_counter++;
    ctx->split_valid = plain;
    ctx->split_version = ctx->hist_version;
    ctx->split_n_below = cfg->n_below;
  }
  CU(cudaGetLastError());
  CU(cudaEventRecord(ctx->ev[1], ctx->stream));
  int64_t counts[3];
  // Without missing parameters the sizes of the two sets follow from the category counts alone
  // (sampler.py:686-722: whole categories in order, the cut inside one of them), which the host
  // mirror knows: no read-back, the builds are queued while the split still runs.
  // TPE_VERIFY_COUNTS=1 reads the device counts back as well and compares.
  static const bool verify_counts = [] { const char* v = getenv("TPE_VERIFY_COUNTS"); return v && v[0] == '1'; }();
  const bool predict = !need_rowok && ctx->M < 2 && (int64_t)ctx->cat_h.size() == N;
  if (predict) {
    const int64_t* cnt = ctx->cat_cnt;
    int64_t remaining = std::max<int64_t>(cfg->n_below, 0), below = 0;
    for (int c = 0; c < 3; ++c) {
      const int64_t take = std::min(remaining, cnt[c]);
      below += take;
      remaining -= take;
      if (take < cnt[c]) break;
    }
    counts[0] = counts[1] = below;
    counts[2] = N - cnt[4] - below;  // TPE_CAT_EXCLUDED rows are in neither set
  }
  if (!predict || verify_counts) {
    int64_t dev[3];
    CU(cudaMemcpyAsync(dev, ctx->counts.p, sizeof(dev), cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    if (predict && (dev[0] != counts[0] || dev[1] != counts[1] || dev[2] != counts[2]))
      return fail(ctx, TPE_E_STATE, "split sizes: host prediction (%lld, %lld, %lld) != device (%lld, %lld, %lld)",
                  (long long)counts[0], (long long)counts[1], (long long)counts[2], (long long)dev[0],
                  (long long)dev[1], (long long)dev[2]);
    counts[0] = dev[0]; counts[1] = dev[1]; counts[2] = dev[2];
  }
  ctx->info.n_below_all = counts[0];
  ctx->info.n_below_obs = counts[1];
  ctx->info.n_above_obs = counts[2];
  ctx->est[0].n = counts[1];
  ctx->est[1].n = counts[2];
  if (info) *info = ctx->info;
  ctx->prepared = true;
  ctx->built = ctx->sampled = false;
  return TPE_OK;
}

int tpe_prepare(tpe_ctx* ctx, const tpe_cfg* cfg, const int32_t* cols, int32_t n_cols, tpe_split_info* info) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  return prepare_locked(ctx, cfg, cols, n_cols, info);
}

static int build_locked(tpe_ctx* ctx, const double* w_below, const double* w_above) {
  if (!ctx->prepared) return fail(ctx, TPE_E_STATE, "tpe_prepare must precede tpe_build");
  if (set_device(ctx)) return TPE_E_CUDA;
  for (int which = 0; which < 2; ++which) {
    const double* w = which == 0 ? w_below : w_above;
    const int64_t n = ctx->est[which].n;
    if (w) {  // the reference's _call_weights_func checks (parzen_estimator.py:88-109)
      double tot = 0;
      for (int64_t i = 0; i < n; ++i) {
        if (w[i] < 0) return fail(ctx, TPE_E_INVALID, "The `weights` function is not allowed to return negative values.");
        if (!isfinite(w[i]))
          return fail(ctx, TPE_E_INVALID, "The `weights`function is not allowed to return infinite or NaN values.");
        tot += w[i];
      }
      if (n > 0 && tot <= 0)
        return fail(ctx, TPE_E_INVALID, "The `weight` function is not allowed to return all-zero values.");
    }
  }
  // multivariate builds share no scratch: g(x)'s estimator (the big one) goes to the second stream
  const bool fork = ctx->cfg.multivariate != 0;
  if (fork) {
    CU(cudaEventRecord(ctx->ev_fork, ctx->stream));
    CU(cudaStreamWaitEvent(ctx->stream2, ctx->ev_fork, 0));
    int rc = build_estimator(ctx, 1, w_above, ctx->stream2);
    if (rc) return rc;
    CU(cudaEventRecord(ctx->ev_join, ctx->stream2));
    ctx->above_pending = true;
    rc = build_estimator(ctx, 0, w_below, ctx->stream);
    if (rc) return rc;
  } else {
    for (int which = 0; which < 2; ++which) {
      int rc = build_estimator(ctx, which, which == 0 ? w_below : w_above, ctx->stream);
      if (rc) return rc;
    }
  }
  CU(cudaEventRecord(ctx->ev[2], ctx->stream));
  ctx->built = true;
  ctx->sampled = false;
  return TPE_OK;
}

int tpe_build(tpe_ctx* ctx, const double* w_below, const double* w_above) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  return build_locked(ctx, w_below, w_above);
}

// Candidates, both log-density grids and the argmax of n_asks asks whose uniforms are resident in ctx->U: launches
// only (ctx->stream); results in ctx->out_x / out_acq / out_best.
static int launch_sample_select(tpe_ctx* ctx, int64_t n_asks, bool used_dev_rng, bool timed) {
  cudaStream_t st = ctx->stream;
  const int32_t C = ctx->cfg.n_candidates;
  const int64_t Ct = n_asks * C;
  const int64_t per_ask = (int64_t)C * (1 + ctx->ncat + ctx->nnum);
  int rc = TPE_OK;
  (void)per_ask;
  if (timed) CU(cudaEventRecord(ctx->ev[3], st));
  ctx->user_points = false;
  Estimator& eb = ctx->est[0];
  k_sample<<<grid_for(Ct * ctx->pc, 128, ctx->sm_count * 16), 128, 0, st>>>(
      ctx->U.as<double>(), n_asks, C, ctx->cols.as<ColMeta>(), ctx->pc, ctx->ncat, ctx->nnum, eb.cdf.as<double>(),
      eb.K, eb.mu.as<double>(), eb.sigma.as<double>(), eb.tab.as<double>(), ctx->S.as<double>(),
      ctx->fast ? ctx->xT.as<double>() : nullptr, ctx->ct_stride, ctx->oob.as<uint8_t>());
  ctx->launch_counter++;
  if (timed) CU(cudaEventRecord(ctx->ev[4], st));
  if (used_dev_rng) {
    // speculative draw for the next ask (same count) from the state this ask's draw ended in; runs on
    // the side stream while the grid kernels of this ask run
    static const bool spec_on = [] { const char* v = getenv("TPE_RNG_SPECULATE"); return !(v && v[0] == '0'); }();
    const int64_t count = n_asks * per_ask;
    if (spec_on) {
      CU(ctx->U2.ensure((size_t)count * 8));
      CU(ctx->mt_spec.ensure(625 * 4));
      CU(cudaMemcpyAsync(ctx->mt_spec.p, ctx->mt_state.p, 625 * 4, cudaMemcpyDeviceToDevice, ctx->stream3));
      if (int rc2 = launch_mt(ctx, ctx->stream3, ctx->mt_spec.as<uint32_t>(), 0, count, ctx->U2.as<double>())) return rc2;
      CU(cudaEventRecord(ctx->ev_spec, ctx->stream3));
      ctx->spec_pending = true;
      ctx->spec_count = count;
    }
    // the generator's end state comes back with the results (tpe_rng_state then needs no device access)
    CU(cudaMemcpyAsync(ctx->mt_host, ctx->mt_state.p, (size_t)625 * 4, cudaMemcpyDeviceToHost, st));
  }
  rc = run_logpdf(ctx, 0, Ct);
  if (rc) return rc;
  if (timed) CU(cudaEventRecord(ctx->ev[5], st));
  rc = run_logpdf(ctx, 1, Ct, timed ? ctx->ev[6] : nullptr);
  if (rc) return rc;
  if (timed) CU(cudaEventRecord(ctx->ev[7], st));
  if (ctx->kshard_world > 1) {
    // one (max, sum) per candidate over this context's slice of g(x); the caller gathers them from all ranks and
    // finishes with tpe_finish_from_partials
    CU(ctx->kpart.ensure((size_t)ctx->ct_stride * 16));
    k_reduce_parts<<<grid_for(Ct, 256, ctx->sm_count * 8), 256, 0, st>>>(ctx->est[1].part.as<double2>(), ctx->est[1].nsplit,
                                                                         ctx->ct_stride, Ct, ctx->kpart.as<double2>());
    ctx->launch_counter++;
    ctx->partial_ready = true;
    return TPE_OK;
  }
  k_acq<<<grid_for(Ct * 32, 256, ctx->sm_count * 8), 256, 0, st>>>(
      ctx->est[0].part.as<double2>(), ctx->est[0].nsplit, ctx->est[1].part.as<double2>(), ctx->est[1].nsplit,
      ctx->ct_stride, ctx->fast ? ctx->oob.as<uint8_t>() : nullptr, ctx->est[0].fix.as<double2>(),
      ctx->est[1].fix.as<double2>(), Ct, ctx->logl.as<double>(), ctx->logg.as<double>());
  k_select<<<(unsigned)n_asks, 256, 0, st>>>(ctx->logl.as<double>(), ctx->logg.as<double>(), C, ctx->S.as<double>(),
                                             ctx->pc, ctx->out_x.as<double>(), ctx->out_acq.as<double>(),
                                             ctx->out_best.as<int64_t>());
  ctx->launch_counter += 2;
  return TPE_OK;
}

// Everything of tpe_sample_and_select up to the last kernel.  defer: the results are also copied into the
// context's page-locked staging area and nothing is waited for (tpe_sample_and_select_async).
static int sample_select_issue(tpe_ctx* ctx, const double* uniforms, int64_t n_asks, bool defer) {
  if (!ctx->built) return fail(ctx, TPE_E_STATE, "tpe_build must precede tpe_sample_and_select");
  if ((!uniforms && !ctx->u_device_rng) || n_asks <= 0)
    return fail(ctx, TPE_E_INVALID, "bad sample arguments");
  if (set_device(ctx, /*join=*/false)) return TPE_E_CUDA;  // est[1] is joined by run_logpdf(ctx, 1)
  cudaStream_t st = ctx->stream;
  const int32_t C = ctx->cfg.n_candidates;
  const int64_t Ct = n_asks * C;
  const int64_t per_ask = (int64_t)C * (1 + ctx->ncat + ctx->nnum);
  ctx->n_asks = n_asks;
  ctx->deferred = false;
  int rc = ensure_candidate_buffers(ctx, Ct);
  if (rc) return rc;
  CU(ctx->U.ensure((size_t)n_asks * per_ask * 8));
  CU(ctx->out_x.ensure((size_t)n_asks * ctx->pc * 8));
  CU(ctx->out_acq.ensure((size_t)n_asks * 8));
  CU(ctx->out_best.ensure((size_t)n_asks * 8));
  const bool used_dev_rng = !uniforms;
  if (!uniforms) {
    if (ctx->u_staged_count != n_asks * per_ask)
      return fail(ctx, TPE_E_INVALID, "device-generated uniforms: %lld staged, %lld needed",
                  (long long)ctx->u_staged_count, (long long)(n_asks * per_ask));
    CU(cudaStreamWaitEvent(st, ctx->ev_u, 0));  // generated by tpe_stage_uniforms_mt19937
    ctx->u_device_rng = false;
  } else if (ctx->u_staged == uniforms && ctx->u_staged_count == n_asks * per_ask) {
    CU(cudaStreamWaitEvent(st, ctx->ev_u, 0));  // uploaded by tpe_suggest while the split ran
  } else {
    if (ctx->u_device_rng) {  // a device draw nobody consumed is still writing U on the side stream
      CU(cudaStreamWaitEvent(st, ctx->ev_u, 0));
      ctx->u_device_rng = false;
    }
    CU(cudaMemcpyAsync(ctx->U.p, uniforms, (size_t)n_asks * per_ask * 8, cudaMemcpyHostToDevice, st));
  }
  ctx->u_staged = nullptr;
  rc = launch_sample_select(ctx, n_asks, used_dev_rng, true);
  if (rc) return rc;
  CU(cudaEventRecord(ctx->ev[8], st));
  CU(cudaGetLastError());
  ctx->issued_dev_rng = used_dev_rng;
  if (defer) {
    const size_t need = (size_t)n_asks * (ctx->pc + 2) * 8;
    if (ctx->res_host_cap < need) {
      if (ctx->res_host) cudaFreeHost(ctx->res_host);
      ctx->res_host = nullptr;
      ctx->res_host_cap = 0;
      CU(cudaHostAlloc(&ctx->res_host, need + 4096, cudaHostAllocDefault));
      ctx->res_host_cap = need + 4096;
    }
    char* h = static_cast<char*>(ctx->res_host);
    CU(cudaMemcpyAsync(h, ctx->out_x.p, (size_t)n_asks * ctx->pc * 8, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(h + (size_t)n_asks * ctx->pc * 8, ctx->out_acq.p, (size_t)n_asks * 8, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(h + (size_t)n_asks * (ctx->pc + 1) * 8, ctx->out_best.p, (size_t)n_asks * 8,
                       cudaMemcpyDeviceToHost, st));
    ctx->deferred = true;
  }
  return TPE_OK;
}

static int sample_select_finish(tpe_ctx* ctx) {
  CU(cudaStreamSynchronize(ctx->stream));
  if (ctx->issued_dev_rng) ctx->mt_host_valid = true;
  for (int i = 0; i < 8; ++i) cudaEventElapsedTime(&ctx->ms[i], ctx->ev[i], ctx->ev[i + 1]);
  cudaEventElapsedTime(&ctx->ms[8], ctx->ev[0], ctx->ev[8]);
  ctx->launches = ctx->launch_counter;
  ctx->sampled = true;
  ctx->deferred = false;
  return TPE_OK;
}

static int sample_select_locked(tpe_ctx* ctx, const double* uniforms, int64_t n_asks, double* out_x, double* out_acq,
                                int64_t* out_best) {
  int rc = sample_select_issue(ctx, uniforms, n_asks, false);
  if (rc) return rc;
  cudaStream_t st = ctx->stream;
  if (out_x) CU(cudaMemcpyAsync(out_x, ctx->out_x.p, (size_t)n_asks * ctx->pc * 8, cudaMemcpyDeviceToHost, st));
  if (out_acq) CU(cudaMemcpyAsync(out_acq, ctx->out_acq.p, (size_t)n_asks * 8, cudaMemcpyDeviceToHost, st));
  if (out_best) CU(cudaMemcpyAsync(out_best, ctx->out_best.p, (size_t)n_asks * 8, cudaMemcpyDeviceToHost, st));
  return sample_select_finish(ctx);
}

int tpe_sample_and_select(tpe_ctx* ctx, const double* uniforms, int64_t n_asks, double* out_x, double* out_acq,
                          int64_t* out_best) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  return sample_select_locked(ctx, uniforms, n_asks, out_x, out_acq, out_best);
}

int tpe_sample_and_select_async(tpe_ctx* ctx, const double* uniforms, int64_t n_asks) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  return sample_select_issue(ctx, uniforms, n_asks, true);
}

int tpe_collect(tpe_ctx* ctx, double* out_x, double* out_acq, int64_t* out_best) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (!ctx->deferred) return fail(ctx, TPE_E_STATE, "tpe_collect needs a pending tpe_sample_and_select_async");
  if (set_device(ctx, /*join=*/false)) return TPE_E_CUDA;
  const int64_t n_asks = ctx->n_asks;
  int rc = sample_select_finish(ctx);
  if (rc) return rc;
  const char* h = static_cast<const char*>(ctx->res_host);
  if (out_x) memcpy(out_x, h, (size_t)n_asks * ctx->pc * 8);
  if (out_acq) memcpy(out_acq, h + (size_t)n_asks * ctx->pc * 8, (size_t)n_asks * 8);
  if (out_best) memcpy(out_best, h + (size_t)n_asks * (ctx->pc + 1) * 8, (size_t)n_asks * 8);
  return TPE_OK;
}

int tpe_set_kernel_shard(tpe_ctx* ctx, int32_t rank, int32_t world) {
  if (!ctx || world < 1 || rank < 0 || rank >= world) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  ctx->kshard_rank = rank;
  ctx->kshard_world = world;
  ctx->partial_ready = false;
  return TPE_OK;
}

int tpe_sample_and_partial(tpe_ctx* ctx, const double* uniforms, int64_t n_asks, double** d_partials, int64_t* stride) {
  if (!ctx || !d_partials) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (ctx->kshard_world < 2) return fail(ctx, TPE_E_STATE, "tpe_set_kernel_shard(rank, world >= 2) must precede tpe_sample_and_partial");
  int rc = sample_select_issue(ctx, uniforms, n_asks, false);
  if (rc) return rc;
  CU(cudaStreamSynchronize(ctx->stream));
  if (ctx->issued_dev_rng) ctx->mt_host_valid = true;
  *d_partials = ctx->kpart.as<double>();
  if (stride) *stride = ctx->ct_stride;
  return TPE_OK;
}

int tpe_finish_from_partials(tpe_ctx* ctx, const double* d_gathered, int32_t world, double* out_x, double* out_acq,
                             int64_t* out_best) {
  if (!ctx || !d_gathered || world < 1) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (!ctx->partial_ready) return fail(ctx, TPE_E_STATE, "tpe_sample_and_partial must precede tpe_finish_from_partials");
  if (set_device(ctx, /*join=*/false)) return TPE_E_CUDA;
  cudaStream_t st = ctx->stream;
  const int64_t n_asks = ctx->n_asks, Ct = n_asks * ctx->cfg.n_candidates;
  k_acq<<<grid_for(Ct * 32, 256, ctx->sm_count * 8), 256, 0, st>>>(
      ctx->est[0].part.as<double2>(), ctx->est[0].nsplit, reinterpret_cast<const double2*>(d_gathered), world,
      ctx->ct_stride, ctx->fast ? ctx->oob.as<uint8_t>() : nullptr, ctx->est[0].fix.as<double2>(),
      ctx->est[1].fix.as<double2>(), Ct, ctx->logl.as<double>(), ctx->logg.as<double>());
  k_select<<<(unsigned)n_asks, 256, 0, st>>>(ctx->logl.as<double>(), ctx->logg.as<double>(), ctx->cfg.n_candidates,
                                             ctx->S.as<double>(), ctx->pc, ctx->out_x.as<double>(),
                                             ctx->out_acq.as<double>(), ctx->out_best.as<int64_t>());
  ctx->launch_counter += 2;
  CU(cudaEventRecord(ctx->ev[8], st));
  CU(cudaGetLastError());
  if (out_x) CU(cudaMemcpyAsync(out_x, ctx->out_x.p, (size_t)n_asks * ctx->pc * 8, cudaMemcpyDeviceToHost, st));
  if (out_acq) CU(cudaMemcpyAsync(out_acq, ctx->out_acq.p, (size_t)n_asks * 8, cudaMemcpyDeviceToHost, st));
  if (out_best) CU(cudaMemcpyAsync(out_best, ctx->out_best.p, (size_t)n_asks * 8, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  for (int i = 0; i < 8; ++i) cudaEventElapsedTime(&ctx->ms[i], ctx->ev[i], ctx->ev[i + 1]);
  cudaEventElapsedTime(&ctx->ms[8], ctx->ev[0], ctx->ev[8]);
  ctx->launches = ctx->launch_counter;
  ctx->partial_ready = false;
  ctx->sampled = true;
  return TPE_OK;
}

int tpe_stage_uniforms_mt19937(tpe_ctx* ctx, const uint32_t* key, int32_t pos, int64_t skip, int64_t count) {
  // key == NULL: continue from the state the previous staged draw ended in (kept on the device)
  if (!ctx || (key && (pos < 0 || pos > 624)) || skip < 0 || count <= 0) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (set_device(ctx, /*join=*/false)) return TPE_E_CUDA;
  if (!key && !ctx->mt_state.p)
    return fail(ctx, TPE_E_STATE, "tpe_stage_uniforms_mt19937(key = NULL) needs a previous staged draw to continue");
  ctx->u_staged = nullptr;
  ctx->u_device_rng = false;
  const bool same_state = !key || (ctx->mt_host_valid && (uint32_t)pos == ctx->mt_host[624] &&
                                   memcmp(key, ctx->mt_host, 624 * 4) == 0);
  if (ctx->spec_pending && skip == 0 && count == ctx->spec_count && same_state) {
    // the caller's generator is where the previous ask left it: the speculative draw is this ask's
    std::swap(ctx->U, ctx->U2);
    std::swap(ctx->mt_state, ctx->mt_spec);
    std::swap(ctx->ev_u, ctx->ev_spec);
    ctx->spec_pending = false;
    ctx->mt_host_valid = false;
    ctx->u_staged_count = count;
    ctx->u_device_rng = true;
    return TPE_OK;
  }
  ctx->spec_pending = false;
  ctx->mt_host_valid = false;
  CU(cudaStreamSynchronize(ctx->stream3));
  CU(ctx->U.ensure((size_t)count * 8));
  CU(ctx->mt_state.ensure(625 * 4));
  if (key) {
    uint32_t h[625];
    memcpy(h, key, 624 * 4);
    h[624] = (uint32_t)pos;
    CU(cudaMemcpyAsync(ctx->mt_state.p, h, sizeof(h), cudaMemcpyHostToDevice, ctx->stream3));
  }
  if (int rc = launch_mt(ctx, ctx->stream3, ctx->mt_state.as<uint32_t>(), skip, count, ctx->U.as<double>())) return rc;
  CU(cudaEventRecord(ctx->ev_u, ctx->stream3));
  ctx->u_staged_count = count;
  ctx->u_device_rng = true;
  return TPE_OK;
}
int tpe_rng_state(tpe_ctx* ctx, uint32_t* key_out, int32_t* pos_out) {
  if (!ctx || !key_out || !pos_out) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (set_device(ctx, /*join=*/false)) return TPE_E_CUDA;
  if (!ctx->mt_state.p) return fail(ctx, TPE_E_STATE, "tpe_stage_uniforms_mt19937 must precede tpe_rng_state");
  if (!ctx->mt_host_valid) {  // not yet read back with the results of an ask
    CU(cudaStreamWaitEvent(ctx->stream, ctx->ev_u, 0));
    CU(cudaMemcpyAsync(ctx->mt_host, ctx->mt_state.p, (size_t)625 * 4, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    ctx->mt_host_valid = true;
  }
  memcpy(key_out, ctx->mt_host, 624 * 4);
  *pos_out = (int32_t)ctx->mt_host[624];
  return TPE_OK;
}
int tpe_result_device_ptrs(tpe_ctx* ctx, double** out_x, double** out_acq, int64_t** out_best) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (!ctx->sampled) return fail(ctx, TPE_E_STATE, "tpe_sample_and_select must precede tpe_result_device_ptrs");
  if (out_x) *out_x = ctx->out_x.as<double>();
  if (out_acq) *out_acq = ctx->out_acq.as<double>();
  if (out_best) *out_best = ctx->out_best.as<int64_t>();
  return TPE_OK;
}
int tpe_rng_state_device(tpe_ctx* ctx, uint32_t** state625) {
  if (!ctx || !state625) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (set_device(ctx, /*join=*/false)) return TPE_E_CUDA;
  if (!ctx->mt_state.p) return fail(ctx, TPE_E_STATE, "tpe_stage_uniforms_mt19937 must precede tpe_rng_state_device");
  CU(cudaStreamSynchronize(ctx->stream3));  // the generator that last wrote the state
  // the caller may overwrite the state (a broadcast from the rank that drew last): forget what the host knows
  ctx->mt_host_valid = false;
  ctx->spec_pending = false;
  *state625 = ctx->mt_state.as<uint32_t>();
  return TPE_OK;
}
int tpe_get_uniforms(tpe_ctx* ctx, double* out, int64_t count) {
  if (!ctx || !out || count <= 0) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (set_device(ctx, /*join=*/false)) return TPE_E_CUDA;
  if ((size_t)count * 8 > ctx->U.cap) return fail(ctx, TPE_E_INVALID, "only %zu uniforms are staged", ctx->U.cap / 8);
  CU(cudaStreamSynchronize(ctx->stream3));
  CU(cudaMemcpyAsync(out, ctx->U.p, (size_t)count * 8, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return TPE_OK;
}

int tpe_host_alloc(tpe_ctx* ctx, size_t bytes, void** out) {
  if (!ctx || !out || bytes == 0) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (set_device(ctx, /*join=*/false)) return TPE_E_CUDA;
  *out = nullptr;
  CU(cudaHostAlloc(out, bytes, cudaHostAllocDefault));
  return TPE_OK;
}
int tpe_host_free(tpe_ctx* ctx, void* p) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (!p) return TPE_OK;
  if (set_device(ctx, /*join=*/false)) return TPE_E_CUDA;
  CU(cudaFreeHost(p));
  return TPE_OK;
}

int tpe_stage_uniforms(tpe_ctx* ctx, const double* uniforms, int64_t count) {
  if (!ctx || !uniforms || count <= 0) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (set_device(ctx, /*join=*/false)) return TPE_E_CUDA;
  ctx->u_staged = nullptr;
  CU(cudaStreamSynchronize(ctx->stream3));  // a previous, unconsumed staging
  CU(ctx->U.ensure((size_t)count * 8));
  CU(cudaMemcpyAsync(ctx->U.p, uniforms, (size_t)count * 8, cudaMemcpyHostToDevice, ctx->stream3));
  CU(cudaEventRecord(ctx->ev_u, ctx->stream3));
  ctx->u_staged = uniforms;
  ctx->u_staged_count = count;
  return TPE_OK;
}

int tpe_suggest(tpe_ctx* ctx, const tpe_cfg* cfg, const int32_t* cols, int32_t n_cols, const double* w_below,
                const double* w_above, const double* uniforms, int64_t n_asks, double* out_x, double* out_acq,
                int64_t* out_best) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  ctx->u_staged = nullptr;
  if (cfg && uniforms && n_asks > 0 && n_cols > 0 && cfg->n_candidates > 0) {
    // every selected column consumes C uniforms, plus C for the kernel choice: the count is known
    // before the split, so the upload overlaps it
    const int64_t count = n_asks * (int64_t)cfg->n_candidates * (1 + n_cols);
    if (set_device(ctx)) return TPE_E_CUDA;
    CU(ctx->U.ensure((size_t)count * 8));
    CU(cudaMemcpyAsync(ctx->U.p, uniforms, (size_t)count * 8, cudaMemcpyHostToDevice, ctx->stream3));
    CU(cudaEventRecord(ctx->ev_u, ctx->stream3));
    ctx->u_staged = uniforms;
    ctx->u_staged_count = count;
  }
  int rc = prepare_locked(ctx, cfg, cols, n_cols, nullptr);
  if (!rc) rc = build_locked(ctx, w_below, w_above);
  if (!rc) rc = sample_select_locked(ctx, uniforms, n_asks, out_x, out_acq, out_best);
  if (ctx->u_staged) {  // an early error left the upload in flight: the caller's buffer must be free on return
    cudaStreamSynchronize(ctx->stream3);
    ctx->u_staged = nullptr;
  }
  return rc;
}

// ---- the P sample_independent calls of one univariate trial, in one go -------------------------------------------

static tpe_ctx* make_sub(tpe_ctx* parent) {
  tpe_ctx* c = new tpe_ctx();
  c->device = parent->device;
  c->is_sub = true;
  c->sm_count = parent->sm_count;
  c->sort_cta_cap = std::max(8, parent->sm_count / 8);   // ~8 column sorts share the GPU at a time
  if (cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) != cudaSuccess ||
      cudaStreamCreateWithFlags(&c->stream2, cudaStreamNonBlocking) != cudaSuccess ||
      cudaStreamCreateWithFlags(&c->stream3, cudaStreamNonBlocking) != cudaSuccess) {
    delete c;
    return nullptr;
  }
  for (auto& e : c->ev) cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
  cudaEventCreateWithFlags(&c->ev_fork, cudaEventDisableTiming);
  cudaEventCreateWithFlags(&c->ev_join, cudaEventDisableTiming);
  cudaEventCreateWithFlags(&c->ev_u, cudaEventDisableTiming);
  cudaEventCreateWithFlags(&c->ev_spec, cudaEventDisableTiming);
  return c;
}

static int uni_batch_locked(tpe_ctx* ctx, const tpe_cfg* cfg, const int32_t* cols, int32_t n_cols,
                            const double* w_below, const double* w_above, const double* uniforms, double* out_x,
                            double* out_acq, int64_t* out_best, bool defer) {
  if (!cfg || !cols || n_cols <= 0 || (!out_x && !defer)) return fail(ctx, TPE_E_INVALID, "bad arguments");
  ctx->deferred_uni = 0;
  if (cfg->multivariate) return fail(ctx, TPE_E_INVALID, "tpe_suggest_univariate_batch is for multivariate = 0");
  if (ctx->M >= 2) return fail(ctx, TPE_E_STATE, "not batchable: multi-objective history (use the per-parameter calls)");
  if (set_device(ctx)) return TPE_E_CUDA;
  const int32_t C = cfg->n_candidates;
  const int64_t per_col = 2ll * C, count = per_col * n_cols;
  // uniforms: uploaded on the side stream now, or already generated there by tpe_stage_uniforms_mt19937
  const bool dev_rng = uniforms == nullptr;
  if (dev_rng) {
    if (!ctx->u_device_rng || ctx->u_staged_count != count)
      return fail(ctx, TPE_E_INVALID, "device-generated uniforms: %lld staged, %lld needed", (long long)ctx->u_staged_count,
                  (long long)count);
  } else {
    if (ctx->u_device_rng) CU(cudaStreamSynchronize(ctx->stream3));
    CU(ctx->U.ensure((size_t)count * 8));
    CU(cudaMemcpyAsync(ctx->U.p, uniforms, (size_t)count * 8, cudaMemcpyHostToDevice, ctx->stream3));
    CU(cudaEventRecord(ctx->ev_u, ctx->stream3));
  }
  ctx->u_device_rng = false;
  ctx->u_staged = nullptr;
  // one split for every column (sampler.py:686-722 does not look at the parameters)
  int rc = prepare_locked(ctx, cfg, cols, n_cols, nullptr);
  if (rc) return rc;
  for (const ColMeta& cm : ctx->cols_h)
    if (ctx->col_missing[cm.src])
      return fail(ctx, TPE_E_STATE, "not batchable: a selected parameter is absent from some trials (their estimators use "
                  "different trials; use the per-parameter calls)");
  for (int which = 0; which < 2; ++which) {   // _call_weights_func checks (parzen_estimator.py:88-109), once
    const double* w = which == 0 ? w_below : w_above;
    const int64_t n = ctx->est[which].n;
    if (!w) continue;
    double tot = 0;
    for (int64_t i = 0; i < n; ++i) {
      if (w[i] < 0) return fail(ctx, TPE_E_INVALID, "The `weights` function is not allowed to return negative values.");
      if (!isfinite(w[i])) return fail(ctx, TPE_E_INVALID, "The `weights`function is not allowed to return infinite or NaN values.");
      tot += w[i];
    }
    if (n > 0 && tot <= 0) return fail(ctx, TPE_E_INVALID, "The `weight` function is not allowed to return all-zero values.");
  }
  {
    // how the above set differs from the previous call's (the column contexts then update their sorted orders
    // instead of sorting: k_order_update); the answer stays on the device
    const int64_t n_new = ctx->est[1].n;
    int cand = 2;
    if (ctx->uni_prev_n >= 0 && ctx->uni_prev_lineage == ctx->hist_lineage)
      cand = n_new == ctx->uni_prev_n ? 0 : n_new == ctx->uni_prev_n + 1 ? 1 : 2;
    CU(ctx->uni_mode.ensure(16));
    CU(cudaMemsetAsync(ctx->uni_mode.p, 0, 4, ctx->stream));
    k_rows_delta<<<cand == 2 ? 1 : grid_for(std::max<int64_t>(ctx->uni_prev_n, 1), 256, ctx->sm_count), 256, 0, ctx->stream>>>(
        ctx->est[1].rows.as<int64_t>(), ctx->uni_prev_rows.as<int64_t>(), cand == 2 ? 0 : ctx->uni_prev_n, cand,
        ctx->uni_mode.as<int>());
    ctx->launch_counter++;
    CU(ctx->uni_prev_rows.ensure((size_t)(n_new + 1) * 8));
    CU(cudaMemcpyAsync(ctx->uni_prev_rows.p, ctx->est[1].rows.p, (size_t)n_new * 8, cudaMemcpyDeviceToDevice, ctx->stream));
    ctx->uni_prev_n = n_new;
    ctx->uni_prev_lineage = ctx->hist_lineage;
    ctx->uni_seq++;
  }
  if (!ctx->ev_uni) CU(cudaEventCreateWithFlags(&ctx->ev_uni, cudaEventDisableTiming));
  CU(cudaEventRecord(ctx->ev_uni, ctx->stream));
  CU(ctx->out_x.ensure((size_t)n_cols * 8));
  CU(ctx->out_acq.ensure((size_t)n_cols * 8));
  CU(ctx->out_best.ensure((size_t)n_cols * 8));
  // all columns continuous: stage by stage over all of them (one launch per stage)
  static const bool staged_on = [] { const char* v = getenv("TPE_UNI_STAGED"); return !(v && v[0] == '0'); }();
  bool staged = staged_on && C <= 4096 && n_cols >= 2;
  for (const ColMeta& cm : ctx->cols_h) staged = staged && cm.cls == COL_CONT;
  if (staged) {
    ctx->launch_counter = 0;
    rc = uni_batch_staged(ctx, cfg, cols, n_cols, w_below, w_above);
    if (rc) return rc;
    if (dev_rng) CU(cudaMemcpyAsync(ctx->mt_host, ctx->mt_state.p, (size_t)625 * 4, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaEventRecord(ctx->ev[8], ctx->stream));
    if (defer) {   // results into the page-locked staging area; tpe_collect_univariate waits and hands them out
      const size_t need = (size_t)n_cols * 3 * 8;
      if (ctx->res_host_cap < need) {
        if (ctx->res_host) cudaFreeHost(ctx->res_host);
        ctx->res_host = nullptr;
        ctx->res_host_cap = 0;
        CU(cudaHostAlloc(&ctx->res_host, need + 4096, cudaHostAllocDefault));
        ctx->res_host_cap = need + 4096;
      }
      char* h = static_cast<char*>(ctx->res_host);
      CU(cudaMemcpyAsync(h, ctx->out_x.p, (size_t)n_cols * 8, cudaMemcpyDeviceToHost, ctx->stream));
      CU(cudaMemcpyAsync(h + (size_t)n_cols * 8, ctx->out_acq.p, (size_t)n_cols * 8, cudaMemcpyDeviceToHost, ctx->stream));
      CU(cudaMemcpyAsync(h + (size_t)n_cols * 16, ctx->out_best.p, (size_t)n_cols * 8, cudaMemcpyDeviceToHost, ctx->stream));
      ctx->deferred_uni = n_cols;
      ctx->deferred_uni_rng = dev_rng;
      ctx->spec_pending = false;
      ctx->launches = ctx->launch_counter;
      ctx->prepared = ctx->built = ctx->sampled = false;
      return TPE_OK;
    }
    CU(cudaMemcpyAsync(out_x, ctx->out_x.p, (size_t)n_cols * 8, cudaMemcpyDeviceToHost, ctx->stream));
    if (out_acq) CU(cudaMemcpyAsync(out_acq, ctx->out_acq.p, (size_t)n_cols * 8, cudaMemcpyDeviceToHost, ctx->stream));
    if (out_best) CU(cudaMemcpyAsync(out_best, ctx->out_best.p, (size_t)n_cols * 8, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    if (dev_rng) ctx->mt_host_valid = true;
    ctx->spec_pending = false;
    for (int i = 0; i < 9; ++i) ctx->ms[i] = 0.0f;
    cudaEventElapsedTime(&ctx->ms[8], ctx->ev[0], ctx->ev[8]);
    ctx->launches = ctx->launch_counter;
    ctx->prepared = ctx->built = ctx->sampled = false;
    return TPE_OK;
  }
  if (defer)
    return fail(ctx, TPE_E_STATE, "not batchable asynchronously: only trials whose parameters are all continuous are "
                "evaluated stage by stage");
  while ((int)ctx->uni_sub.size() < n_cols) {
    tpe_ctx* c = make_sub(ctx);
    if (!c) return fail(ctx, TPE_E_CUDA, "could not create the streams of a column context");
    ctx->uni_sub.push_back(c);
  }
  int launches = ctx->launch_counter;
  // Issuing ~20 launches per column is host work: the columns are independent,
  // so a few host threads issue them side by side.  Each column context is touched by exactly one thread.
  auto issue_column = [&](int j) -> int {
    tpe_ctx* sub = ctx->uni_sub[j];
    int rc = TPE_OK;
    sub->err.clear();
#define CUS(call)                                                                                            \
    do {                                                                                                       \
      cudaError_t e_ = (call);                                                                                 \
      if (e_ != cudaSuccess)                                                                                   \
        return fail(sub, e_ == cudaErrorMemoryAllocation ? TPE_E_NOMEM : TPE_E_CUDA, "%s failed: %s (%s:%d)", \
                    #call, cudaGetErrorString(e_), __FILE__, __LINE__);                                        \
    } while (0)
    CUS(cudaSetDevice(ctx->device));
    sub->space = ctx->space;
    sub->cat_dist_off = ctx->cat_dist_off;
    sub->cat_dist.alias(ctx->cat_dist.p, ctx->cat_dist.cap);
    sub->col_missing = ctx->col_missing;
    sub->col_oor = ctx->col_oor;
    sub->col_offgrid = ctx->col_offgrid;
    sub->X.alias(ctx->X.p, ctx->X.cap);
    sub->cat.alias(ctx->cat.p, ctx->cat.cap);
    sub->key.alias(ctx->key.p, ctx->key.cap);
    sub->N = ctx->N;
    sub->hist_lineage = ctx->hist_lineage;
    sub->uni_seq = ctx->uni_seq;
    sub->uni_mode_ptr = ctx->uni_mode.as<int>();
    sub->M = 1;
    sub->history_set = true;
    sub->cfg = *cfg;
    sub->launch_counter = 0;
    bool rowok_unused = false;
    rc = setup_columns(sub, cfg, cols + j, 1, &rowok_unused);
    if (rc) return rc;
    for (int which = 0; which < 2; ++which) {
      sub->est[which].rows.alias(ctx->est[which].rows.p, ctx->est[which].rows.cap);
      sub->est[which].n = ctx->est[which].n;
    }
    sub->est[0].pos.alias(ctx->est[0].pos.p, ctx->est[0].pos.cap);
    sub->info = ctx->info;
    sub->prepared = true;
    CUS(cudaStreamWaitEvent(sub->stream, ctx->ev_uni, 0));
    for (int which = 0; which < 2; ++which) {
      rc = build_estimator(sub, which, which == 0 ? w_below : w_above, sub->stream);
      if (rc) return rc;
    }
    sub->built = true;
    sub->U.alias(ctx->U.as<double>() + (size_t)j * per_col, (size_t)per_col * 8);
    CUS(cudaStreamWaitEvent(sub->stream, ctx->ev_u, 0));
    sub->n_asks = 1;
    rc = ensure_candidate_buffers(sub, C);
    if (rc) return rc;
    CUS(sub->out_x.ensure(8));
    CUS(sub->out_acq.ensure(8));
    CUS(sub->out_best.ensure(8));
    rc = launch_sample_select(sub, 1, false, false);
    if (rc) return rc;
    CUS(cudaMemcpyAsync(ctx->out_x.as<double>() + j, sub->out_x.p, 8, cudaMemcpyDeviceToDevice, sub->stream));
    CUS(cudaMemcpyAsync(ctx->out_acq.as<double>() + j, sub->out_acq.p, 8, cudaMemcpyDeviceToDevice, sub->stream));
    CUS(cudaMemcpyAsync(ctx->out_best.as<int64_t>() + j, sub->out_best.p, 8, cudaMemcpyDeviceToDevice, sub->stream));
    CUS(cudaEventRecord(sub->ev_join, sub->stream));
#undef CUS
    return TPE_OK;
  };
  static const int n_threads_env = [] { const char* v = getenv("TPE_UNI_THREADS"); return v ? atoi(v) : 6; }();
  const int T = std::max(1, std::min(n_threads_env, (int)n_cols));
  std::vector<int> rcs((size_t)n_cols, TPE_OK);
  if (T == 1) {
    for (int j = 0; j < n_cols; ++j) rcs[(size_t)j] = issue_column(j);
  } else {
    std::vector<std::thread> pool;
    for (int w = 0; w < T; ++w)
      pool.emplace_back([&, w] { for (int j = w; j < n_cols; j += T) rcs[(size_t)j] = issue_column(j); });
    for (auto& th : pool) th.join();
  }
  for (int j = 0; j < n_cols; ++j) {
    if (rcs[(size_t)j]) {
      ctx->err = ctx->uni_sub[(size_t)j]->err;
      for (int q = 0; q < n_cols; ++q) cudaStreamSynchronize(ctx->uni_sub[(size_t)q]->stream);
      return rcs[(size_t)j];
    }
    CU(cudaStreamWaitEvent(ctx->stream, ctx->uni_sub[(size_t)j]->ev_join, 0));
    launches += ctx->uni_sub[(size_t)j]->launch_counter;
  }
  if (dev_rng) CU(cudaMemcpyAsync(ctx->mt_host, ctx->mt_state.p, (size_t)625 * 4, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaEventRecord(ctx->ev[8], ctx->stream));
  CU(cudaMemcpyAsync(out_x, ctx->out_x.p, (size_t)n_cols * 8, cudaMemcpyDeviceToHost, ctx->stream));
  if (out_acq) CU(cudaMemcpyAsync(out_acq, ctx->out_acq.p, (size_t)n_cols * 8, cudaMemcpyDeviceToHost, ctx->stream));
  if (out_best) CU(cudaMemcpyAsync(out_best, ctx->out_best.p, (size_t)n_cols * 8, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  if (dev_rng) ctx->mt_host_valid = true;
  ctx->spec_pending = false;
  for (int i = 0; i < 9; ++i) ctx->ms[i] = 0.0f;
  cudaEventElapsedTime(&ctx->ms[8], ctx->ev[0], ctx->ev[8]);
  ctx->launches = launches;
  ctx->last_kernel = ctx->uni_sub[0]->last_kernel;
  ctx->prepared = ctx->built = ctx->sampled = false;   // the per-column state lives in the column contexts
  return TPE_OK;
}

int tpe_suggest_univariate_batch(tpe_ctx* ctx, const tpe_cfg* cfg, const int32_t* cols, int32_t n_cols,
                                 const double* w_below, const double* w_above, const double* uniforms, double* out_x,
                                 double* out_acq, int64_t* out_best) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  return uni_batch_locked(ctx, cfg, cols, n_cols, w_below, w_above, uniforms, out_x, out_acq, out_best, false);
}

int tpe_suggest_univariate_batch_async(tpe_ctx* ctx, const tpe_cfg* cfg, const int32_t* cols, int32_t n_cols,
                                       const double* w_below, const double* w_above, const double* uniforms) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  return uni_batch_locked(ctx, cfg, cols, n_cols, w_below, w_above, uniforms, nullptr, nullptr, nullptr, true);
}

int tpe_collect_univariate(tpe_ctx* ctx, double* out_x, double* out_acq, int64_t* out_best) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (ctx->deferred_uni <= 0)
    return fail(ctx, TPE_E_STATE, "tpe_collect_univariate needs a pending tpe_suggest_univariate_batch_async");
  if (set_device(ctx, /*join=*/false)) return TPE_E_CUDA;
  const int64_t n = ctx->deferred_uni;
  CU(cudaStreamSynchronize(ctx->stream));
  ctx->deferred_uni = 0;
  if (ctx->deferred_uni_rng) ctx->mt_host_valid = true;
  for (int i = 0; i < 9; ++i) ctx->ms[i] = 0.0f;
  cudaEventElapsedTime(&ctx->ms[8], ctx->ev[0], ctx->ev[8]);
  const char* h = static_cast<const char*>(ctx->res_host);
  if (out_x) memcpy(out_x, h, (size_t)n * 8);
  if (out_acq) memcpy(out_acq, h + (size_t)n * 8, (size_t)n * 8);
  if (out_best) memcpy(out_best, h + (size_t)n * 16, (size_t)n * 8);
  return TPE_OK;
}

int tpe_get_split_info(tpe_ctx* ctx, tpe_split_info* info) {
  if (!ctx || !info) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (!ctx->prepared) return fail(ctx, TPE_E_STATE, "tpe_prepare must precede tpe_get_split_info");
  *info = ctx->info;
  return TPE_OK;
}

int tpe_get_split(tpe_ctx* ctx, int64_t* below_rows, int64_t* above_rows) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (!ctx->prepared) return fail(ctx, TPE_E_STATE, "tpe_prepare must precede tpe_get_split");
  if (set_device(ctx)) return TPE_E_CUDA;
  if (below_rows && ctx->est[0].n)
    CU(cudaMemcpyAsync(below_rows, ctx->est[0].rows.p, (size_t)ctx->est[0].n * 8, cudaMemcpyDeviceToHost, ctx->stream));
  if (above_rows && ctx->est[1].n)
    CU(cudaMemcpyAsync(above_rows, ctx->est[1].rows.p, (size_t)ctx->est[1].n * 8, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return TPE_OK;
}

int tpe_get_mixture(tpe_ctx* ctx, int which, double* weights, double* mu, double* sigma) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (!ctx->built) return fail(ctx, TPE_E_STATE, "tpe_build must precede tpe_get_mixture");
  if (which < 0 || which > 1) return fail(ctx, TPE_E_INVALID, "which must be 0 or 1");
  if (set_device(ctx)) return TPE_E_CUDA;
  Estimator& e = ctx->est[which];
  if (weights) CU(cudaMemcpyAsync(weights, e.w.p, (size_t)e.K * 8, cudaMemcpyDeviceToHost, ctx->stream));
  if (mu) CU(cudaMemcpyAsync(mu, e.mu.p, (size_t)e.K * ctx->pc * 8, cudaMemcpyDeviceToHost, ctx->stream));
  if (sigma) CU(cudaMemcpyAsync(sigma, e.sigma.p, (size_t)e.K * ctx->pc * 8, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return TPE_OK;
}

int tpe_get_candidates(tpe_ctx* ctx, double* samples, double* logl, double* logg) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (!ctx->sampled) return fail(ctx, TPE_E_STATE, "tpe_sample_and_select must precede tpe_get_candidates");
  if (set_device(ctx)) return TPE_E_CUDA;
  if (samples) CU(cudaMemcpyAsync(samples, ctx->S.p, (size_t)ctx->Ct * ctx->pc * 8, cudaMemcpyDeviceToHost, ctx->stream));
  if (logl) CU(cudaMemcpyAsync(logl, ctx->logl.p, (size_t)ctx->Ct * 8, cudaMemcpyDeviceToHost, ctx->stream));
  if (logg) CU(cudaMemcpyAsync(logg, ctx->logg.p, (size_t)ctx->Ct * 8, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return TPE_OK;
}

int tpe_logpdf(tpe_ctx* ctx, int which, const double* x, int64_t n, double* out) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (!ctx->built) return fail(ctx, TPE_E_STATE, "tpe_build must precede tpe_logpdf");
  if (which < 0 || which > 1 || !x || !out || n <= 0) return fail(ctx, TPE_E_INVALID, "bad logpdf arguments");
  if (set_device(ctx)) return TPE_E_CUDA;
  cudaStream_t st = ctx->stream;
  int rc = ensure_candidate_buffers(ctx, n);
  if (rc) return rc;
  ctx->sampled = false;
  ctx->user_points = true;
  CU(cudaMemcpyAsync(ctx->S.p, x, (size_t)n * ctx->pc * 8, cudaMemcpyHostToDevice, st));
  k_prep_points<<<grid_for(n * ctx->pc, 256, ctx->sm_count * 8), 256, 0, st>>>(
      ctx->S.as<double>(), n, ctx->cols.as<ColMeta>(), ctx->pc, ctx->fast ? ctx->xT.as<double>() : nullptr,
      ctx->ct_stride, ctx->oob.as<uint8_t>());
  ctx->launch_counter++;
  rc = run_logpdf(ctx, which, n);
  if (rc) return rc;
  Estimator& e = ctx->est[which];
  k_finish_logpdf<<<grid_for(n, 256, ctx->sm_count * 8), 256, 0, st>>>(
      e.part.as<double2>(), e.nsplit, ctx->ct_stride, ctx->fast ? ctx->oob.as<uint8_t>() : nullptr,
      e.fix.as<double2>(), n, ctx->logl.as<double>());
  ctx->launch_counter++;
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(out, ctx->logl.p, (size_t)n * 8, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  return TPE_OK;
}

int tpe_last_timing(tpe_ctx* ctx, float* ms9, int32_t* launches) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (ms9)
    for (int i = 0; i < 9; ++i) ms9[i] = ctx->ms[i];
  if (launches) *launches = ctx->launches;
  return TPE_OK;
}

int tpe_probe_fp64_tflops(tpe_ctx* ctx, double* tflops) {
  if (!ctx || !tflops) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (set_device(ctx)) return TPE_E_CUDA;
  const int blocks = ctx->sm_count * 4, threads = 512, iters = 20000;
  DevBuf out;
  CU(out.ensure((size_t)blocks * threads * 8));
  float best = 1e30f;
  for (int rep = 0; rep < 4; ++rep) {
    CU(cudaEventRecord(ctx->ev[0], ctx->stream));
    k_fp64_probe<<<blocks, threads, 0, ctx->stream>>>(out.as<double>(), iters);
    CU(cudaEventRecord(ctx->ev[1], ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    float ms = 0;
    cudaEventElapsedTime(&ms, ctx->ev[0], ctx->ev[1]);
    if (rep > 0 && ms < best) best = ms;
  }
  out.release();
  const double flops = 2.0 * 8.0 * (double)iters * blocks * threads;
  *tflops = flops / (best * 1e-3) / 1e12;
  return TPE_OK;
}

// ---- Gaussian process of the terminator's regret bound (tpe_gp.cuh) ------------------------------------------------
static constexpr int64_t kGpQmax = 1024;   // query rows per posterior chunk (cross covariance rows held in A)
static constexpr int kGpGradBlocks = 1024; // CTAs of k_gp_grad at most: fixed, so the partial sums' order is too

static int64_t gp_grad_blocks(int64_t n) {
  const int64_t total = n * (n + 1) / 2;
  return std::min<int64_t>((total + gp::GRAD_THREADS - 1) / gp::GRAD_THREADS, kGpGradBlocks);
}

static void gp_gemm(cudaStream_t st, const double* A, int64_t lda, const double* B, int64_t ldb, double* out,
                    int64_t ldc, int64_t M, int64_t N, int64_t K, double alpha, int flags) {
  if (M <= 0 || N <= 0) return;
  const dim3 grid((unsigned)((N + gp::NB - 1) / gp::NB), (unsigned)((M + gp::NB - 1) / gp::NB));
  gp::k_gp_gemm<<<grid, 128, 0, st>>>(A, lda, B, ldb, out, ldc, (int)M, (int)N, (int)K, alpha, flags);
}

// C at gp.prm into A, then L (right-looking blocked Cholesky) in A and L^-1 (blocked TRTRI) in B; gp.fail is set when
// a pivot is <= 0 or NaN.  Then u = L^-1 y, [sum log L_ii, u.u] in gp.scal and alpha = L^-T u.
static void gp_factor(tpe_ctx* ctx) {
  GpState& g = ctx->gp;
  cudaStream_t st = ctx->stream;
  const int64_t n = g.n;
  const int NB = gp::NB;
  cudaMemsetAsync(g.fail, 0, sizeof(int), st);
  const unsigned nt = (unsigned)((n + 31) / 32);
  gp::k_gp_cov<<<dim3(nt, nt), dim3(32, 32), 0, st>>>(g.X, g.cat, g.prm, g.P, (int)n, g.A);
  double *A = g.A, *B = g.B;
  for (int64_t k0 = 0; k0 < n; k0 += NB) {
    const int64_t nb = std::min<int64_t>(NB, n - k0), r0 = k0 + nb, m = n - r0;
    gp::k_gp_potrf_diag<<<1, 256, 0, st>>>(A, B, (int)n, (int)k0, (int)nb, g.fail);
    if (m > 0) {
      // panel TRSM in place: L21 = A21 L11^-T, with L11^-1 from the diagonal block of B
      gp_gemm(st, A + r0 * n + k0, n, B + k0 * n + k0, n, A + r0 * n + k0, n, m, nb, nb, 1.0, 0);
      // trailing SYRK: A22 -= L21 L21^T over the lower triangle
      gp_gemm(st, A + r0 * n + k0, n, A + r0 * n + k0, n, A + r0 * n + r0, n, m, m, nb, -1.0,
              gp::GF_LOWER | gp::GF_ACCUM);
    }
  }
  // TRTRI, last block column first: L^-1[r0:, k0:r0] = -(L^-1[r0:, r0:] L[r0:, k0:r0]) L^-1[k0:r0, k0:r0]
  for (int64_t k0 = ((n - 1) / NB) * NB; k0 >= 0; k0 -= NB) {
    const int64_t nb = std::min<int64_t>(NB, n - k0), r0 = k0 + nb, m = n - r0;
    if (m == 0) continue;
    gp_gemm(st, B + r0 * n + r0, n, A + r0 * n + k0, n, g.W, NB, m, nb, m, 1.0, gp::GF_TB | gp::GF_KHI_ROW);
    gp_gemm(st, g.W, NB, B + k0 * n + k0, n, B + r0 * n + k0, n, m, nb, nb, -1.0, gp::GF_TB);
  }
  gp::k_gp_trmv_lower<<<(unsigned)((n + 7) / 8), 256, 0, st>>>(B, g.y, (int)n, g.u);
  gp::k_gp_stats<<<1, 256, 0, st>>>(A, g.u, (int)n, g.scal);
  gp::k_gp_trmv_lower_t<<<(unsigned)((n + 31) / 32), 256, 0, st>>>(B, g.u, (int)n, g.alpha);
}

// the allocations and uploads of tpe_gp_set_data; on failure the caller releases what was allocated
static int gp_upload(tpe_ctx* ctx, const double* X, const double* y, const uint8_t* is_categorical, int64_t n,
                     int32_t P, size_t a_elems, size_t b_elems, int64_t part) {
  GpState& g = ctx->gp;
  g.n = n;
  g.P = P;
  CU(cudaMalloc(&g.A, a_elems * 8));
  CU(cudaMalloc(&g.B, b_elems * 8));
  CU(cudaMalloc(&g.W, (size_t)n * gp::NB * 8));
  CU(cudaMalloc(&g.X, (size_t)n * P * 8));
  CU(cudaMalloc(&g.y, n * 8));
  CU(cudaMalloc(&g.u, n * 8));
  CU(cudaMalloc(&g.alpha, n * 8));
  CU(cudaMalloc(&g.prm, (P + 2) * 8));
  CU(cudaMalloc(&g.part, part * 8));
  g.part_cap = part;
  CU(cudaMalloc(&g.scal, 2 * 8));
  CU(cudaMalloc(&g.grad, (P + 2) * 8));
  CU(cudaMalloc(&g.cat, P));
  CU(cudaMalloc(&g.fail, sizeof(int)));
  std::vector<uint8_t> cat(P);
  for (int d = 0; d < P; ++d) cat[d] = is_categorical[d] ? 1 : 0;
  CU(cudaMemsetAsync(g.B, 0, b_elems * 8, ctx->stream));   // L^-1: the upper triangle stays zero
  CU(cudaMemcpyAsync(g.X, X, (size_t)n * P * 8, cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaMemcpyAsync(g.y, y, n * 8, cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaMemcpyAsync(g.cat, cat.data(), P, cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return TPE_OK;
}

// replaces GPRegressor(...) construction (optuna/_gp/gp.py:94-118): the training data of the fit
int tpe_gp_set_data(tpe_ctx* ctx, const double* X, const double* y, const uint8_t* is_categorical, int64_t n,
                    int32_t P) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  ctx->gp.conditioned = false;
  if (n < 1 || P < 1 || n > (int64_t)1 << 30) return fail(ctx, TPE_E_INVALID, "bad GP sizes (n %lld, P %d)", (long long)n, P);
  if (!X || !y || !is_categorical) return fail(ctx, TPE_E_INVALID, "bad GP arguments");
  for (int64_t i = 0; i < n * P; ++i)
    if (!std::isfinite(X[i])) return fail(ctx, TPE_E_INVALID, "GP inputs hold a non-finite value");
  for (int64_t i = 0; i < n; ++i)
    if (!std::isfinite(y[i])) return fail(ctx, TPE_E_INVALID, "GP targets hold a non-finite value");
  if (set_device(ctx)) return TPE_E_CUDA;
  GpState& g = ctx->gp;
  g.release();
  const int64_t npass = (P + gp::GRAD_DC - 1) / gp::GRAD_DC;
  const int64_t part = std::max<int64_t>(npass * kGpGradBlocks * (gp::GRAD_DC + 2), kGpQmax * ((n + gp::NB - 1) / gp::NB));
  const size_t a_elems = (size_t)std::max<int64_t>(n, kGpQmax) * n, b_elems = (size_t)n * n;
  // A, B, the TRTRI panel, X / y / u / alpha, the partial sums and scalars, and the posterior's query buffers for
  // the evaluator's n + 2048 points (Xq, ucb, lcb).  The gradient buffers of tpe_gp_query are allocated and checked
  // by the first query that asks for gradients.
  const size_t n_query = (size_t)n + 2048;
  const size_t need = 8 * (a_elems + b_elems + (size_t)n * gp::NB + (size_t)n * (P + 3) + (size_t)part + 3 * (P + 2) +
                           2 + n_query * (P + 2)) + P + sizeof(int);
  size_t free_b = 0, total_b = 0;
  CU(cudaMemGetInfo(&free_b, &total_b));
  if (need > free_b)
    return fail(ctx, TPE_E_INVALID,
                "the Gaussian process over n = %lld points needs %.2f GB of device memory (two n x n fp64 matrices), "
                "device %d has %.2f GB free",
                (long long)n, need / 1e9, ctx->device, free_b / 1e9);
  const int rc = gp_upload(ctx, X, y, is_categorical, n, P, a_elems, b_elems, part);
  if (rc != TPE_OK) {
    // a partial allocation (free memory can shrink after the check on a shared device) leaves no usable state
    cudaStreamSynchronize(ctx->stream);
    g.release();
    return rc;
  }
  g.ready = true;
  return TPE_OK;
}

// The body of tpe_gp_loss and tpe_gp_loss_fixed_noise, called under the context lock with the arguments checked:
// l_d = exp(raw_d), ks = exp(raw_P), noise_var = noise_excess + noise_base.  The gradient in raw_{P+1} is
// 1/2 noise_excess sum_i W_ii, so noise_excess = 0 (the noise held fixed) makes it 0.
static int gp_loss_run(tpe_ctx* ctx, const double* raw, double noise_excess, double noise_base, double* loss,
                       double* grad) {
  GpState& g = ctx->gp;
  const int P = g.P;
  g.conditioned = false;   // B and prm are overwritten
  if (set_device(ctx)) return TPE_E_CUDA;
  std::vector<double> prm(P + 2);
  for (int d = 0; d < P; ++d) prm[d] = std::exp(raw[d]);
  prm[P] = std::exp(raw[P]);
  prm[P + 1] = noise_excess + noise_base;
  // a NaN or +inf raw parameter (a line-search iterate) makes the reference's covariance non-finite and its
  // Cholesky fail: the same error here, so that the fit retries and falls back the same way
  for (int d = 0; d < P + 2; ++d)
    if (!std::isfinite(prm[d]))
      return fail(ctx, TPE_E_NOTPD, "the GP covariance is not positive definite (non-finite kernel parameters)");
  cudaStream_t st = ctx->stream;
  CU(cudaMemcpyAsync(g.prm, prm.data(), (P + 2) * 8, cudaMemcpyHostToDevice, st));
  gp_factor(ctx);
  const int64_t n = g.n;
  // C^-1 = L^-T L^-1 over the lower triangle, into A
  gp_gemm(st, g.B, n, g.B, n, g.A, n, n, n, n, 1.0, gp::GF_TA | gp::GF_TB | gp::GF_LOWER | gp::GF_KLO_ROW);
  const int64_t nblk = gp_grad_blocks(n);
  for (int d0 = 0; d0 < P; d0 += gp::GRAD_DC) {
    double* part = g.part + (int64_t)(d0 / gp::GRAD_DC) * nblk * (gp::GRAD_DC + 2);
    gp::k_gp_grad<gp::GRAD_DC><<<(unsigned)nblk, gp::GRAD_THREADS, 0, st>>>(g.A, g.X, g.cat, g.prm, g.alpha, P,
                                                                           (int)n, d0, part);
    gp::k_gp_grad_finish<gp::GRAD_DC><<<1, 32, 0, st>>>(part, (int)nblk, g.prm, P, d0, g.grad);
  }
  gp::k_gp_grad_tail<<<1, 1, 0, st>>>(g.prm, noise_excess, P, g.grad);
  CU(cudaGetLastError());
  int failed = 0;
  double scal[2];
  CU(cudaMemcpyAsync(&failed, g.fail, sizeof(int), cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(scal, g.scal, 2 * 8, cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(grad, g.grad, (P + 2) * 8, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  if (failed) return fail(ctx, TPE_E_NOTPD, "the GP covariance is not positive definite (Cholesky pivot <= 0 or NaN)");
  // marginal_log_likelihood's order: (logdet_part + const) + quad_part, negated
  const double mll = (-scal[0] + -0.5 * (double)n * std::log(2.0 * M_PI)) + -0.5 * scal[1];
  *loss = -mll;
  return TPE_OK;
}

// replaces loss_func of GPRegressor._fit_kernel_params without the prior (optuna/_gp/gp.py:312-327, with
// marginal_log_likelihood :252-285 and its autograd backward): -log p(y | raw) and its gradient in raw
int tpe_gp_loss(tpe_ctx* ctx, const double* raw, double minimum_noise, double* loss, double* grad) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (!ctx->gp.ready) return fail(ctx, TPE_E_STATE, "no GP data (tpe_gp_set_data)");
  if (!raw || !loss || !grad) return fail(ctx, TPE_E_INVALID, "bad GP loss arguments");
  if (!std::isfinite(minimum_noise) || minimum_noise < 0.0) return fail(ctx, TPE_E_INVALID, "bad minimum noise");
  return gp_loss_run(ctx, raw, std::exp(raw[ctx->gp.P + 1]), minimum_noise, loss, grad);
}

// the same with deterministic_objective=True (gp.py:317-321): the noise is noise_var, raw[P + 1] is not read and
// grad[P + 1] = 0
int tpe_gp_loss_fixed_noise(tpe_ctx* ctx, const double* raw, double noise_var, double* loss, double* grad) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (!ctx->gp.ready) return fail(ctx, TPE_E_STATE, "no GP data (tpe_gp_set_data)");
  if (!raw || !loss || !grad) return fail(ctx, TPE_E_INVALID, "bad GP loss arguments");
  if (!std::isfinite(noise_var) || noise_var < 0.0) return fail(ctx, TPE_E_INVALID, "bad noise variance");
  return gp_loss_run(ctx, raw, 0.0, noise_var, loss, grad);
}

// Query buffers for m rows: Xq and the two value outputs (ucb / lcb, or mean / var)
static int gp_query_buffers(tpe_ctx* ctx, int64_t m) {
  GpState& g = ctx->gp;
  if (m <= g.xq_cap) return TPE_OK;
  for (double** p : {&g.Xq, &g.ucb, &g.lcb}) {
    if (*p) cudaFree(*p);
    *p = nullptr;
  }
  g.xq_cap = 0;
  CU(cudaMalloc(&g.Xq, (size_t)m * g.P * 8));
  CU(cudaMalloc(&g.ucb, m * 8));
  CU(cudaMalloc(&g.lcb, m * 8));
  g.xq_cap = m;
  return TPE_OK;
}

// The gradient outputs of one query chunk (NB rows x P each), allocated by the first query that asks for gradients:
// the posterior calls never touch them
static int gp_grad_buffers(tpe_ctx* ctx) {
  GpState& g = ctx->gp;
  if (g.dmean) return TPE_OK;
  const size_t bytes = (size_t)gp::NB * g.P * 8;
  size_t free_b = 0, total_b = 0;
  CU(cudaMemGetInfo(&free_b, &total_b));
  if (2 * bytes > free_b)
    return fail(ctx, TPE_E_INVALID, "the GP posterior gradient needs %zu bytes of device memory, device %d has %zu free",
                2 * bytes, ctx->device, free_b);
  if (g.dvar) cudaFree(g.dvar);   // left by an earlier call whose second allocation failed
  g.dvar = nullptr;
  CU(cudaMalloc(&g.dvar, bytes));   // dvar first: dmean != nullptr marks both allocated
  CU(cudaMalloc(&g.dmean, bytes));
  return TPE_OK;
}

// The query rows of g.Xq against the factor in B, alpha and prm (A is scratch).  Per chunk of rows (kGpQmax, or NB
// with grad): the cross covariance into A, the squared norms of L^-1 k* and k_gp_post_finish (moments: mean / var
// into ucb / lcb, else mean +- sqrt(beta var)).  Every row's values depend on that row alone, so they are the same
// whatever the chunk size.  With host gradient outputs dmean_h / dvar_h [m, P] (both or neither) also V = K L^-T into
// the n x 64 TRTRI panel (free after gp_factor), Wm = V L^-1 into rows NB .. 2 NB - 1 of A, k_gp_post_grad into the
// chunk's gradient buffers, and their copy to the host.  V repeats the O(Q n^2) product of the squared norms: the
// values must not depend on whether gradients are asked for, so they come from the same kernels either way.  With
// J > 0 the joint covariance of the first J rows into part [J * J].
static int gp_query_chunks(tpe_ctx* ctx, int64_t m, double beta, bool moments, int J, double* dmean_h,
                           double* dvar_h) {
  GpState& g = ctx->gp;
  cudaStream_t st = ctx->stream;
  const int P = g.P;
  const bool grad = dmean_h != nullptr;
  const int64_t n = g.n, ntiles = (n + gp::NB - 1) / gp::NB, qmax = grad ? gp::NB : kGpQmax;
  double* Wm = g.A + gp::NB * n;   // A has at least kGpQmax >= 2 NB rows of n
  for (int64_t q0 = 0; q0 < m; q0 += qmax) {
    const int64_t Q = std::min(qmax, m - q0);
    gp::k_gp_cross<<<dim3((unsigned)((n + 127) / 128), (unsigned)Q), 128, 0, st>>>(g.Xq + q0 * P, g.X, g.cat, g.prm,
                                                                                  P, (int)n, (int)Q, g.A);
    // squared norms of L^-1 k*, per query and column tile
    gp_gemm(st, g.A, n, g.B, n, g.part, 0, Q, n, n, 1.0, gp::GF_KHI_COL | gp::GF_SQSUM);
    gp::k_gp_post_finish<<<(unsigned)((Q + 7) / 8), 256, 0, st>>>(g.A, g.alpha, g.part, (int)ntiles, g.prm, P, (int)n,
                                                                  (int)Q, beta, moments, g.ucb + q0, g.lcb + q0);
    if (grad) {
      gp_gemm(st, g.A, n, g.B, n, g.W, n, Q, n, n, 1.0, gp::GF_KHI_COL);
      gp_gemm(st, g.W, n, g.B, n, Wm, n, Q, n, n, 1.0, gp::GF_TB | gp::GF_KLO_COL);
      const dim3 grid((unsigned)Q, (unsigned)((P + gp::GRAD_DC - 1) / gp::GRAD_DC));
      gp::k_gp_post_grad<gp::GRAD_DC><<<grid, gp::GRAD_THREADS, 0, st>>>(
          g.Xq + q0 * P, g.X, g.cat, g.prm, g.alpha, Wm, g.part, (int)ntiles, P, (int)n, g.dmean, g.dvar);
      // stream order: the next chunk's k_gp_post_grad writes the buffers after these copies have read them
      CU(cudaMemcpyAsync(dmean_h + q0 * P, g.dmean, (size_t)Q * P * 8, cudaMemcpyDeviceToHost, st));
      CU(cudaMemcpyAsync(dvar_h + q0 * P, g.dvar, (size_t)Q * P * 8, cudaMemcpyDeviceToHost, st));
    }
    if (q0 == 0 && J > 0) {
      // V = K L^-T for the first J rows (J <= min(m, 64), so all in this chunk) into the n x 64 TRTRI panel
      // buffer, free after gp_factor
      gp_gemm(st, g.A, n, g.B, n, g.W, n, J, n, n, 1.0, gp::GF_KHI_COL);
    }
  }
  if (J > 0)   // after the last chunk's k_gp_post_finish has read g.part (>= 18 432 entries, see tpe_gp_set_data)
    gp::k_gp_joint_cov<<<(unsigned)((J * J + 7) / 8), 256, 0, st>>>(g.Xq, g.W, g.cat, g.prm, P, (int)n, J, g.part);
  return TPE_OK;
}

// The body of tpe_gp_posterior and tpe_gp_posterior_moments, called under the context lock with the arguments
// checked: factorise at params, then gp_query_chunks.  The factor in B is this call's: tpe_gp_query needs a new
// tpe_gp_condition.
static int gp_posterior_run(tpe_ctx* ctx, const double* params, const double* Xq, int64_t m, double beta,
                            bool moments, int J, double* out0, double* out1, double* cov) {
  GpState& g = ctx->gp;
  const int P = g.P;
  g.conditioned = false;
  if (set_device(ctx)) return TPE_E_CUDA;
  cudaStream_t st = ctx->stream;
  const int rc = gp_query_buffers(ctx, m);
  if (rc != TPE_OK) return rc;
  CU(cudaMemcpyAsync(g.prm, params, (P + 2) * 8, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(g.Xq, Xq, (size_t)m * P * 8, cudaMemcpyHostToDevice, st));
  gp_factor(ctx);
  gp_query_chunks(ctx, m, beta, moments, J, nullptr, nullptr);   // without gradients it makes no call that can fail
  CU(cudaGetLastError());
  int failed = 0;
  CU(cudaMemcpyAsync(&failed, g.fail, sizeof(int), cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(out0, g.ucb, m * 8, cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(out1, g.lcb, m * 8, cudaMemcpyDeviceToHost, st));
  if (J > 0) CU(cudaMemcpyAsync(cov, g.part, (size_t)J * J * 8, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  if (failed) return fail(ctx, TPE_E_NOTPD, "the GP covariance is not positive definite (Cholesky pivot <= 0 or NaN)");
  return TPE_OK;
}

static int gp_params_check(tpe_ctx* ctx, const double* params) {
  for (int d = 0; d < ctx->gp.P + 2; ++d)
    if (!std::isfinite(params[d])) return fail(ctx, TPE_E_INVALID, "kernel parameters hold a non-finite value");
  return TPE_OK;
}

static int gp_xq_check(tpe_ctx* ctx, const double* Xq, int64_t m) {
  for (int64_t i = 0; i < m * ctx->gp.P; ++i)
    if (!std::isfinite(Xq[i])) return fail(ctx, TPE_E_INVALID, "query points hold a non-finite value");
  return TPE_OK;
}

// the argument checks the two posterior entry points share
static int gp_posterior_check(tpe_ctx* ctx, const double* params, const double* Xq, int64_t m, bool ok) {
  GpState& g = ctx->gp;
  if (!g.ready) return fail(ctx, TPE_E_STATE, "no GP data (tpe_gp_set_data)");
  if (!params || !Xq || !ok || m < 1) return fail(ctx, TPE_E_INVALID, "bad GP posterior arguments");
  const int rc = gp_params_check(ctx, params);
  return rc != TPE_OK ? rc : gp_xq_check(ctx, Xq, m);
}

// replaces GPRegressor._cache_matrix + posterior (optuna/_gp/gp.py:124-149, 215-250) and UCB / LCB.eval_acqf
// (optuna/_gp/acqf.py:185-214): mean +- sqrt(beta var) at m query points, for params = [l_1 .. l_P, ks, noise_var]
int tpe_gp_posterior(tpe_ctx* ctx, const double* params, const double* Xq, int64_t m, double beta, double* ucb,
                     double* lcb) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  const int rc = gp_posterior_check(ctx, params, Xq, m, ucb && lcb);
  if (rc != TPE_OK) return rc;
  if (!std::isfinite(beta) || beta < 0.0) return fail(ctx, TPE_E_INVALID, "bad beta");
  return gp_posterior_run(ctx, params, Xq, m, beta, false, 0, ucb, lcb, nullptr);
}

// replaces GPRegressor._cache_matrix + posterior (gp.py:124-149, 215-250): mean and var at m query points, and with
// n_joint in [2, 64] the joint covariance of the first n_joint of them (joint=True)
int tpe_gp_posterior_moments(tpe_ctx* ctx, const double* params, const double* Xq, int64_t m, int32_t n_joint,
                             double* mean, double* var, double* cov) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  const int rc = gp_posterior_check(ctx, params, Xq, m, mean && var);
  if (rc != TPE_OK) return rc;
  const bool joint_ok = n_joint == 0 ? cov == nullptr
                                     : (n_joint >= 2 && n_joint <= gp::NB && n_joint <= m && cov != nullptr);
  if (!joint_ok) return fail(ctx, TPE_E_INVALID, "bad joint covariance request (n_joint %d, m %lld)", n_joint,
                             (long long)m);
  return gp_posterior_run(ctx, params, Xq, m, 0.0, true, n_joint, mean, var, cov);
}

// replaces GPRegressor._cache_matrix (gp.py:124-149): factorise once at params and keep L^-1 and alpha for
// tpe_gp_query
int tpe_gp_condition(tpe_ctx* ctx, const double* params) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  GpState& g = ctx->gp;
  if (!g.ready) return fail(ctx, TPE_E_STATE, "no GP data (tpe_gp_set_data)");
  if (!params) return fail(ctx, TPE_E_INVALID, "bad GP condition arguments");
  const int rc = gp_params_check(ctx, params);
  if (rc != TPE_OK) return rc;
  g.conditioned = false;
  if (set_device(ctx)) return TPE_E_CUDA;
  cudaStream_t st = ctx->stream;
  CU(cudaMemcpyAsync(g.prm, params, (g.P + 2) * 8, cudaMemcpyHostToDevice, st));
  gp_factor(ctx);
  CU(cudaGetLastError());
  int failed = 0;
  CU(cudaMemcpyAsync(&failed, g.fail, sizeof(int), cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  if (failed) return fail(ctx, TPE_E_NOTPD, "the GP covariance is not positive definite (Cholesky pivot <= 0 or NaN)");
  g.conditioned = true;
  ++ctx->gp_generation;
  return TPE_OK;
}

// replaces GPRegressor.posterior (gp.py:215-250) and its autograd backward in x, against the factor of
// tpe_gp_condition: mean and var at m query points and, with dmean / dvar, their gradients in the query point
int tpe_gp_query(tpe_ctx* ctx, const double* Xq, int64_t m, double* mean, double* var, double* dmean,
                 double* dvar) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  GpState& g = ctx->gp;
  if (!g.ready) return fail(ctx, TPE_E_STATE, "no GP data (tpe_gp_set_data)");
  if (!g.conditioned) return fail(ctx, TPE_E_STATE, "the GP is not conditioned (tpe_gp_condition)");
  if (!Xq || !mean || !var || m < 1 || (dmean == nullptr) != (dvar == nullptr))
    return fail(ctx, TPE_E_INVALID, "bad GP query arguments");
  int rc = gp_xq_check(ctx, Xq, m);
  if (rc != TPE_OK) return rc;
  if (set_device(ctx)) return TPE_E_CUDA;
  rc = gp_query_buffers(ctx, m);
  if (rc == TPE_OK && dmean) rc = gp_grad_buffers(ctx);
  if (rc != TPE_OK) return rc;
  cudaStream_t st = ctx->stream;
  CU(cudaMemcpyAsync(g.Xq, Xq, (size_t)m * g.P * 8, cudaMemcpyHostToDevice, st));
  rc = gp_query_chunks(ctx, m, 0.0, true, 0, dmean, dvar);
  if (rc != TPE_OK) return rc;
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(mean, g.ucb, m * 8, cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(var, g.lcb, m * 8, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  return TPE_OK;
}

// ---- log-EHVI of GPSampler's multi-objective acquisition (tpe_ehvi.cuh) ----------------------------------------------
// ---- Many Gaussian processes at once (tpe_gpbatch.cuh) -------------------------------------------------------------
static size_t gpb_free_bytes(tpe_ctx* ctx) {
  size_t free_b = 0, total_b = 0;
  if (cudaMemGetInfo(&free_b, &total_b) != cudaSuccess) return 0;
  return free_b;
}

// The three kinds of batched call, by the per-job workspace they need
enum GpbCall { GPB_LOSS, GPB_BOUNDS, GPB_MOMENTS };

// Per-job workspace offsets (doubles) of a call: k_gpb_loss needs gpb::ws_doubles(n), k_gpb_bounds also n x NQ
// doubles of cross covariance, k_gpe_moments gpe::ws_doubles(n).  Jobs get their own workspace even when they name the
// same GP.
static int64_t gpb_ws_layout(const GpBatchState& s, const int32_t* gp_idx, int64_t k, GpbCall call,
                             std::vector<int64_t>& wsoff, size_t* smem) {
  int64_t tot = 0;
  *smem = 0;
  wsoff.resize(k);
  for (int64_t b = 0; b < k; ++b) {
    const int64_t n = s.off[gp_idx[b] + 1] - s.off[gp_idx[b]];
    wsoff[b] = tot;
    tot += call == GPB_MOMENTS ? gpe::ws_doubles(n) : gpb::ws_doubles(n) + (call == GPB_BOUNDS ? n * gpb::NQ : 0);
    *smem = std::max(*smem, gpb::smem_bytes((int)n, s.P));
  }
  return tot;
}

static int gpb_check_jobs(tpe_ctx* ctx, int64_t k, const int32_t* gp_idx) {
  const GpBatchState& s = ctx->gpb;
  if (!s.ready) return fail(ctx, TPE_E_STATE, "no batched GP data (tpe_gp_batch_set)");
  if (k < 1 || !gp_idx) return fail(ctx, TPE_E_INVALID, "bad batched GP call (k %lld)", (long long)k);
  for (int64_t b = 0; b < k; ++b)
    if (gp_idx[b] < 0 || gp_idx[b] >= s.n_gp)
      return fail(ctx, TPE_E_INVALID, "GP index %d out of range (%d GPs)", gp_idx[b], s.n_gp);
  return TPE_OK;
}

static int gpb_oom(tpe_ctx* ctx, const char* what, size_t need, int64_t nmax) {
  return fail(ctx, TPE_E_INVALID,
              "%s needs %zu bytes (%.2f GB) of device memory (largest GP: n = %lld), device %d has %zu bytes free",
              what, need, need / 1e9, (long long)nmax, ctx->device, gpb_free_bytes(ctx));
}

// Uploads the job list and sizes the per-job workspace and the launch's shared memory; the caller has checked the
// jobs.  Fails naming the bytes when the workspace does not fit in free device memory.
static int gpb_stage_jobs(tpe_ctx* ctx, int64_t k, const int32_t* gp_idx, GpbCall call, size_t extra,
                          size_t* smem) {
  GpBatchState& s = ctx->gpb;
  std::vector<int64_t> wsoff;
  const int64_t wsd = gpb_ws_layout(s, gp_idx, k, call, wsoff, smem);
  int64_t nmax = 0;
  for (int64_t b = 0; b < k; ++b) nmax = std::max(nmax, s.off[gp_idx[b] + 1] - s.off[gp_idx[b]]);
  const size_t need = (size_t)std::max<int64_t>(wsd, 1) * 8 + extra;
  const size_t have = s.ws.cap;
  if (need > have && need - have > gpb_free_bytes(ctx))
    return gpb_oom(ctx,
                   call == GPB_BOUNDS ? "the batched GP bounds"
                                      : call == GPB_MOMENTS ? "the batched GP moments" : "the batched GP loss",
                   need, nmax);
  cudaStream_t st = ctx->stream;
  CU(s.ws.ensure((size_t)std::max<int64_t>(wsd, 1) * 8));
  CU(s.wsoff.ensure(k * 8));
  CU(s.idx.ensure(k * 4));
  CU(s.status.ensure(k * 4));
  CU(cudaMemcpyAsync(s.wsoff.p, wsoff.data(), k * 8, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(s.idx.p, gp_idx, k * 4, cudaMemcpyHostToDevice, st));
  if (*smem > 48 * 1024) {
    CU(cudaFuncSetAttribute(gpb::k_gpb_loss, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)*smem));
    CU(cudaFuncSetAttribute(gpb::k_gpb_bounds, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)*smem));
    CU(cudaFuncSetAttribute(gpe::k_gpe_moments, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)*smem));
  }
  return TPE_OK;
}

// n_gp Gaussian processes over the rows offsets[i] .. offsets[i + 1] - 1 of X [N, P] / y [N]
int tpe_gp_batch_set(tpe_ctx* ctx, int32_t n_gp, const int64_t* offsets, int32_t P, const double* X, const double* y,
                     const uint8_t* is_categorical) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  GpBatchState& s = ctx->gpb;
  s.ready = false;
  if (n_gp < 1) return fail(ctx, TPE_E_INVALID, "no GPs in the batch (n_gp %d)", n_gp);
  if (P < 1) return fail(ctx, TPE_E_INVALID, "bad batched GP width (P %d)", P);
  if (!offsets || !X || !y || !is_categorical) return fail(ctx, TPE_E_INVALID, "bad batched GP arguments");
  if (offsets[0] != 0) return fail(ctx, TPE_E_INVALID, "batched GP offsets must start at 0");
  int64_t nmax = 0, wsd = 0;
  for (int32_t i = 0; i < n_gp; ++i) {
    const int64_t n = offsets[i + 1] - offsets[i];
    if (n < 1 || n > (int64_t)1 << 20)
      return fail(ctx, TPE_E_INVALID, "GP %d of the batch has n = %lld rows (needs 1 .. 2^20)", i, (long long)n);
    nmax = std::max(nmax, n);
    wsd += gpb::ws_doubles(n);
  }
  const int64_t N = offsets[n_gp];
  for (int64_t i = 0; i < N * P; ++i)
    if (!std::isfinite(X[i])) return fail(ctx, TPE_E_INVALID, "batched GP inputs hold a non-finite value");
  for (int64_t i = 0; i < N; ++i)
    if (!std::isfinite(y[i])) return fail(ctx, TPE_E_INVALID, "batched GP targets hold a non-finite value");
  if (set_device(ctx)) return TPE_E_CUDA;
  s.release();
  // the data, and the workspace of one loss call over every GP (n x n fp64 per GP above the shared-memory size)
  const size_t need = 8 * ((size_t)N * (P + 1) + (size_t)n_gp + 1 + (size_t)wsd) + P;
  if (need > gpb_free_bytes(ctx)) return gpb_oom(ctx, "the batch of Gaussian processes", need, nmax);
  cudaStream_t st = ctx->stream;
  std::vector<uint8_t> cat(P);
  for (int d = 0; d < P; ++d) cat[d] = is_categorical[d] ? 1 : 0;
  s.n_gp = n_gp;
  s.P = P;
  s.off.assign(offsets, offsets + n_gp + 1);
  CU(s.X.ensure((size_t)N * P * 8));
  CU(s.y.ensure((size_t)N * 8));
  CU(s.doff.ensure((size_t)(n_gp + 1) * 8));
  CU(s.cat.ensure(P));
  CU(cudaMemcpyAsync(s.X.p, X, (size_t)N * P * 8, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(s.y.p, y, (size_t)N * 8, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(s.doff.p, offsets, (size_t)(n_gp + 1) * 8, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(s.cat.p, cat.data(), P, cudaMemcpyHostToDevice, st));
  CU(cudaStreamSynchronize(st));
  s.ready = true;
  return TPE_OK;
}

// The body of tpe_gp_batch_loss and tpe_gp_batch_loss_fixed_noise, called under the context lock: job b's noise is
// exp(raw[b][P + 1]) + noise, or with fixed the constant noise with a noise excess of 0, which makes k_gpb_loss's raw
// noise gradient 1/2 * 0 * sum_i W_ii = 0 (k_gp_grad_tail's form, as tpe_gp_loss_fixed_noise gives it)
static int gpb_loss_run(tpe_ctx* ctx, int64_t k, const int32_t* gp_idx, const double* raw, double noise, bool fixed,
                        double* loss, double* grad, int32_t* status) {
  int rc = gpb_check_jobs(ctx, k, gp_idx);
  if (rc != TPE_OK) return rc;
  if (!raw || !loss || !grad || !status) return fail(ctx, TPE_E_INVALID, "bad batched GP loss arguments");
  if (!std::isfinite(noise) || noise < 0.0)
    return fail(ctx, TPE_E_INVALID, fixed ? "bad noise variance" : "bad minimum noise");
  GpBatchState& s = ctx->gpb;
  const int P = s.P;
  if (set_device(ctx)) return TPE_E_CUDA;
  size_t smem = 0;
  rc = gpb_stage_jobs(ctx, k, gp_idx, GPB_LOSS, 0, &smem);
  if (rc != TPE_OK) return rc;
  // the kernel parameters as tpe_gp_loss forms them on the host; a non-finite one is reported by the kernel
  std::vector<double> prm((size_t)k * (P + 2)), nexc(k);
  for (int64_t b = 0; b < k; ++b) {
    const double* r = raw + b * (P + 2);
    double* p = prm.data() + b * (P + 2);
    for (int d = 0; d <= P; ++d) p[d] = std::exp(r[d]);
    nexc[b] = fixed ? 0.0 : std::exp(r[P + 1]);
    p[P + 1] = nexc[b] + noise;
  }
  cudaStream_t st = ctx->stream;
  CU(s.prm.ensure(prm.size() * 8));
  CU(s.nexc.ensure(k * 8));
  CU(s.loss.ensure(k * 8));
  CU(s.grad.ensure(prm.size() * 8));
  CU(cudaMemcpyAsync(s.prm.p, prm.data(), prm.size() * 8, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(s.nexc.p, nexc.data(), k * 8, cudaMemcpyHostToDevice, st));
  gpb::k_gpb_loss<<<(unsigned)k, gpb::THREADS, smem, st>>>(
      s.X.as<double>(), s.y.as<double>(), s.doff.as<int64_t>(), s.cat.as<uint8_t>(), P, s.idx.as<int32_t>(),
      s.prm.as<double>(), s.nexc.as<double>(), s.ws.as<double>(), s.wsoff.as<int64_t>(), s.loss.as<double>(),
      s.grad.as<double>(), s.status.as<int32_t>());
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(loss, s.loss.p, k * 8, cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(grad, s.grad.p, prm.size() * 8, cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(status, s.status.p, k * 4, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  return TPE_OK;
}

// tpe_gp_loss for k jobs at once: job b is GP gp_idx[b] at raw[b] [P + 2]
int tpe_gp_batch_loss(tpe_ctx* ctx, int64_t k, const int32_t* gp_idx, const double* raw, double minimum_noise,
                      double* loss, double* grad, int32_t* status) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  return gpb_loss_run(ctx, k, gp_idx, raw, minimum_noise, false, loss, grad, status);
}

// tpe_gp_loss_fixed_noise for k jobs at once: the noise is noise_var, raw[b][P + 1] is not read, grad[b][P + 1] = 0
int tpe_gp_batch_loss_fixed_noise(tpe_ctx* ctx, int64_t k, const int32_t* gp_idx, const double* raw, double noise_var,
                                  double* loss, double* grad, int32_t* status) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  return gpb_loss_run(ctx, k, gp_idx, raw, noise_var, true, loss, grad, status);
}

// RegretBoundEvaluator's three maxima for k jobs: GP gp_idx[b] at params[b] [P + 2], beta[b], and its S sample rows
// samples[b] [S, P]
int tpe_gp_batch_bounds(tpe_ctx* ctx, int64_t k, const int32_t* gp_idx, const double* params, const double* beta,
                        int32_t S, const double* samples, double* out, int32_t* status) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  int rc = gpb_check_jobs(ctx, k, gp_idx);
  if (rc != TPE_OK) return rc;
  if (!params || !beta || !out || !status || S < 1 || !samples)
    return fail(ctx, TPE_E_INVALID, "bad batched GP bounds arguments");
  GpBatchState& s = ctx->gpb;
  const int P = s.P;
  for (int64_t b = 0; b < k; ++b)
    if (!std::isfinite(beta[b]) || beta[b] < 0.0) return fail(ctx, TPE_E_INVALID, "bad beta");
  const int64_t ns = k * (int64_t)S * P;
  for (int64_t i = 0; i < ns; ++i)
    if (!std::isfinite(samples[i])) return fail(ctx, TPE_E_INVALID, "sample points hold a non-finite value");
  if (set_device(ctx)) return TPE_E_CUDA;
  size_t smem = 0;
  rc = gpb_stage_jobs(ctx, k, gp_idx, GPB_BOUNDS, (size_t)ns * 8, &smem);
  if (rc != TPE_OK) return rc;
  cudaStream_t st = ctx->stream;
  CU(s.prm.ensure((size_t)k * (P + 2) * 8));
  CU(s.beta.ensure(k * 8));
  CU(s.Xs.ensure((size_t)ns * 8));
  CU(s.out.ensure(k * 3 * 8));
  CU(cudaMemcpyAsync(s.prm.p, params, (size_t)k * (P + 2) * 8, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(s.beta.p, beta, k * 8, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(s.Xs.p, samples, (size_t)ns * 8, cudaMemcpyHostToDevice, st));
  gpb::k_gpb_bounds<<<(unsigned)k, gpb::THREADS, smem, st>>>(
      s.X.as<double>(), s.y.as<double>(), s.doff.as<int64_t>(), s.cat.as<uint8_t>(), P, s.idx.as<int32_t>(),
      s.prm.as<double>(), s.beta.as<double>(), s.Xs.as<double>(), S, s.ws.as<double>(), s.wsoff.as<int64_t>(),
      s.out.as<double>(), s.status.as<int32_t>());
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(out, s.out.p, k * 3 * 8, cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(status, s.status.p, k * 4, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  return TPE_OK;
}

// EMMREvaluator's posterior terms for k jobs: GP gp_idx[b] at params[b] [P + 2], at its own train rows rows[b] [m]
int tpe_gp_batch_moments(tpe_ctx* ctx, int64_t k, const int32_t* gp_idx, const double* params, int32_t m,
                         const int32_t* rows, int32_t n_joint, double* mean, double* var, double* cov,
                         int32_t* status) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  int rc = gpb_check_jobs(ctx, k, gp_idx);
  if (rc != TPE_OK) return rc;
  if (!params || !rows || !mean || !var || !status)
    return fail(ctx, TPE_E_INVALID, "bad batched GP moments arguments");
  if (m < 1 || m > gpe::MQ)
    return fail(ctx, TPE_E_INVALID, "batched GP moments take 1 .. %d rows per job, got m = %d", gpe::MQ, m);
  if (!(n_joint == 0 ? cov == nullptr : (n_joint >= 2 && n_joint <= m && cov != nullptr)))
    return fail(ctx, TPE_E_INVALID, "bad joint covariance request (n_joint %d, m %d)", n_joint, m);
  GpBatchState& s = ctx->gpb;
  const int P = s.P;
  for (int64_t b = 0; b < k; ++b) {
    const int64_t n = s.off[gp_idx[b] + 1] - s.off[gp_idx[b]];
    for (int q = 0; q < m; ++q)
      if (rows[b * m + q] < 0 || rows[b * m + q] >= n)
        return fail(ctx, TPE_E_INVALID, "row index %d of job %lld out of range (GP %d has %lld rows)", rows[b * m + q],
                    (long long)b, gp_idx[b], (long long)n);
  }
  if (set_device(ctx)) return TPE_E_CUDA;
  size_t smem = 0;
  rc = gpb_stage_jobs(ctx, k, gp_idx, GPB_MOMENTS, 0, &smem);
  if (rc != TPE_OK) return rc;
  cudaStream_t st = ctx->stream;
  const int64_t J2 = (int64_t)n_joint * n_joint;
  CU(s.prm.ensure((size_t)k * (P + 2) * 8));
  CU(s.rows.ensure((size_t)k * m * 4));
  CU(s.out.ensure((size_t)k * (2 * m + J2) * 8));
  double* dmean = s.out.as<double>();
  double* dvar = dmean + k * m;
  double* dcov = dvar + k * m;
  CU(cudaMemcpyAsync(s.prm.p, params, (size_t)k * (P + 2) * 8, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(s.rows.p, rows, (size_t)k * m * 4, cudaMemcpyHostToDevice, st));
  gpe::k_gpe_moments<<<(unsigned)k, gpe::THREADS, smem, st>>>(
      s.X.as<double>(), s.y.as<double>(), s.doff.as<int64_t>(), s.cat.as<uint8_t>(), P, s.idx.as<int32_t>(),
      s.prm.as<double>(), s.rows.as<int32_t>(), m, n_joint, s.ws.as<double>(), s.wsoff.as<int64_t>(), dmean, dvar,
      dcov, s.status.as<int32_t>());
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(mean, dmean, (size_t)k * m * 8, cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(var, dvar, (size_t)k * m * 8, cudaMemcpyDeviceToHost, st));
  if (n_joint) CU(cudaMemcpyAsync(cov, dcov, (size_t)k * J2 * 8, cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(status, s.status.p, k * 4, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  return TPE_OK;
}

static constexpr int64_t kEhviPartDoubles = (int64_t)1 << 23;   // partial sums of one launch at most (64 MB)

// the chunk kernel for M objectives: register arrays sized for the next of 4, 8, 12, 24 (a 16 spills with gradients)
typedef void (*EhviChunkFn)(const double*, int64_t, const double*, int, int, const double*, const double*, double*);
static EhviChunkFn ehvi_chunk_kernel(int M, bool grad) {
  if (M <= 4) return grad ? ehvi::k_ehvi_chunk<4, true> : ehvi::k_ehvi_chunk<4, false>;
  if (M <= 8) return grad ? ehvi::k_ehvi_chunk<8, true> : ehvi::k_ehvi_chunk<8, false>;
  if (M <= 12) return grad ? ehvi::k_ehvi_chunk<12, true> : ehvi::k_ehvi_chunk<12, false>;
  return grad ? ehvi::k_ehvi_chunk<24, true> : ehvi::k_ehvi_chunk<24, false>;
}

// replaces LogEHVI.__init__'s state (optuna/_gp/acqf.py:245-280): the non-dominated boxes and the fixed QMC samples
// The body of tpe_ehvi_set, called under the context lock (also by tpe_acqf_set)
static int ehvi_upload(tpe_ctx* ctx, const double* lower, const double* intervals, int64_t B, const double* samples,
                       int32_t S, int32_t M) {
  EhviState& e = ctx->ehvi;
  e.ready = false;
  if (M < 2 || M > ehvi::MAX_M) return fail(ctx, TPE_E_INVALID, "EHVI needs 2 <= M <= %d objectives, got %d", ehvi::MAX_M, M);
  if (S < 1 || S > ehvi::MAX_S) return fail(ctx, TPE_E_INVALID, "EHVI needs 1 <= S <= %d samples, got %d", ehvi::MAX_S, S);
  if (B < 1 || B > ((int64_t)1 << 31)) return fail(ctx, TPE_E_INVALID, "EHVI needs 1 <= B <= 2^31 boxes, got %lld", (long long)B);
  if (!lower || !intervals || !samples) return fail(ctx, TPE_E_INVALID, "bad EHVI arguments");
  std::vector<double> lbI((size_t)B * M * 2);
  for (int64_t i = 0; i < B * M; ++i) {
    if (std::isnan(lower[i])) return fail(ctx, TPE_E_INVALID, "EHVI box lower bounds hold a NaN");
    if (std::isnan(intervals[i])) return fail(ctx, TPE_E_INVALID, "EHVI box intervals hold a NaN");
    lbI[2 * i] = lower[i];
    lbI[2 * i + 1] = intervals[i];
  }
  for (int64_t i = 0; i < (int64_t)S * M; ++i)
    if (std::isnan(samples[i])) return fail(ctx, TPE_E_INVALID, "EHVI samples hold a NaN");
  if (set_device(ctx)) return TPE_E_CUDA;
  cudaStream_t st = ctx->stream;
  CU(e.lbI.ensure(lbI.size() * 8));
  CU(e.Z.ensure((size_t)S * M * 8));
  CU(cudaMemcpyAsync(e.lbI.p, lbI.data(), lbI.size() * 8, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(e.Z.p, samples, (size_t)S * M * 8, cudaMemcpyHostToDevice, st));
  for (bool grad : {false, true}) {
    const size_t smem = ehvi::smem_bytes(M, grad);
    if (smem > 48 * 1024)
      CU(cudaFuncSetAttribute(ehvi_chunk_kernel(M, grad), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  }
  CU(cudaStreamSynchronize(st));   // the host copy of the bounds goes out of scope
  e.B = B;
  e.S = S;
  e.M = M;
  e.ready = true;
  return TPE_OK;
}

int tpe_ehvi_set(tpe_ctx* ctx, const double* lower, const double* intervals, int64_t B, const double* samples,
                 int32_t S, int32_t M) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  return ehvi_upload(ctx, lower, intervals, B, samples, S, M);
}

// The bytes ehvi_launch allocates for Q rows that the context does not hold yet
static size_t ehvi_new_bytes(const EhviState& e, int64_t Q, bool grad, bool inputs) {
  const int M = e.M, K = grad ? 1 + 2 * M : 1;
  const int64_t nchunks = (e.B + ehvi::CHUNK - 1) / ehvi::CHUNK;
  const int64_t slab = std::max<int64_t>(1, std::min<int64_t>({Q, kEhviPartDoubles / (nchunks * K), 65535}));
  auto more = [](const DevBuf& b, size_t bytes) { return bytes > b.cap ? bytes : (size_t)0; };
  size_t need = more(e.value, (size_t)Q * 8) + more(e.part, (size_t)slab * nchunks * K * 8);
  if (inputs) need += more(e.mean, (size_t)Q * M * 8) + more(e.sd, (size_t)Q * M * 8);
  if (grad) need += more(e.dmean, (size_t)Q * M * 8) + more(e.dsd, (size_t)Q * M * 8);
  return need;
}

// log-EHVI at Q rows of device means and standard deviations [Q][M] into e.value and, with grad, e.dmean / e.dsd, on
// the context stream
static int ehvi_launch(tpe_ctx* ctx, const double* mean_d, const double* sd_d, int64_t Q, bool grad) {
  EhviState& e = ctx->ehvi;
  const int M = e.M, K = grad ? 1 + 2 * M : 1;
  const int64_t nchunks = (e.B + ehvi::CHUNK - 1) / ehvi::CHUNK;
  // rows per launch: the partial sums stay under kEhviPartDoubles and the grid's y extent under 65 535
  const int64_t slab = std::max<int64_t>(1, std::min<int64_t>({Q, kEhviPartDoubles / (nchunks * K), 65535}));
  cudaStream_t st = ctx->stream;
  CU(e.value.ensure((size_t)Q * 8));
  CU(e.part.ensure((size_t)slab * nchunks * K * 8));
  if (grad) {
    CU(e.dmean.ensure((size_t)Q * M * 8));
    CU(e.dsd.ensure((size_t)Q * M * 8));
  }
  const size_t smem = ehvi::smem_bytes(M, grad);
  const double log_s = std::log((double)e.S);
  for (int64_t r0 = 0; r0 < Q; r0 += slab) {
    const int64_t rows = std::min(slab, Q - r0);
    const dim3 grid((unsigned)nchunks, (unsigned)rows);
    const double* m0 = mean_d + r0 * M;
    const double* s0 = sd_d + r0 * M;
    const unsigned fb = (unsigned)((rows + 127) / 128);
    ehvi_chunk_kernel(M, grad)<<<grid, ehvi::THREADS, smem, st>>>(e.lbI.as<double>(), e.B, e.Z.as<double>(), e.S, M,
                                                                   m0, s0, e.part.as<double>());
    if (grad) {
      ehvi::k_ehvi_finish<true><<<fb, 128, 0, st>>>(e.part.as<double>(), rows, (int)nchunks, M, log_s,
                                                    e.value.as<double>() + r0, e.dmean.as<double>() + r0 * M,
                                                    e.dsd.as<double>() + r0 * M);
    } else {
      ehvi::k_ehvi_finish<false><<<fb, 128, 0, st>>>(e.part.as<double>(), rows, (int)nchunks, M, log_s,
                                                     e.value.as<double>() + r0, nullptr, nullptr);
    }
  }
  return TPE_OK;
}

// replaces LogEHVI.eval_acqf after the posteriors (acqf.py:282-300, with logehvi :45-62) and its autograd backward in
// the posterior mean and standard deviation
int tpe_ehvi(tpe_ctx* ctx, const double* mean, const double* sd, int64_t Q, double* value, double* dmean,
             double* dsd) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  EhviState& e = ctx->ehvi;
  if (!e.ready) return fail(ctx, TPE_E_STATE, "no EHVI boxes and samples (tpe_ehvi_set)");
  if (!mean || !sd || !value || Q < 1 || (dmean == nullptr) != (dsd == nullptr))
    return fail(ctx, TPE_E_INVALID, "bad EHVI arguments");
  if (set_device(ctx)) return TPE_E_CUDA;
  const bool grad = dmean != nullptr;
  const int M = e.M;
  cudaStream_t st = ctx->stream;
  CU(e.mean.ensure((size_t)Q * M * 8));
  CU(e.sd.ensure((size_t)Q * M * 8));
  CU(cudaMemcpyAsync(e.mean.p, mean, (size_t)Q * M * 8, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(e.sd.p, sd, (size_t)Q * M * 8, cudaMemcpyHostToDevice, st));
  const int rc = ehvi_launch(ctx, e.mean.as<double>(), e.sd.as<double>(), Q, grad);
  if (rc != TPE_OK) return rc;
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(value, e.value.p, (size_t)Q * 8, cudaMemcpyDeviceToHost, st));
  if (grad) {
    CU(cudaMemcpyAsync(dmean, e.dmean.p, (size_t)Q * M * 8, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(dsd, e.dsd.p, (size_t)Q * M * 8, cudaMemcpyDeviceToHost, st));
  }
  CU(cudaStreamSynchronize(st));
  return TPE_OK;
}

// ---- GPSampler's acquisition function over the device posteriors (tpe_acqf.cuh) --------------------------------------
// The posterior of the conditioned GP g at the m rows Xq (device) on stream st, into mean / var [m] and, with dmean,
// dmean / dvar [m][P]: gp_query_chunks' kernels in its chunks, on g's factor and scratch (A, W, part), with the
// outputs in the caller's buffers.  A row's values are the same bits as tpe_gp_query's.
static void acqf_posterior(cudaStream_t st, GpState& g, const double* Xq, int64_t m, double* mean, double* var,
                           double* dmean, double* dvar) {
  const int P = g.P;
  const bool grad = dmean != nullptr;
  const int64_t n = g.n, ntiles = (n + gp::NB - 1) / gp::NB, qmax = grad ? gp::NB : kGpQmax;
  double* Wm = g.A + gp::NB * n;
  for (int64_t q0 = 0; q0 < m; q0 += qmax) {
    const int64_t Q = std::min(qmax, m - q0);
    gp::k_gp_cross<<<dim3((unsigned)((n + 127) / 128), (unsigned)Q), 128, 0, st>>>(Xq + q0 * P, g.X, g.cat, g.prm, P,
                                                                                  (int)n, (int)Q, g.A);
    gp_gemm(st, g.A, n, g.B, n, g.part, 0, Q, n, n, 1.0, gp::GF_KHI_COL | gp::GF_SQSUM);
    gp::k_gp_post_finish<<<(unsigned)((Q + 7) / 8), 256, 0, st>>>(g.A, g.alpha, g.part, (int)ntiles, g.prm, P, (int)n,
                                                                  (int)Q, 0.0, true, mean + q0, var + q0);
    if (grad) {
      gp_gemm(st, g.A, n, g.B, n, g.W, n, Q, n, n, 1.0, gp::GF_KHI_COL);
      gp_gemm(st, g.W, n, g.B, n, Wm, n, Q, n, n, 1.0, gp::GF_TB | gp::GF_KLO_COL);
      const dim3 grid((unsigned)Q, (unsigned)((P + gp::GRAD_DC - 1) / gp::GRAD_DC));
      gp::k_gp_post_grad<gp::GRAD_DC><<<grid, gp::GRAD_THREADS, 0, st>>>(
          Xq + q0 * P, g.X, g.cat, g.prm, g.alpha, Wm, g.part, (int)ntiles, P, (int)n, dmean + q0 * P, dvar + q0 * P);
    }
  }
}

// replaces the state of GPSampler's acquisition functions (optuna/_gp/acqf.py: LogEI :116-149, ConstrainedLogEI
// :217-235, LogEHVI :245-280, ConstrainedLogEHVI :303-331)
int tpe_acqf_set(tpe_ctx* ctx, int32_t kind, tpe_ctx* const* gps, int32_t n_gp, int32_t n_obj,
                 const double* thresholds, double stabilizing_noise, const double* lower, const double* intervals,
                 int64_t B, const double* samples, int32_t S) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  AcqfState& a = ctx->acqf;
  a.release();
  if (kind < TPE_ACQF_LOGEI || kind > TPE_ACQF_LOGPI) return fail(ctx, TPE_E_INVALID, "unknown acquisition kind %d", kind);
  const int want_obj = kind == TPE_ACQF_LOGEI ? 1 : kind == TPE_ACQF_LOGPI ? 0 : n_obj;
  if (kind == TPE_ACQF_LOGEHVI && (n_obj < 2 || n_obj > ehvi::MAX_M))
    return fail(ctx, TPE_E_INVALID, "log-EHVI needs 2 <= n_obj <= %d objectives, got %d", ehvi::MAX_M, n_obj);
  if (n_obj != want_obj) return fail(ctx, TPE_E_INVALID, "acquisition kind %d takes %d objective GPs, got %d", kind,
                                     want_obj, n_obj);
  if (!gps || !thresholds || n_gp < std::max(n_obj, 1) || n_gp > 1 << 16)
    return fail(ctx, TPE_E_INVALID, "bad acquisition arguments (%d GPs, %d objectives)", n_gp, n_obj);
  if (!std::isfinite(stabilizing_noise) || stabilizing_noise < 0.0)
    return fail(ctx, TPE_E_INVALID, "bad stabilizing noise");
  for (int i = 0; i < n_gp; ++i) {
    if (std::isnan(thresholds[i])) return fail(ctx, TPE_E_INVALID, "acquisition threshold %d is NaN", i);
    if (i > 0 && !std::isfinite(thresholds[i]))
      return fail(ctx, TPE_E_INVALID, "acquisition threshold %d is not finite", i);
  }
  if (kind == TPE_ACQF_LOGEI && std::isinf(thresholds[0]) && thresholds[0] > 0)
    return fail(ctx, TPE_E_INVALID, "the LogEI threshold is +inf");
  std::vector<uint64_t> gen(n_gp);
  int32_t P = 0;
  for (int i = 0; i < n_gp; ++i) {
    tpe_ctx* g = gps[i];
    if (!g || g == ctx) return fail(ctx, TPE_E_INVALID, "GP context %d is NULL or the acquisition context itself", i);
    for (int j = 0; j < i; ++j)
      if (gps[j] == g) return fail(ctx, TPE_E_INVALID, "GP contexts %d and %d are the same context", j, i);
    if (g->device != ctx->device)
      return fail(ctx, TPE_E_INVALID, "GP context %d is on device %d, the acquisition context on device %d", i,
                  g->device, ctx->device);
    std::lock_guard<std::mutex> gl(g->mu);
    if (!g->gp.ready || !g->gp.conditioned)
      return fail(ctx, TPE_E_STATE, "GP context %d is not conditioned (tpe_gp_condition)", i);
    if (i > 0 && g->gp.P != P)
      return fail(ctx, TPE_E_INVALID, "GP context %d has width %d, GP context 0 has width %d", i, g->gp.P, P);
    P = g->gp.P;
    gen[i] = g->gp_generation;
  }
  if (set_device(ctx)) return TPE_E_CUDA;
  if (kind == TPE_ACQF_LOGEHVI) {
    const int rc = ehvi_upload(ctx, lower, intervals, B, samples, S, n_obj);
    if (rc != TPE_OK) return rc;
  }
  a.gps.assign(gps, gps + n_gp);
  a.gen = gen;
  a.ev.assign(n_gp, nullptr);
  for (auto& e : a.ev) CU(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  CU(a.thr.ensure((size_t)n_gp * 8));
  CU(cudaMemcpyAsync(a.thr.p, thresholds, (size_t)n_gp * 8, cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  a.kind = kind;
  a.n_obj = n_obj;
  a.P = P;
  a.noise = stabilizing_noise;
  a.ready = true;
  return TPE_OK;
}

// The checks and the body of tpe_acqf_eval, called with the acquisition context and every GP context locked
static int acqf_eval_locked(tpe_ctx* ctx, const double* X, int64_t Q, double* value, double* grad_h) {
  AcqfState& a = ctx->acqf;
  const int K = (int)a.gps.size(), P = a.P, M = a.n_obj;
  for (int i = 0; i < K; ++i) {
    const tpe_ctx* g = a.gps[i];
    if (!g->gp.ready || !g->gp.conditioned || g->gp_generation != a.gen[i] || g->gp.P != P)
      return fail(ctx, TPE_E_STATE, "GP context %d was re-conditioned or changed since tpe_acqf_set", i);
  }
  // non-finite query points are evaluated, not refused: NaN propagates through the posterior and the acquisition as
  // in torch, so that an L-BFGS-B run that met a NaN gradient ends as the reference's does
  const bool grad = grad_h != nullptr;
  const bool ehvi_on = a.kind == TPE_ACQF_LOGEHVI;
  auto more = [](const DevBuf& b, size_t bytes) { return bytes > b.cap ? bytes : (size_t)0; };
  size_t need = more(a.X, (size_t)Q * P * 8) + more(a.mean, (size_t)K * Q * 8) + more(a.var, (size_t)K * Q * 8) +
                more(a.value, (size_t)Q * 8);
  if (grad)
    need += more(a.dmean, (size_t)K * Q * P * 8) + more(a.dvar, (size_t)K * Q * P * 8) +
            more(a.coef, (size_t)K * Q * 2 * 8) + more(a.grad, (size_t)Q * P * 8);
  if (ehvi_on) need += ehvi_new_bytes(ctx->ehvi, Q, grad, true);
  if (set_device(ctx)) return TPE_E_CUDA;
  if (need > 0) {
    size_t free_b = 0, total_b = 0;
    CU(cudaMemGetInfo(&free_b, &total_b));
    if (need > free_b)
      return fail(ctx, TPE_E_INVALID,
                  "the acquisition function at Q = %lld rows needs %zu more bytes of device memory, device %d has %zu "
                  "free", (long long)Q, need, ctx->device, free_b);
  }
  cudaStream_t st = ctx->stream;
  CU(a.X.ensure((size_t)Q * P * 8));
  CU(a.mean.ensure((size_t)K * Q * 8));
  CU(a.var.ensure((size_t)K * Q * 8));
  CU(a.value.ensure((size_t)Q * 8));
  if (grad) {
    CU(a.dmean.ensure((size_t)K * Q * P * 8));
    CU(a.dvar.ensure((size_t)K * Q * P * 8));
    CU(a.coef.ensure((size_t)K * Q * 2 * 8));
    CU(a.grad.ensure((size_t)Q * P * 8));
  }
  CU(cudaMemcpyAsync(a.X.p, X, (size_t)Q * P * 8, cudaMemcpyHostToDevice, st));
  double *mean = a.mean.as<double>(), *var = a.var.as<double>();
  for (int i = 0; i < K; ++i) {
    // the GP's factor and scratch are written on its own stream
    CU(cudaEventRecord(a.ev[i], a.gps[i]->stream));
    CU(cudaStreamWaitEvent(st, a.ev[i], 0));
    acqf_posterior(st, a.gps[i]->gp, a.X.as<double>(), Q, mean + (int64_t)i * Q, var + (int64_t)i * Q,
                   grad ? a.dmean.as<double>() + (int64_t)i * Q * P : nullptr,
                   grad ? a.dvar.as<double>() + (int64_t)i * Q * P : nullptr);
  }
  EhviState& e = ctx->ehvi;
  if (ehvi_on) {
    CU(e.mean.ensure((size_t)Q * M * 8));
    CU(e.sd.ensure((size_t)Q * M * 8));
    acqf::k_acqf_ehvi_in<<<(unsigned)((Q * M + 255) / 256), 256, 0, st>>>(mean, var, Q, M, a.noise,
                                                                          e.mean.as<double>(), e.sd.as<double>());
    const int rc = ehvi_launch(ctx, e.mean.as<double>(), e.sd.as<double>(), Q, grad);
    if (rc != TPE_OK) return rc;
  }
  acqf::k_acqf_combine<<<(unsigned)((Q + 127) / 128), 128, 0, st>>>(
      a.kind, K, M, a.thr.as<double>(), a.noise, mean, var, Q, ehvi_on ? e.value.as<double>() : nullptr,
      ehvi_on && grad ? e.dmean.as<double>() : nullptr, ehvi_on && grad ? e.dsd.as<double>() : nullptr,
      ehvi_on ? e.sd.as<double>() : nullptr, a.value.as<double>(), grad ? a.coef.as<double>() : nullptr);
  if (grad)
    acqf::k_acqf_grad<<<(unsigned)((Q * P + 255) / 256), 256, 0, st>>>(K, a.coef.as<double>(), a.dmean.as<double>(),
                                                                       a.dvar.as<double>(), Q, P, a.grad.as<double>());
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(value, a.value.p, (size_t)Q * 8, cudaMemcpyDeviceToHost, st));
  if (grad) CU(cudaMemcpyAsync(grad_h, a.grad.p, (size_t)Q * P * 8, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  return TPE_OK;
}

// replaces eval_acqf of GPSampler's acquisition functions (acqf.py:151-159, 175-182, 237-242, 282-300, 333-337) and
// its autograd backward in x
int tpe_acqf_eval(tpe_ctx* ctx, const double* X, int64_t Q, double* value, double* grad) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  AcqfState& a = ctx->acqf;
  if (!a.ready) return fail(ctx, TPE_E_STATE, "no acquisition function (tpe_acqf_set)");
  if (!X || !value || Q < 1) return fail(ctx, TPE_E_INVALID, "bad acquisition arguments (Q %lld)", (long long)Q);
  // the GP contexts in address order, so that two acquisition contexts sharing GPs cannot deadlock
  std::vector<tpe_ctx*> order(a.gps);
  std::sort(order.begin(), order.end());
  std::vector<std::unique_lock<std::mutex>> held;
  held.reserve(order.size());
  for (tpe_ctx* g : order) held.emplace_back(g->mu);
  return acqf_eval_locked(ctx, X, Q, value, grad);
}

// replaces get_non_dominated_box_bounds (optuna/_hypervolume/box_decomposition.py:138-157), as LogEHVI.__init__ calls
// it (optuna/_gp/acqf.py:255-263)
int tpe_box_decomposition(tpe_ctx* ctx, const double* loss_vals, int64_t n, int32_t M, const double* ref_point,
                          int64_t* n_boxes) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  BoxDecState& d = ctx->boxdec;
  d.ready = false;
  if (M < 2 || M > boxdec::MAX_M)
    return fail(ctx, TPE_E_INVALID, "box decomposition needs 2 <= M <= %d objectives, got %d", boxdec::MAX_M, M);
  if (n < 1 || n >= (1ll << 31) - 4096)
    return fail(ctx, TPE_E_INVALID, "box decomposition needs 1 <= n < 2^31 - 4096 rows, got %lld", (long long)n);
  if (!loss_vals || !ref_point || !n_boxes) return fail(ctx, TPE_E_INVALID, "bad box decomposition arguments");
  for (int64_t q = 0; q < n * M; ++q)
    if (!std::isfinite(loss_vals[q]))
      return fail(ctx, TPE_E_INVALID, "box decomposition: loss values must be finite (row %lld)", (long long)(q / M));
  for (int j = 0; j < M; ++j)
    if (std::isnan(ref_point[j])) return fail(ctx, TPE_E_INVALID, "box decomposition: the reference point holds a NaN");
  if (set_device(ctx)) return TPE_E_CUDA;
  BD_ALLOC(d.rows, (size_t)n * M * 8, n);
  CU(cudaMemcpyAsync(d.rows.p, loss_vals, (size_t)n * M * 8, cudaMemcpyHostToDevice, ctx->stream));
  const int rc = bd_run(ctx, (int)n, M, ref_point);
  if (rc != TPE_OK) return rc;
  *n_boxes = (int64_t)(d.lower.size() / M);
  d.ready = true;
  return TPE_OK;
}

int tpe_get_box_decomposition(tpe_ctx* ctx, double* lower, double* upper, int64_t* stats) {
  if (!ctx) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  const BoxDecState& d = ctx->boxdec;
  if (!d.ready) return fail(ctx, TPE_E_STATE, "no box decomposition (tpe_box_decomposition)");
  if (lower) std::copy(d.lower.begin(), d.lower.end(), lower);
  if (upper) std::copy(d.upper.begin(), d.upper.end(), upper);
  if (stats) std::copy(d.stats, d.stats + 6, stats);
  return TPE_OK;
}

const char* tpe_last_logpdf_kernel(tpe_ctx* ctx) { return ctx ? ctx->last_kernel : "none"; }

#ifdef TPE_LAB
// lab build only (not in the header): the near-term counters of the DBG = 5 tilings summed since the last call (see
// g_mma_lab_count), then cleared
int tpe_lab_mma_counters(tpe_ctx* ctx, unsigned long long* out5) {
  if (!ctx || !out5) return TPE_E_INVALID;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (set_device(ctx)) return TPE_E_CUDA;
  CU(cudaStreamSynchronize(ctx->stream));
  CU(cudaMemcpyFromSymbol(out5, g_mma_lab_count, 5 * sizeof(unsigned long long)));
  const unsigned long long zero[5] = {0, 0, 0, 0, 0};
  CU(cudaMemcpyToSymbol(g_mma_lab_count, zero, sizeof(zero)));
  return TPE_OK;
}
#endif  // TPE_LAB

}  // extern "C"
