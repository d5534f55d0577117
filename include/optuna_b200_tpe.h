/*
 * optuna_b200_tpe.h -- C ABI of the GPU-native (H100, sm_90a) TPE suggestion engine (libtpe_b200.so).
 *
 * This is the drop-in boundary for the reference's TPE hot path.  Each entry point names the
 * reference interface it replaces (paths relative to the optuna checkout @ 4df4b72).  The
 * Python host (optuna_b200/sampler.py) binds these with ctypes; INTEGRATION.md shows the stub a
 * maintainer of the reference would add.
 *
 * Conventions
 *   - every function returns 0 on success or a negative TPE_E_* code; the message is
 *     retrievable with tpe_last_error(ctx) (per context, valid until the next call on it);
 *   - the caller owns all host buffers; the library copies and retains no host pointer;
 *   - the library owns all device memory; one context is bound to one CUDA device;
 *   - no callbacks into the host: Python callables of the reference (gamma, weights,
 *     constraints_func, categorical_distance_func) are evaluated by the host and passed as data;
 *   - all entry points take a per-context mutex (ctypes releases the GIL, and the reference
 *     shares one sampler across n_jobs threads: optuna/study/_optimize.py:87-121);
 *   - doubles are IEEE fp64, indices int64, "internal representation" of a parameter is the
 *     reference's (optuna/distributions.py:182,365,509): float value / int as float / choice index.
 */
#ifndef OPTUNA_B200_TPE_H_
#define OPTUNA_B200_TPE_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* 2: + tpe_history_update, tpe_stage_uniforms, tpe_stage_uniforms_mt19937, tpe_rng_state,
 *      tpe_get_uniforms, tpe_host_alloc / tpe_host_free; tpe_sample_and_select accepts uniforms == NULL
 *      after tpe_stage_uniforms_mt19937 */
/* 3: + TPE_CAT_EXCLUDED; tpe_history_update may extend the history; tpe_sample_and_select accepts out_x == NULL
 *      (results stay on the device: tpe_result_device_ptrs); tpe_rng_state_device; tpe_suggest_univariate_batch */
/* 4: + tpe_sample_and_select_async / tpe_collect */
/* 5: + tpe_suggest_univariate_batch_async / tpe_collect_univariate */
/* 6: + tpe_set_kernel_shard / tpe_sample_and_partial / tpe_finish_from_partials */
/* 7: + tpe_hypervolume_history */
/* 8: + tpe_pareto_front */
/* 9: + tpe_fanova_variances */
/* 10: + tpe_gp_set_data, tpe_gp_loss, tpe_gp_posterior, TPE_E_NOTPD */
/* 11: + tpe_gp_loss_fixed_noise, tpe_gp_posterior_moments */
/* 12: + tpe_gp_condition, tpe_gp_query */
/* 13: + tpe_ehvi_set, tpe_ehvi */
/* 14: + tpe_box_decomposition, tpe_get_box_decomposition */
/* 15: + tpe_gp_batch_set, tpe_gp_batch_loss, tpe_gp_batch_bounds */
/* 16: + tpe_gp_batch_loss_fixed_noise, tpe_gp_batch_moments */
/* 17: + tpe_acqf_set, tpe_acqf_eval */
#define TPE_ABI_VERSION 17

enum {
  TPE_OK = 0,
  TPE_E_INVALID = -1,  /* bad argument (mirrors the reference's ValueError) */
  TPE_E_CUDA = -2,     /* CUDA runtime failure */
  TPE_E_STATE = -3,    /* call order violated (e.g. suggest before history/space are set) */
  TPE_E_NOMEM = -4,
  TPE_E_NOTPD = -5     /* a Gaussian-process covariance is not positive definite (torch's Cholesky LinAlgError) */
};

/* optuna/distributions.py: FloatDistribution :109, IntDistribution :310, CategoricalDistribution :470 */
enum { TPE_KIND_FLOAT = 0, TPE_KIND_INT = 1, TPE_KIND_CAT = 2 };

/* Trial groups of TPESampler._split_trials (optuna/samplers/_tpe/sampler.py:686-722). */
enum {
  TPE_CAT_COMPLETE = 0,
  TPE_CAT_PRUNED = 1,
  TPE_CAT_INFEASIBLE = 2,
  TPE_CAT_RUNNING = 3,
  /* A row that takes part in neither set: the placeholder of a trial the sampler must not see yet (WAITING,
   * RUNNING without constant_liar, the trial being sampled itself -- sampler.py:526-535 filters it out) or ever
   * (FAIL).  Keeps row index == position in the study's trial list, so that a trial finishing late is one
   * tpe_history_update in place instead of a re-upload. */
  TPE_CAT_EXCLUDED = 4
};

typedef struct tpe_ctx tpe_ctx;

typedef struct {
  int32_t kind;      /* TPE_KIND_* */
  int32_t log;       /* 1 = log-scaled domain */
  int32_t has_step;  /* 1 = discretised (always 1 for TPE_KIND_INT) */
  int32_t n_choices; /* categorical only */
  double low, high, step;
} tpe_param_desc;

/* TPESampler constructor arguments that reach the numeric path (sampler.py:305-360) plus the
 * per-call values the host evaluates (gamma(n) -> n_below). */
typedef struct {
  double prior_weight;   /* _ParzenEstimatorParameters.prior_weight */
  int32_t magic_clip;    /* consider_magic_clip */
  int32_t endpoints;     /* consider_endpoints */
  int32_t multivariate;  /* multivariate */
  int32_t n_candidates;  /* n_ei_candidates */
  int64_t n_below;       /* gamma(n_finished), evaluated by the host (sampler.py:538-542) */
} tpe_cfg;

/* Shapes of the two estimators after tpe_prepare. */
typedef struct {
  int64_t n_below_all;  /* |below| before dropping trials that lack a selected param */
  int64_t n_below_obs;  /* observations in l(x) (kernels = +1 prior) */
  int64_t n_above_obs;  /* observations in g(x) */
} tpe_split_info;

int tpe_abi_version(void);
int tpe_ctx_create(int device, tpe_ctx** out);
void tpe_ctx_destroy(tpe_ctx* ctx);
const char* tpe_last_error(tpe_ctx* ctx);

/* Search space = every parameter the study has seen, in the host's column order
 * (replaces the dict[str, BaseDistribution] handed to sample_relative, samplers/_base.py:96).
 * cat_dist: optional concatenation of row-major [n_choices, n_choices] distance tables for the
 * categorical params that have a categorical_distance_func (parzen_estimator.py:152-160),
 * cat_dist_offset[p] = offset into cat_dist or -1. */
int tpe_space_set(tpe_ctx* ctx, const tpe_param_desc* params, int32_t n_params,
                  const double* cat_dist, const int64_t* cat_dist_offset);

/* Trial history (replaces the list[FrozenTrial] walk of _get_internal_repr / _split_trials,
 * sampler.py:511-521, :686-722).
 *   X        [n, n_params] row-major internal representation, NaN = parameter absent
 *   category [n] TPE_CAT_*
 *   key      [n, 2] the reference's sort key inside the category (sampler.py:735-742, :782-821):
 *            COMPLETE (signed value, 0); PRUNED (-last_step, signed value); INFEASIBLE (violation, 0)
 * tpe_history_set replaces everything; tpe_history_append adds rows (after_trial hook). */
int tpe_history_set(tpe_ctx* ctx, const double* X, const int8_t* category, const double* key,
                    int64_t n);
int tpe_history_append(tpe_ctx* ctx, const double* X, const int8_t* category, const double* key,
                       int64_t n);
/* Overwrite rows [at_row, at_row + n) in place: a trial that has finished keeps its position (trial-number order)
 * and only changes its category / key / parameters (a TPE_CAT_EXCLUDED placeholder becoming COMPLETE; with
 * constant_liar=True, sampler.py:526-535, a RUNNING row of the above set).  at_row <= current size; a write that
 * runs past the end extends the history, so "the previous trial finished + the next one started" is one call. */
int tpe_history_update(tpe_ctx* ctx, const double* X, const int8_t* category, const double* key, int64_t n,
                       int64_t at_row);
/* Same, with DEVICE pointers on ctx's device (used after an NCCL broadcast of the history). */
int tpe_history_set_device(tpe_ctx* ctx, const double* dX, const int8_t* dcategory,
                           const double* dkey, int64_t n, const uint8_t* col_has_missing);
/* Multi-objective studies: objective values of rows [at_row, at_row + n), sign-normalised so that
 * every objective is minimised (sampler.py:755).  values [n, n_objectives] row-major.  With
 * n_objectives >= 2 the COMPLETE group is split by non-domination rank + greedy hypervolume subset
 * selection (sampler.py:745-779) and l(x) is weighted by hypervolume contributions (:824-863)
 * unless tpe_build is given explicit below-weights.  n_objectives <= 16; any number of below trials (the exact
 * hypervolumes run over the Pareto front of the below set / the selected subset only; their scratch is O(n^2 M) per
 * warp, TPE_E_NOMEM beyond 16 GB). */
int tpe_history_set_values(tpe_ctx* ctx, const double* values, int64_t n, int32_t n_objectives, int64_t at_row);
int64_t tpe_history_size(tpe_ctx* ctx);
/* Device pointers of the resident history (for the NCCL broadcast done by the host plumbing). */
int tpe_history_device_ptrs(tpe_ctx* ctx, double** dX, int8_t** dcategory, double** dkey);

/* Stage 1: split + observation gathering for the selected columns.
 * Replaces _split_trials + _get_internal_repr.  cols[n_cols] index into the space. */
int tpe_prepare(tpe_ctx* ctx, const tpe_cfg* cfg, const int32_t* cols, int32_t n_cols,
                tpe_split_info* info);

/* Stage 2: build l(x) and g(x) (replaces _ParzenEstimator.__init__, parzen_estimator.py:39-78).
 * w_below / w_above: raw per-observation weights (weights_func(n)[:n], or the MOTPE weights,
 * sampler.py:574-576) or NULL for the reference's default_weights (sampler.py:61-69). */
int tpe_build(tpe_ctx* ctx, const double* w_below, const double* w_above);

/* Stage 3+4: draw candidates from l(x) with host-supplied uniforms and pick the best by
 * log l(x) - log g(x) (replaces mpe_below.sample, _compute_acquisition_func, _compare;
 * sampler.py:553-555).  n_asks independent suggestions share the estimators.
 *   uniforms [n_asks, C * (1 + n_cat + n_num)] per ask in the reference's RNG order
 *            (probability_distributions.py:87,100,138-144): C for rng.choice, then C per
 *            categorical param in column order, then an [n_num, C] block.
 *   out_x    [n_asks, n_cols] chosen candidate (internal representation); NULL = leave the results on the device
 *            (tpe_result_device_ptrs): a multi-GPU caller gathers them with NCCL without a host bounce
 *   out_acq  [n_asks] its acquisition value (may be NULL)
 *   out_best [n_asks] its candidate index (may be NULL) */
int tpe_sample_and_select(tpe_ctx* ctx, const double* uniforms, int64_t n_asks, double* out_x,
                          double* out_acq, int64_t* out_best);

/* The same in two halves: tpe_sample_and_select_async queues the work (and the copy of the results into page-locked
 * memory of the context) and returns; tpe_collect waits for it and hands the results out.  A caller that knows the
 * next suggestion's inputs early -- the sampler at `tell` time: the history with the finished trial, the generator
 * where the last ask left it (BaseSampler.after_trial, optuna/samplers/_base.py:178-203, runs before the next
 * Study.ask) -- overlaps the device work with its own host work; results are those of tpe_sample_and_select.
 * `uniforms` is read before tpe_sample_and_select_async returns.  Any tpe_prepare abandons uncollected results. */
int tpe_sample_and_select_async(tpe_ctx* ctx, const double* uniforms, int64_t n_asks);
int tpe_collect(tpe_ctx* ctx, double* out_x, double* out_acq, int64_t* out_best);

/* ONE suggestion over several GPUs (SURVEY section 8e, the alternative for a single ask): every rank holds the whole
 * history and builds both estimators (cheap), but evaluates g(x) -- the C x K x P grid -- only over its slice of the
 * above kernels.  tpe_set_kernel_shard(rank, world) selects the slice for the following calls (world = 1: off).
 * tpe_sample_and_partial replaces tpe_sample_and_select: candidates (every rank draws the same ones from the same
 * uniforms), l(x) in full, g(x) over the slice, reduced to one (max, sum) pair per candidate:
 *   *d_partials  device pointer, [n_asks * C] double2 padded to *stride pairs.
 * The caller gathers the partials of all ranks into one device buffer [world][*stride] double2 (ncclAllGather) and
 * calls tpe_finish_from_partials on every rank: log-sum-exp across ranks in rank order, acquisition, argmax -- the
 * same numbers on every rank.  Multivariate suggestions over continuous parameters only (TPE_E_STATE otherwise). */
int tpe_set_kernel_shard(tpe_ctx* ctx, int32_t rank, int32_t world);
int tpe_sample_and_partial(tpe_ctx* ctx, const double* uniforms, int64_t n_asks, double** d_partials, int64_t* stride);
int tpe_finish_from_partials(tpe_ctx* ctx, const double* d_gathered, int32_t world, double* out_x, double* out_acq,
                             int64_t* out_best);

/* Device pointers of the results of the last tpe_sample_and_select: out_x [n_asks, n_cols], out_acq [n_asks],
 * out_best [n_asks] (valid until the next call on the context; the work has completed when that call returned). */
int tpe_result_device_ptrs(tpe_ctx* ctx, double** out_x, double** out_acq, int64_t** out_best);

/* One-call convenience = prepare + build + sample_and_select (TPESampler._sample, sampler.py:523-560). */
int tpe_suggest(tpe_ctx* ctx, const tpe_cfg* cfg, const int32_t* cols, int32_t n_cols,
                const double* w_below, const double* w_above, const double* uniforms,
                int64_t n_asks, double* out_x, double* out_acq, int64_t* out_best);

/* Univariate TPE (multivariate = 0, the reference's default): the n_cols sample_independent calls of ONE trial
 * (sampler.py:458-491, one TPESampler._sample per parameter) evaluated together.  Column cols[j] gets its own pair
 * of 1-D estimators (the split is shared: it does not depend on the parameter), its own C candidates from
 * uniforms[j * 2C, (j + 1) * 2C) -- C for rng.choice, then C for the value, the order a sequence of per-parameter
 * calls consumes the generator -- and its own argmax; the columns run concurrently on the device.
 * uniforms == NULL: the n_cols * 2C uniforms staged by tpe_stage_uniforms_mt19937.
 * TPE_E_STATE ("not batchable") when the columns cannot share a split (a parameter absent from some trials) or the
 * history is multi-objective: the caller then makes the per-parameter calls.
 *   out_x [n_cols] chosen value per column (internal representation); out_acq, out_best [n_cols] may be NULL. */
int tpe_suggest_univariate_batch(tpe_ctx* ctx, const tpe_cfg* cfg, const int32_t* cols, int32_t n_cols,
                                 const double* w_below, const double* w_above, const double* uniforms,
                                 double* out_x, double* out_acq, int64_t* out_best);

/* The same in two halves (as tpe_sample_and_select_async / tpe_collect): queue the whole batch and return; collect
 * waits and hands the results out.  Only for trials whose selected parameters are all continuous (the path that runs
 * stage by stage over all columns); TPE_E_STATE "not batchable asynchronously" otherwise.  `uniforms`, `w_below` and
 * `w_above` are read before the call returns. */
int tpe_suggest_univariate_batch_async(tpe_ctx* ctx, const tpe_cfg* cfg, const int32_t* cols, int32_t n_cols,
                                       const double* w_below, const double* w_above, const double* uniforms);
int tpe_collect_univariate(tpe_ctx* ctx, double* out_x, double* out_acq, int64_t* out_best);

/* Optional: start the upload of the uniforms of the NEXT tpe_sample_and_select early (e.g. right
 * after tpe_prepare, so that the copy overlaps tpe_build).  `count` doubles are copied from
 * `uniforms` on a side stream; tpe_sample_and_select called with the same pointer and the matching
 * count then skips its own copy.  Purely a latency hint: no effect on results.  The reference has no
 * counterpart (its uniforms never leave the host, probability_distributions.py:86-152). */
int tpe_stage_uniforms(tpe_ctx* ctx, const double* uniforms, int64_t count);

/* Device-side uniforms: generate the next `count` outputs of numpy.random.RandomState.random_sample
 * (MT19937, legacy 53-bit doubles) on the GPU, after discarding `skip` of them, straight into the
 * buffer tpe_sample_and_select reads -- the exact stream the reference draws on the host
 * (probability_distributions.py:87,100,138-144), without the host RNG and
 * without the upload.  key[624] / pos are RandomState.get_state()[1:3].  The following
 * tpe_sample_and_select must be called with uniforms == NULL and count == n_asks * per_ask.
 * tpe_rng_state returns the generator state after the (skip + count) draws, for set_state().
 * key == NULL continues from the state the previous staged draw ended in (it is kept on the device), so a
 * caller that owns the generator exclusively can defer get_state()/set_state() until somebody else needs it. */
int tpe_stage_uniforms_mt19937(tpe_ctx* ctx, const uint32_t* key, int32_t pos, int64_t skip, int64_t count);
int tpe_rng_state(tpe_ctx* ctx, uint32_t* key_out, int32_t* pos_out);
/* The same state where it lives: 625 words (key[624], pos) in device memory.  For multi-GPU plumbing -- the rank that
 * drew the LAST stretch of a batch broadcasts its end state into every rank's buffer (NCCL, device to device), so all
 * ranks continue as one generator that drew everything (optuna_b200/dist.py).  The library forgets its host copy. */
int tpe_rng_state_device(tpe_ctx* ctx, uint32_t** state625);
/* Inspection: the first `count` staged uniforms (device-generated or uploaded). */
int tpe_get_uniforms(tpe_ctx* ctx, double* out, int64_t count);

/* Page-locked host memory for buffers handed to tpe_sample_and_select / tpe_suggest (uniforms): a copy
 * from pinned memory is a true asynchronous DMA, a copy from pageable memory is staged by the host
 * thread first.  Optional; any host pointer is accepted everywhere. */
int tpe_host_alloc(tpe_ctx* ctx, size_t bytes, void** out);
int tpe_host_free(tpe_ctx* ctx, void* p);

/* ---- parity / inspection entry points (used by tests and by custom _parzen_estimator_cls-style
 * consumers, sampler.py:358-359) ------------------------------------------------------------- */
/* Shapes of the last tpe_prepare / tpe_suggest. */
int tpe_get_split_info(tpe_ctx* ctx, tpe_split_info* info);
/* Index lists produced by the last tpe_prepare (ascending trial order). */
int tpe_get_split(tpe_ctx* ctx, int64_t* below_rows, int64_t* above_rows);
/* Estimator parameters of the last tpe_build.  which: 0 = below, 1 = above.
 * weights [K]; mu, sigma [K, n_cols] (categorical columns hold the observed choice index / 0);
 * K = n_obs + 1.  Any pointer may be NULL. */
int tpe_get_mixture(tpe_ctx* ctx, int which, double* weights, double* mu, double* sigma);
/* MOTPE: raw hypervolume weights of ALL below trials (length n_below_all) of the last tpe_build. */
int tpe_get_mo_weights(tpe_ctx* ctx, double* weights);

/* ---- analysis ------------------------------------------------------------------------------ */
/* Hypervolume history of a multi-objective study (replaces _get_hypervolume_history_info,
 * optuna/visualization/_hypervolume_history.py:83-138).  values [n, n_objectives]: objective values of the
 * COMPLETE trials in trial order, multiplied by +1 (minimise) or -1 (maximise); ref [n_objectives]: the
 * reference point with the same signs; feasible [n]: 0 = a constraint is violated (NULL: all feasible).
 * out [n]: the hypervolume after each trial.  2 <= n_objectives <= 16; NaN in values or ref is
 * TPE_E_INVALID.  Uses its own device memory and leaves the context's history and suggestion state alone. */
int tpe_hypervolume_history(tpe_ctx* ctx, const double* values, const uint8_t* feasible, int64_t n,
                            int32_t n_objectives, const double* ref, double* out);
/* Pareto front of a set of objective vectors (replaces _is_pareto_front, optuna/study/_multi_objective.py:171-184,
 * behind Study.best_trials and plot_pareto_front).  values [n, n_objectives]: the candidate rows, multiplied by +1
 * (minimise) or -1 (maximise).  on_front [n]: 1 iff no row is <= the row in every objective and < in one; identical
 * rows never dominate each other, so every copy of a front vector is on the front.  IEEE comparisons (-0.0 == 0.0,
 * +-inf are ordinary values).  1 <= n_objectives <= 16; NaN in values is TPE_E_INVALID.  Uses its own device memory
 * and leaves the context's history and suggestion state alone. */
int tpe_pareto_front(tpe_ctx* ctx, const double* values, int64_t n, int32_t n_objectives, uint8_t* on_front);
/* fANOVA variances of a fitted random forest (replaces the per-tree work of optuna/importance/_fanova: the
 * _FanovaTree precomputation, _tree.py:144-236, its variance, :33-45, and get_marginal_variance with its tree walk per
 * grid cell, :47-142, as _Fanova.fit / _compute_variances, _fanova.py:53-108, call them).
 * Trees t = 0..n_trees-1 are the nodes [node_offsets[t], node_offsets[t+1]) of the concatenated arrays left, right
 * (children, indices within the tree), feature (< 0: leaf), threshold (x <= threshold goes left) and value (the
 * node's prediction), as sklearn's tree_.children_left / children_right / feature / threshold / value[:, 0, 0].
 * bounds [n_features, 2]: the search space of the raw features.  Parameter p is the raw features
 * raw_features[param_offsets[p] .. param_offsets[p+1]) (one column, or the one-hot columns of a categorical).
 * Out: tree_variance [n_trees] and marginal_variance [n_params, n_trees] (unclipped).
 * TPE_E_INVALID: a child index not in (parent, tree size), a node with no or two parents, an internal node's feature
 * >= n_features, a NaN threshold or one outside its feature's bounds, a raw feature out of range or in two
 * parameters, and a parameter whose grid (the product of its columns' midpoint counts) exceeds 2^20 cells in some
 * tree -- the reference would walk that tree 2^20 times per parameter; this is the one input it accepts that is
 * refused here.  TPE_E_NOMEM when the device memory runs out.  Uses its own device memory and leaves the context's
 * history and suggestion state alone. */
int tpe_fanova_variances(tpe_ctx* ctx, int32_t n_trees, const int64_t* node_offsets, const int32_t* left,
                         const int32_t* right, const int32_t* feature, const double* threshold, const double* value,
                         int32_t n_features, const double* bounds, int32_t n_params, const int32_t* param_offsets,
                         const int32_t* raw_features, double* tree_variance, double* marginal_variance);
/* Gaussian process of the terminator's improvement evaluators (RegretBoundEvaluator, optuna/terminator/improvement/
 * evaluator.py:142-177, and EMMREvaluator, emmr.py:123-237) and of GPSampler (optuna/samplers/_gp/sampler.py), fp64.
 * Kept apart from the history and the suggestion state.
 * tpe_gp_set_data replaces the GPRegressor's training data (optuna/_gp/gp.py:94-118): X [n, P] normalised
 * parameters, y [n] standardised values, is_categorical [P] (0 / 1); n >= 1, P >= 1, all finite.  Allocates two
 * n x n matrices; TPE_E_INVALID naming the need when the device lacks the memory.
 * tpe_gp_loss replaces loss_func of GPRegressor._fit_kernel_params without its prior term (gp.py:312-327,
 * marginal_log_likelihood :252-285 and its backward): raw [P + 2] = log inverse squared lengthscales, log kernel
 * scale, log(noise_var - minimum_noise).  *loss = -log p(y), grad [P + 2] its gradient in raw.
 * tpe_gp_posterior replaces _cache_matrix / posterior (gp.py:124-149, 215-250) and UCB / LCB (optuna/_gp/acqf.py:
 * 185-214): params [P + 2] = inverse squared lengthscales, kernel scale, noise_var; Xq [m, P]; ucb, lcb [m] =
 * mean +- sqrt(beta var), var clamped at 0.
 * tpe_gp_loss_fixed_noise is tpe_gp_loss with deterministic_objective=True (gp.py:312-327): the noise is fixed at
 * noise_var, raw[P + 1] is ignored and grad[P + 1] = 0.
 * tpe_gp_posterior_moments replaces GPRegressor.posterior (gp.py:215-250) at m points: mean [m], var [m] clamped at
 * 0; with n_joint in [2, 64] (and <= m) also the joint covariance of the first n_joint points, cov [n_joint *
 * n_joint] row-major, diagonal clamped at 0 (joint=True); n_joint = 0 and cov = NULL for none.  One factorisation
 * per call.
 * tpe_gp_condition replaces GPRegressor._cache_matrix (gp.py:124-149) and, after a new tpe_gp_set_data of the train
 * and running rows, append_running_data (gp.py:151-183): it factorises once at params [P + 2] and keeps L^-1 and
 * C^-1 y for tpe_gp_query.  tpe_gp_set_data, the loss calls and the posterior calls overwrite that factor and undo it.
 * tpe_gp_query replaces GPRegressor.posterior (gp.py:215-250, joint=False) and its autograd backward in x, as the
 * acquisition functions of optuna/_gp/acqf.py and optim_mixed.optimize_acqf_mixed call it: at m query rows Xq [m, P],
 * mean [m] and var [m] clamped at 0 against the conditioned factor, with no refactorisation; with dmean and dvar
 * non-NULL also their gradients in x, [m, P] each, 0 in categorical columns and, for dvar, where var was clamped.  The
 * values do not depend on whether gradients are asked for.  TPE_E_STATE when the context is not conditioned.
 * All return TPE_E_NOTPD when a Cholesky pivot is <= 0 or NaN; the loss calls also when a raw parameter they read is
 * NaN or large enough that a kernel parameter is not finite (the reference's Cholesky fails there too). */
int tpe_gp_set_data(tpe_ctx* ctx, const double* X, const double* y, const uint8_t* is_categorical, int64_t n,
                    int32_t P);
int tpe_gp_loss(tpe_ctx* ctx, const double* raw, double minimum_noise, double* loss, double* grad);
int tpe_gp_posterior(tpe_ctx* ctx, const double* params, const double* Xq, int64_t m, double beta, double* ucb,
                     double* lcb);
int tpe_gp_loss_fixed_noise(tpe_ctx* ctx, const double* raw, double noise_var, double* loss, double* grad);
int tpe_gp_posterior_moments(tpe_ctx* ctx, const double* params, const double* Xq, int64_t m, int32_t n_joint,
                             double* mean, double* var, double* cov);
int tpe_gp_condition(tpe_ctx* ctx, const double* params);
int tpe_gp_query(tpe_ctx* ctx, const double* Xq, int64_t m, double* mean, double* var, double* dmean, double* dvar);
/* Many independent Gaussian processes at once, fp64: the per-prefix fits of plot_terminator_improvement
 * (optuna/visualization/_terminator_improvement.py:83-132, one RegretBoundEvaluator.evaluate per trial).  Kept apart
 * from the history, the suggestion state and the single-GP state.
 * tpe_gp_batch_set sets n_gp GPs: GP i has the rows offsets[i] .. offsets[i + 1] - 1 of X [N, P] and y [N]
 * (offsets [n_gp + 1], offsets[0] = 0, N = offsets[n_gp]), all share is_categorical [P].  n_gp >= 1, every
 * n_i >= 1, P >= 1, X and y finite.  TPE_E_INVALID naming the bytes when the device lacks the memory for the data
 * and one loss call over every GP.
 * tpe_gp_batch_loss is tpe_gp_loss for k jobs: job b is GP gp_idx[b] at raw[b] [P + 2] (the raw parameters of
 * tpe_gp_loss); loss[b] = -log p(y), grad[b] [P + 2].  status[b] = 0, or 1 when the kernel parameters are not finite
 * or the covariance is not positive definite (tpe_gp_loss's TPE_E_NOTPD), with loss and grad NaN; the other jobs are
 * unaffected.
 * tpe_gp_batch_bounds: job b is GP gp_idx[b] at params[b] [P + 2] (inverse squared lengthscales, kernel scale,
 * noise_var) with beta[b] >= 0 and the S sample rows samples[b] [S, P]; out[b] [3] = max over the GP's train rows of
 * mean + sqrt(beta var), the same over the sample rows, and max over the train rows of mean - sqrt(beta var), var
 * clamped at 0 and NaN propagating as np.max propagates it (RegretBoundEvaluator.evaluate, optuna/terminator/
 * improvement/evaluator.py:50-84).  status as for the loss.
 * tpe_gp_batch_loss_fixed_noise is tpe_gp_loss_fixed_noise for k jobs: the noise is fixed at noise_var, raw[b][P + 1]
 * is not read and grad[b][P + 1] = 0; status as for tpe_gp_batch_loss.
 * tpe_gp_batch_moments replaces the posterior calls of EMMREvaluator.evaluate (optuna/terminator/improvement/emmr.py:
 * 165-185) for k jobs: job b is GP gp_idx[b] at params[b] [P + 2] (inverse squared lengthscales, kernel scale,
 * noise_var), queried at m (1 to 3) of its own train rows, rows[b] [m] row indices within the GP.  mean[b] [m] and
 * var[b] [m] clamped at 0; with n_joint in [2, m] also cov[b] [n_joint * n_joint] row-major, the joint covariance of
 * the first n_joint rows with its diagonal clamped at 0 (tpe_gp_posterior_moments's); n_joint = 0 and cov = NULL for
 * none.  status as for the loss, with the outputs NaN.  TPE_E_INVALID for a row index outside its GP or a bad n_joint.
 * Several jobs may name the same GP.  A job's outputs are the same bits whatever the other jobs of the call are. */
int tpe_gp_batch_set(tpe_ctx* ctx, int32_t n_gp, const int64_t* offsets, int32_t P, const double* X, const double* y,
                     const uint8_t* is_categorical);
int tpe_gp_batch_loss(tpe_ctx* ctx, int64_t k, const int32_t* gp_idx, const double* raw, double minimum_noise,
                      double* loss, double* grad, int32_t* status);
int tpe_gp_batch_bounds(tpe_ctx* ctx, int64_t k, const int32_t* gp_idx, const double* params, const double* beta,
                        int32_t S, const double* samples, double* out, int32_t* status);
int tpe_gp_batch_loss_fixed_noise(tpe_ctx* ctx, int64_t k, const int32_t* gp_idx, const double* raw, double noise_var,
                                  double* loss, double* grad, int32_t* status);
int tpe_gp_batch_moments(tpe_ctx* ctx, int64_t k, const int32_t* gp_idx, const double* params, int32_t m,
                         const int32_t* rows, int32_t n_joint, double* mean, double* var, double* cov,
                         int32_t* status);
/* Log expected hypervolume improvement of GPSampler's multi-objective acquisition (LogEHVI, optuna/_gp/acqf.py:245-300,
 * with logehvi :45-62), fp64.  Kept apart from the history, the suggestion state and the GP state.
 * tpe_ehvi_set replaces the state LogEHVI.__init__ builds (acqf.py:245-280): lower [B, M] the lower bounds of the
 * non-dominated boxes, intervals [B, M] their widths already clamped at 1e-12, samples [S, M] the fixed QMC samples
 * (standard normal).  2 <= M <= 24 (a product of M factors of at least 1e-12 stays a normal double), 1 <= S <= 1024,
 * B >= 1, no NaN; infinities are allowed and follow IEEE arithmetic as torch does (an interval is often +inf, a sample
 * can be -inf).  TPE_E_INVALID naming the violated condition.
 * tpe_ehvi replaces LogEHVI.eval_acqf after the posteriors (acqf.py:282-300) and its autograd backward: at Q rows of
 * posterior means mean [Q, M] and standard deviations sd [Q, M], value [Q] = log(1/S sum_{s,b} prod_j
 * min(max(mean_j + sd_j z_sj - lower_bj, 1e-12), intervals_bj)), the reference's logsumexp of sum_j log; with dmean and
 * dsd non-NULL (both or neither) also its gradients [Q, M] in mean and sd, through torch's inclusive clamp mask.  A
 * row's value is the same bits whatever Q, the row's position and the gradient request, and repeated calls return the
 * same bits.  TPE_E_STATE before tpe_ehvi_set. */
int tpe_ehvi_set(tpe_ctx* ctx, const double* lower, const double* intervals, int64_t B, const double* samples,
                 int32_t S, int32_t M);
int tpe_ehvi(tpe_ctx* ctx, const double* mean, const double* sd, int64_t Q, double* value, double* dmean, double* dsd);
/* GPSampler's acquisition function (optuna/_gp/acqf.py) over the posteriors of conditioned GP contexts, fp64, with its
 * gradient in the query point.  Kept apart from every other state of the acquisition context except its log-EHVI
 * boxes and samples, which tpe_acqf_set replaces for TPE_ACQF_LOGEHVI.
 * tpe_acqf_set: kind TPE_ACQF_LOGEI (n_obj = 1: LogEI of gps[0], acqf.py:151-159), TPE_ACQF_LOGEHVI (2 <= n_obj <= 24:
 * log-EHVI of gps[0 .. n_obj - 1] over lower / intervals [B, M] and samples [S, M] as tpe_ehvi_set takes them) or
 * TPE_ACQF_LOGPI (n_obj = 0: no objective part).  gps[n_obj .. n_gp - 1] are constraints: their LogPI terms
 * (acqf.py:175-182) are summed as ConstrainedLogEI / ConstrainedLogEHVI sum them.  thresholds [n_gp]: LogEI's f0
 * (-inf gives the reference's zeros), then the constraints' thresholds (finite).  stabilizing_noise is added to every
 * variance.  Every GP context must be conditioned (tpe_gp_condition), distinct, of one width P and on this context's
 * device, and must outlive the calls; TPE_E_STATE / TPE_E_INVALID naming the violated condition.
 * tpe_acqf_eval: value [Q] at the rows of X [Q, P] and, with grad non-NULL, d value / dx [Q, P].  The GP posteriors
 * are computed on this context's stream after the work queued on each GP context's stream, with one synchronise per
 * call.  A row's value is the same bits whatever Q, the row's position and the gradient request.  TPE_E_STATE when a
 * GP context was conditioned again or changed since tpe_acqf_set; TPE_E_INVALID for Q < 1, or naming the bytes when
 * the device lacks the memory.  Non-finite entries of X are evaluated: NaN propagates as in torch. */
enum { TPE_ACQF_LOGEI = 0, TPE_ACQF_LOGEHVI = 1, TPE_ACQF_LOGPI = 2 };
int tpe_acqf_set(tpe_ctx* ctx, int32_t kind, tpe_ctx* const* gps, int32_t n_gp, int32_t n_obj,
                 const double* thresholds, double stabilizing_noise, const double* lower, const double* intervals,
                 int64_t B, const double* samples, int32_t S);
int tpe_acqf_eval(tpe_ctx* ctx, const double* X, int64_t Q, double* value, double* grad);
/* Non-dominated box decomposition of LogEHVI (get_non_dominated_box_bounds, optuna/_hypervolume/box_decomposition.py:
 * 138-157, as optuna/_gp/acqf.py:255-263 calls it).  Kept apart from every other state of the context.
 * tpe_box_decomposition decomposes the space that the rows of loss_vals [n, M] (minimised) do not dominate, below
 * ref_point [M], into *n_boxes boxes and keeps them: the reference's arrays bit for bit, in its row order.  The one
 * freedom is numpy's: of rows that np.unique merges because they differ only in the sign of a zero, which one it keeps.
 * 2 <= M <= 24, n >= 1, loss values finite, no NaN in ref_point; TPE_E_INVALID naming the violated condition, or the
 * bytes needed when the device lacks the memory of the bounds' pool.  *n_boxes = 0 is a valid result.
 * tpe_get_box_decomposition copies out the last decomposition: lower, upper [n_boxes, M] (each may be NULL) and, if
 * stats is non-NULL, stats[6] = the front's size, the first pass's bounds made and kept, the second pass's front,
 * bounds made and kept.  TPE_E_STATE before a successful tpe_box_decomposition. */
int tpe_box_decomposition(tpe_ctx* ctx, const double* loss_vals, int64_t n, int32_t M, const double* ref_point,
                          int64_t* n_boxes);
int tpe_get_box_decomposition(tpe_ctx* ctx, double* lower, double* upper, int64_t* stats);
/* Candidates / log-densities of the last tpe_sample_and_select (all asks).
 * samples [n_asks * C, n_cols]; logl, logg [n_asks * C].  Any pointer may be NULL. */
int tpe_get_candidates(tpe_ctx* ctx, double* samples, double* logl, double* logg);
/* log-density of arbitrary points under the last-built estimator
 * (replaces _ParzenEstimator.log_pdf, parzen_estimator.py:84-86).  x [n, n_cols]. */
int tpe_logpdf(tpe_ctx* ctx, int which, const double* x, int64_t n, double* out);

/* CUDA-event timing (ms, on the context stream) of the stages of the last prepare / build /
 * sample_and_select sequence: [0] split, [1] estimator build, [2] uniforms H2D, [3] sample,
 * [4] log-density under l(x), [5] main log-density kernel under g(x), [6] its fix-up pass,
 * [7] select, [8] first-to-last span.  launches = kernels launched by the sequence. */
int tpe_last_timing(tpe_ctx* ctx, float* ms9, int32_t* launches);
/* Peak-probe: fp64 FMA throughput of this device (TFLOP/s), measured by a dependent-chain-free
 * DFMA kernel; used by bench.py as the compute-roof denominator. */
int tpe_probe_fp64_tflops(tpe_ctx* ctx, double* tflops);
/* Which kernel variant the last log-density pass used (static string). */
const char* tpe_last_logpdf_kernel(tpe_ctx* ctx);

#ifdef __cplusplus
}
#endif
#endif /* OPTUNA_B200_TPE_H_ */
