"""Array-level Python face of the C ABI: one ``TPEEngine`` = one ``tpe_ctx`` on one GPU.

This is the thin layer ``B200TPESampler`` (sampler.py) drives; it is also what the parity tests
call so that every check goes through the C ABI.  It holds no algorithmic logic: inputs are
validated and copied by the library (include/optuna_b200_tpe.h).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Sequence

import numpy as np

from . import _lib


@dataclass(frozen=True)
class ParamSpec:
    """One column of the search space (mirror of optuna.distributions.*Distribution fields)."""

    kind: int  # _lib.KIND_*
    low: float = 0.0
    high: float = 0.0
    step: float | None = None
    log: bool = False
    n_choices: int = 0
    dist_table: np.ndarray | None = None  # categorical_distance_func evaluated on all pairs


def _ptr(a: np.ndarray | None):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _f64(a, shape=None) -> np.ndarray:
    out = np.ascontiguousarray(a, dtype=np.float64)
    if shape is not None:
        out = out.reshape(shape)
    return out


class GPCholeskyError(RuntimeError):
    """The Gaussian-process covariance is not positive definite: a Cholesky pivot was <= 0 or NaN.  A
    ``RuntimeError``, like the ``LinAlgError`` torch's Cholesky raises, so that optuna's fit retries and falls back
    the same way."""


class TPEEngine:
    def __init__(self, device: int = 0) -> None:
        self._lib = _lib.load()
        handle = C.c_void_p()
        rc = self._lib.tpe_ctx_create(int(device), C.byref(handle))
        if rc != 0:
            raise RuntimeError(f"tpe_ctx_create(device={device}) failed with code {rc}: a CUDA device is required")
        self._h = handle
        self.device = int(device)
        self.n_params = 0
        self._cfg = None
        self._pc = 0
        self._ncat = self._nnum = 0
        self._specs: list[ParamSpec] = []
        self._cols: list[int] = []
        self._gp_P = 0
        self._ehvi_M = 0
        self._acqf_P = 0

    # -- lifecycle -----------------------------------------------------------------------------
    def close(self) -> None:
        if getattr(self, "_h", None):
            for p in getattr(self, "_pinned", []):
                self._lib.tpe_host_free(self._h, C.c_void_p(p))
            self._pinned = []
            self._lib.tpe_ctx_destroy(self._h)
            self._h = None

    def __del__(self) -> None:  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc: int) -> None:
        if rc == 0:
            return
        msg = self._lib.tpe_last_error(self._h).decode()
        if rc == _lib.TPE_E_INVALID:
            raise ValueError(msg)
        if rc == _lib.TPE_E_NOTPD:
            raise GPCholeskyError(msg)
        raise RuntimeError(f"libtpe_b200 error {rc}: {msg}")

    # -- space / history -------------------------------------------------------------------------
    def set_space(self, specs: Sequence[ParamSpec]) -> None:
        n = len(specs)
        arr = (_lib.ParamDesc * max(n, 1))()
        offs = np.full(max(n, 1), -1, dtype=np.int64)
        tables = []
        at = 0
        for i, s in enumerate(specs):
            arr[i].kind = s.kind
            arr[i].log = int(bool(s.log))
            arr[i].has_step = int(s.step is not None)
            arr[i].n_choices = int(s.n_choices)
            arr[i].low = float(s.low)
            arr[i].high = float(s.high)
            arr[i].step = float(s.step) if s.step is not None else 0.0
            if s.dist_table is not None:
                t = _f64(s.dist_table, (s.n_choices, s.n_choices))
                tables.append(t.ravel())
                offs[i] = at
                at += t.size
        flat = np.concatenate(tables) if tables else None
        self._check(self._lib.tpe_space_set(self._h, arr, n, _ptr(flat), _ptr(offs) if tables else None))
        self._specs = list(specs)
        self.n_params = n

    def set_history(self, X, category, key) -> None:
        X = _f64(X, (-1, self.n_params))
        cat = np.ascontiguousarray(category, dtype=np.int8)
        key = _f64(key, (-1, 2))
        assert X.shape[0] == cat.shape[0] == key.shape[0]
        self._check(self._lib.tpe_history_set(self._h, _ptr(X), _ptr(cat), _ptr(key), X.shape[0]))

    def append_history(self, X, category, key) -> None:
        X = _f64(X, (-1, self.n_params))
        cat = np.ascontiguousarray(category, dtype=np.int8).reshape(-1)
        key = _f64(key, (-1, 2))
        self._check(self._lib.tpe_history_append(self._h, _ptr(X), _ptr(cat), _ptr(key), X.shape[0]))

    def update_history(self, X, category, key, at_row: int) -> None:
        """Overwrite rows [at_row, at_row + n) in place (a trial that finished keeps its position); a write
        past the end extends the history."""
        X = _f64(X, (-1, self.n_params))
        cat = np.ascontiguousarray(category, dtype=np.int8).reshape(-1)
        key = _f64(key, (-1, 2))
        self._check(self._lib.tpe_history_update(self._h, _ptr(X), _ptr(cat), _ptr(key), X.shape[0], int(at_row)))

    def set_values(self, values, at_row: int = 0, n_objectives: int | None = None) -> None:
        """Sign-normalised objective values [n, M] of history rows [at_row, at_row + n) (MOTPE).  Pass
        `n_objectives` when n may be 0 (the shape of an empty array does not say)."""
        v = _f64(values)
        m = int(n_objectives) if n_objectives is not None else (v.shape[1] if v.ndim == 2 else 1)
        v = v.reshape(-1, m)
        self._check(self._lib.tpe_history_set_values(self._h, _ptr(v), v.shape[0], m, int(at_row)))

    def set_history_device(self, dX: int, dcat: int, dkey: int, n: int, col_has_missing=None) -> None:
        miss = None if col_has_missing is None else np.ascontiguousarray(col_has_missing, dtype=np.uint8)
        self._check(self._lib.tpe_history_set_device(self._h, C.c_void_p(dX), C.c_void_p(dcat), C.c_void_p(dkey),
                                                     int(n), _ptr(miss)))

    def history_device_ptrs(self) -> tuple[int, int, int]:
        a, b, c = C.c_void_p(), C.c_void_p(), C.c_void_p()
        self._check(self._lib.tpe_history_device_ptrs(self._h, C.byref(a), C.byref(b), C.byref(c)))
        return a.value, b.value, c.value

    @property
    def history_size(self) -> int:
        return int(self._lib.tpe_history_size(self._h))

    # -- stages ------------------------------------------------------------------------------------
    def _make_cfg(self, *, n_below: int, n_candidates: int, multivariate: bool, prior_weight: float = 1.0,
                  magic_clip: bool = True, endpoints: bool = False) -> _lib.Cfg:
        return _lib.Cfg(float(prior_weight), int(magic_clip), int(endpoints), int(multivariate),
                        int(n_candidates), int(n_below))

    def _note_cols(self, cols: Sequence[int], n_candidates: int) -> np.ndarray:
        self._cols = [int(c) for c in cols]
        self._pc = len(self._cols)
        self._ncat = sum(1 for c in self._cols if 0 <= c < self.n_params and self._specs[c].kind == _lib.KIND_CAT)
        self._nnum = self._pc - self._ncat
        self._C = int(n_candidates)
        return np.ascontiguousarray(self._cols, dtype=np.int32)

    def uniforms_per_ask(self) -> int:
        return self._C * (1 + self._ncat + self._nnum)

    def prepare(self, cols: Sequence[int], **cfg) -> tuple[int, int, int]:
        c = self._make_cfg(**cfg)
        cols_a = self._note_cols(cols, c.n_candidates)
        info = _lib.SplitInfo()
        self._check(self._lib.tpe_prepare(self._h, C.byref(c), _ptr(cols_a), len(cols_a), C.byref(info)))
        self._info = (int(info.n_below_all), int(info.n_below_obs), int(info.n_above_obs))
        return self._info

    def build(self, w_below=None, w_above=None) -> None:
        wb = None if w_below is None else _f64(w_below)
        wa = None if w_above is None else _f64(w_above)
        if wb is not None:
            assert wb.size == self._info[1], (wb.size, self._info)
        if wa is not None:
            assert wa.size == self._info[2], (wa.size, self._info)
        self._check(self._lib.tpe_build(self._h, _ptr(wb), _ptr(wa)))

    def sample_and_select(self, uniforms, n_asks: int = 1):
        """uniforms=None: consume the device-generated uniforms of ``stage_rng``."""
        u = None
        if uniforms is not None:
            u = _f64(uniforms).reshape(-1)
            assert u.size == n_asks * self.uniforms_per_ask(), (u.size, n_asks, self.uniforms_per_ask())
        x = np.empty((n_asks, self._pc), dtype=np.float64)
        acq = np.empty(n_asks, dtype=np.float64)
        best = np.empty(n_asks, dtype=np.int64)
        self._check(self._lib.tpe_sample_and_select(self._h, _ptr(u), int(n_asks), _ptr(x), _ptr(acq), _ptr(best)))
        self._last_asks = n_asks
        return x, acq, best

    def sample_and_select_async(self, uniforms, n_asks: int = 1) -> None:
        """Queue ``sample_and_select`` and return; ``collect()`` waits and returns the results."""
        u = None
        if uniforms is not None:
            u = _f64(uniforms).reshape(-1)
            assert u.size == n_asks * self.uniforms_per_ask(), (u.size, n_asks, self.uniforms_per_ask())
        self._check(self._lib.tpe_sample_and_select_async(self._h, _ptr(u), int(n_asks)))
        self._last_asks = n_asks

    def collect(self):
        n_asks = self._last_asks
        x = np.empty((n_asks, self._pc), dtype=np.float64)
        acq = np.empty(n_asks, dtype=np.float64)
        best = np.empty(n_asks, dtype=np.int64)
        self._check(self._lib.tpe_collect(self._h, _ptr(x), _ptr(acq), _ptr(best)))
        return x, acq, best

    def rng_snapshot(self) -> tuple:
        """The generator state the device holds (after the last staged draw) as ``RandomState.set_state`` takes it."""
        key = np.empty(624, dtype=np.uint32)
        pos = C.c_int32()
        self._check(self._lib.tpe_rng_state(self._h, _ptr(key), C.byref(pos)))
        name, has_gauss, cached = self._rng_tail
        return (name, key, int(pos.value), has_gauss, cached)

    def set_kernel_shard(self, rank: int, world: int) -> None:
        """This engine evaluates g(x) over slice `rank` of `world` of the above kernels (world = 1: off)."""
        self._check(self._lib.tpe_set_kernel_shard(self._h, int(rank), int(world)))

    def sample_and_partial(self, uniforms, n_asks: int = 1) -> tuple[int, int]:
        """Candidates, l(x) and this engine's slice of g(x): (device address of the [n_asks * C] (max, sum) pairs,
        their padded count)."""
        u = None
        if uniforms is not None:
            u = _f64(uniforms).reshape(-1)
            assert u.size == n_asks * self.uniforms_per_ask()
        ptr, stride = C.c_void_p(), C.c_int64()
        self._check(self._lib.tpe_sample_and_partial(self._h, _ptr(u), int(n_asks), C.byref(ptr), C.byref(stride)))
        self._last_asks = n_asks
        return int(ptr.value), int(stride.value)

    def finish_from_partials(self, gathered_ptr: int, world: int):
        n_asks = self._last_asks
        x = np.empty((n_asks, self._pc), dtype=np.float64)
        acq = np.empty(n_asks, dtype=np.float64)
        best = np.empty(n_asks, dtype=np.int64)
        self._check(self._lib.tpe_finish_from_partials(self._h, C.c_void_p(int(gathered_ptr)), int(world), _ptr(x), _ptr(acq),
                                                       _ptr(best)))
        return x, acq, best

    def sample_and_select_device(self, n_asks: int = 1) -> int:
        """Like ``sample_and_select(None, n_asks)`` but the results stay on the device; returns the device
        address of out_x [n_asks, n_cols] fp64 (valid until the next call on this engine)."""
        self._check(self._lib.tpe_sample_and_select(self._h, None, int(n_asks), None, None, None))
        self._last_asks = n_asks
        px = C.c_void_p()
        self._check(self._lib.tpe_result_device_ptrs(self._h, C.byref(px), None, None))
        return int(px.value)

    def rng_state_device(self) -> int:
        """Device address of the generator state (625 uint32) kept by ``stage_rng``; see tpe_rng_state_device."""
        p = C.c_void_p()
        self._check(self._lib.tpe_rng_state_device(self._h, C.byref(p)))
        return int(p.value)

    def stage_rng(self, rng: np.random.RandomState | None, count: int, skip: int = 0, state=None) -> None:
        """Generate the next `count` outputs of ``rng.random_sample`` on the device (after dropping
        `skip`); the following ``sample_and_select(None, n_asks)`` consumes them.  ``finish_rng(rng)``
        then moves `rng` to the state after the draws.  ``rng=None`` continues from the state the
        previous staged draw ended in (the host generator is then stale until ``finish_rng``)."""
        if rng is None:
            self._check(self._lib.tpe_stage_uniforms_mt19937(self._h, None, 0, int(skip), int(count)))
            return
        st = rng.get_state() if state is None else state
        key = np.ascontiguousarray(st[1], dtype=np.uint32)
        self._rng_tail = (st[0], st[3], st[4])
        self._check(self._lib.tpe_stage_uniforms_mt19937(self._h, _ptr(key), int(st[2]), int(skip), int(count)))

    def get_uniforms(self, count: int) -> np.ndarray:
        out = np.empty(int(count), dtype=np.float64)
        self._check(self._lib.tpe_get_uniforms(self._h, _ptr(out), int(count)))
        return out

    def finish_rng(self, rng: np.random.RandomState) -> None:
        key = np.empty(624, dtype=np.uint32)
        pos = C.c_int32()
        self._check(self._lib.tpe_rng_state(self._h, _ptr(key), C.byref(pos)))
        name, has_gauss, cached = self._rng_tail
        rng.set_state((name, key, int(pos.value), has_gauss, cached))

    def pinned_empty(self, n: int) -> np.ndarray:
        """float64[n] in page-locked host memory (freed with the engine): copies from it are async DMAs."""
        p = C.c_void_p()
        self._check(self._lib.tpe_host_alloc(self._h, C.c_size_t(int(n) * 8), C.byref(p)))
        if not hasattr(self, "_pinned"):
            self._pinned = []
        self._pinned.append(p.value)
        return np.ctypeslib.as_array((C.c_double * int(n)).from_address(p.value))

    def stage_uniforms(self, uniforms: np.ndarray) -> np.ndarray:
        """Start uploading the uniforms of the next `sample_and_select` now (latency hint); pass the
        returned array (same memory) to `sample_and_select`."""
        u = _f64(uniforms).reshape(-1)
        self._check(self._lib.tpe_stage_uniforms(self._h, _ptr(u), int(u.size)))
        return u

    def suggest(self, cols: Sequence[int], uniforms, n_asks: int = 1, w_below=None, w_above=None, **cfg):
        c = self._make_cfg(**cfg)
        cols_a = self._note_cols(cols, c.n_candidates)
        u = _f64(uniforms).reshape(-1)
        assert u.size == n_asks * self.uniforms_per_ask()
        wb = None if w_below is None else _f64(w_below)
        wa = None if w_above is None else _f64(w_above)
        x = np.empty((n_asks, self._pc), dtype=np.float64)
        acq = np.empty(n_asks, dtype=np.float64)
        best = np.empty(n_asks, dtype=np.int64)
        self._check(self._lib.tpe_suggest(self._h, C.byref(c), _ptr(cols_a), len(cols_a), _ptr(wb), _ptr(wa),
                                          _ptr(u), int(n_asks), _ptr(x), _ptr(acq), _ptr(best)))
        self._last_asks = n_asks
        self._info = self.split_info()
        return x, acq, best

    def suggest_univariate_batch(self, cols: Sequence[int], uniforms, w_below=None, w_above=None, **cfg):
        """The per-parameter suggestions of one univariate trial together (tpe_suggest_univariate_batch);
        uniforms=None consumes the device-generated uniforms of ``stage_rng(.., len(cols) * 2 * C)``.
        Raises RuntimeError("... not batchable ...") when the columns cannot share a split."""
        c = self._make_cfg(**cfg)
        cols_a = np.ascontiguousarray([int(v) for v in cols], dtype=np.int32)
        u = None
        if uniforms is not None:
            u = _f64(uniforms).reshape(-1)
            assert u.size == len(cols_a) * 2 * c.n_candidates
        wb = None if w_below is None else _f64(w_below)
        wa = None if w_above is None else _f64(w_above)
        x = np.empty(len(cols_a), dtype=np.float64)
        acq = np.empty(len(cols_a), dtype=np.float64)
        best = np.empty(len(cols_a), dtype=np.int64)
        self._check(self._lib.tpe_suggest_univariate_batch(self._h, C.byref(c), _ptr(cols_a), len(cols_a), _ptr(wb),
                                                           _ptr(wa), _ptr(u), _ptr(x), _ptr(acq), _ptr(best)))
        return x, acq, best

    def suggest_univariate_batch_async(self, cols: Sequence[int], uniforms, w_below=None, w_above=None, **cfg) -> None:
        """Queue ``suggest_univariate_batch`` and return; ``collect_univariate()`` waits and returns the results."""
        c = self._make_cfg(**cfg)
        cols_a = np.ascontiguousarray([int(v) for v in cols], dtype=np.int32)
        u = None
        if uniforms is not None:
            u = _f64(uniforms).reshape(-1)
            assert u.size == len(cols_a) * 2 * c.n_candidates
        wb = None if w_below is None else _f64(w_below)
        wa = None if w_above is None else _f64(w_above)
        self._check(self._lib.tpe_suggest_univariate_batch_async(self._h, C.byref(c), _ptr(cols_a), len(cols_a), _ptr(wb),
                                                                 _ptr(wa), _ptr(u)))
        self._uni_pending = len(cols_a)

    def collect_univariate(self):
        n = self._uni_pending
        x = np.empty(n, dtype=np.float64)
        acq = np.empty(n, dtype=np.float64)
        best = np.empty(n, dtype=np.int64)
        self._check(self._lib.tpe_collect_univariate(self._h, _ptr(x), _ptr(acq), _ptr(best)))
        return x, acq, best

    def split_info(self) -> tuple[int, int, int]:
        info = _lib.SplitInfo()
        self._check(self._lib.tpe_get_split_info(self._h, C.byref(info)))
        return int(info.n_below_all), int(info.n_below_obs), int(info.n_above_obs)

    # -- analysis ----------------------------------------------------------------------------------
    def hypervolume_history(self, values, feasible, ref) -> np.ndarray:
        """Hypervolume after each trial of ``values`` [n, M] (sign-normalised, trial order) against the
        sign-normalised reference point ``ref`` [M]; ``feasible`` [n] bools or None (all feasible).  Leaves the
        history and the suggestion state of this engine unchanged (tpe_hypervolume_history)."""
        v = _f64(values)
        r = _f64(ref).reshape(-1)
        if v.ndim != 2 or v.shape[1] != r.size:
            raise ValueError(f"values must be [n, {r.size}], got shape {v.shape}")
        f = None
        if feasible is not None:
            f = np.ascontiguousarray(feasible, dtype=np.uint8).reshape(-1)
            if f.size != v.shape[0]:
                raise ValueError(f"feasible has {f.size} entries for {v.shape[0]} trials")
        out = np.empty(v.shape[0], dtype=np.float64)
        self._check(self._lib.tpe_hypervolume_history(self._h, _ptr(v), _ptr(f), v.shape[0], r.size, _ptr(r),
                                                      _ptr(out)))
        return out

    def pareto_front(self, values) -> np.ndarray:
        """Pareto-front flags of the rows of ``values`` [n, M] (sign-normalised: every objective minimised): True
        where no row is <= the row everywhere and < somewhere.  Leaves the history and the suggestion state of
        this engine unchanged (tpe_pareto_front)."""
        v = _f64(values)
        if v.ndim != 2:
            raise ValueError(f"values must be [n, n_objectives], got shape {v.shape}")
        out = np.empty(v.shape[0], dtype=np.uint8)
        self._check(self._lib.tpe_pareto_front(self._h, _ptr(v), v.shape[0], v.shape[1], _ptr(out)))
        return out.view(bool)

    def fanova_variances(self, node_offsets, left, right, feature, threshold, value, bounds, param_offsets,
                         raw_features) -> tuple[np.ndarray, np.ndarray]:
        """fANOVA variances of a forest (tpe_fanova_variances): ``(tree_variance [T], marginal_variance
        [n_params, T])``.  Tree t is the nodes ``[node_offsets[t], node_offsets[t + 1])`` of the concatenated
        sklearn arrays (children indexed within their tree); parameter p is the raw features
        ``raw_features[param_offsets[p]:param_offsets[p + 1]]``.  Leaves the history and the suggestion state of
        this engine unchanged."""
        off = np.ascontiguousarray(node_offsets, dtype=np.int64)
        i32 = [np.ascontiguousarray(a, dtype=np.int32) for a in (left, right, feature)]
        thr, val = _f64(threshold), _f64(value)
        bnd = _f64(bounds)
        po = np.ascontiguousarray(param_offsets, dtype=np.int32)
        cols = np.ascontiguousarray(raw_features, dtype=np.int32)
        T, n_params = off.size - 1, po.size - 1
        if bnd.ndim != 2 or bnd.shape[1] != 2:
            raise ValueError(f"bounds must be [n_features, 2], got shape {bnd.shape}")
        n = int(off[-1]) if off.size else 0
        if T < 1 or any(a.shape != (n,) for a in (*i32, thr, val)) or n_params < 0 or cols.size != int(po[-1]):
            raise ValueError("inconsistent fANOVA forest arrays")
        tree_var = np.empty(T)
        marg = np.empty((max(n_params, 0), T))
        self._check(self._lib.tpe_fanova_variances(self._h, T, _ptr(off), *(_ptr(a) for a in i32), _ptr(thr),
                                                   _ptr(val), bnd.shape[0], _ptr(bnd), n_params, _ptr(po),
                                                   _ptr(cols), _ptr(tree_var), _ptr(marg)))
        return tree_var, marg

    def gp_set_data(self, X, y, is_categorical) -> None:
        """Training data of the terminator's Gaussian process (tpe_gp_set_data): ``X`` [n, P] normalised parameters,
        ``y`` [n] standardised values, ``is_categorical`` [P].  Allocates two n x n fp64 matrices on the device;
        ``ValueError`` naming the need when it lacks the memory.  Leaves the history and the suggestion state of
        this engine unchanged."""
        Xa, ya = _f64(X), _f64(y)
        cat = np.ascontiguousarray(is_categorical, dtype=np.uint8)
        if Xa.ndim != 2 or ya.shape != (Xa.shape[0],) or cat.shape != (Xa.shape[1],):
            raise ValueError(f"GP data must be X [n, P], y [n], is_categorical [P]; got {Xa.shape}, {ya.shape}, "
                             f"{cat.shape}")
        self._gp_P = 0   # a failed call leaves no GP data in the context either
        self._check(self._lib.tpe_gp_set_data(self._h, _ptr(Xa), _ptr(ya), _ptr(cat), Xa.shape[0], Xa.shape[1]))
        self._gp_P = Xa.shape[1]

    def gp_loss(self, raw_params, minimum_noise: float, deterministic: bool = False) -> tuple[float, np.ndarray]:
        """Negative marginal log-likelihood of the GP data and its gradient in the raw kernel parameters (log
        inverse squared lengthscales, log kernel scale, log(noise_var - minimum_noise)) (tpe_gp_loss).  With
        ``deterministic`` the noise is fixed at ``minimum_noise``, the last raw parameter is ignored and its gradient
        is 0 (tpe_gp_loss_fixed_noise).  Raises ``GPCholeskyError`` when the covariance is not positive definite."""
        raw = _f64(raw_params)
        if self._gp_P and raw.shape != (self._gp_P + 2,):   # without GP data the library reports that first
            raise ValueError(f"raw_params must have {self._gp_P + 2} entries, got shape {raw.shape}")
        loss = C.c_double()
        grad = np.empty(raw.size)
        fn = self._lib.tpe_gp_loss_fixed_noise if deterministic else self._lib.tpe_gp_loss
        self._check(fn(self._h, _ptr(raw), float(minimum_noise), C.byref(loss), _ptr(grad)))
        return loss.value, grad

    def gp_posterior(self, params, Xq, beta: float) -> tuple[np.ndarray, np.ndarray]:
        """``(mean + sqrt(beta var), mean - sqrt(beta var))`` of the GP posterior at the rows of ``Xq`` [m, P], for
        ``params`` = (inverse squared lengthscales, kernel scale, noise_var) (tpe_gp_posterior).  Raises
        ``GPCholeskyError`` when the covariance is not positive definite."""
        prm, xq = _f64(params), _f64(Xq)
        if xq.ndim != 2 or (self._gp_P and (prm.shape != (self._gp_P + 2,) or xq.shape[1] != self._gp_P)):
            raise ValueError(f"params must have {self._gp_P + 2} entries and Xq {self._gp_P} columns")
        ucb, lcb = np.empty(xq.shape[0]), np.empty(xq.shape[0])
        self._check(self._lib.tpe_gp_posterior(self._h, _ptr(prm), _ptr(xq), xq.shape[0], float(beta), _ptr(ucb),
                                               _ptr(lcb)))
        return ucb, lcb

    def gp_posterior_moments(self, params, Xq, n_joint: int = 0) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
        """``(mean, var, cov)`` of the GP posterior at the rows of ``Xq`` [m, P], for ``params`` = (inverse squared
        lengthscales, kernel scale, noise_var) (tpe_gp_posterior_moments).  ``var`` is clamped at 0.  ``cov`` is the
        joint covariance [n_joint, n_joint] of the first ``n_joint`` rows (0, or 2 to 64), diagonal clamped at 0.
        Raises ``GPCholeskyError`` when the covariance is not positive definite."""
        prm, xq = _f64(params), _f64(Xq)
        if xq.ndim != 2 or (self._gp_P and (prm.shape != (self._gp_P + 2,) or xq.shape[1] != self._gp_P)):
            raise ValueError(f"params must have {self._gp_P + 2} entries and Xq {self._gp_P} columns")
        n_joint = int(n_joint)
        mean, var = np.empty(xq.shape[0]), np.empty(xq.shape[0])
        cov = np.empty((max(n_joint, 0), max(n_joint, 0)))
        self._check(self._lib.tpe_gp_posterior_moments(self._h, _ptr(prm), _ptr(xq), xq.shape[0], n_joint, _ptr(mean),
                                                       _ptr(var), _ptr(cov) if n_joint else None))
        return mean, var, cov

    def gp_condition(self, params) -> None:
        """Factorise the GP covariance once at ``params`` = (inverse squared lengthscales, kernel scale, noise_var) and
        keep the factor for ``gp_query`` (tpe_gp_condition).  ``gp_set_data``, ``gp_loss`` and the posterior calls
        undo it.  Raises ``GPCholeskyError`` when the covariance is not positive definite."""
        prm = _f64(params)
        if self._gp_P and prm.shape != (self._gp_P + 2,):
            raise ValueError(f"params must have {self._gp_P + 2} entries, got shape {prm.shape}")
        self._check(self._lib.tpe_gp_condition(self._h, _ptr(prm)))

    def gp_query(self, Xq, grad: bool = False):
        """The GP posterior at the rows of ``Xq`` [m, P] against the factor of ``gp_condition`` (tpe_gp_query):
        ``(mean, var)``, ``var`` clamped at 0, and with ``grad`` also ``(dmean, dvar)`` [m, P], their gradients in the
        query point.  The values are the same bits with and without ``grad``."""
        xq = _f64(Xq)
        if xq.ndim != 2 or (self._gp_P and xq.shape[1] != self._gp_P):
            raise ValueError(f"Xq must be [m, {self._gp_P}], got shape {xq.shape}")
        mean, var = np.empty(xq.shape[0]), np.empty(xq.shape[0])
        dmean = np.empty(xq.shape) if grad else None
        dvar = np.empty(xq.shape) if grad else None
        self._check(self._lib.tpe_gp_query(self._h, _ptr(xq), xq.shape[0], _ptr(mean), _ptr(var), _ptr(dmean),
                                           _ptr(dvar)))
        return (mean, var, dmean, dvar) if grad else (mean, var)

    def gp_batch_set(self, offsets, X, y, is_categorical) -> None:
        """Many independent GPs at once (tpe_gp_batch_set): GP i is fitted to the rows ``offsets[i] ..
        offsets[i + 1] - 1`` of ``X`` [N, P] and ``y`` [N]; all share ``is_categorical`` [P].  ``ValueError`` on bad
        input, or naming the bytes when the device lacks the memory.  Leaves the other state of this engine
        unchanged."""
        off = np.ascontiguousarray(offsets, dtype=np.int64)
        Xa, ya = _f64(X), _f64(y)
        cat = np.ascontiguousarray(is_categorical, dtype=np.uint8)
        if off.ndim != 1 or Xa.ndim != 2 or ya.shape != (Xa.shape[0],) or cat.shape != (Xa.shape[1],) or (
                off.size and off[-1] != Xa.shape[0]):
            raise ValueError(f"batched GP data must be offsets [n_gp + 1] ending at N, X [N, P], y [N], "
                             f"is_categorical [P]; got {off.shape}, {Xa.shape}, {ya.shape}, {cat.shape}")
        self._gpb_P = 0   # a failed call leaves no batched GP data in the context either
        self._check(self._lib.tpe_gp_batch_set(self._h, off.size - 1, _ptr(off), Xa.shape[1], _ptr(Xa), _ptr(ya),
                                               _ptr(cat)))
        self._gpb_P = Xa.shape[1]

    def gp_batch_loss(self, gp_idx, raw, minimum_noise: float, deterministic: bool = False):
        """``gp_loss`` for k jobs at once (tpe_gp_batch_loss): job b is GP ``gp_idx[b]`` at ``raw[b]`` [P + 2].
        Returns ``(loss [k], grad [k, P + 2], status [k])``; status 1 marks a job whose covariance is not positive
        definite (or whose kernel parameters are not finite), its loss and gradient NaN.  With ``deterministic`` the
        noise is fixed at ``minimum_noise``, the last raw parameter is ignored and its gradient is 0
        (tpe_gp_batch_loss_fixed_noise)."""
        idx = np.ascontiguousarray(gp_idx, dtype=np.int32)
        r = _f64(raw)
        P = getattr(self, "_gpb_P", 0)
        if idx.ndim != 1 or (P and r.shape != (idx.size, P + 2)):
            raise ValueError(f"raw must be [k, {P + 2}] for k = {idx.size} GP indices, got shape {r.shape}")
        loss, grad = np.empty(idx.size), np.empty(r.shape)
        status = np.empty(idx.size, dtype=np.int32)
        fn = self._lib.tpe_gp_batch_loss_fixed_noise if deterministic else self._lib.tpe_gp_batch_loss
        self._check(fn(self._h, idx.size, _ptr(idx), _ptr(r), float(minimum_noise), _ptr(loss), _ptr(grad),
                       _ptr(status)))
        return loss, grad, status

    def gp_batch_bounds(self, gp_idx, params, beta, samples):
        """RegretBoundEvaluator's three maxima for k jobs (tpe_gp_batch_bounds): job b is GP ``gp_idx[b]`` at
        ``params[b]`` [P + 2] (inverse squared lengthscales, kernel scale, noise_var) with ``beta[b]`` and the sample
        rows ``samples[b]`` [S, P].  Returns ``(out [k, 3], status [k])``: max UCB over the train rows, max UCB over
        the samples, max LCB over the train rows; status as for ``gp_batch_loss``."""
        idx = np.ascontiguousarray(gp_idx, dtype=np.int32)
        prm, bt, xs = _f64(params), _f64(beta), _f64(samples)
        P = getattr(self, "_gpb_P", 0)
        if idx.ndim != 1 or bt.shape != idx.shape or xs.ndim != 3 or xs.shape[0] != idx.size or (
                P and (prm.shape != (idx.size, P + 2) or xs.shape[2] != P)):
            raise ValueError(f"bounds need params [k, {P + 2}], beta [k], samples [k, S, {P}]; got {prm.shape}, "
                             f"{bt.shape}, {xs.shape}")
        out = np.empty((idx.size, 3))
        status = np.empty(idx.size, dtype=np.int32)
        self._check(self._lib.tpe_gp_batch_bounds(self._h, idx.size, _ptr(idx), _ptr(prm), _ptr(bt), xs.shape[1],
                                                  _ptr(xs), _ptr(out), _ptr(status)))
        return out, status

    def gp_batch_moments(self, gp_idx, params, rows, n_joint: int = 0):
        """EMMREvaluator's posterior terms for k jobs (tpe_gp_batch_moments): job b is GP ``gp_idx[b]`` at
        ``params[b]`` [P + 2] (inverse squared lengthscales, kernel scale, noise_var), queried at its own train rows
        ``rows[b]`` [m] (row indices within the GP, 1 <= m <= 3).  Returns ``(mean [k, m], var [k, m], cov [k, J, J],
        status [k])``: ``var`` clamped at 0, ``cov`` the joint covariance of the first ``J = n_joint`` rows (0, or 2
        to m), diagonal clamped at 0; status as for ``gp_batch_loss``."""
        idx = np.ascontiguousarray(gp_idx, dtype=np.int32)
        prm = _f64(params)
        rw = np.ascontiguousarray(rows, dtype=np.int32)
        P = getattr(self, "_gpb_P", 0)
        if idx.ndim != 1 or rw.ndim != 2 or rw.shape[0] != idx.size or (P and prm.shape != (idx.size, P + 2)):
            raise ValueError(f"moments need params [k, {P + 2}] and rows [k, m]; got {prm.shape}, {rw.shape}")
        n_joint = int(n_joint)
        m = rw.shape[1]
        mean, var = np.empty((idx.size, m)), np.empty((idx.size, m))
        J = max(n_joint, 0)
        cov = np.empty((idx.size, J, J))
        status = np.empty(idx.size, dtype=np.int32)
        self._check(self._lib.tpe_gp_batch_moments(self._h, idx.size, _ptr(idx), _ptr(prm), m, _ptr(rw), n_joint,
                                                   _ptr(mean), _ptr(var), _ptr(cov) if n_joint else None,
                                                   _ptr(status)))
        return mean, var, cov, status

    def ehvi_set(self, lower, intervals, samples) -> None:
        """The non-dominated boxes and fixed QMC samples of a log-EHVI acquisition (tpe_ehvi_set): ``lower`` and
        ``intervals`` [B, M] (intervals already clamped at 1e-12), ``samples`` [S, M].  2 <= M <= 24, 1 <= S <= 1024,
        no NaN (infinities are allowed).  Leaves the history, suggestion and GP state of this engine unchanged."""
        lb, iv, z = _f64(lower), _f64(intervals), _f64(samples)
        if lb.ndim != 2 or iv.shape != lb.shape or z.ndim != 2 or z.shape[1] != lb.shape[1]:
            raise ValueError(f"EHVI inputs must be lower [B, M], intervals [B, M], samples [S, M]; got {lb.shape}, "
                             f"{iv.shape}, {z.shape}")
        self._ehvi_M = 0   # a failed call leaves no EHVI state in the context either
        self._check(self._lib.tpe_ehvi_set(self._h, _ptr(lb), _ptr(iv), lb.shape[0], _ptr(z), z.shape[0], z.shape[1]))
        self._ehvi_M = lb.shape[1]

    def ehvi(self, mean, sd, grad: bool = False):
        """log-EHVI at the rows of ``mean`` and ``sd`` [Q, M], the posterior means and standard deviations of the M
        objectives, against the boxes and samples of ``ehvi_set`` (tpe_ehvi): ``value`` [Q] and with ``grad`` also
        ``(dmean, dsd)`` [Q, M], its gradients.  The values are the same bits with and without ``grad``."""
        m, s = _f64(mean), _f64(sd)
        M = self._ehvi_M
        if m.ndim != 2 or s.shape != m.shape or (M and m.shape[1] != M):
            raise ValueError(f"mean and sd must be [Q, {M}], got shapes {m.shape}, {s.shape}")
        value = np.empty(m.shape[0])
        dmean = np.empty(m.shape) if grad else None
        dsd = np.empty(m.shape) if grad else None
        self._check(self._lib.tpe_ehvi(self._h, _ptr(m), _ptr(s), m.shape[0], _ptr(value), _ptr(dmean), _ptr(dsd)))
        return (value, dmean, dsd) if grad else value

    ACQF_LOGEI, ACQF_LOGEHVI, ACQF_LOGPI = 0, 1, 2   # tpe_acqf_set's kinds

    def acqf_set(self, kind: int, gp_engines, n_obj: int, thresholds, stabilizing_noise: float = 1e-12,
                 lower=None, intervals=None, samples=None) -> None:
        """GPSampler's acquisition function over the conditioned GPs of ``gp_engines`` (tpe_acqf_set): ``ACQF_LOGEI``
        (``n_obj`` = 1, LogEI of the first GP), ``ACQF_LOGEHVI`` (2 <= ``n_obj`` <= 24, log-EHVI of the first
        ``n_obj`` GPs over ``lower`` / ``intervals`` [B, M] and ``samples`` [S, M]) or ``ACQF_LOGPI`` (``n_obj`` = 0);
        the GPs after the objectives' are constraints whose LogPI terms are added.  ``thresholds`` holds one value
        per GP (LogEI's may be -inf).  The engines must stay open while this one evaluates; conditioning one of them
        again invalidates the acquisition."""
        engines = list(gp_engines)
        thr = _f64(thresholds).reshape(-1)
        if thr.shape != (len(engines),):
            raise ValueError(f"one threshold per GP engine: {len(engines)} engines, {thr.size} thresholds")
        handles = (C.c_void_p * max(len(engines), 1))(*[e._h for e in engines])
        lb = iv = z = None
        B = S = 0
        if kind == self.ACQF_LOGEHVI:
            lb, iv, z = _f64(lower), _f64(intervals), _f64(samples)
            if lb.ndim != 2 or iv.shape != lb.shape or z.ndim != 2 or z.shape[1] != lb.shape[1]:
                raise ValueError(f"EHVI inputs must be lower [B, M], intervals [B, M], samples [S, M]; got {lb.shape}, "
                                 f"{iv.shape}, {z.shape}")
            B, S = lb.shape[0], z.shape[0]
        self._acqf_P = 0
        self._check(self._lib.tpe_acqf_set(self._h, int(kind), handles, len(engines), int(n_obj), _ptr(thr),
                                           float(stabilizing_noise), _ptr(lb), _ptr(iv), B, _ptr(z), S))
        self._acqf_P = engines[0]._gp_P
        self._acqf_engines = engines   # kept open with this acquisition

    def acqf_eval(self, X, grad: bool = False):
        """The acquisition function of ``acqf_set`` at the rows of ``X`` [Q, P] (tpe_acqf_eval): ``value`` [Q] and
        with ``grad`` also d value / dx [Q, P], in one device call.  A row's value is the same bits whatever the batch
        and the gradient request."""
        x = _f64(X)
        if x.ndim != 2 or (self._acqf_P and x.shape[1] != self._acqf_P):
            raise ValueError(f"X must be [Q, {self._acqf_P}], got shape {x.shape}")
        value = np.empty(x.shape[0])
        g = np.empty(x.shape) if grad else None
        self._check(self._lib.tpe_acqf_eval(self._h, _ptr(x), x.shape[0], _ptr(value), _ptr(g)))
        return (value, g) if grad else value

    def box_decomposition(self, loss_vals, ref_point) -> tuple[np.ndarray, np.ndarray]:
        """``get_non_dominated_box_bounds(loss_vals, ref_point)`` (optuna/_hypervolume/box_decomposition.py:138-157)
        without its warning: ``(lower, upper)`` [B, M], the reference's bits in its row order (tpe_box_decomposition).
        ``loss_vals`` [n, M] finite, minimised; ``ref_point`` [M] without NaN; 2 <= M <= 24.  B may be 0.  The counts
        of the last call (front size, bounds made and kept by each pass) are in ``last_box_stats``.  Leaves every
        other state of this engine unchanged."""
        v, r = _f64(loss_vals), _f64(ref_point).reshape(-1)
        if v.ndim != 2 or v.shape[1] != r.size:
            raise ValueError(f"loss_vals must be [n, {r.size}] for a reference point of {r.size} objectives, got shape "
                             f"{v.shape}")
        n_boxes = C.c_int64()
        self._check(self._lib.tpe_box_decomposition(self._h, _ptr(v), v.shape[0], v.shape[1], _ptr(r),
                                                    C.byref(n_boxes)))
        lower = np.empty((n_boxes.value, r.size))
        upper = np.empty((n_boxes.value, r.size))
        stats = np.empty(6, dtype=np.int64)
        self._check(self._lib.tpe_get_box_decomposition(self._h, _ptr(lower), _ptr(upper), _ptr(stats)))
        self.last_box_stats = dict(zip(("front", "born1", "bounds1", "front2", "born2", "bounds2"), stats.tolist()))
        return lower, upper

    # -- inspection --------------------------------------------------------------------------------
    def get_split(self) -> tuple[np.ndarray, np.ndarray]:
        below = np.empty(self._info[1], dtype=np.int64)
        above = np.empty(self._info[2], dtype=np.int64)
        self._check(self._lib.tpe_get_split(self._h, _ptr(below), _ptr(above)))
        return below, above

    def get_mixture(self, which: int):
        K = self._info[1 + which] + 1
        w = np.empty(K)
        mu = np.empty((K, self._pc))
        sg = np.empty((K, self._pc))
        self._check(self._lib.tpe_get_mixture(self._h, int(which), _ptr(w), _ptr(mu), _ptr(sg)))
        return w, mu, sg

    def get_mo_weights(self) -> np.ndarray:
        w = np.empty(self._info[0])
        self._check(self._lib.tpe_get_mo_weights(self._h, _ptr(w)))
        return w

    def get_candidates(self):
        ct = self._last_asks * self._C
        s = np.empty((ct, self._pc))
        ll = np.empty(ct)
        lg = np.empty(ct)
        self._check(self._lib.tpe_get_candidates(self._h, _ptr(s), _ptr(ll), _ptr(lg)))
        return s, ll, lg

    def logpdf(self, which: int, x) -> np.ndarray:
        x = _f64(x, (-1, self._pc))
        out = np.empty(x.shape[0])
        self._check(self._lib.tpe_logpdf(self._h, int(which), _ptr(x), x.shape[0], _ptr(out)))
        return out

    def last_timing(self) -> tuple[np.ndarray, int]:
        ms = np.zeros(9, dtype=np.float32)
        n = C.c_int32()
        self._check(self._lib.tpe_last_timing(self._h, _ptr(ms), C.byref(n)))
        return ms, int(n.value)

    def probe_fp64_tflops(self) -> float:
        v = C.c_double()
        self._check(self._lib.tpe_probe_fp64_tflops(self._h, C.byref(v)))
        return float(v.value)

    def last_logpdf_kernel(self) -> str:
        return self._lib.tpe_last_logpdf_kernel(self._h).decode()
