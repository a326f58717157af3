"""Thin Python layer over the C ABI: Engine (handle) and Dataset objects.

Host logic only -- argument marshalling and sklearn-compatible parameter scaling.  All
arithmetic happens inside libcnmf_b200.so on the GPU.
"""
import ctypes

import numpy as np

from . import _lib
from ._lib import (LOSS_FROBENIUS, LOSS_ITAKURA_SAITO, LOSS_KULLBACK_LEIBLER, NmfParams, PRECISION_FP32,
                   PRECISION_F16X2, PRECISION_TF32X3, PRECISION_TF32X3_GENERAL, SOLVER_CD, SOLVER_MU, check, f32c, ptr)

# default: split-operand tensor-core products with fp32-class accuracy -- 2 f16 passes when X is recognised as
# scaled integer counts (what the reference factorizes), 3 tf32 passes otherwise
_DEFAULT_PRECISION = PRECISION_F16X2


def precision_code(p):
    """'fp32' | 'tf32x3' (default; 2-pass products when X is scaled integer counts) | 'f16x2' (like tf32x3, but the
    2-pass products of scaled-integer-count matrices run on f16 MMAs) | 'tf32x3-general' (always 3-pass)."""
    if p in (PRECISION_FP32, PRECISION_TF32X3, PRECISION_TF32X3_GENERAL, PRECISION_F16X2):
        return p
    return {"fp32": PRECISION_FP32, "tf32x3": PRECISION_TF32X3, "tf32x3-general": PRECISION_TF32X3_GENERAL,
            "f16x2": PRECISION_F16X2}[p]


def _params_precision(p):
    return PRECISION_TF32X3 if p in (PRECISION_TF32X3_GENERAL, PRECISION_F16X2) else p


def check_supported(ks=None, init="random", beta_loss="frobenius"):
    """Options the CUDA path does not implement are refused where the user states them (prepare / the CLI), not
    hours later inside factorize: n_components > 32, an init scikit-learn does not know, beta_loss outside
    {frobenius, kullback-leibler, itakura-saito}.  init: 'random' (the reference default, cnmf.py:335; generated on
    the device) and the NNDSVD family ('nndsvd' is the CLI's other choice, cnmf.py:1252; starting factors computed on
    the host by cnmf_b200.nndsvd, then the same batched solve)."""
    from .nndsvd import INITS
    if ks is not None:
        bad = [int(k) for k in np.atleast_1d(ks) if int(k) < 1 or int(k) > _lib.MAX_COMPONENTS]
        if bad:
            raise ValueError("cnmf_b200: n_components must be in [1, %d] on the CUDA path (got %s); the batched "
                             "kernels keep a restart's K x K Gram matrix and its K factor values per item on chip"
                             % (_lib.MAX_COMPONENTS, bad))
    if init is not None and init not in INITS:
        raise ValueError("Invalid init parameter: got %r instead of one of %r" % (init, (None,) + INITS))
    loss_code(beta_loss)


def nndsvd_starts(X, ks, seeds, init):
    """Packed starting factors (W^T rows: sum ks x cells, H rows: sum ks x genes; fp32) of every restart (k, seed) for
    init in {'nndsvd', 'nndsvda', 'nndsvdar', None}: scikit-learn's `_initialize_nmf` as the reference's call reaches it
    (cnmf.py:672), restated in cnmf_b200/nndsvd.py.  One randomized SVD per restart on the host (threads: LAPACK / BLAS
    release the GIL)."""
    import concurrent.futures
    import os
    from .nndsvd import nndsvd_init, resolve_init
    ks = [int(k) for k in ks]
    n, g = X.shape
    offs = np.concatenate([[0], np.cumsum(ks)]).astype(np.int64)
    W0 = np.empty((int(offs[-1]), n), np.float32)
    H0 = np.empty((int(offs[-1]), g), np.float32)

    def one(r):
        which = resolve_init(init, ks[r], n, g)
        if which == "random":
            raise ValueError("init=None resolves to 'random' for n_components > min(shape): use the seeded device generator")
        W, H = nndsvd_init(X, ks[r], int(seeds[r]), which)
        W0[offs[r]:offs[r + 1]] = W.T
        H0[offs[r]:offs[r + 1]] = H

    workers = max(1, min(8, (os.cpu_count() or 1) // 4, len(ks)))
    if workers == 1:
        for r in range(len(ks)):
            one(r)
    else:
        with concurrent.futures.ThreadPoolExecutor(max_workers=workers) as ex:
            list(ex.map(one, range(len(ks))))
    return W0, H0


def make_params(nmf_kwargs, n_samples, n_features, precision, for_refit=False):
    """nmf_kwargs dict of cnmf.py:618-631 -> struct cnmf_nmf_params.

    Regularisation scaling follows sklearn/decomposition/_nmf.py:1249-1260.  Only what the CUDA
    path implements is accepted; anything else raises (no silent fallback)."""
    solver = nmf_kwargs.get("solver", "mu")
    beta = nmf_kwargs.get("beta_loss", "frobenius")
    loss = loss_code(beta)
    if loss != LOSS_FROBENIUS and solver != "mu":      # sklearn _nmf.py:1195-1199
        raise ValueError("Invalid beta_loss parameter: solver %r does not handle beta_loss = %r" % (solver, beta))
    if not for_refit:                                   # a refit (update_H=False) has no initialisation to choose
        check_supported(None, nmf_kwargs.get("init", "random"), beta)
    if solver not in ("mu", "cd"):
        raise ValueError("solver must be 'mu' or 'cd'")
    alpha_W = float(nmf_kwargs.get("alpha_W", 0.0))
    alpha_H = nmf_kwargs.get("alpha_H", 0.0)
    alpha_H = alpha_W if alpha_H == "same" else float(alpha_H)
    l1_ratio = float(nmf_kwargs.get("l1_ratio", 0.0))
    p = NmfParams()
    p.solver = SOLVER_MU if solver == "mu" else SOLVER_CD
    p.precision = _params_precision(precision_code(precision))
    rng = nmf_kwargs.get("rng", "device")
    if rng not in ("device", "host"):
        raise ValueError("rng must be 'device' or 'host'")
    p.reserved = 1 if rng == "host" else 0          # bit 0: draw the random init on the host
    p.max_iter = int(nmf_kwargs.get("max_iter", 1000))
    p.tol = float(nmf_kwargs.get("tol", 1e-4))
    p.l1_reg_W = n_features * alpha_W * l1_ratio
    p.l1_reg_H = n_samples * alpha_H * l1_ratio
    p.l2_reg_W = n_features * alpha_W * (1.0 - l1_ratio)
    p.l2_reg_H = n_samples * alpha_H * (1.0 - l1_ratio)
    p.beta_loss = loss
    return p


def loss_code(beta):
    """'frobenius' | 2 -> tensor-core path; 'kullback-leibler' | 1 and 'itakura-saito' | 0 -> streaming MU kernels
    (sklearn _nmf.py:52-58 `_beta_loss_to_float`).  Other beta values are not implemented on the CUDA path."""
    table = {"frobenius": LOSS_FROBENIUS, 2: LOSS_FROBENIUS, "kullback-leibler": LOSS_KULLBACK_LEIBLER,
             1: LOSS_KULLBACK_LEIBLER, "itakura-saito": LOSS_ITAKURA_SAITO, 0: LOSS_ITAKURA_SAITO}
    try:
        return table[beta]
    except (KeyError, TypeError):
        raise NotImplementedError("cnmf_b200: beta_loss must be 'frobenius' (2), 'kullback-leibler' (1) or "
                                  "'itakura-saito' (0) on the CUDA path (got %r)" % (beta,))


class Engine:
    """One per process and GPU: owns the library handle and its cached device workspace."""

    def __init__(self, device=0):
        self.lib = _lib.load()
        self._h = ctypes.c_void_p()
        check(self.lib.cnmf_create(ctypes.byref(self._h), int(device)))
        self.device = int(device)

    def close(self):
        if self._h:
            self.lib.cnmf_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def launch_count(self):
        return int(self.lib.cnmf_launch_count(self._h))

    def profile(self, on=True):
        """Start (and reset) / stop per-launch CUDA-event timing of the batched GEMM."""
        check(self.lib.cnmf_profile_enable(self._h, 1 if on else 0))

    def profile_get(self, kernel_class=0):
        """(total device ms, launches, algorithmic work) of a kernel class since profile(True):
        0 = batched GEMM (work in FLOPs), 1 = fused update kernels (work in bytes)."""
        ms, n, fl = ctypes.c_double(), ctypes.c_longlong(), ctypes.c_double()
        check(self.lib.cnmf_profile_get_class(self._h, int(kernel_class), ctypes.byref(ms), ctypes.byref(n),
                                              ctypes.byref(fl)))
        return ms.value, int(n.value), fl.value

    def mem_info(self):
        """(free, total, cached) device bytes: cudaMemGetInfo plus what the handle's own pool / workspace holds."""
        v = [ctypes.c_longlong() for _ in range(3)]
        check(self.lib.cnmf_mem_info(self._h, *[ctypes.byref(x) for x in v]))
        return tuple(int(x.value) for x in v)

    def last_timing(self):
        """Host wall-clock phases (ms) of the last factorize: dict(rng, h2d, solve, d2h)."""
        v = [ctypes.c_double() for _ in range(4)]
        check(self.lib.cnmf_last_timing(self._h, *[ctypes.byref(x) for x in v]))
        return dict(zip(("rng_ms", "h2d_ms", "solve_ms", "d2h_ms"), [x.value for x in v]))

    def dataset(self, X, precision=_DEFAULT_PRECISION, stream=None):
        return Dataset(self, X, precision, stream)

    def gemm_abt(self, A, B, precision=PRECISION_TF32X3, splits=1, reps=1):
        """C = A @ B.T through the solver's GEMM kernels (test / micro-benchmark hook)."""
        A, B = f32c(A), f32c(B)
        M, Kd = A.shape
        N = B.shape[0]
        assert B.shape[1] == Kd
        C = np.empty((M, N), np.float32)
        ms = ctypes.c_float(0)
        pc = precision_code(precision)
        pc = PRECISION_TF32X3 if pc == PRECISION_TF32X3_GENERAL else pc      # f16x2: B must hold integers <= 2048
        check(self.lib.cnmf_gemm_abt_host(self._h, pc, ptr(A), ptr(B), M, N, Kd, splits,
                                          ptr(C), reps, ctypes.byref(ms), None))
        return C, float(ms.value)


class Dataset:
    """A cells x genes matrix resident on the GPU (norm_counts.X / tpm.X of the reference)."""

    def __init__(self, engine, X, precision=_DEFAULT_PRECISION, stream=None, _handle=None):
        self.engine = engine
        self.lib = engine.lib
        self.precision = precision_code(precision)
        self._d = ctypes.c_void_p()
        if _handle is not None:
            self._d = _handle
        else:
            if hasattr(X, "toarray"):       # scipy sparse: the CUDA path is dense (DESIGN.md)
                X = X.toarray()
            X = f32c(X)
            n, g = X.shape
            check(self.lib.cnmf_dataset_create(engine._h, ptr(X), n, g, g, 0, self.precision, stream,
                                               ctypes.byref(self._d)))
        n, g = ctypes.c_int(), ctypes.c_int()
        check(self.lib.cnmf_dataset_shape(self._d, ctypes.byref(n), ctypes.byref(g)))
        self.shape = (n.value, g.value)

    def close(self):
        if self._d:
            self.lib.cnmf_dataset_destroy(self._d)
            self._d = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def ld(self):
        """(row stride of packed W^T rows, row stride of packed H rows), both padded to 32 floats."""
        a, b = ctypes.c_int(), ctypes.c_int()
        check(self.lib.cnmf_dataset_ld(self._d, ctypes.byref(a), ctypes.byref(b)))
        return a.value, b.value

    def solve_bytes_per_row(self):
        """Device bytes one packed factor row costs in a batched solve (workspace sizing for restart groups)."""
        return int(self.lib.cnmf_solve_bytes_per_row(self._d))

    def max_rows_per_solve(self, fraction=0.8):
        """How many packed rows (sum of n_components over restarts) fit one batched solve in the device memory that
        is free or already cached by this handle."""
        free, _, cached = self.engine.mem_info()
        return max(1, int(fraction * (free + cached)) // max(1, self.solve_bytes_per_row()))

    def random_init_dev(self, ks, seeds, Wt_ptr, H_ptr):
        """sklearn's random init for every (k, seed), generated on the GPU into packed padded device buffers."""
        ks = np.ascontiguousarray(ks, dtype=np.int32)
        seeds = np.ascontiguousarray(seeds, dtype=np.uint32)
        check(self.lib.cnmf_random_init_dev(self._d, len(ks), ptr(ks), ptr(seeds), ctypes.c_void_p(Wt_ptr),
                                            ctypes.c_void_p(H_ptr), None))

    def factorize_seeds_dev(self, ks, seeds, out_ptr, ld_out, nmf_kwargs):
        """cnmf_factorize (same seeds, same device RNG) with the spectra left on the device: out_ptr is a
        (sum ks) x ld_out fp32 device buffer.  Returns (n_iter, err)."""
        ks = np.ascontiguousarray(ks, dtype=np.int32)
        seeds = np.ascontiguousarray(seeds, dtype=np.uint32)
        R = len(ks)
        if nmf_kwargs.get("init", "random") != "random":
            raise ValueError("factorize_seeds_dev draws the seeded random init on the device; init=%r goes through "
                             "Dataset.factorize(X_host=...)" % (nmf_kwargs.get("init"),))
        p = self.params(nmf_kwargs)
        self._check_loss(p)
        n_iter = np.zeros(R, np.int32)
        err = np.zeros(R, np.float64)
        check(self.lib.cnmf_factorize_seeds_dev(self._d, R, ptr(ks), ptr(seeds), ctypes.byref(p), ctypes.c_void_p(out_ptr),
                                                int(ld_out), ptr(n_iter), ptr(err), None))
        return n_iter, err

    def factorize_dev(self, ks, Wt0_ptr, H0_ptr, out_ptr, nmf_kwargs):
        """Device-resident factorize: raw device pointers (e.g. torch.Tensor.data_ptr()) of the packed,
        padded initial factors and of the output spectra slab.  Returns (n_iter, err)."""
        ks = np.ascontiguousarray(ks, dtype=np.int32)
        R = len(ks)
        p = self.params(nmf_kwargs)
        self._check_loss(p)
        n_iter = np.zeros(R, np.int32)
        err = np.zeros(R, np.float64)
        check(self.lib.cnmf_factorize_dev(self._d, R, ptr(ks), ctypes.c_void_p(Wt0_ptr), ctypes.c_void_p(H0_ptr),
                                          ctypes.byref(p), ctypes.c_void_p(out_ptr), ptr(n_iter), ptr(err), None))
        return n_iter, err

    @property
    def exact(self):
        """True when X was recognised as scaled integer counts (2-pass tensor-core products)."""
        return bool(self.lib.cnmf_dataset_is_exact(self._d))

    @property
    def f16(self):
        """True when the big products run as 2 f16 passes (exact dataset created with precision='f16x2')."""
        return self.lib.cnmf_dataset_is_exact(self._d) == 2

    def min(self):
        m = ctypes.c_float()
        check(self.lib.cnmf_dataset_min(self._d, ctypes.byref(m), None))
        return float(m.value)

    def _check_loss(self, p):
        # sklearn _nmf.py:1675-1680
        if p.beta_loss == LOSS_ITAKURA_SAITO and self.min() == 0:
            raise ValueError("When beta_loss <= 0 and X contains zeros, the solver may diverge. Please add small values "
                             "to X, or use a positive beta_loss.")

    def sums(self):
        s, q = ctypes.c_double(), ctypes.c_double()
        check(self.lib.cnmf_dataset_sums(self._d, ctypes.byref(s), ctypes.byref(q)))
        return s.value, q.value

    def col_stats(self, row_scale=None):
        """Per-column (mean, population variance) in float64; with row_scale: of diag(row_scale) @ X, accumulated
        from the stored values (TPM gene statistics straight from the raw counts, cnmf.py:192-242, 436-445)."""
        g = self.shape[1]
        mean, var = np.empty(g), np.empty(g)
        if row_scale is None:
            check(self.lib.cnmf_dataset_col_stats(self._d, ptr(mean), ptr(var), None))
        else:
            rs = np.ascontiguousarray(row_scale, dtype=np.float64)
            assert rs.shape == (self.shape[0],)
            check(self.lib.cnmf_dataset_scaled_col_stats(self._d, ptr(rs), ptr(mean), ptr(var), None))
        return mean, var

    def row_sums(self):
        """Per-row (cell) totals in float64 (the TPM denominators, cnmf.py:245-251)."""
        out = np.empty(self.shape[0])
        check(self.lib.cnmf_dataset_row_sums(self._d, ptr(out), None))
        return out

    def scale_rows(self, row_scale):
        """New resident dataset diag(row_scale) @ X (TPM from counts without a trip through the host)."""
        rs = f32c(row_scale)
        assert rs.shape == (self.shape[0],)
        out = ctypes.c_void_p()
        check(self.lib.cnmf_dataset_scale_rows(self._d, ptr(rs), None, ctypes.byref(out)))
        return Dataset(self.engine, None, self.precision, _handle=out)

    def from_columns(self, cols, scale):
        cols = np.ascontiguousarray(cols, dtype=np.int32)
        scale = f32c(scale)
        out = ctypes.c_void_p()
        check(self.lib.cnmf_dataset_from_columns(self._d, ptr(cols), ptr(scale), len(cols), None, ctypes.byref(out)))
        return Dataset(self.engine, None, self.precision, _handle=out)

    def params(self, nmf_kwargs):
        return make_params(nmf_kwargs, self.shape[0], self.shape[1], self.precision)

    def factorize(self, ks, seeds, nmf_kwargs, return_usages=False, W0=None, H0=None, X_host=None):
        """All restarts (ks[r], seeds[r]) at once.  Returns (spectra_list, usages_list|None, n_iter, err).
        W0 / H0: packed starting factors (sum ks x cells, sum ks x genes) instead of the seeded random init; X_host: the
        host matrix, needed only when nmf_kwargs['init'] is one of the NNDSVD family (starts computed from it)."""
        ks = np.ascontiguousarray(ks, dtype=np.int32)
        R = len(ks)
        SK = int(ks.sum())
        n, g = self.shape
        p = self.params(nmf_kwargs)
        self._check_loss(p)
        spectra = np.empty((SK, g), np.float32)
        usages = np.empty((SK, n), np.float32) if return_usages else None
        n_iter = np.zeros(R, np.int32)
        err = np.zeros(R, np.float64)
        init = nmf_kwargs.get("init", "random")
        if W0 is None and init != "random":
            # NNDSVD family (cnmf.py:1252 / SK _nmf.py:309-369): starting factors from cnmf_b200.nndsvd on the host, one
            # randomized SVD per restart (the seed enters through its test matrix), then the ordinary batched solve
            if X_host is None:
                raise ValueError("init=%r: pass X_host (the matrix the dataset was created from) or W0 / H0; the "
                                 "device generator only covers init='random'" % (init,))
            W0, H0 = nndsvd_starts(X_host, ks, seeds, init)
        if W0 is None:
            seeds = np.ascontiguousarray(seeds, dtype=np.uint32)
            check(self.lib.cnmf_factorize(self._d, R, ptr(ks), ptr(seeds), ctypes.byref(p), ptr(spectra), ptr(usages),
                                          ptr(n_iter), ptr(err), None))
        else:
            W0, H0 = f32c(W0), f32c(H0)      # packed (SK x n), (SK x g)
            assert W0.shape == (SK, n) and H0.shape == (SK, g)
            check(self.lib.cnmf_factorize_init(self._d, R, ptr(ks), ptr(W0), ptr(H0), ctypes.byref(p), ptr(spectra),
                                               ptr(usages), ptr(n_iter), ptr(err), None))
        offs = np.concatenate([[0], np.cumsum(ks)])
        sp = [spectra[offs[r]:offs[r + 1]] for r in range(R)]
        us = [usages[offs[r]:offs[r + 1]].T for r in range(R)] if return_usages else None
        return sp, us, n_iter, err

    def refit(self, fixed, nmf_kwargs, transposed=False):
        """NMF with `fixed` held constant (update_H=False).  transposed=False: fixed = H (k x genes),
        returns W (cells x k).  transposed=True: fixed = W^T (k x cells), returns H^T (genes x k)."""
        fixed = f32c(fixed)
        k = fixed.shape[0]
        n, g = self.shape
        n_r, n_c = (g, n) if transposed else (n, g)
        assert fixed.shape[1] == n_c
        p = make_params(nmf_kwargs, n_r, n_c, self.precision, for_refit=True)
        self._check_loss(p)
        out = np.empty((n_r, k), np.float32)
        it = ctypes.c_int32(0)
        err = ctypes.c_double(0)
        check(self.lib.cnmf_refit(self._d, 1 if transposed else 0, k, ptr(fixed), ctypes.byref(p), ptr(out),
                                  ctypes.byref(it), ctypes.byref(err), None))
        return out, int(it.value), float(err.value)

    def project_rows(self, Ut):
        """Ut (k x cells) @ X -> (k x genes)."""
        Ut = f32c(Ut)
        k = Ut.shape[0]
        assert Ut.shape[1] == self.shape[0]
        out = np.empty((k, self.shape[1]), np.float32)
        check(self.lib.cnmf_project_rows(self._d, k, ptr(Ut), ptr(out), None))
        return out
