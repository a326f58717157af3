"""Thin Python layer over the C ABI: Engine (handle) and Dataset objects.

Host logic only -- argument marshalling and sklearn-compatible parameter scaling.  All
arithmetic happens inside libcnmf_b200.so on the GPU.
"""
import ctypes

import numpy as np

from . import _lib
from ._lib import (LOSS_FROBENIUS, LOSS_ITAKURA_SAITO, LOSS_KULLBACK_LEIBLER, NmfParams, PRECISION_FP32,
                   PRECISION_F16X2, PRECISION_FP64, PRECISION_TF32X3, PRECISION_TF32X3_GENERAL, SOLVER_CD, SOLVER_MU,
                   check, f32c, f64c, ptr)

# default: split-operand tensor-core products with fp32-class accuracy -- 2 f16 passes when X is recognised as
# scaled integer counts (what the reference factorizes), 3 tf32 passes otherwise
_DEFAULT_PRECISION = PRECISION_F16X2


def precision_code(p):
    """'fp32' | 'tf32x3' (default; 2-pass products when X is scaled integer counts) | 'f16x2' (like tf32x3, but the
    2-pass products of scaled-integer-count matrices run on f16 MMAs) | 'tf32x3-general' (always 3-pass) | 'fp64'
    (X, factors and products in float64 on the fp64 tensor cores: the reference's own float64 numbers)."""
    if p in (PRECISION_FP32, PRECISION_TF32X3, PRECISION_TF32X3_GENERAL, PRECISION_F16X2, PRECISION_FP64):
        return p
    return {"fp32": PRECISION_FP32, "tf32x3": PRECISION_TF32X3, "tf32x3-general": PRECISION_TF32X3_GENERAL,
            "f16x2": PRECISION_F16X2, "fp64": PRECISION_FP64}[p]


def is_fp64(precision):
    return precision is not None and precision_code(precision) == PRECISION_FP64


def check_fp64_supported(precision, beta_loss="frobenius", rng="device"):
    """What precision='fp64' does not cover is refused where the user states it: beta_loss other than frobenius, and the
    host random generator (fp64 starts come from the device generator or the NNDSVD family)."""
    if not is_fp64(precision):
        return
    if loss_code(beta_loss) != LOSS_FROBENIUS:
        raise NotImplementedError("cnmf_b200: precision='fp64' supports beta_loss='frobenius' only (got %r)"
                                  % (beta_loss,))
    if rng == "host":
        raise NotImplementedError("cnmf_b200: precision='fp64' draws its random starts on the device; rng='host' "
                                  "serves the float precisions only")


def _params_precision(p):
    return PRECISION_TF32X3 if p in (PRECISION_TF32X3_GENERAL, PRECISION_F16X2) else p


def check_supported(ks=None, init="random", beta_loss="frobenius"):
    """Options the CUDA path does not implement are refused where the user states them (prepare / the CLI), not
    hours later inside factorize: n_components > 32, an init scikit-learn does not know, beta_loss outside
    {frobenius, kullback-leibler, itakura-saito}.  init: 'random' (the reference default, cnmf.py:335) and the NNDSVD
    family ('nndsvd' is the CLI's other choice, cnmf.py:1252), both generated on the device before the same batched
    solve (cnmf_b200.nndsvd restates the NNDSVD family on the host)."""
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


def init_code(init, ks, n_samples, n_features):
    """CNMF_INIT_* of one call: init (None resolved as scikit-learn does, per n_components) must name the same
    initialisation for every restart."""
    from .nndsvd import resolve_init
    which = {resolve_init(init, int(k), n_samples, n_features) for k in np.atleast_1d(ks)}
    if len(which) > 1:
        raise ValueError("init=%r resolves to %s for different n_components of one call; split the call by K"
                         % (init, sorted(which)))
    return _lib.INIT_CODES[which.pop()]


def nndsvd_starts(X, ks, seeds, init, dtype=np.float32):
    """Packed starting factors (W^T rows: sum ks x cells, H rows: sum ks x genes; dtype) of every restart (k, seed) for
    init in {'nndsvd', 'nndsvda', 'nndsvdar', None}: scikit-learn's `_initialize_nmf` as the reference's call reaches it
    (cnmf.py:672), restated in cnmf_b200/nndsvd.py.  One randomized SVD per restart on the host (threads: LAPACK / BLAS
    release the GIL).  Dataset.nndsvd_init_dev computes the same starts on the GPU."""
    import concurrent.futures
    import os
    from .nndsvd import nndsvd_init, resolve_init
    ks = [int(k) for k in ks]
    n, g = X.shape
    offs = np.concatenate([[0], np.cumsum(ks)]).astype(np.int64)
    W0 = np.empty((int(offs[-1]), n), dtype)
    H0 = np.empty((int(offs[-1]), g), dtype)

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
    check_fp64_supported(precision, beta, rng)
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


def _csr_arrays(C, dtype):
    """(row_ptr int64, col_idx int32, values as dtype) of the scipy CSR matrix C in canonical form: column indices sorted
    within each row, duplicates summed in C's own dtype (C itself is left as it is)."""
    if not C.has_canonical_format:
        C = C.copy()
        C.sum_duplicates()
    return (np.ascontiguousarray(C.indptr, dtype=np.int64), np.ascontiguousarray(C.indices, dtype=np.int32),
            np.ascontiguousarray(C.data, dtype=dtype))


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
        0 = batched GEMM (work in FLOPs), 1 = fused update kernels (work in bytes), 2 = sparse-dataset products
        (work in bytes), 3 = fp64 GEMM of the NNDSVD starts (work in FLOPs), 4 = fp64 GEMM of the float64 solver
        (work in FLOPs), 5 = fp64 GEMMs of the Harmony ridge correction (work in FLOPs)."""
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

    def nndsvd_chunk_limit(self, max_restarts):
        """Test hook: at most max_restarts restarts per chunk of the device NNDSVD starts (0 = sized from free memory)."""
        check(self.lib.cnmf_nndsvd_chunk_limit(self._h, int(max_restarts)))

    def dataset(self, X, precision=_DEFAULT_PRECISION, stream=None):
        return Dataset(self, X, precision, stream)

    def sparse_dataset(self, X, precision=_DEFAULT_PRECISION, stream=None):
        """X (any scipy sparse matrix or an ndarray) resident on the GPU as canonical float32 CSC, 8 bytes per stored
        entry; no dense copy is made on the host or the device.  Serves the consensus step's TPM uses: sums, col_stats,
        project_rows, from_columns (returns a dense dataset) and refit(transposed=True) with the Frobenius loss; and
        prepare's uses of raw counts: tpm_stats, col_stats, from_columns.  Everything else raises CnmfError.
        precision='fp64' has no sparse form.  A CSR matrix is transposed on the device (only its stored entries are
        copied); any other input is converted to CSC on the host."""
        if is_fp64(precision):
            raise NotImplementedError("cnmf_b200: precision='fp64' needs a dense dataset; sparse (CSC) datasets hold "
                                      "float32 values")
        import scipy.sparse as sp
        out = ctypes.c_void_p()
        if sp.issparse(X) and X.format == "csr":
            n, g = X.shape
            row_ptr, col_idx, vals = _csr_arrays(sp.csr_matrix(X, dtype=np.float32), np.float32)
            check(self.lib.cnmf_dataset_create_csr(self._h, n, g, int(row_ptr[-1]), ptr(row_ptr), ptr(col_idx),
                                                   ptr(vals), precision_code(precision), stream, ctypes.byref(out)))
            return Dataset(self, None, precision, _handle=out, sparse=True)
        C = sp.csc_matrix(X, dtype=np.float32)
        if not C.has_canonical_format:          # sorted row indices, no duplicates: the library does not sort
            C = C.copy()
            C.sum_duplicates()
        n, g = C.shape
        col_ptr = np.ascontiguousarray(C.indptr, dtype=np.int64)
        row_idx = np.ascontiguousarray(C.indices, dtype=np.int32)
        vals = np.ascontiguousarray(C.data, dtype=np.float32)
        check(self.lib.cnmf_dataset_create_csc(self._h, n, g, int(col_ptr[-1]), ptr(col_ptr), ptr(row_idx), ptr(vals),
                                               precision_code(precision), stream, ctypes.byref(out)))
        return Dataset(self, None, precision, _handle=out, sparse=True)

    def dataset_from_device(self, X_ptr, n_rows, n_cols, ld, precision=_DEFAULT_PRECISION, stream=None):
        """Dataset of a float32 device matrix (n_rows x n_cols, row stride ld elements, e.g. torch.Tensor.data_ptr())."""
        out = ctypes.c_void_p()
        check(self.lib.cnmf_dataset_create(self._h, ctypes.c_void_p(X_ptr), int(n_rows), int(n_cols), int(ld), 1,
                                           precision_code(precision), stream, ctypes.byref(out)))
        return Dataset(self, None, precision, _handle=out)

    def dense_dataset_bytes(self, n_rows, n_cols, precision=_DEFAULT_PRECISION):
        """Worst-case device bytes dataset() of an n_rows x n_cols matrix needs while it is built."""
        peak = ctypes.c_longlong()
        check(self.lib.cnmf_dataset_dense_bytes(int(n_rows), int(n_cols), precision_code(precision), ctypes.byref(peak)))
        return int(peak.value)

    def gemm_abt(self, A, B, precision=PRECISION_TF32X3, splits=1, reps=1, b_exact=False, k_scale=None,
                 out_col_scale=None, tile_n=0):
        """C = A @ B.T through the solver's GEMM kernels (test / micro-benchmark hook).  The exact-count forms:
        b_exact (tf32x3; implied by f16x2) takes B as exact tf32 values, and then C = A diag(k_scale) B^T
        diag(out_col_scale) with the scales applied where the solver applies a dataset's (either may be None).
        tile_n: columns per output tile, 0 = the launcher's choice by shape; 128, or 168 / 192 in the exact forms,
        forces that width."""
        A, B = f32c(A), f32c(B)
        M, Kd = A.shape
        N = B.shape[0]
        assert B.shape[1] == Kd
        ks = None if k_scale is None else f32c(k_scale)
        cs = None if out_col_scale is None else f32c(out_col_scale)
        assert ks is None or ks.shape == (Kd,)
        assert cs is None or cs.shape == (N,)
        C = np.empty((M, N), np.float32)
        ms = ctypes.c_float(0)
        pc = precision_code(precision)
        pc = PRECISION_TF32X3 if pc == PRECISION_TF32X3_GENERAL else pc      # f16x2: B must hold integers <= 2048
        check(self.lib.cnmf_gemm_abt_host(self._h, pc, ptr(A), ptr(B), M, N, Kd, splits, 1 if b_exact else 0,
                                          ptr(ks), ptr(cs), int(tile_n), ptr(C), reps, ctypes.byref(ms), None))
        return C, float(ms.value)

    def update_step(self, ks, rids, done, n, F, num, gram_in, solver="mu", pieces=None, gram=None, want_scalar=False,
                    cpb_tiles=1, l1=0.0, l2=0.0, piece_scale=None, pieces_hi=None, pieces_lo=None, tile_scale=None,
                    gram_out=None, scal_out=None):
        """Test hook: one launch of the solver's update kernel (solver 'mu' / 'cd') or, with solver=None, the
        stand-alone Gram / <NUM, F> / piece launches that start a solve, on packed host data (slot s holds restart
        rids[s] with ks[s] components; F is (sum ks) x ld with ld = ceil(n / 32) * 32, num nsplit x (sum ks) x ld,
        gram_in n_rids x 32 x 32 float64).  pieces: None | 'tf32' | 'f16'; gram: None | 'fused' | 'standalone'.
        The optional in/out arrays (pieces, tile scales, Gram, scalar) are uploaded as given, so a caller can pre-fill
        them with a sentinel; missing ones start as zeros.  Returns dict(F, hi, lo, tile_scale, gram, scal)."""
        ks = np.ascontiguousarray(ks, np.int32)
        rids = np.ascontiguousarray(rids, np.int32)
        done = np.ascontiguousarray(done, np.int32)
        F = f32c(F).copy()
        SK, ld = F.shape
        assert SK == int(ks.sum()) and ld == -(-int(n) // 32) * 32
        num = f32c(num).reshape(-1, SK, ld) if num is not None else None
        gram_in = np.ascontiguousarray(gram_in, np.float64)
        n_rids = len(done)
        assert gram_in.shape == (n_rids, 32, 32)
        pmode = {None: _lib.UNIT_PIECES_NONE, "tf32": _lib.UNIT_PIECES_TF32, "f16": _lib.UNIT_PIECES_F16}[pieces]
        gmode = {None: _lib.UNIT_GRAM_NONE, "fused": _lib.UNIT_GRAM_FUSED, "standalone": _lib.UNIT_GRAM_STANDALONE}[gram]
        smode = {None: _lib.UNIT_SOLVER_NONE, "mu": SOLVER_MU, "cd": SOLVER_CD}[solver]
        pdt = np.float16 if pieces == "f16" else np.float32
        hi = lo = ts = None
        if pieces is not None:
            hi = np.zeros((SK, ld), pdt) if pieces_hi is None else np.ascontiguousarray(pieces_hi, pdt).copy()
            lo = np.zeros((SK, ld), pdt) if pieces_lo is None else np.ascontiguousarray(pieces_lo, pdt).copy()
        if pieces == "f16":
            nt = (ld + 511) // 512
            ts = np.zeros((SK, nt), np.float32) if tile_scale is None else f32c(tile_scale).copy()
        g_out = np.zeros((n_rids, 32, 32)) if gram_out is None else np.ascontiguousarray(gram_out, np.float64).copy()
        s_out = np.zeros(n_rids) if scal_out is None else np.ascontiguousarray(scal_out, np.float64).copy()
        ps = None if piece_scale is None else f32c(piece_scale)
        assert ps is None or ps.shape == (ld,)
        a = _lib.UpdateStepArgs()
        a.n_slots, a.n_rids, a.n, a.cpb_tiles = len(ks), n_rids, int(n), int(cpb_tiles)
        a.ks, a.rids, a.done = ptr(ks), ptr(rids), ptr(done)
        a.solver, a.pieces, a.gram, a.want_scalar = smode, pmode, gmode, 1 if want_scalar else 0
        a.nsplit = 1 if num is None else num.shape[0]
        a.l1, a.l2 = float(l1), float(l2)
        a.F, a.num, a.gram_in, a.piece_scale = ptr(F), ptr(num), ptr(gram_in), ptr(ps)
        a.pieces_hi, a.pieces_lo, a.tile_scale = ptr(hi), ptr(lo), ptr(ts)
        a.gram_out, a.scal_out = ptr(g_out), ptr(s_out)
        check(self.lib.cnmf_update_step_host(self._h, ctypes.byref(a), None))
        return dict(F=F, hi=hi, lo=lo, tile_scale=ts, gram=g_out, scal=s_out)

    def beta_step(self, ks, rids, done, side, loss, D, F_own, F_other, n_items, n_contract, op="update", l1=0.0, l2=0.0,
                  last=None, totals=None):
        """Test hook: one launch of the KL / IS solver's update kernel (op 'update', loss 'kullback-leibler' /
        'itakura-saito') or one divergence evaluation (op 'divergence', those losses or 'frobenius'), on packed host data
        (slot s holds restart rids[s] with ks[s] components; done has one entry per rid).  side 'W' or 'H' names the
        half whose flags the solver would use (only H maps a zero KL sum to 1; W clips only for IS).  D is n_contract x
        ld_items with the item index contiguous, F_own (sum ks) x ld_items, F_other (sum ks) x ld_contract, ld_* =
        ceil(n / 32) * 32; their padding is passed as given.  last (n_rids) and totals (n_rids x 2) are uploaded as given,
        so a caller can pre-fill them with a sentinel; missing ones start as zeros.  Returns dict(F, oth_sum, last,
        totals): the updated F_own and, for KL updates, the fp64 row sums of F_other; for divergences the statistic
        sqrt(2 max(res, 0)) (||X - WH||_F for frobenius) and the fp64 (sum of terms, sum of x over x > eps) per rid."""
        ks = np.ascontiguousarray(ks, np.int32)
        rids = np.ascontiguousarray(rids, np.int32)
        done = np.ascontiguousarray(done, np.int32)
        SK, n_rids = int(ks.sum()), len(done)
        ld_i, ld_k = -(-int(n_items) // 32) * 32, -(-int(n_contract) // 32) * 32
        D = f32c(D)
        F = f32c(F_own).copy()
        Fo = f32c(F_other)
        assert D.shape == (n_contract, ld_i) and F.shape == (SK, ld_i) and Fo.shape == (SK, ld_k)
        lcode = {"kullback-leibler": LOSS_KULLBACK_LEIBLER, "itakura-saito": LOSS_ITAKURA_SAITO,
                 "frobenius": LOSS_FROBENIUS}[loss]
        oth = np.zeros(SK)
        lo = np.zeros(n_rids) if last is None else np.ascontiguousarray(last, np.float64).copy()
        tt = np.zeros((n_rids, 2)) if totals is None else np.ascontiguousarray(totals, np.float64).copy()
        assert lo.shape == (n_rids,) and tt.shape == (n_rids, 2)
        a = _lib.BetaStepArgs()
        a.n_slots, a.n_rids = len(ks), n_rids
        a.ks, a.rids, a.done = ptr(ks), ptr(rids), ptr(done)
        a.op = {"update": _lib.UNIT_BETA_UPDATE, "divergence": _lib.UNIT_BETA_DIVERGENCE}[op]
        a.side = {"W": _lib.UNIT_SIDE_W, "H": _lib.UNIT_SIDE_H}[side]
        a.loss, a.n_items, a.n_contract = lcode, int(n_items), int(n_contract)
        a.l1, a.l2 = float(l1), float(l2)
        a.D, a.F_own, a.F_other = ptr(D), ptr(F), ptr(Fo)
        a.oth_sum, a.last, a.totals = ptr(oth), ptr(lo), ptr(tt)
        check(self.lib.cnmf_beta_step_host(self._h, ctypes.byref(a), None))
        return dict(F=F, oth_sum=oth, last=lo, totals=tt)

    def update_step_f64(self, ks, rids, done, n, F, op="update", num=None, gram_in=None, solver="mu", want_scalar=False,
                        l1=0.0, l2=0.0, gram_out=None, scal_out=None):
        """Test hook: one launch of the float64 solver on packed fp64 host data (slot s holds restart rids[s] with
        ks[s] components; F and num are (sum ks) x ld with ld = ceil(n / 32) * 32, gram_in n_rids x 32 x 32).  op
        'update' (solver 'mu' / 'cd'; with want_scalar also MU <NUM, F_new> / CD sum |projected gradient|), 'gram' (the
        Gram of F) or 'cross' (<NUM, F>).  gram_out and scal_out are uploaded as given, so a caller can pre-fill them
        with a sentinel; missing ones start as zeros.  Returns dict(F, gram, scal)."""
        ks = np.ascontiguousarray(ks, np.int32)
        rids = np.ascontiguousarray(rids, np.int32)
        done = np.ascontiguousarray(done, np.int32)
        F = f64c(F).copy()
        SK, ld = F.shape
        assert SK == int(ks.sum()) and ld == -(-int(n) // 32) * 32
        num = None if num is None else f64c(num)
        assert num is None or num.shape == (SK, ld)
        n_rids = len(done)
        gin = None if gram_in is None else f64c(gram_in)
        assert gin is None or gin.shape == (n_rids, 32, 32)
        g_out = np.zeros((n_rids, 32, 32)) if gram_out is None else f64c(gram_out).copy()
        s_out = np.zeros(n_rids) if scal_out is None else f64c(scal_out).copy()
        a = _lib.UpdateStepF64Args()
        a.n_slots, a.n_rids, a.n = len(ks), n_rids, int(n)
        a.ks, a.rids, a.done = ptr(ks), ptr(rids), ptr(done)
        a.op = {"update": _lib.UNIT_F64_UPDATE, "gram": _lib.UNIT_F64_GRAM, "cross": _lib.UNIT_F64_CROSS}[op]
        a.solver = {"mu": SOLVER_MU, "cd": SOLVER_CD}[solver]
        a.want_scalar = 1 if want_scalar else 0
        a.l1, a.l2 = float(l1), float(l2)
        a.F, a.num, a.gram_in, a.gram_out, a.scal_out = ptr(F), ptr(num), ptr(gin), ptr(g_out), ptr(s_out)
        check(self.lib.cnmf_update_step_f64_host(self._h, ctypes.byref(a), None))
        return dict(F=F, gram=g_out, scal=s_out)

    def conv_check(self, ks, rids, solver, it, tol, max_iter, done, n_iter, err0, prev, last, normX2=0.0, cross=None,
                   gramA=None, gramB=None, violA=None, violB=None):
        """Test hook: one launch of the shared convergence kernel (solver 'mu': mu_check_kernel, 'cd': cd_check_kernel)
        on host state, with it / tol / max_iter as the solvers pass them.  Per-restart arrays have one entry per rid
        (gramA / gramB n_rids x 32 x 32); the state (done, n_iter, err0, prev, last) is uploaded as given.  Returns
        dict(done, n_iter, err0, prev, last) after the launch."""
        ks = np.ascontiguousarray(ks, np.int32)
        rids = np.ascontiguousarray(rids, np.int32)
        st = dict(done=np.array(done, np.int32), n_iter=np.array(n_iter, np.int32), err0=np.array(err0, np.float64),
                  prev=np.array(prev, np.float64), last=np.array(last, np.float64))
        n_rids = len(st["done"])
        assert all(len(v) == n_rids for v in st.values())
        opt = {k: (None if v is None else f64c(v)) for k, v in
               dict(cross=cross, gramA=gramA, gramB=gramB, violA=violA, violB=violB).items()}
        a = _lib.ConvCheckArgs()
        a.n_slots, a.n_rids = len(ks), n_rids
        a.ks, a.rids = ptr(ks), ptr(rids)
        a.solver = {"mu": SOLVER_MU, "cd": SOLVER_CD}[solver]
        a.it, a.max_iter, a.tol, a.normX2 = int(it), int(max_iter), float(tol), float(normX2)
        for k, v in opt.items():
            setattr(a, k, ptr(v))
        for k, v in st.items():
            setattr(a, k, ptr(v))
        check(self.lib.cnmf_conv_check_host(self._h, ctypes.byref(a), None))
        return st


class Dataset:
    """A cells x genes matrix resident on the GPU (norm_counts.X / tpm.X of the reference).  precision='fp64' keeps X
    in float64 and runs everything in float64: factorize / refit / project_rows then take and return float64 arrays."""

    def __init__(self, engine, X, precision=_DEFAULT_PRECISION, stream=None, _handle=None, sparse=False):
        self.engine = engine
        self.lib = engine.lib
        self.precision = precision_code(precision)
        self.fp64 = self.precision == PRECISION_FP64
        self.sparse = sparse        # CSC-resident (Engine.sparse_dataset)
        self._d = ctypes.c_void_p()
        if _handle is not None:
            self._d = _handle
        elif hasattr(X, "toarray"):
            # scipy sparse: the stored entries go to the device and are scattered into the dense dataset there -- the
            # same dataset X.toarray() would give, without a cells x genes array on the host
            import scipy.sparse as sp
            n, g = X.shape
            row_ptr, col_idx, vals = _csr_arrays(sp.csr_matrix(X), np.float64 if self.fp64 else np.float32)
            nnz = int(row_ptr[-1])
            if self.fp64:
                check(self.lib.cnmf_dataset_create_from_csr_f64(engine._h, n, g, nnz, ptr(row_ptr), ptr(col_idx),
                                                                ptr(vals), stream, ctypes.byref(self._d)))
            else:
                check(self.lib.cnmf_dataset_create_from_csr(engine._h, n, g, nnz, ptr(row_ptr), ptr(col_idx), ptr(vals),
                                                            self.precision, stream, ctypes.byref(self._d)))
        else:
            if self.fp64:
                X = f64c(X)
                n, g = X.shape
                check(self.lib.cnmf_dataset_create_f64(engine._h, ptr(X), n, g, g, 0, stream, ctypes.byref(self._d)))
            else:
                X = f32c(X)
                n, g = X.shape
                check(self.lib.cnmf_dataset_create(engine._h, ptr(X), n, g, g, 0, self.precision, stream,
                                                   ctypes.byref(self._d)))
        n, g = ctypes.c_int(), ctypes.c_int()
        check(self.lib.cnmf_dataset_shape(self._d, ctypes.byref(n), ctypes.byref(g)))
        self.shape = (n.value, g.value)

    def close(self):
        # cnmf_dataset_destroy hands the dataset's buffers back to its handle's pool, so it must not run once the
        # handle is destroyed: it would write to freed host memory.  That happens after an explicit Engine.close, and
        # when the garbage collector finalizes an Engine before a Dataset of the same reference cycle (a failed
        # test's traceback holds both); the dataset's device memory then stays allocated until the process exits
        if self._d and self.engine._h:
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

    def nndsvd_init_dev(self, ks, seeds, init, Wt_ptr, H_ptr):
        """scikit-learn's NNDSVD starts (init 'nndsvd' | 'nndsvda' | 'nndsvdar' | None, resolved per n_components as
        scikit-learn does) of every (k, seed), computed on the GPU in float64 into packed padded device buffers laid
        out as for random_init_dev."""
        ks = np.ascontiguousarray(ks, dtype=np.int32)
        seeds = np.ascontiguousarray(seeds, dtype=np.uint32)
        code = init_code(init, ks, *self.shape)
        if code == _lib.INIT_RANDOM:
            raise ValueError("nndsvd_init_dev: init=%r is the random init (random_init_dev)" % (init,))
        check(self.lib.cnmf_nndsvd_init_dev(self._d, len(ks), ptr(ks), ptr(seeds), code, ctypes.c_void_p(Wt_ptr),
                                            ctypes.c_void_p(H_ptr), None))

    def nndsvd_gemm(self, A, to_genes):
        """The fp64 GEMM hook, for both element types of X (the NNDSVD starts on an fp32 X; the float64 solver's two
        products and NNDSVD starts on a float64 X): A (M x genes) @ X.T, or with to_genes A (M x cells) @ X, in float64.
        Sparse datasets are refused."""
        A = np.ascontiguousarray(A, dtype=np.float64)
        n, g = self.shape
        assert A.shape[1] == (n if to_genes else g)
        C = np.empty((A.shape[0], g if to_genes else n))
        check(self.lib.cnmf_nndsvd_gemm_host(self._d, 1 if to_genes else 0, A.shape[0], ptr(A), ptr(C), None))
        return C

    def _init_params(self, ks, nmf_kwargs):
        """params with the initialisation of the call in bits 1-2 of `reserved`"""
        p = self.params(nmf_kwargs)
        p.reserved |= init_code(nmf_kwargs.get("init", "random"), ks, *self.shape) << 1
        return p

    def factorize_seeds_dev(self, ks, seeds, out_ptr, ld_out, nmf_kwargs):
        """cnmf_factorize (same seeds, same device starts: random or NNDSVD) with the spectra left on the device:
        out_ptr is a (sum ks) x ld_out fp32 device buffer.  Returns (n_iter, err)."""
        ks = np.ascontiguousarray(ks, dtype=np.int32)
        seeds = np.ascontiguousarray(seeds, dtype=np.uint32)
        R = len(ks)
        p = self._init_params(ks, nmf_kwargs)
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

    @property
    def form(self):
        """Operand form decided at creation: 'fp32', 'tf32', 'tf32_exact', 'f16_exact' or 'fp64' (sparse datasets: the
        form their detection chose)."""
        f = self.lib.cnmf_dataset_form(self._d)
        if f < 0:
            check(f)
        return _lib.FORM_NAMES[f]

    def operand(self, name):
        """Test hook: copy of one resident array, padding included (None when the dataset does not hold it):
        X, X_hi, X_lo (n_rows x ld_cols float32), Xt, Xt_hi, Xt_lo (n_cols x ld_rows float32), X_h16 / Xt_h16 (the
        same shapes in float16), row_scale (ld_rows), col_scale (ld_cols); on sparse datasets csc_col_ptr (n_cols + 1,
        int64), csc_row_idx (nnz, int32), csc_values (nnz)."""
        ld_r, ld_c = self.ld()
        n, g = self.shape
        if name == "csc_col_ptr":
            shape, dtype = (g + 1,), np.int64
        elif name in ("csc_row_idx", "csc_values"):
            col_ptr = self.operand("csc_col_ptr")
            if col_ptr is None:
                return None
            shape, dtype = (int(col_ptr[-1]),), np.int32 if name == "csc_row_idx" else np.float32
        else:
            shape = {"X": (n, ld_c), "X_hi": (n, ld_c), "X_lo": (n, ld_c), "X_h16": (n, ld_c),
                     "Xt": (g, ld_r), "Xt_hi": (g, ld_r), "Xt_lo": (g, ld_r), "Xt_h16": (g, ld_r),
                     "row_scale": (ld_r,), "col_scale": (ld_c,)}[name]
            dtype = np.float16 if name.endswith("h16") else np.float32
        out = np.empty(shape, dtype)
        rc = self.lib.cnmf_dataset_operand_host(self._d, _lib.OPERANDS[name], ptr(out), out.nbytes)
        if rc == -3:
            return None
        check(rc)
        return out

    def gemm(self, F, side, transposed=False):
        """Test hook: one of the solver's two products on this dataset's view, through the solver's own launch.
        side 0: F (SK x n_c of the view) @ B_rows^T; side 1: F (SK x n_r of the view) @ B_cols^T (untransposed:
        n_r = cells, n_c = genes).  Returns the raw split-K slices, splits x SK x n_out (their sum is the product).
        Sparse datasets run the transposed refit's product only (transposed, side 0, SK <= 32; one slice)."""
        F = f32c(F)
        n_r, n_c = self.shape[::-1] if transposed else self.shape
        assert F.ndim == 2 and F.shape[1] == (n_c if side == 0 else n_r)
        splits = ctypes.c_int()
        check(self.lib.cnmf_dataset_gemm_host(self._d, int(transposed), int(side), F.shape[0], None, None,
                                              ctypes.byref(splits)))
        out = np.empty((splits.value, F.shape[0], n_r if side == 0 else n_c), np.float32)
        check(self.lib.cnmf_dataset_gemm_host(self._d, int(transposed), int(side), F.shape[0], ptr(F), ptr(out),
                                              ctypes.byref(splits)))
        return out

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

    def tpm_stats(self, target_sum=1e6):
        """Sparse (CSC) counts only: (cell totals, mean, population variance) in float64, the statistics being those of
        the TPM matrix diag(target_sum / total) @ X (a cell without counts stays at zero), computed on the device
        without forming it (cnmf.py:245-251, 436-445).  A dense dataset has row_sums() and col_stats(row_scale=...)."""
        n, g = self.shape
        totals, mean, var = np.empty(n), np.empty(g), np.empty(g)
        check(self.lib.cnmf_dataset_tpm_stats(self._d, float(target_sum), ptr(totals), ptr(mean), ptr(var), None))
        return totals, mean, var

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

    def from_columns_div(self, cols, divisor):
        """float64 datasets: new float64 dataset X[:, cols] / divisor, each entry one IEEE division (bit for bit what
        numpy gives for X[:, cols] / divisor on the host)."""
        cols = np.ascontiguousarray(cols, dtype=np.int32)
        div = f64c(divisor)
        assert div.shape == cols.shape
        out = ctypes.c_void_p()
        check(self.lib.cnmf_dataset_from_columns_f64(self._d, ptr(cols), ptr(div), len(cols), None, ctypes.byref(out)))
        return Dataset(self.engine, None, self.precision, _handle=out)

    def params(self, nmf_kwargs):
        return make_params(nmf_kwargs, self.shape[0], self.shape[1], self.precision)

    def factorize(self, ks, seeds, nmf_kwargs, return_usages=False, W0=None, H0=None, X_host=None):
        """All restarts (ks[r], seeds[r]) at once.  Returns (spectra_list, usages_list|None, n_iter, err).
        W0 / H0: packed starting factors (sum ks x cells, sum ks x genes) instead of the seeded init.  The NNDSVD family
        of nmf_kwargs['init'] runs on the device, unless X_host (the host matrix the dataset was created from) is
        given: then its starts come from cnmf_b200.nndsvd on the host."""
        ks = np.ascontiguousarray(ks, dtype=np.int32)
        R = len(ks)
        SK = int(ks.sum())
        n, g = self.shape
        p = self.params(nmf_kwargs)
        self._check_loss(p)
        dt = np.float64 if self.fp64 else np.float32
        spectra = np.empty((SK, g), dt)
        usages = np.empty((SK, n), dt) if return_usages else None
        n_iter = np.zeros(R, np.int32)
        err = np.zeros(R, np.float64)
        init = nmf_kwargs.get("init", "random")
        if W0 is None and init != "random" and X_host is not None:
            # NNDSVD family (cnmf.py:1252 / SK _nmf.py:309-369) on the host: starting factors from cnmf_b200.nndsvd, one
            # randomized SVD per restart (the seed enters through its test matrix), then the ordinary batched solve
            W0, H0 = nndsvd_starts(X_host, ks, seeds, init, dtype=dt)
        if self.fp64:
            if W0 is None:
                p.reserved |= init_code(init, ks, n, g) << 1
                seeds = np.ascontiguousarray(seeds, dtype=np.uint32)
                check(self.lib.cnmf_factorize_f64(self._d, R, ptr(ks), ptr(seeds), ctypes.byref(p), ptr(spectra),
                                                  ptr(usages), ptr(n_iter), ptr(err), None))
            else:
                W0, H0 = f64c(W0), f64c(H0)
                assert W0.shape == (SK, n) and H0.shape == (SK, g)
                check(self.lib.cnmf_factorize_init_f64(self._d, R, ptr(ks), ptr(W0), ptr(H0), ctypes.byref(p),
                                                       ptr(spectra), ptr(usages), ptr(n_iter), ptr(err), None))
        elif W0 is None:
            p.reserved |= init_code(init, ks, n, g) << 1
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
        fixed = f64c(fixed) if self.fp64 else f32c(fixed)
        k = fixed.shape[0]
        n, g = self.shape
        n_r, n_c = (g, n) if transposed else (n, g)
        assert fixed.shape[1] == n_c
        p = make_params(nmf_kwargs, n_r, n_c, self.precision, for_refit=True)
        self._check_loss(p)
        out = np.empty((n_r, k), fixed.dtype)
        it = ctypes.c_int32(0)
        err = ctypes.c_double(0)
        fn = self.lib.cnmf_refit_f64 if self.fp64 else self.lib.cnmf_refit
        check(fn(self._d, 1 if transposed else 0, k, ptr(fixed), ctypes.byref(p), ptr(out), ctypes.byref(it),
                 ctypes.byref(err), None))
        return out, int(it.value), float(err.value)

    def project_rows(self, Ut):
        """Ut (k x cells) @ X -> (k x genes)."""
        Ut = f64c(Ut) if self.fp64 else f32c(Ut)
        k = Ut.shape[0]
        assert Ut.shape[1] == self.shape[0]
        out = np.empty((k, self.shape[1]), Ut.dtype)
        fn = self.lib.cnmf_project_rows_f64 if self.fp64 else self.lib.cnmf_project_rows
        check(fn(self._d, k, ptr(Ut), ptr(out), None))
        return out
