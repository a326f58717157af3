"""Preprocessing before `cnmf prepare` (the reference's src/cnmf/preprocess.py): Harmony batch correction of the
normalised cells x genes matrix, and variance scaling with a quantile ceiling, on the GPU.

Harmony itself (the soft clustering of the PCs) runs on the host through harmonypy, as in the reference; its
mixture-of-experts ridge correction of every gene -- K ridge solves, each two passes over the N x G matrix in numpy --
runs as fp64 GEMMs and a fused epilogue (cnmf_moe_grams / cnmf_moe_correct).  The scanpy-bound plumbing (filtering,
seurat_v3 HVGs, PCA, mutual-information features) is not provided.

Importing this module needs neither a GPU, harmonypy nor scanpy.
"""
import ctypes

import numpy as np
import scipy.sparse as sp

from . import _lib

_ENGINE = None

HARMONYPY_MISSING = "harmonypy is not installed. Please install it using 'pip install harmonypy' before proceeding."


def _engine():
    global _ENGINE
    if _ENGINE is None:
        from .engine import Engine
        _ENGINE = Engine(0)
    return _ENGINE


def _dtype_code(a):
    if a.dtype == np.float32:
        return 0
    if a.dtype == np.float64:
        return 1
    raise TypeError("expected a float32 or float64 matrix, got %s" % a.dtype)


def moe_grams(R, Phi_moe, lamb):
    """A_i = (Phi_moe * R[i]) Phi_moe^T + lamb for every cluster i, (K, B+1, B+1) float64, computed on the GPU."""
    R = _lib.f64c(R)
    Phi = _lib.f64c(Phi_moe)
    lamb = _lib.f64c(lamb)
    K, N = R.shape
    B1 = Phi.shape[0]
    if Phi.shape[1] != N or lamb.shape != (B1, B1):
        raise ValueError("R (K x N), Phi_moe (B+1 x N) and lamb (B+1 x B+1) do not agree")
    eng = _engine()
    A = np.empty((K, B1, B1), np.float64)
    _lib.check(eng.lib.cnmf_moe_grams(eng._h, _lib.ptr(R), _lib.ptr(Phi), _lib.ptr(lamb), K, B1, N, _lib.ptr(A),
                                      None))
    return A


def moe_correct_cells(X, R, Phi_moe, lamb, clamp_zero=False, want_cos=False):
    """Ridge correction of a cells x genes matrix X (float32 or float64, returned in the same type):
    X - sum_i W_i^T (Phi_moe * R[i]) with W_i = inv(A_i) (Phi_moe * R[i]) X and row 0 of W_i zeroed.
    A singular A_i raises numpy.linalg.LinAlgError.  Returns (X_corr, X_cos or None, W of the last cluster)."""
    X = np.ascontiguousarray(np.asarray(X))
    code = _dtype_code(X)
    R = _lib.f64c(R)
    Phi = _lib.f64c(Phi_moe)
    N, G = X.shape
    K = R.shape[0]
    B1 = Phi.shape[0]
    if R.shape[1] != N or Phi.shape[1] != N:
        raise ValueError("R and Phi_moe must have one column per cell (%d)" % N)
    Ainv = np.ascontiguousarray(np.linalg.inv(moe_grams(R, Phi, lamb)))
    eng = _engine()
    out = np.empty_like(X)
    cos = np.empty_like(X) if want_cos else None
    W = np.empty((B1, G), np.float64)
    _lib.check(eng.lib.cnmf_moe_correct(eng._h, _lib.ptr(X), code, N, G, G, 0, _lib.ptr(R), _lib.ptr(Phi),
                                        _lib.ptr(Ainv), K, B1, 1 if clamp_zero else 0, _lib.ptr(out), G, 0,
                                        _lib.ptr(cos), _lib.ptr(W), None))
    return out, cos, W


def moe_correct_ridge(Z_orig, Z_cos, Z_corr, R, W, K, Phi_Rk, Phi_moe, lamb):
    """The reference's moe_correct_ridge (preprocess.py:9-18) on the GPU: Z_orig is genes x cells.  Returns
    (Z_cos, Z_corr, W, Phi_Rk) with W and Phi_Rk of the last cluster, as the reference does."""
    R = np.asarray(R)[:int(K)]
    Phi_moe = np.asarray(Phi_moe)
    Zc, Zcos, W = moe_correct_cells(np.asarray(Z_orig).T, R, Phi_moe, lamb, want_cos=True)
    Phi_Rk = np.multiply(Phi_moe, R[-1, :])
    return Zcos.T, Zc.T, W, Phi_Rk


def harmony_layout(harmony_res, pca):
    """(R as K x cells, Phi_moe as (B+1) x cells, X_pca_harmony as cells x PCs) from a Harmony result in either
    harmonypy layout: older versions keep cells as columns, newer ones as rows (told apart by Z_corr's shape, as
    preprocess.py:405-414 does)."""
    Z_corr = np.asarray(harmony_res.Z_corr)
    R = np.asarray(harmony_res.R)
    Phi_moe = np.asarray(harmony_res.Phi_moe)
    if Z_corr.shape[0] == np.shape(pca)[0]:
        return R.T, Phi_moe.T, Z_corr
    return R, Phi_moe, Z_corr.T


def quantile_ranks(n, q, dtype):
    """(k_lo, k_hi, gamma) of np.quantile(a, q) (linear method) for n values of a float array of `dtype`: the ranks
    of the two order statistics it interpolates and the weight, computed in the types numpy computes them in."""
    if isinstance(q, (int, float)):
        q = np.asanyarray(q, dtype=dtype)
    else:
        q = np.asanyarray(q)
    if q.ndim != 0 or not (0 <= q <= 1):
        raise ValueError("Quantiles must be in the range [0, 1]")
    v = np.asanyarray((n - 1) * q)
    prev = np.asanyarray(np.floor(v))
    nxt = np.asanyarray(prev + 1)
    if v >= n - 1:
        prev, nxt = np.asanyarray(prev * 0 - 1), np.asanyarray(nxt * 0 - 1)
    prev_i = prev.astype(np.intp)
    nxt_i = nxt.astype(np.intp)
    gamma = np.asanyarray(np.asanyarray(v - prev_i), dtype=v.dtype)
    return int(prev_i) % n, int(nxt_i) % n, float(gamma)


def scale_quantile_ceiling(X, max_value=None, quantile_thresh=None):
    """Dense or CSR X -> (dense result in X's float type, threshold or None): each column divided by its ddof = 1
    std (a zero std counts as 1), clipped at max_value, then values above np.quantile(result, quantile_thresh) set to
    that quantile.  Integer input is scaled as float64."""
    csr = None
    if sp.issparse(X):
        csr = sp.csr_matrix(X)
        csr.sum_duplicates()
        csr.sort_indices()
        vals = csr.data if csr.data.dtype in (np.float32, np.float64) else csr.data.astype(np.float64)
        vals = np.ascontiguousarray(vals)
        N, G = csr.shape
        dtype = vals.dtype
        row_ptr = np.ascontiguousarray(csr.indptr, dtype=np.int64)
        col_idx = np.ascontiguousarray(csr.indices, dtype=np.int32)
        src, nnz = vals, int(csr.nnz)
    else:
        src = np.asarray(X)
        if src.dtype not in (np.float32, np.float64):
            src = src.astype(np.float64)
        src = np.ascontiguousarray(src)
        N, G = src.shape
        dtype = src.dtype
        row_ptr = col_idx = None
        nnz = 0
    k_lo = k_hi = -1
    gamma = 0.0
    if quantile_thresh is not None:
        k_lo, k_hi, gamma = quantile_ranks(N * G, quantile_thresh, dtype)
    eng = _engine()
    out = np.empty((N, G), dtype)
    thresh = ctypes.c_double()
    _lib.check(eng.lib.cnmf_scale_quantile_ceiling(
        eng._h, _lib.ptr(src), _dtype_code(out), N, G, G, 0, _lib.ptr(row_ptr), _lib.ptr(col_idx), nnz,
        float(max_value) if max_value is not None else 0.0, 0 if max_value is None else 1, k_lo, k_hi, gamma,
        _lib.ptr(out), G, 0, ctypes.byref(thresh), None))
    return out, (dtype.type(thresh.value) if quantile_thresh is not None else None), csr


def stdscale_quantile_celing(_adata, max_value=None, quantile_thresh=None):
    """The reference's stdscale_quantile_celing (preprocess.py:21-29) on the GPU, in place on _adata.X (anything with
    an .X: CellGeneMatrix, AnnData).  A CSR .X is densified on the device and stays CSR with its sparsity pattern."""
    out, _, csr = scale_quantile_ceiling(_adata.X, max_value, quantile_thresh)
    if csr is None:
        _adata.X = out
    else:
        rows = np.repeat(np.arange(csr.shape[0]), np.diff(csr.indptr))
        _adata.X = sp.csr_matrix((out[rows, csr.indices], csr.indices.copy(), csr.indptr.copy()), shape=csr.shape)


_SCANPY_BOUND = ("%s needs scanpy's AnnData, seurat_v3 highly variable genes and PCA, which cnmf_b200 does not "
                 "provide: run it with the reference package, or call Preprocess.harmony_correct_X and "
                 "stdscale_quantile_celing on the matrices directly")


class Preprocess():
    """Batch correction for cNMF on the GPU: Harmony's ridge correction applied to the normalised counts rather than
    the PCs (the reference's Preprocess, preprocess.py:41)."""

    def __init__(self, random_seed=None):
        np.random.seed(random_seed)

    def filter_adata(self, *args, **kwargs):
        raise NotImplementedError(_SCANPY_BOUND % "Preprocess.filter_adata")

    def preprocess_for_cnmf(self, *args, **kwargs):
        raise NotImplementedError(_SCANPY_BOUND % "Preprocess.preprocess_for_cnmf")

    def normalize_batchcorrect(self, *args, **kwargs):
        raise NotImplementedError(_SCANPY_BOUND % "Preprocess.normalize_batchcorrect")

    def select_features_MI(self, *args, **kwargs):
        raise NotImplementedError(_SCANPY_BOUND % "Preprocess.select_features_MI")

    def harmony_correct_X(self, X, obs, pca, harmony_vars, theta=1, max_iter_harmony=20, harmony_res=None):
        """Fit Harmony on the PCs (harmonypy, host) and remove each cluster's batch effect from every gene of the
        cells x genes matrix X on the GPU; negatives are set to 0.  Returns (X_corr, X_pca_harmony).

        harmony_res: an already fitted Harmony result (attributes Z_corr, R, Phi_moe, K, lamb, in either harmonypy
        layout); harmonypy is then not needed and obs, harmony_vars, theta and max_iter_harmony are unused."""
        if harmony_res is None:
            try:
                import harmonypy
            except ImportError:
                raise ImportError(HARMONYPY_MISSING)
            harmony_res = harmonypy.run_harmony(pca, obs, harmony_vars, max_iter_harmony=max_iter_harmony,
                                                theta=theta)
        R, Phi_moe, X_pca_harmony = harmony_layout(harmony_res, pca)
        R = R[:int(harmony_res.K)]
        X_corr, _, _ = moe_correct_cells(np.asarray(X), R, Phi_moe, harmony_res.lamb, clamp_zero=True)
        return X_corr, X_pca_harmony
