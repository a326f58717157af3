"""ctypes binding of libcnmf_b200.so (the C ABI in include/cnmf_b200.h).

The CUDA library is the product: there is no Python / numpy / torch fallback.  Importing this
module never needs a GPU (so CPU-only hosts can check the ABI), but every compute entry point
raises ``CnmfError`` when no sm_90 (H100) device is present.
"""
import ctypes
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libcnmf_b200.so")

SOLVER_MU, SOLVER_CD = 0, 1
PRECISION_FP32, PRECISION_TF32X3, PRECISION_TF32X3_GENERAL, PRECISION_F16X2, PRECISION_FP64 = 0, 1, 2, 3, 4
LOSS_FROBENIUS, LOSS_KULLBACK_LEIBLER, LOSS_ITAKURA_SAITO = 0, 1, 2
INIT_RANDOM, INIT_NNDSVD, INIT_NNDSVDA, INIT_NNDSVDAR = 0, 1, 2, 3
INIT_CODES = {"random": INIT_RANDOM, "nndsvd": INIT_NNDSVD, "nndsvda": INIT_NNDSVDA, "nndsvdar": INIT_NNDSVDAR}
MAX_COMPONENTS = 32


class CnmfError(RuntimeError):
    pass


class NmfParams(ctypes.Structure):
    """struct cnmf_nmf_params (include/cnmf_b200.h)."""
    _fields_ = [("solver", ctypes.c_int32), ("precision", ctypes.c_int32), ("max_iter", ctypes.c_int32),
                ("reserved", ctypes.c_int32), ("tol", ctypes.c_double),
                ("l1_reg_W", ctypes.c_double), ("l2_reg_W", ctypes.c_double),
                ("l1_reg_H", ctypes.c_double), ("l2_reg_H", ctypes.c_double),
                ("beta_loss", ctypes.c_int32), ("reserved2", ctypes.c_int32)]


UNIT_SOLVER_NONE = -1
UNIT_PIECES_NONE, UNIT_PIECES_TF32, UNIT_PIECES_F16 = 0, 1, 2
UNIT_GRAM_NONE, UNIT_GRAM_FUSED, UNIT_GRAM_STANDALONE = 0, 1, 2


class UpdateStepArgs(ctypes.Structure):
    """struct cnmf_update_step_args (include/cnmf_b200.h): arguments of the cnmf_update_step_host test hook."""
    _fields_ = [("n_slots", ctypes.c_int32), ("n_rids", ctypes.c_int32),
                ("ks", ctypes.c_void_p), ("rids", ctypes.c_void_p), ("done", ctypes.c_void_p),
                ("n", ctypes.c_int32), ("cpb_tiles", ctypes.c_int32), ("solver", ctypes.c_int32),
                ("pieces", ctypes.c_int32), ("gram", ctypes.c_int32), ("want_scalar", ctypes.c_int32),
                ("nsplit", ctypes.c_int32), ("l1", ctypes.c_float), ("l2", ctypes.c_float),
                ("F", ctypes.c_void_p), ("num", ctypes.c_void_p), ("gram_in", ctypes.c_void_p),
                ("piece_scale", ctypes.c_void_p), ("pieces_hi", ctypes.c_void_p), ("pieces_lo", ctypes.c_void_p),
                ("tile_scale", ctypes.c_void_p), ("gram_out", ctypes.c_void_p), ("scal_out", ctypes.c_void_p)]


UNIT_BETA_UPDATE, UNIT_BETA_DIVERGENCE = 0, 1
UNIT_SIDE_W, UNIT_SIDE_H = 0, 1


class BetaStepArgs(ctypes.Structure):
    """struct cnmf_beta_step_args (include/cnmf_b200.h): arguments of the cnmf_beta_step_host test hook."""
    _fields_ = [("n_slots", ctypes.c_int32), ("n_rids", ctypes.c_int32),
                ("ks", ctypes.c_void_p), ("rids", ctypes.c_void_p), ("done", ctypes.c_void_p),
                ("op", ctypes.c_int32), ("side", ctypes.c_int32), ("loss", ctypes.c_int32),
                ("n_items", ctypes.c_int32), ("n_contract", ctypes.c_int32), ("l1", ctypes.c_float), ("l2", ctypes.c_float),
                ("D", ctypes.c_void_p), ("F_own", ctypes.c_void_p), ("F_other", ctypes.c_void_p),
                ("oth_sum", ctypes.c_void_p), ("last", ctypes.c_void_p), ("totals", ctypes.c_void_p)]


UNIT_F64_UPDATE, UNIT_F64_GRAM, UNIT_F64_CROSS = 0, 1, 2


class UpdateStepF64Args(ctypes.Structure):
    """struct cnmf_update_step_f64_args (include/cnmf_b200.h): arguments of the cnmf_update_step_f64_host test hook."""
    _fields_ = [("n_slots", ctypes.c_int32), ("n_rids", ctypes.c_int32),
                ("ks", ctypes.c_void_p), ("rids", ctypes.c_void_p), ("done", ctypes.c_void_p),
                ("n", ctypes.c_int32), ("op", ctypes.c_int32), ("solver", ctypes.c_int32),
                ("want_scalar", ctypes.c_int32), ("l1", ctypes.c_double), ("l2", ctypes.c_double),
                ("F", ctypes.c_void_p), ("num", ctypes.c_void_p), ("gram_in", ctypes.c_void_p),
                ("gram_out", ctypes.c_void_p), ("scal_out", ctypes.c_void_p)]


FORM_FP32, FORM_TF32, FORM_TF32_EXACT, FORM_F16_EXACT, FORM_FP64 = 0, 1, 2, 3, 4
FORM_NAMES = {FORM_FP32: "fp32", FORM_TF32: "tf32", FORM_TF32_EXACT: "tf32_exact", FORM_F16_EXACT: "f16_exact",
              FORM_FP64: "fp64"}
# resident arrays of cnmf_dataset_operand_host
OPERANDS = {"X": 0, "Xt": 1, "X_hi": 2, "X_lo": 3, "Xt_hi": 4, "Xt_lo": 5, "X_h16": 6, "Xt_h16": 7, "row_scale": 8,
            "col_scale": 9, "csc_col_ptr": 10, "csc_row_idx": 11, "csc_values": 12}


class ConvCheckArgs(ctypes.Structure):
    """struct cnmf_conv_check_args (include/cnmf_b200.h): arguments of the cnmf_conv_check_host test hook."""
    _fields_ = [("n_slots", ctypes.c_int32), ("n_rids", ctypes.c_int32),
                ("ks", ctypes.c_void_p), ("rids", ctypes.c_void_p),
                ("solver", ctypes.c_int32), ("it", ctypes.c_int32), ("max_iter", ctypes.c_int32),
                ("tol", ctypes.c_double), ("normX2", ctypes.c_double),
                ("cross", ctypes.c_void_p), ("gramA", ctypes.c_void_p), ("gramB", ctypes.c_void_p),
                ("violA", ctypes.c_void_p), ("violB", ctypes.c_void_p),
                ("done", ctypes.c_void_p), ("n_iter", ctypes.c_void_p),
                ("err0", ctypes.c_void_p), ("prev", ctypes.c_void_p), ("last", ctypes.c_void_p)]


_c = ctypes
_vp, _i, _ll, _d = _c.c_void_p, _c.c_int, _c.c_longlong, _c.c_double
_pp = _c.POINTER

# name -> (restype, argtypes); every symbol declared in include/cnmf_b200.h
SIGNATURES = {
    "cnmf_abi_version": (_i, []),
    "cnmf_last_error": (_c.c_char_p, []),
    "cnmf_create": (_i, [_pp(_vp), _i]),
    "cnmf_destroy": (_i, [_vp]),
    "cnmf_launch_count": (_ll, [_vp]),
    "cnmf_mem_info": (_i, [_vp, _pp(_ll), _pp(_ll), _pp(_ll)]),
    "cnmf_solve_bytes_per_row": (_ll, [_vp]),
    "cnmf_profile_enable": (_i, [_vp, _i]),
    "cnmf_profile_get": (_i, [_vp, _pp(_d), _pp(_ll), _pp(_d)]),
    "cnmf_profile_get_class": (_i, [_vp, _i, _pp(_d), _pp(_ll), _pp(_d)]),
    "cnmf_last_timing": (_i, [_vp, _pp(_d), _pp(_d), _pp(_d), _pp(_d)]),
    "cnmf_dataset_create": (_i, [_vp, _vp, _i, _i, _ll, _i, _i, _vp, _pp(_vp)]),
    "cnmf_dataset_create_csc": (_i, [_vp, _i, _i, _ll, _vp, _vp, _vp, _i, _vp, _pp(_vp)]),
    "cnmf_dataset_create_csr": (_i, [_vp, _i, _i, _ll, _vp, _vp, _vp, _i, _vp, _pp(_vp)]),
    "cnmf_dataset_create_from_csr": (_i, [_vp, _i, _i, _ll, _vp, _vp, _vp, _i, _vp, _pp(_vp)]),
    "cnmf_dataset_create_from_csr_f64": (_i, [_vp, _i, _i, _ll, _vp, _vp, _vp, _vp, _pp(_vp)]),
    "cnmf_dataset_dense_bytes": (_i, [_i, _i, _i, _pp(_ll)]),
    "cnmf_dataset_from_columns": (_i, [_vp, _vp, _vp, _i, _vp, _pp(_vp)]),
    "cnmf_dataset_destroy": (_i, [_vp]),
    "cnmf_dataset_shape": (_i, [_vp, _pp(_i), _pp(_i)]),
    "cnmf_dataset_ld": (_i, [_vp, _pp(_i), _pp(_i)]),
    "cnmf_dataset_is_exact": (_i, [_vp]),
    "cnmf_dataset_sums": (_i, [_vp, _pp(_d), _pp(_d)]),
    "cnmf_dataset_min": (_i, [_vp, _pp(_c.c_float), _vp]),
    "cnmf_dataset_col_stats": (_i, [_vp, _vp, _vp, _vp]),
    "cnmf_dataset_row_sums": (_i, [_vp, _vp, _vp]),
    "cnmf_dataset_scaled_col_stats": (_i, [_vp, _vp, _vp, _vp, _vp]),
    "cnmf_dataset_scale_rows": (_i, [_vp, _vp, _vp, _pp(_vp)]),
    "cnmf_dataset_tpm_stats": (_i, [_vp, _d, _vp, _vp, _vp, _vp]),
    "cnmf_random_init_host": (_i, [_c.c_uint32, _d, _i, _i, _i, _vp, _ll, _vp, _ll]),
    "cnmf_random_init_dev": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _vp]),
    "cnmf_nndsvd_init_dev": (_i, [_vp, _i, _vp, _vp, _i, _vp, _vp, _vp]),
    "cnmf_nndsvd_chunk_limit": (_i, [_vp, _i]),
    "cnmf_nndsvd_gemm_host": (_i, [_vp, _i, _i, _vp, _vp, _vp]),
    "cnmf_dataset_create_f64": (_i, [_vp, _vp, _i, _i, _ll, _i, _vp, _pp(_vp)]),
    "cnmf_dataset_from_columns_f64": (_i, [_vp, _vp, _vp, _i, _vp, _pp(_vp)]),
    "cnmf_factorize_f64": (_i, [_vp, _i, _vp, _vp, _pp(NmfParams), _vp, _vp, _vp, _vp, _vp]),
    "cnmf_factorize_init_f64": (_i, [_vp, _i, _vp, _vp, _vp, _pp(NmfParams), _vp, _vp, _vp, _vp, _vp]),
    "cnmf_refit_f64": (_i, [_vp, _i, _i, _vp, _pp(NmfParams), _vp, _pp(_c.c_int32), _pp(_d), _vp]),
    "cnmf_project_rows_f64": (_i, [_vp, _i, _vp, _vp, _vp]),
    "cnmf_factorize": (_i, [_vp, _i, _vp, _vp, _pp(NmfParams), _vp, _vp, _vp, _vp, _vp]),
    "cnmf_factorize_seeds_dev": (_i, [_vp, _i, _vp, _vp, _pp(NmfParams), _vp, _ll, _vp, _vp, _vp]),
    "cnmf_allgather_spectra": (_i, [_vp, _vp, _ll, _ll, _vp, _vp]),
    "cnmf_comm_unique_id": (_i, [_vp]),
    "cnmf_comm_create": (_i, [_vp, _vp, _i, _i, _pp(_vp)]),
    "cnmf_comm_destroy": (_i, [_vp]),
    "cnmf_factorize_init": (_i, [_vp, _i, _vp, _vp, _vp, _pp(NmfParams), _vp, _vp, _vp, _vp, _vp]),
    "cnmf_factorize_dev": (_i, [_vp, _i, _vp, _vp, _vp, _pp(NmfParams), _vp, _vp, _vp, _vp]),
    "cnmf_refit": (_i, [_vp, _i, _i, _vp, _pp(NmfParams), _vp, _pp(_c.c_int32), _pp(_d), _vp]),
    "cnmf_project_rows": (_i, [_vp, _i, _vp, _vp, _vp]),
    "cnmf_gemm_abt_host": (_i, [_vp, _i, _vp, _vp, _i, _i, _i, _i, _i, _vp, _vp, _i, _vp, _i, _pp(_c.c_float), _vp]),
    "cnmf_update_step_host": (_i, [_vp, _pp(UpdateStepArgs), _vp]),
    "cnmf_beta_step_host": (_i, [_vp, _pp(BetaStepArgs), _vp]),
    "cnmf_update_step_f64_host": (_i, [_vp, _pp(UpdateStepF64Args), _vp]),
    "cnmf_conv_check_host": (_i, [_vp, _pp(ConvCheckArgs), _vp]),
    "cnmf_dataset_form": (_i, [_vp]),
    "cnmf_dataset_operand_host": (_i, [_vp, _i, _vp, _ll]),
    "cnmf_dataset_gemm_host": (_i, [_vp, _i, _i, _i, _vp, _vp, _pp(_i)]),
    "cnmf_l2_normalize_rows": (_i, [_vp, _vp, _i, _i, _i, _vp]),
    "cnmf_local_density": (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp]),
    "cnmf_col_stats_dev": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _vp]),
    "cnmf_gather_rows": (_i, [_vp, _vp, _i, _vp, _i, _i, _vp, _i, _vp]),
    "cnmf_sq_dists_to_rows": (_i, [_vp, _vp, _i, _i, _i, _vp, _i, _vp, _vp]),
    "cnmf_kmeans_step": (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _pp(_c.c_int32), _pp(_c.c_int32), _pp(_d), _vp]),
    "cnmf_kmeans_fit": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _i, _d, _vp, _vp, _i, _vp, _vp, _vp, _pp(_c.c_int32), _vp]),
    "cnmf_kmeans_assign": (_i, [_vp, _vp, _i, _i, _i, _vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "cnmf_cluster_dist_sums": (_i, [_vp, _vp, _i, _i, _i, _vp, _i, _vp, _vp]),
    "cnmf_cluster_median": (_i, [_vp, _vp, _i, _i, _i, _vp, _i, _vp, _i, _vp]),
    "cnmf_l2_normalize_rows_f64": (_i, [_vp, _vp, _i, _i, _i, _vp]),
    "cnmf_local_density_f64": (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp]),
    "cnmf_col_stats_dev_f64": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _vp]),
    "cnmf_gather_rows_f64": (_i, [_vp, _vp, _i, _vp, _i, _i, _vp, _i, _vp]),
    "cnmf_sq_dists_to_rows_f64": (_i, [_vp, _vp, _i, _i, _i, _vp, _i, _vp, _vp]),
    "cnmf_kmeans_step_f64": (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _pp(_c.c_int32), _pp(_c.c_int32), _pp(_d), _vp]),
    "cnmf_kmeans_fit_f64": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _i, _d, _vp, _vp, _i, _vp, _vp, _vp, _pp(_c.c_int32), _vp]),
    "cnmf_kmeans_assign_f64": (_i, [_vp, _vp, _i, _i, _i, _vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "cnmf_cluster_dist_sums_f64": (_i, [_vp, _vp, _i, _i, _i, _vp, _i, _vp, _vp]),
    "cnmf_cluster_median_f64": (_i, [_vp, _vp, _i, _i, _i, _vp, _i, _vp, _i, _vp]),
    "cnmf_moe_grams": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _vp, _vp]),
    "cnmf_moe_correct": (_i, [_vp, _vp, _i, _i, _i, _ll, _i, _vp, _vp, _vp, _i, _i, _i, _vp, _ll, _i, _vp, _vp, _vp]),
    "cnmf_scale_quantile_ceiling": (_i, [_vp, _vp, _i, _i, _i, _ll, _i, _vp, _vp, _ll, _d, _i, _ll, _ll, _d, _vp, _ll,
                                         _i, _pp(_d), _vp]),
}

_lib = None


ABI_VERSION = 19     # include/cnmf_b200.h CNMF_B200_ABI_VERSION


def load():
    """Load the shared library (once) and attach the signatures. Fails loudly if it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise CnmfError(
            "libcnmf_b200.so not found at %s -- build it with `python -m cnmf_b200.build` "
            "(cnmf_b200 has no CPU / PyTorch fallback)" % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)        # AttributeError here = ABI mismatch: let it propagate
        fn.restype = res
        fn.argtypes = args
    if lib.cnmf_abi_version() != ABI_VERSION:
        raise CnmfError("libcnmf_b200.so ABI version mismatch")
    _lib = lib
    return lib


def check(rc):
    if rc != 0:
        msg = load().cnmf_last_error()
        raise CnmfError("cnmf_b200 error %d: %s" % (rc, msg.decode() if msg else "?"))


def ptr(a):
    """Raw data pointer of a C-contiguous numpy array (or None)."""
    if a is None:
        return None
    assert a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(ctypes.c_void_p)


def f32c(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def f64c(a):
    return np.ascontiguousarray(a, dtype=np.float64)
