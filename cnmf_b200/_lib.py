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
PRECISION_FP32, PRECISION_TF32X3, PRECISION_TF32X3_GENERAL, PRECISION_F16X2 = 0, 1, 2, 3
LOSS_FROBENIUS, LOSS_KULLBACK_LEIBLER, LOSS_ITAKURA_SAITO = 0, 1, 2
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
    "cnmf_random_init_host": (_i, [_c.c_uint32, _d, _i, _i, _i, _vp, _ll, _vp, _ll]),
    "cnmf_random_init_dev": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _vp]),
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
    "cnmf_gemm_abt_host": (_i, [_vp, _i, _vp, _vp, _i, _i, _i, _i, _vp, _i, _pp(_c.c_float), _vp]),
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
}

_lib = None


ABI_VERSION = 7      # include/cnmf_b200.h CNMF_B200_ABI_VERSION


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
