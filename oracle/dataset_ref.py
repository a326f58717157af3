"""What dataset creation leaves resident on the device, restated in numpy in the device's own arithmetic, so that the
operands can be compared bit for bit (tests/test_dataset_units.py; pinned by tests/test_oracle_golden.py).

  cnmf_dataset_create -> dataset_resolve_form (capi.cu): exact-count detection, min_positive_kernel / fix_scale_kernel /
                         check_scaled_int_kernel (nmf_kernels.cu), csc_detect_exact (sparse_kernels.cu) on CSC input
                      -> dataset_finish (capi.cu): split_tf32_kernel, transpose_kernel, build_counts_kernel,
                         to_half_kernel
  cnmf_dataset_from_columns (capi_refit.cu): gather_cols_kernel, combine_scale_kernel, then dataset_finish

Every operation is IEEE float32 with round-to-nearest-even (the library is built without fast-math, so the device `/`
is correctly rounded, and rintf rounds ties to even), except to_tf32, which rounds ties away from zero
(cvt.rna.tf32.f32 as common.cuh writes it: add 0x1000 to the bit pattern and clear the low 13 bits).
"""
import numpy as np

F32 = np.float32
MAX_COUNT = 2048          # largest integer the exact forms hold (exact in fp16)
ADMIT = F32(5e-7)         # is_scaled_int: |q - n| <= 5e-7 n
SCALE_CAP = F32(1e30)     # fix_scale: a smallest positive entry at or above this is no scale
NO_ENTRY = np.uint32(0x7f7f7f7f).view(F32)    # what min_positive starts from (cudaMemset 0x7f)

FORMS = ("fp32", "tf32", "tf32_exact", "f16_exact")


def pad_ld(n):
    return -(-int(n) // 32) * 32


def to_tf32(x):
    """cvt.rna.tf32.f32 on finite fp32 values, as an fp32 bit pattern (common.cuh to_tf32)."""
    b = np.asarray(x, F32).view(np.uint32)
    return ((b + np.uint32(0x1000)) & np.uint32(0xffffe000)).view(F32)


def split_tf32(x):
    """hi = to_tf32(x), lo = to_tf32(x - hi) (common.cuh split_tf32)."""
    x = np.asarray(x, F32)
    hi = to_tf32(x)
    return hi, to_tf32((x - hi).astype(F32))


def is_scaled_int(v, sc):
    """Elementwise is_scaled_int (common.cuh): is v an integer n in [1, 2048] times sc, within 5e-7 n?"""
    v = np.asarray(v, F32)
    sc = np.asarray(sc, F32)
    with np.errstate(all="ignore"):
        q = (v / sc).astype(F32)
        n = np.rint(q).astype(F32)
        return (v > 0) & (n >= 1) & (n <= MAX_COUNT) & (np.abs((q - n).astype(F32)) <= (ADMIT * n).astype(F32))


def fix_scale(v, n_pad):
    """fix_scale_kernel: a line without a positive entry (or with a non-finite or >= 1e30 minimum) gets scale 1; the
    padding up to n_pad is 0."""
    v = np.asarray(v, F32)
    out = np.zeros(n_pad, F32)
    with np.errstate(all="ignore"):
        ok = np.isfinite(v) & (v > 0) & (v < SCALE_CAP)
    out[:len(v)] = np.where(ok, v, F32(1))
    return out


def min_positive(X, axis):
    """Smallest entry with 0 < x < inf along `axis` (0: per column, 1: per row); NO_ENTRY where there is none
    (min_positive_kernel, csc_min_positive_kernel: +inf orders like their sentinel, NaN is not positive)."""
    X = np.asarray(X, F32)
    with np.errstate(invalid="ignore"):
        pos = (X > 0) & np.isfinite(X)
    return np.where(pos, X, NO_ENTRY).min(axis=axis).astype(F32)


def scales(X):
    """(column scale of length ld_c, row scale of length ld_r): fix_scale of the minimum positive entries."""
    n, g = X.shape
    return fix_scale(min_positive(X, 0), pad_ld(g)), fix_scale(min_positive(X, 1), pad_ld(n))


def decide(X, precision):
    """dataset_resolve_form: (form, row_scale or None, col_scale or None).  fp32 and tf32x3-general never detect; tf32x3
    and f16x2 test the column scale first, then the row scale.  Zero entries are skipped; a negative, NaN or infinite
    entry fails both tests."""
    X = np.asarray(X, F32)
    if precision == "fp32":
        return "fp32", None, None
    if precision == "tf32x3-general":
        return "tf32", None, None
    assert precision in ("tf32x3", "f16x2"), precision
    exact = "f16_exact" if precision == "f16x2" else "tf32_exact"
    n, g = X.shape
    cs, rs = scales(X)
    nz = X != 0
    if is_scaled_int(X, cs[None, :g])[nz].all():
        return exact, None, cs
    if is_scaled_int(X, rs[:n, None])[nz].all():
        return exact, rs, None
    return "tf32", None, None


def counts(X, rs, cs):
    """build_counts_kernel: C = rint(x / fl(rs cs)) (0 where x == 0), n_rows x ld_c with zero padding."""
    X = np.asarray(X, F32)
    n, g = X.shape
    sc = np.ones((n, g), F32)
    if rs is not None:
        sc = sc * np.asarray(rs, F32)[:n, None]
    if cs is not None:
        sc = (sc * np.asarray(cs, F32)[None, :g]).astype(F32)
    C = np.zeros((n, pad_ld(g)), F32)
    with np.errstate(all="ignore"):
        C[:, :g] = np.where(X == 0, F32(0), np.rint((X / sc).astype(F32)))
    return C


def padded(X):
    X = np.asarray(X, F32)
    out = np.zeros((X.shape[0], pad_ld(X.shape[1])), F32)
    out[:, :X.shape[1]] = X
    return out


def transposed(A, n_cols, n_rows):
    """A (n_rows x ld_c, padded) -> n_cols x ld_r with zero padding, as transpose_kernel writes into a zeroed array."""
    out = np.zeros((n_cols, pad_ld(n_rows)), A.dtype)
    out[:, :n_rows] = A[:n_rows, :n_cols].T
    return out


def operands(X, form, rs=None, cs=None):
    """Every array dataset_finish leaves resident for a dense matrix X of the given form and scales (what
    cnmf_dataset_operand_host returns; arrays a form does not hold are absent)."""
    X = np.asarray(X, F32)
    n, g = X.shape
    Xp = padded(X)
    out = {"X": Xp}
    if form == "fp32":
        out["Xt"] = transposed(Xp, g, n)
    elif form == "tf32":
        hi, lo = split_tf32(Xp)
        out.update(X_hi=hi, X_lo=lo, Xt_hi=transposed(hi, g, n), Xt_lo=transposed(lo, g, n))
    else:
        C = counts(X, rs, cs)
        Ct = transposed(C, g, n)
        if form == "f16_exact":
            out.update(X_h16=C.astype(np.float16), Xt_h16=Ct.astype(np.float16))
        else:
            out.update(X_hi=C, Xt_hi=Ct)
        if rs is not None:
            out["row_scale"] = np.asarray(rs, F32)
        if cs is not None:
            out["col_scale"] = np.asarray(cs, F32)
    return out


def combine_scale(scale, src_cs, cols, n_pad):
    """combine_scale_kernel: fl(scale[c] * src_cs[cols[c]]) (src_cs None: scale[c]), zero padding to n_pad."""
    out = np.zeros(n_pad, F32)
    s = np.asarray(scale, F32)
    out[:len(s)] = s if src_cs is None else (s * np.asarray(src_cs, F32)[np.asarray(cols)]).astype(F32)
    return out
