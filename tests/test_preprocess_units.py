"""The preprocessing kernels (preprocess_kernels.cu) one C call at a time, against extended precision and the reference:

  * cnmf_moe_grams alone: A_i = P_i Phi^T + lambda against a long-double restatement, at N around the 64-cell tiles and
    every split-K plan (one slice up to 4 096 cells, 32 slices longer than 4 096 above 131 072), K from 1 to 100 and
    B + 1 from 1 to 64, one-hot and signed Phi;
  * cnmf_moe_correct with an inverse the test supplies (independent of the grams): the corrected X, W_i of every
    cluster (a call with the single cluster R[i:i+1] returns it as W_last) and Z_cos, at K(B + 1) around the 32-row
    shared-memory stage of moe_apply_kernel, G around the 64-gene tiles, clamp on and off, strided host and device
    operands, and bit-identical repeats over several split-K slices;
  * cnmf_scale_quantile_ceiling: the scaled matrix equal bit for bit to the reference's scaling
    (oracle/make_golden_preprocess._scale) for G >= 2, on constant non-integer, zero, integer, negative, large-mean and
    NaN-producing columns; the radix select at every rank of a small matrix with ties, negatives, +-0, subnormals and
    float64 values that share their top 7 bytes, and at the digit edges of a larger one; NaN in the scaled matrix;
    CSR input equal to the dense path.

u = 2^-53.  Products too large for long double on the host (C = P X and the per-cluster terms) use float64 BLAS, and
the bound adds the BLAS result's own rounding; the small ones (A_i, W_i, the running subtraction) run in np.longdouble
(unit roundoff UL = 2^-64 on x86-64).  gamma(n) = n u / (1 - n u).  Every matrix comes from a seed here.
"""
import ctypes

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import make_golden_preprocess as mg

U = 2.0 ** -53
U32 = 2.0 ** -24
LD = np.longdouble
UL = 2.0 ** -(np.finfo(LD).nmant + 1)
SECOND = 1 + 2.0 ** -10          # second-order terms, relative to a first-order bound
RATIOS = {}
NEAR = {}


def gam(n):
    return n * U / (1 - n * U)


@pytest.fixture(scope="module")
def eng():
    from cnmf_b200.engine import Engine
    return Engine(0)


@pytest.fixture(scope="module", autouse=True)
def report_ratios():
    """Largest error-to-bound ratio per check and the near-midpoint roundings seen, printed after the module (-s)."""
    yield
    for k in sorted(RATIOS):
        print("ratio %-24s %.3g" % (k, RATIOS[k]))
    for k in sorted(NEAR):
        print("near midpoint %-16s %d" % (k, NEAR[k]))


def note(key, err, bound):
    err, bound = np.asarray(err, np.float64), np.asarray(bound, np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.where(bound > 0, err / bound, np.where(err > 0, np.inf, 0.0))
    r = float(q.max()) if q.size else 0.0
    RATIOS[key] = max(RATIOS.get(key, 0.0), r)
    assert r <= 1.0, (key, r)


def ptr(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def moe_chunk(n):
    """the kernel's split-K plan: slices of a length that depends on N only"""
    splits = min((n + 4095) // 4096, 32)
    return ((n + splits - 1) // splits + 15) // 16 * 16


def moe_splits(n):
    c = moe_chunk(n)
    return (n + c - 1) // c


def design(n, b1, kind, rng):
    """(B+1) x n: row 0 the intercept, then one-hot batch indicators or signed covariates"""
    if b1 == 1:
        return np.ones((1, n))
    if kind == "onehot":
        lab = rng.randint(0, b1 - 1, size=n)
        lab[:min(n, b1 - 1)] = np.arange(min(n, b1 - 1))
        return np.vstack([np.ones(n)] + [(lab == j).astype(np.float64) for j in range(b1 - 1)])
    return np.vstack([np.ones(n), rng.randn(b1 - 1, n) * 10.0 ** rng.uniform(-1, 1, (b1 - 1, 1))])


def assignments(k, n, rng):
    logits = rng.normal(scale=2.0, size=(k, n))
    R = np.exp(logits - logits.max(0))
    return R / R.sum(0)


# ------------------------------------------------------------------------------------------------------------ grams
GRAM_CASES = [
    # N, K, B+1, Phi
    (1, 1, 1, "onehot"),
    (2, 2, 2, "signed"),
    (63, 20, 3, "onehot"),
    (64, 100, 5, "signed"),
    (65, 2, 64, "signed"),
    (4095, 20, 33, "onehot"),
    (4096, 1, 32, "signed"),
    (4097, 100, 2, "signed"),
    (8193, 2, 5, "onehot"),
    (131072, 1, 3, "signed"),
    (131073, 2, 2, "onehot"),
]


def test_gram_cases_cover_every_axis_value():
    assert {c[0] for c in GRAM_CASES} == {1, 2, 63, 64, 65, 4095, 4096, 4097, 8193, 131072, 131073}
    assert {c[1] for c in GRAM_CASES} == {1, 2, 20, 100}
    assert {c[2] for c in GRAM_CASES} == {1, 2, 3, 5, 32, 33, 64}
    assert {c[3] for c in GRAM_CASES} == {"onehot", "signed"}
    assert moe_splits(4096) == 1 and moe_splits(4097) == 2 and moe_splits(131073) == 32
    assert moe_chunk(131073) > 4096


@pytest.mark.gpu
@pytest.mark.parametrize("n,k,b1,kind", GRAM_CASES)
def test_moe_grams_against_longdouble(eng, n, k, b1, kind):
    """|A - A_ref| <= gamma(N + splits + 1) sum_n |P_b Phi_c| + u |A| (the last rounding, of + lambda), plus the long
    double reference's own (N + 1) UL sum |P_b Phi_c|.  P = Phi * R[i] is the same fp64 product on both sides."""
    from cnmf_b200 import _lib
    rng = np.random.RandomState(n * 131 + k * 7 + b1)
    Phi = design(n, b1, kind, rng)
    R = assignments(k, n, rng)
    lamb = np.diag(np.concatenate([[0.0], np.full(b1 - 1, 1.0)])) + 0.25 * (kind == "signed") * np.eye(b1)
    A = np.empty((k, b1, b1))
    _lib.check(eng.lib.cnmf_moe_grams(eng._h, ptr(R), ptr(Phi), ptr(lamb), k, b1, n, ptr(A), None))
    PhiL, PhiA = Phi.astype(LD), np.abs(Phi)
    g = gam(n + moe_splits(n) + 1)
    for i in range(k):
        P = Phi * R[i]
        ref = P.astype(LD) @ PhiL.T + lamb.astype(LD)
        mag = np.abs(P) @ PhiA.T
        bound = ((g + (n + 1) * UL) * mag + U * np.abs(ref.astype(np.float64))) * SECOND
        note("grams", np.abs(A[i] - ref).astype(np.float64), bound)


# ------------------------------------------------------------------------------------------------------- correction
def correct(eng, X, R, Phi, Ainv, clamp=False, want_cos=False):
    """cnmf_moe_correct on host operands: (X_corr, X_cos or None, W of the last cluster)"""
    from cnmf_b200 import _lib
    X = np.ascontiguousarray(X)
    N, G = X.shape
    out = np.empty_like(X)
    cos = np.empty_like(X) if want_cos else None
    W = np.empty((Phi.shape[0], G))
    _lib.check(eng.lib.cnmf_moe_correct(
        eng._h, ptr(X), 0 if X.dtype == np.float32 else 1, N, G, G, 0, ptr(np.ascontiguousarray(R)),
        ptr(np.ascontiguousarray(Phi)), ptr(np.ascontiguousarray(Ainv)), R.shape[0], Phi.shape[0], int(clamp),
        ptr(out), G, 0, ptr(cos), ptr(W), None))
    return out, cos, W


def inverses(R, Phi):
    """A_i^-1 of the Grams with a unit ridge (always invertible), from numpy: the correction does not depend on them"""
    return np.ascontiguousarray(np.linalg.inv(np.stack([(Phi * r) @ Phi.T for r in R]) + np.eye(Phi.shape[0])))


def ulp32(x):
    x = np.abs(np.asarray(x, np.float32))
    return (np.nextafter(x, np.float32(np.inf)) - x).astype(np.float64)


def near_midpoint(v, e):
    """True where the long double value v lies within e of an fp32 rounding midpoint (or of the fp32 range's edge)"""
    r = v.astype(np.float32)
    up = np.nextafter(r, np.float32(np.inf)).astype(LD)
    dn = np.nextafter(r, np.float32(-np.inf)).astype(LD)
    rl = r.astype(LD)
    d = np.minimum(np.abs(v - (rl + up) / 2), np.abs(v - (rl + dn) / 2))
    return (d <= e) | ~np.isfinite(d)


class Restatement:
    """X - sum_i P_i^T W_i composed in the kernel's order, with the forward bound of every stage:
      C = P_i X            fp64 BLAS here; kernel and BLAS each within gamma(N + splits) |P_i| |X|
      W_i = A_i^-1 C_i     long double here; the kernel's B+1-term fp64 sums add gamma(B+1) |A_i^-1| |C_i|
      t = P_i^T W_i        fp64 BLAS here over rows b >= 1; each side gamma(B) |P_i| |W_i|, plus |P_i| e_W
      z <- z - t           long double here, rounded to fp64 (and, for fp32 X, then to fp32) as the kernel does
    For float64 X, ez bounds |kernel z - z| (both sides' roundings).  For float32 X, z is the fp32 value the kernel
    must reproduce: a cluster flags an entry when its value before rounding lies within its bound of an fp32 rounding
    midpoint; from the first flag on, the entry may differ by one fp32 ulp per cluster (allow)."""

    def __init__(self, X, R, Phi, Ainv):
        N, G = X.shape
        B1 = Phi.shape[0]
        X64 = X.astype(np.float64)
        absX = np.abs(X64)
        self.f32 = X.dtype == np.float32
        z = X64.astype(LD)
        ez = np.zeros((N, G))
        allow = np.zeros((N, G))
        flagged = np.zeros((N, G), bool)
        self.W, self.eW = [], []
        gC = gam(N + moe_splits(N))
        for i in range(R.shape[0]):
            P = Phi * R[i]
            C = P @ X64
            eC = 2 * gC * (np.abs(P) @ absX)
            Ai = Ainv[i]
            W = Ai.astype(LD) @ C.astype(LD)
            eW = (np.abs(Ai) @ eC + (gam(B1) + B1 * UL) * (np.abs(Ai) @ np.abs(C))) * SECOND
            W[0] = 0
            eW[0] = 0
            self.W.append(W)
            self.eW.append(eW)
            Wf = W.astype(np.float64)
            if B1 == 1:
                continue
            t = P[1:].T @ Wf[1:]
            eT = ((2 * gam(B1) + U) * (np.abs(P[1:]).T @ np.abs(Wf[1:])) + np.abs(P[1:]).T @ eW[1:]) * SECOND
            v = z - t.astype(LD)
            av = np.abs(v).astype(np.float64)
            if self.f32:
                e = (eT + U * av + UL * av) * SECOND
                hit = near_midpoint(v, e)
                flagged |= hit
                allow = np.where(flagged, allow + ulp32(av + allow) * 2, 0.0)
                z = v.astype(np.float32).astype(LD)
                NEAR["correct fp32"] = NEAR.get("correct fp32", 0) + int(hit.sum())
            else:
                z = v.astype(np.float64).astype(LD)
                ez = (ez + eT + 2 * U * av + UL * av) * SECOND
        self.z = z.astype(X.dtype)
        self.ez, self.allow, self.flagged = ez, allow, flagged

    def check(self, key, out, clamp):
        want = np.where(self.z < 0, 0, self.z).astype(self.z.dtype) if clamp else self.z
        if not self.f32:
            note(key, np.abs(out - want), self.ez)
            return
        same = out.view(np.uint32) == want.view(np.uint32)
        assert same[~self.flagged].all(), (key, int((~same & ~self.flagged).sum()))
        note(key + " near midpoint", np.abs(out.astype(np.float64) - want)[self.flagged], self.allow[self.flagged])

    def check_w(self, key, i, W):
        note(key, np.abs(W - self.W[i]).astype(np.float64), self.eW[i])


def correction_inputs(n, g, k, b1, dtype, seed, kind="onehot"):
    rng = np.random.RandomState(seed)
    X = (rng.gamma(0.6, 1.5, size=(n, g)) * (rng.rand(n, g) < 0.6)).astype(dtype)
    Phi = design(n, b1, kind, rng)
    R = assignments(k, n, rng)
    return X, R, Phi, inverses(R, Phi)


CORRECT_CASES = [
    # N, G, K, B+1, dtype, clamp, Phi
    (63, 31, 15, 2, np.float64, False, "onehot"),    # M = 30
    (64, 32, 16, 2, np.float32, True, "onehot"),     # M = 32: one whole stage
    (65, 33, 11, 3, np.float32, False, "signed"),    # M = 33: cluster 10 straddles rows 30-32
    (130, 63, 13, 5, np.float64, True, "onehot"),    # M = 65: clusters straddle rows 32 and 64
    (1, 64, 2, 33, np.float32, False, "signed"),     # M = 66, one cell
    (64, 32, 1, 64, np.float64, False, "signed"),    # M = 64, B + 1 at its limit
    (200, 2000, 3, 3, np.float32, False, "onehot"),
    (4095, 65, 2, 4, np.float64, False, "onehot"),
    (4096, 64, 20, 2, np.float32, False, "onehot"),
    (4097, 1, 5, 3, np.float32, False, "onehot"),    # two slices
    (8193, 33, 3, 2, np.float32, True, "signed"),    # three slices
    (131073, 2, 2, 3, np.float64, False, "onehot"),  # 32 slices of 4 112 cells
]


def test_correction_cases_cover_the_stage_and_slice_edges():
    ms = {c[2] * c[3] for c in CORRECT_CASES}
    assert {30, 32, 33, 64, 65, 66} <= ms
    assert {1, 31, 32, 33, 63, 64, 65, 2000} <= {c[1] for c in CORRECT_CASES}
    assert {63, 64, 65, 4095, 4096, 4097, 8193, 131073} <= {c[0] for c in CORRECT_CASES}
    assert {True, False} == {c[5] for c in CORRECT_CASES}


@pytest.mark.gpu
@pytest.mark.parametrize("n,g,k,b1,dtype,clamp,kind", CORRECT_CASES)
def test_moe_correct_against_restatement(eng, n, g, k, b1, dtype, clamp, kind):
    X, R, Phi, Ainv = correction_inputs(n, g, k, b1, dtype, n * 17 + g + k, kind)
    ref = Restatement(X, R, Phi, Ainv)
    out, cos, W = correct(eng, X, R, Phi, Ainv, clamp, want_cos=not clamp)
    tag = "correct " + np.dtype(dtype).name
    ref.check(tag, out, clamp)
    ref.check_w("W_last", k - 1, W)
    if not clamp:
        # Z_cos from the kernel's own corrected rows: fp64 sum of squares, sqrt rounded to X's type, one division
        o = out.astype(LD)
        norm = np.sqrt((o * o).sum(1, keepdims=True))
        want = (o / norm).astype(np.float64)
        u_t = U32 if dtype == np.float32 else U
        note("Z_cos " + np.dtype(dtype).name, np.abs(cos - want), np.abs(want) * (2 * u_t + gam(g) + 2 * U) * SECOND)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_moe_correct_every_cluster_w(eng, dtype):
    X, R, Phi, Ainv = correction_inputs(65, 33, 11, 3, dtype, 5, "signed")
    ref = Restatement(X, R, Phi, Ainv)
    for i in range(R.shape[0]):
        _, _, W = correct(eng, X, R[i:i + 1], Phi, Ainv[i:i + 1])
        assert not W[0].any()
        ref.check_w("W_i", i, W)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_moe_correct_intercept_only_is_identity(eng, dtype):
    """B + 1 = 1: W is the zeroed intercept row, nothing is subtracted, the output is X (clamped where asked)"""
    rng = np.random.RandomState(9)
    X = (rng.randn(65, 33) * 10.0 ** rng.uniform(-3, 3, (65, 33))).astype(dtype)
    X[0, :5] = (-0.0, 0.0, np.finfo(dtype).tiny / 4, -np.finfo(dtype).tiny / 4, np.finfo(dtype).max)
    R = assignments(3, 65, rng)
    Phi = np.ones((1, 65))
    Ainv = rng.rand(3, 1, 1)
    out, _, W = correct(eng, X, R, Phi, Ainv)
    assert np.array_equal(out.view(np.uint8), X.view(np.uint8)) and not W.any()
    out, _, _ = correct(eng, X, R, Phi, Ainv, clamp=True)
    assert np.array_equal(out.view(np.uint8), np.where(X < 0, dtype(0), X).view(np.uint8))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_moe_correct_zero_row_gives_nan_cosine(eng, dtype):
    """a cell with no cluster weight and a zero row stays zero; its Z_cos row is 0 / 0 = NaN, as in numpy"""
    X, R, Phi, Ainv = correction_inputs(70, 40, 4, 3, dtype, 11)
    X[17] = 0
    R[:, 17] = 0
    out, cos, _ = correct(eng, X, R, Phi, Ainv, want_cos=True)
    assert not out[17].any() and np.isnan(cos[17]).all()
    assert np.isfinite(np.delete(cos, 17, axis=0)).all()
    with np.errstate(invalid="ignore"):
        assert np.isnan(out[17] / np.linalg.norm(out[17])).all()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_moe_correct_strides_and_device_operands(eng, dtype):
    """ld / ld_out > G on host and device (torch) operands give the contiguous host call's bits and leave the padding
    of the output rows untouched"""
    import torch
    from cnmf_b200 import _lib
    X, R, Phi, Ainv = correction_inputs(65, 33, 3, 3, dtype, 21)
    want, want_cos, want_w = correct(eng, X, R, Phi, Ainv, want_cos=True)
    N, G = X.shape
    ld, ld_out = 40, 37
    code = 0 if dtype == np.float32 else 1
    sentinel = dtype(-7.25)
    for src_dev in (0, 1):
        for dst_dev in (0, 1):
            Xs = np.full((N, ld), dtype(3.5), dtype)
            Xs[:, :G] = X
            outs = [np.full((N, ld_out), sentinel, dtype) for _ in range(2)]
            if src_dev:
                Xs = torch.from_numpy(Xs).cuda()
            if dst_dev:
                outs = [torch.from_numpy(o).cuda() for o in outs]
            W = np.empty((3, G))
            torch.cuda.synchronize()
            p = (lambda t: ctypes.c_void_p(t.data_ptr()) if isinstance(t, torch.Tensor) else ptr(t))
            _lib.check(eng.lib.cnmf_moe_correct(eng._h, p(Xs), code, N, G, ld, src_dev, ptr(R), ptr(Phi), ptr(Ainv),
                                                3, 3, 0, p(outs[0]), ld_out, dst_dev, p(outs[1]), ptr(W), None))
            got = [o.cpu().numpy() if dst_dev else o for o in outs]
            for o, w in zip(got, (want, want_cos)):
                assert o.dtype == np.dtype(dtype)
                assert np.array_equal(o[:, :G].view(np.uint8), w.view(np.uint8)), (src_dev, dst_dev)
                assert (o[:, G:] == sentinel).all(), (src_dev, dst_dev)
            assert np.array_equal(W, want_w)


@pytest.mark.gpu
def test_moe_correct_repeats_bit_for_bit_over_slices(eng):
    X, R, Phi, Ainv = correction_inputs(8193, 70, 3, 3, np.float32, 31)
    assert moe_splits(8193) == 3
    a = correct(eng, X, R, Phi, Ainv, want_cos=True)
    b = correct(eng, X, R, Phi, Ainv, want_cos=True)
    for x, y in zip(a, b):
        assert np.array_equal(x.view(np.uint8), y.view(np.uint8))


def test_restatement_bound_holds_against_longdouble():
    """the float64 restatement's bound covers its own error against an all-long-double computation (CPU)"""
    X, R, Phi, Ainv = correction_inputs(65, 33, 4, 3, np.float64, 3, "signed")
    ref = Restatement(X, R, Phi, Ainv)
    z = X.astype(LD)
    for i in range(R.shape[0]):
        P = (Phi * R[i]).astype(LD)
        W = Ainv[i].astype(LD) @ (P @ X.astype(LD))
        W[0] = 0
        z = z - P.T @ W
    note("restatement vs long double", np.abs(ref.z - z).astype(np.float64), ref.ez)


# ---------------------------------------------------------------------------------------------------------- scaling
SCALE_N = [2, 3, 2047, 2048, 2049, 4097, 20000]
SCALE_G = [2, 31, 32, 33, 257]
CONSTANTS = [0.1, 1 / 3, 7.123, 1e-3, 2.7, 0.3, 1e4 + 0.1, 12.34, 5e-5, 0.7]


def scale_matrix(n, g, dtype, seed):
    """columns of every kind the moments have to reproduce: constant non-integer (whose variance cancels to a few ulps
    of either sign, or 0), all-zero, integer counts, negative, large mean with small variance, continuous, sparse,
    and a NaN entry"""
    rng = np.random.RandomState(seed)
    X = np.empty((n, g), dtype)
    for c in range(g):
        kind = (c + seed) % 8 if c else 0
        if kind == 0:
            X[:, c] = CONSTANTS[(c // 8 + seed) % len(CONSTANTS)]
        elif kind == 1:
            X[:, c] = 0
        elif kind == 2:
            X[:, c] = rng.poisson(1.5, n)
        elif kind == 3:
            X[:, c] = -rng.gamma(0.5, 2.0, n)
        elif kind == 4:
            X[:, c] = 1e4 + rng.rand(n)
        elif kind == 5:
            X[:, c] = rng.gamma(0.5, 2.0, n)
        elif kind == 6:
            X[:, c] = rng.gamma(0.5, 2.0, n) * (rng.rand(n) < 0.1)
        else:
            X[:, c] = rng.randn(n)
            X[rng.randint(n), c] = np.nan
    return X


def reference_scale(X, max_value=None):
    from oracle.refshim import AnnDataLite
    a = AnnDataLite(X.copy())
    with np.errstate(invalid="ignore", divide="ignore"):
        mg._scale(a, max_value=max_value)
    return a.X


def row_order_scale(X, max_value=None):
    """the kernel's scaling restated: per column one sequential fp64 chain for sum(x) and one for sum(x^2) in row
    order (cumsum is sequential), then the reference's formulas"""
    X64 = X.astype(np.float64)
    n = X.shape[0]
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        mean = np.cumsum(X64, axis=0)[-1] / n
        msq = np.cumsum(X64 * X64, axis=0)[-1] / n
        std = np.sqrt((msq - mean * mean) * (n / (n - 1)))
        std[std == 0] = 1
        Y = (X64 / std).astype(X.dtype)
        if max_value is not None:
            Y[Y > max_value] = max_value
    return Y


def same_bits(a, b):
    """equal values, NaN where NaN, and identical bits wherever not NaN (signed zeros included)"""
    if a.dtype != b.dtype or a.shape != b.shape or not np.array_equal(np.isnan(a), np.isnan(b)):
        return False
    m = ~np.isnan(a)
    u = np.uint32 if a.dtype == np.float32 else np.uint64
    return np.array_equal(a.view(u)[m], b.view(u)[m])


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_row_order_restatement_is_the_reference_scaling(dtype):
    """numpy sums a 2-D array over axis 0 row after row: the row-order restatement is the reference for G >= 2 (CPU),
    and on these columns the order decides NaN and ~1e8-scaled genes"""
    nans = 0
    for n in SCALE_N:
        for g in SCALE_G:
            X = scale_matrix(n, g, dtype, n + g)
            want = reference_scale(X)
            assert same_bits(row_order_scale(X), want), (n, g)
            nans += int(np.isnan(want[:, 0]).any())
    assert nans > 0             # some constant first column cancels to a negative variance


@pytest.mark.gpu
@pytest.mark.parametrize("n", SCALE_N)
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_scaling_is_the_reference_bit_for_bit(eng, n, dtype):
    from cnmf_b200.preprocess import scale_quantile_ceiling
    for g in SCALE_G:
        X = scale_matrix(n, g, dtype, n + g)
        for mv in (None, 2.5):
            out, t, _ = scale_quantile_ceiling(X, max_value=mv)
            assert t is None
            assert same_bits(out, reference_scale(X, mv)), (n, g, mv)


@pytest.mark.gpu
def test_constant_columns_match_the_reference(eng):
    """constant non-integer columns: the std is the rounding residue of msq - mean^2, so only the reference's summation
    order gives the reference's NaN, 1 or ~1e-8 std"""
    from cnmf_b200.preprocess import scale_quantile_ceiling
    for dtype in (np.float32, np.float64):
        for n in (40, 300, 1000, 2049, 4097, 10000):
            X = np.empty((n, len(CONSTANTS)), dtype)
            X[:] = np.array(CONSTANTS, dtype)
            out, _, _ = scale_quantile_ceiling(X)
            assert same_bits(out, reference_scale(X)), (np.dtype(dtype).name, n)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_single_column_scaling(eng, dtype):
    """G = 1: numpy sums one column pairwise, the kernel in row order.  Contract: the kernel's result is the row-order
    restatement bit for bit, and within the two summation orders' rounding of the reference: each sum within
    gamma(N) of the exact one, so |d var| <= f (2 gamma(N) msq + 4 gamma(N) |mean| mean|x| + 4 u (msq + mean^2)),
    f = N / (N - 1), |d std| / std <= |d var| / (2 var), and the output moves by that relative amount plus one rounding
    to X's type.  Below 8 rows numpy's pairwise sum is the row-order sum and the results are equal."""
    from cnmf_b200.preprocess import scale_quantile_ceiling
    u_t = U32 if dtype == np.float32 else U
    for n in (2, 3, 2049, 20000):
        rng = np.random.RandomState(n)
        for X in (rng.gamma(0.5, 2.0, (n, 1)).astype(dtype), rng.poisson(2.0, (n, 1)).astype(dtype),
                  (rng.randn(n, 1) - 3).astype(dtype)):
            out, _, _ = scale_quantile_ceiling(X)
            assert same_bits(out, row_order_scale(X)), n
            x = X.astype(np.float64)[:, 0]
            mean, msq, f = x.mean(), (x * x).mean(), n / (n - 1)
            var = (msq - mean * mean) * f
            dvar = f * (2 * gam(n) * msq + 4 * gam(n) * abs(mean) * np.abs(x).mean() + 4 * U * (msq + mean ** 2))
            want = reference_scale(X)
            if n < 8:
                assert same_bits(out, want)     # numpy's pairwise sum adds fewer than 8 terms in order
                continue
            assert var > 100 * dvar
            rel = dvar / (2 * var) * SECOND
            note("G = 1", np.abs(out - want.astype(np.float64))[:, 0],
                 np.abs(want[:, 0]) * (rel + 2 * u_t) * SECOND)


# ------------------------------------------------------------------------------------------------------------ select
def order_key(a):
    """the radix select's order-preserving unsigned key of each float"""
    if a.dtype == np.float32:
        u = a.view(np.uint32).astype(np.uint64)
        return np.where(u >> 31, ~u & 0xFFFFFFFF, u | 0x80000000), 32
    u = a.view(np.uint64)
    return np.where(u >> np.uint64(63), ~u, u | np.uint64(1 << 63)), 64


def select(eng, X, r_lo, r_hi=None, gamma=0.0):
    """cnmf_scale_quantile_ceiling with ranks k_lo, k_hi: (ceiled matrix, threshold)"""
    from cnmf_b200 import _lib
    X = np.ascontiguousarray(X)
    N, G = X.shape
    out = np.empty_like(X)
    t = ctypes.c_double()
    r_hi = r_lo if r_hi is None else r_hi
    _lib.check(eng.lib.cnmf_scale_quantile_ceiling(eng._h, ptr(X), 0 if X.dtype == np.float32 else 1, N, G, G, 0,
                                                   None, None, 0, 0.0, 0, r_lo, r_hi, gamma, ptr(out), G, 0,
                                                   ctypes.byref(t), None))
    return out, t.value


def small_select_matrix(dtype):
    """12 x 4: ties and +-0; subnormals next to values that keep the std near 1; near-1 values one ulp apart (float64:
    equal in their top 7 bytes) next to values that keep the std away from 0"""
    tiny = np.finfo(dtype).smallest_subnormal
    sub = [tiny, -tiny, 3 * tiny, 1000 * tiny, -1000 * tiny, 0.0, 4.0, -4.0, 4.0, 0.0, -0.0, 2.0]
    near = [1 + k * np.finfo(dtype).eps for k in range(1, 9)] + [8.0, -8.0, 1.0, 1.0]
    ties = [3.0, 3.0, 3.0, -3.0, 0.0, -0.0, 3.0, 1.0, 1.0, -3.0, -0.0, 0.0]
    neg = [-5.0, -1.5, -1.5, -2.5, 0.5, 7.0, -0.0, 0.0, -5.0, 2.0, 2.0, -9.0]
    return np.array([ties, sub, near, neg], dtype).T.copy()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_select_every_rank_of_a_small_matrix(eng, dtype):
    from cnmf_b200.preprocess import scale_quantile_ceiling
    X = small_select_matrix(dtype)
    scaled, _, _ = scale_quantile_ceiling(X)
    assert same_bits(scaled, reference_scale(X))
    v = scaled.reshape(-1)
    assert (v < 0).any() and (np.signbit(v) & (v == 0)).any() and (~np.signbit(v) & (v == 0)).any()
    assert ((v != 0) & (np.abs(v) < np.finfo(dtype).tiny)).sum() >= 3
    assert len(np.unique(v)) < v.size
    if dtype == np.float64:
        k = np.unique(order_key(v)[0])
        assert len(np.unique(k >> np.uint64(8))) < len(k)      # distinct values equal in their top 7 bytes
    s = np.sort(v)
    for r in range(v.size):
        out, t = select(eng, X, r)
        assert t == s[r], (r, t, s[r])
        assert same_bits(out, np.where(scaled > dtype(t), dtype(t), scaled)), r


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_select_at_ends_and_digit_edges(eng, dtype):
    """ranks 0, 1, n - 2, n - 1 and both sides of the first, middle and last bin edge of every 8-bit digit"""
    from cnmf_b200.preprocess import scale_quantile_ceiling
    rng = np.random.RandomState(17)
    X = (rng.randn(3000, 50) * rng.gamma(0.5, 2.0, (3000, 50))).astype(dtype)
    X[rng.rand(3000, 50) < 0.05] = 0
    scaled, _, _ = scale_quantile_ceiling(X)
    s = np.sort(scaled.reshape(-1))
    n = s.size
    keys, bits = order_key(s)
    ranks = {0, 1, n - 2, n - 1}
    for shift in range(bits - 8, -1, -8):
        edge = np.flatnonzero(np.diff(keys >> type(keys[0])(shift)) != 0) + 1
        for i in (edge[:1], edge[len(edge) // 2:len(edge) // 2 + 1], edge[-1:]):
            for e in i:
                ranks |= {int(e) - 1, int(e)}
    for r in sorted(ranks):
        _, t = select(eng, X, r)
        assert t == s[r], (r, t, s[r])
    lo, hi = n // 3, n // 3 + 1
    _, t = select(eng, X, lo, hi, 0.75)
    d = s[hi] - s[lo]
    assert t == s[hi] - d * dtype(0.25)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_nan_gives_nan_threshold_and_no_ceiling(eng, dtype):
    """np.quantile of values that include a NaN is NaN and `X[X > nan] = nan` changes nothing: a NaN in X, or a column
    whose variance cancels to a negative value, gives a NaN threshold and the scaled matrix unchanged"""
    from cnmf_b200.preprocess import scale_quantile_ceiling
    rng = np.random.RandomState(2)
    X = rng.gamma(0.5, 2.0, (300, 20)).astype(dtype)
    X[40, 3] = np.nan
    Y = rng.gamma(0.5, 2.0, (300, 20)).astype(dtype)
    Y[:, 5] = 0.1
    for M in (X, Y):
        scaled = reference_scale(M)
        assert np.isnan(scaled).any() and np.isnan(np.quantile(scaled, 0.9))
        for mv in (None, 2.0):
            out, t, _ = scale_quantile_ceiling(M, max_value=mv, quantile_thresh=0.9)
            assert np.isnan(t) and t.dtype == np.dtype(dtype)
            assert same_bits(out, reference_scale(M, mv))
        out, t = select(eng, M, 0)
        assert np.isnan(t) and same_bits(out, scaled)


def test_nan_constant_column_exists():
    """the constant columns of test_nan_gives_nan_threshold_and_no_ceiling give the reference a NaN std (CPU)"""
    for dtype in (np.float32, np.float64):
        X = np.full((300, 2), 0.1, dtype)
        X[:, 1] = np.arange(300)
        assert np.isnan(reference_scale(X)[:, 0]).all()


# --------------------------------------------------------------------------------------------------------------- CSR
def csr_counts(n, g, dtype, seed):
    """CSR counts with empty rows, explicit zeros and duplicate entries (summed as the dense form is)"""
    rng = np.random.RandomState(seed)
    rows, cols, vals = [], [], []
    for r in range(n):
        if r % 7 == 3:
            continue                                        # empty row
        m = rng.randint(1, g + 1)
        c = rng.randint(0, g, m)                            # repeats: duplicates
        v = rng.poisson(1.0, m)                             # zeros: explicit zeros
        rows += [r] * m
        cols += list(c)
        vals += list(v)
    order = np.lexsort((cols, rows))
    rows, cols, vals = np.array(rows)[order], np.array(cols)[order], np.array(vals)[order]
    indptr = np.concatenate([[0], np.cumsum(np.bincount(rows, minlength=n))])
    M = sp.csr_matrix((vals.astype(dtype), cols, indptr), shape=(n, g))
    assert (M.data == 0).any() and not M.has_canonical_format
    return M


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.int64, np.float32, np.float64])
@pytest.mark.parametrize("n,g", [(300, 40), (2049, 33)])
def test_csr_equals_dense_bit_for_bit(eng, dtype, n, g):
    from cnmf_b200.preprocess import scale_quantile_ceiling, stdscale_quantile_celing
    from oracle.refshim import AnnDataLite
    M = csr_counts(n, g, dtype, n + g)
    D = M.toarray()
    assert (D == 0).all(1).any()
    for mv, q in ((None, None), (2.0, None), (None, 0.99), (3.0, 0.5)):
        d, td, _ = scale_quantile_ceiling(D, max_value=mv, quantile_thresh=q)
        s, ts, csr = scale_quantile_ceiling(M.copy(), max_value=mv, quantile_thresh=q)
        assert csr is not None and same_bits(s, d) and (td is None or td == ts)
        if q is None:
            assert same_bits(d, reference_scale(D.astype(np.float64) if dtype == np.int64 else D, mv))
    a = AnnDataLite(M.copy())
    stdscale_quantile_celing(a, quantile_thresh=0.99)
    d, _, _ = scale_quantile_ceiling(D, quantile_thresh=0.99)
    assert sp.issparse(a.X) and np.array_equal(a.X.toarray(), d)
