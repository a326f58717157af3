"""What dataset creation leaves on the device (`-m gpu`), through the cnmf_dataset_form / cnmf_dataset_operand_host /
cnmf_dataset_gemm_host test hooks, against oracle/dataset_ref.py (the device's arithmetic restated in numpy, pinned by
tests/test_oracle_golden.py) and float64:

  * the operand form and both scale vectors of every precision, from host, from a strided device matrix and from CSC;
  * every resident array bit for bit, padding included, around the 32 x 32 transpose tile;
  * the derived datasets of cnmf_dataset_from_columns / cnmf_dataset_scale_rows;
  * both of the solver's products in both orientations and every scale kind (view_gemm, the solver's own launch);
  * datasets with more rows than one launch's grid.y covers (the transpose and the detection stride over row blocks).
"""
import math

import numpy as np
import pytest

from oracle import dataset_ref as dr

pytestmark = pytest.mark.gpu

TOL_GEMM = 2e-6          # fp32-class GEMM vs float64, as in test_kernel_units.py
PRECISIONS = ["fp32", "tf32x3", "tf32x3-general", "f16x2"]
ARRAYS = ["X", "Xt", "X_hi", "X_lo", "Xt_hi", "Xt_lo", "X_h16", "Xt_h16", "row_scale", "col_scale"]


@pytest.fixture(scope="module")
def eng():
    from cnmf_b200.engine import Engine
    return Engine(0)


def make(eng, X, precision, how):
    """The dataset of X created from host memory, from a device matrix with row stride ld > n_cols (the extra columns
    hold NaN: they must not be read) or from its CSC form."""
    X = np.ascontiguousarray(X, np.float32)
    if how == "host":
        return eng.dataset(X, precision)
    if how == "csc":
        import scipy.sparse as sp
        return eng.sparse_dataset(sp.csc_matrix(X), precision)
    import torch
    n, g = X.shape
    t = torch.full((n, g + 7), float("nan"), dtype=torch.float32, device="cuda")
    t[:, :g] = torch.from_numpy(X).cuda()
    torch.cuda.synchronize()
    return eng.dataset_from_device(t.data_ptr(), n, g, g + 7, precision)


# ------------------------------------------------------------------------------------------------ matrices
def counts(rng, n, g, lam=2.0, ones="row0"):
    """Poisson counts; ones='row0' puts a 1 in every column (the column scale is the column's scale), 'col0' a 1 in
    every row, 'both' both."""
    C = rng.poisson(lam, (n, g)).astype(np.float32)
    if ones in ("row0", "both"):
        C[0, :] = 1
    if ones in ("col0", "both"):
        C[:, 0] = 1
    return C


def col_scaled(rng, n, g, spread=1.0):
    C = counts(rng, n, g, ones="row0")
    cs = (10.0 ** rng.uniform(-spread, spread, g)).astype(np.float32)
    return (C * cs[None, :]).astype(np.float32)


def row_scaled(rng, n, g):
    C = counts(rng, n, g, ones="col0")
    return (C * (np.float32(1e6) / C.sum(axis=1, keepdims=True))).astype(np.float32)


def form_cases():
    rng = np.random.RandomState(11)
    n, g = 37, 45
    cases = {
        "col_scaled": col_scaled(rng, n, g),
        "row_scaled_tpm": row_scaled(rng, n, g),
        "integers": counts(rng, n, g),
        "general": rng.uniform(0.1, 3.0, (n, g)).astype(np.float32),
    }
    C = counts(rng, n, g, ones="both")
    for top in (2048, 2049):
        M = C.copy()
        M[5, 9] = top
        cases["max_%d" % top] = M
    cs = (10.0 ** rng.uniform(-1, 1, g)).astype(np.float32)
    base = (C * cs).astype(np.float32)
    base[7, 3] = np.float32(1000.0) * cs[3]
    for rel in (3e-7, 8e-7):
        M = base.copy()
        M[7, 3] = np.float32(1000.0 * (1.0 + rel) * np.float64(cs[3]))
        cases["perturbed_%g" % rel] = M
    for name, v in (("negative", -1.0), ("nan", np.nan), ("inf", np.inf), ("subnormal", 1e-40)):
        M = C.copy()
        M[3, 4] = v
        cases[name] = M
    M = col_scaled(rng, n, g)
    M[[2, 30], :] = 0
    M[:, [0, 17, 44]] = 0
    cases["zero_lines"] = M
    cases["zeros"] = np.zeros((n, g), np.float32)
    cases["1x1"] = np.float32([[3.5]])
    cases["1xn"] = col_scaled(rng, 1, 70)
    cases["nx1"] = row_scaled(rng, 70, 1)
    return cases


FORM_CASES = form_cases()


def check_form_and_scales(ds, X, precision):
    form, rs, cs = dr.decide(X, precision)
    assert ds.form == form
    for name, want in (("row_scale", rs), ("col_scale", cs)):
        got = ds.operand(name)
        if want is None:
            assert got is None, name
        else:
            assert got is not None and got.view(np.uint32).tolist() == want.view(np.uint32).tolist(), name
    return form, rs, cs


@pytest.mark.parametrize("how", ["host", "device", "csc"])
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("case", list(FORM_CASES))
def test_form_and_scales(eng, case, precision, how):
    """Form and both scale vectors equal the restatement bit for bit: the column scale is tried first, then the row
    scale; fp32 and tf32x3-general never detect; a count of 2049, an entry 8e-7 n off an integer, a negative, NaN or
    infinite entry take the general form; a line without a positive entry has scale 1 and padding is 0.  The dense and
    CSC forms of a matrix give the same dataset form and scales."""
    X = FORM_CASES[case]
    ds = make(eng, X, precision, how)
    check_form_and_scales(ds, X, precision)
    if how == "csc":
        assert not ds.exact
    else:
        assert ds.exact == (ds.form in ("tf32_exact", "f16_exact"))
        assert ds.f16 == (ds.form == "f16_exact")


# ------------------------------------------------------------------------------------------------ resident operands
SHAPES = [(31, 33), (32, 32), (33, 31), (63, 65), (64, 64), (65, 63), (1000, 33), (33, 1000), (1, 65), (65, 1)]


def operand_matrix(kind, n, g):
    rng = np.random.RandomState(n * 1009 + g)
    if kind == "col_scaled":
        return col_scaled(rng, n, g)
    if kind == "row_scaled":
        return row_scaled(rng, n, g) if g > 1 else col_scaled(rng, n, g)
    X = rng.uniform(0.0, 5.0, (n, g)).astype(np.float32)
    X[rng.rand(n, g) < 0.3] = 0
    return X


def check_operands(ds, want):
    for name in ARRAYS:
        got = ds.operand(name)
        if name not in want:
            assert got is None, "%s is held but the form has no such array" % name
            continue
        w = want[name]
        assert got is not None and got.shape == w.shape, name
        bits = np.uint16 if w.dtype == np.float16 else np.uint32
        assert np.array_equal(got.view(bits), w.view(bits)), name


def check_sums(ds, X):
    s, q = ds.sums()
    x = X.astype(np.float64).ravel()
    m = x.size
    ref_s, ref_q, abs_s = math.fsum(x), math.fsum(x * x), math.fsum(np.abs(x))
    assert abs(s - ref_s) <= m * 2.0 ** -53 * abs_s
    assert abs(q - ref_q) <= m * 2.0 ** -53 * ref_q


def check_admission(want, X):
    """rs C cs represents X within the admission bound: 5e-7 |x| plus the rounding of the quotient and of the scale
    product (2^-24 each)."""
    C = (want["X_hi"] if "X_hi" in want else want["X_h16"]).astype(np.float64)[:, :X.shape[1]]
    n, g = X.shape
    rs = want["row_scale"][:n].astype(np.float64)[:, None] if "row_scale" in want else 1.0
    cs = want["col_scale"][:g].astype(np.float64)[None, :] if "col_scale" in want else 1.0
    x = X.astype(np.float64)
    assert (np.abs(rs * C * cs - x) <= (5e-7 + 2.0 ** -23) * np.abs(x)).all()


@pytest.mark.parametrize("how", ["host", "device"])
@pytest.mark.parametrize("kind", ["col_scaled", "row_scaled", "general"])
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "%dx%d" % s)
def test_resident_operands(eng, shape, precision, kind, how):
    """Every array the dataset holds, padding included, bit for bit: X and X^T (fp32), the tf32 hi / lo pieces of X
    and of X^T (X^T's pieces are the transpose of X's), C and C^T of the exact forms (F16_EXACT: only their fp16
    copies; the fp32 ones are released); every padding row and column exactly 0; no array the form does not use.
    Exact forms: rs C cs represents X within the admission bound.  sum / sum_sq within (entries) 2^-53 of float64."""
    n, g = shape
    X = operand_matrix(kind, n, g)
    ds = make(eng, X, precision, how)
    form, rs, cs = check_form_and_scales(ds, X, precision)
    want = dr.operands(X, form, rs, cs)
    check_operands(ds, want)
    if form in ("tf32_exact", "f16_exact"):
        check_admission(want, X)
    check_sums(ds, X)


# ------------------------------------------------------------------------------------------------ derived datasets
def derived_sources():
    rng = np.random.RandomState(5)
    n, g = 70, 41
    return {"general": rng.uniform(0.1, 2.0, (n, g)).astype(np.float32), "col_scaled": col_scaled(rng, n, g),
            "row_scaled": row_scaled(rng, n, g)}


DERIVED = derived_sources()


@pytest.mark.parametrize("precision", ["tf32x3", "f16x2", "fp32"])
@pytest.mark.parametrize("source", list(DERIVED))
def test_from_columns(eng, source, precision):
    """from_columns (the HVG refit's tpm[:, hvgs] / std) with repeated and reversed columns: X = fl(X[:, cols] *
    scale); an exact source stays exact with the source's C columns bit for bit, the row scale kept and the column
    scale fl(scale[c] * src_cs[cols[c]]); a general source is detected afresh.  The dense-derived and the CSC-derived
    datasets hold the same bits in every array."""
    X = DERIVED[source]
    n, g = X.shape
    cols = np.array([g - 1, 3, 3, 0, 17, 16, 15, 14, 40, 2, 2, 39], np.int32)
    rng = np.random.RandomState(9)
    scale = (1.0 / rng.uniform(0.5, 3.0, len(cols))).astype(np.float32)
    Xd = (X[:, cols] * scale[None, :]).astype(np.float32)
    out = {}
    for how in ("host", "csc"):
        src = make(eng, X, precision, how)
        sform, srs, scs = check_form_and_scales(src, X, precision)
        d = src.from_columns(cols, scale)
        exact = sform in ("tf32_exact", "f16_exact")
        if exact:
            assert d.form == sform
            ld_c = dr.pad_ld(len(cols))
            cs = dr.combine_scale(scale, scs, cols, ld_c)
            want = dr.operands(Xd, sform, srs, cs)
            C_src = dr.counts(X, srs, scs)[:, :g]
            C_new = (want["X_hi"] if "X_hi" in want else want["X_h16"].astype(np.float32))[:, :len(cols)]
            assert np.array_equal(C_new, C_src[:, cols]), "derived C is not the source's columns"
            check_admission(want, Xd)
        else:
            form, rs, cs = dr.decide(Xd, precision)
            want = dr.operands(Xd, form, rs, cs)
            assert d.form == form
        check_operands(d, want)
        out[how] = {name: d.operand(name) for name in ARRAYS}
    for name in ARRAYS:
        a, b = out["host"][name], out["csc"][name]
        assert (a is None) == (b is None), name
        if a is not None:
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), name


@pytest.mark.parametrize("precision", ["tf32x3", "f16x2"])
def test_scale_rows_is_detected_as_row_scaled(eng, precision):
    """scale_rows of counts by 1e6 / total (TPM made on the device) is detected again, from scratch, as row-scaled."""
    rng = np.random.RandomState(4)
    C = counts(rng, 90, 50, ones="col0")
    rs = (np.float32(1e6) / C.sum(axis=1)).astype(np.float32)
    t = eng.dataset(C, precision).scale_rows(rs)
    T = (C * rs[:, None]).astype(np.float32)
    form, r, c = check_form_and_scales(t, T, precision)
    assert r is not None and c is None and form in ("tf32_exact", "f16_exact")
    check_operands(t, dr.operands(T, form, r, c))


# ------------------------------------------------------------------------------------------------ both products
def splits_of(Kd, f16):
    bke = 64 if f16 else 32
    return max(1, min(16, (-(-Kd // bke) + 63) // 64))


def effective_matrix(ds, X):
    """float64 matrix the products multiply: rs C cs on the exact forms (from the device's own C and scales), X
    otherwise."""
    n, g = X.shape
    if ds.form not in ("tf32_exact", "f16_exact"):
        return X.astype(np.float64)
    C = ds.operand("X_hi") if ds.form == "tf32_exact" else ds.operand("X_h16")
    M = C.astype(np.float64)[:, :g]
    rs, cs = ds.operand("row_scale"), ds.operand("col_scale")
    if rs is not None:
        M = M * rs[:n].astype(np.float64)[:, None]
    if cs is not None:
        M = M * cs[:g].astype(np.float64)[None, :]
    return M


def check_products(ds, X, sks, f16, seed):
    """Every (transposed, side) against float64, per row within 4 TOL_GEMM of the magnitude product (non-negative
    factors: the product itself), and per entry within (2^-20 + 2 (Kd + 2) 2^-24) of it: the factor's pieces carry 22
    significant bits, any order of Kd fp32 additions of non-negative terms is within (Kd - 1) u of their sum, and the
    output scale is one more rounding; 2 u per addition leaves room for the tensor cores' accumulator.  Per entry, so
    that an error confined to the output columns of small scale is not hidden behind the row norm.  The split count
    is the solver's plan for the reduction length."""
    M = effective_matrix(ds, X)
    n, g = X.shape
    rng = np.random.RandomState(seed)
    worst = 0.0
    for transposed in (False, True):
        for side in (0, 1):
            use_t = (side == 0) != transposed           # out = F @ M^T, else F @ M
            Kd = g if use_t else n
            F = rng.uniform(0.05, 1.0, (max(sks), Kd)).astype(np.float32)
            ref = F.astype(np.float64) @ (M.T if use_t else M)
            for sk in sks:
                sl = ds.gemm(F[:sk], side, transposed)
                assert sl.shape[0] == splits_of(Kd, f16), (transposed, side, sl.shape)
                out = sl.astype(np.float64).sum(axis=0)
                err = np.linalg.norm(out - ref[:sk], axis=1) / np.linalg.norm(ref[:sk], axis=1)
                assert np.isfinite(out).all()
                worst = max(worst, float(err.max()))
                assert err.max() <= 4 * TOL_GEMM, (transposed, side, sk, err.max())
                entry = (2.0 ** -20 + 2 * (Kd + 2) * 2.0 ** -24) * ref[:sk]
                assert (np.abs(out - ref[:sk]) <= entry).all(), (transposed, side, sk)
    return worst


def gemm_matrix(kind, n, g, rng):
    """none: integers (unit scales); col: column scales 1e-6 .. 1e6 inside every 512-column group; row: TPM-like row
    scales; both: the row-scaled matrix times column scales (from_columns of the row-scaled dataset)."""
    if kind == "none":
        return counts(rng, n, g, lam=1.0, ones="both")
    if kind == "col":
        return col_scaled(rng, n, g, spread=6.0)
    return row_scaled(rng, n, g)


GEMM_SHAPE = {"fp32": (2048, 2049), "tf32x3": (2048, 2049), "tf32x3-general": (2048, 2049), "f16x2": (4096, 4097)}


@pytest.mark.parametrize("kind", ["none", "col", "row", "both"])
@pytest.mark.parametrize("precision", PRECISIONS)
def test_products_every_orientation(eng, precision, kind):
    """Both of the solver's products (view_gemm) in both orientations at SK = 1, 7, 33, 129, 193, on reduction lengths
    either side of a split-plan change (2 048 / 2 049; f16: 4 096 / 4 097), against float64 F (rs C cs)^T (exact forms)
    or F X^T (general forms)."""
    rng = np.random.RandomState(PRECISIONS.index(precision) * 10 + len(kind))
    n, g = GEMM_SHAPE[precision]
    X = gemm_matrix(kind, n, g, rng)
    ds = eng.dataset(X, precision)
    if kind == "both":
        cs = (10.0 ** rng.uniform(-6, 6, g)).astype(np.float32)
        ds = ds.from_columns(np.arange(g, dtype=np.int32), cs)
        X = (X * cs[None, :]).astype(np.float32)
    form = ds.form
    if precision in ("tf32x3", "f16x2"):
        assert form == ("f16_exact" if precision == "f16x2" else "tf32_exact")
        if kind == "both":
            assert ds.operand("row_scale") is not None and ds.operand("col_scale") is not None
    check_products(ds, X, [1, 7, 33, 129, 193], precision == "f16x2", seed=n + g)


@pytest.mark.parametrize("precision", ["tf32x3", "f16x2"])
def test_products_scale_orientation(eng, precision):
    """A dataset with both scales, each spanning 1e-6 .. 1e6, in both orientations: a row scale applied where the
    column scale belongs (or either one dropped) is off by orders of magnitude, not by a rounding.  Square, so that
    both scale vectors have the same length."""
    rng = np.random.RandomState(2)
    n = g = 300
    C = counts(rng, n, g, lam=1.0, ones="both")
    rs = (10.0 ** rng.uniform(-6, 6, n)).astype(np.float32)
    cs = (10.0 ** rng.uniform(-6, 6, g)).astype(np.float32)
    T = (C * rs[:, None]).astype(np.float32)
    ds = eng.dataset(T, precision).from_columns(np.arange(g, dtype=np.int32), cs)
    X = (T * cs[None, :]).astype(np.float32)
    assert ds.operand("row_scale") is not None and ds.operand("col_scale") is not None
    check_products(ds, X, [1, 33], precision == "f16x2", seed=7)


def test_products_need_a_dense_float_dataset(eng):
    """The product hook refuses datasets the solver runs no tensor-core product on: float64 (gemm_f64 runs those), and
    on sparse (CSC) datasets every product but the transposed refit's one (transposed, side 0, SK <= 32), which it runs
    through csc_project in one slice."""
    from cnmf_b200._lib import CnmfError
    X = counts(np.random.RandomState(3), 40, 30)
    with pytest.raises(CnmfError):
        eng.dataset(X, "fp64").gemm(np.ones((2, 30), np.float32), 0)
    ds = make(eng, X, "tf32x3", "csc")
    for transposed, side, sk in ((False, 0, 2), (False, 1, 2), (True, 1, 2), (True, 0, 33)):
        n_r, n_c = (30, 40) if transposed else (40, 30)
        with pytest.raises(CnmfError, match="sparse"):
            ds.gemm(np.ones((sk, n_c if side == 0 else n_r), np.float32), side, transposed)
    F = np.random.RandomState(4).uniform(0.1, 1.0, (3, 40)).astype(np.float32)
    sl = ds.gemm(F, 0, transposed=True)
    assert sl.shape == (1, 3, 30)
    assert np.allclose(sl[0], F.astype(np.float64) @ X, rtol=1e-6, atol=0)


# ------------------------------------------------------------------------------------------------ row limits
def last_strip_counts(rng, n, g):
    """Column-scaled counts whose every column has its smallest count (1) only in the last row; every other count is
    even, so a column minimum taken without the last row (2 cs) gives another, wrong, exact dataset."""
    C = (2 * rng.poisson(1.0, (n, g)) + 2).astype(np.float32)
    C[-1, :] = 1
    cs = (10.0 ** rng.uniform(-1, 1, g)).astype(np.float32)
    return (C * cs[None, :]).astype(np.float32)


@pytest.mark.parametrize("kind", ["row_scaled", "col_min_in_last_row"])
@pytest.mark.parametrize("precision", ["tf32x3", "f16x2"])
@pytest.mark.parametrize("n_rows", [65535 * 32 + 1, 65535 * 64 + 1])
def test_more_rows_than_one_grid_column(eng, n_rows, precision, kind):
    """Count datasets with more rows than 65 535 transpose tiles (2 097 121) and than 65 535 detection strips
    (4 194 241), on data where the last rows decide the scales: TPM (every row's minimum makes its row scale, the last
    strip's included) and column-scaled counts whose column minima lie only in the last row (4 194 240 is the one row
    of strip 65 535).  Created, detected as exact with the restatement's scales, C and C^T equal to the restatement
    (C on sampled rows around the block boundaries, C^T in full) and C^T's padding zero."""
    g = 8
    rng = np.random.RandomState(n_rows % 977)
    X = row_scaled(rng, n_rows, g) if kind == "row_scaled" else last_strip_counts(rng, n_rows, g)
    ds = eng.dataset(X, precision)
    form, rs, cs = dr.decide(X, precision)
    assert form == ("f16_exact" if precision == "f16x2" else "tf32_exact")
    assert (rs is not None) == (kind == "row_scaled") and (cs is not None) == (kind != "row_scaled")
    assert ds.form == form
    for name, want in (("row_scale", rs), ("col_scale", cs)):
        got = ds.operand(name)
        assert (got is None) == (want is None), name
        if want is not None:
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), name
    C = dr.counts(X, rs, cs)
    f16 = precision == "f16x2"
    got = ds.operand("X_h16" if f16 else "X_hi").astype(np.float32)
    gott = ds.operand("Xt_h16" if f16 else "Xt_hi").astype(np.float32)
    edges = [0, 1, 31, 32, 65535 * 32 - 1, 65535 * 32, 65535 * 32 + 1, 65535 * 64 - 1, 65535 * 64, n_rows - 1]
    rows = np.unique(np.concatenate([[r for r in edges if r < n_rows], rng.randint(0, n_rows, 4000)]))
    assert np.array_equal(got[rows], C[rows])
    assert not gott[:, n_rows:].any()
    assert np.array_equal(gott[:, :n_rows], C[:, :g].T)
