"""The sparse (CSC) kernels and both OLS projections one launch at a time (`-m gpu`), against extended precision:

  * csc_project_kernel + csc_project_reduce_kernel through project_rows on a sparse dataset, at every k from 1 to 32
    (strand widths G = kp / 4 = 1 ... 8, including 3, 5, 6 and 7, where 32 is not a multiple of G and the top lanes
    idle), at column lengths around every strand count and every 4 096-entry chunk, with more chunk items than one grid
    pass covers, and with planted cancellation in the signed product;
  * the transposed refit's staged product (stage_rows from the strided factor, csc_project into NUM_r at stride ld_r)
    through cnmf_dataset_gemm_host, at every k;
  * csc_col_stats_kernel / csc_totals_kernel, and the three tpm_stats kernels at every slab-count regime;
  * the dense projection cnmf_project_rows in every operand form, on both sides of its split plan's cap.

u = 2^-53 is the unit roundoff of float64.  The references run in np.longdouble (unit roundoff UL = 2^-64 on x86-64)
where the kernel accumulates in fp64; each CSC sum is np.add.reduceat over the exact fp64 products (fp32 x fp32 is exact
in fp64).  Every bound adds the reference's own error, n UL per n-term sum.  Every matrix comes from a seed here.
"""
import numpy as np
import pytest
import scipy.sparse as sp

pytestmark = pytest.mark.gpu

U = 2.0 ** -53
U32 = 2.0 ** -24
LD = np.longdouble
UL = 2.0 ** -(np.finfo(LD).nmant + 1)
SECOND = 1 + 2.0 ** -10          # second-order terms, relative to a first-order bound
CHUNK = 4096                     # CSC_CHUNK: entries per chunk item of csc_project_kernel
WARPS = 8                        # warps per block of the warp-per-column / warp-per-chunk kernels
TPM_SLABS = 128

RATIOS = {}
NOT_NEAREST = {}


@pytest.fixture(scope="module")
def eng():
    from cnmf_b200.engine import Engine
    return Engine(0)


@pytest.fixture(scope="module")
def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module", autouse=True)
def report_ratios():
    """Largest error-to-bound ratio seen per check, printed after the module (visible with -s)."""
    yield
    for k in sorted(RATIOS):
        print("ratio %-22s %.3g" % (k, RATIOS[k]))
    for k in sorted(NOT_NEAREST):
        print("not nearest %-16s %d" % (k, NOT_NEAREST[k]))


def ratio(err, bound):
    err, bound = np.asarray(err, np.float64), np.asarray(bound, np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.where(bound > 0, err / bound, np.where(err > 0, np.inf, 0.0))
    return float(q.max()) if q.size else 0.0


def note(key, r):
    RATIOS[key] = max(RATIOS.get(key, 0.0), r)
    assert r <= 1.0, (key, r)


def csc(n_rows, cols):
    """canonical CSC from a list of (rows, values) per column"""
    lens = np.array([len(r) for r, _ in cols], np.int64)
    col_ptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    idx = np.concatenate([np.asarray(r, np.int32) for r, _ in cols] + [np.zeros(0, np.int32)])
    val = np.concatenate([np.asarray(v, np.float32) for _, v in cols] + [np.zeros(0, np.float32)])
    M = sp.csc_matrix((val, idx, col_ptr), shape=(n_rows, len(cols)))
    M.has_sorted_indices = True
    return M


def col_sums(M, terms):
    """per-column longdouble sums of `terms` (one per stored entry, in CSC order); empty columns give 0"""
    starts = M.indptr[:-1]
    t = np.concatenate([np.asarray(terms, LD), np.zeros((1,) + np.shape(terms)[1:], LD)])
    out = np.add.reduceat(t, np.minimum(starts, M.nnz), axis=0)
    out[np.diff(M.indptr) == 0] = 0
    return out


# ------------------------------------------------------------------------------------------------ A / B: csc_project
H = 8200                  # rows [0, H): signed random U; [H, 2H): -U of the first block
D = 2100                  # rows [2H, 2H + D): small integers; [2H + D, 2H + 2D): their negatives
EXTRA = 7                 # rows of the residual entries; n_rows = 20 607, not a multiple of 32 (the factor's ld is)
N_ROWS = 2 * H + 2 * D + EXTRA
P_COUNTS = (32, 16, 10, 8, 6, 5, 4)      # strands per warp, 32 // G, for G = 1 ... 8
LENGTHS = sorted({0, 1} | {p + d for p in P_COUNTS for d in (-1, 0, 1)}
                 | {4095, 4096, 4097, 8192, 8193, 3 * CHUNK + 1})


def strands(k):
    return 32 // (((k + 3) // 4 * 4) // 4)


@pytest.fixture(scope="module")
def proj(sm_count):
    """One n_rows x G CSC matrix and the signed n_rows x 32 factor whose first k columns are U for every k:
      * a column of every length in LENGTHS (0, 1, P - 1, P, P + 1 for every strand count, one to four chunks), positive
        lognormal values over six decades, rows from the signed block;
      * exact cancellation: pairs (r, r + D) of the integer block with equal integer values, 1, 16 and 2 049 pairs (the
        last crosses a chunk).  Every product and partial sum is an integer below 2^53, so the kernel's sum is 0;
      * planted cancellation: pairs (r, r + H) with equal values (their products cancel exactly) and one residual entry
        of a tiny value, so that the true sum is >= 2^20 times smaller than sum |u x|;
      * more non-empty columns than the grid's 8 * 16 * sm_count warps cover in one pass, and an empty last column."""
    rng = np.random.RandomState(20)
    Uf = np.zeros((N_ROWS, 32), np.float32)
    Uf[:H] = rng.randn(H, 32).astype(np.float32) * np.float32(10.0) ** rng.uniform(-2, 2, (H, 1)).astype(np.float32)
    Uf[H:2 * H] = -Uf[:H]
    Uf[2 * H:2 * H + D] = rng.randint(-100, 101, (D, 32))
    Uf[2 * H + D:2 * H + 2 * D] = -Uf[2 * H:2 * H + D]
    Uf[2 * H + 2 * D:] = rng.randn(EXTRA, 32)
    U64 = Uf.astype(np.float64)
    cols, kinds = [], []

    def add(rows, vals, kind):
        o = np.argsort(rows)
        cols.append((np.asarray(rows)[o], np.asarray(vals, np.float32)[o]))
        kinds.append(kind)

    for m in LENGTHS:
        add(rng.choice(2 * H, m, replace=False), 10.0 ** rng.uniform(-3, 3, m), "length")
    for p in (1, 16, 2049):
        r = rng.choice(D, p, replace=False) + 2 * H
        v = rng.randint(1, 41, p)
        add(np.concatenate([r, r + D]), np.concatenate([v, v]), "exact")
    for i, p in enumerate((4, 50, 300)):
        r = rng.choice(H, p, replace=False)
        v = (10.0 ** rng.uniform(-1, 1, p)).astype(np.float32)
        e = 2 * H + 2 * D + i
        mag = (np.abs(U64[r]) * v[:, None].astype(np.float64)).sum(axis=0) * 2       # sum |u x| per component
        x0 = np.float32(2.0 ** -21 * mag.min() / np.abs(U64[e]).max())
        add(np.concatenate([r, r + H, [e]]), np.concatenate([v, v, [x0]]), "residual")
    n_short = WARPS * 16 * sm_count + 2000
    starts = rng.randint(0, 2 * H - 3, n_short)
    lens = rng.randint(1, 4, n_short)
    for s, m in zip(starts, lens):
        add(s + np.arange(m), 10.0 ** rng.uniform(-3, 3, m), "short")
    add([], [], "length")
    M = csc(N_ROWS, cols)
    kinds = np.array(kinds)
    items = int((-(-np.diff(M.indptr) // CHUNK)).sum())
    assert items > WARPS * 16 * sm_count                 # the grid-stride loop takes a second pass
    return dict(M=M, U=Uf, kinds=kinds, items=items)


@pytest.fixture(scope="module")
def proj_ds(eng, proj):
    ds = eng.sparse_dataset(proj["M"])
    assert ds.sparse and ds.shape == proj["M"].shape
    yield ds
    ds.close()


def project_reference(M, Uk):
    """exact sum and sum |u x| per (component, column) in longdouble: k x G each"""
    prod = Uk.astype(np.float64)[M.indices] * M.data.astype(np.float64)[:, None]     # exact in fp64
    return col_sums(M, prod).T, col_sums(M, np.abs(prod)).T


def check_projection(key, out, M, Uk, kinds):
    """out (k x G, fp32) against the exact sum s per entry.  The kernel: strand t of P sums the products of its
    entries of one chunk in fp64 FMAs from 0 (the first exact, one rounding per later entry), the P strand partials are
    added in order from 0, the chunk partials of the column in order from 0, and the result is rounded to fp32 once.
    Every product is exact, so each term of sum |u x| reaches the fp64 result through at most m + P + chunks
    roundings (m the column's entry count), and the longdouble reference adds m UL:
        |t - s| <= eps = ((m + P + chunks + 1) u + m UL) sum |u x|.
    Rounding to nearest is monotone, so out = fl32(t) lies in [fl32(s - eps), fl32(s + eps)]: one of the two fp32
    neighbours of s, and the nearest one unless s lies within eps of their midpoint.  With fp32 accumulators the error
    is ~m 2^-24 sum |u x|, far outside.  The exactly cancelling integer columns give exactly 0."""
    k = Uk.shape[1]
    s, S = project_reference(M, Uk)
    m = np.diff(M.indptr)[None, :].astype(np.float64)
    chunks = -(-m // CHUNK)
    eps = ((m + strands(k) + chunks + 1) * U + m * UL) * S.astype(np.float64) * SECOND
    lo = (s - eps.astype(LD)).astype(np.float32)
    hi = (s + eps.astype(LD)).astype(np.float32)
    assert np.isfinite(out).all()
    bad = (out < lo) | (out > hi)
    assert not bad.any(), (key, k, np.argwhere(bad)[:5])
    nearest = s.astype(np.float32)
    NOT_NEAREST[key] = NOT_NEAREST.get(key, 0) + int((out != nearest).sum())
    assert not out[:, kinds == "exact"].any()
    assert not out[:, np.diff(M.indptr) == 0].any()
    res = kinds == "residual"
    assert (S[:, res] >= 2.0 ** 20 * np.abs(s[:, res])).all()        # the planted cancellation is as deep as claimed


@pytest.mark.parametrize("k", list(range(1, 33)))
def test_csc_project_every_k(proj, proj_ds, k):
    """project_rows on the sparse dataset at k (strand width G = ceil(k / 4)): per entry as check_projection, twice
    with the same bits."""
    Uk = proj["U"][:, :k]
    out = proj_ds.project_rows(np.ascontiguousarray(Uk.T))
    check_projection("csc_project", out, proj["M"], Uk, proj["kinds"])
    assert np.array_equal(out, proj_ds.project_rows(np.ascontiguousarray(Uk.T)))


@pytest.mark.parametrize("k", list(range(1, 33)))
def test_refit_product_every_k(proj, proj_ds, k):
    """The transposed refit's product as cnmf_refit issues it (the factor at stride ld_rows staged by stage_rows,
    csc_project into the zeroed NUM_r at stride ld_cols, one slice), through cnmf_dataset_gemm_host: per entry as
    check_projection.  n_rows is not a multiple of 32, so a factor read at stride n_rows instead of ld shifts every
    component after the first."""
    Uk = proj["U"][:, :k]
    sl = proj_ds.gemm(np.ascontiguousarray(Uk.T), 0, transposed=True)
    assert sl.shape == (1, k, proj["M"].shape[1])
    check_projection("refit_product", sl[0], proj["M"], Uk, proj["kinds"])
    assert np.array_equal(sl, proj_ds.gemm(np.ascontiguousarray(Uk.T), 0, transposed=True))


def test_csc_project_edges(eng):
    """nnz = 0 gives exact zeros; k = 33 is refused on a sparse dataset; the product hook refuses every combination
    but the transposed refit's product, and SK > 32."""
    from cnmf_b200._lib import CnmfError
    ds = eng.sparse_dataset(sp.csc_matrix((37, 45), dtype=np.float32))
    Ut = np.random.RandomState(1).randn(32, 37).astype(np.float32)
    for k in (1, 5, 32):
        out = ds.project_rows(Ut[:k])
        assert out.shape == (k, 45) and not out.any()
    with pytest.raises(CnmfError, match="k must be <= 32 on a sparse dataset"):
        ds.project_rows(np.ones((33, 37), np.float32))
    ds.close()
    M = csc(40, [(np.arange(3), np.ones(3))] * 30)
    ds = eng.sparse_dataset(M)
    for transposed, side, sk in ((False, 0, 2), (False, 1, 2), (True, 1, 2), (True, 0, 33)):
        with pytest.raises(CnmfError, match="sparse"):
            n_c = 40 if transposed else 30
            n_r = 30 if transposed else 40
            ds.gemm(np.ones((sk, n_c if side == 0 else n_r), np.float32), side, transposed)
    assert ds.gemm(np.ones((2, 40), np.float32), 0, transposed=True).shape == (1, 2, 30)
    ds.close()


# ------------------------------------------------------------------------------------------------ C: column statistics
def lane_depth(m):
    """roundings on the way of one term of a warp-per-column sum: lane strides of 32 (ceil(m / 32) terms from 0, the
    first exact) then the 5-level xor tree"""
    return -(-np.asarray(m, np.float64) // 32) + 5


@pytest.mark.parametrize("n_cols", [253, 255, 256, 257])
def test_csc_col_stats(eng, n_cols):
    """col_stats and sums on CSC: columns of 0, 1, 31, 32, 33 and 4 097 entries, then random lengths, signed values.
    Per column the kernel's Sigma x and Sigma x^2 (FMA: v^2 is exact in fp64, one rounding per step) carry
    d = ceil(m / 32) + 5 roundings per term; mean = s / n is one more, variance = fl(fl(q / n) - fl(m^2)) adds one
    rounding of q / n, 2 (d + 1) + 1 of m^2 and one of the difference: (2 d + 5) u (q / n + m^2).  The dataset
    totals (csc_totals_kernel) add the column sums at thread strides of 256 and in an 8-level tree:
    (max d + ceil(G / 256) + 8) u sum |x|."""
    rng = np.random.RandomState(n_cols)
    n = 5000
    lens = [0, 1, 31, 32, 33, 4097] + list(rng.randint(0, 81, n_cols - 6))
    cols = [(np.sort(rng.choice(n, m, replace=False)),
             rng.choice([-1.0, 1.0], m) * 10.0 ** rng.uniform(-3, 3, m)) for m in lens]
    M = csc(n, cols)
    ds = eng.sparse_dataset(M)
    x = M.data.astype(np.float64)
    s, q, a = col_sums(M, x), col_sums(M, x * x), col_sums(M, np.abs(x))
    m = np.diff(M.indptr)
    d = lane_depth(m)
    mean, var = ds.col_stats()
    m_ref = s / n
    note("col_stats.mean", ratio(np.abs(mean - m_ref), ((d + 1) * U + m * UL) * (a / n) * SECOND))
    v_ref = q / n - m_ref ** 2
    note("col_stats.var", ratio(np.abs(var - v_ref), ((2 * d + 5) * U + m * UL) * (q / n + m_ref ** 2) * SECOND))
    tot, tot_sq = ds.sums()
    depth = d.max() + -(-n_cols // 256) + 8
    note("csc_totals.sum", ratio(abs(tot - s.sum()), (depth * U + M.nnz * UL) * a.sum() * SECOND))
    note("csc_totals.sq", ratio(abs(tot_sq - q.sum()), (depth * U + M.nnz * UL) * q.sum() * SECOND))
    ds.close()


def slab_plan(M):
    """csc_tpm_sums' slab count and csc_row_partials_kernel's column range per slab"""
    n, g = M.shape
    S = max(1, min(TPM_SLABS, g, (1 << 25) // n))
    cp = M.indptr

    def first_col(target):
        return int(np.searchsorted(cp[:g], target, side="left"))

    bounds = []
    for s in range(S):
        c0 = 0 if s == 0 else first_col(M.nnz * s // S)
        c1 = g if s == S - 1 else first_col(M.nnz * (s + 1) // S)
        bounds.append((c0, c1))
    return S, bounds


def restated_totals(M, bounds):
    """the cell totals in the kernels' fp64 order: slab s adds its columns into its own row vector from 0, one column
    at a time (distinct rows within a column: one addition per entry), then the slab vectors are added in slab order"""
    t = np.zeros(M.shape[0])
    for c0, c1 in bounds:
        p = np.zeros(M.shape[0])
        for c in range(c0, c1):
            sl = slice(M.indptr[c], M.indptr[c + 1])
            p[M.indices[sl]] += M.data[sl].astype(np.float64)
        t += p
    return t


def tpm_case(name):
    rng = np.random.RandomState(len(name))
    if name == "slabs_eq_cols":                 # G = 5: S = G, and slab 1 holds two columns
        n, lens, integer = 1000, [600, 500, 500, 900, 400], False
    elif name == "slabs_111":                   # N = 300 000: S = floor(2^25 / N) = 111
        n, lens, integer = 300_000, list(rng.randint(1000, 3000, 300)), True
    elif name == "one_slab":                    # N just above 2^24: S = 1
        n, lens, integer = (1 << 24) + 5, [5000, 4097, 3000], True
    elif name == "dominant_column":             # one column holds most entries: most slabs are empty
        n, lens, integer = 20_000, [20_000] + [5] * 199, False
    elif name == "unrolled_edges":              # around the row pass's 4 x 512-entry unrolled step
        n, lens, integer = 6000, [1536, 1537, 2048, 2049, 4097, 1], False
    else:                                       # the same lengths, integer counts
        n, lens, integer = 6000, [1536, 1537, 2048, 2049, 4097, 1], True
    cols = []
    for m in lens:
        r = np.arange(n) if m == n else np.sort(rng.choice(n, m, replace=False))
        v = rng.randint(1, 6, m).astype(np.float64) if integer else 2.0 ** rng.uniform(-30, 30, m)
        cols.append((r, v))
    if name == "slabs_eq_cols":
        # x0 in [1, 2) (an fp32 value: its last fp64 bit is 0) and 2^-53 in columns 1 and 2, which share slab 1:
        # x0 + (2^-53 + 2^-53) = x0 + 2^-52, while column by column x0 + 2^-53 ties to x0 twice
        cols[0] = (cols[0][0], 2.0 ** rng.uniform(0, 1, lens[0]))
        cols[1] = (cols[1][0], np.full(lens[1], 2.0 ** -53))
        cols[2] = (cols[2][0], np.full(lens[2], 2.0 ** -53))
    return csc(n, cols), integer


TPM_CASES = ["slabs_eq_cols", "slabs_111", "one_slab", "dominant_column", "unrolled_edges", "unrolled_edges_counts"]


@pytest.mark.parametrize("case", TPM_CASES)
def test_tpm_stats(eng, case):
    """tpm_stats on CSC.  The cell totals equal, bit for bit, the kernels' order restated in numpy (slab plan from the
    shape, columns in order into each slab's vector, slabs in order): a plan that ignores n_cols groups the columns
    differently, which the G = 5 case turns into different bits with a planted rounding tie.  Integer counts: the totals are exact.  The scale
    rs = 1e6 / total is one IEEE division of those totals.  The TPM column sums run as csc_col_stats_kernel on
    v = fl(x rs): one more rounding per term, d = ceil(m / 32) + 6, then mean and variance as in test_csc_col_stats.
    Against the dense twins of the same matrix (row_sums, col_stats(row_scale=rs)), within the sum of both bounds:
    row_sums is a warp per row (ceil(G / 32) + 5 roundings against at most G column and G slab additions), the strip sums of the dense col_stats carry per + strips
    + 1 roundings per term (per rows per strip, then the strips in order) and square with a separate multiply."""
    M, integer = tpm_case(case)
    n, g = M.shape
    S, bounds = slab_plan(M)
    expect_S = {"slabs_eq_cols": 5, "slabs_111": 111, "one_slab": 1}.get(case)
    if expect_S is not None:
        assert S == expect_S
    if case == "slabs_eq_cols":
        assert any(c1 - c0 > 1 for c0, c1 in bounds)
    if case == "dominant_column":
        assert sum(c1 == c0 for c0, c1 in bounds) >= S // 2
    ds = eng.sparse_dataset(M)
    totals, mean, var = ds.tpm_stats()
    t_ref = restated_totals(M, bounds)
    assert np.array_equal(totals, t_ref), (case, np.flatnonzero(totals != t_ref)[:5])
    if integer:
        exact = np.bincount(M.indices, weights=M.data.astype(np.int64), minlength=n)
        assert np.array_equal(totals, exact)
    with np.errstate(divide="ignore"):
        rs = np.where(t_ref != 0, 1e6 / t_ref, 0.0)
    v = M.data.astype(np.float64) * rs[M.indices]
    s, q = col_sums(M, v.astype(LD)), col_sums(M, v.astype(LD) ** 2)
    m = np.diff(M.indptr)
    d = lane_depth(m) + 1
    m_ref = s / n
    b_mean = (((d + 1) * U + m * UL) * (s / n) * SECOND).astype(np.float64)
    b_var = (((2 * d + 5) * U + m * UL) * (q / n + m_ref ** 2) * SECOND).astype(np.float64)
    note("tpm_stats.mean", ratio(np.abs(mean - m_ref), b_mean))
    note("tpm_stats.var", ratio(np.abs(var - (q / n - m_ref ** 2)), b_var))
    ds.close()
    if n * g > 50_000_000:
        return
    dd = eng.dataset(M.toarray(), "fp32")
    rsum = dd.row_sums()
    row_abs = np.asarray(abs(M).sum(axis=1)).ravel()
    b_rows = (2 * g + -(-g // 32) + 5) * U * row_abs * SECOND
    if integer:
        assert np.array_equal(rsum, totals)
    assert (np.abs(rsum - totals) <= b_rows).all()
    dmean, dvar = dd.col_stats(row_scale=rs)
    strips = max(1, min(64, n // 64))
    dd_depth = -(-n // strips) + strips + 1
    note("tpm_stats.dense_mean", ratio(np.abs(dmean - mean), b_mean + ((dd_depth + 2) * U) * (s / n).astype(np.float64)))
    note("tpm_stats.dense_var", ratio(np.abs(dvar - var),
                                      b_var + ((2 * dd_depth + 7) * U) * (q / n + m_ref ** 2).astype(np.float64)))
    dd.close()


# ------------------------------------------------------------------------------------------------ D: dense project_rows
DENSE_FORMS = ["f16x2-tpm", "f16x2-col", "tf32x3", "tf32x3-general", "fp32"]
DENSE_SHAPES = [(1, 257), (255, 256), (256, 255), (257, 2000), (4097, 1), (4097, 257), (50_000, 256), (50_000, 257)]
BK = 32                   # fp32 elements per k-block of the GEMMs; 64 fp16 elements in the f16 form


def dense_matrix(form, n, g, rng):
    if form in ("tf32x3-general", "fp32"):
        return (10.0 ** rng.uniform(-2, 2, (n, g)) * (rng.rand(n, g) < 0.5)).astype(np.float32)
    C = rng.poisson(1.0, (n, g)).astype(np.float32)
    if form == "f16x2-tpm":
        C[:, 0] = 1
        return (C * (np.float32(1e6) / C.sum(axis=1, keepdims=True))).astype(np.float32)
    C[0, :] = 1
    return (C * (10.0 ** rng.uniform(-3, 3, g)).astype(np.float32)[None, :]).astype(np.float32)


def project_plan(k, n, g, sm_count, f16):
    """cnmf_project_rows' split plan: (requested splits before the 32 cap, effective splits, k-blocks per slice)"""
    tiles = -(-k // 128) * -(-g // 256)
    want = -(-2 * sm_count // tiles) if tiles < 2 * sm_count else 1
    want = min(want, max(1, -(-n // 32) // 8))
    bke = 2 * BK if f16 else BK
    total_kb = -(-n // bke)
    s = max(1, min(min(want, 32), total_kb))
    per = -(-total_kb // s)
    if f16 and per % 2:
        per += 1
    return want, -(-total_kb // per), per * bke


def signed_rows(rng, k, n):
    """centred signed rows; the last row (k >= 2) holds in its first 512-element group one negative entry 2^30 times
    the group's other entries, which puts them under the f16 group-scale floor"""
    Ut = rng.randn(k, n)
    Ut -= Ut.mean(axis=1, keepdims=True)
    if k >= 2:
        Ut[-1] = rng.uniform(0.5, 1.0, n) * rng.choice([-1.0, 1.0], n)
        Ut[-1, min(n - 1, 3)] = -(2.0 ** 30)
    return Ut.astype(np.float32)


@pytest.mark.parametrize("shape", DENSE_SHAPES, ids=["%dx%d" % s for s in DENSE_SHAPES])
@pytest.mark.parametrize("form", DENSE_FORMS)
def test_dense_project_rows(eng, sm_count, form, shape):
    """cnmf_project_rows (Ut @ X through the operand pieces and the split-K GEMM, slices summed on the host in fp64) at
    k = 1, 7, 32 and 33, against float64 Ut @ X_eff (X_eff = rs C cs, the device's own integer matrix and scales, on
    the exact forms).  Per entry, relative to the magnitude product mag = |Ut| |X_eff|:
      * the pieces: 22 significant bits of each factor entry (2^-22); the general form also splits X and drops
        lo x lo (3 x 2^-22); fp32 has none;
      * L fp32 additions per slice (L = k-blocks per slice x block depth), 2 u32 each to leave room for the tensor
        cores' accumulator, plus 2;
      * the output scale (one rounding) and the host's fp32 rounding of the fp64 slice sum: 2 u32;
      * f16: entries far below their 512-row group's maximum lose up to 2^-39 of it: 2^-39 max|a rs|_group
        sum_group |C cs| per group.
    The plan reaches its 32-split cap at 50 000 rows.  Two calls give the same bits."""
    n, g = shape
    precision = {"f16x2-tpm": "f16x2", "f16x2-col": "f16x2"}.get(form, form)
    rng = np.random.RandomState(n + g + DENSE_FORMS.index(form))
    X = dense_matrix(form, n, g, rng)
    ds = eng.dataset(X, precision)
    expect = {"f16x2": "f16_exact", "tf32x3": "tf32_exact", "tf32x3-general": "tf32", "fp32": "fp32"}[precision]
    assert ds.form == expect
    f16 = expect == "f16_exact"
    if expect in ("tf32_exact", "f16_exact"):
        C = (ds.operand("X_hi") if expect == "tf32_exact" else ds.operand("X_h16")).astype(np.float64)[:, :g]
        rs, cs = ds.operand("row_scale"), ds.operand("col_scale")
        rs = np.ones(n) if rs is None else rs[:n].astype(np.float64)
        cs = np.ones(g) if cs is None else cs[:g].astype(np.float64)
        Xe = C * rs[:, None] * cs[None, :]
    else:
        C, rs, cs = None, np.ones(n), np.ones(g)
        Xe = X.astype(np.float64)
    pieces = {"f16_exact": 1, "tf32_exact": 1, "tf32": 3, "fp32": 0}[expect]
    for k in (1, 7, 32, 33):
        want, splits, L = project_plan(k, n, g, sm_count, f16)
        if n == 50_000:
            assert want > 32 and splits >= 31, (want, splits)
        Ut = signed_rows(rng, k, n)
        out = ds.project_rows(Ut)
        A = Ut.astype(np.float64)
        ref = A @ Xe
        mag = np.abs(A) @ np.abs(Xe)
        bound = (pieces * 2.0 ** -22 + (2 * (L + 2) + 2) * U32) * mag
        if f16:
            ng = -(-n // 512)
            Ag = np.zeros((k, ng))
            Yg = np.zeros((ng, g))
            for j in range(ng):
                sl = slice(512 * j, 512 * (j + 1))
                Ag[:, j] = np.abs(A[:, sl] * rs[None, sl]).max(axis=1)
                Yg[j] = (C[sl] * cs[None, :]).sum(axis=0)
            bound += 2.0 ** -39 * (Ag @ Yg)
        bound *= SECOND
        assert np.isfinite(out).all(), (form, shape, k)
        note("project_rows." + expect, ratio(np.abs(out - ref), bound))
        assert np.array_equal(out, ds.project_rows(Ut))
    ds.close()
