"""The float64 solver's kernels one launch at a time (`-m gpu`), through the cnmf_update_step_f64_host /
cnmf_conv_check_host / cnmf_nndsvd_gemm_host test hooks, against references of oracle/kernel_ref.py -- at every K from 1
to 32 (the 8 / 16 / 32-wide update bodies are chosen per slot from K), at item counts around the 256-item update blocks,
the 64-item Gram staging tiles and the 2 048-item Gram chunks, at the GEMM's 64 x 128 output tiles and 16-deep K tiles
-- and bit for bit where batch independence rests on equal bits (DESIGN.md sections 4.6, 4.7).

u = 2^-53 is the unit roundoff of float64.  The references run in np.longdouble, whose unit roundoff UL (2^-64 on x86-64)
is 2^-11 of u: every bound adds the reference's own error, n UL per sum of n terms, so no float64 rounding of the
reference counts against the kernel.  Block sums of the update / cross kernels (block_sum) add 32 lanes in a 5-level
shuffle tree and then 8 warps in a chain: 12 roundings deep.  finalize_kernel adds a restart's chunks in order.
"""
import numpy as np
import pytest

from oracle import kernel_ref as kr

pytestmark = pytest.mark.gpu

U = 2.0 ** -53
LD = np.longdouble
UL = 2.0 ** -(np.finfo(LD).nmant + 1)
SECOND = 1 + 2.0 ** -10          # second-order terms and the reference's own rounding, relative to a first-order bound
TREE = 12                        # block_sum depth
ITEMS, GRAM_COLS = 256, 2048     # items per block of the update / cross kernels, of the Gram kernel
SENTINEL = -12345.0

ALL_K = list(np.random.RandomState(7).permutation(np.arange(1, 33)))      # every K in one batch, in no order
L12 = [(0.0, 0.0), (0.25, 0.0), (0.0, 0.5), (0.125, 0.375)]


@pytest.fixture(scope="module")
def eng():
    from cnmf_b200.engine import Engine
    return Engine(0)


def ld_of(n):
    return -(-n // 32) * 32


def offsets(ks):
    return np.concatenate([[0], np.cumsum(ks)]).astype(int)


def chunks(n):
    return -(-n // ITEMS)


def gram_blocks(rng, n_rids, m=48):
    """Per rid a symmetric 32 x 32 Gram-like block: unit diagonal plus coupling of about 1/32 per pair (enough that a
    Jacobi order of the CD sweep moves every coordinate after the first far outside the tolerance)."""
    out = np.zeros((n_rids, 32, 32))
    for r in range(n_rids):
        P = rng.uniform(0, 1, (32, m))
        out[r] = np.eye(32) + (P @ P.T) / (8 * m)
    return out


def make_batch(ks, n, seed, solver="mu", rids=None, n_rids=None):
    """Packed fp64 data of one launch.  Product columns >= n hold garbage; factor padding is zero (the layout's
    invariant)."""
    rng = np.random.RandomState(seed)
    ks = [int(k) for k in ks]
    R, SK, ld = len(ks), sum(ks), ld_of(n)
    rids = np.arange(R) if rids is None else np.asarray(rids)
    n_rids = int(rids.max()) + 1 if n_rids is None else n_rids
    off = offsets(ks)
    F = np.zeros((SK, ld))
    F[:, :n] = rng.uniform(0.1, 2.0, (SK, n))
    gin = gram_blocks(rng, n_rids)
    num = np.full((SK, ld), 7.0)
    if solver == "mu":
        num[:, :n] = rng.uniform(0.05, 1.5, (SK, n))
    else:
        F[:, :n][rng.rand(SK, n) < 0.1] = 0.0                                  # the projected gradient's min(0, g)
        for s, (k, r) in enumerate(zip(ks, rids)):
            target = rng.uniform(-0.3, 1.5, (k, n))                            # negative targets: clipped at 0
            num[off[s]:off[s + 1], :n] = gin[r, :k, :k] @ target
    return dict(ks=ks, rids=rids, n_rids=n_rids, off=off, n=n, F=F, num=num, gin=gin)


def run(eng, b, op="update", solver="mu", done=None, **kw):
    done = np.zeros(b["n_rids"], np.int32) if done is None else done
    return eng.update_step_f64(b["ks"], b["rids"], done, b["n"], b["F"], op=op, num=b["num"], gram_in=b["gin"],
                               solver=solver, **kw)


def slots(b):
    for s, (k, r) in enumerate(zip(b["ks"], b["rids"])):
        yield k, int(r), slice(b["off"][s], b["off"][s + 1])


def ratio(err, bound):
    """largest err / bound over entries with a positive bound (0 where both are 0)"""
    err, bound = np.asarray(err, np.float64), np.asarray(bound, np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.where(bound > 0, err / bound, np.where(err > 0, np.inf, 0.0))
    return float(q.max()) if q.size else 0.0


RATIOS = {}


@pytest.fixture(scope="module", autouse=True)
def report_ratios():
    """Largest error-to-bound ratio seen per check, printed after the module (visible with -s)."""
    yield
    for k in sorted(RATIOS):
        print("ratio %-18s %.3g" % (k, RATIOS[k]))


def note(key, r):
    RATIOS[key] = max(RATIOS.get(key, 0.0), r)
    assert r <= 1.0, (key, r)


def sum_bound(depth, S, terms):
    """|fl(sum) - sum| for a sum whose terms have absolute sum S, each partial sum rounded at most `depth` times on its
    way to the result, against a longdouble reference over `terms` products: depth u S + terms UL S."""
    return (depth * U + terms * UL) * S * SECOND


# ------------------------------------------------------------------------------------------------ MU
def mu_check(b, out, l1, l2, want_scalar=True):
    """MU per entry: den is a chain of K fp64 FMAs over non-negative terms (K roundings), then + l1 (1) and + l2 F (2);
    the quotient num / den and the product F * q round once each (IEEE): |F - ref| <= (K + 5) u |ref| to first order,
    no cancellation anywhere.  A zero den takes float32 eps, a positive one below FLT_MIN is used as it is.
    The scalar <NUM, F_new> is a chain of K FMAs per item, the block tree and the chunk chain over non-negative terms:
    against the kernel's own F_new it is within (K + TREE + chunks) u S, S = sum NUM F_new."""
    n = b["n"]
    for k, r, rows in slots(b):
        ref = kr.mu_half_step(b["F"][rows, :n], b["num"][rows, :n], b["gin"][r, :k, :k], l1, l2, eps_rule="zero",
                              dtype=LD)
        got = out["F"][rows, :n].astype(LD)
        note("mu.F", ratio(np.abs(got - ref), (k + 5) * U * SECOND * np.abs(ref)))
        if want_scalar:
            S = float((b["num"][rows, :n].astype(LD) * got).sum())
            note("mu.scal", ratio(abs(out["scal"][r] - S), sum_bound(k + TREE + chunks(n), S, n * k)))


@pytest.mark.parametrize("l12", L12, ids=lambda p: "l1_%g-l2_%g" % p)
@pytest.mark.parametrize("n", [1, 255, 256, 257, 2049])
def test_mu_update_against_float64_every_k(eng, n, l12):
    l1, l2 = l12
    for ks in (ALL_K, list(range(1, 9)), list(range(9, 17))):
        b = make_batch(ks, n, seed=n + len(ks) + int(8 * l1 + 16 * l2))
        out = run(eng, b, "update", "mu", want_scalar=True, l1=l1, l2=l2)
        mu_check(b, out, l1, l2)
        assert not out["F"][:, n:].any(), "factor padding columns must stay exactly 0"


def test_mu_denominator_eps_rule_is_sklearns(eng):
    """A zero Gram row with l1 = l2 = 0 gives den = 0 exactly: float32 eps, like scikit-learn.  A Gram row of about
    1e-300 gives 0 < den < FLT_MIN, which scikit-learn -- and so the float64 kernel -- divides by as it is (the fp32
    kernels floor it to eps)."""
    n = 513
    b = make_batch(ALL_K, n, seed=5)
    b["gin"][:, 0, :] = 0.0
    b["gin"][:, 1, :] *= 1e-300
    out = run(eng, b, "update", "mu")
    mu_check(b, out, 0.0, 0.0, want_scalar=False)
    for k, r, rows in slots(b):
        F, num = b["F"][rows, :n], b["num"][rows, :n]
        assert np.array_equal(out["F"][rows][0, :n], F[0] * (num[0] / kr.EPSILON))
        if k > 1:
            den = b["gin"][r, 1, :k] @ F
            assert (den > 0).all() and (den < kr.FLT_MIN).all()


# ------------------------------------------------------------------------------------------------ CD
def cd_check(b, out, l1, l2, viol=True):
    """CD per entry.  The gradient g of coordinate t is -(num - l1) (1 rounding) plus a chain of K FMAs: its error is
    <= (K + 1) u mag (mag = |num - l1| + sum |G F|) plus sum_{r<t} |G[t, r]| |dF_r| from the coordinates the sweep
    already moved differently.  g / h and F - g / h round once each: u mag / h and u (|F| + mag / h).  So
        |dF_t| <= ((K + 3) u mag + sum_{r<t} |G[t, r]| |dF_r|) / h + u |F_old|.
    (An entry-relative bound cannot work: F - g / h cancels for coordinates the sweep drives towards 0.)  h = G[t, t]
    + l2 rounds identically in the kernel and here.  The violation sums |projected gradient| in a chain of K per item,
    the block tree and the chunk chain, each term off by its gradient's error:
        |viol - ref| <= (K + TREE + chunks) u sum mag + sum_t ((K + 1) u mag_t + sum_{r<t} |G[t, r]| |dF_r|)."""
    n = b["n"]
    for k, r, rows in slots(b):
        G = b["gin"][r, :k, :k] + l2 * np.eye(k)          # the kernel's load_gram: one fp64 add on the diagonal
        F0 = b["F"][rows, :n]
        ref, vref, mag = kr.cd_sweep(F0, b["num"][rows, :n], G, l1, 0.0, dtype=LD)
        got = out["F"][rows, :n].astype(LD)
        d = np.abs(got - ref).astype(np.float64)
        mag = mag.astype(np.float64)
        lower = np.tril(np.abs(G), -1)
        h = np.abs(np.diag(G))[:, None]
        with np.errstate(divide="ignore", invalid="ignore"):
            bound = np.where(h > 0, (((k + 3) * U * mag + lower @ d) / h + U * np.abs(F0)) * SECOND, 0.0)
        note("cd.F", ratio(d, bound))
        if viol:
            bound = ((2 * k + 1 + TREE + chunks(n)) * U * mag.sum() + (lower @ d).sum()) * SECOND
            note("cd.viol", ratio(abs(out["scal"][r] - vref), bound))


@pytest.mark.parametrize("l12", L12, ids=lambda p: "l1_%g-l2_%g" % p)
@pytest.mark.parametrize("n", [1, 255, 257, 2049])
def test_cd_update_against_float64_every_k(eng, n, l12):
    l1, l2 = l12
    for ks in (ALL_K, list(range(1, 9)), list(range(9, 17))):
        b = make_batch(ks, n, seed=3 * n + len(ks), solver="cd")
        out = run(eng, b, "update", "cd", want_scalar=True, l1=l1, l2=l2)
        cd_check(b, out, l1, l2)
        assert not out["F"][:, n:].any(), "factor padding columns must stay exactly 0"


def test_cd_is_gauss_seidel_and_zero_diagonal_is_left_alone(eng):
    """The fixtures couple the coordinates strongly enough that a Jacobi order lands far outside the tolerance; a zero
    Gram diagonal (l2 = 0) leaves its coordinate bitwise unchanged."""
    b = make_batch(ALL_K, 2049, seed=11, solver="cd")
    b["gin"][:, 5, 5] = 0.0
    out = run(eng, b, "update", "cd", want_scalar=True)
    cd_check(b, out, 0.0, 0.0)
    far = 0
    for k, r, rows in slots(b):
        if k > 5:
            assert np.array_equal(out["F"][rows][5], b["F"][rows][5])
        if k > 1:
            jac, _, _ = kr.cd_sweep(b["F"][rows, :2049], b["num"][rows, :2049], b["gin"][r, :k, :k], jacobi=True)
            far += np.abs(out["F"][rows, :2049] - jac).max() > 1e-6
    assert far == 31


# ------------------------------------------------------------------------------------------------ Gram
GRAM_N = [1, 63, 64, 65, 2047, 2048, 2049, 6145]
KP_GROUPS = [list(range(q - 3, q + 1)) for q in range(4, 33, 4)]       # [1..4], [5..8], ... [29..32]: kp = 4 .. 32


def gram_check(b, out, key="gram"):
    """Entry (c, i) is one FMA chain over the chunk's items -- the 64-item stages continue it, zero-padded items add
    exactly 0 -- then finalize's chain over the chunks: at most min(n, 2048) + chunks roundings of partial sums of
    non-negative terms.  Entries with c or i in [K, KP) are exactly 0, those beyond KP are not written (sentinel), and
    the Gram is exactly symmetric (entry and mirror are the same chain with the factors swapped)."""
    n = b["n"]
    depth = min(n, GRAM_COLS) + -(-n // GRAM_COLS)
    for k, r, rows in slots(b):
        F = b["F"][rows, :n].astype(LD)
        ref = F @ F.T
        g = out["gram"][r]
        note(key, ratio(np.abs(g[:k, :k].astype(LD) - ref), sum_bound(depth, ref.astype(np.float64), n)))
        assert np.array_equal(g[:k, :k], g[:k, :k].T), ("Gram not exactly symmetric", k)
        kp = -(-k // 4) * 4
        assert not g[:kp, k:kp].any() and not g[k:kp, :kp].any(), ("entries c or i in [K, KP) must be 0", k)
        assert (g[kp:, :] == SENTINEL).all() and (g[:, kp:] == SENTINEL).all(), ("entries beyond KP written", k)


@pytest.mark.parametrize("n", GRAM_N)
def test_gram_against_float64_every_k(eng, n):
    """Every K in batches whose kp runs from 4 to 32, each after a batch that leaves non-zero partials where its
    [K, KP) entries go, and a restart's Gram has the same bits in its own kp group as beside every other K."""
    sent = np.full((32, 32, 32), SENTINEL)
    grams = {}
    for ks in KP_GROUPS:
        kp = ks[-1]
        prime = make_batch([kp] * len(ks), n, seed=n + kp)
        run(eng, prime, "gram")
        b = make_batch(ks, n, seed=n)
        b["F"] = np.vstack([make_batch([k], n, seed=1000 * k + n)["F"] for k in ks])
        out = run(eng, b, "gram", gram_out=sent[:len(ks)])
        gram_check(b, out)
        for k, r, _ in slots(b):
            grams[k] = out["gram"][r].copy()
    b = make_batch(ALL_K, n, seed=n)
    b["F"] = np.vstack([make_batch([k], n, seed=1000 * k + n)["F"] for k in ALL_K])
    out = run(eng, b, "gram", gram_out=sent)
    gram_check(b, out)
    for k, r, _ in slots(b):
        assert np.array_equal(out["gram"][r], grams[k]), ("Gram bits depend on the batch's kmax", k)


# ------------------------------------------------------------------------------------------------ cross
@pytest.mark.parametrize("n", GRAM_N)
def test_cross_against_float64_every_k(eng, n):
    """<NUM, F> is a chain of K FMAs per item, the block tree and the chunk chain over non-negative terms:
    within (K + TREE + chunks) u S of the exact sum, S = sum NUM F."""
    b = make_batch(ALL_K, n, seed=n + 1)
    out = run(eng, b, "cross", scal_out=np.full(b["n_rids"], SENTINEL))
    for k, r, rows in slots(b):
        S = float((b["num"][rows, :n].astype(LD) * b["F"][rows, :n].astype(LD)).sum())
        note("cross", ratio(abs(out["scal"][r] - S), sum_bound(k + TREE + chunks(n), S, n * k)))
    assert np.array_equal(out["F"], b["F"])


# ------------------------------------------------------------------------------------------------ slots
@pytest.mark.parametrize("op,solver", [("update", "mu"), ("update", "cd"), ("gram", "mu"), ("cross", "mu")])
def test_frozen_and_foreign_restarts_are_untouched(eng, op, solver):
    """Slots in a permuted rid order, two rids in no slot, two slots frozen: the frozen restarts' factor rows and every
    result of a frozen or foreign rid keep their sentinels; the live ones match a batch without them."""
    ks = [3, 17, 8, 32, 1, 12]
    rids = [4, 0, 7, 2, 5, 1]                 # rids 3 and 6 are in no slot
    done = np.zeros(8, np.int32)
    done[[7, 5]] = 1                          # the K = 8 and K = 1 slots
    b = make_batch(ks, 700, seed=21, solver=solver, rids=rids, n_rids=8)
    kw = dict(gram_out=np.full((8, 32, 32), SENTINEL), scal_out=np.full(8, SENTINEL))
    out = run(eng, b, op, solver, done=done, want_scalar=True, l1=0.125, l2=0.25, **kw)
    live = [s for s, r in enumerate(rids) if not done[r]]
    sub = make_batch([ks[s] for s in live], 700, seed=0, solver=solver)
    sub["F"] = np.vstack([b["F"][b["off"][s]:b["off"][s + 1]] for s in live])
    sub["num"] = np.vstack([b["num"][b["off"][s]:b["off"][s + 1]] for s in live])
    sub["gin"] = b["gin"][[rids[s] for s in live]]
    ref = run(eng, sub, op, solver, want_scalar=True, l1=0.125, l2=0.25)
    for s, (k, r) in enumerate(zip(ks, rids)):
        rows = slice(b["off"][s], b["off"][s + 1])
        if done[r]:
            assert np.array_equal(out["F"][rows], b["F"][rows])
            continue
        i = live.index(s)
        assert np.array_equal(out["F"][rows], ref["F"][sub["off"][i]:sub["off"][i + 1]])
        if op == "gram":
            assert np.array_equal(out["gram"][r][:k, :k], ref["gram"][i][:k, :k])
        else:
            assert out["scal"][r] == ref["scal"][i]
    for r in (3, 6, 7, 5):
        assert (out["gram"][r] == SENTINEL).all() and out["scal"][r] == SENTINEL, r
    assert not out["F"][:, 700:].any()


# ------------------------------------------------------------------------------------------------ fp64 GEMM
GEMM_M = [1, 15, 16, 63, 64, 65, 528]
GEMM_OUT = [1, 127, 128, 129, 257]
GEMM_RED = [1, 15, 16, 17, 31, 33, 2049]


@pytest.mark.parametrize("to_genes", [False, True])
@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_fp64_gemm_against_float64(eng, dtype, to_genes):
    """C = A X^T (output over X's rows) or A X (over its columns) through the GEMM hook, which runs the <*, float> or
    <*, double> instantiation on the dataset's own X.  A is signed (projections of centred usages are).  Per entry the
    order inside a 16-deep DMMA tile is unspecified, so the bound is the order-free (K + 1) u sum_k |a||x| of a K-term
    fp64 dot product.  No output is NaN (C starts as NaN bytes), and an output row has the same bits at any M and
    wherever its row sits in the 64-row tile (rows prepended to A)."""
    rng = np.random.RandomState(17 + to_genes + 2 * (dtype == "float64"))
    for n_out in GEMM_OUT:
        for red in GEMM_RED:
            shape = (red, n_out) if to_genes else (n_out, red)
            X = np.abs(rng.randn(*shape)).astype(dtype)
            ds = eng.dataset(X, precision="fp64" if dtype == "float64" else "fp32")
            A = rng.randn(max(GEMM_M), red)
            XL = X.astype(LD)
            ref = A.astype(LD) @ (XL if to_genes else XL.T)
            absum = np.abs(A) @ np.abs(X.astype(np.float64) if to_genes else X.astype(np.float64).T)
            bound = ((red + 1) * U + red * UL) * absum * SECOND
            full = ds.nndsvd_gemm(A, to_genes)
            assert np.isfinite(full).all(), (n_out, red)
            note("gemm.%s" % dtype, ratio(np.abs(full.astype(LD) - ref), bound))
            for M in GEMM_M[:-1]:
                C = ds.nndsvd_gemm(A[:M], to_genes)
                assert np.array_equal(C, full[:M]), ("output rows depend on M", M, n_out, red)
            for p in (1, 17, 64):
                C = ds.nndsvd_gemm(np.vstack([rng.randn(p, red), A[:65]]), to_genes)
                assert np.array_equal(C[p:], full[:65]), ("output rows depend on their position", p, n_out, red)
            ds.close()


def test_fp64_gemm_hook_refuses_sparse_datasets(eng):
    import scipy.sparse as sp
    from cnmf_b200._lib import CnmfError
    ds = eng.sparse_dataset(sp.random(50, 40, density=0.2, format="csc", random_state=0))
    with pytest.raises(CnmfError, match="sparse"):
        ds.nndsvd_gemm(np.ones((2, 40)), False)


# ------------------------------------------------------------------------------------------------ convergence
def conv(eng, solver, it, tol, max_iter, st, **kw):
    R = len(st["done"])
    return eng.conv_check(kw.pop("ks", [4] * R), kw.pop("rids", list(range(R))), solver, it, tol, max_iter,
                          st["done"], st["n_iter"], st["err0"], st["prev"], st["last"], **kw)


def mu_state(err0, prev, R=1):
    return dict(done=np.zeros(R, np.int32), n_iter=np.zeros(R, np.int32), err0=np.full(R, err0),
                prev=np.full(R, prev), last=np.zeros(R))


def mu_tol_eff(it, tol):
    """what the batched solve passes to mu_check_kernel at iteration it (solve_frobenius, nmf_engine.cu)"""
    return tol if (tol > 0 and it % 10 == 0) else -1.0


def mu_errs(err, R=1):
    """err = sqrt(normX2 - 2 cross + <gA, gB>) with grams 0 and cross 0: normX2 = err^2 (exact for the values used)"""
    return dict(normX2=err ** 2, cross=np.zeros(R), gramA=np.zeros((R, 32, 32)), gramB=np.zeros((R, 32, 32)))


def mu_drive(eng, errs, tol, max_iter):
    """The solver's sequence of mu_check launches (it = 0, then the checks) against kernel_ref.mu_stop over the same
    errors (errs[it], held until the next iteration listed): the same stopping iteration and last error."""
    st = mu_state(0.0, 0.0)
    st = conv(eng, "mu", 0, tol, max_iter, st, **mu_errs(errs[0]))
    assert st["err0"][0] == errs[0] and st["prev"][0] == errs[0]
    prev, n_ref = errs[0], None
    for it in range(1, max_iter + 1):
        err = errs[max(e for e in errs if e <= it)]
        stop, prev = kr.mu_stop(it, err, errs[0], prev, tol, max_iter)
        if (tol > 0 and it % 10 == 0) or it == max_iter:
            st = conv(eng, "mu", it, mu_tol_eff(it, tol), max_iter, st, **mu_errs(err))
            if not st["done"][0]:
                assert st["prev"][0] == prev
        if stop:
            n_ref = it
            break
    assert st["done"][0] == 1 and st["n_iter"][0] == n_ref, (st, n_ref)
    return st


def test_mu_check_follows_the_loop_decision(eng):
    """tol boundary (< is strict), err0 = 0 runs to max_iter, a max_iter off the multiples of 10 stops there with
    that iteration's error, and the plain case."""
    e = {0: 4.0, 10: 3.0, 20: 2.0, 30: 1.75, 40: 1.5}
    assert mu_drive(eng, e, 0.25, 100)["n_iter"][0] == 30           # (3 - 2) / 4 = 0.25: not < 0.25, continues
    assert mu_drive(eng, e, np.nextafter(0.25, 1), 100)["n_iter"][0] == 10
    z = {0: 0.0, 10: 0.0}
    assert mu_drive(eng, z, 1e-4, 35)["n_iter"][0] == 35
    st = mu_drive(eng, {0: 4.0, 10: 3.0, 13: 2.5}, 1e-4, 13)
    assert st["n_iter"][0] == 13 and st["last"][0] == 2.5
    st = mu_drive(eng, {0: 4.0, 7: 3.5}, 0.0, 7)
    assert st["n_iter"][0] == 7 and st["last"][0] == 3.5


def test_mu_check_error_and_clamp(eng):
    """err = sqrt(max(normX2 - 2 cross + <gA, gB>, 0)): the dot is K^2 / 32 terms per lane plus a 5-level tree, then two
    adds (and the product's own rounding if it is not fused): |err^2 - ref| <= (K^2 / 32 + 9) u (normX2 + 2 |cross| + sum |gA gB|), and sqrt adds u err.  A negative
    residual gives err = 0 (never NaN); frozen restarts and their n_iter are untouched."""
    rng = np.random.RandomState(2)
    ks = ALL_K
    R = len(ks)
    gA, gB = rng.uniform(0, 1, (R, 32, 32)), rng.uniform(0, 1, (R, 32, 32))
    cross = rng.uniform(0, 1, R) * 50
    normX2 = 4000.0
    st = dict(done=np.zeros(R, np.int32), n_iter=np.zeros(R, np.int32), err0=np.zeros(R), prev=np.zeros(R),
              last=np.full(R, SENTINEL))
    st["done"][3] = 1
    st["n_iter"][3] = 77
    out = conv(eng, "mu", 0, 1e-4, 100, st, ks=ks, normX2=normX2, cross=cross, gramA=gA, gramB=gB)
    for r, k in enumerate(ks):
        if r == 3:
            assert out["done"][r] == 1 and out["n_iter"][r] == 77 and out["last"][r] == SENTINEL
            continue
        dot = (gA[r, :k, :k].astype(LD) * gB[r, :k, :k]).sum()
        e2 = LD(normX2) - 2 * LD(cross[r]) + dot
        ref = float(np.sqrt(e2))
        b2 = ((k * k / 32 + 9) * U + k * k * UL) * (normX2 + 2 * cross[r] + float(dot))
        bound = (b2 / (2 * ref) + U * ref) * SECOND
        note("mu_check.err", ratio(abs(out["last"][r] - ref), bound))
        assert out["err0"][r] == out["last"][r] == out["prev"][r]
    neg = conv(eng, "mu", 0, 1e-4, 100, mu_state(0.0, 0.0), normX2=1.0, cross=np.ones(1),
               gramA=np.zeros((1, 32, 32)), gramB=np.zeros((1, 32, 32)))
    assert neg["last"][0] == 0.0 and neg["err0"][0] == 0.0


def cd_drive(eng, viols, tol, max_iter, violB=None):
    st = dict(done=np.zeros(1, np.int32), n_iter=np.zeros(1, np.int32), err0=np.zeros(1), prev=np.zeros(1),
              last=np.zeros(1))
    v0, n_ref = None, None
    for it in range(1, max_iter + 1):
        v = viols[min(it, len(viols)) - 1]
        vb = None if violB is None else np.array([violB])
        stop, v0 = kr.cd_stop(it, v + (0.0 if violB is None else violB), v0, tol, max_iter)
        st = conv(eng, "cd", it, tol, max_iter, st, violA=np.array([v]), violB=vb)
        if stop:
            n_ref = it
            break
    assert st["done"][0] == 1 and st["n_iter"][0] == n_ref
    return st


def test_cd_check_follows_the_loop_decision(eng):
    """<= at the tol boundary, viol0 = 0 stops at iteration 1, violB is added, max_iter ends the loop."""
    assert cd_drive(eng, [4.0, 2.0, 1.0, 0.5], 0.25, 50)["n_iter"][0] == 3          # 1 / 4 <= 0.25
    assert cd_drive(eng, [4.0, 2.0, 1.0, 0.5], np.nextafter(0.25, 0), 50)["n_iter"][0] == 4
    assert cd_drive(eng, [0.0, 0.0], 1e-4, 50)["n_iter"][0] == 1
    assert cd_drive(eng, [3.5, 0.5], 0.25, 50, violB=0.5)["n_iter"][0] == 2          # (0.5 + 0.5) / (3.5 + 0.5)
    st = cd_drive(eng, [4.0, 3.5, 3.25], 1e-4, 6)
    assert st["n_iter"][0] == 6 and st["last"][0] == 3.25 and st["err0"][0] == 4.0


def test_cd_check_leaves_frozen_restarts_alone(eng):
    st = dict(done=np.array([1, 0], np.int32), n_iter=np.array([9, 0], np.int32), err0=np.array([5.0, 0.0]),
              prev=np.zeros(2), last=np.array([SENTINEL, 0.0]))
    out = conv(eng, "cd", 1, 1e-4, 10, st, violA=np.array([0.0, 2.0]))
    assert out["done"][0] == 1 and out["n_iter"][0] == 9 and out["last"][0] == SENTINEL and out["err0"][0] == 5.0
    assert out["done"][1] == 0 and out["err0"][1] == 2.0 and out["last"][1] == 2.0


# ------------------------------------------------------------------------------------------------ dataset sums
@pytest.mark.parametrize("rows", [63, 64, 65, 4095, 4097])
def test_float64_dataset_sums_and_col_stats(eng, rows):
    """matrix_sums_f64: each thread adds rows_per_block (64) x ceil(cols / 256) values, then the block tree and the
    chain over blocks; col_stats_kernel<double>: a chain over a strip of per = ceil(rows / strips) rows (2 roundings per
    term for v^2), strips = clamp(rows / 64, 1, 64) added in order, then mean = s / n and var = q / n - mean^2.  Against
    exact sums (math.fsum on the values; x^2 rounds once, which the bound adds)."""
    import math
    cols = 300
    rng = np.random.RandomState(rows)
    X = rng.uniform(0, 3, (rows, cols))
    ds = eng.dataset(X, precision="fp64")
    s, q = ds.sums()
    S, Q = math.fsum(X.ravel()), math.fsum((X * X).ravel())
    nb = -(-rows // 64)
    depth = 64 * -(-cols // 256) + TREE + nb
    note("sums", ratio(abs(s - S), depth * U * S * SECOND))
    note("sums.sq", ratio(abs(q - Q), (depth + 1) * U * Q * SECOND))
    mean, var = ds.col_stats()
    strips = max(1, min(64, rows // 64))
    per = -(-rows // strips)
    for c in range(cols):
        sc, qc = math.fsum(X[:, c]), math.fsum(X[:, c] * X[:, c])
        m = sc / rows
        bm = (per + strips + 1) * U * m * SECOND
        note("col_stats.mean", ratio(abs(mean[c] - m), bm))
        v = float(LD(qc) / rows - (LD(sc) / rows) ** 2)
        bv = ((2 * per + strips + 3) * U * qc / rows + 2 * m * bm + 2 * U * m * m + U * v) * SECOND
        note("col_stats.var", ratio(abs(var[c] - v), bv))
    ds.close()
