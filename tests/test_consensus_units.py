"""The consensus kernels one entry point at a time (`-m gpu`), in both element types (float32, and float64 for
precision='fp64'), against float64 references computed from the same T inputs -- at the sizes where the kernels change
form: the 64-row distance tiles, the ragged G % 4 tail and the NC = 2 / 4 / 8 forms of the candidate distances and the
tile fallback beyond 8 candidates, the 1024-row chunks of the batched member lists, K = 32 of the batched fit and
K = 1024 of the per-run kernels, the 48 KB dynamic shared-memory threshold of the k-means++ select kernel, and the
R <= 25 600 limit of the batched fit.

u_T is the unit roundoff of T (2^-24 or 2^-53); u = 2^-53 that of the float64 accumulators.  Every bound is derived
from the kernel's own arithmetic in the docstring of its check.  The batched fit is compared with
oracle/kmeans_device_ref.py, a restatement of it in the device's order of operations.
"""
import ctypes
import math

import numpy as np
import pytest

from oracle import kmeans_device_ref as kd

pytestmark = pytest.mark.gpu

U64 = 2.0 ** -53
UT = {np.float32: 2.0 ** -24, np.float64: 2.0 ** -53}
DTYPES = [np.float32, np.float64]
SENTINEL = -12345.0
dtypes = pytest.mark.parametrize("dt", DTYPES, ids=["f32", "f64"])


@pytest.fixture(scope="module")
def eng():
    from cnmf_b200.engine import Engine
    return Engine(0)


def mat(eng, X, dt):
    from cnmf_b200.consensus import SpectraMatrix
    return SpectraMatrix(eng, np.asarray(X), dtype=dt)


def ivec(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).cuda()


def vp(t):
    return ctypes.c_void_p(t.data_ptr())


def call(S, name, *args):
    from cnmf_b200._lib import check
    check(S.fn(name)(S.engine._h, S.p, *args))


def ceil_div(a, b):
    return -(-a // b)


# ------------------------------------------------------------------------------------------------ C1
@dtypes
@pytest.mark.parametrize("G", [1, 3, 31, 33, 4097])
def test_l2_normalize_rows(eng, dt, G):
    """q = sum x^2 in float64 (each thread a strided chain of ceil(G / 256), then an 8-level block tree: relative error
    <= (ceil(G / 256) + 8) u), sqrt, 1 / sqrt and x * inv each round once in float64, then one rounding to T:
    |out - ref| <= u_T |ref| + ((ceil(G / 256) + 8) / 2 + 3) u |ref|, i.e. within about 1 ulp of T.  Rows span
    2^-60 ... 2^60; the padding columns keep their sentinel."""
    rng = np.random.RandomState(G)
    R = 40
    X = (rng.uniform(0.5, 2.0, (R, G)) * rng.choice([-1.0, 1.0], (R, G))).astype(dt)
    X *= (2.0 ** np.linspace(-60, 60, R).round()).astype(dt)[:, None]
    S = mat(eng, X, dt)
    S.t[:, G:] = SENTINEL
    S.l2_normalize()
    got = S.numpy().astype(np.float64)
    X64 = X.astype(np.float64)
    ref = X64 / np.sqrt((X64 ** 2).sum(axis=1, keepdims=True))
    bound = (UT[dt] + ((ceil_div(G, 256) + 8) / 2 + 3) * U64) * np.abs(ref)
    assert (np.abs(got - ref) <= bound).all(), float((np.abs(got - ref) / np.abs(ref)).max())
    assert (S.t[:, G:].cpu().numpy() == SENTINEL).all()


# ------------------------------------------------------------------------------------------------ C2 / C3
def dist_bound(G, dt):
    """One T chain of G fmas over non-negative terms (G roundings), each difference rounded once (2 in its square),
    then a square root (half the relative error, plus its own rounding): ((G + 2) / 2 + 1) u_T relative."""
    return ((G + 2) / 2 + 1) * UT[dt] * (1 + 1e-6)


def exact_dist(X):
    from scipy.spatial.distance import cdist
    X64 = X.astype(np.float64)
    return cdist(X64, X64)


def spectra(rng, R, G, dt):
    X = np.abs(rng.randn(R, G)) + 0.05
    if R >= 3:
        X[R - 1] = X[0]                    # identical rows: distance exactly 0
    return X.astype(dt)


@dtypes
@pytest.mark.parametrize("R,G", [(2, 1), (63, 17), (64, 16), (65, 15), (129, 2001), (1000, 17), (257, 1)])
def test_pair_distances(eng, dt, R, G):
    """D of local_density(return_dist=True) within dist_bound of the float64 distances; exactly symmetric, exactly
    zero on the diagonal and between identical rows."""
    X = spectra(np.random.RandomState(R + G), R, G, dt)
    S = mat(eng, X, dt)
    _, D = S.local_density(1, return_dist=True)
    D64 = D.astype(np.float64)
    ref = exact_dist(X)
    err = np.abs(D64 - ref)
    assert (err <= dist_bound(G, dt) * ref).all(), float((err / np.maximum(ref, 1e-300)).max())
    assert (D == D.T).all() and (np.diag(D) == 0).all()
    if R >= 3:
        assert D[0, R - 1] == 0 and D[R - 1, 0] == 0


def density_ref(D, m, n):
    """Sum of the m smallest entries of every row, exactly (fsum of the sorted row), over n."""
    Ds = np.sort(D, axis=1)[:, :m]
    return np.array([math.fsum(r) for r in Ds]) / n


def density_cases(rng, dt):
    yield "random", spectra(rng, 200, 33, dt)
    X = spectra(rng, 97, 9, dt)
    X[50:60] = X[10]                       # ten duplicates of one row: ten zero distances in its row
    yield "duplicates", X
    yield "equidistant", (0.75 * np.eye(65, 70)).astype(dt)      # every off-diagonal distance the same value


@dtypes
def test_local_density(eng, dt):
    """Against the device's own D the selection is exact, so the density is a float64 sum (each thread a strided
    chain of ceil(R / 256), then a 10-level tree, and the (m - less) tau term), one division and one rounding to T:
    |dens - ref| <= u_T ref + (ceil(R / 256) + 12) u ref.  Against the float64 distances, every entry of D is within
    dist_bound relative, and so is any sum of its m smallest (each subset sum moves by at most that much).  Keep / drop
    at a threshold equals the reference's wherever the reference is farther than the bound from it."""
    rng = np.random.RandomState(7)
    for name, X in density_cases(rng, dt):
        R, G = X.shape
        S = mat(eng, X, dt)
        ref64 = exact_dist(X)
        for n in sorted({1, 2, R - 2, R - 1}):
            dens, D = S.local_density(n, return_dist=True)
            own = density_ref(D.astype(np.float64), n + 1, n)
            b_own = UT[dt] + (ceil_div(R, 256) + 12) * U64
            assert (np.abs(dens - own) <= b_own * own).all(), (name, n, float(np.abs(dens / own - 1).max()))
            ref = density_ref(ref64, n + 1, n)
            b_ref = b_own + dist_bound(G, dt) * (1 + b_own)
            assert (np.abs(dens - ref) <= b_ref * ref).all(), (name, n, float(np.abs(dens / ref - 1).max()))
            thr = float(np.median(ref))
            clear = np.abs(ref - thr) > b_ref * ref
            assert clear.sum() >= R // 4 or name == "equidistant"
            assert np.array_equal((dens < thr)[clear], (ref < thr)[clear]), (name, n)
        if name == "equidistant":       # all off-diagonal distances equal: n copies of the threshold value, over n
            d1 = float(D[0, 1])
            assert (D[~np.eye(R, dtype=bool)] == D[0, 1]).all()
            for n in (1, 2, R - 1):
                dens, _ = S.local_density(n)
                assert (np.abs(dens - d1) <= 2 * UT[dt] * d1).all(), (n, dens[:3], d1)


# ------------------------------------------------------------------------------------------------ C4
@dtypes
@pytest.mark.parametrize("G", [1, 2, 3, 5, 7, 2001])
def test_sq_dists_to_rows(eng, dt, G):
    """n_c <= 8 runs cand_dist_kernel (NC = 2 / 4 / 8, unused slots read candidate 0): differences in T (2 u_T in the
    square), float64 sums (G u, negligible), one rounding to T: <= 3 u_T + G u relative.  n_c > 8 gathers the
    candidates and runs the T distance tile: one T chain of G fmas, (G + 2) u_T.  A candidate equal to the row gives
    exactly 0; repeated candidates give equal rows."""
    rng = np.random.RandomState(G)
    R = 300
    X = spectra(rng, R, G, dt)
    S = mat(eng, X, dt)
    X64 = X.astype(np.float64)
    for n_c in (1, 2, 3, 4, 5, 8, 9, 70):
        idx = rng.randint(0, R, n_c)
        if n_c >= 2:
            idx[-1] = idx[0]                    # a repeated candidate
        out = S.sq_dists_to_rows(idx)
        ref = ((X64[None, :, :] - X64[idx][:, None, :]) ** 2).sum(axis=2)
        rel = (3 * UT[dt] + (G + 4) * U64) if n_c <= 8 else (G + 2) * UT[dt] * (1 + 1e-6)
        err = np.abs(out - ref)
        assert (err <= rel * ref).all(), (n_c, float((err / np.maximum(ref, 1e-300)).max()))
        assert (out[np.arange(n_c), idx] == 0).all()     # each candidate against its own row
        if n_c >= 2:
            assert np.array_equal(out[-1], out[0])


# ------------------------------------------------------------------------------------------------ C5
def canonical(C):
    """Index of the first centre equal to each centre."""
    first = {}
    return np.array([first.setdefault(c.tobytes(), j) for j, c in enumerate(C)])


def assign_ref(X, C):
    """float64 E step: labels (first minimum), distances, and the relative gap to the nearest centre that is not a copy
    of the chosen one (copies give bit-equal distances in T, so their tie goes to the lower index exactly)."""
    X64, C64 = X.astype(np.float64), C.astype(np.float64)
    D = ((X64[:, None, :] - C64[None, :, :]) ** 2).sum(axis=2)
    lab = np.argmin(D, axis=1)
    best = D[np.arange(len(X)), lab]
    canon = canonical(C)
    other = np.where(canon[None, :] == canon[lab][:, None], np.inf, D)
    second = other.min(axis=1)
    with np.errstate(invalid="ignore"):             # K = 1 or only copies: no runner-up, the gap is infinite
        gap = np.where(np.isinf(second), np.inf, (second - best) / np.maximum(second + best, 1e-300))
    return lab, best, gap


def make_centres(rng, X, K, dt):
    R, G = X.shape
    C = X[rng.randint(0, R, K)].astype(np.float64) + 0.3 * rng.randn(K, G)
    C[: min(K, R) // 2] = X[: min(K, R) // 2]       # centres equal to rows: distance 0
    if K >= 4:
        C[3] = C[1]                                 # a copy of a centre: its rows must take the lower index
    return np.ascontiguousarray(C, dtype=dt)


@dtypes
@pytest.mark.parametrize("K", [1, 2, 32, 33, 512, 1024])
@pytest.mark.parametrize("R", [1, 31, 33, 1025])
def test_kmeans_assign(eng, dt, K, R):
    """Labels: first minimum; where the gap to the runner-up exceeds kd.e_step_bound the label equals float64's (and
    most rows have such gaps).  mind within e_step_bound of the float64 distance.  counts and the float64 centre sums
    exact: a sequential row-order float64 sum (the kernel's order) reproduced bit for bit.  inertia: the mind values
    (each within e_step_bound) summed in float64 by one block of 1024 (ceil(R / 1024) + 10 roundings)."""
    import torch
    G = 7 if K >= 512 else 19
    rng = np.random.RandomState(K * 7 + R)
    X = (rng.rand(R, G) * 2).astype(dt)
    S = mat(eng, X, dt)
    C = make_centres(rng, X, K, dt)
    lab_in = rng.randint(0, K, R)
    labels_t = ivec(lab_in)
    mind_t = torch.empty(R, dtype=S.torch_dtype, device="cuda")
    sums = np.empty((K, G)); counts = np.empty(K, np.int32)
    n_changed = np.zeros(1, np.int32); inertia = np.zeros(1)
    from cnmf_b200._lib import ptr
    call(S, "cnmf_kmeans_assign", R, G, S.ld, ptr(C), K, vp(labels_t), ptr(sums), ptr(counts), vp(mind_t),
         ptr(n_changed), ptr(inertia), None)
    lab = labels_t.cpu().numpy()
    mind = mind_t.cpu().numpy().astype(np.float64)
    lref, dref, gap = assign_ref(X, C)
    eb = kd.e_step_bound(G, dt)
    decided = gap > eb
    assert decided.mean() > 0.5
    assert np.array_equal(lab[decided], lref[decided]), int((lab != lref)[decided].sum())
    canon = canonical(C)
    assert (canon[lab] == lab).all(), "a copy of a centre won over its lower-index original"
    assert (np.abs(mind - dref) <= eb * dref).all()
    assert n_changed[0] == int((lab != lab_in).sum())
    assert np.array_equal(counts, np.bincount(lab, minlength=K))
    ref_sums = np.zeros((K, G))
    np.add.at(ref_sums, lab, X.astype(np.float64))
    assert np.array_equal(sums, ref_sums)
    b = eb + (ceil_div(R, 1024) + 10) * U64
    assert abs(inertia[0] - dref.sum()) <= b * dref.sum() + 1e-300


@dtypes
@pytest.mark.parametrize("K,R", [(1, 1), (2, 31), (32, 1025), (33, 33), (1024, 1025)])
def test_kmeans_step(eng, dt, K, R):
    """One per-run Lloyd step from given float64 centres: labels and mind as in test_kmeans_assign; n_changed against
    the labels passed in, counts and any_empty exact; the centre sums bit for bit a sequential row-order float64 sum;
    the new centres sums * (1 / count) and their T copy bit for bit; the shift (a float64 block sum per centre, the
    centres summed on the host) within (ceil(G / 256) + K + 12) u."""
    import torch
    G = 7 if K >= 512 else 37
    rng = np.random.RandomState(K + 3 * R)
    X = (rng.rand(R, G) * 2).astype(dt)
    S = mat(eng, X, dt)
    C64 = make_centres(rng, X, K, np.float64)
    CT = C64.astype(dt)
    lab_in = rng.randint(0, K, R)
    labels_t = ivec(lab_in)
    mind_t = torch.empty(R, dtype=S.torch_dtype, device="cuda")
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()      # noqa: E731
    C64_cur, C64_new = dev(C64), torch.full((K, G), np.nan, dtype=torch.float64, device="cuda")
    sums_t = torch.empty((K, G), dtype=torch.float64, device="cuda")
    counts_t = torch.empty(K, dtype=torch.int32, device="cuda")
    n_changed, any_empty, shift = ctypes.c_int32(), ctypes.c_int32(), ctypes.c_double()
    tail = (vp(labels_t), vp(mind_t), vp(sums_t), vp(counts_t), ctypes.byref(n_changed), ctypes.byref(any_empty),
            ctypes.byref(shift), None)
    if dt == np.float64:
        call(S, "cnmf_kmeans_step", R, G, S.ld, K, vp(C64_cur), vp(C64_new), *tail)
        CT_new = None
    else:
        CT_cur, CT_new = dev(CT), torch.full((K, G), np.nan, dtype=torch.float32, device="cuda")
        call(S, "cnmf_kmeans_step", R, G, S.ld, K, vp(CT_cur), vp(C64_cur), vp(C64_new), vp(CT_new), *tail)
    lab = labels_t.cpu().numpy()
    lref, dref, gap = assign_ref(X, CT)
    eb = kd.e_step_bound(G, dt)
    decided = gap > eb
    assert decided.mean() > 0.5 and np.array_equal(lab[decided], lref[decided])
    assert (np.abs(mind_t.cpu().numpy() - dref) <= eb * dref).all()
    counts = np.bincount(lab, minlength=K)
    assert n_changed.value == int((lab != lab_in).sum())
    assert np.array_equal(counts_t.cpu().numpy(), counts)
    assert any_empty.value == int((counts == 0).any())
    ref_sums = np.zeros((K, G))
    np.add.at(ref_sums, lab, X.astype(np.float64))
    assert np.array_equal(sums_t.cpu().numpy(), ref_sums)
    full = counts > 0
    new = C64_new.cpu().numpy()
    ref_new = ref_sums * (1.0 / np.maximum(counts, 1))[:, None]
    assert np.array_equal(new[full], ref_new[full])
    if CT_new is not None:
        assert np.array_equal(CT_new.cpu().numpy()[full], ref_new[full].astype(np.float32))
    ref_shift = float(((ref_new - C64)[full] ** 2).sum())
    assert abs(shift.value - ref_shift) <= (ceil_div(G, 256) + K + 12) * U64 * ref_shift


# ------------------------------------------------------------------------------------------------ C5b
def blobs(R, G, n_blobs, seed, spread=0.35):
    rng = np.random.RandomState(seed)
    cen = rng.rand(n_blobs, G) * 2
    return cen[rng.randint(0, n_blobs, R)] + spread * rng.randn(R, G)


def draws(R, K, n_init, n_trials, seed):
    rng = np.random.RandomState(seed)
    return (rng.randint(0, R, n_init).astype(np.int32),
            rng.uniform(size=(n_init, max(K - 1, 1), n_trials)))


def kmeans_fit(S, K, first, unif, n_trials, max_iter, tol_abs):
    from cnmf_b200._lib import ptr
    n_init = len(first)
    labels = np.zeros((n_init, S.R), np.int32)
    inertia = np.zeros(n_init)
    n_iter = np.zeros(n_init, np.int32)
    flag = ctypes.c_int32(-1)
    call(S, "cnmf_kmeans_fit", S.R, S.G, S.ld, K, n_init, max_iter, float(tol_abs), ptr(first),
         ptr(np.ascontiguousarray(unif)), n_trials, ptr(labels), ptr(inertia), ptr(n_iter), ctypes.byref(flag), None)
    return labels, inertia, n_iter, flag.value


def check_fit(S, X, K, first, unif, n_trials, max_iter, tol_abs, dt):
    """Every run of the batched fit against the device-order restatement.  The data must decide every E step and every
    shift test the same way in T as in float64 (asserted from the restatement's gaps), so labels and n_iter are equal;
    inertia is the final mind values (each within e_step_bound) summed in float64 by 256 threads per run
    (ceil(R / 256) + 9 roundings)."""
    R, G = X.shape
    runs = kd.kmeans_fit(X, K, first, unif, n_trials, max_iter, tol_abs)
    eb = kd.e_step_bound(G, dt)
    for r in runs:
        assert not r["empty"]
        assert r["min_gap"] > eb, ("data too close to a tie", r["min_gap"], eb)
        assert r["tol_gap"] > 1e-9
    labels, inertia, n_iter, flag = kmeans_fit(S, K, first, unif, n_trials, max_iter, tol_abs)
    assert flag == 0
    b = eb + (ceil_div(R, 256) + 9) * U64
    for t, r in enumerate(runs):
        assert np.array_equal(labels[t], r["labels"]), (t, int((labels[t] != r["labels"]).sum()))
        assert n_iter[t] == r["n_iter"], (t, int(n_iter[t]), r["n_iter"])
        assert abs(inertia[t] - r["inertia"]) <= b * r["inertia"] + 1e-300, (t, inertia[t], r["inertia"])
    return runs, n_iter


FIT_CASES = [  # K, n_init, n_trials, R, G, max_iter, tol on (tol * mean variance)
    (1, 1, 1, 1, 3, 300, 1e-4),
    (2, 10, 2, 2, 5, 300, 1e-4),
    (5, 10, 3, 1023, 6, 300, 1e-4),
    (5, 32, 8, 1024, 6, 1, 1e-4),
    (31, 3, 8, 1024, 4, 2, 1e-4),
    (32, 10, 2, 1025, 5, 300, 0.0),
    (32, 32, 1, 32, 3, 300, 1e-4),
    (5, 10, 2, 6100, 4, 300, 1e-2),
    (2, 3, 2, 25600, 4, 300, 1e-4),
]


@dtypes
@pytest.mark.parametrize("case", FIT_CASES, ids=lambda c: "K%d-n%d-t%d-R%d-i%d" % (c[0], c[1], c[2], c[3], c[5]))
def test_kmeans_fit_every_run(eng, dt, case):
    K, n_init, n_trials, R, G, max_iter, tol = case
    X = blobs(R, G, max(K, 2), seed=K + R + G).astype(dt)
    S = mat(eng, X, dt)
    first, unif = draws(R, K, n_init, n_trials, seed=R + n_init)
    tol_abs = tol * float(np.var(X.astype(np.float64), axis=0).mean())
    runs, n_iter = check_fit(S, X, K, first, unif, n_trials, max_iter, tol_abs, dt)
    if max_iter == 300 and n_init >= 10 and 2 < K < R:
        assert len(set(n_iter.tolist())) > 1, "every run stopped at the same iteration"
    if max_iter < 300:
        assert (n_iter == max_iter).all()


@dtypes
def test_kmeans_fit_select_shared_memory_window(eng, dt):
    """R = 6135 ... 6145: the k-means++ select kernel's R doubles of dynamic shared memory cross 48 KB minus its static
    shared memory (6135) and 48 KB itself (6145).  Every R fits and matches the restatement."""
    for R in range(6135, 6146):
        X = blobs(R, 4, 5, seed=R).astype(dt)
        S = mat(eng, X, dt)
        first, unif = draws(R, 5, 2, 3, seed=R)
        tol_abs = 1e-4 * float(np.var(X.astype(np.float64), axis=0).mean())
        check_fit(S, X, 5, first, unif, 3, 300, tol_abs, dt)


def tie_rows(dt):
    """1-D rows -2, -2, 0, 0, 2, 2 with the k-means++ centres -2 (first) and 2 (the uniform 0.4 lands on row 4).
    Both rows 0 are exactly 2 from either centre: the first minimum puts them with -2, the means are -1 and 2 (counts
    4 and 2, all arithmetic exact) and the final labels are 0 0 0 0 1 1 with inertia 4.  A last-minimum rule would
    give the means -2 and 1 and labels 0 0 1 1 1 1."""
    X = np.array([[-2.0], [-2.0], [0.0], [0.0], [2.0], [2.0]], dtype=dt)
    return X, np.array([0], np.int32), np.array([[[0.4]]])


@dtypes
@pytest.mark.parametrize("max_iter", [1, 300])
def test_kmeans_fit_exact_ties_take_the_lower_centre(eng, dt, max_iter):
    X, first, unif = tie_rows(dt)
    S = mat(eng, X, dt)
    labels, inertia, n_iter, flag = kmeans_fit(S, 2, first, unif, 1, max_iter, 0.0)
    assert flag == 0
    assert labels[0].tolist() == [0, 0, 0, 0, 1, 1] and inertia[0] == 4.0
    assert n_iter[0] == min(max_iter, 2)


@dtypes
def test_kmeans_fit_runs_stop_at_different_parities(eng, dt):
    """max_iter = 1 stops every run after one step, so the final E step must read the buffer that step wrote (index 1),
    not the k-means++ centres; with max_iter = 300 the runs stop at iterations of both parities."""
    X = blobs(700, 6, 6, seed=3).astype(dt)
    S = mat(eng, X, dt)
    first, unif = draws(700, 6, 12, 3, seed=9)
    tol_abs = 1e-4 * float(np.var(X.astype(np.float64), axis=0).mean())
    _, n1 = check_fit(S, X, 6, first, unif, 3, 1, tol_abs, dt)
    _, n = check_fit(S, X, 6, first, unif, 3, 300, tol_abs, dt)
    assert (n1 == 1).all() and {0, 1} <= set((n % 2).tolist()), n


@dtypes
def test_kmeans_fit_empty_cluster_in_one_run_hands_over(eng, dt, monkeypatch):
    """Run 3 of 10 starts at row 0 and draws the uniform 0: the cumulative sum reaches 0 at row 0 itself, so its second
    centre is row 0 again.  The copy loses every tie to the original, its cluster is empty after the first E step, and
    the fit reports it (needs_host_path) instead of labels; consensus.kmeans then runs the per-run path once."""
    from cnmf_b200 import consensus as cs
    R, K = 200, 4
    X = blobs(R, 5, K, seed=8).astype(dt)
    first, unif = draws(R, K, 10, 1, seed=6)
    first[3], unif[3, 0, 0] = 0, 0.0
    runs = kd.kmeans_fit(X, K, first, unif, 1, 300, 0.0)
    assert [r["empty"] for r in runs] == [t == 3 for t in range(10)]
    assert runs[3]["centre_idx"][1] == 0 and runs[3]["n_iter"] == 1
    S = mat(eng, X, dt)
    _, _, _, flag = kmeans_fit(S, K, first, unif, 1, 300, 0.0)
    assert flag == 1
    calls = []
    per_run = cs._kmeans_per_run
    monkeypatch.setattr(cs, "_kmeans_per_run", lambda *a: calls.append(1) or per_run(*a))
    monkeypatch.setattr(cs, "_kmeans_draws", lambda rng, n, k, n_init: (first, unif, 1))
    labels, _, _, _ = cs.kmeans(S, K)
    assert calls == [1] and labels.shape == (R,) and 0 <= labels.min() and labels.max() < K


@dtypes
def test_kmeans_beyond_the_batched_limit_takes_the_per_run_path(eng, dt, monkeypatch):
    """R = 25 601 rows do not fit the select kernel's shared memory: the library refuses the batched fit and
    consensus.kmeans runs the per-run path (once)."""
    from cnmf_b200 import consensus as cs
    from cnmf_b200._lib import CnmfError
    R = 25601
    X = blobs(R, 3, 3, seed=2).astype(dt)
    S = mat(eng, X, dt)
    first, unif = draws(R, 3, 1, 2, seed=1)
    with pytest.raises(CnmfError, match="too many rows"):
        kmeans_fit(S, 3, first, unif, 2, 10, 0.0)
    calls = []
    per_run = cs._kmeans_per_run
    monkeypatch.setattr(cs, "_kmeans_per_run", lambda *a: calls.append(1) or per_run(*a))
    labels, _, _, _ = cs.kmeans(S, 3, n_init=2, max_iter=50)
    assert calls == [1] and labels.shape == (R,)


@dtypes
def test_kmeans_batched_matches_per_run(eng, dt):
    """consensus.kmeans' batched fit and its per-run path from the same draws: equal labels (same E / M arithmetic;
    the k-means++ potentials differ only in association).  The inertia is the same mind values summed by 256 threads
    per run or by one block of 1024: within (ceil(R / 256) + ceil(R / 1024) + 20) u, not bit for bit."""
    from cnmf_b200 import consensus as cs
    R = 1023
    X = blobs(R, 6, 5, seed=12).astype(dt)
    S = mat(eng, X, dt)
    lb, _, ib, _ = cs.kmeans(S, 5)
    mean, var = np.empty(S.G), np.empty(S.G)
    call(S, "cnmf_col_stats_dev", S.R, S.G, S.ld, mean.ctypes.data_as(ctypes.c_void_p),
         var.ctypes.data_as(ctypes.c_void_p), None)
    lp, _, ip, _ = cs._kmeans_per_run(S, 5, 10, 1, 300, float(var.mean()) * 1e-4)
    assert np.array_equal(lb, lp)
    assert abs(ib - ip) <= (ceil_div(R, 256) + ceil_div(R, 1024) + 20) * U64 * ip


# ------------------------------------------------------------------------------------------------ C6
def median_labels(rng, K, sizes):
    lab = np.concatenate([np.full(sizes[c % len(sizes)], c) for c in range(K)])
    return lab[rng.permutation(len(lab))]          # members interleaved in row order


@dtypes
@pytest.mark.parametrize("K,G", [(1, 33), (32, 7), (32, 130), (1024, 5)])
def test_cluster_median(eng, dt, K, G):
    """The median in T is bit-exact (the middle value, or T(0.5) * (v1 + v2) in T); each row is then divided by its
    float64 sum (at most G - 1 roundings), one division, one rounding to T: within u_T + G u relative of
    median / fsum(median).  An empty cluster gives a NaN row and leaves the others alone.  Values are multiples of 1/8
    with many zeros, so even clusters often have equal (or zero) middle values."""
    import torch
    rng = np.random.RandomState(K + G)
    sizes = [64] if K == 1 else [1, 2, 3, 4, 5, 64, 65, 0, 6] if K < 1024 else [1, 2, 3, 4, 5, 0, 6]
    lab = median_labels(rng, K, sizes)
    R = len(lab)
    X = (rng.randint(0, 6, (R, G)) / 8.0) * (rng.rand(R, G) < 0.6)
    X[:, G // 2:] += rng.rand(R, G - G // 2) * (rng.rand(R, G - G // 2) < 0.5)
    X[:, 0] += 0.125                                 # no all-zero median row
    X = X.astype(dt)
    S = mat(eng, X, dt)
    M = torch.full((K, S.ld), SENTINEL, dtype=S.torch_dtype, device="cuda")
    call(S, "cnmf_cluster_median", S.R, S.G, S.ld, vp(ivec(lab)), K, vp(M), S.ld, None)
    got = M[:, :G].cpu().numpy().astype(np.float64)
    assert (M[:, G:].cpu().numpy() == SENTINEL).all()
    half = dt(0.5)
    for c in range(K):
        v = np.sort(X[lab == c], axis=0)
        n = len(v)
        if n == 0:
            assert np.isnan(got[c]).all()
            continue
        med = v[n // 2] if n % 2 else half * (v[n // 2 - 1] + v[n // 2])
        med64 = med.astype(np.float64)
        ref = med64 / math.fsum(med64)
        assert (np.abs(got[c] - ref) <= (UT[dt] + G * U64) * np.abs(ref)).all(), (c, n)


# ------------------------------------------------------------------------------------------------ C7
@dtypes
@pytest.mark.parametrize("R", [1, 2, 7, 8, 9, 33, 257, 1001])
@pytest.mark.parametrize("K", [1, 2, 512])
def test_cluster_dist_sums(eng, dt, R, K):
    """Per row and cluster, the float64 sum of the device's own distances to the cluster's members: R - 1 roundings
    at most, so within R u relative of fsum.  Some of the 8 per-warp slices are empty at small R; clusters without
    members give exactly 0.  A second call gives the same bits."""
    rng = np.random.RandomState(R + K)
    X = spectra(rng, R, 11, dt)
    S = mat(eng, X, dt)
    lab = rng.randint(0, max(1, K // 2), R) if K > 1 else np.zeros(R, int)   # the upper half of the clusters is empty
    out = np.empty((R, K))
    out2 = np.empty((R, K))
    labels_t = ivec(lab)
    from cnmf_b200._lib import ptr
    call(S, "cnmf_cluster_dist_sums", R, S.G, S.ld, vp(labels_t), K, ptr(out), None)
    call(S, "cnmf_cluster_dist_sums", R, S.G, S.ld, vp(labels_t), K, ptr(out2), None)
    assert np.array_equal(out, out2)
    D = S.local_density(1, return_dist=True)[1].astype(np.float64) if R >= 2 else np.zeros((1, 1))
    ref = np.array([[math.fsum(D[r, lab == c]) for c in range(K)] for r in range(R)])
    assert (np.abs(out - ref) <= R * U64 * ref).all()
    if K > 1:
        assert (out[:, K // 2:] == 0).all()


# ------------------------------------------------------------------------------------------------ C8
@dtypes
@pytest.mark.parametrize("R", [1, 256, 1000])
def test_col_stats(eng, dt, R):
    """Column sums s and q = sum x^2 in float64 in row order (R - 1 roundings each; squares of float32 are exact).
    mean = s / R within (R + 1) u of the two-pass mean (relative to mean |x|); var = q / R - mean^2 loses at most
    3 (R + 2) u E[x^2] to cancellation (q / R carries (R + 1) u E[x^2], mean^2 twice the mean's error), is clamped at 0, and is exactly 0 for a constant 0.75 column when R is a power
    of two (every sum exact)."""
    from cnmf_b200._lib import ptr
    rng = np.random.RandomState(R)
    G = 6
    X = np.empty((R, G))
    X[:, 0] = rng.rand(R)
    X[:, 1] = 1000.0 + rng.randn(R)                 # large mean, unit variance
    X[:, 2] = 1.0 + 1e-6 * rng.randn(R)             # near-constant
    X[:, 3] = 0.75                                  # constant, exact sums
    X[:, 4] = 0.1                                   # constant, inexact sums
    X[:, 5] = rng.randn(R) * 2.0 ** rng.randint(-20, 20, R)
    X = X.astype(dt)
    S = mat(eng, X, dt)
    mean, var = np.empty(G), np.empty(G)
    call(S, "cnmf_col_stats_dev", R, G, S.ld, ptr(mean), ptr(var), None)
    X64 = X.astype(np.float64)
    m_ref = np.array([math.fsum(c) for c in X64.T]) / R
    v_ref = np.array([math.fsum(c) for c in ((X64 - m_ref) ** 2).T]) / R
    ex2 = (X64 ** 2).mean(axis=0)
    assert (np.abs(mean - m_ref) <= (R + 1) * U64 * np.abs(X64).mean(axis=0)).all()
    assert (var >= 0).all()
    assert (np.abs(var - v_ref) <= 3 * (R + 2) * U64 * ex2).all(), (var, v_ref)
    if R & (R - 1) == 0:
        assert var[3] == 0.0 and mean[3] == 0.75


# ------------------------------------------------------------------------------------------------ C9
@dtypes
def test_gather_rows(eng, dt):
    """A device row gather: bit for bit, with repeated and reversed indices."""
    from cnmf_b200.consensus import SpectraMatrix
    rng = np.random.RandomState(0)
    X = rng.randn(50, 37).astype(dt)
    S = mat(eng, X, dt)
    for idx in (np.arange(50)[::-1], np.array([3, 3, 3, 49, 0, 3]), rng.randint(0, 50, 200)):
        assert np.array_equal(S.take_rows(idx).numpy(), X[idx])
        T = SpectraMatrix.from_device_rows(eng, S.t.data_ptr(), S.ld, idx, 37, dtype=dt)
        assert np.array_equal(T.numpy(), X[idx])


# ------------------------------------------------------------------------------------------------ workspace reuse
def workspace_results(eng, dt, X, lab, K, first, unif):
    """Every entry point with a named cached buffer: consensus.D (local_density without a D argument,
    cluster_dist_sums), kmeans.cnt / kmeans.order (cluster_median, kmeans_assign) and kmb.* (kmeans_fit)."""
    import torch
    from cnmf_b200._lib import ptr
    S = mat(eng, X, dt)
    R, G = X.shape
    out = {"density": S.local_density(3)[0]}
    sums = np.empty((R, K))
    labels_t = ivec(lab)
    call(S, "cnmf_cluster_dist_sums", R, G, S.ld, vp(labels_t), K, ptr(sums), None)
    out["dist_sums"] = sums
    M = torch.empty((K, S.ld), dtype=S.torch_dtype, device="cuda")
    call(S, "cnmf_cluster_median", R, G, S.ld, vp(labels_t), K, vp(M), S.ld, None)
    out["median"] = M[:, :G].cpu().numpy()
    C = np.ascontiguousarray(X[:K])
    mind_t = torch.empty(R, dtype=S.torch_dtype, device="cuda")
    cs, cn = np.empty((K, G)), np.empty(K, np.int32)
    call(S, "cnmf_kmeans_assign", R, G, S.ld, ptr(C), K, vp(labels_t), ptr(cs), ptr(cn), vp(mind_t),
         None, None, None)
    out["assign"] = (labels_t.cpu().numpy(), cs, cn)
    out["fit"] = kmeans_fit(S, K, first, unif, 3, 300, 0.0)
    return out


def same(a, b):
    if isinstance(a, tuple):
        return all(same(x, y) for x, y in zip(a, b))
    return np.array_equal(a, b, equal_nan=True) if np.asarray(a).dtype.kind == "f" else np.array_equal(a, b)


@dtypes
def test_reused_workspace_gives_fresh_bits(eng, dt):
    """A call after a larger and after a smaller one gives the same bits as on a fresh Engine."""
    from cnmf_b200.engine import Engine
    cases = []
    for R, G, K, seed in ((300, 21, 6, 1), (1100, 9, 12, 2), (300, 21, 6, 1)):
        X = blobs(R, G, K, seed=seed).astype(dt)
        rng = np.random.RandomState(seed)
        first, unif = draws(R, K, 4, 3, seed=seed)
        cases.append((X, rng.randint(0, K, R), K, first, unif))
    fresh = []
    for c in cases[:2]:
        e = Engine(0)
        fresh.append(workspace_results(e, dt, *c))
        e.close()
    shared = [workspace_results(eng, dt, *c) for c in cases]
    for got, want in ((shared[0], fresh[0]), (shared[1], fresh[1]), (shared[2], fresh[0])):
        for key in want:
            assert same(got[key], want[key]), key
