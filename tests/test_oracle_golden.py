"""Pin the oracle (oracle/nmf_ref.py, oracle/consensus_ref.py) against fixtures produced by
the UNMODIFIED reference (oracle/make_golden.py -> tests/golden/*.npz), and against live
scikit-learn calls with the kwargs the reference passes (cnmf.py:618-631,738-741).
CPU only."""
import warnings

import numpy as np
import pytest

from oracle import consensus_ref, nmf_ref
from cnmf_b200.synth import restart_table


def rel_l2(a, b):
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


def test_seed_rule_matches_reference(golden):
    # cnmf.py:597-610 -- seeds drawn with np.random.seed(seed); randint(1, 2**31-1, n_runs)
    rows = restart_table(list(golden["ks"]), int(golden["n_iter"]), int(golden["seed"]))
    assert np.array_equal(np.array(rows, dtype=np.int64), golden["table"])


def test_factorize_restatement_matches_reference(golden):
    X = golden["X"]
    solver = golden["solver"]
    for k in golden["ks"]:
        merged = golden["merged_k%d" % k]
        rows = [r for r in golden["table"] if r[0] == k]
        for (kk, it, seed) in rows:
            W, H, n_it = nmf_ref.nmf(X, int(kk), int(seed), solver=solver, beta=golden["beta"], init=golden["init"])
            ref = merged[it * k:(it + 1) * k]
            assert rel_l2(H, ref) < 1e-10, (solver, k, it)


def test_trace_form_error_equals_dense_form(golden):
    # the CUDA path evaluates ||X-WH|| through the trace identity (SK/_nmf.py:116-120)
    X = golden["X"]
    W, H = nmf_ref.init_random(X.mean(), X.shape[0], X.shape[1], 5, 7)
    a = nmf_ref.frobenius_error(X, W, H)
    b = nmf_ref.frobenius_error_trace(X, W, H)
    assert abs(a - b) / a < 1e-12
    W2, H2, it2 = nmf_ref.mu_frobenius(X, W, H, error_fn=nmf_ref.frobenius_error_trace)
    W1, H1, it1 = nmf_ref.mu_frobenius(X, W, H)
    assert it1 == it2 and rel_l2(H2, H1) < 1e-12


def test_consensus_restatement_matches_reference(golden):
    solver = golden["solver"]
    for k in golden["ks"]:
        out = consensus_ref.consensus(golden["merged_k%d" % k], golden["X"], golden["tpm"],
                                      golden["tpm_std"], golden["hvg_idx"], int(k),
                                      density_threshold=float(golden["dt"]), solver=solver, beta=golden["beta"])
        # ||x||^2+||y||^2-2x.y cancels catastrophically for near-identical unit rows (d ~ 1e-4 here):
        # fp64 summation-order noise of 1e-16 in d^2 is 1e-8 relative -- hence rtol 1e-6, not 1e-12
        # (init='nndsvd': the restarts differ by ~1e-8 -- every density is that cancellation noise itself, compared as "zero")
        atol = 1e-12 if golden["init"] == "random" else 1e-7
        assert np.allclose(out["local_density"], golden["density_k%d" % k], rtol=1e-6, atol=atol)
        # the reference test's own criterion: sum of squared differences < 1e-4
        # (tests/test_reproducibility.py:111-112), plus a much tighter relative bound
        for name, key in (("consensus_spectra", "cspectra"), ("consensus_usages", "cusages"),
                          ("gene_spectra_tpm", "tpmspec"), ("gene_spectra_score", "score")):
            ref = golden["%s_k%d" % (key, k)]
            assert rel_l2(out[name], ref) < 1e-8, (name, k, rel_l2(out[name], ref))


def test_kmeans_restatement_matches_sklearn():
    from sklearn.cluster import KMeans
    rng = np.random.RandomState(3)
    centres = rng.rand(6, 40)
    X = np.vstack([c + 0.05 * rng.randn(30, 40) for c in centres])
    X = np.abs(X)
    X /= np.linalg.norm(X, axis=1, keepdims=True)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        km = KMeans(n_clusters=6, n_init=10, random_state=1).fit(X)
    labels, inertia, centers = consensus_ref.kmeans(X, 6)
    assert np.array_equal(labels, km.labels_)
    assert abs(inertia - km.inertia_) / km.inertia_ < 1e-10
    assert np.allclose(centers, km.cluster_centers_, atol=1e-12)


@pytest.mark.parametrize("k,n_init,seed", [(1, 3, 0), (2, 10, 1), (5, 10, 2), (7, 4, 3)])
def test_kmeans_device_order_restatement_matches_sklearn(k, n_init, seed):
    """oracle/kmeans_device_ref.py (the batched fit in the device's order) in float64 against scikit-learn: every run's
    k-means++ centre indices equal kmeans_plusplus' from the same RandomState stream, and the best run's labels equal
    KMeans'.  Overlapping blobs, so Lloyd takes several iterations; no E-step decision is within 1e-9 of a tie."""
    from sklearn.cluster import KMeans, kmeans_plusplus
    from cnmf_b200.consensus import _kmeans_draws
    from oracle import kmeans_device_ref as kd
    rng = np.random.RandomState(40 + seed)
    centres = rng.rand(max(k, 2) + 1, 12)
    X = np.vstack([c + 0.25 * rng.randn(60, 12) for c in centres])
    first, unif, n_trials = _kmeans_draws(np.random.RandomState(seed), X.shape[0], k, n_init)
    tol_abs = float(np.var(X, axis=0).mean()) * 1e-4
    runs = kd.kmeans_fit(X, k, first, unif, n_trials, 300, tol_abs)
    sk_rng = np.random.RandomState(seed)
    for r in runs:
        _, idx = kmeans_plusplus(X, k, random_state=sk_rng)
        assert np.array_equal(r["centre_idx"], idx)
        assert r["min_gap"] > 1e-9 and not r["empty"]
    assert len({r["n_iter"] for r in runs}) > 1 or n_init == 1 or k == 1
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        km = KMeans(n_clusters=k, n_init=n_init, random_state=seed).fit(X)
    best = kd.best_run(runs, k)
    assert np.array_equal(best["labels"], km.labels_)
    assert abs(best["inertia"] - km.inertia_) <= 1e-10 * km.inertia_


def test_distance_and_density_match_sklearn():
    from sklearn.metrics.pairwise import euclidean_distances
    rng = np.random.RandomState(0)
    S = consensus_ref.l2_normalize_rows(np.abs(rng.randn(50, 30)))
    D = euclidean_distances(S)
    assert np.allclose(consensus_ref.euclidean_distances(S), D, atol=1e-13)
    n = 7
    part = np.argpartition(D, n + 1)[:, :n + 1]
    dens = D[np.arange(50)[:, None], part].sum(1) / n      # cnmf.py:893-896
    assert np.allclose(consensus_ref.local_density(D, n), dens, atol=1e-13)


def test_silhouette_matches_sklearn():
    from sklearn.metrics import silhouette_score
    rng = np.random.RandomState(1)
    X = rng.rand(60, 10)
    labels = rng.randint(0, 4, 60)
    assert abs(consensus_ref.silhouette(X, labels) - silhouette_score(X, labels)) < 1e-12


def test_stats_branch_matches_reference(golden):
    # cnmf.py:922-936 (k_selection statistics): no density filter; silhouette + ||X - W H||^2
    solver = golden["solver"]
    for k in golden["ks"]:
        merged = golden["merged_k%d" % k]
        l2 = consensus_ref.l2_normalize_rows(merged)
        labels, _, _ = consensus_ref.kmeans(l2, int(k))
        med = consensus_ref.cluster_medians(l2, labels, int(k))
        rf, _ = nmf_ref.refit(golden["X"], med, solver, beta=golden["beta"])
        err = ((golden["X"] - rf @ med) ** 2).sum()
        stats = golden["stats_k%d" % k]
        # (init='nndsvd': intra-cluster distances are ~1e-8 cancellation noise, so the silhouette is 1 - noise)
        assert abs(consensus_ref.silhouette(l2, labels) - stats[2]) < (1e-9 if golden["init"] == "random" else 1e-7)
        assert abs(err - stats[3]) / stats[3] < 1e-9


@pytest.mark.parametrize("l1,l2", [(0.0, 0.0), (0.3, 0.0), (0.0, 0.7), (0.25, 1.5)])
def test_kernel_step_references_match_sklearn(l1, l2):
    """oracle/kernel_ref.py's one-launch references -- what tests/test_kernel_units.py holds the update kernels to --
    against scikit-learn's own update functions in float64 (MU: _multiplicative_update_w; CD:
    _update_coordinate_descent with shuffle=False), in the kernels' layout F = W^T, num = (X H^T)^T, G = H H^T."""
    from sklearn.decomposition import _nmf
    from oracle import kernel_ref
    rng = np.random.RandomState(int(10 * l1 + 100 * l2))
    n, g, K = 60, 45, 7
    X = np.abs(rng.randn(n, g))
    W = np.abs(rng.randn(n, K))
    W[::5, 2] = 0.0                     # zero coordinates: the projected gradient's min(0, g) branch
    H = np.abs(rng.randn(K, g))
    num, G = (X @ H.T).T, H @ H.T
    Wm, *_ = _nmf._multiplicative_update_w(X, W.copy(), H, 2, l1, l2, 1.0)
    assert np.allclose(kernel_ref.mu_half_step(W.T, num, G, l1, l2), Wm.T, rtol=1e-13, atol=0)
    Wc = W.copy()
    viol = _nmf._update_coordinate_descent(X, Wc, H.T, l1, l2, False, None)
    Fc, v, mag = kernel_ref.cd_sweep(W.T, num, G, l1, l2)
    assert np.allclose(Fc, Wc.T, rtol=1e-12, atol=1e-13) and abs(v - viol) <= 1e-12 * viol
    assert (mag >= 0).all()
    Fj, _, _ = kernel_ref.cd_sweep(W.T, num, G, l1, l2, jacobi=True)
    assert np.abs(Fj - Fc).max() > 1e-3                 # the coupling is strong enough to tell the orders apart
    # the kernel's denominator floor: below FLT_MIN -> eps, exactly as sklearn's den == 0 -> eps on a zero row
    G0 = G.copy()
    G0[3] = 0.0
    ref = kernel_ref.mu_half_step(W.T, num, G0, 0.0, 0.0)
    assert np.allclose(ref[3], W.T[3] * num[3] / kernel_ref.EPSILON, rtol=1e-15)


@pytest.mark.parametrize("l1,l2", [(0.0, 0.0), (0.3, 0.0), (0.0, 0.7), (0.25, 1.5)])
@pytest.mark.parametrize("beta", [1, 0])
def test_beta_step_references_match_sklearn(beta, l1, l2):
    """oracle/kernel_ref.py's KL / IS references -- what tests/test_beta_units.py holds the beta kernels to -- against
    scikit-learn in float64: _multiplicative_update_w / _h (gamma = 1 / (2 - beta) for beta < 1, else 1) plus the flush
    of _fit_multiplicative_update, and _beta_divergence.  Layout: W half F = W^T, Foth = H, D = X^T; H half F = H,
    Foth = W^T, D = X.  The data has a zero component (zero KL sums, zero IS numerators and denominators), entries of
    WH below eps, exact zeros and values at float32 eps in X, and values that the update drives below float64 eps."""
    from sklearn.decomposition import _nmf
    from oracle import kernel_ref
    rng = np.random.RandomState(int(10 * l1 + 100 * l2) + beta)
    n, g, K = 50, 40, 6
    X = rng.uniform(0.2, 3.0, (n, g))
    X[3, :5] = 0.0
    X[4, :3] = kernel_ref.EPSILON
    X[5, :3] = 2 * kernel_ref.EPSILON
    W = rng.uniform(0.1, 1.5, (n, K))
    H = rng.uniform(0.1, 1.5, (K, g))
    W[:, 2] = 0.0                        # dead component: zero W sum (KL), zero numerator and denominator of H row 2
    H[4, :] = 0.0                        # dead component for the W half
    W[7, :] = 0.0                        # WH = 0 on a whole row: floored at eps
    W[9, 1] = 1e-20                      # driven towards 0: below float64 eps after the update
    H[1, 8] = 1e-20
    gamma = 0.5 if beta == 0 else 1.0
    Wn, *_ = _nmf._multiplicative_update_w(X, W.copy(), H, beta, l1, l2, gamma)
    Wc = Wn.copy()
    if beta < 1:
        Wc[Wc < np.finfo(np.float64).eps] = 0.0
    Fw = kernel_ref.beta_half_step(W.T, X.T, H, beta, "W", l1, l2)
    assert np.allclose(Fw, Wc.T, rtol=1e-13, atol=0)
    assert (Fw.T[9, 1] == 0.0) == (beta < 1) and (Fw.T[9, 1] > 0) == (beta == 1)
    Hn = _nmf._multiplicative_update_h(X, W, H.copy(), beta, l1, l2, gamma)
    Hn[Hn < np.finfo(np.float64).eps] = 0.0
    Fh = kernel_ref.beta_half_step(H, X, W.T, beta, "H", l1, l2)
    assert np.allclose(Fh, Hn, rtol=1e-13, atol=0)
    assert Fh[1, 8] == 0.0 and np.isfinite(Fh).all() and np.isfinite(Fw).all()
    for b in (beta, 2):
        ref = _nmf._beta_divergence(X, W, H, b, square_root=True)
        t, sx, res, err = kernel_ref.beta_terms(X.T, W.T, H, b)
        assert abs(err - ref) <= 1e-12 * ref, (b, err, ref)
        half = 2.0 if b == 2 else 1.0              # scikit-learn's Frobenius res is half the squared norm
        assert res == pytest.approx(half * _nmf._beta_divergence(X, W, H, b, square_root=False), rel=1e-12)
        assert kernel_ref.beta_terms(X, H, W.T, b)[3] == pytest.approx(err, rel=1e-13)
        WH = W @ H
        keep = X > kernel_ref.EPSILON
        if b == 1:         # the kernel's split: sum(WH) over the dropped entries, plus the floor's share on the rest
            assert sx == pytest.approx(WH[~keep].sum() + (WH[keep] - np.maximum(WH[keep], kernel_ref.EPSILON)).sum(),
                                       rel=1e-13)
            assert (WH[keep] < kernel_ref.EPSILON).any()
        elif b == 0:
            assert sx == keep.sum() and t >= 0


def test_float64_eps_rule_matches_sklearn():
    """kernel_ref.mu_half_step(eps_rule='zero') -- what tests/test_fp64_units.py holds the float64 MU kernel to --
    against scikit-learn's _multiplicative_update_w on denominators that are exactly 0 (-> float32 eps) and positive
    below FLT_MIN (used as they are), where the fp32 kernels' floor rule differs."""
    from sklearn.decomposition import _nmf
    from oracle import kernel_ref
    rng = np.random.RandomState(3)
    n, K = 40, 6
    W = np.abs(rng.randn(n, K)) + 0.1
    G = np.abs(rng.randn(K, K))
    G = G @ G.T
    G[2] = 0.0                           # den == 0 on row 2 of the update (sklearn reads G transposed: HHt = G.T)
    G[4] = 1e-300 * np.abs(rng.rand(K))   # 0 < den < FLT_MIN on row 4
    num = np.abs(rng.randn(K, n))
    Wm, *_ = _nmf._multiplicative_update_w(np.zeros((n, 3)), W.copy(), np.zeros((K, 3)), 2, 0.0, 0.0, 1.0,
                                           HHt=G.T.copy(), XHt=num.T.copy(), update_H=False)
    ref = kernel_ref.mu_half_step(W.T, num, G, eps_rule="zero")
    assert np.allclose(ref, Wm.T, rtol=1e-13, atol=0)
    den = G @ W.T
    assert (den[4] > 0).all() and (den[4] < kernel_ref.FLT_MIN).all()
    assert np.array_equal(ref[2], W.T[2] * num[2] / kernel_ref.EPSILON)
    floor = kernel_ref.mu_half_step(W.T, num, G)
    assert np.array_equal(floor[2], ref[2]) and not np.allclose(floor[4], ref[4])
    ld = kernel_ref.mu_half_step(W.T, num, G, eps_rule="zero", dtype=np.longdouble)
    assert np.allclose(ld.astype(np.float64), ref, rtol=1e-15, atol=0)


def _mu_replay(errors, tol, max_iter):
    """n_iter of the MU loop driven by kernel_ref.mu_stop over errors[it] (it = 0 is the error at init)."""
    from oracle import kernel_ref
    prev = errors[0]
    for it in range(1, max_iter + 1):
        stop, prev = kernel_ref.mu_stop(it, errors.get(it), errors[0], prev, tol, max_iter)
        if stop:
            return it
    raise AssertionError("mu_stop never stopped the loop")


@pytest.mark.parametrize("tol,max_iter", [(1e-3, 400), (1e-2, 400), (1e-4, 13), (0.0, 25), (1e-4, 30)])
def test_mu_stop_restates_the_mu_loop(golden, tol, max_iter):
    """kernel_ref.mu_stop -- the decision the MU convergence kernel is held to -- replayed over the errors
    nmf_ref.mu_frobenius evaluates gives its n_iter: checks at multiples of 10 only, strict <, the end at max_iter."""
    X = golden["X"]
    W, H = nmf_ref.init_random(X.mean(), X.shape[0], X.shape[1], 4, 11)
    seen = []

    def record(X_, W_, H_):
        e = nmf_ref.frobenius_error(X_, W_, H_)
        seen.append(e)
        return e

    _, _, n_iter = nmf_ref.mu_frobenius(X, W, H, tol=tol, max_iter=max_iter, error_fn=record)
    errors = {0: seen[0]}
    errors.update({10 * (i + 1): e for i, e in enumerate(seen[1:])})
    assert _mu_replay(errors, tol, max_iter) == n_iter


def test_mu_stop_edges():
    """The branches the fixtures never reach: err0 == 0 with err == 0 (NaN quotient: runs on), the tol boundary
    (equality continues), prev advancing only on a continue, no look at the error off the multiples of 10."""
    from oracle import kernel_ref as kr
    assert kr.mu_stop(10, 0.0, 0.0, 0.0, 1e-4, 100) == (False, 0.0)
    assert kr.mu_stop(100, 0.0, 0.0, 0.0, 1e-4, 100) == (True, 0.0)
    assert kr.mu_stop(10, 2.0, 4.0, 3.0, 0.25, 100) == (False, 2.0)        # (3 - 2) / 4 == tol: continues
    assert kr.mu_stop(10, 2.0, 4.0, 3.0, np.nextafter(0.25, 1), 100) == (True, 3.0)
    assert kr.mu_stop(13, None, 4.0, 3.0, 0.25, 13) == (True, 3.0)
    assert kr.mu_stop(7, None, 4.0, 3.0, 0.25, 100) == (False, 3.0)


@pytest.mark.parametrize("tol,max_iter,l2", [(1e-4, 200, 0.0), (1e-2, 200, 0.5), (0.0, 7, 0.0)])
def test_cd_stop_restates_the_cd_loop(golden, tol, max_iter, l2):
    """kernel_ref.cd_stop replayed over nmf_ref's own half-sweeps gives cd_frobenius's n_iter and factors (<=, viol0
    from iteration 1), and an all-zero problem -- viol0 == 0 -- stops at iteration 1."""
    from oracle import kernel_ref as kr
    X = golden["X"]
    W0, H0 = nmf_ref.init_random(X.mean(), X.shape[0], X.shape[1], 4, 5)
    Wr, Hr, n_ref = nmf_ref.cd_frobenius(X, W0, H0, tol=tol, max_iter=max_iter, l2_reg_W=l2, l2_reg_H=l2)
    W, Ht = W0.copy(), np.ascontiguousarray(H0.T.copy())
    viol0 = None
    for it in range(1, max_iter + 1):
        HHt = Ht.T @ Ht + l2 * np.eye(4)
        viol = nmf_ref._cd_sweep(W, HHt, X @ Ht)
        WtW = W.T @ W + l2 * np.eye(4)
        viol += nmf_ref._cd_sweep(Ht, WtW, X.T @ W)
        stop, viol0 = kr.cd_stop(it, viol, viol0, tol, max_iter)
        if stop:
            break
    assert it == n_ref and np.array_equal(W, Wr) and np.array_equal(Ht.T, Hr)
    Z = np.zeros_like(X)
    _, _, n_zero = nmf_ref.cd_frobenius(Z, np.zeros_like(W0), np.zeros_like(H0), tol=tol, max_iter=max_iter)
    assert n_zero == 1 and kr.cd_stop(1, 0.0, None, tol, max_iter) == (True, 0.0)
    assert kr.cd_stop(3, 0.25, 1.0, 0.25, 100)[0] and not kr.cd_stop(3, 0.25, 1.0, np.nextafter(0.25, 0), 100)[0]


# ------------------------------------------------------------------------------------ dataset operand restatement
def test_dataset_ref_detection_pins_todays_policy():
    """oracle/dataset_ref.py restates exact-count detection (tests/test_dataset_units.py compares the device with it
    bit for bit).  The reference's own matrices take the exact forms: the normalised HVG counts (counts / std) with a
    column scale, TPM (counts * 1e6 / total) with a row scale.  A count of 2049, a column whose smallest count is 2 and
    a matrix with both a row and a column scale take the general form."""
    from cnmf_golden import load_golden
    from oracle import dataset_ref as dr
    g = load_golden("sim_mu")
    X, tpm = g["X"].astype(np.float32), g["tpm"].astype(np.float32)
    for precision, exact in (("tf32x3", "tf32_exact"), ("f16x2", "f16_exact")):
        form, rs, cs = dr.decide(X, precision)
        assert form == exact and rs is None and cs is not None
        assert np.array_equal(dr.counts(X, rs, cs)[:, :X.shape[1]], g["counts"][:, g["hvg_idx"]])
        form, rs, cs = dr.decide(tpm, precision)
        assert form == exact and rs is not None and cs is None
        assert np.array_equal(dr.counts(tpm, rs, cs)[:, :tpm.shape[1]], g["counts"])
    assert dr.decide(X, "tf32x3-general") == ("tf32", None, None)
    assert dr.decide(X, "fp32") == ("fp32", None, None)
    rng = np.random.RandomState(0)
    C = rng.poisson(3.0, (40, 30)).astype(np.float32)
    C[:, 0] = np.maximum(C[:, 0], 1)
    assert dr.decide(C, "tf32x3")[0] == "tf32_exact"
    C2 = C.copy()
    C2[5, 7] = 2049
    assert dr.decide(C2, "tf32x3")[0] == "tf32"
    C3 = C.copy()
    C3[:, 4] = np.where(C3[:, 4] > 0, 2 * C3[:, 4] + 1, 0)         # odd counts ...
    C3[np.flatnonzero(C3[:, 4])[0], 4] = 2                          # ... and one 2: the column scale 2 fails them
    assert dr.decide(C3, "tf32x3")[0] == "tf32"
    both = (C * (1.0 + rng.rand(40, 1)) * (1.0 + rng.rand(1, 30))).astype(np.float32)
    assert dr.decide(both, "tf32x3")[0] == "tf32"
    # the admission bound: 3e-7 n is admitted, 8e-7 n is not (n = 1000: far from the other rounding terms)
    base = np.full((4, 4), 1000.0, np.float32)
    base[0, 0] = 1.0
    for rel, exact in ((3e-7, True), (8e-7, False)):
        P = base.copy()
        P[2, 3] = np.float32(1000.0 * (1.0 + rel))
        assert (dr.decide(P, "tf32x3")[0] == "tf32_exact") == exact, rel


def test_dataset_ref_to_tf32_is_cvt_rna():
    """to_tf32 (the add-0x1000-and-mask form of common.cuh) is cvt.rna.tf32.f32: the nearest value with 10 stored
    mantissa bits, ties away from zero, on a few thousand bit patterns (all exponents, the tie and its neighbours)."""
    from oracle import dataset_ref as dr
    rng = np.random.RandomState(1)
    exps = rng.randint(1, 254, 4000).astype(np.uint32)
    mant = rng.randint(0, 1 << 23, 4000).astype(np.uint32)
    mant[:600] = (mant[:600] & ~np.uint32(0x1fff)) | np.uint32(0x1000)        # exact ties
    mant[600:900] = (mant[600:900] & ~np.uint32(0x1fff)) | np.uint32(0x0fff)  # just below
    mant[900:1200] = (mant[900:1200] & ~np.uint32(0x1fff)) | np.uint32(0x1001)  # just above
    mant[1200:1300] = np.uint32(0x7fffff)                                     # carries into the exponent
    sign = (rng.rand(4000) < 0.5).astype(np.uint32) << np.uint32(31)
    bits = sign | (exps << np.uint32(23)) | mant
    x = bits.view(np.float32)
    got = dr.to_tf32(x)
    # direct definition: |x| = m * 2^e with m = mant / 2^13 (step 1 of the kept mantissa), round half away from zero
    ax = np.abs(x.astype(np.float64))
    e = np.frexp(ax)[1] - 1                    # ax in [2^e, 2^(e + 1))
    step = np.ldexp(1.0, e - 10)
    want = np.sign(x) * np.floor(ax / step + 0.5) * step
    assert np.array_equal(got.astype(np.float64), want)
    assert (got.view(np.uint32) & np.uint32(0x1fff) == 0).all()
    hi, lo = dr.split_tf32(x)
    normal = (ax > 2.0 ** -100) & (ax < 2.0 ** 100)        # lo neither subnormal nor beyond fp32
    assert np.array_equal(hi, got)
    assert (np.abs(x.astype(np.float64) - hi - lo) <= ax * 2.0 ** -22)[normal].all()
