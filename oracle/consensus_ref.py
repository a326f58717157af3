"""ORACLE (test infrastructure) -- numpy restatement of the numerics of ``cNMF.consensus``
(cnmf.py:823-985) and of the scikit-learn 1.9.0 routines it calls (``SK/`` = site-packages/
sklearn; third-party, not part of the reference).  Each function cites what it restates.
Pinned by tests/test_oracle_golden.py against fixtures the reference itself produced
(oracle/make_golden.py).
"""
import numpy as np

from . import nmf_ref


def l2_normalize_rows(S):
    """cnmf.py:882."""
    return (S.T / np.sqrt((S ** 2).sum(axis=1))).T


def euclidean_distances(X):
    """SK/metrics/pairwise.py:376-427 for Y is X, float64 input:
    sqrt(max(||x||^2 + ||y||^2 - 2 x.y, 0)), diagonal forced to 0."""
    XX = (X * X).sum(axis=1)[:, None]
    D = -2.0 * (X @ X.T)
    D += XX
    D += XX.T
    np.maximum(D, 0, out=D)
    np.fill_diagonal(D, 0)
    return np.sqrt(D)


def local_density(D, n_neighbors):
    """cnmf.py:893-896: mean over the n nearest neighbours = (sum of the n+1 smallest
    entries of each row, which include the 0 self-distance) / n."""
    part = np.partition(D, n_neighbors + 1, axis=1)[:, : n_neighbors + 1]
    return part.sum(axis=1) / n_neighbors


# ---------------------------------------------------------------- KMeans -----------------

def _sq_dists(C, X, x_sq):
    """SK/metrics/pairwise.py:_euclidean_distances(squared=True): ||c||^2 - 2 c.x + ||x||^2,
    clamped at 0 (and exactly 0 is NOT forced for identical rows when X is not Y)."""
    cc = (C * C).sum(axis=1)[:, None]
    D = -2.0 * (C @ X.T)
    D += cc
    D += x_sq[None, :]
    np.maximum(D, 0, out=D)
    return D


def kmeans_plusplus(X, k, x_sq, rng):
    """SK/cluster/_kmeans.py:180-278 with unit sample weights."""
    n = X.shape[0]
    n_local_trials = 2 + int(np.log(k))
    w = np.ones(n)
    centers = np.empty((k, X.shape[1]), dtype=X.dtype)
    cid = rng.choice(n, p=w / w.sum())
    indices = [cid]
    centers[0] = X[cid]
    closest = _sq_dists(centers[0:1], X, x_sq)
    pot = closest @ w
    for c in range(1, k):
        rand_vals = rng.uniform(size=n_local_trials) * pot
        cand = np.searchsorted(np.cumsum(w * closest), rand_vals)
        np.clip(cand, None, closest.size - 1, out=cand)
        d = _sq_dists(X[cand], X, x_sq)
        np.minimum(closest, d, out=d)
        cpot = d @ w.reshape(-1, 1)
        best = int(np.argmin(cpot))
        pot = cpot[best]
        closest = d[best][None, :]
        centers[c] = X[cand[best]]
        indices.append(int(cand[best]))
    return centers, np.array(indices)


def _lloyd_iter(X, centers, update_centers=True):
    """SK/cluster/_k_means_lloyd.pyx:168-219 (E+M for all rows) + empty-cluster relocation
    (_k_means_common.pyx:167-211) + _average_centers (:274-298) + _center_shift (:301-316)."""
    k = centers.shape[0]
    pd_ = (centers * centers).sum(axis=1)[None, :] - 2.0 * (X @ centers.T)
    labels = np.argmin(pd_, axis=1).astype(np.int32)   # first minimum wins, like the strict '<'
    if not update_centers:
        return labels, None, None
    weight = np.bincount(labels, minlength=k).astype(X.dtype)
    new = np.zeros_like(centers)
    np.add.at(new, labels, X)
    empty = np.where(weight == 0)[0]
    if len(empty) > 0:
        dist = ((X - centers[labels]) ** 2).sum(axis=1)
        if dist.max() != 0:
            far = np.argpartition(dist, -len(empty))[: -len(empty) - 1: -1]
            for idx, new_id in enumerate(empty):
                fi = far[idx]
                old_id = labels[fi]
                new[old_id] -= X[fi]
                new[new_id] = X[fi]
                weight[new_id] = 1
                weight[old_id] -= 1
    amax = int(np.argmax(weight))
    for j in range(k):
        if weight[j] > 0:
            new[j] *= 1.0 / weight[j]
        else:
            new[j] = new[amax]
    shift = np.sqrt(((new - centers) ** 2).sum(axis=1))
    return labels, new, shift


def kmeans_single_lloyd(X, centers_init, max_iter=300, tol=1e-4):
    """SK/cluster/_kmeans.py:630-758."""
    centers = centers_init.copy()
    labels_old = np.full(X.shape[0], -1, dtype=np.int32)
    strict = False
    it = 0
    for it in range(max_iter):
        labels, new, shift = _lloyd_iter(X, centers)
        centers = new
        if np.array_equal(labels, labels_old):
            strict = True
            break
        if (shift ** 2).sum() <= tol:
            break
        labels_old = labels
    if not strict:
        labels, _, _ = _lloyd_iter(X, centers, update_centers=False)
    inertia = ((X - centers[labels]) ** 2).sum()
    return labels, inertia, centers, it + 1


def _same_clustering(l1, l2, k):
    """SK/cluster/_k_means_common.pyx:319-330."""
    mapping = np.full(k, -1, dtype=np.int64)
    for a, b in zip(l1, l2):
        if mapping[a] == -1:
            mapping[a] = b
        elif mapping[a] != b:
            return False
    return True


def kmeans(X, k, n_init=10, random_state=1, max_iter=300, tol=1e-4):
    """KMeans(n_clusters=k, n_init=10, random_state=1).fit(X).labels_ (cnmf.py:908-910),
    SK/cluster/_kmeans.py:1436-1563 (lloyd, k-means++ init, unit weights)."""
    X = np.array(X, dtype=np.float64, order="C")
    rng = np.random.RandomState(random_state)
    mean = X.mean(axis=0)
    X = X - mean
    tol_abs = np.mean(np.var(X, axis=0)) * tol       # _tolerance, :285-293 (on centred X: same var)
    x_sq = (X * X).sum(axis=1)
    best = None
    for _ in range(n_init):
        c0, _idx = kmeans_plusplus(X, k, x_sq, rng)
        labels, inertia, centers, n_it = kmeans_single_lloyd(X, c0, max_iter, tol_abs)
        if best is None or (inertia < best[1] and not _same_clustering(labels, best[0], k)):
            best = (labels, inertia, centers, n_it)
    return best[0], best[1], best[2] + mean


# ---------------------------------------------------------------- medians / OLS ----------

def cluster_medians(l2, labels, k):
    """cnmf.py:913-916: per-cluster, per-gene median (pandas groupby.median: mean of the two
    middle values for even counts), then each row divided by its sum. labels are 0-based."""
    M = np.vstack([np.median(l2[labels == c], axis=0) for c in range(k)])
    return (M.T / M.sum(axis=1)).T


def ols_zscore(U, T):
    """efficient_ols_all_cols(U, T, normalize_y=True) (cnmf.py:55-125): z-score the columns of
    T with the population mean/variance (StandardScaler, cnmf.py:131-134; var floored at 1e-12),
    accumulate the normal equations, lstsq."""
    mean = T.mean(axis=0)
    var = T.var(axis=0)
    var[var < 1e-12] = 1e-12
    Z = (T - mean) / np.sqrt(var)
    XtX = U.T @ U
    XtY = U.T @ Z
    beta, *_ = np.linalg.lstsq(XtX, XtY, rcond=None)
    return beta


def silhouette(l2, labels):
    """sklearn.metrics.silhouette_score(metric='euclidean') (cnmf.py:923)."""
    D = euclidean_distances(l2)
    ks = np.unique(labels)
    n = len(labels)
    A = np.zeros(n)
    B = np.full(n, np.inf)
    for c in ks:
        m = labels == c
        s = D[:, m].sum(axis=1)
        cnt = m.sum()
        inn = m
        A[inn] = s[inn] / max(cnt - 1, 1)
        out = ~m
        B[out] = np.minimum(B[out], s[out] / cnt)
    sil = (B - A) / np.maximum(A, B)
    sizes = np.array([(labels == labels[i]).sum() for i in range(n)])
    sil[sizes == 1] = 0
    return float(np.nan_to_num(sil).mean())


def consensus(merged, X, tpm, tpm_std, hvg_idx, k, density_threshold=0.5,
              local_neighborhood_size=0.30, solver="mu", tol=1e-4, max_iter=1000,
              refit_usage=True, beta=2):
    """Numeric part of cNMF.consensus (cnmf.py:871-975) on plain arrays.

    merged   R x G stacked spectra (f64)       X    N x G normalised counts
    tpm      N x G_all                          tpm_std  per-gene std(ddof=0) (tpm_stats.__std)
    hvg_idx  positions of the G HVGs inside the G_all TPM columns
    Returns a dict with every intermediate the CUDA path is compared on.
    """
    R = merged.shape[0]
    n_neighbors = int(local_neighborhood_size * R / k)
    l2 = l2_normalize_rows(merged)
    D = euclidean_distances(l2)
    dens = local_density(D, n_neighbors)
    keep = dens < density_threshold
    l2f = l2[keep]
    if l2f.shape[0] == 0:
        raise RuntimeError("Zero components remain after density filtering. Consider increasing density threshold")
    labels, inertia, _ = kmeans(l2f, k)
    med = cluster_medians(l2f, labels, k)
    rf, _ = nmf_ref.refit(X, med, solver, tol, max_iter, beta=beta)
    norm_usages = rf / rf.sum(axis=1, keepdims=True)
    order = np.argsort(-norm_usages.sum(axis=0), kind="stable")
    rf = rf[:, order]
    norm_usages = norm_usages[:, order]
    med = med[order]
    spectra_tpm_T, _ = nmf_ref.refit(tpm.T, norm_usages.T, solver, tol, max_iter, beta=beta)
    spectra_tpm = spectra_tpm_T.T
    score = ols_zscore(rf, tpm)
    usages = rf
    if refit_usage:
        norm_tpm = tpm[:, hvg_idx] / tpm[:, hvg_idx].std(axis=0, ddof=1)
        sp_rf = spectra_tpm[:, hvg_idx] / tpm_std[hvg_idx]
        usages, _ = nmf_ref.refit(norm_tpm, sp_rf, solver, tol, max_iter, beta=beta)
    return dict(l2=l2, local_density=dens, keep=keep, labels=labels, inertia=inertia,
                consensus_spectra=med, consensus_usages=usages,
                gene_spectra_tpm=spectra_tpm, gene_spectra_score=score, order=order)
