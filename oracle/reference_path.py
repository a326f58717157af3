"""ORACLE / CPU BASELINE (test infrastructure) -- the reference's own call sequence for the hot path,
executed on scikit-learn exactly as the reference's src/cnmf/cnmf.py does:

  factorize : one `non_negative_factorization(X, **kwargs)` per (k, seed) job, sequentially
              (cnmf.py:735-745 -> _nmf, cnmf.py:661-674), kwargs from get_nmf_iter_params (cnmf.py:618-631)
  consensus : the numeric steps of cnmf.py:871-975 with sklearn KMeans / euclidean_distances

scikit-learn is a third-party dependency of the reference that IS part of the image, so this module
runs anywhere (unlike the reference checkout itself).  Only tests/, __graft_entry__.smoke() and
bench.py's cpu_baseline / --impl reference arm may call it.
"""
import time
import warnings

import numpy as np


def nmf_kwargs(solver="mu", tol=1e-4, max_iter=1000, beta_loss=None):
    """cnmf.py:618-631: beta_loss='frobenius' -> solver 'cd' (the reference default); a float
    beta_loss=2.0 keeps solver 'mu' (SURVEY.md fact 3); 'kullback-leibler' / 'itakura-saito' keep 'mu'."""
    kw = dict(alpha_W=0.0, alpha_H=0.0, l1_ratio=0.0, beta_loss="frobenius", solver="mu", tol=tol,
              max_iter=max_iter, init="random")
    if beta_loss not in (None, "frobenius", 2, 2.0):
        kw["beta_loss"] = beta_loss
    elif solver == "cd":
        kw["solver"] = "cd"
    else:
        kw["beta_loss"] = 2.0
    return kw


def factorize(X, jobs, solver="mu", tol=1e-4, max_iter=1000, beta_loss=None):
    """jobs: list of (k, seed).  Returns (list of spectra, list of n_iter, seconds)."""
    from sklearn.decomposition import non_negative_factorization
    kw = nmf_kwargs(solver, tol, max_iter, beta_loss)
    X = np.asarray(X, dtype=np.float64)              # cnmf.py:534
    out, its = [], []
    t0 = time.perf_counter()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for (k, seed) in jobs:
            kw["random_state"] = int(seed)
            kw["n_components"] = int(k)
            W, H, it = non_negative_factorization(X, **kw)
            out.append(H)
            its.append(int(it))
    return out, its, time.perf_counter() - t0


def consensus_cluster(merged, k, density_threshold=0.5, local_neighborhood_size=0.30):
    """cnmf.py:879-916 on sklearn: returns (local_density, keep mask, labels, median_spectra)."""
    from sklearn.cluster import KMeans
    from sklearn.metrics.pairwise import euclidean_distances
    merged = np.asarray(merged, dtype=np.float64)
    n_neighbors = int(local_neighborhood_size * merged.shape[0] / k)
    l2 = (merged.T / np.sqrt((merged ** 2).sum(axis=1))).T
    D = euclidean_distances(l2)
    part = np.argpartition(D, n_neighbors + 1)[:, :n_neighbors + 1]
    dens = D[np.arange(D.shape[0])[:, None], part].sum(1) / n_neighbors
    keep = dens < density_threshold
    l2f = l2[keep]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        labels = KMeans(n_clusters=k, n_init=10, random_state=1).fit(l2f).labels_
    med = np.vstack([np.median(l2f[labels == c], axis=0) for c in range(k)])
    med = (med.T / med.sum(1)).T
    return dens, keep, labels, med
