"""ORACLE (test infrastructure) -- numpy restatement of the batched KMeans fit (cnmf_b200/csrc/kmeans_batched.cu,
cnmf_kmeans_fit) in the device's order of operations, run by run.

T is the element type of the spectra (float32, or float64 under precision='fp64').  The rules:
  * k-means++ closest distances: differences in T, squares summed in float64, rounded to T;
  * potentials: blocks of 8 rows summed in row order, then the blocks summed sequentially;
  * candidates: searchsorted(side='left') on a sequential float64 cumulative sum, clipped to R - 1;
  * argmin and the E step: the first minimum wins;
  * M step: float64 column sums in member (row) order, centre = sums * (1 / count), the E step reading the centres
    rounded to T; stop when no label changed, the total squared shift is <= tol_abs, or max_iter iterations ran;
    then a final E step against the last centres.
The E-step distances here are float64 sums; the device's are T sums.  Every E-step decision is returned with its
relative gap, so a test can check that the data decides it the same way in T (see `e_step_bound`).
"""
import numpy as np


def row_dists(S, idx):
    """Squared distances of every row of S to rows `idx` of S (n_c x R, float64 holding T values)."""
    T = S.dtype
    d = (S[None, :, :] - S[np.asarray(idx)][:, None, :]).astype(T)       # differences in T
    return (d.astype(np.float64) ** 2).sum(axis=2).astype(T).astype(np.float64)


def block_potential(v):
    """Sum of v in the device's order: blocks of 8 rows in order, then the blocks sequentially."""
    n = len(v)
    P = np.zeros(((n + 7) // 8) * 8)
    P[:n] = v
    P = P.reshape(-1, 8)
    part = P[:, 0].copy()
    for w in range(1, 8):
        part = part + P[:, w]
    return float(np.cumsum(part)[-1])


def kmeans_plusplus(S, k, first, unif, n_trials):
    """Centre indices of one run.  first: the first centre; unif: (k - 1) x n_trials uniforms."""
    R = S.shape[0]
    closest = row_dists(S, [first])[0]
    pot = block_potential(closest)
    idx = [int(first)]
    for step in range(1, k):
        rv = np.asarray(unif[step - 1][:n_trials], dtype=np.float64) * pot
        cand = np.minimum(np.searchsorted(np.cumsum(closest), rv, side="left"), R - 1)
        d = np.minimum(closest[None, :], row_dists(S, cand))
        cpot = np.array([block_potential(dj) for dj in d])
        best = int(np.argmin(cpot))
        pot = float(cpot[best])
        closest = d[best]
        idx.append(int(cand[best]))
    return np.array(idx, dtype=np.int64)


def _e_step(S64, CE64):
    """Labels (first minimum), float64 distances to the chosen centre, relative gap of every decision."""
    D = ((S64[:, None, :] - CE64[None, :, :]) ** 2).sum(axis=2)
    labels = np.argmin(D, axis=1)
    best = D[np.arange(len(D)), labels]
    if D.shape[1] > 1:
        rest = D.copy()
        rest[np.arange(len(D)), labels] = np.inf
        second = rest.min(axis=1)
        gap = (second - best) / np.maximum(second + best, 1e-300)
    else:
        gap = np.full(len(D), np.inf)
    return labels.astype(np.int32), best, gap


def e_step_bound(G, T):
    """Relative error of one device E-step distance (kmeans_assign_kernel / kmb_assign_kernel): each difference rounds
    once in T (2 u in its square), each lane chains ceil(G / 32) fmas over non-negative terms, and the warp tree adds
    5 roundings.  A decision whose relative gap (d2 - d1) / (d2 + d1) exceeds this is the same in T as in float64."""
    u = 2.0 ** -24 if np.dtype(T) == np.float32 else 2.0 ** -53
    return (-(-G // 32) + 8) * u * 1.01


def lloyd(S, centre_idx, max_iter, tol_abs):
    """One run's Lloyd loop from k-means++ centres.  Returns a dict: labels, inertia (float64 sum of float64 distances
    to the final T centres), n_iter, empty (an empty cluster stopped the run: the device hands over to the host path),
    min_gap (smallest relative gap of any E-step decision), tol_gap (smallest |shift - tol_abs| / tol_abs of the
    shift tests that ran), centres (float64)."""
    T = S.dtype
    S64 = S.astype(np.float64)
    k = len(centre_idx)
    C64 = S64[centre_idx].copy()
    prev = np.full(S.shape[0], -1, np.int32)
    min_gap, tol_gap = np.inf, np.inf
    n_iter = 0
    while True:
        labels, _, gap = _e_step(S64, C64.astype(T).astype(np.float64))
        min_gap = min(min_gap, float(gap.min()))
        n_changed = int((labels != prev).sum())
        prev = labels
        counts = np.bincount(labels, minlength=k)
        n_iter += 1
        if (counts == 0).any():
            return dict(labels=labels, inertia=None, n_iter=n_iter, empty=True, min_gap=min_gap, tol_gap=tol_gap,
                        centres=C64)
        sums = np.zeros((k, S.shape[1]))
        np.add.at(sums, labels, S64)                      # row order, per cluster
        new = sums * (1.0 / counts.astype(np.float64))[:, None]
        shift = float(((new - C64) ** 2).sum())
        C64 = new
        if n_changed == 0:
            break
        if tol_abs > 0:
            tol_gap = min(tol_gap, abs(shift - tol_abs) / tol_abs)
        if shift <= tol_abs or n_iter >= max_iter:
            break
    labels, dist, gap = _e_step(S64, C64.astype(T).astype(np.float64))
    min_gap = min(min_gap, float(gap.min()))
    return dict(labels=labels, inertia=float(dist.sum()), n_iter=n_iter, empty=False, min_gap=min_gap,
                tol_gap=tol_gap, centres=C64)


def kmeans_fit(S, k, first, unif, n_trials, max_iter, tol_abs):
    """Every run of cnmf_kmeans_fit.  first: n_init first-centre indices; unif: n_init x (k - 1) x n_trials uniforms
    (consensus._kmeans_draws).  Returns one lloyd() dict per run, with its centre_idx."""
    runs = []
    for t in range(len(first)):
        idx = kmeans_plusplus(S, k, first[t], unif[t], n_trials)
        r = lloyd(S, idx, max_iter, tol_abs)
        r["centre_idx"] = idx
        runs.append(r)
    return runs


def best_run(runs, k):
    """scikit-learn's choice of run (_kmeans.py:1534-1541): lower inertia and a different clustering."""
    from .consensus_ref import _same_clustering
    best = None
    for r in runs:
        if best is None or (r["inertia"] < best["inertia"] and not _same_clustering(r["labels"], best["labels"], k)):
            best = r
    return best
