"""Host orchestration of the consensus stage (cnmf.py:871-975) over the CUDA kernels.

What runs where
  * GPU (libcnmf_b200.so): L2 normalisation, all-pairs distances, k-NN local density, the Lloyd
    E+M steps, k-means++ candidate distances, per-cluster medians, the three NNLS refits and the
    OLS projection GEMM.
  * Host (numpy, O(R) or O(K*G) work only): the k-means++ random draws (they must consume the
    legacy RandomState(1) stream exactly like sklearn/cluster/_kmeans.py:231-262), centre averaging,
    the K x K least-squares solve, bookkeeping.

torch is used purely as the device-memory container (allocation + memcpy); no torch op touches
the data.  There is no CPU fallback: without the CUDA library / a GPU this module raises.
"""
import ctypes

import numpy as np

from ._lib import check, ptr


# work counters of the last consensus_numerics call (bench.py's consensus roofline): Lloyd iterations summed over the
# n_init runs, (rows, cols, n_iter) of every refit
STATS = {}


class _few_blas_threads:
    """The host-side linear algebra of this stage is tiny (K x K solves, N x K Gram products).  On a 128-core host a
    BLAS pool of 128 threads wakes up for each of them and the wake-up, not the arithmetic, becomes the cost (tens of ms
    at random points of a stage whose GPU work takes milliseconds).  Four threads for the duration of the stage."""

    def __enter__(self):
        try:
            from threadpoolctl import threadpool_limits
            self._ctx = threadpool_limits(limits=4)
            self._ctx.__enter__()
        except Exception:
            self._ctx = None
        return self

    def __exit__(self, *exc):
        if self._ctx is not None:
            self._ctx.__exit__(*exc)
        return False


def _torch():
    import torch
    if not torch.cuda.is_available():
        raise RuntimeError("cnmf_b200.consensus needs a CUDA device (no CPU fallback)")
    return torch


class SpectraMatrix:
    """R x G matrix on the device (row stride ld = G padded to 32), float32 or float64 (dtype).  A float64 matrix
    (precision='fp64') runs every consensus kernel on its _f64 entry point: distances, densities, KMeans centres and
    medians stay in float64."""

    def __init__(self, engine, array=None, shape=None, dtype=np.float32):
        torch = _torch()
        self.engine = engine
        self.lib = engine.lib
        self.dtype = np.dtype(dtype)
        if self.dtype not in (np.float32, np.float64):
            raise ValueError("SpectraMatrix: dtype must be float32 or float64, not %s" % self.dtype)
        self.fp64 = self.dtype == np.float64
        if array is not None:
            array = np.ascontiguousarray(array, dtype=self.dtype)
            shape = array.shape
        self.R, self.G = int(shape[0]), int(shape[1])
        self.ld = (self.G + 31) // 32 * 32
        self.t = torch.zeros((self.R, self.ld), dtype=self.torch_dtype, device="cuda:%d" % engine.device)
        if array is not None:
            self.t[:, :self.G].copy_(torch.from_numpy(array))     # H2D memcpy

    @property
    def torch_dtype(self):
        return _torch().float64 if self.fp64 else _torch().float32

    def fn(self, name):
        """The library entry point `name` for this matrix's element type (name + '_f64' for a float64 matrix)."""
        return getattr(self.lib, name + "_f64" if self.fp64 else name)

    @classmethod
    def from_device_rows(cls, engine, src_ptr, ld_src, rows, n_cols, dtype=np.float32):
        """Rows `rows` of a device-resident slab of `dtype` (e.g. the all-gathered spectra of every restart) as a new
        matrix: a device-side row gather, no trip through the host."""
        rows = np.ascontiguousarray(rows, dtype=np.int32)
        out = cls(engine, shape=(len(rows), n_cols), dtype=dtype)
        check(out.fn("cnmf_gather_rows")(engine._h, ctypes.c_void_p(int(src_ptr)), int(ld_src), ptr(rows), len(rows),
                                         int(n_cols), out.p, out.ld, None))
        return out

    @property
    def p(self):
        return ctypes.c_void_p(self.t.data_ptr())

    def numpy(self):
        return self.t[:, :self.G].cpu().numpy()

    def l2_normalize(self):
        check(self.fn("cnmf_l2_normalize_rows")(self.engine._h, self.p, self.R, self.G, self.ld, None))
        return self

    def local_density(self, n_neighbors, return_dist=False):
        torch = _torch()
        dens = torch.empty(self.R, dtype=self.torch_dtype, device=self.t.device)
        D = torch.empty((self.R, self.R), dtype=self.torch_dtype, device=self.t.device) if return_dist else None
        check(self.fn("cnmf_local_density")(self.engine._h, self.p, self.R, self.G, self.ld, int(n_neighbors),
                                          ctypes.c_void_p(dens.data_ptr()),
                                          ctypes.c_void_p(D.data_ptr()) if D is not None else None, None))
        torch.cuda.synchronize(self.t.device)
        return dens.cpu().numpy().astype(np.float64), (D.cpu().numpy() if D is not None else None)

    def take_rows(self, idx):
        idx = np.ascontiguousarray(idx, dtype=np.int32)
        out = SpectraMatrix(self.engine, shape=(len(idx), self.G), dtype=self.dtype)
        check(self.fn("cnmf_gather_rows")(self.engine._h, self.p, self.ld, ptr(idx), len(idx), self.G, out.p, out.ld, None))
        return out

    def sq_dists_to_rows(self, idx):
        idx = np.ascontiguousarray(idx, dtype=np.int32)
        out = np.empty((len(idx), self.R), self.dtype)
        check(self.fn("cnmf_sq_dists_to_rows")(self.engine._h, self.p, self.R, self.G, self.ld, ptr(idx), len(idx),
                                               ptr(out), None))
        return out.astype(np.float64)


# ------------------------------------------------------------------------------ KMeans
def _kmeans_plusplus(S, k, rng):
    """sklearn/cluster/_kmeans.py:180-278 with unit weights; distances from the GPU, draws on the host."""
    n = S.R
    n_local_trials = 2 + int(np.log(k))
    w = np.ones(n)
    center_id = rng.choice(n, p=w / w.sum())
    indices = [int(center_id)]
    closest = S.sq_dists_to_rows([center_id])          # (1, n)
    pot = closest @ w
    for _ in range(1, k):
        rand_vals = rng.uniform(size=n_local_trials) * pot
        cand = np.searchsorted(np.cumsum(w * closest), rand_vals)
        np.clip(cand, None, closest.size - 1, out=cand)
        d = S.sq_dists_to_rows(cand)
        np.minimum(closest, d, out=d)
        cpot = d @ w.reshape(-1, 1)
        best = int(np.argmin(cpot))
        pot = cpot[best]
        closest = d[best][None, :]
        indices.append(int(cand[best]))
    return np.array(indices, dtype=np.int32)


def _same_clustering(l1, l2, k):
    mapping = np.full(k, -1, dtype=np.int64)
    for a, b in zip(l1, l2):
        if mapping[a] == -1:
            mapping[a] = b
        elif mapping[a] != b:
            return False
    return True


def _kmeans_draws(rng, n, k, n_init):
    """The random numbers k-means++ consumes, in sklearn's order (SK/cluster/_kmeans.py:231, 249-251): per run one
    rng.choice(n, p=uniform) for the first centre, then rng.uniform(size=n_local_trials) per further centre.  They do not
    depend on the data, so the whole fit can run on the device without handing control back for a draw."""
    n_trials = 2 + int(np.log(k))
    w = np.ones(n)
    first = np.empty(n_init, np.int32)
    unif = np.empty((n_init, max(k - 1, 1), n_trials), np.float64)
    for t in range(n_init):
        first[t] = rng.choice(n, p=w / w.sum())
        for c in range(k - 1):
            unif[t, c] = rng.uniform(size=n_trials)
    return first, unif, n_trials


def kmeans(S, k, n_init=10, random_state=1, max_iter=300, tol=1e-4):
    """KMeans(n_clusters=k, n_init=10, random_state=1).fit(l2_spectra).labels_ (cnmf.py:908-910).
    Returns (labels int32 numpy, labels device tensor, inertia, centers or None).

    Default path: ONE library call (cnmf_kmeans_fit) -- k-means++ and Lloyd for all n_init runs resident on the device,
    the host only pre-draws the random numbers and applies sklearn's best-run rule.  When a cluster comes out empty
    (sklearn's relocation rule) the per-run host-assisted path below is used instead."""
    torch = _torch()
    lib, h = S.lib, S.engine._h
    G, R = S.G, S.R
    # tolerance: mean of the per-feature variances * tol (sklearn _kmeans.py:285-293)
    mean = np.empty(G)
    var = np.empty(G)
    check(S.fn("cnmf_col_stats_dev")(h, S.p, R, G, S.ld, ptr(mean), ptr(var), None))
    tol_abs = float(var.mean()) * tol
    if k <= 32 and n_init <= 32 and R * 8 <= 200 * 1024:
        rng = np.random.RandomState(random_state)
        first, unif, n_trials = _kmeans_draws(rng, R, k, n_init)
        labels_all = np.empty((n_init, R), np.int32)
        inertia = np.empty(n_init, np.float64)
        n_it = np.zeros(n_init, np.int32)
        fallback = ctypes.c_int32(0)
        check(S.fn("cnmf_kmeans_fit")(h, S.p, R, G, S.ld, int(k), int(n_init), int(max_iter), tol_abs, ptr(first),
                                      ptr(unif), int(n_trials), ptr(labels_all), ptr(inertia), ptr(n_it),
                                      ctypes.byref(fallback), None))
        if not fallback.value:
            STATS["lloyd_iters"] = STATS.get("lloyd_iters", 0) + int(n_it.sum())
            best = None
            for t in range(n_init):            # sklearn _kmeans.py:1534-1541
                if best is None or (inertia[t] < best[1] and not _same_clustering(labels_all[t], best[0], k)):
                    best = (labels_all[t], float(inertia[t]))
            labels_t = torch.from_numpy(np.ascontiguousarray(best[0])).to(S.t.device)
            return best[0].copy(), labels_t, best[1], None
    return _kmeans_per_run(S, k, n_init, random_state, max_iter, tol_abs)


def _kmeans_per_run(S, k, n_init, random_state, max_iter, tol_abs):
    """One run at a time, k-means++ draws and the empty-cluster relocation rule on the host (sklearn
    _k_means_common.pyx:167-211), distances and Lloyd steps on the device.  A float32 matrix runs its E steps against an
    fp32 copy of the fp64 centres; a float64 one against the fp64 centres themselves."""
    torch = _torch()
    lib, h = S.lib, S.engine._h
    rng = np.random.RandomState(random_state)
    G, R = S.G, S.R

    dev = S.t.device
    labels_t = torch.empty(R, dtype=torch.int32, device=dev)
    mind_t = torch.empty(R, dtype=S.torch_dtype, device=dev)
    # centres stay on the device across Lloyd iterations (fp64 master + fp32 copy for the E step, ping-pong):
    # an iteration returns three scalars instead of a K x G round trip
    C64 = [torch.empty((k, G), dtype=torch.float64, device=dev) for _ in range(2)]
    C32 = None if S.fp64 else [torch.empty((k, G), dtype=torch.float32, device=dev) for _ in range(2)]
    sums_t = torch.empty((k, G), dtype=torch.float64, device=dev)
    counts_t = torch.empty(k, dtype=torch.int32, device=dev)
    vp = lambda t: ctypes.c_void_p(t.data_ptr())        # noqa: E731
    n_changed = ctypes.c_int32(0)
    any_empty = ctypes.c_int32(0)
    shift = ctypes.c_double(0)
    inertia = ctypes.c_double(0)
    best = None
    for _ in range(n_init):
        idx = _kmeans_plusplus(S, k, rng)
        centers = S.take_rows(idx).numpy().astype(np.float64)
        cur = 0
        C64[cur].copy_(torch.from_numpy(centers))
        if C32 is not None:
            C32[cur].copy_(torch.from_numpy(np.ascontiguousarray(centers, dtype=np.float32)))
        labels_t.fill_(-1)
        n_it = 0
        for n_it in range(max_iter):
            new = 1 - cur
            flags = (vp(labels_t), vp(mind_t), vp(sums_t), vp(counts_t), ctypes.byref(n_changed),
                     ctypes.byref(any_empty), ctypes.byref(shift), None)
            if S.fp64:
                check(lib.cnmf_kmeans_step_f64(h, S.p, R, G, S.ld, k, vp(C64[cur]), vp(C64[new]), *flags))
            else:
                check(lib.cnmf_kmeans_step(h, S.p, R, G, S.ld, k, vp(C32[cur]), vp(C64[cur]), vp(C64[new]),
                                           vp(C32[new]), *flags))
            shift_tot = shift.value
            if any_empty.value:                       # rare: relocation rule on the host, sklearn _k_means_common.pyx:167-211
                centers = C64[cur].cpu().numpy()
                nc = sums_t.cpu().numpy().copy()
                weight = counts_t.cpu().numpy().astype(np.float64)
                empty = np.where(weight == 0)[0]
                dist = mind_t.cpu().numpy().astype(np.float64)
                if dist.max() != 0:
                    lab = labels_t.cpu().numpy()
                    far = np.argpartition(dist, -len(empty))[: -len(empty) - 1: -1]
                    rows = S.take_rows(far).numpy().astype(np.float64)
                    for j, new_id in enumerate(empty):
                        old_id = lab[far[j]]
                        nc[old_id] -= rows[j]
                        nc[new_id] = rows[j]
                        weight[new_id] = 1
                        weight[old_id] -= 1
                amax = int(np.argmax(weight))
                for j in range(k):                    # _average_centers, _k_means_common.pyx:274-298
                    if weight[j] > 0:
                        nc[j] *= 1.0 / weight[j]
                    else:
                        nc[j] = nc[amax]
                shift_tot = float(((nc - centers) ** 2).sum())
                C64[new].copy_(torch.from_numpy(nc))
                if C32 is not None:
                    C32[new].copy_(torch.from_numpy(np.ascontiguousarray(nc, dtype=np.float32)))
            cur = new
            if n_changed.value == 0:
                break
            if shift_tot <= tol_abs:
                break
        STATS["lloyd_iters"] = STATS.get("lloyd_iters", 0) + n_it + 1
        centers = C64[cur].cpu().numpy()
        ce = np.ascontiguousarray(centers, dtype=S.dtype)
        # final E step (labels consistent with the final centres) + inertia
        check(S.fn("cnmf_kmeans_assign")(h, S.p, R, G, S.ld, ptr(ce), k, ctypes.c_void_p(labels_t.data_ptr()),
                                         None, None, ctypes.c_void_p(mind_t.data_ptr()), ctypes.byref(n_changed),
                                         ctypes.byref(inertia), None))
        labels = labels_t.cpu().numpy().copy()
        if best is None or (inertia.value < best[1] and not _same_clustering(labels, best[0], k)):
            best = (labels, float(inertia.value), centers.copy(), n_it + 1)
    labels_t.copy_(torch.from_numpy(best[0]))
    return best[0], labels_t, best[1], best[2]


def cluster_medians(S, labels_t, k):
    """cnmf.py:913-916 on the device; returns K x G float64 (rows sum to 1)."""
    torch = _torch()
    M = torch.empty((k, S.ld), dtype=S.torch_dtype, device=S.t.device)
    check(S.fn("cnmf_cluster_median")(S.engine._h, S.p, S.R, S.G, S.ld, ctypes.c_void_p(labels_t.data_ptr()), k,
                                    ctypes.c_void_p(M.data_ptr()), S.ld, None))
    torch.cuda.synchronize(S.t.device)
    return M[:, :S.G].cpu().numpy().astype(np.float64)


def silhouette(S, labels, labels_t, k):
    """sklearn.metrics.silhouette_score(l2_spectra, labels, metric='euclidean') (cnmf.py:923): the R x R
    distances and the per-sample per-cluster distance sums come from the GPU, the O(R*K) rest is numpy."""
    sums = np.empty((S.R, k), np.float64)
    check(S.fn("cnmf_cluster_dist_sums")(S.engine._h, S.p, S.R, S.G, S.ld, ctypes.c_void_p(labels_t.data_ptr()), k,
                                         ptr(sums), None))
    counts = np.bincount(labels, minlength=k).astype(np.float64)
    own = counts[labels]
    idx = np.arange(S.R)
    with np.errstate(divide="ignore", invalid="ignore"):
        a = sums[idx, labels] / (own - 1.0)
        mean_other = sums / counts[None, :]
        mean_other[idx, labels] = np.inf
        b = mean_other.min(axis=1)
        sil = (b - a) / np.maximum(a, b)
    sil[own == 1] = 0.0
    return float(np.nan_to_num(sil).mean())


def ols_zscore(usages, tpm_ds):
    """efficient_ols_all_cols(rf_usages, tpm.X, normalize_y=True) (cnmf.py:55-125).
    U^T Z with Z = (T - mean)/std equals (U - mean(U))^T T / std because the columns of T - mean sum to
    zero; centring U instead of T keeps the GEMM free of catastrophic cancellation in fp32 accumulation."""
    U = np.asarray(usages, dtype=np.float64)
    mean, var = tpm_ds.col_stats()
    var[var < 1e-12] = 1e-12
    std = np.sqrt(var)
    Uc = U - U.mean(axis=0)
    dt = np.float64 if getattr(tpm_ds, "fp64", False) else np.float32     # a float64 dataset projects in float64
    UtZ = tpm_ds.project_rows(np.ascontiguousarray(Uc.T, dtype=dt)).astype(np.float64) / std
    UtU = U.T @ U
    beta, *_ = np.linalg.lstsq(UtU, UtZ, rcond=None)
    return beta


# ------------------------------------------------------------------------------ the consensus step as one function
def consensus_numerics(eng, merged, k, norm_ds, kw, **kwargs):
    """See _consensus_numerics; runs it with a small host BLAS pool."""
    with _few_blas_threads():
        return _consensus_numerics(eng, merged, k, norm_ds, kw, **kwargs)


def _consensus_numerics(eng, merged, k, norm_ds, kw, density_threshold=0.5, n_neighbors=None,
                       local_neighborhood_size=0.30, stats_only=False, local_density=None, want_dist=False,
                       tpm_ds=None, hvg_idx=None, tpm_std_hvg=None, refit_usage=True, tpm_sparse=False,
                       on_density=None):
    """Every numeric step of cNMF.consensus (cnmf.py:879-975) for one K, on the GPU, without files or labels:
    the facade (pipeline.cNMF.consensus) wraps it in the reference's DataFrames / ledger, bench.py times it.

    merged        R x G stacked spectra: numpy array or a SpectraMatrix already on the device (not yet normalised)
    norm_ds       resident normalised counts (refit a, cnmf.py:919);  tpm_ds: resident TPM (refits b, c and the OLS)
    local_density optional cached densities (cnmf.py:887-888); else computed (and returned); on_density(array) is
                  called as soon as they exist -- the reference writes its cache before the filter can raise
    Returns a dict: local_density, keep (indices), labels (0-based), median_spectra (K x G, rows sum to 1), rf_usages,
    refit_err and, unless stats_only: order (program permutation, cnmf.py:939-946), norm_usages, spectra_tpm,
    usage_coef, final rf_usages; with stats_only: silhouette, prediction_error (cnmf.py:922-936)."""
    import pandas as pd
    import time
    phases = STATS.setdefault("phases_ms", {})
    t_last = [time.perf_counter()]

    def mark(name):          # host wall clock per phase (every phase ends in a host-visible result, i.e. synchronised)
        now = time.perf_counter()
        phases[name] = phases.get(name, 0.0) + 1e3 * (now - t_last[0])
        t_last[0] = now

    # a float64 analysis (precision='fp64') keeps the spectra in float64 through every consensus kernel
    dtype = np.float64 if getattr(norm_ds, "fp64", False) else np.float32
    S = merged if isinstance(merged, SpectraMatrix) else SpectraMatrix(eng, merged, dtype=dtype)
    S.l2_normalize()                                                            # cnmf.py:882
    R = S.R
    if n_neighbors is None:
        n_neighbors = int(local_neighborhood_size * R / k)                      # cnmf.py:879
    out = {"S_all": S, "topics_dist": None, "keep": np.arange(R)}
    if not stats_only:
        if local_density is None:
            local_density, out["topics_dist"] = S.local_density(n_neighbors, return_dist=want_dist)   # cnmf.py:891-896
        out["local_density"] = np.asarray(local_density, dtype=np.float64)
        if on_density is not None:
            on_density(out["local_density"])
        keep = np.where(out["local_density"] < density_threshold)[0]             # cnmf.py:903
        if len(keep) == 0:
            raise RuntimeError("Zero components remain after density filtering. Consider increasing density threshold")
        if len(keep) < R:
            S = S.take_rows(keep)
        out["keep"] = keep
        mark("l2_dist_density_filter")
    out["S"] = S
    labels0, labels_t, _, _ = kmeans(S, k)                                        # cnmf.py:908-910
    out["labels"] = labels0
    mark("kmeans")
    med = cluster_medians(S, labels_t, k)                                         # cnmf.py:913-916
    out["median_spectra"] = med
    mark("median")
    rf, it_a, err = norm_ds.refit(med, kw)                                        # cnmf.py:919
    STATS.setdefault("refits", []).append((norm_ds.shape[0], norm_ds.shape[1], it_a))
    rf = rf.astype(np.float64)
    out["rf_usages"], out["refit_err"] = rf, err
    mark("refit_usage_norm_counts")
    if stats_only:                                                                # cnmf.py:922-936
        out["silhouette"] = silhouette(S, labels0, labels_t, k)
        out["prediction_error"] = err ** 2
        mark("silhouette")
        return out
    norm_usages = rf / rf.sum(axis=1, keepdims=True)                              # cnmf.py:939-946
    order = pd.Series(norm_usages.sum(axis=0)).sort_values(ascending=False).index.values
    rf, norm_usages, med = rf[:, order], norm_usages[:, order], med[order]
    out.update(order=order, rf_usages=rf, norm_usages=norm_usages, median_spectra=med)
    if tpm_ds is None:
        return out
    Ht, it_b, _ = tpm_ds.refit(np.ascontiguousarray(norm_usages.T), kw, transposed=True)   # cnmf.py:952 (refit_spectra)
    STATS.setdefault("refits", []).append((tpm_ds.shape[1], tpm_ds.shape[0], it_b))
    spectra_tpm = Ht.T.astype(np.float64)
    out["spectra_tpm"] = spectra_tpm
    mark("refit_spectra_tpm")
    out["usage_coef"] = ols_zscore(rf, tpm_ds)                                     # cnmf.py:958
    mark("ols")
    if refit_usage and hvg_idx is not None:                                        # cnmf.py:961-975
        _, var = tpm_ds.col_stats()
        n = tpm_ds.shape[0]
        std1 = np.sqrt(var[hvg_idx] * n / (n - 1.0))                              # std(ddof=1)
        if tpm_sparse:
            std1[std1 == 0] = 1.0                                                 # sc.pp.scale, cnmf.py:967
        if getattr(tpm_ds, "fp64", False):      # X /= std as the host divides (cnmf.py:967-969), bit for bit
            norm_tpm_ds = tpm_ds.from_columns_div(hvg_idx, std1)
        else:
            norm_tpm_ds = tpm_ds.from_columns(hvg_idx, 1.0 / std1)
        sp_rf = spectra_tpm[:, hvg_idx] / np.asarray(tpm_std_hvg, dtype=np.float64)[None, :]
        rf2, it_c, _ = norm_tpm_ds.refit(sp_rf, kw)
        STATS.setdefault("refits", []).append((norm_tpm_ds.shape[0], norm_tpm_ds.shape[1], it_c))
        norm_tpm_ds.close()
        out["rf_usages"] = rf2.astype(np.float64)
        mark("refit_usage_tpm_hvg")
    return out
