"""`cNMF` facade: the reference's class / file ledger / method signatures (cnmf.py:265-1210) over the
H100 engine.  Host logic only (paths, seeds, job split, DataFrame labelling, file I/O); the numerics of
factorize and consensus run in libcnmf_b200.so.  Nothing here falls back to scikit-learn.

Drop-in points (reference file:line -> here)
  cNMF.__init__/_initialize_dirs  cnmf.py:268-330   same directory layout and path templates
  prepare                         cnmf.py:333-459   host numpy (dense); same outputs and seed rule
  factorize                       cnmf.py:692-745   ALL of this worker's (k, seed) jobs in one batched GPU solve
  combine / combine_nmf           cnmf.py:462-483,748-773
  refit_usage / refit_spectra     cnmf.py:776-820   cnmf_refit
  consensus                       cnmf.py:823-1082  GPU kernels via cnmf_b200.consensus
  k_selection_plot                cnmf.py:1119-1158 statistics (+ figure when matplotlib is available)
  load_results                    cnmf.py:1161-1210
"""
import datetime
import errno
import itertools
import os
import uuid
import warnings

import numpy as np
import pandas as pd
import yaml

from . import io as cio
from .io import load_df_from_npz, save_df_to_npz, save_df_to_text

_TMP = "cnmf_tmp"
# (key, in cnmf_tmp?, suffix) -- expands to the path table of cnmf.py:298-330
_PATH_SPECS = [
    ("normalized_counts", True, ".norm_counts.h5ad"),
    ("nmf_replicate_parameters", True, ".nmf_params.df.npz"),
    ("nmf_run_parameters", True, ".nmf_idvrun_params.yaml"),
    ("nmf_genes_list", False, ".overdispersed_genes.txt"),
    ("tpm", True, ".tpm.h5ad"),
    ("tpm_stats", True, ".tpm_stats.df.npz"),
    ("iter_spectra", True, ".spectra.k_%d.iter_%d.df.npz"),
    ("iter_usages", True, ".usages.k_%d.iter_%d.df.npz"),
    ("merged_spectra", True, ".spectra.k_%d.merged.df.npz"),
    ("local_density_cache", True, ".local_density_cache.k_%d.merged.df.npz"),
    ("consensus_spectra", True, ".spectra.k_%d.dt_%s.consensus.df.npz"),
    ("consensus_spectra__txt", False, ".spectra.k_%d.dt_%s.consensus.txt"),
    ("consensus_usages", True, ".usages.k_%d.dt_%s.consensus.df.npz"),
    ("consensus_usages__txt", False, ".usages.k_%d.dt_%s.consensus.txt"),
    ("consensus_stats", True, ".stats.k_%d.dt_%s.df.npz"),
    ("clustering_plot", False, ".clustering.k_%d.dt_%s.png"),
    ("gene_spectra_score", True, ".gene_spectra_score.k_%d.dt_%s.df.npz"),
    ("gene_spectra_score__txt", False, ".gene_spectra_score.k_%d.dt_%s.txt"),
    ("gene_spectra_tpm", True, ".gene_spectra_tpm.k_%d.dt_%s.df.npz"),
    ("gene_spectra_tpm__txt", False, ".gene_spectra_tpm.k_%d.dt_%s.txt"),
    ("starcat_spectra", True, ".starcat_spectra.k_%d.dt_%s.df.npz"),
    ("starcat_spectra__txt", False, ".starcat_spectra.k_%d.dt_%s.txt"),
    ("k_selection_plot", False, ".k_selection.png"),
    ("k_selection_stats", False, ".k_selection_stats.df.npz"),
]


def worker_filter(iterable, worker_index, total_workers):
    """cnmf.py:52-53."""
    return (p for i, p in enumerate(iterable) if (i - worker_index) % total_workers == 0)


def _highvar_from_stats(mean, var, numgenes):
    """V-score over-dispersion ranking from per-gene TPM mean / population variance (cnmf.py:192-242)."""
    mean = pd.Series(np.asarray(mean, dtype=float))
    var = pd.Series(np.asarray(var, dtype=float))
    fano = var / mean
    top = mean.sort_values(ascending=False)[:20].index
    A = (np.sqrt(var) / mean)[top].min()
    m_lo, m_hi = mean.quantile([0.10, 0.90])
    f_lo, f_hi = fano.quantile([0.10, 0.90])
    box = (fano > f_lo) & (fano < f_hi) & (mean > m_lo) & (mean < m_hi)
    B = np.sqrt(fano[box].median())
    ratio = fano / ((A ** 2) * mean + (B ** 2))
    chosen = ratio.sort_values(ascending=False).index[:numgenes]
    return ratio.index.isin(chosen)


def _maybe_csr(X, sparse):
    if not sparse:
        return X
    import scipy.sparse as sp
    return sp.csr_matrix(X)


def _highvar_genes(tpm, numgenes):
    """Same ranking on a dense TPM matrix held on the host."""
    return _highvar_from_stats(tpm.mean(axis=0), tpm.var(axis=0, ddof=0), numgenes)


def plan_groups(ks, max_rows):
    """Consecutive job ranges [lo, hi) whose packed rows (sum of k) fit `max_rows`; a single job always forms a
    group of its own even when it alone exceeds the budget (the allocation then reports the shortage)."""
    groups, lo, rows = [], 0, 0
    for i, k in enumerate(ks):
        if i > lo and rows + k > max_rows:
            groups.append((lo, i))
            lo, rows = i, 0
        rows += k
    if lo < len(ks):
        groups.append((lo, len(ks)))
    return groups


class cNMF:
    """Same constructor, attributes and methods as the reference class (cnmf.py:265)."""

    def __init__(self, output_dir=".", name=None, precision="f16x2", device=None):
        self.output_dir = output_dir
        if name is None:
            name = "%s_%s" % (datetime.datetime.now().strftime("%Y_%m_%d"), uuid.uuid4().hex[:6])
        self.name = name
        self.precision = precision
        self.device = device
        self.paths = None
        self._engine = None
        self._resident_norm = None      # normalised counts left in HBM by prepare(on_device=True)
        self._initialize_dirs()

    # ------------------------------------------------------------------ ledger
    def _initialize_dirs(self):
        if self.paths is not None:
            return
        base = os.path.join(self.output_dir, self.name)
        os.makedirs(os.path.join(base, _TMP), exist_ok=True)
        self.paths = {key: os.path.join(base, _TMP if tmp else "", self.name + suffix) if tmp
                      else os.path.join(base, self.name + suffix) for key, tmp, suffix in _PATH_SPECS}

    def engine(self):
        """The GPU engine (created on first use; raises without an H100 -- there is no CPU path)."""
        if self._engine is None:
            from .engine import Engine
            dev = self.device
            if dev is None:
                dev = int(os.environ.get("LOCAL_RANK", "0"))
            self._engine = Engine(dev)
        return self._engine

    # ------------------------------------------------------------------ prepare
    def prepare(self, counts_fn, components, n_iter=100, densify=False, tpm_fn=None, seed=None,
                beta_loss="frobenius", num_highvar_genes=2000, genes_file=None,
                alpha_usage=0.0, alpha_spectra=0.0, init="random", max_NMF_iter=1000, on_device=False):
        """Same outputs as reference prepare() (cnmf.py:333-459) for dense inputs.  The CUDA path holds the
        matrix dense, so sparse inputs are densified (numerically identical to the reference's --densify).

        on_device=True (cnmf_b200 extension, `--prepare-on-device`): the raw counts are made resident and the
        per-cell totals, the TPM gene statistics behind the over-dispersion ranking and `tpm_stats`, the per-gene
        scale of the HVG matrix and the HVG matrix itself are computed by CUDA kernels (float64 accumulation from the
        exact integer counts); the normalised matrix stays in HBM for factorize().  Raises without a GPU."""
        from .engine import check_supported
        check_supported(components, init, beta_loss)                  # fail here, not hours later in factorize
        counts = cio.read_counts(counts_fn)
        # the reference keeps X sparse (CSR) unless --densify: text / npz inputs are converted to CSR, .h5ad keeps
        # what the file holds (cnmf.py:383-405).  The CUDA path is dense, but the two branches differ in one rule
        # -- sc.pp.scale(zero_center=False) maps a zero standard deviation to 1 (cnmf.py:538, 967) where the dense
        # branch divides by it (cnmf.py:542) -- and the stored matrices stay CSR like the reference's
        sparse_sem = (not densify) and (counts.is_sparse or not counts_fn.endswith(".h5ad"))
        C = counts.dense(np.float64)
        dev = None
        if on_device:
            if tpm_fn is not None:
                raise ValueError("on_device=True derives TPM from the counts; it cannot be combined with tpm_fn")
            dev = self.engine().dataset(C, precision=self.precision)       # raw counts resident in HBM
            totals = dev.row_sums()
            tpm_X = C / totals[:, None] * 1e6                              # host copy only for the tpm file
            tpm = cio.CellGeneMatrix(_maybe_csr(tpm_X, sparse_sem), counts.obs_names, counts.var_names)
            t_mean, t_var = dev.col_stats(row_scale=1e6 / totals)
            t_std = np.sqrt(t_var)
        elif tpm_fn is None:
            tpm_X = C / C.sum(axis=1, keepdims=True) * 1e6           # cnmf.py:245-251
            tpm = cio.CellGeneMatrix(_maybe_csr(tpm_X, sparse_sem), counts.obs_names, counts.var_names)
        else:
            tpm = cio.read_counts(tpm_fn)
            tpm_X = tpm.dense(np.float64)
            tpm = cio.CellGeneMatrix(_maybe_csr(tpm_X, sparse_sem), tpm.obs_names, tpm.var_names)
        cio.write_matrix(self.paths["tpm"], tpm)
        T = tpm_X
        if dev is None:
            t_mean, t_std = T.mean(axis=0), T.std(axis=0, ddof=0)
        stats = pd.DataFrame([t_mean, t_std], index=["__mean", "__std"], columns=tpm.var_names).T   # cnmf.py:439-445
        save_df_to_npz(stats, self.paths["tpm_stats"])

        if genes_file is not None:
            hvgs = open(genes_file).read().rstrip().split("\n")
        elif dev is not None:
            hvgs = list(tpm.var_names[_highvar_from_stats(t_mean, t_var, num_highvar_genes)])
        else:
            hvgs = list(tpm.var_names[_highvar_genes(T, num_highvar_genes)])
        norm, idx = cio.CellGeneMatrix(C, counts.obs_names, counts.var_names).subset_genes(hvgs)
        X = norm.X.astype(np.float64)
        if dev is not None:
            n = C.shape[0]
            _, c_var = dev.col_stats()
            std1 = np.sqrt(c_var[idx] * n / (n - 1.0))                 # std(ddof=1) of the selected count columns
            if sparse_sem:
                std1[std1 == 0] = 1.0
            X /= std1
            with np.errstate(divide="ignore"):
                self._resident_norm = dev.from_columns(idx, 1.0 / std1)   # counts[:, hvgs] / std, built on the device
            dev.close()
        else:
            std1 = X.std(axis=0, ddof=1)
            if sparse_sem:
                std1[std1 == 0] = 1.0                                  # sc.pp.scale(zero_center=False), cnmf.py:538
            X /= std1                                                  # cnmf.py:542 (no centring)
        if np.isnan(X).sum() > 0:
            print("Warning NaNs in normalized counts matrix")
        norm.X = _maybe_csr(X, sparse_sem)
        with open(self.paths["nmf_genes_list"], "w") as F:
            F.write("\n".join(hvgs))
        zero = np.asarray(X.sum(axis=1)).reshape(-1) == 0
        if zero.sum() > 0:                                             # cnmf.py:551-554
            ex = norm.obs_names[np.ravel(zero)]
            raise Exception("Error: %d cells have zero counts of overdispersed genes. E.g. %s. Filter those cells "
                            "and re-run or adjust the number of overdispersed genes. Quitting!"
                            % (zero.sum(), ", ".join(ex[:4])))
        self.save_norm_counts(norm)
        rp, run = self.get_nmf_iter_params(ks=components, n_iter=n_iter, random_state_seed=seed, beta_loss=beta_loss,
                                           alpha_usage=alpha_usage, alpha_spectra=alpha_spectra, init=init,
                                           max_iter=max_NMF_iter)
        self.save_nmf_iter_params(rp, run)

    def save_norm_counts(self, norm_counts):
        self._initialize_dirs()
        cio.write_matrix(self.paths["normalized_counts"], norm_counts)

    def get_nmf_iter_params(self, ks, n_iter=100, random_state_seed=None, beta_loss="kullback-leibler",
                            alpha_usage=0.0, alpha_spectra=0.0, init="random", max_iter=1000):
        """(k, iter, seed, completed) table + solver kwargs; identical seed rule to cnmf.py:593-633."""
        if type(ks) is int:
            ks = [ks]
        from .engine import check_supported
        check_supported(ks, init, beta_loss)
        k_list = sorted(set(list(ks)))
        n_runs = len(ks) * n_iter
        np.random.seed(seed=random_state_seed)
        nmf_seeds = np.random.randint(low=1, high=(2 ** 31) - 1, size=n_runs)
        rows = []
        for i, (k, r) in enumerate(itertools.product(k_list, range(n_iter))):
            rows.append([k, r, nmf_seeds[i], os.path.exists(self.paths["iter_spectra"] % (k, r))])
        rp = pd.DataFrame(rows, columns=["n_components", "iter", "nmf_seed", "completed"])
        if rp["completed"].sum() > 0:
            warnings.warn("%d runs already appear completed. If this is unexpected, consider re-initializing the "
                          "cnmf object with a different run name or output directory" % rp["completed"].sum(), UserWarning)
        kw = dict(alpha_W=alpha_usage, alpha_H=alpha_spectra, l1_ratio=0.0, beta_loss=beta_loss, solver="mu",
                  tol=1e-4, max_iter=max_iter, init=init)
        if beta_loss == "frobenius":      # cnmf.py:629-631: the reference's default solver for Frobenius is CD
            kw["solver"] = "cd"
        return rp, kw

    def update_nmf_iter_params(self):
        kw = yaml.load(open(self.paths["nmf_run_parameters"]), Loader=yaml.FullLoader)
        rp = load_df_from_npz(self.paths["nmf_replicate_parameters"])
        for i in rp.index:
            rp.at[i, "completed"] = os.path.exists(self.paths["iter_spectra"] % (rp.at[i, "n_components"], rp.at[i, "iter"]))
        print("%d NMF runs are currently incomplete" % (rp["completed"] == False).sum())  # noqa: E712
        self.save_nmf_iter_params(rp, kw)

    def save_nmf_iter_params(self, replicate_params, run_params):
        self._initialize_dirs()
        save_df_to_npz(replicate_params, self.paths["nmf_replicate_parameters"])
        with open(self.paths["nmf_run_parameters"], "w") as F:
            yaml.dump(run_params, F)

    # ------------------------------------------------------------------ the seam
    def _dataset(self, X):
        from .engine import Dataset
        if isinstance(X, Dataset):
            return X
        return self.engine().dataset(X, precision=self.precision)

    def _nmf(self, X, nmf_kwargs):
        """Drop-in for the reference seam cNMF._nmf (cnmf.py:661-674): one sklearn-style NMF call,
        returns (spectra, usages).  factorize() uses the batched form _nmf_batched instead."""
        kw = dict(nmf_kwargs)
        ds = self._dataset(X)
        if kw.get("update_H", True) is False:
            H = np.asarray(kw["H"])
            W, _, _ = ds.refit(H, kw)
            return H, W.astype(np.float64)
        from .engine import Dataset
        sp, us, _, _ = ds.factorize([int(kw["n_components"])], [int(kw["random_state"])], kw, return_usages=True,
                                    X_host=None if isinstance(X, Dataset) else X)
        return sp[0].astype(np.float64), us[0].astype(np.float64)

    def _nmf_batched(self, X, ks, seeds, nmf_kwargs, X_host=None):
        """All restarts at once; returns list of spectra (float64) and per-restart iteration counts.  X_host: the host
        matrix, used only for the NNDSVD family of initialisations (their SVD runs on the host)."""
        ds = self._dataset(X)
        sp, _, n_iter, err = ds.factorize(ks, seeds, nmf_kwargs, X_host=X_host)
        return [s.astype(np.float64) for s in sp], n_iter, err

    # ------------------------------------------------------------------ factorize / combine
    def factorize(self, worker_i=0, total_workers=1, skip_completed_runs=False):
        """cnmf.py:692-745, but every job of this worker goes through ONE batched GPU solve."""
        run_params = load_df_from_npz(self.paths["nmf_replicate_parameters"])
        norm = cio.read_matrix(self.paths["normalized_counts"])
        kw = yaml.load(open(self.paths["nmf_run_parameters"]), Loader=yaml.FullLoader)
        if not skip_completed_runs:
            jobs = list(worker_filter(range(len(run_params)), worker_i, total_workers))
        else:
            jobs = list(worker_filter(run_params.index[run_params["completed"] == False], worker_i, total_workers))  # noqa: E712
        if not jobs:
            return
        ks = [int(run_params.iloc[j]["n_components"]) for j in jobs]
        seeds = [int(run_params.iloc[j]["nmf_seed"]) for j in jobs]
        X = norm.X
        if self._resident_norm is not None and self._resident_norm.shape == tuple(norm.X.shape):
            X = self._resident_norm                    # already in HBM (prepare(on_device=True)): no H2D
        ds = self._dataset(X)
        # Restart groups sized from the device memory that is actually free: a solve's workspace grows with
        # sum(k) x cells, so a large K-sweep on a large atlas goes through several batched solves instead of
        # failing in cudaMalloc; each group's files are written as soon as it finishes, so an interrupted run
        # resumes with skip_completed_runs exactly like the reference's per-job loop (cnmf.py:735-745).
        groups = plan_groups(ks, ds.max_rows_per_solve())
        print("[Worker %d]. Starting %d tasks in %d batched solve%s." % (worker_i, len(jobs), len(groups),
                                                                        "" if len(groups) == 1 else "s"))
        hit_max = False
        for lo, hi in groups:
            spectra, n_iter, _ = self._nmf_batched(ds, ks[lo:hi], seeds[lo:hi], kw, X_host=norm.X)
            hit_max = hit_max or int(np.max(n_iter)) >= int(kw["max_iter"])
            for j, sp in zip(jobs[lo:hi], spectra):
                p = run_params.iloc[j]
                df = pd.DataFrame(sp, index=np.arange(1, int(p["n_components"]) + 1), columns=norm.var_names)
                save_df_to_npz(df, self.paths["iter_spectra"] % (p["n_components"], p["iter"]))
        if hit_max:
            from sklearn.exceptions import ConvergenceWarning
            warnings.warn("Maximum number of iterations %d reached. Increase it to improve convergence." % kw["max_iter"],
                          ConvergenceWarning)

    def combine(self, components=None, skip_missing_files=False):
        if type(components) is int:
            ks = [components]
        elif components is None:
            ks = sorted(set(load_df_from_npz(self.paths["nmf_replicate_parameters"]).n_components))
        else:
            ks = components
        for k in ks:
            self.combine_nmf(k, skip_missing_files=skip_missing_files)

    def combine_nmf(self, k, skip_missing_files=False, remove_individual_iterations=False):
        """cnmf.py:748-773."""
        run_params = load_df_from_npz(self.paths["nmf_replicate_parameters"])
        print("Combining factorizations for k=%d." % k)
        sub = run_params[run_params.n_components == k].sort_values("iter")
        parts = []
        for _, p in sub.iterrows():
            fn = self.paths["iter_spectra"] % (p["n_components"], p["iter"])
            if not os.path.exists(fn):
                if not skip_missing_files:
                    print("Missing file: %s, run with skip_missing=True to override" % fn)
                    raise FileNotFoundError(errno.ENOENT, os.strerror(errno.ENOENT), fn)
                print("Missing file: %s. Skipping." % fn)
                continue
            sp = load_df_from_npz(fn)
            sp.index = ["iter%d_topic%d" % (p["iter"], t + 1) for t in range(k)]
            parts.append(sp)
        if parts:
            merged = pd.concat(parts, axis=0)
            save_df_to_npz(merged, self.paths["merged_spectra"] % k)
            return merged
        print("No spectra found for k=%d" % k)
        return parts

    # ------------------------------------------------------------------ refits
    def _run_kwargs(self):
        return yaml.load(open(self.paths["nmf_run_parameters"]), Loader=yaml.FullLoader)

    def refit_usage(self, X, spectra):
        """cnmf.py:776-802."""
        H = spectra.values if isinstance(spectra, pd.DataFrame) else np.asarray(spectra)
        Xv = X.values if isinstance(X, pd.DataFrame) else X
        W, _, _ = self._dataset(Xv).refit(H, self._run_kwargs())
        W = W.astype(np.float64)
        if isinstance(X, pd.DataFrame) and isinstance(spectra, pd.DataFrame):
            W = pd.DataFrame(W, index=X.index, columns=spectra.index)
        return W

    def refit_spectra(self, X, usage):
        """cnmf.py:805-820: refit_usage(X.T, usage.T).T -- the engine solves the transposed problem
        on the same resident dataset instead of materialising X.T."""
        U = usage.values if isinstance(usage, pd.DataFrame) else np.asarray(usage)
        Xv = X.values if isinstance(X, pd.DataFrame) else X
        Ht, _, _ = self._dataset(Xv).refit(np.ascontiguousarray(U.T), self._run_kwargs(), transposed=True)
        return Ht.T.astype(np.float64)

    # ------------------------------------------------------------------ consensus
    def consensus(self, k, density_threshold=0.5, local_neighborhood_size=0.30, show_clustering=True,
                  build_ref=True, skip_density_and_return_after_stats=False, close_clustergram_fig=False,
                  refit_usage=True, normalize_tpm_spectra=False, norm_counts=None):
        """cnmf.py:823-1082 with every numeric step on the GPU (see cnmf_b200/consensus.py)."""
        from . import consensus as cs
        eng = self.engine()
        merged = load_df_from_npz(self.paths["merged_spectra"] % k)
        if norm_counts is None:
            norm_counts = cio.read_matrix(self.paths["normalized_counts"])
        if not hasattr(norm_counts, "_ds"):
            norm_counts._ds = self._dataset(norm_counts.X)
        norm_ds = norm_counts._ds
        kw = self._run_kwargs()

        dt_str = "2" if skip_density_and_return_after_stats else str(density_threshold)
        dt_repl = dt_str.replace(".", "_")
        stats_only = bool(skip_density_and_return_after_stats)
        cached = None
        cache = self.paths["local_density_cache"] % k
        if not stats_only and os.path.isfile(cache):                                # cnmf.py:887-888 (keyed by k only)
            local_density = load_df_from_npz(cache)
            cached = local_density.iloc[:, 0].values
        tpm = tpm_ds = hv_idx = tpm_std_hvg = None
        if not stats_only:
            tpm = cio.read_matrix(self.paths["tpm"])                                # cnmf.py:950-953
            tpm_stats = load_df_from_npz(self.paths["tpm_stats"])
            tpm_ds = self._dataset(tpm.X)
            if refit_usage:
                hvgs = open(self.paths["nmf_genes_list"]).read().split("\n")
                hv_idx = tpm.var_names.get_indexer(hvgs)
                tpm_std_hvg = tpm_stats.loc[hvgs, "__std"].values
        def save_density(dens):                                                     # cnmf.py:897-899
            if cached is None:
                save_df_to_npz(pd.DataFrame(dens, columns=["local_density"], index=merged.index), cache)

        res = cs.consensus_numerics(eng, merged.values, k, norm_ds, kw, density_threshold=density_threshold,
                                    local_neighborhood_size=local_neighborhood_size, stats_only=stats_only,
                                    local_density=cached, want_dist=show_clustering, tpm_ds=tpm_ds, hvg_idx=hv_idx,
                                    tpm_std_hvg=tpm_std_hvg, refit_usage=refit_usage,
                                    tpm_sparse=bool(tpm is not None and tpm.is_sparse), on_density=save_density)
        if tpm_ds is not None:
            tpm_ds.close()
        if stats_only:                                                              # cnmf.py:922-936
            return pd.DataFrame([k, density_threshold, res["silhouette"], res["prediction_error"]],
                                index=["k", "local_density_threshold", "silhouette", "prediction_error"],
                                columns=["stats"])
        if cached is None:
            local_density = pd.DataFrame(res["local_density"], columns=["local_density"], index=merged.index)
        density_filter = local_density.iloc[:, 0] < density_threshold               # cnmf.py:903
        l2_index = merged.index[res["keep"]]
        cluster_labels = pd.Series(res["labels"] + 1, index=l2_index)
        programs = np.arange(1, k + 1)                                              # relabelled 1..K in usage order
        median_spectra = pd.DataFrame(res["median_spectra"], index=programs, columns=merged.columns)
        rf_usages = pd.DataFrame(res["rf_usages"], index=norm_counts.obs_names, columns=programs)
        spectra_tpm = pd.DataFrame(res["spectra_tpm"], index=programs, columns=tpm.var_names)
        if normalize_tpm_spectra:
            spectra_tpm = spectra_tpm.div(spectra_tpm.sum(axis=1), axis=0) * 1e6
        usage_coef = pd.DataFrame(res["usage_coef"], index=programs, columns=tpm.var_names)
        S, topics_dist = res["S"], res["topics_dist"]

        tag = (k, dt_repl)
        save_df_to_npz(median_spectra, self.paths["consensus_spectra"] % tag)
        save_df_to_npz(rf_usages, self.paths["consensus_usages"] % tag)
        save_df_to_text(median_spectra, self.paths["consensus_spectra__txt"] % tag)
        save_df_to_text(rf_usages, self.paths["consensus_usages__txt"] % tag)
        save_df_to_npz(spectra_tpm, self.paths["gene_spectra_tpm"] % tag)
        save_df_to_text(spectra_tpm, self.paths["gene_spectra_tpm__txt"] % tag)
        save_df_to_npz(usage_coef, self.paths["gene_spectra_score"] % tag)
        save_df_to_text(usage_coef, self.paths["gene_spectra_score__txt"] % tag)
        if show_clustering:
            self._clustergram(S, topics_dist, density_filter, cluster_labels, local_density, density_threshold, tag,
                              close_clustergram_fig)
        if build_ref:
            self.build_reference(k, density_threshold)

    @staticmethod
    def clustergram_order(S, topics_dist, density_filter, labels):
        """Row order of the clustergram (cnmf.py:986-1010): clusters in label order, inside a cluster the leaf order
        of an average-linkage tree over the pairwise distances.  The distances come from the GPU (the R x R matrix
        the density step already produced, or a fresh one for the filtered spectra); the O(R) tree is scipy, as in
        the reference.  Returns (order, filtered distance matrix)."""
        from scipy.cluster.hierarchy import leaves_list, linkage
        from scipy.spatial.distance import squareform
        if topics_dist is None:
            _, topics_dist = S.local_density(1, return_dist=True)
        else:
            keep = np.asarray(density_filter.values if hasattr(density_filter, "values") else density_filter, dtype=bool)
            topics_dist = topics_dist[keep, :][:, keep]
        labels = np.asarray(labels.values if hasattr(labels, "values") else labels)
        order = []
        for cl in sorted(set(labels)):
            f = labels == cl
            if f.sum() > 1:
                d = squareform(topics_dist[f, :][:, f], checks=False)
                d[d < 0] = 0
                order += list(np.where(f)[0][leaves_list(linkage(d, "average"))])
            else:
                order += list(np.where(f)[0])
        return order, topics_dist

    def _clustergram(self, S, topics_dist, density_filter, labels, local_density, density_threshold, tag, close_fig):
        """Figure of cnmf.py:986-1079 -- visualisation, outside the accelerated path; needs matplotlib."""
        order, topics_dist = self.clustergram_order(S, topics_dist, density_filter, labels)
        self.last_clustergram_order = order
        try:
            import matplotlib.pyplot as plt
        except Exception:
            warnings.warn("matplotlib is not installed: skipping the clustergram figure", UserWarning)
            return
        fig = plt.figure(figsize=(10, 9.5))
        ax = fig.add_axes([0.08, 0.05, 0.6, 0.85])
        D = topics_dist[order, :][:, order]
        im = ax.imshow(D, interpolation="none", cmap="viridis", aspect="auto", rasterized=True)
        ax.set_xticks([]); ax.set_yticks([])
        hax = fig.add_axes([0.75, 0.6, 0.22, 0.3])
        hax.hist(local_density.values, bins=np.linspace(0, 1, 50))
        hax.axvline(density_threshold, linestyle="--", color="k")
        hax.set_title("Local density histogram")
        fig.colorbar(im, cax=fig.add_axes([0.75, 0.45, 0.22, 0.02]), orientation="horizontal")
        fig.savefig(self.paths["clustering_plot"] % tag, dpi=250)
        if close_fig:
            plt.close(fig)

    def build_reference(self, k, density_threshold=0.5, target_sum=1e6):
        """cnmf.py:1085-1116 (small pandas post-step)."""
        dt_repl = str(density_threshold).replace(".", "_")
        spectra_tpm = pd.read_csv(self.paths["gene_spectra_tpm__txt"] % (k, dt_repl), index_col=0, sep="\t")
        hvgs = open(self.paths["nmf_genes_list"]).read().split("\n")
        tpm_stats = load_df_from_npz(self.paths["tpm_stats"])
        tpm_stats.index = spectra_tpm.columns
        renorm = spectra_tpm.div(spectra_tpm.sum(axis=1), axis=0) * target_sum
        ref = renorm.div(tpm_stats["__std"])[hvgs].copy()
        ref.index = "GEP" + ref.index.astype("str")
        save_df_to_npz(ref, self.paths["starcat_spectra"] % (k, dt_repl))
        save_df_to_text(ref, self.paths["starcat_spectra__txt"] % (k, dt_repl))

    def k_selection_plot(self, close_fig=False):
        """cnmf.py:1119-1158: stability (silhouette) and prediction error for every K."""
        run_params = load_df_from_npz(self.paths["nmf_replicate_parameters"])
        norm_counts = cio.read_matrix(self.paths["normalized_counts"])
        stats = []
        for k in sorted(set(run_params.n_components)):
            stats.append(self.consensus(int(k), skip_density_and_return_after_stats=True, show_clustering=False,
                                        close_clustergram_fig=True, norm_counts=norm_counts).stats)
        stats = pd.DataFrame(stats)
        stats.reset_index(drop=True, inplace=True)
        save_df_to_npz(stats, self.paths["k_selection_stats"])
        try:
            import matplotlib.pyplot as plt
        except Exception:
            warnings.warn("matplotlib is not installed: k_selection statistics saved, figure skipped", UserWarning)
            return stats
        fig = plt.figure(figsize=(6, 4))
        ax1 = fig.add_subplot(111)
        ax2 = ax1.twinx()
        ax1.plot(stats.k, stats.silhouette, "o-", color="b")
        ax1.set_ylabel("Stability", color="b", fontsize=15)
        ax2.plot(stats.k, stats.prediction_error, "o-", color="r")
        ax2.set_ylabel("Error", color="r", fontsize=15)
        ax1.set_xlabel("Number of Components", fontsize=15)
        ax1.grid("on")
        plt.tight_layout()
        fig.savefig(self.paths["k_selection_plot"], dpi=250)
        if close_fig:
            plt.close(fig)
        return stats

    def load_results(self, K, density_threshold, n_top_genes=100, norm_usage=True):
        """cnmf.py:1161-1210."""
        dt = str(density_threshold).replace(".", "_")
        scores = pd.read_csv(self.paths["gene_spectra_score__txt"] % (K, dt), sep="\t", index_col=0).T
        tpm = pd.read_csv(self.paths["gene_spectra_tpm__txt"] % (K, dt), sep="\t", index_col=0).T
        usage = pd.read_csv(self.paths["consensus_usages__txt"] % (K, dt), sep="\t", index_col=0)
        if norm_usage:
            usage = usage.div(usage.sum(axis=1), axis=0)
        try:
            usage.columns = [int(x) for x in usage.columns]
        except Exception:
            print("Usage matrix columns include non integer values")
        top = [list(scores.sort_values(by=g, ascending=False).index[:n_top_genes]) for g in scores.columns]
        top_genes = pd.DataFrame(top, index=scores.columns).T
        return usage, scores, tpm, top_genes


def main():
    """`cnmf {prepare,factorize,combine,consensus,k_selection_plot}` with the reference's flags (cnmf.py:1213-1294)."""
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("command", type=str, choices=["prepare", "factorize", "combine", "consensus", "k_selection_plot"])
    ap.add_argument("--name", type=str, nargs="?", default="cNMF")
    ap.add_argument("--output-dir", type=str, nargs="?", default=".")
    ap.add_argument("-c", "--counts", type=str)
    ap.add_argument("-k", "--components", type=int, nargs="+")
    ap.add_argument("-n", "--n-iter", type=int, default=100)
    ap.add_argument("--total-workers", type=int, default=1)
    ap.add_argument("--seed", type=int, default=None)
    ap.add_argument("--genes-file", type=str, default=None)
    ap.add_argument("--numgenes", type=int, default=2000)
    ap.add_argument("--tpm", type=str, default=None)
    ap.add_argument("--max-nmf-iter", type=int, default=1000)
    ap.add_argument("--beta-loss", type=str, choices=["frobenius", "kullback-leibler", "itakura-saito"], default="frobenius")
    ap.add_argument("--init", type=str, choices=["random", "nndsvd"], default="random",
                    help="Initialization algorithm for NMF (cnmf.py:1252); 'nndsvd' starts every restart from a "
                         "host-side randomized SVD of the normalised counts")
    ap.add_argument("--densify", dest="densify", action="store_true", default=False)
    ap.add_argument("--worker-index", type=int, default=0)
    ap.add_argument("--skip-completed-runs", action="store_true", default=False)
    ap.add_argument("--local-density-threshold", type=float, default=0.5)
    ap.add_argument("--local-neighborhood-size", type=float, default=0.30)
    ap.add_argument("--show-clustering", dest="show_clustering", action="store_true")
    ap.add_argument("--build-reference", dest="build_reference", action="store_true", default=True)
    ap.add_argument("--prepare-on-device", dest="prepare_on_device", action="store_true", default=False,
                    help="[cnmf_b200] prepare: cell totals, TPM gene statistics and the HVG matrix computed on the GPU")
    ap.add_argument("--precision", type=str, choices=["f16x2", "tf32x3", "fp32"], default="f16x2",
                    help="[cnmf_b200] big products: split-fp16 wgmma MMAs for scaled-integer-count matrices, split-TF32 "
                         "otherwise (default); split-TF32 always; or FFMA fp32")
    a = ap.parse_args()
    obj = cNMF(output_dir=a.output_dir, name=a.name, precision=a.precision)
    if a.command == "prepare":
        obj.prepare(a.counts, components=a.components, n_iter=a.n_iter, densify=a.densify, tpm_fn=a.tpm, seed=a.seed,
                    beta_loss=a.beta_loss, max_NMF_iter=a.max_nmf_iter, num_highvar_genes=a.numgenes,
                    genes_file=a.genes_file, init=a.init, on_device=a.prepare_on_device)
    elif a.command == "factorize":
        obj.factorize(worker_i=a.worker_index, total_workers=a.total_workers, skip_completed_runs=a.skip_completed_runs)
    elif a.command == "combine":
        obj.combine(components=a.components)
    elif a.command == "consensus":
        rp = load_df_from_npz(obj.paths["nmf_replicate_parameters"])
        ks = sorted(set(rp.n_components)) if a.components is None else a.components
        for k in ks:
            obj.consensus(int(k), a.local_density_threshold, a.local_neighborhood_size, a.show_clustering,
                          a.build_reference, close_clustergram_fig=True)
    elif a.command == "k_selection_plot":
        obj.k_selection_plot(close_fig=True)


if __name__ == "__main__":
    main()
