"""precision='fp64' consensus: the consensus kernels on a float64 SpectraMatrix.

CPU test (unmarked): every float consensus entry point has its _f64 twin in the header and the binding table.
GPU tests (`-m gpu`) hold each kernel to two float64 references -- scipy's cdist (the direct sqrt(sum (x - y)^2) form
the kernels compute) and oracle/consensus_ref + scikit-learn (whose euclidean_distances uses the expanded
||x||^2 + ||y||^2 - 2 x.y form) -- and the whole cNMF(precision='fp64') pipeline to the reference's own files at 1e-8.
Lines starting with MEASURE report the deviations DESIGN.md records (run with -s to see them).
"""
import os
import re
import warnings

import numpy as np
import pytest

from cnmf_golden import load_golden

gpu = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FLOAT_CONSENSUS_CALLS = ["cnmf_l2_normalize_rows", "cnmf_local_density", "cnmf_gather_rows", "cnmf_sq_dists_to_rows",
                         "cnmf_kmeans_fit", "cnmf_kmeans_assign", "cnmf_kmeans_step", "cnmf_col_stats_dev",
                         "cnmf_cluster_dist_sums", "cnmf_cluster_median"]


def rel(a, b):
    a = np.asarray(a, dtype=np.float64)
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


def test_every_consensus_call_has_an_f64_twin():
    from cnmf_b200 import _lib
    header = open(os.path.join(ROOT, "include", "cnmf_b200.h")).read()
    for name in FLOAT_CONSENSUS_CALLS:
        assert re.search(r"\bint %s_f64\(" % name, header), name
        assert name + "_f64" in _lib.SIGNATURES, name
    assert "int cnmf_kmeans_step_f64(" in header and "C32" not in header.split("int cnmf_kmeans_step_f64(")[1].split(";")[0]


# ------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def eng():
    from cnmf_b200.engine import Engine
    return Engine(0)


def _planted():
    """R = 3000 x G = 2000: 12 planted clusters of 240 plus 120 outliers (test_consensus_kernels_larger_random)."""
    rng = np.random.RandomState(5)
    cen = np.abs(rng.randn(12, 2000))
    return np.vstack([c + 0.05 * np.abs(rng.randn(240, 2000)) for c in cen] + [np.abs(rng.randn(120, 2000))])


def _tight_threshold():
    """Replicates whose local densities straddle density_threshold = 0.01 (test_density_filter_decision_near_tight_
    threshold): K = 20 clusters of 60, nearest margin to the threshold ~8e-4 relative."""
    rng = np.random.RandomState(11)
    K, reps, G = 20, 60, 2000
    cen = rng.gamma(0.3, 1.0, size=(K, G)) + 1e-3
    spread = np.geomspace(1e-3, 3e-2, reps)
    pts = np.vstack([cen[c] * (1.0 + spread[:, None] * rng.randn(reps, G)).clip(0.0) for c in range(K)])
    return pts[rng.permutation(len(pts))]


def _case(name):
    """(merged spectra, K, n_neighbors, density_threshold)"""
    if name == "planted":
        return _planted(), 12, 72, 0.5
    if name == "tight":
        pts = _tight_threshold()
        return pts, 20, int(0.3 * len(pts) / 20), 0.01
    tag, k = name.split(":")
    g = load_golden(tag)
    merged, k = g["merged_k%s" % k], int(k)
    return merged, k, int(0.3 * merged.shape[0] / k), float(g["dt"])


def _silhouette(D, labels):
    """oracle/consensus_ref.silhouette's formula on a given distance matrix."""
    n = len(labels)
    A = np.zeros(n)
    B = np.full(n, np.inf)
    for c in np.unique(labels):
        m = labels == c
        s = D[:, m].sum(axis=1)
        cnt = m.sum()
        A[m] = s[m] / max(cnt - 1, 1)
        B[~m] = np.minimum(B[~m], s[~m] / cnt)
    sil = (B - A) / np.maximum(A, B)
    sizes = np.bincount(labels)[labels]
    sil[sizes == 1] = 0
    return float(np.nan_to_num(sil).mean())


def _tol_abs(S, tol=1e-4):
    from cnmf_b200._lib import check, ptr
    mean, var = np.empty(S.G), np.empty(S.G)
    check(S.fn("cnmf_col_stats_dev")(S.engine._h, S.p, S.R, S.G, S.ld, ptr(mean), ptr(var), None))
    return float(var.mean()) * tol


# sklearn's expanded form ||x||^2 + ||y||^2 - 2 x.y loses ~eps in d^2 to cancellation, so a distance d between
# L2-normalised rows is off by up to ~eps / d, and by up to sqrt(few eps) ~ 3e-8 as d -> 0 (near-identical restarts).
# The reference's local densities (means of such distances) and its silhouette carry that error; the direct form does not.
SKLEARN_FORM_ABS = 5e-8


@gpu
@pytest.mark.parametrize("case", ["sim_mu:4", "sim_mu:5", "sim_nndsvd:4", "c1_cd:7", "planted", "tight"])
def test_consensus_kernels_fp64_against_float64(eng, case):
    import torch
    from scipy.spatial.distance import cdist
    from sklearn.cluster import KMeans
    from sklearn.metrics import silhouette_score
    from cnmf_b200 import consensus as cs
    from oracle import consensus_ref as cr
    merged, k, n_nb, dt = _case(case)
    S = cs.SpectraMatrix(eng, merged, dtype=np.float64).l2_normalize()
    assert S.t.dtype == torch.float64 and S.ld % 32 == 0
    l2 = cr.l2_normalize_rows(merged)
    ulps = np.abs(S.numpy() - l2) / np.spacing(np.abs(l2).max(axis=1, keepdims=True))
    assert ulps.max() <= 4, ulps.max()
    # C2: the direct form to 1e-13, exactly symmetric, zero diagonal
    dens, D = S.local_density(n_nb, return_dist=True)
    assert D.dtype == np.float64
    Dc = cdist(l2, l2)
    err_cdist = float(np.abs(D - Dc).max())
    assert err_cdist < 1e-13, err_cdist
    assert (D == D.T).all() and (np.diag(D) == 0).all()
    Dsk = cr.euclidean_distances(l2)
    # C3: density within 1e-12 of the direct-form density, relative to max(density, threshold): the keep decision
    # compares with the threshold, and below it near-identical restarts (sim_nndsvd) have densities of ~1e-15 whose last
    # digits follow the ulps in which the device's and numpy's L2 rows differ.  Keep / drop exactly the reference's.
    dref = cr.local_density(Dc, n_nb)
    dens_sk = cr.local_density(Dsk, n_nb)
    err_dens = float((np.abs(dens - dref) / np.maximum(dref, dt)).max())
    assert err_dens < 1e-12, err_dens
    keep = dens < dt
    assert np.array_equal(keep, dens_sk < dt), int((keep != (dens_sk < dt)).sum())
    dev_dens_sk = float(np.abs(dens - dens_sk).max())
    print("MEASURE %s dist-vs-cdist %.2e dist-vs-sklearn %.2e density-vs-sklearn-abs %.2e" % (
        case, err_cdist, float(np.abs(D - Dsk).max()), dev_dens_sk))
    assert dev_dens_sk < SKLEARN_FORM_ABS
    # KMeans on the kept rows: labels of the oracle and of scikit-learn, inertia to 1e-12
    idx = np.where(keep)[0]
    S2 = S.take_rows(idx) if len(idx) < S.R else S
    l2k = l2[keep]
    labels, labels_t, inertia, _ = cs.kmeans(S2, k)
    lref, iref, _ = cr.kmeans(l2k, k)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        sk = KMeans(n_clusters=k, n_init=10, random_state=1).fit(l2k)
    assert np.array_equal(labels, lref) and np.array_equal(labels, sk.labels_)
    assert abs(inertia - iref) <= 1e-12 * iref + 1e-28, (inertia, iref)      # + 1e-28: clusters of identical rows
    # the per-run path: same labels, same inertia to 1e-12
    lp, _, ip, _ = cs._kmeans_per_run(S2, k, 10, 1, 300, _tol_abs(S2))
    assert np.array_equal(lp, labels) and abs(ip - inertia) <= 1e-12 * inertia + 1e-28, (ip, inertia)
    # C6: medians (normalised rows) within 1e-15
    med = cs.cluster_medians(S2, labels_t, k)
    err_med = float(np.abs(med - cr.cluster_medians(l2k, lref, k)).max())
    assert err_med < 1e-15, err_med
    # silhouette: the oracle's formula on the direct-form distances within 1e-12; sklearn's deviation is reported
    sil = cs.silhouette(S2, labels, labels_t, k)
    err_sil = abs(sil - _silhouette(cdist(l2k, l2k), labels))
    assert err_sil < 1e-12, err_sil
    print("MEASURE %s median %.2e silhouette-vs-cdist %.2e silhouette-vs-sklearn %.2e" % (
        case, err_med, err_sil, abs(sil - silhouette_score(l2k, labels))))


@gpu
def test_kmeans_fp64_empty_cluster_takes_the_per_run_path(eng, monkeypatch):
    """Three distinct rows repeated 16, 32 and 16 times, K = 5: k-means++ has to pick duplicate centres, a cluster comes
    out empty and the batched fit hands over to the per-run path (sklearn's relocation rule); labels equal the oracle's
    and sklearn's.  The rows are multiples of 1/8 and the counts powers of two, so every mean (sklearn's centring
    included) and every centre is exact: all distances to the centres are exactly 0 and no tie is decided by rounding."""
    from sklearn.cluster import KMeans
    from cnmf_b200 import consensus as cs
    from oracle import consensus_ref as cr
    rng = np.random.RandomState(3)
    base = rng.randint(1, 8, size=(3, 300)) / 8.0
    pts = base[rng.permutation(np.repeat([0, 1, 2], [16, 32, 16]))]
    calls = []
    per_run = cs._kmeans_per_run
    monkeypatch.setattr(cs, "_kmeans_per_run", lambda *a: calls.append(1) or per_run(*a))
    S = cs.SpectraMatrix(eng, pts, dtype=np.float64)
    labels, _, inertia, _ = cs.kmeans(S, 5)
    assert calls, "the batched fit did not hand over"
    lref, iref, _ = cr.kmeans(pts, 5)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        sk = KMeans(n_clusters=5, n_init=10, random_state=1).fit(pts)
    assert np.array_equal(labels, lref) and np.array_equal(labels, sk.labels_)
    assert inertia == 0.0 and iref == 0.0


# The fixture's densities and silhouettes come from sklearn's expanded-form distances: the densities are held to
# SKLEARN_FORM_ABS, and so is the silhouette of sim_nndsvd, whose deterministic starts make every restart of a K the same
# spectra (zero true distances, each off by up to ~3e-8 in the expanded form); every other silhouette to 1e-9.
SILHOUETTE_TOL = {"sim_nndsvd": SKLEARN_FORM_ABS}


@gpu
@pytest.mark.parametrize("tag", ["sim_mu", "sim_cd", "sim_nndsvd", "c1_mu", "c1_cd"])
def test_pipeline_fp64_consensus_matches_reference_files(tmp_path, tag):
    """cNMF(precision='fp64'): prepare -> factorize -> combine -> consensus; every consensus file within 1e-8 of the
    reference's (sim_mu K = 4 included), the k-selection statistics within 1e-9, every keep / drop decision equal."""
    import pandas as pd
    from cnmf_b200 import cNMF, load_df_from_npz, save_df_to_npz
    g = load_golden(tag)
    counts = g["counts"].astype(np.float64)
    df = pd.DataFrame(counts, index=["c%d" % i for i in range(counts.shape[0])],
                      columns=["g%d" % i for i in range(counts.shape[1])])
    fn = str(tmp_path / "counts.df.npz")
    save_df_to_npz(df, fn)
    obj = cNMF(output_dir=str(tmp_path), name="run", precision="fp64")
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        obj.prepare(fn, components=list(g["ks"]), n_iter=int(g["n_iter"]), seed=int(g["seed"]), densify=True,
                    beta_loss=g["beta_loss_arg"], num_highvar_genes=len(g["hvg_idx"]), init=g["init"])
        obj.factorize()
        obj.combine()
        dt = float(g["dt"])
        for k in g["ks"]:
            k = int(k)
            stats = obj.consensus(k, skip_density_and_return_after_stats=True, show_clustering=False)
            ref_stats = g["stats_k%d" % k]
            e_sil = abs(stats.loc["silhouette", "stats"] - ref_stats[2])
            e_pe = abs(stats.loc["prediction_error", "stats"] - ref_stats[3]) / ref_stats[3]
            obj.consensus(k, density_threshold=dt, show_clustering=False)
            dens = load_df_from_npz(obj.paths["local_density_cache"] % k).values[:, 0]
            dref = g["density_k%d" % k]
            e_dens = float(np.abs(dens - dref).max())
            errs = {}
            dts = str(dt).replace(".", "_")
            for key, name in (("consensus_spectra", "cspectra"), ("consensus_usages", "cusages"),
                              ("gene_spectra_tpm", "tpmspec"), ("gene_spectra_score", "score"),
                              ("starcat_spectra", "starcat")):
                got = load_df_from_npz(obj.paths[key] % (k, dts)).values
                errs[key] = rel(got, g["%s_k%d" % (name, k)])
            print("MEASURE %s K=%d silhouette %.2e prediction_error %.2e density-abs %.2e %s" % (
                tag, k, e_sil, e_pe, e_dens, " ".join("%s %.2e" % kv for kv in errs.items())))
            for key, e in errs.items():
                assert e < 1e-8, (tag, k, key, e)
            assert e_pe < 1e-9, (tag, k, e_pe)
            assert e_sil < SILHOUETTE_TOL.get(tag, 1e-9), (tag, k, e_sil)
            assert np.array_equal(dens < dt, dref < dt), (tag, k)
            assert e_dens < SKLEARN_FORM_ABS, (tag, k, e_dens)
