"""Sparse (CSC) TPM datasets (`-m gpu`): the consensus step's three TPM uses -- refit_spectra, the OLS z-scores and the
HVG refit (cnmf.py:950-969) -- on a matrix that stays CSC on the device, against float64 and against the dense dataset
of the same matrix.  Every fixture is generated here from a seed."""
import ctypes
import os
import warnings

import numpy as np
import pytest
import scipy.sparse as sp

from cnmf_golden import load_golden

pytestmark = pytest.mark.gpu

TOL_SPECTRA = 1e-4


def rel(a, b):
    a = np.asarray(a, dtype=np.float64)
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


@pytest.fixture(scope="module")
def eng():
    from cnmf_b200.engine import Engine
    return Engine(0)


def ragged_csc(n, g, density, seed, counts):
    """Random n x g CSC with an empty row, an empty column, a column with one entry and a fully dense column longer
    than one project chunk when n > 4096.  counts=True: TPM-like (row-scaled integer counts, recognised as exact: every
    row holds a count of 1), else arbitrary values."""
    rng = np.random.RandomState(seed)
    M = sp.random(n, g, density=density, format="lil", random_state=rng,
                  data_rvs=lambda m: rng.randint(1, 40, size=m).astype(np.float64))
    M[:, 0] = 0
    M[:, 1] = 0
    M[n // 2, 1] = 7.0
    M[:, 2] = rng.randint(1, 9, size=(n, 1)).astype(np.float64) if not counts else 1.0   # counts: a 1 in every row
    M[3, :] = 0
    M = M.tocsr()
    if counts:
        tot = np.asarray(M.sum(axis=1)).ravel()
        tot[tot == 0] = 1.0
        M = sp.diags(1e6 / tot) @ M
    else:
        M.data = M.data * rng.lognormal(0.0, 2.0, size=M.nnz)
    C = M.tocsc().astype(np.float32)
    C.eliminate_zeros()
    return C


MATRICES = [(3000, 400, 0.05, 1, True), (9000, 257, 0.02, 2, False)]


@pytest.mark.parametrize("shape", MATRICES)
def test_primitives_match_float64(eng, shape):
    T = ragged_csc(*shape)
    n = T.shape[0]
    ds = eng.sparse_dataset(T)
    assert ds.sparse and ds.shape == T.shape and not ds.exact
    T64 = T.astype(np.float64)
    s, q = ds.sums()
    assert abs(s - T64.data.sum()) <= 1e-12 * abs(T64.data.sum())
    assert abs(q - (T64.data ** 2).sum()) <= 1e-12 * (T64.data ** 2).sum()
    cs = np.asarray(T64.sum(axis=0)).ravel()
    cq = np.asarray(T64.multiply(T64).sum(axis=0)).ravel()
    mean, var = ds.col_stats()
    m_ref = cs / n
    v_ref = np.maximum(cq / n - m_ref ** 2, 0.0)          # col_stats_impl's formula
    assert np.all(np.abs(mean - m_ref) <= 1e-12 * np.abs(m_ref))
    assert np.all(np.abs(var - v_ref) <= 1e-12 * cq / n)
    rng = np.random.RandomState(5)
    for k in (1, 7, 32):
        Ut = rng.randn(k, n).astype(np.float32)           # signed, like the centred usages of the OLS step
        P = ds.project_rows(Ut)
        ref = (T64.T @ Ut.astype(np.float64).T).T
        nz = np.linalg.norm(ref, axis=1) > 0
        assert nz.all()
        err = np.linalg.norm(P - ref, axis=1) / np.linalg.norm(ref, axis=1)
        assert err.max() < 2e-7, (k, err.max())
        assert not P[:, [0]].any()                       # the empty column
        assert np.array_equal(P, ds.project_rows(Ut))     # fixed order, no atomics: bit-identical
    ds.close()


@pytest.mark.parametrize("solver", ["mu", "cd"])
@pytest.mark.parametrize("k", [1, 6, 9, 14, 19, 23, 27, 32])
def test_transposed_refit_matches_oracle_and_dense(eng, solver, k):
    from oracle import nmf_ref
    T = ragged_csc(2500, 300, 0.08, 11, True)
    Td = T.toarray()
    rng = np.random.RandomState(k)
    W = (np.abs(rng.randn(T.shape[0], k)) + 0.05).astype(np.float32)
    kw = dict(solver=solver, tol=1e-4, max_iter=400)
    sds = eng.sparse_dataset(T)
    Ht, it, _ = sds.refit(np.ascontiguousarray(W.T), kw, transposed=True)
    Hr, itr = nmf_ref.refit(Td.T.astype(np.float64), W.T.astype(np.float64), solver, max_iter=400)
    assert it == itr and rel(Ht, Hr) < TOL_SPECTRA, (it, itr, rel(Ht, Hr))
    # the dense dataset's product runs as 2 f16 passes (fp32-class, ~2^-22 relative) where the sparse one is exact
    # in fp64; the solve carries that rounding further the more components it has: measured on an H100, up to
    # 9.2e-7 at k <= 9 and 1.2e-6 (k = 14) to 1.7e-6 (k = 32, CD) above
    dds = eng.dataset(Td)
    Htd, itd, _ = dds.refit(np.ascontiguousarray(W.T), kw, transposed=True)
    assert itd == it and rel(Ht, Htd) < (2e-6 if k >= 14 else 1e-6), (itd, it, rel(Ht, Htd))
    sds.close()
    dds.close()


@pytest.mark.parametrize("counts", [True, False])
def test_from_columns_matches_dense(eng, counts):
    T = ragged_csc(3000, 400, 0.05, 3, counts)
    Td = T.toarray()
    sds, dds = eng.sparse_dataset(T), eng.dataset(Td)
    hv = np.random.RandomState(4).choice(np.arange(3, 400), 120, replace=False)
    std1 = Td[:, hv].astype(np.float64).std(axis=0, ddof=1)
    a, b = dds.from_columns(hv, 1.0 / std1), sds.from_columns(hv, 1.0 / std1)
    assert not b.sparse and (a.exact, a.f16) == (b.exact, b.f16) and a.exact == counts
    H = np.abs(np.random.RandomState(6).randn(6, len(hv))) + 0.1
    for solver in ("mu", "cd"):
        Wa, ita, _ = a.refit(H, dict(solver=solver, tol=1e-4, max_iter=400))
        Wb, itb, _ = b.refit(H, dict(solver=solver, tol=1e-4, max_iter=400))
        assert ita == itb and rel(Wb, Wa) < 1e-6


def test_refused_entry_points(eng):
    import torch
    from cnmf_b200._lib import CnmfError
    T = ragged_csc(500, 64, 0.1, 7, True)
    ds = eng.sparse_dataset(T)
    n, g = T.shape
    kw = dict(solver="mu", tol=1e-4, max_iter=50)
    ld_r, ld_c = ds.ld()
    Wt = torch.zeros((4, ld_r), dtype=torch.float32, device="cuda")
    H = torch.zeros((4, ld_c), dtype=torch.float32, device="cuda")
    calls = {
        "factorize": lambda: ds.factorize([4], [1], kw),
        "factorize_init": lambda: ds.factorize([4], [1], kw, W0=np.ones((4, n)), H0=np.ones((4, g))),
        "factorize_dev": lambda: ds.factorize_dev([4], Wt.data_ptr(), H.data_ptr(), H.data_ptr(), kw),
        "factorize_seeds_dev": lambda: ds.factorize_seeds_dev([4], [1], H.data_ptr(), ld_c, kw),
        "random_init_dev": lambda: ds.random_init_dev([4], [1], Wt.data_ptr(), H.data_ptr()),
        "scale_rows": lambda: ds.scale_rows(np.ones(n)),
        "scaled_col_stats": lambda: ds.col_stats(row_scale=np.ones(n)),
        "row_sums": lambda: ds.row_sums(),
        "min": lambda: ds.min(),
        "refit": lambda: ds.refit(np.ones((4, g)), kw),
        "refit kl": lambda: ds.refit(np.ones((4, n)), dict(kw, beta_loss="kullback-leibler"), transposed=True),
        "refit is": lambda: ds.refit(np.ones((4, n)), dict(kw, beta_loss="itakura-saito"), transposed=True),
    }
    for name, fn in calls.items():
        with pytest.raises(CnmfError, match="sparse"):
            fn()
    # the dataset is still usable after the refusals
    mean, _ = ds.col_stats()
    assert np.allclose(mean, np.asarray(T.astype(np.float64).mean(axis=0)).ravel(), rtol=1e-12)
    peak = ctypes.c_longlong()
    assert eng.lib.cnmf_dataset_dense_bytes(0, 5, 3, ctypes.byref(peak)) == -1
    ds.close()


@pytest.fixture
def force_sparse_tpm(monkeypatch):
    from cnmf_b200 import pipeline
    from cnmf_b200.engine import Engine
    made = []
    orig = Engine.sparse_dataset

    def counted(self, X, *a, **kw):
        made.append(X.shape)
        return orig(self, X, *a, **kw)

    monkeypatch.setattr(pipeline, "TPM_DENSE_FRACTION", 0.0)
    monkeypatch.setattr(Engine, "sparse_dataset", counted)
    return made


def _prepare(tmp_path, g):
    import pandas as pd
    from cnmf_b200 import cNMF, save_df_to_npz
    counts = g["counts"].astype(np.float64)
    df = pd.DataFrame(counts, index=["c%d" % i for i in range(counts.shape[0])],
                      columns=["g%d" % i for i in range(counts.shape[1])])
    fn = str(tmp_path / "counts.df.npz")
    save_df_to_npz(df, fn)
    obj = cNMF(output_dir=str(tmp_path), name="run")
    obj.prepare(fn, components=list(g["ks"]), n_iter=int(g["n_iter"]), seed=int(g["seed"]), densify=True,
                beta_loss=g["beta_loss_arg"], num_highvar_genes=len(g["hvg_idx"]), init=g["init"])
    obj.factorize()
    obj.combine()
    return obj


@pytest.mark.parametrize("tag", ["sim_mu", "sim_cd", "c1_mu", "c1_cd"])
def test_pipeline_with_sparse_tpm_matches_reference_outputs(tmp_path, tag, force_sparse_tpm):
    """The facade with the TPM forced onto the sparse path reproduces every reference file, with the assertions and
    tolerances of test_gpu_parity.test_pipeline_matches_reference_outputs."""
    from cnmf_b200 import load_df_from_npz
    g = load_golden(tag)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        obj = _prepare(tmp_path, g)
        dt = float(g["dt"])
        for k in g["ks"]:
            k = int(k)
            stats = obj.consensus(k, skip_density_and_return_after_stats=True, show_clustering=False)
            ref_stats = g["stats_k%d" % k]
            assert abs(stats.loc["silhouette", "stats"] - ref_stats[2]) < 1e-4
            assert abs(stats.loc["prediction_error", "stats"] - ref_stats[3]) / ref_stats[3] < 1e-5
            obj.consensus(k, density_threshold=dt, show_clustering=False)
            dts = str(dt).replace(".", "_")
            for key, name in (("consensus_spectra", "cspectra"), ("consensus_usages", "cusages"),
                              ("gene_spectra_tpm", "tpmspec"), ("gene_spectra_score", "score"),
                              ("starcat_spectra", "starcat")):
                got = load_df_from_npz(obj.paths[key] % (k, dts)).values
                e = rel(got, g["%s_k%d" % (name, k)])
                limit = 3e-4 if (tag, k) == ("sim_mu", 4) else TOL_SPECTRA
                assert e < limit, (tag, k, key, e)
                assert os.path.exists(obj.paths[key + "__txt"] % (k, dts))
    assert len(force_sparse_tpm) == len(g["ks"])


def test_pipeline_kl_with_sparse_tpm_raises(tmp_path, force_sparse_tpm):
    g = load_golden("sim_kl")
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        obj = _prepare(tmp_path, g)
        k = int(g["ks"][0])
        obj.consensus(k, skip_density_and_return_after_stats=True, show_clustering=False)    # no TPM involved
        with pytest.raises(NotImplementedError, match="sparse KL / IS refit is not implemented"):
            obj.consensus(k, density_threshold=float(g["dt"]), show_clustering=False)
    assert not force_sparse_tpm


def atlas_tpm(n, g, per_col, seed):
    """n x g TPM-like CSC: about per_col distinct cells per gene, counts 1..5 times 1e6 / (cell total), plus two
    ubiquitous genes (every cell non-zero).  Built column-wise; never dense."""
    rng = np.random.default_rng(seed)
    rows = np.sort(rng.integers(0, n, size=(g, per_col), dtype=np.int32), axis=1)
    keep = np.ones(rows.shape, bool)
    keep[:, 1:] = rows[:, 1:] != rows[:, :-1]
    lens = keep.sum(axis=1)
    lens[:2] = n
    col_ptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    idx = np.empty(col_ptr[-1], np.int32)
    idx[:2 * n] = np.tile(np.arange(n, dtype=np.int32), 2)
    idx[2 * n:] = rows[2:][keep[2:]]
    counts = rng.integers(1, 6, size=idx.size).astype(np.float64)
    tot = np.bincount(idx, weights=counts, minlength=n)
    vals = (counts * (1e6 / tot[idx])).astype(np.float32)
    return sp.csc_matrix((vals, idx, col_ptr), shape=(n, g))


def test_atlas_shape_takes_sparse_path(eng):
    """500 000 cells x 30 000 genes at ~0.5 % density (75 M entries): its dense dataset needs ~300 GB, so consensus
    keeps it sparse without forcing and completes for K = 6.  Device footprint of the library after the run (the
    sparse TPM, the dense HVG dataset, the solver workspace and the buffer pool): under 24 GB."""
    from cnmf_b200 import consensus as cs
    from cnmf_b200.pipeline import tpm_dataset
    n, g, k = 500_000, 30_000, 6
    T = atlas_tpm(n, g, 2500, 0)
    free0, _, _ = eng.mem_info()
    tds = tpm_dataset(eng, T, "f16x2")
    assert tds.sparse
    mean, var = tds.col_stats()
    # the two ubiquitous genes keep every cell's HVG row non-zero (cnmf.py:551-554 refuses cells without counts)
    order = np.argsort(-var / np.maximum(mean, 1e-12))
    hvg = np.concatenate([[0, 1], order[order > 1][:1998]])
    std1 = np.sqrt(var[hvg] * n / (n - 1.0))
    rng = np.random.RandomState(0)
    true = np.abs(rng.randn(k, len(hvg)))
    merged = np.vstack([true * (1 + 0.05 * np.abs(rng.randn(k, len(hvg)))) for _ in range(8)])
    norm_ds = tds.from_columns(hvg, 1.0 / std1)
    kw = dict(solver="cd", beta_loss="frobenius", tol=1e-4, max_iter=200)
    out = cs.consensus_numerics(eng, merged, k, norm_ds, kw, density_threshold=2.0, tpm_ds=tds, hvg_idx=hvg,
                                tpm_std_hvg=std1)
    norm_ds.close()
    assert out["spectra_tpm"].shape == (k, g) and np.isfinite(out["spectra_tpm"]).all()
    assert out["usage_coef"].shape == (k, g) and np.isfinite(out["usage_coef"]).all()
    assert out["rf_usages"].shape == (n, k)
    U = out["rf_usages"]
    Uc = (U - U.mean(axis=0)).astype(np.float32)
    P = tds.project_rows(np.ascontiguousarray(Uc.T))
    genes = np.concatenate([[0, 1], rng.choice(np.arange(2, g), 62, replace=False)])
    ref = (T[:, genes].astype(np.float64).T @ Uc.astype(np.float64)).T
    err = np.linalg.norm(P[:, genes] - ref, axis=0) / np.linalg.norm(ref, axis=0)
    assert err.max() < 1e-6, err.max()
    free1, _, _ = eng.mem_info()
    used = free0 - free1
    print("atlas: nnz %d, dense peak %.1f GB, library footprint after consensus %.2f GB"
          % (T.nnz, eng.dense_dataset_bytes(n, g, "f16x2") / 1e9, used / 1e9))
    assert used < 24e9
    tds.close()
