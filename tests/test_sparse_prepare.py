"""prepare(on_device=True) on counts stored sparse whose dense dataset does not fit: the counts stay CSC on the device
(Dataset.tpm_stats, col_stats, from_columns) and no cells x all-genes dense matrix is formed.  The GPU tests check the
new primitive against float64, the branch against the dense on-device branch and the reference fixtures, and a
500 000 x 30 000 atlas end to end; the CPU test checks which inputs take the branch.  Every fixture is generated here
from a seed."""
import os
import warnings

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sp

from cnmf_golden import load_golden

TOL_SPECTRA = 1e-4


def rel(a, b):
    a = np.asarray(a, dtype=np.float64)
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


def ragged_counts(n, g, density, seed, integer, empty_row=True):
    """Random n x g CSC (float32 values) with an empty column (0), a one-entry column (1), a fully stored column (2,
    longer than one warp's stride) and, with empty_row, an empty row (3).  integer=False: non-integer values."""
    rng = np.random.RandomState(seed)
    R = sp.random(n, g - 3, density=density, format="csc", random_state=rng,
                  data_rvs=lambda m: rng.randint(1, 30, size=m).astype(np.float64))
    one = sp.csc_matrix((np.array([7.0]), (np.array([n // 2]), np.array([0]))), shape=(n, 1))
    full = sp.csc_matrix(rng.randint(1, 9, size=(n, 1)).astype(np.float64))
    M = sp.hstack([sp.csc_matrix((n, 1)), one, full, R], format="csc")
    if not integer:
        M.data = M.data * rng.lognormal(0.0, 1.0, size=M.nnz)
    if empty_row:
        keep = np.ones(n)
        keep[3] = 0.0
        M = sp.diags(keep) @ M
    M = sp.csc_matrix(M, dtype=np.float32)
    M.eliminate_zeros()
    M.sort_indices()
    return M


@pytest.fixture(scope="module")
def eng():
    from cnmf_b200.engine import Engine
    return Engine(0)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(3000, 400, 0.05, 1, True), (9000, 257, 0.02, 2, False),
                                   (70001, 300, 0.01, 3, True)])
def test_tpm_stats_match_float64(eng, shape):
    from cnmf_b200._lib import CnmfError
    C = ragged_counts(*shape)
    integer = shape[4]
    n = C.shape[0]
    C64 = C.astype(np.float64)
    ds = eng.sparse_dataset(C)
    tot, mean, var = ds.tpm_stats()
    tot_ref = np.asarray(C64.sum(axis=1)).ravel()
    if integer:
        assert np.array_equal(tot, tot_ref)                                 # integer counts: exact
    else:
        assert np.allclose(tot, tot_ref, rtol=1e-13, atol=0)
    assert tot[3] == 0.0
    rs = np.where(tot_ref > 0, 1e6 / np.where(tot_ref > 0, tot_ref, 1.0), 0.0)   # a cell without counts stays at 0
    T = (sp.diags(rs) @ C64).toarray()
    assert np.allclose(mean, T.mean(axis=0), rtol=1e-13, atol=0)
    assert np.allclose(var, T.var(axis=0), rtol=1e-10, atol=1e-9)
    assert mean[0] == 0.0 and var[0] == 0.0                               # the empty column
    # the zero-total row contributes nothing: the other rows alone give the same sums
    live = np.delete(T, 3, axis=0)
    assert np.allclose(mean * n, live.sum(axis=0), rtol=1e-13, atol=0)
    again = ds.tpm_stats()
    assert all(np.array_equal(a, b) for a, b in zip((tot, mean, var), again))    # fixed order: bit-identical
    ds.close()

    # without empty rows: totals equal the dense dataset's row_sums exactly, statistics its scaled col_stats
    Cf = ragged_counts(*shape, empty_row=False)
    sds, dds = eng.sparse_dataset(Cf), eng.dataset(Cf.toarray())
    tot_s, mean_s, var_s = sds.tpm_stats()
    tot_d = dds.row_sums()
    assert (tot_d > 0).all()
    if integer:
        assert np.array_equal(tot_s, tot_d)
    else:
        assert np.allclose(tot_s, tot_d, rtol=1e-13, atol=0)
    mean_d, var_d = dds.col_stats(row_scale=1e6 / tot_d)
    assert np.allclose(mean_s, mean_d, rtol=1e-12, atol=0)
    assert np.allclose(var_s, var_d, rtol=1e-12, atol=0)
    with pytest.raises(CnmfError, match="row_sums"):
        dds.tpm_stats()
    sds.close()
    dds.close()


@pytest.fixture
def sparse_calls(monkeypatch):
    """Shapes Engine.sparse_dataset is called with; force() makes every cells x all-genes matrix take the sparse form
    (TPM_DENSE_FRACTION = 0)."""
    from cnmf_b200 import pipeline
    from cnmf_b200.engine import Engine
    orig = Engine.sparse_dataset

    class Calls(list):
        def force(self):
            monkeypatch.setattr(pipeline, "TPM_DENSE_FRACTION", 0.0)

    made = Calls()

    def counted(self, X, *a, **kw):
        made.append(tuple(X.shape))
        return orig(self, X, *a, **kw)

    monkeypatch.setattr(Engine, "sparse_dataset", counted)
    return made


def write_sparse_counts(path, counts):
    """counts (cells x genes) stored CSR as `<path>`: a real .h5ad with anndata, else the `<path>.npz` side file."""
    from cnmf_b200 import io as cio
    X = sp.csr_matrix(np.asarray(counts, dtype=np.float64)) if not sp.issparse(counts) else counts.tocsr()
    n, g = X.shape
    cio.write_matrix(path, cio.CellGeneMatrix(X, ["c%d" % i for i in range(n)], ["g%d" % i for i in range(g)]))
    return path


def prepare(tmp_path, name, fn, g, **kw):
    from cnmf_b200 import cNMF
    obj = cNMF(output_dir=str(tmp_path), name=name)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        obj.prepare(fn, components=list(g["ks"]), n_iter=int(g["n_iter"]), seed=int(g["seed"]), densify=False,
                    beta_loss=g["beta_loss_arg"], num_highvar_genes=len(g["hvg_idx"]), init=g["init"], on_device=True,
                    **kw)
    return obj


def same_csr(a, b):
    a, b = a.tocsr(), b.tocsr()
    return (a.shape == b.shape and np.array_equal(a.indptr, b.indptr) and np.array_equal(a.indices, b.indices)
            and np.array_equal(a.data, b.data))


@pytest.mark.gpu
@pytest.mark.parametrize("tag", ["sim_mu", "c1_cd"])
def test_sparse_prepare_matches_dense_branch_and_reference(tmp_path, tag, sparse_calls):
    from cnmf_b200 import io as cio
    from cnmf_b200 import load_df_from_npz
    g = load_golden(tag)
    fn = write_sparse_counts(str(tmp_path / "counts.h5ad"), g["counts"])
    dense = prepare(tmp_path, "dense", fn, g)                         # fits: the dense on-device branch
    assert not sparse_calls
    sparse_calls.force()
    sparse = prepare(tmp_path, "sparse", fn, g)
    assert sparse_calls == [g["counts"].shape]
    hv_d = open(dense.paths["nmf_genes_list"]).read().split("\n")
    hv_s = open(sparse.paths["nmf_genes_list"]).read().split("\n")
    assert hv_d == hv_s
    for key in ("tpm", "normalized_counts"):
        a, b = cio.read_matrix(sparse.paths[key]), cio.read_matrix(dense.paths[key])
        assert a.is_sparse and same_csr(a.X, b.X), key
    sa, sb = load_df_from_npz(sparse.paths["tpm_stats"]), load_df_from_npz(dense.paths["tpm_stats"])
    assert np.allclose(sa.values, sb.values, rtol=1e-12, atol=0)
    # the two resident HVG matrices hold the same fp32 values, so the solves are expected to be bit-identical
    kw = dict(solver="cd" if str(g["beta_loss_arg"]) == "frobenius" else "mu", tol=1e-4, max_iter=1000)
    ks, seeds = [int(k) for k in g["ks"] for _ in range(3)], list(range(1, 3 * len(g["ks"]) + 1))
    sp_s, _, it_s, _ = sparse._resident_norm.factorize(ks, seeds, kw)
    sp_d, _, it_d, _ = dense._resident_norm.factorize(ks, seeds, kw)
    assert np.array_equal(it_s, it_d)
    assert max(rel(a, b) for a, b in zip(sp_s, sp_d)) < 1e-6
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        sparse.factorize()
        sparse.combine()
        dt = float(g["dt"])
        for k in g["ks"]:
            k = int(k)
            stats = sparse.consensus(k, skip_density_and_return_after_stats=True, show_clustering=False)
            ref_stats = g["stats_k%d" % k]
            assert abs(stats.loc["silhouette", "stats"] - ref_stats[2]) < 1e-4
            assert abs(stats.loc["prediction_error", "stats"] - ref_stats[3]) / ref_stats[3] < 1e-5
            sparse.consensus(k, density_threshold=dt, show_clustering=False)
            dts = str(dt).replace(".", "_")
            for key, name in (("consensus_spectra", "cspectra"), ("consensus_usages", "cusages"),
                              ("gene_spectra_tpm", "tpmspec"), ("gene_spectra_score", "score"),
                              ("starcat_spectra", "starcat")):
                got = load_df_from_npz(sparse.paths[key] % (k, dts)).values
                e = rel(got, g["%s_k%d" % (name, k)])
                limit = 3e-4 if (tag, k) == ("sim_mu", 4) else TOL_SPECTRA
                assert e < limit, (tag, k, key, e)
                assert os.path.exists(sparse.paths[key + "__txt"] % (k, dts))


@pytest.mark.gpu
def test_sparse_prepare_never_densifies(tmp_path, sparse_calls, monkeypatch):
    from cnmf_b200 import io as cio
    from cnmf_b200.engine import Dataset
    g = load_golden("sim_mu")
    n, g_all = g["counts"].shape
    fn = write_sparse_counts(str(tmp_path / "counts.h5ad"), g["counts"])
    dense_shapes = []
    orig_dense, orig_init = cio.CellGeneMatrix.dense, Dataset.__init__

    def dense(self, *a, **kw):
        dense_shapes.append(tuple(self.shape))
        return orig_dense(self, *a, **kw)

    def init(self, engine, X, *a, **kw):
        if X is not None:
            dense_shapes.append(tuple(X.shape))
        orig_init(self, engine, X, *a, **kw)

    monkeypatch.setattr(cio.CellGeneMatrix, "dense", dense)
    monkeypatch.setattr(Dataset, "__init__", init)
    sparse_calls.force()
    obj = prepare(tmp_path, "run", fn, g)
    assert sparse_calls == [(n, g_all)]
    assert (n, g_all) not in dense_shapes, dense_shapes
    assert obj._resident_norm.shape == (n, len(g["hvg_idx"]))


@pytest.mark.gpu
def test_sparse_prepare_refuses_zero_count_cell(tmp_path, sparse_calls):
    g = load_golden("sim_mu")
    counts = g["counts"].astype(np.float64)
    counts[5] = 0.0
    fn = write_sparse_counts(str(tmp_path / "counts.h5ad"), counts)
    sparse_calls.force()
    with pytest.raises(Exception, match="cells have zero counts of overdispersed genes"):
        prepare(tmp_path, "run", fn, g)
    assert sparse_calls == [counts.shape]


def atlas_counts(n, g, per_col, seed):
    """n x g integer counts as CSC: about per_col distinct cells per gene with counts 1..5, plus two ubiquitous genes
    (every cell non-zero).  Built column-wise; never dense."""
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
    vals = rng.integers(1, 6, size=idx.size).astype(np.float64)
    return sp.csc_matrix((vals, idx, col_ptr), shape=(n, g))


@pytest.mark.gpu
def test_atlas_prepare_to_consensus_stays_sparse(tmp_path, sparse_calls):
    """500 000 cells x 30 000 genes (~75 M stored counts): the dense counts dataset needs ~300 GB, so prepare keeps the
    counts sparse without forcing, and factorize -> combine -> consensus complete for one K."""
    from cnmf_b200 import cNMF, load_df_from_npz
    n, g, k = 500_000, 30_000, 5
    C = atlas_counts(n, g, 2500, 0)
    fn = write_sparse_counts(str(tmp_path / "atlas.h5ad"), C)
    genes = np.concatenate([[0, 1], np.random.RandomState(0).choice(np.arange(2, g), 1998, replace=False)])
    genes_file = str(tmp_path / "genes.txt")
    with open(genes_file, "w") as f:
        f.write("\n".join("g%d" % i for i in genes))
    del C
    obj = cNMF(output_dir=str(tmp_path), name="atlas")
    eng = obj.engine()
    free0, _, _ = eng.mem_info()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        obj.prepare(fn, components=[k], n_iter=4, seed=1, densify=False, genes_file=genes_file, max_NMF_iter=50,
                    on_device=True)
        free1, _, _ = eng.mem_info()
        print("atlas prepare: dense counts dataset %.1f GB, library footprint after prepare %.2f GB"
              % (eng.dense_dataset_bytes(n, g, obj.precision) / 1e9, (free0 - free1) / 1e9))
        assert sparse_calls == [(n, g)]
        assert obj._resident_norm.shape == (n, len(genes))
        obj.factorize()
        obj.combine()
        obj.consensus(k, density_threshold=2.0, show_clustering=False)
    assert sparse_calls == [(n, g), (n, g)]                           # consensus kept the TPM sparse too
    tag = (k, "2_0")
    usages = load_df_from_npz(obj.paths["consensus_usages"] % tag).values
    spectra_tpm = load_df_from_npz(obj.paths["gene_spectra_tpm"] % tag).values
    score = load_df_from_npz(obj.paths["gene_spectra_score"] % tag).values
    assert usages.shape == (n, k) and spectra_tpm.shape == (k, g) and score.shape == (k, g)
    assert np.isfinite(usages).all() and np.isfinite(spectra_tpm).all() and np.isfinite(score).all()
    stats = load_df_from_npz(obj.paths["tpm_stats"])
    assert stats.shape == (g, 2) and np.isfinite(stats.values).all()


# ------------------------------------------------------------------------------------ branch choice (CPU)
class _FakeDataset:
    """numpy stand-in for a resident dataset: what prepare(on_device=True) calls, in float64 from the fp32 values."""

    def __init__(self, X, sparse):
        self.X = (sp.csc_matrix(X, dtype=np.float32) if sparse else np.asarray(X, np.float32)).astype(np.float64)
        self.sparse = sparse
        self.shape = self.X.shape

    def _stats(self, rs=None):
        T = self.X if rs is None else sp.diags(rs) @ self.X
        m = np.asarray(T.sum(axis=0)).ravel() / self.shape[0]
        q = np.asarray((T.multiply(T) if sp.issparse(T) else T * T).sum(axis=0)).ravel() / self.shape[0]
        return m, np.maximum(q - m * m, 0.0)

    def row_sums(self):
        assert not self.sparse
        return self.X.sum(axis=1)

    def col_stats(self, row_scale=None):
        assert row_scale is None or not self.sparse
        return self._stats(row_scale)

    def tpm_stats(self, target_sum=1e6):
        assert self.sparse
        tot = np.asarray(self.X.sum(axis=1)).ravel()
        rs = np.where(tot != 0, target_sum / np.where(tot != 0, tot, 1.0), 0.0)
        return (tot,) + self._stats(rs)

    def from_columns(self, cols, scale):
        sub = self.X[:, cols]
        return _FakeDataset((sub.toarray() if self.sparse else sub) * np.asarray(scale, np.float32), False)

    def close(self):
        pass


class _FakeEngine:
    def __init__(self, free_bytes):
        self.free = free_bytes
        self.made = []

    def mem_info(self):
        return self.free, self.free, 0

    def dense_dataset_bytes(self, n, g, precision=None):
        return 20 * n * g

    def dataset(self, X, precision=None):
        self.made.append(("dense", X.shape))
        return _FakeDataset(X, False)

    def sparse_dataset(self, X, precision=None):
        self.made.append(("sparse", X.shape))
        return _FakeDataset(X, True)


def test_branch_choice_and_outputs_without_gpu(tmp_path):
    """Only sparse counts with densify=False whose dense dataset does not fit take the sparse branch, and its files
    equal the dense on-device branch's (same host arithmetic on the same totals)."""
    from cnmf_b200 import cNMF, load_df_from_npz, save_df_to_npz
    from cnmf_b200 import io as cio
    g = load_golden("c1_cd")
    n, g_all = g["counts"].shape
    sparse_fn = write_sparse_counts(str(tmp_path / "counts.h5ad"), g["counts"])
    df = pd.DataFrame(g["counts"].astype(np.float64), index=["c%d" % i for i in range(n)],
                      columns=["g%d" % i for i in range(g_all)])
    dense_fn = str(tmp_path / "counts.df.npz")
    save_df_to_npz(df, dense_fn)
    fits, tight = 2 * 20 * n * g_all, 20 * n * g_all          # _FakeEngine: 20 B per entry against 0.8 x free
    runs = {}
    for name, fn, free, densify in (("fits", sparse_fn, fits, False), ("densify", sparse_fn, tight, True),
                                    ("dense_input", dense_fn, tight, False), ("sparse", sparse_fn, tight, False)):
        obj = cNMF(output_dir=str(tmp_path), name=name)
        obj._engine = _FakeEngine(free)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            obj.prepare(fn, components=[7], n_iter=2, seed=1, densify=densify, num_highvar_genes=500, on_device=True)
        runs[name] = obj
        kinds = [kind for kind, shape in obj._engine.made if shape == (n, g_all)]
        assert kinds == (["sparse"] if name == "sparse" else ["dense"]), (name, obj._engine.made)
    a, b = runs["sparse"], runs["fits"]
    assert open(a.paths["nmf_genes_list"]).read() == open(b.paths["nmf_genes_list"]).read()
    for key in ("tpm", "normalized_counts"):
        assert same_csr(cio.read_matrix(a.paths[key]).X, cio.read_matrix(b.paths[key]).X), key
    assert np.allclose(load_df_from_npz(a.paths["tpm_stats"]).values, load_df_from_npz(b.paths["tpm_stats"]).values,
                       rtol=1e-12, atol=0)
    assert a._resident_norm.shape == (n, 500)
    assert np.array_equal(a._resident_norm.X, b._resident_norm.X)
