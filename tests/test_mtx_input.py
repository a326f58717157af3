"""10x Matrix Market input (`prepare -c <dir>/matrix.mtx[.gz]`, `--tpm` likewise) and the device builds of datasets from
CSR matrices.  The CPU tests check io.read_10x_mtx against what each test wrote (expected values from the triplets with
numpy) and prepare on an mtx directory against prepare on the same counts as .df.npz; the GPU tests check that a CSC
dataset transposed on the device and a dense dataset scattered on the device are bit-identical to the host-built ones,
and a whole run from an mtx directory against the same run from .h5ad.  Every fixture is generated here."""
import gzip
import os
import warnings
import zlib

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sp


# ------------------------------------------------------------------------------------ fixtures
def write_10x(path, n_genes, n_cells, triplets, ids=None, symbols=None, types=None, barcodes=None, legacy=False,
              field="integer"):
    """A 10x directory: triplets = (gene, cell, value) 0-based, written in the given order (duplicates kept).  v3
    (gz, features with a type column) unless legacy.  field 'pattern' writes no values."""
    os.makedirs(path, exist_ok=True)
    ids = ids if ids is not None else ["ENSG%05d" % i for i in range(n_genes)]
    symbols = symbols if symbols is not None else ["G%d" % i for i in range(n_genes)]
    types = types if types is not None else ["Gene Expression"] * n_genes
    barcodes = barcodes if barcodes is not None else ["AAAC-%d" % i for i in range(n_cells)]
    lines = ["%%%%MatrixMarket matrix coordinate %s general" % field, "%", "%d %d %d" % (n_genes, n_cells, len(triplets))]
    for gi, ci, v in triplets:
        lines.append("%d %d" % (gi + 1, ci + 1) if field == "pattern" else
                     "%d %d %s" % (gi + 1, ci + 1, repr(float(v)) if field == "real" else int(v)))
    mtx = "\n".join(lines) + "\n"
    feats = "".join("%s\t%s\n" % (i, s) if legacy else "%s\t%s\t%s\n" % (i, s, t) for i, s, t in zip(ids, symbols, types))
    bcs = "".join(b + "\n" for b in barcodes)
    files = {"matrix.mtx": mtx, "genes.tsv" if legacy else "features.tsv": feats, "barcodes.tsv": bcs}
    for name, text in files.items():
        if legacy:
            with open(os.path.join(path, name), "w") as f:
                f.write(text)
        else:
            with gzip.open(os.path.join(path, name + ".gz"), "wt") as f:
                f.write(text)
    return path


def expected_dense(n_genes, n_cells, triplets, keep=None, pattern=False):
    """cells x genes float32 from the triplets: values rounded to float32, then repeated coordinates added"""
    E = np.zeros((n_cells, n_genes), np.float32)
    for gi, ci, v in triplets:
        E[ci, gi] += np.float32(1.0 if pattern else v)
    return E if keep is None else E[:, keep]


def random_triplets(n_genes, n_cells, density, seed, shuffle=True):
    rng = np.random.RandomState(seed)
    M = sp.random(n_genes, n_cells, density=density, format="coo", random_state=rng,
                  data_rvs=lambda m: rng.randint(1, 40, size=m).astype(np.float64))
    t = list(zip(M.row.tolist(), M.col.tolist(), M.data.tolist()))
    if shuffle:
        rng.shuffle(t)
    return t


def assert_canonical_csr(X, E):
    assert sp.issparse(X) and X.format == "csr" and X.dtype == np.float32
    assert X.has_canonical_format
    assert np.array_equal(X.toarray(), E)


# ------------------------------------------------------------------------------------ io (CPU)
def test_v3_layout_drops_other_feature_types(tmp_path):
    from cnmf_b200 import io as cio
    n_genes, n_cells = 7, 9
    types = ["Gene Expression"] * 3 + ["Antibody Capture"] + ["Gene Expression"] * 3
    t = random_triplets(n_genes, n_cells, 0.5, 1)
    t.append((3, 0, 11.0))                                             # the antibody row holds counts
    d = write_10x(str(tmp_path / "v3"), n_genes, n_cells, t, types=types)
    keep = [0, 1, 2, 4, 5, 6]
    m = cio.read_counts(os.path.join(d, "matrix.mtx.gz"))
    assert_canonical_csr(m.X, expected_dense(n_genes, n_cells, t, keep))
    assert list(m.var_names) == ["G%d" % i for i in keep]
    assert list(m.obs_names) == ["AAAC-%d" % i for i in range(n_cells)]


def test_v2_layout(tmp_path):
    from cnmf_b200 import io as cio
    n_genes, n_cells = 6, 5
    t = random_triplets(n_genes, n_cells, 0.6, 2)
    d = write_10x(str(tmp_path / "v2"), n_genes, n_cells, t, legacy=True)
    m = cio.read_counts(os.path.join(d, "matrix.mtx"))
    assert_canonical_csr(m.X, expected_dense(n_genes, n_cells, t))
    assert list(m.var_names) == ["G%d" % i for i in range(n_genes)]
    assert list(m.obs_names) == ["AAAC-%d" % i for i in range(n_cells)]


@pytest.mark.parametrize("legacy", [False, True])
def test_file_name_is_ignored_only_the_directory_counts(tmp_path, legacy):
    from cnmf_b200 import io as cio
    t = random_triplets(5, 4, 0.5, 3)
    d = write_10x(str(tmp_path / "d"), 5, 4, t, legacy=legacy)
    a = cio.read_counts(os.path.join(d, "matrix.mtx"))
    b = cio.read_counts(os.path.join(d, "matrix.mtx.gz"))
    assert (a.X != b.X).nnz == 0 and a.X.shape == b.X.shape
    assert a.var_names.equals(b.var_names) and a.obs_names.equals(b.obs_names)


def test_symbols_made_unique_as_anndata_does(tmp_path):
    from cnmf_b200 import io as cio
    d = write_10x(str(tmp_path / "u"), 5, 2, [(0, 0, 1), (4, 1, 2)], symbols=["A", "A", "A-1", "B", "A"])
    m = cio.read_counts(os.path.join(d, "matrix.mtx.gz"))
    assert list(m.var_names) == ["A", "A-2", "A-1", "B", "A-3"]
    assert list(cio.make_index_unique(["x", "y"])) == ["x", "y"]


def test_real_values_round_through_float32_and_pattern_gives_ones(tmp_path):
    from cnmf_b200 import io as cio
    t = [(0, 0, 0.1), (1, 2, 1.0 / 3.0), (2, 1, 123456.789), (1, 0, 2.5)]
    d = write_10x(str(tmp_path / "real"), 3, 3, t, field="real")
    m = cio.read_counts(os.path.join(d, "matrix.mtx.gz"))
    E = expected_dense(3, 3, t)
    assert_canonical_csr(m.X, E)
    assert float(E[0, 0]) == float(np.float32(0.1)) != 0.1              # rounded, not kept in float64
    d = write_10x(str(tmp_path / "pattern"), 3, 3, t, field="pattern")
    m = cio.read_counts(os.path.join(d, "matrix.mtx.gz"))
    assert_canonical_csr(m.X, expected_dense(3, 3, t, pattern=True))


def test_unsorted_triplets_with_a_repeated_coordinate_are_summed(tmp_path):
    from cnmf_b200 import io as cio
    t = [(2, 3, 4), (0, 1, 1), (2, 3, 5), (1, 0, 7), (0, 1, 2), (2, 0, 1), (2, 3, 1)]
    d = write_10x(str(tmp_path / "dup"), 3, 4, t)
    m = cio.read_counts(os.path.join(d, "matrix.mtx.gz"))
    E = expected_dense(3, 4, t)
    assert E[3, 2] == 10 and E[1, 0] == 3
    assert_canonical_csr(m.X, E)
    assert m.X.nnz == 4


def test_missing_file_is_named(tmp_path):
    from cnmf_b200 import io as cio
    d = write_10x(str(tmp_path / "miss"), 3, 3, [(0, 0, 1)])
    os.remove(os.path.join(d, "barcodes.tsv.gz"))
    with pytest.raises(FileNotFoundError, match="barcodes.tsv.gz"):
        cio.read_counts(os.path.join(d, "matrix.mtx.gz"))


def counts_as_10x(path, counts, extra_antibody=True):
    """cells x genes integer counts as a v3 directory named c%d / g%d, plus (extra_antibody) one Antibody Capture
    feature with counts in every cell, which the reader drops"""
    n, g = counts.shape
    C = sp.coo_matrix(np.asarray(counts).T)
    t = list(zip(C.row.tolist(), C.col.tolist(), C.data.tolist()))
    symbols, types = ["g%d" % i for i in range(g)], ["Gene Expression"] * g
    if extra_antibody:
        t += [(g, c, 1 + c % 5) for c in range(n)]
        symbols, types = symbols + ["CD3"], types + ["Antibody Capture"]
    write_10x(path, len(symbols), n, t, symbols=symbols, types=types, barcodes=["c%d" % i for i in range(n)])
    return os.path.join(path, "matrix.mtx.gz")


def counts_as_df_npz(fn, counts):
    from cnmf_b200 import save_df_to_npz
    n, g = counts.shape
    save_df_to_npz(pd.DataFrame(np.asarray(counts, np.float64), index=["c%d" % i for i in range(n)],
                                columns=["g%d" % i for i in range(g)]), fn)
    return fn


def assert_same_files(dir_a, dir_b):
    """every file under dir_a exists under dir_b with the same content: .npz array by array (names included), the
    rest byte for byte"""
    files_a = sorted(os.path.relpath(os.path.join(r, f), dir_a) for r, _, fs in os.walk(dir_a) for f in fs)
    files_b = sorted(os.path.relpath(os.path.join(r, f), dir_b) for r, _, fs in os.walk(dir_b) for f in fs)
    assert files_a == files_b
    for rel in files_a:
        pa, pb = os.path.join(dir_a, rel), os.path.join(dir_b, rel)
        if rel.endswith(".npz"):
            with np.load(pa, allow_pickle=True) as a, np.load(pb, allow_pickle=True) as b:
                assert sorted(a.files) == sorted(b.files), rel
                for k in a.files:
                    assert a[k].dtype == b[k].dtype and np.array_equal(a[k], b[k]), (rel, k)
        else:
            assert open(pa, "rb").read() == open(pb, "rb").read(), rel
    return files_a


def run_prepare(out, fn, **kw):
    from cnmf_b200 import cNMF
    obj = cNMF(output_dir=str(out), name="run")
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        obj.prepare(fn, components=[3, 4], n_iter=3, seed=5, num_highvar_genes=30, **kw)
    return obj


def test_prepare_from_mtx_writes_what_prepare_from_df_npz_writes(tmp_path):
    from cnmf_b200.synth import make_counts
    counts = make_counts(300, 60, k_true=3, seed=2, libsize=300.0)
    mtx = counts_as_10x(str(tmp_path / "tenx"), counts)
    npz = counts_as_df_npz(str(tmp_path / "counts.df.npz"), counts)
    run_prepare(tmp_path / "a", mtx, on_device=False)
    run_prepare(tmp_path / "b", npz, on_device=False)
    files = assert_same_files(str(tmp_path / "a"), str(tmp_path / "b"))
    assert any("tpm_stats" in f for f in files) and any("norm_counts" in f for f in files)
    assert any("overdispersed_genes" in f for f in files) and any("nmf_params" in f for f in files)
    # -c <dir>/matrix.mtx names the same directory
    run_prepare(tmp_path / "c", os.path.join(str(tmp_path / "tenx"), "matrix.mtx"), on_device=False)
    assert_same_files(str(tmp_path / "c"), str(tmp_path / "b"))


def test_tpm_given_as_mtx(tmp_path):
    from cnmf_b200.synth import make_counts
    counts = make_counts(300, 60, k_true=3, seed=4, libsize=300.0)
    tpm = np.round(counts / counts.sum(axis=1, keepdims=True) * 1e4)     # integer-valued, as an mtx 'integer' file
    npz = counts_as_df_npz(str(tmp_path / "counts.df.npz"), counts)
    tpm_mtx = counts_as_10x(str(tmp_path / "tpm10x"), tpm)
    tpm_npz = counts_as_df_npz(str(tmp_path / "tpm.df.npz"), tpm)
    run_prepare(tmp_path / "a", npz, tpm_fn=tpm_mtx)
    run_prepare(tmp_path / "b", npz, tpm_fn=tpm_npz)
    assert_same_files(str(tmp_path / "a"), str(tmp_path / "b"))


# ------------------------------------------------------------------------------------ device builds (GPU)
@pytest.fixture(scope="module")
def eng():
    from cnmf_b200.engine import Engine
    return Engine(0)


def csr_case(name):
    """(CSR float32 matrix) of one named shape"""
    rng = np.random.RandomState(zlib.crc32(name.encode()))
    ints = lambda m: rng.randint(1, 30, size=m).astype(np.float32)     # noqa: E731
    if name == "empty_rows_and_cols":
        M = sp.random(400, 90, density=0.05, format="lil", random_state=rng, data_rvs=ints)
        M[7, :] = 0
        M[:, 11] = 0
        M[:, 89] = 0
        M = M.tocsr()
    elif name == "nnz0":
        M = sp.csr_matrix((50, 40), dtype=np.float32)
    elif name == "one_row":
        M = sp.random(1, 300, density=0.3, format="csr", random_state=rng, data_rvs=ints)
    elif name == "one_col":
        M = sp.random(300, 1, density=0.3, format="csr", random_state=rng, data_rvs=ints)
    elif name == "full_col_500k":
        n = 500_000
        R = sp.random(n, 3, density=0.01, format="csc", random_state=rng, data_rvs=ints)
        M = sp.hstack([R[:, :1], sp.csc_matrix(rng.randint(1, 9, size=(n, 1)).astype(np.float32)), R[:, 1:]]).tocsr()
    elif name == "cols_70000":
        M = sp.random(3000, 70_000, density=0.002, format="csr", random_state=rng, data_rvs=ints)
    else:                                                              # "rows_<n>": around the row-block size
        M = sp.random(int(name.split("_")[1]), 50, density=0.2, format="csr", random_state=rng, data_rvs=ints)
    M = sp.csr_matrix(M, dtype=np.float32)
    M.sort_indices()
    return M


ROW_BLOCK = 256      # CSR_ROW_BLOCK (engine.h): rows per block of the device transpose at these widths
SHAPES = (["empty_rows_and_cols", "nnz0", "one_row", "one_col", "full_col_500k", "cols_70000"]
          + ["rows_%d" % (m * ROW_BLOCK + d) for m in (1, 2) for d in (-1, 0, 1)])


@pytest.mark.gpu
@pytest.mark.parametrize("name", SHAPES)
def test_device_transpose_equals_host_tocsc(eng, name):
    M = csr_case(name)
    a, b = eng.sparse_dataset(M), eng.sparse_dataset(M.tocsc())
    ref = M.tocsc()
    for key, want in (("csc_col_ptr", ref.indptr.astype(np.int64)), ("csc_row_idx", ref.indices.astype(np.int32)),
                      ("csc_values", ref.data.astype(np.float32))):
        got, host = a.operand(key), b.operand(key)
        assert got.dtype == host.dtype and np.array_equal(got, host), key
        assert np.array_equal(got, want), key
    assert a.form == b.form and a.sums() == b.sums() and a.shape == b.shape
    for x, y in zip(a.tpm_stats(), b.tpm_stats()):
        assert np.array_equal(x, y, equal_nan=True)
    for x, y in zip(a.col_stats(), b.col_stats()):
        assert np.array_equal(x, y)
    g = M.shape[1]
    cols = np.arange(g)[::-1][: max(1, g // 2)].copy()
    scale = (1.0 / (1.0 + np.arange(len(cols)))).astype(np.float32)
    fa, fb = a.from_columns(cols, scale), b.from_columns(cols, scale)
    assert fa.form == fb.form
    assert np.array_equal(fa.operand("X"), fb.operand("X"))
    for ds in (a, b, fa, fb):
        ds.close()


def dense_inputs():
    from cnmf_b200.synth import make_counts
    counts = make_counts(500, 160, k_true=4, seed=11, libsize=600.0).astype(np.float64)
    counts[3, :] = 0.0                                                 # an empty row
    hvg = counts / np.where(counts.std(axis=0, ddof=1) > 0, counts.std(axis=0, ddof=1), 1.0)
    tot = counts.sum(axis=1, keepdims=True)
    tpm = np.divide(counts, tot, out=np.zeros_like(counts), where=tot > 0) * 1e6
    return {"counts": counts, "hvg": hvg, "tpm": tpm}


OPERAND_NAMES = ["X", "Xt", "X_hi", "X_lo", "Xt_hi", "Xt_lo", "X_h16", "Xt_h16", "row_scale", "col_scale"]


def assert_same_dataset(a, b):
    assert a.shape == b.shape and a.form == b.form and a.sums() == b.sums()
    for name in OPERAND_NAMES:
        x, y = a.operand(name), b.operand(name)
        assert (x is None) == (y is None), name
        if x is not None:
            assert np.array_equal(x.view(np.uint8), y.view(np.uint8)), name     # bit for bit
    if a.fp64:                                                        # X64 read back through an identity product
        eye = np.eye(a.shape[1])
        assert np.array_equal(a.nndsvd_gemm(eye, False).view(np.uint64), b.nndsvd_gemm(eye, False).view(np.uint64))


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["f16x2", "tf32x3", "tf32x3-general", "fp32", "fp64"])
@pytest.mark.parametrize("kind", ["counts", "hvg", "tpm"])
def test_dense_dataset_from_csr_equals_dataset_from_toarray(eng, precision, kind):
    X = sp.csr_matrix(dense_inputs()[kind])
    a, b = eng.dataset(X, precision=precision), eng.dataset(X.toarray(), precision=precision)
    if kind == "counts" and precision in ("f16x2", "tf32x3"):
        assert a.form.endswith("exact")
    assert_same_dataset(a, b)
    a.close()
    b.close()


@pytest.mark.gpu
def test_dense_dataset_from_csr_in_several_slices(eng):
    """more than 2^24 stored entries: the entries cross in several slices (CSR_STAGE_ENTRIES)"""
    rng = np.random.RandomState(5)
    X = sp.random(40_000, 1500, density=0.5, format="csr", random_state=rng,
                  data_rvs=lambda m: rng.randint(1, 20, size=m).astype(np.float32))
    assert X.nnz > 2 ** 24
    a, b = eng.dataset(X, precision="fp32"), eng.dataset(X.toarray(), precision="fp32")
    assert_same_dataset(a, b)
    a.close()
    b.close()


def test_sparse_inputs_reach_the_csr_entry_points(monkeypatch):
    """Engine.sparse_dataset hands CSR to the device transpose and other matrices to the host CSC route, fp64 is
    refused before either; Dataset hands any scipy matrix to the CSR scatter (float or float64) -- checked with a
    recording stand-in for the library"""
    from cnmf_b200 import engine as E
    calls = []

    class Lib:
        def __getattr__(self, name):
            def f(*a):
                calls.append(name)
                return 0
            return f

    class Eng:
        lib = Lib()
        _h = None

    monkeypatch.setattr(E.Dataset, "close", lambda self: None)
    X = sp.random(20, 10, density=0.3, format="csr", random_state=0)
    E.Engine.sparse_dataset(Eng(), X)
    E.Engine.sparse_dataset(Eng(), X.tocoo())
    E.Dataset(Eng(), X.tocsc())
    E.Dataset(Eng(), X, precision="fp64")
    with pytest.raises(NotImplementedError):
        E.Engine.sparse_dataset(Eng(), X, precision="fp64")
    created = [c for c in calls if c.startswith("cnmf_dataset_create")]
    assert created == ["cnmf_dataset_create_csr", "cnmf_dataset_create_csc", "cnmf_dataset_create_from_csr",
                       "cnmf_dataset_create_from_csr_f64"]


@pytest.mark.gpu
def test_run_from_mtx_equals_run_from_h5ad_and_never_densifies(tmp_path, monkeypatch):
    from cnmf_b200 import cNMF, pipeline
    from cnmf_b200 import io as cio
    from cnmf_b200.engine import Dataset
    from cnmf_golden import load_golden
    g = load_golden("sim_mu")
    counts = g["counts"].astype(np.float64)
    n, g_all = counts.shape
    n_hvg = len(g["hvg_idx"])
    mtx = counts_as_10x(str(tmp_path / "tenx"), counts)
    h5ad = str(tmp_path / "counts.h5ad")
    cio.write_matrix(h5ad, cio.CellGeneMatrix(sp.csr_matrix(counts), ["c%d" % i for i in range(n)],
                                              ["g%d" % i for i in range(g_all)]))
    monkeypatch.setattr(pipeline, "TPM_DENSE_FRACTION", 0.0)          # the sparse branch everywhere
    ks = [int(k) for k in g["ks"]]
    dt = float(g["dt"])
    dense_shapes = []

    def run(out, fn, watch):
        obj = cNMF(output_dir=str(out), name="run")
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            obj.prepare(fn, components=ks, n_iter=int(g["n_iter"]), seed=int(g["seed"]), densify=False,
                        beta_loss=g["beta_loss_arg"], num_highvar_genes=n_hvg, init=g["init"], on_device=True)
            obj = cNMF(output_dir=str(out), name="run")               # factorize / consensus as separate commands do
            if watch:
                watch()
            obj.factorize()
            obj.combine()
            for k in ks:
                obj.consensus(k, density_threshold=dt, show_clustering=False)

    def watch():
        orig_dense, orig_init = cio.CellGeneMatrix.dense, Dataset.__init__
        orig_toarray = {cls: cls.toarray for cls in (sp.csr_matrix, sp.csc_matrix, sp.coo_matrix)}

        def dense(self, *a, **kw):
            dense_shapes.append(tuple(self.shape))
            return orig_dense(self, *a, **kw)

        def init(self, engine, X, *a, **kw):
            if X is not None and not sp.issparse(X):
                dense_shapes.append(tuple(np.shape(X)))
            orig_init(self, engine, X, *a, **kw)

        monkeypatch.setattr(cio.CellGeneMatrix, "dense", dense)
        monkeypatch.setattr(Dataset, "__init__", init)
        for cls, f in orig_toarray.items():
            def toarray(self, *a, _f=f, **kw):
                dense_shapes.append(tuple(self.shape))
                return _f(self, *a, **kw)
            monkeypatch.setattr(cls, "toarray", toarray)

    run(tmp_path / "h5ad", h5ad, None)
    run(tmp_path / "mtx", mtx, watch)
    assert not [s for s in dense_shapes if s[0] == n and s[1] in (g_all, n_hvg)], dense_shapes
    files = assert_same_files(str(tmp_path / "mtx"), str(tmp_path / "h5ad"))
    for k in ks:
        assert any(("spectra.k_%d.dt_" % k) in f and f.endswith(".consensus.txt") for f in files)
        assert any(("gene_spectra_score.k_%d" % k) in f for f in files)
