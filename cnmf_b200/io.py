"""On-disk codecs of the cNMF file ledger (host code).

``.df.npz``  = np.savez_compressed(data=values, index=index, columns=columns), read back with
               allow_pickle (reference cnmf.py:31-40) -- byte-layout compatible, so files written by
               either implementation are readable by the other.
``.txt``     = tab-separated DataFrame.to_csv (cnmf.py:34-35).
cells x genes matrices (``norm_counts``, ``tpm``): the reference stores AnnData ``.h5ad`` through
scanpy (cnmf.py:410,561).  anndata / h5py are optional here: with anndata installed real ``.h5ad``
files are read and written; without it the same matrix goes to ``<path>.npz`` (dense, with
obs / var names) and a note is printed once.
"""
import os
import warnings

import numpy as np
import pandas as pd


def save_df_to_npz(obj, filename):
    np.savez_compressed(filename, data=obj.values, index=obj.index.values, columns=obj.columns.values)


def save_df_to_text(obj, filename):
    obj.to_csv(filename, sep="\t")


def load_df_from_npz(filename):
    with np.load(filename, allow_pickle=True) as f:
        obj = pd.DataFrame(**f)
    return obj


class CellGeneMatrix:
    """Minimal cells x genes container (dense ndarray or scipy sparse) with obs / var names."""

    def __init__(self, X, obs_names, var_names):
        self.X = X
        self.obs_names = pd.Index(obs_names)
        self.var_names = pd.Index(var_names)

    @property
    def shape(self):
        return self.X.shape

    @property
    def is_sparse(self):
        return hasattr(self.X, "tocsr")

    def dense(self, dtype=np.float64):
        X = self.X.toarray() if hasattr(self.X, "toarray") else np.asarray(self.X)
        return np.ascontiguousarray(X, dtype=dtype)

    def subset_genes(self, names):
        idx = self.var_names.get_indexer(list(names))
        if (idx < 0).any():
            raise KeyError("genes not found: %s" % list(np.asarray(names)[idx < 0][:4]))
        return CellGeneMatrix(self.X[:, idx], self.obs_names, self.var_names[idx]), idx


def _have_anndata():
    try:
        import anndata  # noqa: F401
        return True
    except Exception:
        return False


_warned = False


def write_matrix(path, mat):
    global _warned
    if _have_anndata():
        import anndata
        ad = anndata.AnnData(X=mat.X, obs=pd.DataFrame(index=mat.obs_names), var=pd.DataFrame(index=mat.var_names))
        ad.write(path)
        return path
    if not _warned:
        warnings.warn("anndata is not installed: cells x genes matrices are stored as '<name>.h5ad.npz' "
                      "instead of '.h5ad'", UserWarning)
        _warned = True
    names = dict(obs=np.asarray(mat.obs_names, dtype=object), var=np.asarray(mat.var_names, dtype=object))
    if hasattr(mat.X, "tocsr"):       # sparse stays sparse (the reference keeps CSR unless --densify, cnmf.py:399-405)
        csr = mat.X.tocsr()
        np.savez(path + ".npz", csr_data=csr.data.astype(np.float64), csr_indices=csr.indices, csr_indptr=csr.indptr,
                 csr_shape=np.asarray(csr.shape), **names)
    else:
        np.savez(path + ".npz", X=mat.dense(np.float64), **names)
    return path + ".npz"


def read_matrix(path):
    if os.path.exists(path) and _have_anndata():
        import anndata
        ad = anndata.read_h5ad(path)
        return CellGeneMatrix(ad.X, ad.obs.index, ad.var.index)
    if os.path.exists(path + ".npz"):
        with np.load(path + ".npz", allow_pickle=True) as f:
            if "csr_data" in f:
                import scipy.sparse as sp
                X = sp.csr_matrix((f["csr_data"], f["csr_indices"], f["csr_indptr"]), shape=tuple(f["csr_shape"]))
                return CellGeneMatrix(X, f["obs"], f["var"])
            return CellGeneMatrix(f["X"], f["obs"], f["var"])
    if os.path.exists(path):
        raise RuntimeError("%s is an .h5ad file but anndata is not installed" % path)
    raise FileNotFoundError(path)


def make_index_unique(names, join="-"):
    """anndata.utils.make_index_unique: the first occurrence keeps its name, each later duplicate v becomes v-1, v-2, ...
    (one counter per name), skipping any candidate already present."""
    names = pd.Index(names)
    if names.is_unique:
        return names
    values = names.values.copy()
    dup = names.duplicated(keep="first")
    taken = set(values)
    counter = {}
    renamed = []
    for v in values[dup]:
        while True:
            counter[v] = counter.get(v, 0) + 1
            candidate = v + join + str(counter[v])
            if candidate not in taken:
                taken.add(candidate)
                renamed.append(candidate)
                break
    values[dup] = renamed
    return pd.Index(values)


def _read_tsv_column(path, col):
    if not os.path.exists(path):
        raise FileNotFoundError(path)
    # names are the file's text (no NA parsing): 10x identifiers and symbols are strings
    return pd.read_csv(path, header=None, sep="\t", dtype=str, keep_default_na=False, usecols=[col])[col].values


def read_10x_mtx(path):
    """scanpy.read_10x_mtx(path) with its defaults (var_names='gene_symbols', make_unique=True, gex_only=True) as a
    CellGeneMatrix holding canonical float32 CSR (cells x genes).  The legacy (Cell Ranger 2) layout, recognised by
    genes.tsv, is matrix.mtx / genes.tsv / barcodes.tsv; otherwise matrix.mtx.gz / features.tsv.gz / barcodes.tsv.gz,
    of which only the 'Gene Expression' features are kept.  The genes x cells matrix is cast to float32 before its
    duplicates are summed, as scanpy's read_mtx does.  Needs scipy only."""
    import scipy.io
    import scipy.sparse as sp
    legacy = os.path.isfile(os.path.join(path, "genes.tsv"))
    suffix = "" if legacy else ".gz"
    mtx = os.path.join(path, "matrix.mtx" + suffix)
    features = os.path.join(path, ("genes" if legacy else "features") + ".tsv" + suffix)
    barcodes = os.path.join(path, "barcodes.tsv" + suffix)
    for fn in (mtx, features, barcodes):
        if not os.path.exists(fn):
            raise FileNotFoundError(fn)
    with warnings.catch_warnings():        # scipy >= 1.18 announces sparse arrays as mmread's future return type
        warnings.simplefilter("ignore", DeprecationWarning)
        M = scipy.io.mmread(mtx)
    X = sp.csr_matrix(sp.coo_matrix(M).astype(np.float32).T)      # duplicates summed here
    var_names = make_index_unique(_read_tsv_column(features, 1))
    obs_names = _read_tsv_column(barcodes, 0)
    if len(var_names) != X.shape[1] or len(obs_names) != X.shape[0]:
        raise ValueError("%s is %d genes x %d cells, but %s names %d and %s %d" % (
            mtx, X.shape[1], X.shape[0], features, len(var_names), barcodes, len(obs_names)))
    if not legacy:
        gex = _read_tsv_column(features, 2) == "Gene Expression"
        X, var_names = X[:, np.flatnonzero(gex)], var_names[gex]
    X.sum_duplicates()            # canonical: sorted column indices (a no-op when they already are)
    return CellGeneMatrix(X, obs_names, var_names)


def read_counts(counts_fn):
    """Input counts as accepted by the reference's prepare() (cnmf.py:383-414): .h5ad, df.npz, tab-delimited text, or
    10x Matrix Market output given as <dir>/matrix.mtx or <dir>/matrix.mtx.gz: the directory is read as
    scanpy.read_10x_mtx reads it (read_10x_mtx), whatever the file name."""
    if counts_fn.endswith(".h5ad"):
        return read_matrix(counts_fn)
    if counts_fn.endswith(".mtx") or counts_fn.endswith(".mtx.gz"):
        return read_10x_mtx(os.path.dirname(counts_fn))
    if counts_fn.endswith(".npz"):
        df = load_df_from_npz(counts_fn)
    else:
        df = pd.read_csv(counts_fn, sep="\t", index_col=0)
    return CellGeneMatrix(df.values, df.index, df.columns)
