"""Load the UNMODIFIED reference module src/cnmf/cnmf.py of a dylkot/cNMF checkout named by the CNMF_REFERENCE
environment variable (test infrastructure for the fixture generators; see oracle/__init__.py).

The reference imports ``scanpy`` and ``matplotlib`` at module level (cnmf.py:24,26); neither
is installed here and there is no network.  This file registers minimal stand-ins in
``sys.modules`` that cover exactly what the hot path touches (SURVEY.md appendix,
"Oracle shim requirements"):

  sc.AnnData(X=, obs=, var=)   cnmf.py:396-402,425-431
  sc.read / sc.write           cnmf.py:384,410,561,726,873,950   (pickle on disk)
  sc.pp.normalize_total        cnmf.py:250
  sc.pp.scale(zero_center=False)  cnmf.py:538,967  (sparse X only)
  adata[:, names], .copy(), .X assignment, .obs.index, .var.index

and then loads cnmf.py by file path so that ``cnmf/__init__.py`` (which imports
preprocess.py -> scanpy/harmonypy) is not executed.

This module only works where such a checkout exists.  No test imports it: the tests compare against the fixtures
it produced (tests/golden/).
"""
import importlib.util
import os
import pickle
import sys
import types

import numpy as np
import pandas as pd
import scipy.sparse as sp

def reference_file():
    """src/cnmf/cnmf.py of the checkout named by CNMF_REFERENCE (an explicit error when the variable is unset)."""
    root = os.environ.get("CNMF_REFERENCE")
    if not root:
        raise RuntimeError("CNMF_REFERENCE is not set: point it at a dylkot/cNMF checkout")
    return os.path.join(root, "src", "cnmf", "cnmf.py")


class AnnDataLite:
    """Dense/CSR cells x genes container with the few attributes cnmf.py uses."""

    def __init__(self, X=None, obs=None, var=None):
        self.X = X
        self.obs = obs if obs is not None else pd.DataFrame(index=[str(i) for i in range(X.shape[0])])
        self.var = var if var is not None else pd.DataFrame(index=[str(i) for i in range(X.shape[1])])

    @property
    def shape(self):
        return self.X.shape

    def copy(self):
        return AnnDataLite(self.X.copy(), self.obs.copy(), self.var.copy())

    def __getitem__(self, key):
        rows, cols = key
        assert rows == slice(None)
        idx = self.var.index.get_indexer(list(cols))
        assert (idx >= 0).all()
        X = self.X[:, idx]
        return AnnDataLite(X.copy(), self.obs.copy(), self.var.iloc[idx].copy())


def _read(path):
    with open(path, "rb") as f:
        return pickle.load(f)


def _write(path, adata):
    with open(path, "wb") as f:
        pickle.dump(adata, f, protocol=4)


def _normalize_total(adata, target_sum=1e6):
    X = adata.X
    if sp.issparse(X):
        tot = np.asarray(X.sum(axis=1)).reshape(-1)
        scale = target_sum / tot
        adata.X = sp.diags(scale) @ X
        adata.X = sp.csr_matrix(adata.X)
    else:
        X = X.astype(np.float64) if not np.issubdtype(X.dtype, np.floating) else X
        tot = X.sum(axis=1, keepdims=True)
        adata.X = X / tot * target_sum


def _scale(adata, zero_center=False):
    assert not zero_center
    X = sp.csc_matrix(adata.X, dtype=np.float64)
    n = X.shape[0]
    mean = np.asarray(X.mean(axis=0)).reshape(-1)
    sq = np.asarray(X.multiply(X).mean(axis=0)).reshape(-1)
    var = (sq - mean ** 2) * (n / (n - 1))
    std = np.sqrt(var)
    std[std == 0] = 1
    adata.X = sp.csr_matrix(X @ sp.diags(1.0 / std))


def _install_stubs():
    if "scanpy" not in sys.modules:
        sc = types.ModuleType("scanpy")
        sc.AnnData = AnnDataLite
        sc.read = _read
        sc.write = _write
        pp = types.ModuleType("scanpy.pp")
        pp.normalize_total = _normalize_total
        pp.scale = _scale
        sc.pp = pp
        sys.modules["scanpy"] = sc
        sys.modules["scanpy.pp"] = pp
    if "matplotlib" not in sys.modules:
        mpl = types.ModuleType("matplotlib")
        plt = types.ModuleType("matplotlib.pyplot")
        mpl.pyplot = plt
        sys.modules["matplotlib"] = mpl
        sys.modules["matplotlib.pyplot"] = plt


_REF = None


def load_reference():
    """Return the reference ``cnmf`` module object (unmodified source, loaded by path)."""
    global _REF
    if _REF is not None:
        return _REF
    path = reference_file()
    if not os.path.exists(path):
        raise RuntimeError("reference source not found: %s (CNMF_REFERENCE)" % path)
    _install_stubs()
    spec = importlib.util.spec_from_file_location("cnmf_reference_module", path)
    mod = importlib.util.module_from_spec(spec)
    # AnnDataLite must be picklable under a stable module name
    spec.loader.exec_module(mod)
    _REF = mod
    return mod
