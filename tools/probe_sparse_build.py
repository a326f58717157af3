#!/usr/bin/env python
"""GPU probe: what reading 10x counts and building datasets from CSR matrices costs, host route against device route.

  python tools/probe_sparse_build.py [atlas] [hvg]

  atlas  500 000 cells x 30 000 genes, ~75 M stored integer counts:
         - io.read_10x_mtx of the counts written as a legacy (uncompressed) 10x directory: the Matrix Market parse;
           a .gz directory adds the single-threaded inflate on top
         - sparse (CSC) dataset: host tocsc + upload of the CSC arrays (Engine.sparse_dataset of the CSC matrix)
           against upload of the CSR arrays + device transpose (Engine.sparse_dataset of the CSR matrix)
  hvg    2 000 000 cells x 2 000 genes at density 0.3 (~1.2 G stored entries):
         - dense dataset (precision fp32: X and X^T): host toarray + upload of the dense matrix against upload of the
           stored entries + device scatter (Engine.dataset of the dense / the CSR matrix)
Each time is host wall clock around a call that ends in a device synchronisation; both routes run once after a small
warm-up and their results are compared.  Inputs come from a seeded generator.  Prints the card's name and power limit
with the numbers.
"""
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import scipy.sparse as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from cnmf_b200 import io as cio  # noqa: E402
from cnmf_b200.engine import Engine  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:          # the numbers are still printed; the card line says why it is missing
        return "unknown (%s)" % e


def timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return out, round(time.perf_counter() - t0, 3)


def atlas_counts(n, g, per_col, seed=0):
    """integer counts 1..5, about per_col distinct cells per gene, as CSR (float32)"""
    rng = np.random.default_rng(seed)
    lens = np.empty(g, np.int64)
    parts = []
    for c0 in range(0, g, 1000):
        rows = np.sort(rng.integers(0, n, size=(min(1000, g - c0), per_col), dtype=np.int32), axis=1)
        keep = np.ones(rows.shape, bool)
        keep[:, 1:] = rows[:, 1:] != rows[:, :-1]
        lens[c0:c0 + rows.shape[0]] = keep.sum(axis=1)
        parts.append(rows[keep])
    idx = np.concatenate(parts)
    col_ptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    vals = rng.integers(1, 6, size=idx.size).astype(np.float32)
    return sp.csc_matrix((vals, idx, col_ptr), shape=(n, g)).tocsr()


def dense_density_counts(n, g, density, seed=0, rows_per_chunk=100_000):
    """n x g CSR (float32 integers 1..5), each entry stored with probability `density`, built in row chunks"""
    rng = np.random.default_rng(seed)
    indptr = [np.zeros(1, np.int64)]
    idx, vals = [], []
    for r0 in range(0, n, rows_per_chunk):
        m = rng.random((min(rows_per_chunk, n - r0), g), dtype=np.float32) < density
        indptr.append(indptr[-1][-1] + np.cumsum(m.sum(axis=1), dtype=np.int64))
        idx.append(np.nonzero(m)[1].astype(np.int32))
        vals.append(rng.integers(1, 6, size=idx[-1].size).astype(np.float32))
        del m
    return sp.csr_matrix((np.concatenate(vals), np.concatenate(idx), np.concatenate(indptr)), shape=(n, g))


def write_legacy_10x(path, C):
    """C (cells x genes CSR) as matrix.mtx (genes x cells) / genes.tsv / barcodes.tsv"""
    import scipy.io
    n, g = C.shape
    scipy.io.mmwrite(os.path.join(path, "matrix.mtx"), C.T.tocoo())
    with open(os.path.join(path, "genes.tsv"), "w") as f:
        f.write("".join("ENSG%06d\tg%d\n" % (i, i) for i in range(g)))
    with open(os.path.join(path, "barcodes.tsv"), "w") as f:
        f.write("".join("c%d\n" % i for i in range(n)))


def probe_atlas(eng):
    n, g = 500_000, 30_000
    C, gen_s = timed(lambda: atlas_counts(n, g, 2500))
    res = {"shape": [n, g], "nnz": int(C.nnz), "generate_s": gen_s}
    with tempfile.TemporaryDirectory() as d:
        _, res["mtx_write_s"] = timed(lambda: write_legacy_10x(d, C))
        res["mtx_bytes"] = os.path.getsize(os.path.join(d, "matrix.mtx"))
        m, res["mtx_read_s"] = timed(lambda: cio.read_counts(os.path.join(d, "matrix.mtx")))
        res["mtx_read_matches"] = bool(m.X.shape == C.shape and (m.X != C).nnz == 0)
        del m
    small = C[:1000]
    eng.sparse_dataset(small).close()
    eng.sparse_dataset(small.tocsc()).close()
    csc, res["host_tocsc_s"] = timed(lambda: C.tocsc())
    a, res["csc_upload_and_build_s"] = timed(lambda: eng.sparse_dataset(csc))
    b, res["csr_upload_and_device_transpose_s"] = timed(lambda: eng.sparse_dataset(C))
    res["host_route_s"] = round(res["host_tocsc_s"] + res["csc_upload_and_build_s"], 3)
    res["device_route_s"] = res["csr_upload_and_device_transpose_s"]
    res["csc_arrays_equal"] = all(np.array_equal(a.operand(k), b.operand(k))
                                  for k in ("csc_col_ptr", "csc_row_idx", "csc_values"))
    a.close()
    b.close()
    return res


def probe_hvg(eng):
    n, g = 2_000_000, 2000
    C, gen_s = timed(lambda: dense_density_counts(n, g, 0.3))
    res = {"shape": [n, g], "nnz": int(C.nnz), "generate_s": gen_s, "precision": "fp32"}
    small = C[:1000]
    eng.dataset(small, precision="fp32").close()
    eng.dataset(small.toarray(), precision="fp32").close()
    D, res["host_toarray_s"] = timed(lambda: C.toarray())
    a, res["dense_upload_and_build_s"] = timed(lambda: eng.dataset(D, precision="fp32"))
    sums_a = a.sums()
    a.close()
    del D
    b, res["csr_upload_and_device_scatter_s"] = timed(lambda: eng.dataset(C, precision="fp32"))
    res["host_route_s"] = round(res["host_toarray_s"] + res["dense_upload_and_build_s"], 3)
    res["device_route_s"] = res["csr_upload_and_device_scatter_s"]
    res["sums_equal"] = sums_a == b.sums()
    b.close()
    return res


def main():
    probes = {"atlas": probe_atlas, "hvg": probe_hvg}
    names = [a for a in sys.argv[1:] if a in probes] or list(probes)
    eng = Engine(0)
    print("card (name, power limit):", card(), flush=True)
    for name in names:
        print(json.dumps({name: probes[name](eng)}), flush=True)


if __name__ == "__main__":
    main()
