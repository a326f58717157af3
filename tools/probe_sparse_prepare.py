#!/usr/bin/env python
"""GPU probe: prepare(on_device=True)'s stages on raw counts kept sparse (CSC) on the device and on the dense counts
dataset.

For each shape: wall clock (host; every stage ends in a host-visible result) of the counts dataset build, the TPM
totals and gene statistics (`tpm_stats` sparse, `row_sums` + `col_stats(row_scale)` dense), the HVG dataset
(`col_stats` + `from_columns`) and the writes of the TPM and normalised-counts files, with the device memory in use
after each; then `tpm_stats` alone over 10 calls as achieved GB/s of algorithmic bytes against the 3.35 TB/s HBM3
data-sheet bound of the H100 SXM.  The stages are the ones `pipeline.cNMF.prepare` runs; the HVGs are ranked by
`_highvar_from_stats` as there.

  python tools/probe_sparse_prepare.py [mid] [atlas]

  mid    50 000 x 20 000 at ~10 % density: both forms (and the rel-L2 between their statistics)
  atlas  400 000 x 30 000 at ~2 % density: sparse only (the dense counts dataset does not fit)
Inputs are integer counts from a seeded generator.  Prints the card's name and power limit with the numbers.
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
from cnmf_b200.pipeline import _highvar_from_stats, fits_dense  # noqa: E402

SHAPES = {"mid": (50_000, 20_000, 5_000), "atlas": (400_000, 30_000, 8_000)}   # cells, genes, draws per gene
N_HVG = 2000
HBM_GBS = 3350.0
SLABS = 128     # sparse_kernels.cu TPM_SLABS


def seeded_counts(n, g, per_col, seed=0):
    """Integer counts 1..5, per_col row draws per gene (duplicates dropped), built as CSC and returned as CSR (the
    form prepare reads)."""
    rng = np.random.default_rng(seed)
    lens = np.empty(g, np.int64)
    idx_parts = []
    for c0 in range(0, g, 1000):                       # blocks of genes bound the host memory of the sort
        rows = np.sort(rng.integers(0, n, size=(min(1000, g - c0), per_col), dtype=np.int32), axis=1)
        keep = np.ones(rows.shape, bool)
        keep[:, 1:] = rows[:, 1:] != rows[:, :-1]
        lens[c0:c0 + rows.shape[0]] = keep.sum(axis=1)
        idx_parts.append(rows[keep])
    idx = np.concatenate(idx_parts)
    col_ptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    vals = rng.integers(1, 6, size=idx.size).astype(np.float64)
    return sp.csc_matrix((vals, idx, col_ptr), shape=(n, g)).tocsr()


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:          # the numbers are still printed; the card line says why it is missing
        return "unknown (%s)" % e


def used_gb(eng):
    free, total, _ = eng.mem_info()
    return round((total - free) / 1e9, 2)


def tpm_stats_bytes(n, g, nnz):
    """Algorithmic bytes of one tpm_stats call: pass 1 reads every entry (8 B) and read-modify-writes its fp64 row
    partial (16 B); the fold reads the slab partials and writes totals and scale; the column pass reads every entry
    again with its row scale (16 B) and writes two fp64 sums per column; col_ptr is read twice."""
    slabs = max(1, min(SLABS, g, (1 << 25) // n))
    return 40.0 * nnz + 8.0 * slabs * n + 16.0 * n + 16.0 * g + 16.0 * (g + 1)


def stages(eng, C, sparse, out_dir):
    """prepare's on-device stages on the CSR counts C; returns (timings / memory, (totals, mean, var), HVG dataset)."""
    n, g = C.shape
    obs, var_names = ["c%d" % i for i in range(n)], ["g%d" % i for i in range(g)]
    res = {}

    def mark(name, t0):
        res[name + "_ms"] = round(1e3 * (time.perf_counter() - t0), 1)
        res[name + "_used_gb"] = used_gb(eng)

    t0 = time.perf_counter()
    ds = eng.sparse_dataset(C) if sparse else eng.dataset(C.toarray())
    mark("build", t0)
    t0 = time.perf_counter()
    if sparse:
        tot, mean, var = ds.tpm_stats()
    else:
        tot = ds.row_sums()
        mean, var = ds.col_stats(row_scale=1e6 / tot)
    mark("tpm_stats", t0)
    t0 = time.perf_counter()
    hv = np.where(_highvar_from_stats(mean, var, N_HVG))[0]
    _, c_var = ds.col_stats()
    std1 = np.sqrt(c_var[hv] * n / (n - 1.0))
    std1[std1 == 0] = 1.0
    hvg_ds = ds.from_columns(hv, 1.0 / std1)
    mark("hvg_dataset", t0)
    if sparse:
        reps = 10
        t0 = time.perf_counter()
        for _ in range(reps):
            ds.tpm_stats()
        ms = 1e3 * (time.perf_counter() - t0) / reps
        gb = tpm_stats_bytes(n, g, C.nnz) / 1e9
        res["tpm_stats_alone"] = {"ms_per_call": round(ms, 2), "algorithmic_gb": round(gb, 2),
                                  "achieved_gbs": round(gb / ms * 1e3, 1),
                                  "share_of_hbm_bound": round(gb / ms * 1e3 / HBM_GBS, 3)}
    ds.close()
    t0 = time.perf_counter()
    T = C.copy()
    T.data /= np.repeat(tot, np.diff(C.indptr))
    T.data *= 1e6
    cio.write_matrix(os.path.join(out_dir, "tpm.h5ad"), cio.CellGeneMatrix(T, obs, var_names))
    del T
    X = C[:, hv].astype(np.float64)
    X.sort_indices()
    X.data /= std1[X.indices]
    cio.write_matrix(os.path.join(out_dir, "norm.h5ad"), cio.CellGeneMatrix(X, obs, [var_names[i] for i in hv]))
    mark("file_writes", t0)
    return res, (tot, mean, var), hvg_ds


def probe(eng, name, out_dir):
    n, g, per_col = SHAPES[name]
    t0 = time.perf_counter()
    C = seeded_counts(n, g, per_col)
    res = {"shape": [n, g], "nnz": int(C.nnz), "density": round(C.nnz / (n * g), 4),
           "generate_s": round(time.perf_counter() - t0, 1),
           "dense_peak_gb": round(eng.dense_dataset_bytes(n, g) / 1e9, 1)}
    res["sparse"], st_s, hvg_s = stages(eng, C, True, out_dir)
    s_sums = hvg_s.sums()
    hvg_s.close()
    if fits_dense(eng, (n, g), "f16x2"):
        res["dense"], st_d, hvg_d = stages(eng, C, False, out_dir)
        res["sparse_vs_dense_rel"] = {k: float(np.linalg.norm(a - b) / np.linalg.norm(b))
                                      for k, a, b in zip(("totals", "mean", "var"), st_s, st_d)}
        res["hvg_dataset_sums_equal"] = s_sums == hvg_d.sums()
        hvg_d.close()
    else:
        res["dense"] = "skipped: the dense counts dataset does not fit"
    return res


def main():
    names = [a for a in sys.argv[1:] if a in SHAPES] or list(SHAPES)
    eng = Engine(0)
    print("card (name, power limit):", card())
    with tempfile.TemporaryDirectory() as out_dir:
        for name in names:
            print(json.dumps({name: probe(eng, name, out_dir)}), flush=True)


if __name__ == "__main__":
    main()
