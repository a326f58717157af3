#!/usr/bin/env python
"""GPU probe: the consensus step's TPM stages on a dense and on a sparse (CSC) TPM dataset.

For each shape: wall clock (host, every stage ends in a host-visible result) of the TPM dataset build, refit_spectra
(transposed refit), the OLS z-score products (col_stats + project_rows) and the HVG refit (from_columns + refit), with
the device memory in use after each; then the sparse product kernels alone (CUDA events, profile class 2) as achieved
GB/s of algorithmic bytes against the 3.35 TB/s HBM3 data-sheet bound of the H100 SXM.

  python tools/probe_sparse_consensus.py [mid] [atlas]

  mid    50 000 x 20 000 at ~10 % density: both forms fit
  atlas  400 000 x 30 000 at ~2 % density: only the sparse form fits (the dense one is reported as skipped)
Inputs come from a seeded generator.  Prints the card's name and power limit with the numbers.
"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import scipy.sparse as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from cnmf_b200.engine import Engine  # noqa: E402
from cnmf_b200.pipeline import TPM_DENSE_FRACTION  # noqa: E402

SHAPES = {"mid": (50_000, 20_000, 5_000), "atlas": (400_000, 30_000, 8_000)}   # cells, genes, draws per gene
K = 10
KW = dict(solver="cd", beta_loss="frobenius", tol=1e-4, max_iter=200)
HBM_GBS = 3350.0


def seeded_tpm(n, g, per_col, seed=0):
    """TPM-like CSC: per_col row draws per gene (duplicates dropped), counts 1..5 scaled by 1e6 / cell total."""
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
    counts = rng.integers(1, 6, size=idx.size).astype(np.float32)
    tot = np.bincount(idx, weights=counts, minlength=n)
    tot[tot == 0] = 1.0
    vals = counts * (1e6 / tot).astype(np.float32)[idx]
    return sp.csc_matrix((vals, idx, col_ptr), shape=(n, g))


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


def stages(eng, T, make):
    """Time the TPM stages on the dataset make() builds; returns a dict of ms and GB in use after each."""
    n, g = T.shape
    rng = np.random.RandomState(1)
    W = (np.abs(rng.randn(n, K)) + 0.05).astype(np.float32)
    out = {}

    def mark(name, t0):
        out[name + "_ms"] = round(1e3 * (time.perf_counter() - t0), 1)
        out[name + "_used_gb"] = used_gb(eng)

    t0 = time.perf_counter()
    ds = make()
    mark("build", t0)
    t0 = time.perf_counter()
    Ht, it, _ = ds.refit(np.ascontiguousarray(W.T), KW, transposed=True)
    mark("refit_spectra", t0)
    out["refit_spectra_iters"] = it
    t0 = time.perf_counter()
    mean, var = ds.col_stats()
    Uc = (W - W.mean(axis=0)).astype(np.float32)
    P = ds.project_rows(np.ascontiguousarray(Uc.T))
    mark("ols", t0)
    t0 = time.perf_counter()
    hvg = np.argsort(-var / np.maximum(mean, 1e-12))[:2000]
    std1 = np.sqrt(var[hvg] * n / (n - 1.0))
    sub = ds.from_columns(hvg, 1.0 / std1)
    rf, it_c, _ = sub.refit(np.abs(Ht.T[:, hvg]) / std1 + 1e-3, KW)
    sub.close()
    mark("hvg_refit", t0)
    out["hvg_refit_iters"] = it_c
    out["_results"] = (Ht, P, rf)
    return ds, out


def probe(eng, name):
    n, g, per_col = SHAPES[name]
    t0 = time.perf_counter()
    T = seeded_tpm(n, g, per_col)
    res = {"shape": [n, g], "nnz": int(T.nnz), "density": round(T.nnz / (n * g), 4),
           "generate_s": round(time.perf_counter() - t0, 1)}
    free, _, cached = eng.mem_info()
    peak = eng.dense_dataset_bytes(n, g)
    res["dense_peak_gb"] = round(peak / 1e9, 1)
    res["dense_budget_gb"] = round(TPM_DENSE_FRACTION * (free + cached) / 1e9, 1)
    sds, res["sparse"] = stages(eng, T, lambda: eng.sparse_dataset(T))
    # the sparse product kernels alone: k = K products of the staged usages, CUDA events around both kernels
    Ut = np.ascontiguousarray(np.random.RandomState(2).randn(K, n).astype(np.float32))
    sds.project_rows(Ut)
    eng.profile(True)
    for _ in range(10):
        sds.project_rows(Ut)
    ms, launches, work = eng.profile_get(2)
    eng.profile(False)
    gbs = work / (ms * 1e6)
    res["csc_project"] = {"k": K, "ms_per_call": round(ms / launches, 3), "algorithmic_gb": round(work / launches / 1e9, 3),
                          "achieved_gbs": round(gbs, 1), "share_of_hbm_bound": round(gbs / HBM_GBS, 3)}
    sds.close()
    if peak <= TPM_DENSE_FRACTION * (free + cached):
        Td = T.toarray()
        dds, res["dense"] = stages(eng, T, lambda: eng.dataset(Td))
        dds.close()
        del Td
        a, b = res["sparse"].pop("_results"), res["dense"].pop("_results")
        res["sparse_vs_dense_rel"] = [float(np.linalg.norm(x - y) / np.linalg.norm(y)) for x, y in zip(a, b)]
    else:
        res["sparse"].pop("_results")
        res["dense"] = "skipped: the dense dataset does not fit"
    return res


def main():
    names = [a for a in sys.argv[1:] if a in SHAPES] or list(SHAPES)
    eng = Engine(0)
    print("card (name, power limit):", card())
    for name in names:
        print(json.dumps({name: probe(eng, name)}), flush=True)


if __name__ == "__main__":
    main()
