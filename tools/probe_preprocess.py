"""Time Harmony's ridge correction on the GPU (cnmf_b200.preprocess.moe_correct_cells) against the reference's numpy
loop (preprocess.py:9-18), at atlas size: 200 000 cells x 2 000 genes, K = 100 clusters, B + 1 = 3 and 11.

    python tools/probe_preprocess.py [--cells 200000] [--genes 2000] [--clusters 100] [--ref-clusters 3]

The numpy loop costs the same for every cluster, so it is timed over --ref-clusters clusters and scaled to K (the
JSON says so).  GPU times are host wall clock around the synchronising calls after one warm-up call, median of
--reps, and include the host <-> device copies of X, R and Phi.  Prints one JSON line; with --out, writes it there too.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from cnmf_b200.preprocess import _engine, moe_correct_cells  # noqa: E402


def inputs(n, g, k, b1, seed=0):
    rng = np.random.RandomState(seed)
    X = (rng.gamma(0.6, 1.5, size=(n, g)) * (rng.rand(n, g) < 0.3)).astype(np.float32)
    lab = rng.randint(0, b1 - 1, size=n)
    Phi = np.vstack([np.ones(n)] + [(lab == j).astype(np.float64) for j in range(b1 - 1)])
    logits = rng.normal(scale=2.0, size=(k, n))
    R = np.exp(logits - logits.max(0))
    R /= R.sum(0)
    lamb = np.diag(np.concatenate([[0.0], np.ones(b1 - 1)]))
    return X, R, Phi, lamb


def numpy_loop(Z_orig, R, Phi_moe, lamb, clusters):
    Z_corr = Z_orig.copy()
    for i in range(clusters):
        Phi_Rk = np.multiply(Phi_moe, R[i, :])
        W = np.dot(np.dot(np.linalg.inv(np.dot(Phi_Rk, Phi_moe.T) + lamb), Phi_Rk), Z_orig.T)
        W[0, :] = 0
        Z_corr -= np.dot(W.T, Phi_Rk)
    return Z_corr


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cells", type=int, default=200000)
    ap.add_argument("--genes", type=int, default=2000)
    ap.add_argument("--clusters", type=int, default=100)
    ap.add_argument("--ref-clusters", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", type=str, default=None)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    eng = _engine()
    rows = []
    for b1 in (3, 11):
        X, R, Phi, lamb = inputs(a.cells, a.genes, a.clusters, b1)
        moe_correct_cells(X, R, Phi, lamb, clamp_zero=True)
        ts = []
        eng.profile(True)
        for _ in range(a.reps):
            t0 = time.perf_counter()
            moe_correct_cells(X, R, Phi, lamb, clamp_zero=True)
            ts.append(time.perf_counter() - t0)
        gemm_ms, gemm_n, gemm_flops = eng.profile_get(5)
        eng.profile(False)
        t0 = time.perf_counter()
        numpy_loop(X.T, R, Phi, lamb, a.ref_clusters)
        t_ref = (time.perf_counter() - t0) * a.clusters / a.ref_clusters
        rows.append(dict(b1=b1, gpu_s=float(np.median(ts)), gpu_s_all=ts, gemm_ms_per_call=gemm_ms / a.reps,
                         gemm_tflops=gemm_flops / (gemm_ms * 1e-3) / 1e12 if gemm_ms else None,
                         numpy_s_scaled=t_ref, numpy_clusters_timed=a.ref_clusters,
                         speedup=t_ref / float(np.median(ts))))
    res = dict(probe="preprocess_moe", gpu=gpu, cells=a.cells, genes=a.genes, clusters=a.clusters, rows=rows)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
