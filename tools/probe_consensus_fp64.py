#!/usr/bin/env python
"""GPU probe: cost of the float64 consensus kernels (precision='fp64') against the float ones, per phase.

  * c3's K = 5..13 sweep: R = 100 K stacked spectra x G = 2000, consensus_numerics on the c3 normalised counts (refit
    of the usages included), float32 matrix + f16x2 dataset against float64 matrix + fp64 dataset, alternated.
  * a c5-sized R = 6000 x G = 5000, K = 30 case: L2 + distances + density, and KMeans, alternated; then one
    torch.profiler pass per type for the distance and density kernels alone (fp64 FLOP/s from 3 R^2 G / 2 FLOPs).
The spectra are planted clusters (K centres, 100 noisy replicates each), so no factorize run is needed.  Prints JSON
lines; the card name and power limit come from the same run.
"""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import bench  # noqa: E402
from cnmf_b200 import consensus as cs  # noqa: E402
from cnmf_b200.engine import Engine  # noqa: E402

TYPES = {"fp32": (np.float32, "f16x2"), "fp64": (np.float64, "fp64")}


def planted(k, reps, G, seed):
    rng = np.random.RandomState(seed)
    cen = rng.gamma(0.5, 1.0, size=(k, G)) + 1e-4
    return np.vstack([c * np.abs(1.0 + 0.1 * rng.randn(reps, G)) for c in cen])


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().split("\n")[0]
    return q


def sweep_c3(eng, reps=3):
    X, _, _ = bench.make_data("c3")
    ds = {t: eng.dataset(X, precision=p) for t, (_, p) in TYPES.items()}
    for k in bench.WORKLOADS["c3"]["ks"]:
        merged = planted(k, 100, X.shape[1], seed=k)
        res = {t: [] for t in TYPES}
        for rep in range(reps + 1):                          # rep 0 warms every shape up
            for t in TYPES:
                cs.STATS.clear()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                cs.consensus_numerics(eng, merged, k, ds[t], bench.NMF_KW)
                torch.cuda.synchronize()
                tot = 1e3 * (time.perf_counter() - t0)
                if rep:
                    res[t].append(dict(cs.STATS["phases_ms"], total=tot))
        out = {"case": "c3", "k": k, "R": merged.shape[0], "G": merged.shape[1]}
        for t in TYPES:
            out[t] = {p: round(float(np.median([r[p] for r in res[t]])), 2) for p in res[t][0]}
        print(json.dumps(out), flush=True)
    for d in ds.values():
        d.close()


def kernel_ms(fn, names, n=3):
    """Mean device time per call of the kernels whose name contains one of `names` (torch.profiler, its own pass)."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
    out = {nm: 0.0 for nm in names}
    for ev in prof.key_averages():
        for nm in names:
            if nm in ev.key:
                out[nm] += ev.device_time_total / 1e3 / n
    return out


def c5_case(eng, reps=3):
    R, G, k = 6000, 5000, 30
    merged = planted(k, R // k, G, seed=5)
    n_nb = int(0.3 * R / k)
    res = {t: {"l2_dist_density_ms": [], "kmeans_ms": []} for t in TYPES}
    for rep in range(reps + 1):
        for t, (dt, _) in TYPES.items():
            S = cs.SpectraMatrix(eng, merged, dtype=dt)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            S.l2_normalize()
            S.local_density(n_nb)
            t1 = time.perf_counter()
            cs.kmeans(S, k)
            torch.cuda.synchronize()
            t2 = time.perf_counter()
            if rep:
                res[t]["l2_dist_density_ms"].append(1e3 * (t1 - t0))
                res[t]["kmeans_ms"].append(1e3 * (t2 - t1))
    out = {"case": "c5-size", "R": R, "G": G, "k": k}
    flops = 3.0 * R * R * G / 2
    for t, (dt, _) in TYPES.items():
        S = cs.SpectraMatrix(eng, merged, dtype=dt).l2_normalize()
        km = kernel_ms(lambda: S.local_density(n_nb), ["pair_dist_kernel", "knn_density_kernel"])
        out[t] = {p: round(float(np.median(v)), 2) for p, v in res[t].items()}
        out[t].update(dist_kernel_ms=round(km["pair_dist_kernel"], 3), density_kernel_ms=round(km["knn_density_kernel"], 3),
                      dist_tflops=round(flops / (km["pair_dist_kernel"] * 1e-3) / 1e12, 2))
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    print(json.dumps({"card": card()}), flush=True)
    eng = Engine(0)
    sweep_c3(eng)
    c5_case(eng)
    print(json.dumps({"card": card()}), flush=True)
