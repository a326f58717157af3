"""precision='fp64' on BASELINE c3's shape (50 000 x 2 000, K = 5..13 x 100 restarts) against 'f16x2' on the same card:
restarts/s of the whole batched factorize (host clock around the call, which ends in a device synchronise), the share
of the float64 solver's fp64 GEMM (profiling class 4) in a separate profiled run with its algorithmic TFLOP/s, and the
device memory in use.  The two precisions are run alternately, --reps times each, per solver.

    python tools/probe_fp64.py [--restarts-per-k 100] [--reps 2] [--solvers cd,mu] [--out probe_fp64.json]

Prints one JSON line; --out also writes it to a file.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

FP64_TC_PEAK = 67e12        # NVIDIA H100 SXM data sheet, FP64 tensor core, dense


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=60).stdout
        name, power, clock, cur = [x.strip() for x in out.strip().splitlines()[0].split(",")]
        return dict(gpu=name, power_limit=power, max_sm_clock=clock, sm_clock_at_start=cur)
    except Exception as e:          # the measurement itself still needs the GPU below
        return dict(gpu="unknown (%s)" % e)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--restarts-per-k", type=int, default=100)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--solvers", default="cd,mu")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    from cnmf_b200.engine import Engine
    from cnmf_b200.synth import make_counts, normalise, restart_table

    X, _ = normalise(make_counts(50000, 2000, k_true=12, seed=0, libsize=1500.0), np.float64)
    rows = restart_table(range(5, 14), a.restarts_per_k, seed=14)
    ks = np.array([r[0] for r in rows], np.int32)
    seeds = np.array([r[2] for r in rows], np.uint32)
    eng = Engine(0)
    ds = {"f16x2": eng.dataset(X, precision="f16x2"), "fp64": eng.dataset(X, precision="fp64")}
    n, g = X.shape
    out = dict(gpu_info(), shape=[n, g], restarts=len(ks), sum_k=int(ks.sum()), runs={})
    for solver in a.solvers.split(","):
        kw = dict(solver=solver, tol=1e-4, max_iter=1000, beta_loss=2.0 if solver == "mu" else "frobenius")
        for prec, d in ds.items():                               # warm-up: every kernel and workspace of the shape
            d.factorize(ks[:3], seeds[:3], dict(kw, max_iter=20))
        res = {p: [] for p in ds}
        n_iter = {}
        for _ in range(a.reps):
            for prec, d in ds.items():                           # alternated: f16x2, fp64, f16x2, fp64, ...
                t0 = time.perf_counter()
                _, _, it, _ = d.factorize(ks, seeds, kw)
                res[prec].append(time.perf_counter() - t0)
                n_iter[prec] = int(np.sum(it))
        free, total, cached = eng.mem_info()
        eng.profile(True)                                        # separate profiled fp64 run: class 4 = its GEMM
        t0 = time.perf_counter()
        ds["fp64"].factorize(ks, seeds, kw)
        prof_s = time.perf_counter() - t0
        gemm_ms, gemm_launches, gemm_flops = eng.profile_get(4)
        upd_ms, _, _ = eng.profile_get(1)
        eng.profile(False)
        out["runs"][solver] = dict(
            seconds={p: [round(x, 3) for x in v] for p, v in res.items()},
            restarts_per_s={p: round(len(ks) / float(np.median(v)), 2) for p, v in res.items()},
            total_iterations=n_iter,
            fp64_profiled_s=round(prof_s, 3), fp64_gemm_ms=round(gemm_ms, 1), fp64_gemm_launches=gemm_launches,
            fp64_gemm_share_of_solve=round(gemm_ms / 1e3 / prof_s, 3),
            fp64_update_ms=round(upd_ms, 1),
            fp64_gemm_tflops=round(gemm_flops / (gemm_ms / 1e3) / 1e12, 2) if gemm_ms > 0 else None,
            fp64_gemm_share_of_datasheet=round(gemm_flops / (gemm_ms / 1e3) / FP64_TC_PEAK, 3) if gemm_ms > 0 else None,
            device_bytes_in_use=int(total - free), engine_cached_bytes=int(cached))
    out.update({"sm_clock_at_end": gpu_info().get("sm_clock_at_start")})
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
