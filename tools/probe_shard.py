"""One rank's share of the c3 job table (idx % WORLD == 0) on ONE GPU: where the time of a small shard goes.

The strong-scaling loss from 1 to N GPUs is the part of a solve that does not shrink with the number of restarts; this
probe times the shard alone (wall, CUDA events, per-class kernel time) so that `wall - GEMM - update` can be read off.
usage: python tools/probe_shard.py [world=8] [reps=3]      env: SHARD_RANKS=0,1,.. (default 0), PROFILE=0 (no per-launch events)"""
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    import torch
    import bench
    from cnmf_b200.engine import Engine
    from cnmf_b200.parallel import shard_jobs
    world = int(sys.argv[1]) if len(sys.argv) > 1 else 8
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    X, _, _ = bench.make_data("c3")
    ks_all, seeds_all, _ = bench.job_table("c3", 1, "strong")
    eng = Engine(0)
    ds = eng.dataset(X)
    _, ld = ds.ld()
    ranks = [int(r) for r in os.environ.get("SHARD_RANKS", "0").split(",")]
    prof = os.environ.get("PROFILE", "1") != "0"
    cases = [(world, r) for r in ranks] + ([(1, 0)] if os.environ.get("SHARD_RANKS") is None else [])
    for w, rk in cases:
        jobs = shard_jobs(len(ks_all), rk, w)
        ks = [ks_all[j] for j in jobs]
        seeds = [seeds_all[j] for j in jobs]
        slab = torch.zeros((sum(ks), ld), dtype=torch.float32, device="cuda:0")
        for _ in range(2 if reps > 1 else 1):
            ds.factorize_seeds_dev(ks, seeds, slab.data_ptr(), ld, bench.NMF_KW)
        torch.cuda.synchronize()
        eng.profile(prof)
        l0 = eng.launch_count
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        e0.record()
        for _ in range(reps):
            n_iter, _ = ds.factorize_seeds_dev(ks, seeds, slab.data_ptr(), ld, bench.NMF_KW)
        e1.record()
        torch.cuda.synchronize()
        wall = 1e3 * (time.perf_counter() - t0) / reps
        dev = e0.elapsed_time(e1) / reps
        g_ms, g_n, _ = eng.profile_get(0)
        u_ms, u_n, _ = eng.profile_get(1)
        eng.profile(False)
        print(json.dumps({"world": w, "rank": rk, "profile": prof, "restarts": len(jobs), "rows": int(sum(ks)), "wall_ms": round(wall, 2),
                          "device_ms": round(dev, 2), "gemm_ms": round(g_ms / reps, 2), "gemm_launches": g_n // reps,
                          "update_ms": round(u_ms / reps, 2), "update_launches": u_n // reps,
                          "other_ms": round(dev - (g_ms + u_ms) / reps, 2),
                          "launches": (eng.launch_count - l0) // reps, "n_iter_mean": float(np.mean(n_iter)),
                          "n_iter_max": int(np.max(n_iter))}), flush=True)


if __name__ == "__main__":
    main()
