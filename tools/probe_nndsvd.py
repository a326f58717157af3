"""Where the time of `--init nndsvd` goes on BASELINE c3's shape (50 000 x 2 000, K = 5..13 x 100 restarts):
the device starts (cnmf_nndsvd_init_dev, CUDA events after a warm-up), the share of its fp64 GEMM and that GEMM's
algorithmic rate, the work-space bytes, and the host restatement (cnmf_b200.nndsvd, what `X_host=` runs) on a sample
of restarts, extrapolated, with the starts' deviation between the two.

    python tools/probe_nndsvd.py [--restarts-per-k 100] [--host-sample 3] [--out probe_nndsvd.json]

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
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in out.split(",")]
        return dict(gpu=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:          # the measurement itself still needs the GPU below
        return dict(gpu="unknown (%s)" % e)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--restarts-per-k", type=int, default=100)
    ap.add_argument("--host-sample", type=int, default=3)
    ap.add_argument("--init", default="nndsvd")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    import torch
    from cnmf_b200.engine import Engine
    from cnmf_b200.nndsvd import nndsvd_init
    from cnmf_b200.synth import make_counts, normalise, restart_table

    X, _ = normalise(make_counts(50000, 2000, k_true=12, seed=3), np.float32)
    rows = restart_table(range(5, 14), a.restarts_per_k, seed=14)
    ks = np.array([r[0] for r in rows], np.int32)
    seeds = np.array([r[2] for r in rows], np.uint32)
    eng = Engine(0)
    ds = eng.dataset(X)
    n, g = ds.shape
    ld_r, ld_c = ds.ld()
    SK = int(ks.sum())
    Wt = torch.empty((SK, ld_r), dtype=torch.float32, device="cuda:0")
    H = torch.empty((SK, ld_c), dtype=torch.float32, device="cuda:0")

    warm = [0, a.restarts_per_k * 4, len(ks) - 1]            # K = 5, 9, 13: both power-iteration classes
    ds.nndsvd_init_dev(ks[warm], seeds[warm], a.init, Wt.data_ptr(), H.data_ptr())
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    ds.nndsvd_init_dev(ks, seeds, a.init, Wt.data_ptr(), H.data_ptr())
    ev1.record()
    torch.cuda.synchronize()
    dev_ms = ev0.elapsed_time(ev1)
    eng.profile(True)
    ds.nndsvd_init_dev(ks, seeds, a.init, Wt.data_ptr(), H.data_ptr())
    gemm_ms, gemm_launches, gemm_flops = eng.profile_get(3)
    eng.profile(False)
    sum_p = int(np.minimum(ks + 10, min(n, g)).sum())
    n_iter = np.where(ks < 0.1 * min(n, g), 7, 4)
    algo_flops = float((2.0 * n * g * np.minimum(ks + 10, min(n, g)) * (2 * n_iter + 2)).sum())

    # host restatement on a sample, same matrix (float64 of the fp32 X), starts compared
    X64 = X.astype(np.float64)
    Wh = Wt.cpu().numpy()
    Hh = H.cpu().numpy()
    offs = np.concatenate([[0], np.cumsum(ks)])
    sample = sorted(set(np.linspace(0, len(ks) - 1, a.host_sample).astype(int).tolist()))
    host_s, dev_w, dev_h = {}, [], []
    for r in sample:
        k = int(ks[r])
        t0 = time.perf_counter()
        W0, H0 = nndsvd_init(X64, k, int(seeds[r]), a.init)
        host_s.setdefault(k, []).append(time.perf_counter() - t0)
        Wd = Wh[offs[r]:offs[r + 1], :n].T.astype(np.float64)
        Hd = Hh[offs[r]:offs[r + 1], :g].astype(np.float64)
        dev_w.append(float(np.linalg.norm(Wd - W0) / np.linalg.norm(W0)))
        dev_h.append(float(np.linalg.norm(Hd - H0) / np.linalg.norm(H0)))
    per_k = {k: float(np.mean(v)) for k, v in host_s.items()}
    ks_known = np.array(sorted(per_k))
    host_total = float(sum(np.interp(k, ks_known, [per_k[x] for x in ks_known]) for k in ks))

    out = dict(gpu_info(), shape=[n, g], restarts=len(ks), init=a.init, sum_p=sum_p,
               device_init_ms=round(dev_ms, 2), restarts_per_s=round(len(ks) / (dev_ms / 1e3), 1),
               fp64_gemm_ms=round(gemm_ms, 2), fp64_gemm_launches=gemm_launches,
               fp64_gemm_tflops=round(gemm_flops / (gemm_ms / 1e3) / 1e12, 2) if gemm_ms > 0 else None,
               fp64_gemm_share_of_datasheet=round(gemm_flops / (gemm_ms / 1e3) / FP64_TC_PEAK, 3) if gemm_ms > 0 else None,
               algorithmic_flops=algo_flops, workspace_bytes=8 * sum_p * (ld_r + ld_c),
               host_cores=os.cpu_count(), host_s_per_restart=per_k, host_extrapolated_s=round(host_total, 1),
               host_sample=[int(ks[r]) for r in sample], rel_dev_W=dev_w, rel_dev_H=dev_h)
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
