"""Time the variance scaling with a quantile ceiling (cnmf_scale_quantile_ceiling) at atlas size: 200 000 cells x
2 000 genes, float32, quantile 0.9999 (what stdscale_quantile_celing runs).

    python tools/probe_scale.py [--cells 200000] [--genes 2000] [--reps 5] [--out FILE]

Two timings, each the median of --reps calls after one warm-up call, host wall clock around the synchronising call:
  host_s    host matrix in and out (scale_quantile_ceiling, pageable copies included);
  device_s  device-resident matrix in and out (torch tensors through the C ABI): staging copy, moments, std, scaling,
            the radix select's histogram passes and the ceiling.
Prints one JSON line with the GPU's name, power limit and maximum SM clock; with --out, writes it there too.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from cnmf_b200 import _lib  # noqa: E402
from cnmf_b200.preprocess import _engine, quantile_ranks, scale_quantile_ceiling  # noqa: E402


def timed(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)), ts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cells", type=int, default=200000)
    ap.add_argument("--genes", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", type=str, default=None)
    a = ap.parse_args()
    import torch
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    rng = np.random.RandomState(0)
    X = (rng.gamma(0.6, 1.5, size=(a.cells, a.genes)) * (rng.rand(a.cells, a.genes) < 0.3)).astype(np.float32)
    eng = _engine()
    host_s, host_all = timed(lambda: scale_quantile_ceiling(X, quantile_thresh=0.9999), a.reps)

    Xd = torch.from_numpy(X).cuda()
    Od = torch.empty_like(Xd)
    k_lo, k_hi, gamma = quantile_ranks(X.size, 0.9999, X.dtype)
    thresh = ctypes.c_double()
    torch.cuda.synchronize()

    def device_call():
        _lib.check(eng.lib.cnmf_scale_quantile_ceiling(
            eng._h, ctypes.c_void_p(Xd.data_ptr()), 0, a.cells, a.genes, a.genes, 1, None, None, 0, 0.0, 0, k_lo, k_hi,
            gamma, ctypes.c_void_p(Od.data_ptr()), a.genes, 1, ctypes.byref(thresh), None))

    device_s, device_all = timed(device_call, a.reps)
    host_out, host_t, _ = scale_quantile_ceiling(X, quantile_thresh=0.9999)
    same = bool(np.array_equal(Od.cpu().numpy(), host_out)) and float(host_t) == thresh.value
    res = dict(probe="scale_quantile_ceiling", gpu=gpu, cells=a.cells, genes=a.genes, dtype="float32",
               quantile=0.9999, host_s=host_s, host_s_all=host_all, device_s=device_s, device_s_all=device_all,
               threshold=thresh.value, device_equals_host=same)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
