#!/usr/bin/env python
"""GPU probe: a multi-tile, mixed-K batch against the numpy oracle, for whichever kernel variant the environment
selects (CNMF_FUSE_W, CNMF_UPD_VARIANT)."""
import json, os, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from cnmf_b200.engine import Engine
from cnmf_b200.synth import make_counts, normalise, restart_table
from oracle import nmf_ref

n_cells = int(os.environ.get("PROBE_CELLS", "1000"))
n_rep = int(os.environ.get("PROBE_REPS", "5"))
X, _ = normalise(make_counts(n_cells, 500, k_true=7, seed=0, libsize=800.0), np.float64)
rows = restart_table(list(range(5, 14)), n_rep, seed=14)
eng = Engine(0)
ds = eng.dataset(X)
kw = dict(solver="mu", beta_loss=2.0, tol=1e-4, max_iter=400)
t0 = time.perf_counter()
sp, _, n_iter, err = ds.factorize([r[0] for r in rows], [r[2] for r in rows], kw)
dt = time.perf_counter() - t0
out = {"fuse": os.environ.get("CNMF_FUSE_W", "0"), "variant": os.environ.get("CNMF_UPD_VARIANT", ""), "SK": int(sum(r[0] for r in rows)), "sec": round(dt, 3), "n_iter": [int(x) for x in n_iter]}
worst, bad = 0.0, []
for i in range(0, len(rows), 4):
    k, _, seed = rows[i]
    W, H, it = nmf_ref.nmf(X, k, seed, solver="mu", max_iter=400)
    e = float(np.linalg.norm(sp[i] - H) / np.linalg.norm(H))
    worst = max(worst, e)
    if it != int(n_iter[i]) or e > 1e-4:
        bad.append((i, k, it, int(n_iter[i]), e))
out["worst_rel"] = worst
out["bad"] = bad
print(json.dumps(out))
