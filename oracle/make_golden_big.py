#!/usr/bin/env python
"""Generate tests/golden/big_samples.npz: the reference's own NMF call on SAMPLED restarts of the
BASELINE.json configurations whose full run would take hours on the host.

    python -m oracle.make_golden_big [case ...]        # from the repo root (scikit-learn only)

Test infrastructure (see oracle/__init__.py).  What the reference executes per (k, seed) job is one
`sklearn.decomposition.non_negative_factorization(X, **kwargs)` (cnmf.py:661-674, called at cnmf.py:741
with the kwargs of cnmf.py:618-631) on the float64 normalised counts (cnmf.py:534-542);
`oracle/reference_path.factorize` issues exactly that call.  Inputs are the deterministic synthetic
matrices of SURVEY.md section 8d (cnmf_b200.synth, seeds of cnmf.py:597-610), so only the OUTPUTS are
stored: per sample `H_<name>` (k x G, the reference's float64 result rounded to float32: 6e-8 relative, far
inside the 1e-4 tolerance, and it keeps the file under 1 MB), `it_<name>` (n_iter) and `meta_<name>` =
[n_cells, n_genes, k, iter index, seed, solver is cd].

Cases (name: shape, K-list of the job table, sampled (k, iter) jobs, solver)
  c2     BASELINE configs[1]  20 000 x 2 000, K=10 x100           iters 0,1,2      mu   (+ iter 3 with cd)
  c3     BASELINE configs[2]  50 000 x 2 000, K=5..13 x100        (5,0) (9,0) (13,0)  mu
  k20    configs[3]-shaped     4 000 x 2 000, K=20 (kp = 32 path)  iter 0           mu and cd
  k30    configs[4]-shaped     2 000 x 1 000, K=30 (kp = 32 path)  iter 0           mu and cd
"""
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from cnmf_b200.synth import make_counts, normalise, restart_table  # noqa: E402
from oracle import reference_path  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "big_samples.npz")

# name: (n_cells, n_genes, k_true, libsize, ks, n_iter, [(k, iter, solver), ...])
CASES = {
    "c2": (20000, 2000, 12, 1500.0, [10], 100, [(10, 0, "mu"), (10, 1, "mu"), (10, 2, "mu"), (10, 3, "cd")]),
    "c3": (50000, 2000, 12, 1500.0, list(range(5, 14)), 100, [(5, 0, "mu"), (9, 0, "mu"), (13, 0, "mu")]),
    "k20": (4000, 2000, 12, 1500.0, [20], 200, [(20, 0, "mu"), (20, 0, "cd")]),
    "k30": (2000, 1000, 12, 1500.0, [30], 200, [(30, 0, "mu"), (30, 0, "cd")]),
}


def case_inputs(name):
    """(X float64, job table) of a case -- also imported by tests/test_gpu_parity.py so both sides build
    the identical matrix."""
    n_cells, n_genes, k_true, libsize, ks, n_iter, _ = CASES[name]
    X, _ = normalise(make_counts(n_cells, n_genes, k_true=k_true, seed=0, libsize=libsize), np.float64)
    return X, restart_table(ks, n_iter, seed=14)


def main():
    want = sys.argv[1:] or list(CASES)
    out = dict(np.load(OUT)) if os.path.exists(OUT) else {}
    for name in want:
        X, table = case_inputs(name)
        lookup = {(k, it): seed for k, it, seed in table}
        for k, it, solver in CASES[name][6]:
            tag = "%s_k%d_i%d_%s" % (name, k, it, solver)
            seed = lookup[(k, it)]
            t0 = time.perf_counter()
            H, n_it, _ = reference_path.factorize(X, [(k, seed)], solver)
            out["H_" + tag] = H[0].astype(np.float32)
            out["it_" + tag] = np.int64(n_it[0])
            out["meta_" + tag] = np.array([X.shape[0], X.shape[1], k, it, seed, int(solver == "cd")], dtype=np.int64)
            print(tag, "n_iter", n_it[0], "%.1f s" % (time.perf_counter() - t0), flush=True)
            np.savez_compressed(OUT, **out)


if __name__ == "__main__":
    main()
