#!/usr/bin/env python
"""Generate tests/golden/preprocess_moe.npz by running the UNMODIFIED reference src/cnmf/preprocess.py of a dylkot/cNMF
checkout on seeded inputs.

    CNMF_REFERENCE=<cNMF checkout> python -m oracle.make_golden_preprocess      # from the repo root

preprocess.py imports scanpy, matplotlib and sklearn at module level and harmonypy inside harmony_correct_X.  The
stand-ins of oracle/refshim.py cover scanpy and matplotlib; sc.pp.scale is extended here to dense X and max_value
(scanpy's zero_center=False semantics: per gene std with ddof = 1 from float64 moments, a zero std counts as 1, X
divided by it in float64 and stored in X's type, then clipped at max_value).  harmonypy is a stand-in whose
run_harmony returns the seeded Harmony result of the case being generated, in the layout the case names.

Cases (CASES): harmony variables 1 or 2, K 1 or 20, float32 or float64 X, old (cells as columns) or new
(cells as rows) harmonypy layout.  The inputs are regenerated from their seeds (make_case, make_scale_input) rather
than stored: the fixture keeps their digest (inputs_digest) so that a changed generator is caught.  Per case <c>: the
reference outputs X_corr (Preprocess.harmony_correct_X), the digest of its X_pca_harmony, and Z_corr_ridge / W /
Phi_Rk (moe_correct_ridge on X.T) with the per-cell norms Z_cos = Z_corr_ridge / Z_cos_norms was divided by.  Scaling cases s32 / s64: integer-valued matrix with ties and all-zero genes, the
reference's stdscale_quantile_celing at quantile 0.9999 and max_value None / 3.
"""
import hashlib
import importlib.util
import os
import sys
import types

import numpy as np

from oracle import refshim

CASES = {
    # name: (harmony variables, K, dtype, layout)
    "v1_k20_f64_old": (1, 20, np.float64, "old"),
    "v2_k20_f32_new": (2, 20, np.float32, "new"),
    "v1_k1_f32_old": (1, 1, np.float32, "old"),
    "v2_k1_f64_new": (2, 1, np.float64, "new"),
    "v2_k20_f32_old": (2, 20, np.float32, "old"),
    "v1_k20_f64_new": (1, 20, np.float64, "new"),
}
N_CELLS, N_GENES, N_PCS = 65, 65, 10          # one 64-row / 64-column tile + a ragged one
LEVELS = (3, 2)


class HarmonyResult:
    """The attributes of a harmonypy Harmony object that harmony_correct_X reads."""

    def __init__(self, Z_corr, R, Phi_moe, K, lamb):
        self.Z_corr, self.R, self.Phi_moe, self.K, self.lamb = Z_corr, R, Phi_moe, K, lamb


def make_case(name):
    """Seeded inputs of a case: (X, pca, HarmonyResult in the case's layout)."""
    n_vars, K, dtype, layout = CASES[name]
    rng = np.random.RandomState(sorted(CASES).index(name) + 11)
    X = (rng.gamma(0.6, 1.5, size=(N_CELLS, N_GENES)) * (rng.rand(N_CELLS, N_GENES) < 0.5)).astype(dtype)
    pca = rng.normal(size=(N_CELLS, N_PCS))
    rows = [np.ones(N_CELLS)]
    for v in range(n_vars):
        lab = rng.randint(0, LEVELS[v], size=N_CELLS)
        rows += [(lab == j).astype(np.float64) for j in range(LEVELS[v])]
    Phi = np.vstack(rows)                                             # (B+1) x cells
    logits = rng.normal(scale=2.0, size=(K, N_CELLS))
    R = np.exp(logits - logits.max(0))
    R /= R.sum(0)                                                     # K x cells
    lamb = np.diag(np.concatenate([[0.0], np.full(Phi.shape[0] - 1, 1.0)]))
    Z = pca + 0.1 * rng.normal(size=pca.shape)                        # cells x PCs
    if layout == "old":
        res = HarmonyResult(Z.T.copy(), R, Phi, K, lamb)
    else:
        res = HarmonyResult(Z.copy(), R.T.copy(), Phi.T.copy(), K, lamb)
    return X, pca, res


def make_scale_input(dtype):
    rng = np.random.RandomState(5)
    X = rng.poisson(0.8, size=(300, 70)).astype(dtype)
    X[:, [3, 40]] = 0                                                 # zero-std genes
    X[rng.rand(300, 70) < 0.002] = 40                                 # a heavy tail for the ceiling to cut
    return X


def inputs_digest(arrays):
    """sha256 of the dtype, shape and bytes of each array, in order."""
    h = hashlib.sha256()
    for a in arrays:
        a = np.ascontiguousarray(a)
        h.update(("%s%s" % (a.dtype.str, a.shape)).encode())
        h.update(a.tobytes())
    return h.hexdigest()


def case_inputs(name):
    """The arrays of a case that inputs_digest covers."""
    X, pca, res = make_case(name)
    return [X, pca, res.Z_corr, res.R, res.Phi_moe, res.lamb]


def _scale(adata, zero_center=False, max_value=None):
    assert not zero_center
    if hasattr(adata.X, "tocsr"):
        refshim._scale(adata, zero_center)
        if max_value is not None:
            adata.X.data[adata.X.data > max_value] = max_value
        return
    X = np.asarray(adata.X)
    X64 = X.astype(np.float64)
    n = X.shape[0]
    mean = X64.mean(axis=0)
    sq = (X64 * X64).mean(axis=0)
    std = np.sqrt((sq - mean ** 2) * (n / (n - 1)))
    std[std == 0] = 1
    Y = (X64 / std).astype(X.dtype)
    if max_value is not None:
        Y[Y > max_value] = max_value
    adata.X = Y


_CURRENT = {}


def load_reference_preprocess():
    root = os.environ.get("CNMF_REFERENCE")
    if not root:
        raise RuntimeError("CNMF_REFERENCE is not set: point it at a dylkot/cNMF checkout")
    refshim._install_stubs()
    sys.modules["scanpy"].pp.scale = _scale
    hp = types.ModuleType("harmonypy")
    hp.run_harmony = lambda pca, obs, harmony_vars, **kw: _CURRENT["res"]
    sys.modules["harmonypy"] = hp
    path = os.path.join(root, "src", "cnmf", "preprocess.py")
    spec = importlib.util.spec_from_file_location("cnmf_reference_preprocess", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def generate():
    ref = load_reference_preprocess()
    out = {}
    for name in sorted(CASES):
        X, pca, res = make_case(name)
        _CURRENT["res"] = res
        X_corr, X_pca_h = ref.Preprocess(random_seed=0).harmony_correct_X(X.copy(), None, pca, ["batch"])
        R, Phi = (res.R, res.Phi_moe) if CASES[name][3] == "old" else (res.R.T, res.Phi_moe.T)
        Z_cos, Z_corr, W, Phi_Rk = ref.moe_correct_ridge(X.T.copy(), None, None, R, None, res.K, None, Phi, res.lamb)
        out[name + "__inputs_digest"] = np.array(inputs_digest(case_inputs(name)))
        # Z_cos is Z_corr_ridge divided by these per-cell norms, and X_pca_harmony is Harmony's Z_corr re-laid: both are
        # kept in compact forms that give back the reference's arrays bit for bit
        norms = np.linalg.norm(Z_corr, ord=2, axis=0)
        assert np.array_equal(Z_corr / norms, Z_cos)
        out[name + "__X_pca_harmony_digest"] = np.array(inputs_digest([X_pca_h]))
        for k, v in dict(X_corr=X_corr, Z_cos_norms=norms, Z_corr_ridge=Z_corr, W=W, Phi_Rk=Phi_Rk).items():
            out["%s__%s" % (name, k)] = np.asarray(v)
    for tag, dtype in (("s32", np.float32), ("s64", np.float64)):
        X = make_scale_input(dtype)
        out[tag + "__inputs_digest"] = np.array(inputs_digest([X]))
        for mv in (None, 3.0):
            a = refshim.AnnDataLite(X.copy())
            ref.stdscale_quantile_celing(a, max_value=mv, quantile_thresh=0.9999)
            out["%s__out_%s" % (tag, "none" if mv is None else "3")] = np.asarray(a.X)
    return out


if __name__ == "__main__":
    dst = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                       "preprocess_moe.npz")
    np.savez_compressed(dst, **generate())
    print("wrote", dst, os.path.getsize(dst), "bytes")
