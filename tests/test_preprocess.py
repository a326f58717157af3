"""Preprocess: Harmony's ridge correction and the variance scaling with a quantile ceiling, against the reference's
outputs (tests/golden/preprocess_moe.npz from oracle/make_golden_preprocess.py) and float64 numpy."""
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import make_golden_preprocess as mg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "preprocess_moe.npz")
HARMONYPY_TEXT = "harmonypy is not installed. Please install it using 'pip install harmonypy' before proceeding."


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(GOLDEN))


def case(gold, name):
    """The reference's outputs of a case with its inputs, regenerated from their seeds."""
    p = name + "__"
    c = {k[len(p):]: v for k, v in gold.items() if k.startswith(p)}
    X, pca, res = mg.make_case(name)
    c.update(X=X, pca=pca, Z_corr=res.Z_corr, R=res.R, Phi_moe=res.Phi_moe, lamb=res.lamb, K=res.K)
    c["Z_cos"] = c["Z_corr_ridge"] / c["Z_cos_norms"]         # the reference's own division, bit for bit
    return c


def fitted(c):
    return mg.HarmonyResult(c["Z_corr"], c["R"], c["Phi_moe"], int(c["K"]), c["lamb"])


def ridge_f64(X, R, Phi, lamb):
    """X - sum_i W_i^T P_i in float64 numpy, W_i = inv(P_i Phi^T + lamb) P_i X with row 0 zeroed; also the
    elementwise sum of |terms| that bounds its rounding error."""
    X = np.asarray(X, np.float64)
    out, mag = X.copy(), np.abs(X)
    for i in range(R.shape[0]):
        P = Phi * R[i]
        W = np.linalg.inv(P @ Phi.T + lamb) @ (P @ X)
        W[0] = 0
        out -= P.T @ W
        mag += np.abs(P.T) @ np.abs(W)
    return out, mag


# ---------------------------------------------------------------------------------------------------- CPU


def test_oracle_inputs_reproduce_fixture(gold):
    for name in mg.CASES:
        assert mg.inputs_digest(mg.case_inputs(name)) == str(gold[name + "__inputs_digest"]), name
    for tag, dt in (("s32", np.float32), ("s64", np.float64)):
        assert mg.inputs_digest([mg.make_scale_input(dt)]) == str(gold[tag + "__inputs_digest"]), tag


def test_fixture_outputs_match_float64_restatement(gold):
    from cnmf_b200.preprocess import harmony_layout
    for name in mg.CASES:
        c = case(gold, name)
        R, Phi, Zp = harmony_layout(fitted(c), c["pca"])
        ref, mag = ridge_f64(c["X"], R, Phi, c["lamb"])
        tol = (1e-10 if c["X"].dtype == np.float64 else 1e-5) * np.abs(ref).max()
        assert np.abs(c["Z_corr_ridge"].T - ref).max() <= tol, name
        assert np.abs(c["X_corr"] - np.maximum(ref, 0)).max() <= tol, name
        assert mg.inputs_digest([Zp]) == str(c["X_pca_harmony_digest"]), name
        if os.environ.get("CNMF_REFERENCE"):
            again = mg.generate()
            assert all(np.array_equal(again[k], gold[k]) for k in gold)
            break


def test_layout_detection_with_fake_results():
    from cnmf_b200.preprocess import harmony_layout
    n, pcs, K, B1 = 7, 3, 4, 2
    rng = np.random.RandomState(0)
    Z, R, Phi = rng.rand(n, pcs), rng.rand(K, n), rng.rand(B1, n)
    old = mg.HarmonyResult(Z.T, R, Phi, K, None)
    new = mg.HarmonyResult(Z, R.T, Phi.T, K, None)
    for res in (old, new):
        r, p, z = harmony_layout(res, np.zeros((n, pcs)))
        assert np.array_equal(r, R) and np.array_equal(p, Phi) and np.array_equal(z, Z)


def test_harmonypy_missing_message():
    from cnmf_b200 import Preprocess
    try:
        import harmonypy  # noqa: F401
        pytest.skip("harmonypy is installed")
    except ImportError:
        pass
    with pytest.raises(ImportError) as e:
        Preprocess().harmony_correct_X(np.zeros((3, 2)), None, np.zeros((3, 2)), ["batch"])
    assert str(e.value) == HARMONYPY_TEXT


@pytest.mark.parametrize("method", ["filter_adata", "preprocess_for_cnmf", "normalize_batchcorrect",
                                    "select_features_MI"])
def test_scanpy_bound_methods_refuse(method):
    from cnmf_b200 import Preprocess
    with pytest.raises(NotImplementedError, match="harmony_correct_X"):
        getattr(Preprocess(random_seed=1), method)(None)


def test_import_needs_no_gpu_harmonypy_or_scanpy():
    code = ("import sys, cnmf_b200; from cnmf_b200 import Preprocess; "
            "assert 'harmonypy' not in sys.modules and 'scanpy' not in sys.modules; print('ok')")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True)
    assert r.returncode == 0 and r.stdout.strip() == "ok", r.stderr


def _lerp(a, b, t):
    # numpy's _lerp in the element type, as cnmf_scale_quantile_ceiling applies it
    d = b - a
    return b - d * (1 - t) if t >= 0.5 else a + d * t


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_quantile_ranks_match_np_quantile(dtype):
    from cnmf_b200.preprocess import quantile_ranks
    rng = np.random.RandomState(3)
    for n in (1, 2, 7, 1000, 123457):
        a = np.round(rng.gamma(0.5, 2.0, size=n), 1).astype(dtype)      # ties
        s = np.sort(a)
        for q in (0.0, 0.5, 0.9999, 1.0, 0.3, 1 / 3):
            lo, hi, g = quantile_ranks(n, q, dtype)
            t = _lerp(s[lo], s[hi], dtype(g))
            want = np.quantile(a, q)
            assert t.dtype == want.dtype and t == want, (n, q, t, want)


# ---------------------------------------------------------------------------------------------------- GPU


def _ulps32(a, b):
    ia = np.asarray(a, np.float32).view(np.int32).astype(np.int64)
    ib = np.asarray(b, np.float32).view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7fffffff), ia)
    ib = np.where(ib < 0, -(ib & 0x7fffffff), ib)
    return np.abs(ia - ib)


def _check_against_reference(got, want):
    assert got.dtype == want.dtype and got.shape == want.shape
    if want.dtype == np.float64:
        assert np.abs(got - want).max() <= 1e-12 * np.abs(want).max()
    else:
        u = _ulps32(got, want)
        assert u.max() <= 1, u.max()
        assert (u == 0).mean() >= 0.999, (u == 0).mean()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(mg.CASES))
def test_harmony_correct_X_reproduces_reference(gold, name):
    from cnmf_b200 import Preprocess
    c = case(gold, name)
    X_corr, X_pca_h = Preprocess().harmony_correct_X(c["X"], None, c["pca"], ["batch"], harmony_res=fitted(c))
    _check_against_reference(X_corr, c["X_corr"])
    assert mg.inputs_digest([X_pca_h]) == str(c["X_pca_harmony_digest"])


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(mg.CASES))
def test_moe_correct_ridge_reproduces_reference(gold, name):
    from cnmf_b200.preprocess import harmony_layout, moe_correct_ridge
    c = case(gold, name)
    R, Phi, _ = harmony_layout(fitted(c), c["pca"])
    Z_cos, Z_corr, W, Phi_Rk = moe_correct_ridge(c["X"].T, None, None, R, None, int(c["K"]), None, Phi, c["lamb"])
    _check_against_reference(np.ascontiguousarray(Z_corr), c["Z_corr_ridge"])
    tol = 1e-12 if c["X"].dtype == np.float64 else 1e-6
    assert np.abs(Z_cos - c["Z_cos"]).max() <= tol * np.abs(c["Z_cos"]).max()
    assert np.abs(W - c["W"]).max() <= 1e-9 * np.abs(c["W"]).max()
    assert np.array_equal(Phi_Rk, c["Phi_Rk"])


@pytest.mark.gpu
@pytest.mark.parametrize("n,g", [(63, 127), (65, 129), (64, 128), (4097, 65), (2, 63), (200, 1)])
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_correction_shape_edges_against_float64(n, g, dtype):
    from cnmf_b200.preprocess import moe_correct_cells
    rng = np.random.RandomState(n * 7 + g)
    X = rng.gamma(0.7, 1.0, size=(n, g)).astype(dtype)
    lab = rng.randint(0, 2, size=n)
    lab[:2] = (0, 1)                                                       # both batches present: A is invertible
    Phi = np.vstack([np.ones(n), (lab == 1).astype(np.float64)])           # B = 1
    R = np.ones((1, n))                                                    # K = 1
    lamb = np.diag([1.0, 0.0])                                             # zero except the intercept
    out, _, _ = moe_correct_cells(X, R, Phi, lamb)
    ref, mag = ridge_f64(X, R, Phi, lamb)
    # every term is a dot product over n cells (Gram, P X) or B + 1 rows, each rounded in fp64 and amplified by the
    # ridge system's condition number; fp32 adds one rounding of the result per cluster
    cond = np.linalg.cond((Phi * R[0]) @ Phi.T + lamb)
    bound = 4 * (n + 8) * cond * np.finfo(np.float64).eps * mag
    if dtype == np.float32:
        bound = bound + np.finfo(np.float32).eps * np.abs(ref)
    assert (np.abs(out - ref) <= bound).all()


@pytest.mark.gpu
def test_correction_is_deterministic_and_singular_gram_raises(gold):
    from cnmf_b200.preprocess import harmony_layout, moe_correct_cells
    c = case(gold, "v2_k20_f32_new")
    R, Phi, _ = harmony_layout(fitted(c), c["pca"])
    a = moe_correct_cells(c["X"], R, Phi, c["lamb"], want_cos=True)
    b = moe_correct_cells(c["X"], R, Phi, c["lamb"], want_cos=True)
    for x, y in zip(a, b):
        assert np.array_equal(x.view(np.uint8), y.view(np.uint8))
    n = c["X"].shape[0]
    with pytest.raises(np.linalg.LinAlgError):
        moe_correct_cells(c["X"], R, np.vstack([np.ones(n), np.ones(n)]), np.zeros((2, 2)))


@pytest.mark.gpu
@pytest.mark.parametrize("tag,dtype", [("s32", np.float32), ("s64", np.float64)])
@pytest.mark.parametrize("mv", [None, 3.0])
def test_scale_quantile_reproduces_reference(gold, tag, dtype, mv):
    from cnmf_b200.preprocess import stdscale_quantile_celing
    from oracle.refshim import AnnDataLite
    a = AnnDataLite(mg.make_scale_input(dtype))
    stdscale_quantile_celing(a, max_value=mv, quantile_thresh=0.9999)
    want = gold["%s__out_%s" % (tag, "none" if mv is None else "3")]
    assert a.X.dtype == want.dtype
    assert np.array_equal(a.X, want)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_quantile_threshold_is_np_quantile_bit_for_bit(gold, dtype):
    from cnmf_b200.preprocess import scale_quantile_ceiling
    X = mg.make_scale_input(dtype)
    X = np.vstack([X, X[:37]])                                  # more ties; zero-std genes stay
    scaled, _, _ = scale_quantile_ceiling(X)
    for q in (0.0, 0.5, 0.9999, 1.0):
        out, t, _ = scale_quantile_ceiling(X, quantile_thresh=q)
        want = np.quantile(scaled.reshape(-1), q)
        assert t.dtype == want.dtype and t == want, (q, t, want)
        assert np.array_equal(out, np.where(scaled > want, want, scaled))
    for mv in (None, 2.5):
        d, td, _ = scale_quantile_ceiling(X, max_value=mv, quantile_thresh=0.9)
        s, ts, csr = scale_quantile_ceiling(sp.csr_matrix(X), max_value=mv, quantile_thresh=0.9)
        assert csr is not None and td == ts and np.array_equal(d, s)
