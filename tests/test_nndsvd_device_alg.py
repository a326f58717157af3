"""CPU: the device NNDSVD algorithm (restated in numpy, tests/nndsvd_device_alg.py) gives scikit-learn's starts:
CholeskyQR2 spans the same subspaces as the LU-normalised range finder, and the Jacobi SVD of the small factor gives
the same triplets."""
import numpy as np
import pytest

from cnmf_golden import load_golden
from nndsvd_device_alg import device_nndsvd_init, orth_rows
from cnmf_b200.nndsvd import nndsvd_init

TOL = 1e-11


def rel(a, b):
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


def _counts(n, g, seed):
    rng = np.random.RandomState(seed)
    X = rng.poisson(rng.gamma(0.6, 2.0, size=(1, g)) * rng.gamma(2.0, 0.5, size=(n, 1))).astype(np.float64)
    X[0, X.sum(axis=0) == 0] = 1.0          # no constant column
    return X / X.std(axis=0, ddof=1)


def _cases():
    sim = load_golden("sim_nndsvd")["X"]
    c1 = load_golden("c1_mu")["X"]
    return [("sim", sim, 4, 11), ("sim", sim, 5, 3), ("c1", c1, 7, 5), ("c1", c1, 32, 2), ("c1", c1, 1, 9),
            ("transposed", _counts(120, 300, 0), 20, 4), ("transposed", _counts(60, 90, 1), 1, 8),
            ("p_capped", _counts(30, 12, 2), 5, 1), ("p_capped_t", _counts(12, 30, 3), 12, 6)]


@pytest.mark.parametrize("init", ["nndsvd", "nndsvda", "nndsvdar"])
@pytest.mark.parametrize("case", range(9))
def test_device_algorithm_matches_nndsvd_init(case, init):
    _, X, k, seed = _cases()[case]
    W0, H0 = nndsvd_init(X, k, seed, init)
    W1, H1 = device_nndsvd_init(X, k, seed, init)
    assert rel(W1, W0) < TOL and rel(H1, H0) < TOL, (rel(W1, W0), rel(H1, H0))
    assert ((W1 == 0) == (W0 == 0)).all() and ((H1 == 0) == (H0 == 0)).all()


def test_nndsvdar_fills_zeros_in_w_then_h_row_major_order():
    """The 'ar' fill draws one normal per zero of the 'nndsvd' start: W's zeros (cells x k, row-major) first, then
    H's, from a fresh RandomState(seed) -- the values the host restatement puts at the same places."""
    X = load_golden("sim_nndsvd")["X"]
    k, seed = 5, 7
    W, H = device_nndsvd_init(X, k, seed, "nndsvd")
    Wr, Hr = device_nndsvd_init(X, k, seed, "nndsvdar")
    Wh, Hh = nndsvd_init(X, k, seed, "nndsvdar")
    zw, zh = W == 0, H == 0
    assert zw.sum() > 0 and zh.sum() > 0
    z = np.random.RandomState(seed).standard_normal(int(zw.sum() + zh.sum()))
    avg = X.mean()
    np.testing.assert_array_equal(Wr[zw], np.abs(avg * z[:zw.sum()] / 100))
    np.testing.assert_array_equal(Hr[zh], np.abs(avg * z[zw.sum():] / 100))
    np.testing.assert_array_equal(Wr[zw], Wh[zw])
    np.testing.assert_array_equal(Hr[zh], Hh[zh])


def test_rank_deficient_rows_are_dropped_not_amplified():
    """Duplicated rows: CholeskyQR2 keeps the independent rows orthonormal and zeroes the dependent ones."""
    rng = np.random.RandomState(0)
    A = rng.randn(6, 200)
    A[3] = A[1]
    A[5] = 2.0 * A[0] - A[2]
    Q, _ = orth_rows(A)
    assert np.isfinite(Q).all()
    assert not Q[3].any() and not Q[5].any()
    keep = [0, 1, 2, 4]
    np.testing.assert_allclose(Q[keep] @ Q[keep].T, np.eye(4), atol=1e-14)
