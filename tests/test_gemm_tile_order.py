"""The batched GEMM on problems whose factor operand is larger than half the L2, where the launcher runs the tiles in
grouped orders (several groups of m-tiles or of n-tiles, the last group partial): every tile is written exactly where
it belongs and matches float64.  The m-tile-fastest order of smaller problems is covered by test_gpu_parity.py."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

TOL_GEMM = 2e-6          # fp32-class GEMM vs float64, as in test_gpu_parity.py


@pytest.fixture(scope="module")
def eng():
    from cnmf_b200.engine import Engine
    return Engine(0)


def tile_rows(M):
    """First and last row of every 128-row tile: the sampled rows see every output tile."""
    r = sorted({x for t in range(0, M, 128) for x in (t, min(t + 127, M - 1))})
    return np.asarray(r)


# (M, N, K, splits, precision): with an H100's 50 MB L2 these take, in order, 2 groups of n-tiles (16 + 15), 2 groups of
# m-tiles (20 + 19) and 3 groups of n-tiles (11 + 11 + 9)
@pytest.mark.parametrize("shape", [(1600, 3900, 4096, 1, "f16x2"), (4900, 20000, 2000, 1, "f16x2"),
                                   (1600, 3900, 2048, 1, "tf32x3")])
def test_gemm_grouped_tile_order_against_float64(eng, shape):
    M, N, K, sp, precision = shape
    rng = np.random.RandomState(M + N + K)
    A = np.abs(rng.standard_normal((M, K))).astype(np.float32)
    B = rng.poisson(1.5, size=(N, K)).astype(np.float32)
    C, _ = eng.gemm_abt(A, B, precision=precision, splits=sp)
    assert not np.isnan(C).any()                          # the output starts as NaN: every tile was written
    rows = tile_rows(M)
    ref = A[rows].astype(np.float64) @ B.astype(np.float64).T
    err = np.linalg.norm(C[rows] - ref, axis=1) / np.linalg.norm(ref, axis=1)
    assert err.max() < TOL_GEMM, err.max()
