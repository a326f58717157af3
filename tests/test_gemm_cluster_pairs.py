"""The batched GEMM runs in clusters of two CTAs that share (multicast) the A panel of an m-tile, each computing one n-tile
of an adjacent pair.  Which CTA of a pair computes a tile must not change a bit of it; grouped tile orders over n-pairs
with an odd number of n-tiles (the last pair's second CTA has no tile) must write every tile where it belongs; and
launches with fewer pairs than the device can run at once must be complete."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

TOL_GEMM = 2e-6          # fp32-class GEMM vs float64, as in test_gpu_parity.py


@pytest.fixture(scope="module")
def eng():
    from cnmf_b200.engine import Engine
    return Engine(0)


def operands(M, N, K, seed):
    rng = np.random.RandomState(seed)
    A = np.abs(rng.standard_normal((M, K))).astype(np.float32)
    B = rng.poisson(1.5, size=(N, K)).astype(np.float32)
    return A, B


def tile_rows(M):
    """First and last row of every 128-row tile: the sampled rows see every output tile."""
    return np.asarray(sorted({x for t in range(0, M, 128) for x in (t, min(t + 127, M - 1))}))


# 128 extra rows in front of B move every n-tile to the other CTA of its pair; each output element is still formed by
# the same chains in the same order, so it must come out bit for bit the same.
@pytest.mark.parametrize("shape", [(300, 700, 3000, 1, "f16x2"), (300, 700, 20000, 5, "f16x2"),
                                   (300, 700, 1000, 1, "tf32x3")])
def test_gemm_pair_position_invariance(eng, shape):
    M, N, K, sp, precision = shape
    A, B = operands(M, N, K, M + N + K)
    extra = np.random.RandomState(1).poisson(1.5, size=(128, K)).astype(np.float32)
    C, _ = eng.gemm_abt(A, B, precision=precision, splits=sp)
    Cs, _ = eng.gemm_abt(A, np.vstack([extra, B]), precision=precision, splits=sp)
    assert not np.isnan(C).any() and not np.isnan(Cs).any()
    assert np.array_equal(Cs[:, 128:], C)


# (M, N, K, splits, precision): with an H100's 50 MB L2 and 66 pairs at once these take, in order, 2 groups of m-tiles
# (19 + 18) over 157 n-tiles, 2 groups of n-pairs (8 + 7) over 29 n-tiles, and 3 groups of n-pairs (6 + 6 + 4) over
# 31 n-tiles: each has an odd number of n-tiles and a partial last group.
@pytest.mark.parametrize("shape", [(4700, 20000, 2000, 1, "f16x2"), (1600, 3700, 4096, 1, "f16x2"),
                                   (1700, 3900, 2048, 1, "tf32x3")])
def test_gemm_grouped_pair_orders_against_float64(eng, shape):
    M, N, K, sp, precision = shape
    A, B = operands(M, N, K, M + N + K)
    C, _ = eng.gemm_abt(A, B, precision=precision, splits=sp)
    assert not np.isnan(C).any()                          # the output starts as NaN: every tile was written
    rows = tile_rows(M)
    ref = A[rows].astype(np.float64) @ B.astype(np.float64).T
    err = np.linalg.norm(C[rows] - ref, axis=1) / np.linalg.norm(ref, axis=1)
    assert err.max() < TOL_GEMM, err.max()


# Fewer pair items than pairs the device runs at once, so the grid is cut to the items: 2 x 2 pairs, 3 x 1 pairs in
# 2 slices, and 1 pair.
@pytest.mark.parametrize("shape", [(200, 300, 1000, 1, "f16x2"), (300, 130, 3000, 2, "f16x2"),
                                   (100, 200, 700, 1, "tf32x3")])
def test_gemm_fewer_pairs_than_clusters(eng, shape):
    M, N, K, sp, precision = shape
    A, B = operands(M, N, K, M + N + K)
    C, _ = eng.gemm_abt(A, B, precision=precision, splits=sp)
    ref = A.astype(np.float64) @ B.astype(np.float64).T
    err = np.linalg.norm(C - ref, axis=1) / np.linalg.norm(ref, axis=1)
    assert err.max() < TOL_GEMM, err.max()
