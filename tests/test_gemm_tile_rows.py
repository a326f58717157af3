"""Split-K products of at least 2 048 rows in the exact-B forms of the batched GEMM (f16x2 and tf32x3 with an exact B)
run on 192-row output tiles with three consumer warpgroups of 64 rows; everything else on 128-row tiles.  Row counts
around the 192-row boundaries (including last tiles whose third, or second and third, warpgroup lies wholly past M),
odd n-tile counts and split-K slices must match float64, and a row's output must not depend on where in a tile it
lands, nor on which tile height computed it: every element is formed by the same chains in the same order."""
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


def gemm(eng, A, B, precision, splits):
    return eng.gemm_abt(A, B, precision=precision, splits=splits, b_exact=True)[0]


def sampled_rows(M):
    """First and last row of every 64-row warpgroup block: the sampled rows see every warpgroup of every tile."""
    return np.asarray(sorted({x for t in range(0, M, 64) for x in (t, min(t + 63, M - 1))}))


# (M, N, K, splits): N = 600 is 5 n-tiles (the last pair's second CTA has none).  Last 192-row tiles: 191 rows (2111),
# full (2112), 1 row (2113, 2305: warpgroups 2-3 empty), 88 rows (2200: warpgroup 3 empty), 36 rows (8100).
SHAPES = [(2111, 600, 5000, 3), (2112, 600, 5000, 3), (2113, 600, 5000, 3), (2200, 600, 5000, 3),
          (2305, 600, 5000, 3), (8100, 600, 5000, 3)]


@pytest.mark.parametrize("precision", ["f16x2", "tf32x3"])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_gemm_tile_rows_against_float64(eng, shape, precision):
    M, N, K, sp = shape
    A, B = operands(M, N, K, M + N + K)
    C = gemm(eng, A, B, precision, sp)
    assert not np.isnan(C).any()
    rows = sampled_rows(M)
    ref = A[rows].astype(np.float64) @ B.astype(np.float64).T
    err = np.linalg.norm(C[rows] - ref, axis=1) / np.linalg.norm(ref, axis=1)
    assert err.max() < TOL_GEMM, err.max()


# Extra rows in front of A move every row to another warpgroup, tile and pair of the launch; the first 2 047 rows alone
# run on 128-row tiles.
@pytest.mark.parametrize("precision", ["f16x2", "tf32x3"])
def test_gemm_tile_rows_position_and_height_invariance(eng, precision):
    M, N, K, sp = 2113, 600, 5000, 3
    A, B = operands(M, N, K, M + N + K)
    C = gemm(eng, A, B, precision, sp)
    extra = np.abs(np.random.RandomState(1).standard_normal((191, K))).astype(np.float32)
    for shift in (1, 64, 96, 128, 191):
        Cs = gemm(eng, np.vstack([extra[:shift], A]), B, precision, sp)
        assert np.array_equal(Cs[shift:], C), shift
    assert np.array_equal(gemm(eng, A[:2047], B, precision, sp), C[:2047])
