"""Output-tile widths of the exact-B forms of the batched GEMM (f16x2 and tf32x3 with an exact B): 128, 168 and 192
columns, forced through tile_n or chosen by shape (tile_n = 0).  Column counts around the width boundaries (a last tile
with one column, a full one, odd n-tile counts whose last pair has one CTA with no tile), row counts around one and two
warpgroups, split-K slices and products as wide as a cell count must match float64, and the outputs must be
bit-identical across the widths and when B gains leading rows: every element is formed by the same chains in the same
order, whichever tile, CTA and width computes it."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

TOL_GEMM = 2e-6          # fp32-class GEMM vs float64, as in test_gpu_parity.py
TILE_N = (0, 128, 168, 192)


@pytest.fixture(scope="module")
def eng():
    from cnmf_b200.engine import Engine
    return Engine(0)


def operands(M, N, K, seed):
    rng = np.random.RandomState(seed)
    A = np.abs(rng.standard_normal((M, K))).astype(np.float32)
    B = rng.poisson(1.5, size=(N, K)).astype(np.float32)
    return A, B


def gemm(eng, A, B, precision, splits, tile_n):
    return eng.gemm_abt(A, B, precision=precision, splits=splits, b_exact=True, tile_n=tile_n)[0]


# (M, N, K, splits).  N: 167-169 and 191-193 around one tile of each wide width, 337 = 2 * 168 + 1 and 385 = 2 * 192 + 1
# (three n-tiles: the second pair's second CTA has none), 2000 (the gene count of the benchmark: 12 tiles of 168, 11 of
# 192), 50000 (its cell count).  M: 64, 65, 127, 128, 129 rows; 2113 rows with split-K run on 192-row tiles at 128
# columns and on 128-row tiles at the wide widths.
SHAPES = [(128, 167, 1000, 1), (64, 168, 1000, 1), (65, 169, 1000, 1), (127, 191, 1000, 1), (128, 192, 1000, 1),
          (129, 193, 1000, 1), (129, 337, 1000, 1), (200, 385, 3000, 2), (130, 2000, 5000, 3), (64, 50000, 512, 1),
          (2113, 400, 5000, 3)]


@pytest.mark.parametrize("precision", ["f16x2", "tf32x3"])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_gemm_tile_cols_against_float64(eng, shape, precision):
    M, N, K, sp = shape
    A, B = operands(M, N, K, M + N + K)
    C = gemm(eng, A, B, precision, sp, 0)
    assert not np.isnan(C).any()
    rows = np.arange(M) if M <= 256 else np.arange(0, M, 7)
    ref = A[rows].astype(np.float64) @ B.astype(np.float64).T
    err = np.linalg.norm(C[rows] - ref, axis=1) / np.linalg.norm(ref, axis=1)
    assert err.max() < TOL_GEMM, err.max()
    for tn in TILE_N[1:]:
        assert np.array_equal(gemm(eng, A, B, precision, sp, tn), C), tn


# Extra rows in front of B move every column to another place in its tile, another tile and another CTA of the pair.
@pytest.mark.parametrize("precision", ["f16x2", "tf32x3"])
@pytest.mark.parametrize("tile_n", TILE_N)
def test_gemm_tile_cols_position_invariance(eng, precision, tile_n):
    M, N, K, sp = 130, 2000, 5000, 3
    A, B = operands(M, N, K, M + N + K)
    C = gemm(eng, A, B, precision, sp, tile_n)
    extra = np.random.RandomState(2).poisson(1.5, size=(191, K)).astype(np.float32)
    for shift in (1, 8, 40, 168, 191):
        Cs = gemm(eng, A, np.vstack([extra[:shift], B]), precision, sp, tile_n)
        assert np.array_equal(Cs[:, shift:], C), shift


def test_gemm_tile_n_is_checked(eng):
    from cnmf_b200._lib import CnmfError
    A, B = operands(64, 200, 256, 0)
    with pytest.raises(CnmfError):
        eng.gemm_abt(A, B, precision="f16x2", tile_n=160)
    with pytest.raises(CnmfError):
        eng.gemm_abt(A, B, precision="tf32x3", tile_n=168)      # the general 3-pass form has 128-column tiles only
