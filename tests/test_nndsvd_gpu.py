"""GPU (`-m gpu`): NNDSVD starting factors computed on the device (cnmf_nndsvd_init_dev) against scikit-learn's
algorithm on the host (cnmf_b200.nndsvd.nndsvd_init), and the solves that start from them."""
import numpy as np
import pytest

from cnmf_golden import load_golden

pytestmark = pytest.mark.gpu

ULP32 = 2.0 ** -23


def rel(a, b):
    a = np.asarray(a, dtype=np.float64)
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


@pytest.fixture(scope="module")
def eng():
    from cnmf_b200.engine import Engine
    return Engine(0)


def _counts(n, g, seed, k_true=6):
    from cnmf_b200.synth import make_counts, normalise
    X, _ = normalise(make_counts(n, g, k_true=k_true, seed=seed, libsize=600.0), np.float32)
    return X


def device_starts(ds, ks, seeds, init):
    """(list of W n x k, list of H k x g) of cnmf_nndsvd_init_dev, fp32, padding checked"""
    import torch
    ld_r, ld_c = ds.ld()
    n, g = ds.shape
    SK = int(np.sum(ks))
    Wt = torch.full((SK, ld_r), 7.0, dtype=torch.float32, device="cuda:0")
    H = torch.full((SK, ld_c), 7.0, dtype=torch.float32, device="cuda:0")
    ds.nndsvd_init_dev(ks, seeds, init, Wt.data_ptr(), H.data_ptr())
    Wt, H = Wt.cpu().numpy(), H.cpu().numpy()
    assert not Wt[:, n:].any() and not H[:, g:].any()
    offs = np.concatenate([[0], np.cumsum(ks)])
    return ([Wt[offs[r]:offs[r + 1], :n].T for r in range(len(ks))],
            [H[offs[r]:offs[r + 1], :g] for r in range(len(ks))])


def assert_fp32_of(dev, host, eps=1e-6):
    """dev (fp32) is host (fp64) rounded to fp32 up to rounding-boundary flips: at most 1 ulp apart anywhere, equal
    in all but 1e-3 of the entries, zero exactly where the host is zero except within 1e-9 of eps."""
    h32 = host.astype(np.float32).astype(np.float64)
    d = dev.astype(np.float64)
    diff = np.abs(d - h32)
    near_eps = np.abs(host - eps) < 1e-9
    assert (((d == 0) == (host == 0)) | near_eps).all()
    ok = diff <= ULP32 * np.abs(host) * 1.0001
    assert (ok | near_eps).all(), float((diff / np.maximum(np.abs(host), 1e-300))[~(ok | near_eps)].max())
    assert (diff > 0).mean() <= 1e-3, float((diff > 0).mean())
    assert rel(d, host) < 1e-7


# ------------------------------------------------------------------------------------ fp64 GEMM
@pytest.mark.parametrize("shape", [(333, 97, 45), (97, 333, 45), (1000, 500, 130), (70, 40, 1), (129, 257, 65)])
@pytest.mark.parametrize("to_genes", [False, True])
def test_fp64_gemm_against_numpy(eng, shape, to_genes):
    n, g, M = shape
    rng = np.random.RandomState(n + g + M)
    X = np.abs(rng.randn(n, g)).astype(np.float32)
    ds = eng.dataset(X)
    A = rng.randn(M, n if to_genes else g)
    C = ds.nndsvd_gemm(A, to_genes)
    X64 = X.astype(np.float64)
    ref = A @ X64 if to_genes else A @ X64.T
    assert rel(C, ref) < 1e-13


# ------------------------------------------------------------------------------------ starts
def _start_cases():
    return [("sim_nndsvd", [4, 5, 1], [11, 3, 9]), ("c1_mu", [7, 32, 1], [5, 2, 9]),
            ("transposed", [20, 1], [4, 8]), ("p_capped", [5], [1])]


def _matrix(tag):
    if tag == "transposed":
        return _counts(120, 300, 0)
    if tag == "p_capped":
        return _counts(30, 12, 2, k_true=3)
    return load_golden(tag)["X"]


@pytest.mark.parametrize("init", ["nndsvd", "nndsvda", "nndsvdar"])
@pytest.mark.parametrize("case", range(4))
def test_device_starts_equal_host_on_the_fp32_matrix(eng, case, init):
    """Against scikit-learn's algorithm in float64 on the matrix the device holds (fp32 X): the starts agree to
    rounding to fp32 (the float64 values are within ~1e-11)."""
    from cnmf_b200.nndsvd import nndsvd_init
    tag, ks, seeds = _start_cases()[case]
    X = _matrix(tag)
    ds = eng.dataset(X)
    X64 = np.asarray(X, dtype=np.float32).astype(np.float64)
    Ws, Hs = device_starts(ds, ks, seeds, init)
    for r, (k, seed) in enumerate(zip(ks, seeds)):
        W0, H0 = nndsvd_init(X64, k, seed, init)
        assert_fp32_of(Ws[r], W0)
        assert_fp32_of(Hs[r], H0)


@pytest.mark.parametrize("tag", ["sim_nndsvd", "c1_mu"])
def test_device_starts_near_host_on_the_fixture_matrix(eng, tag):
    from cnmf_b200.nndsvd import nndsvd_init
    X = load_golden(tag)["X"]
    ds = eng.dataset(X)
    ks, seeds = [4, 7], [21, 22]
    Ws, Hs = device_starts(ds, ks, seeds, "nndsvda")
    for r, (k, seed) in enumerate(zip(ks, seeds)):
        W0, H0 = nndsvd_init(X, k, seed, "nndsvda")
        assert rel(Ws[r], W0) < 1e-6 and rel(Hs[r], H0) < 1e-6


@pytest.mark.parametrize("init", ["nndsvd", "nndsvdar"])
def test_restart_starts_do_not_depend_on_the_batch_or_the_chunking(eng, init):
    """One restart alone, and in a mixed-K batch processed one, two or all restarts per chunk (the chunk cap of the
    test hook; by default chunks are sized from free device memory): bit-identical.  min(N, G) <= 200 puts the
    power-iteration threshold at <= 20, so the batch runs both iteration classes (k >= 20: 4, else 7)."""
    X = _counts(20000, 200, 5)
    ds = eng.dataset(X)
    n, g = ds.shape
    ks = [13, 3, 30, 9, 25, 2, 20]
    seeds = [7, 1, 2, 3, 4, 5, 6]
    assert any(k >= 0.1 * min(n, g) for k in ks) and any(k < 0.1 * min(n, g) for k in ks)
    Wa, Ha = device_starts(ds, [13], [7], init)
    runs = {}
    try:
        for cap in (1, 2, 0):
            eng.nndsvd_chunk_limit(cap)
            runs[cap] = device_starts(ds, ks, seeds, init)
    finally:
        eng.nndsvd_chunk_limit(0)
    Wb, Hb = runs[0]
    assert np.array_equal(Wa[0], Wb[0]) and np.array_equal(Ha[0], Hb[0])
    for cap in (1, 2):
        for r in range(len(ks)):
            assert np.array_equal(runs[cap][0][r], Wb[r]), (cap, r)
            assert np.array_equal(runs[cap][1][r], Hb[r]), (cap, r)


def test_rank_deficient_matrix_gives_finite_starts(eng):
    """X of rank 3 with k = 5 (P = 15): finite starts; the components inside the rank agree with the host."""
    from cnmf_b200.nndsvd import nndsvd_init
    rng = np.random.RandomState(3)
    X = (rng.gamma(1.0, 1.0, size=(300, 3)) @ rng.gamma(1.0, 1.0, size=(3, 80))).astype(np.float32)
    X[:, 40:] = X[:, :40]                      # duplicated columns as well
    ds = eng.dataset(X, precision="tf32x3-general")
    Ws, Hs = device_starts(ds, [5], [4], "nndsvd")
    assert np.isfinite(Ws[0]).all() and np.isfinite(Hs[0]).all()
    W0, H0 = nndsvd_init(X.astype(np.float64), 5, 4, "nndsvd")
    assert rel(Ws[0][:, :3], W0[:, :3]) < 1e-6 and rel(Hs[0][:3], H0[:3]) < 1e-6


def test_sparse_dataset_is_refused(eng):
    import scipy.sparse as sp
    import torch
    from cnmf_b200._lib import CnmfError
    X = load_golden("sim_nndsvd")["X"]
    ds = eng.sparse_dataset(sp.csc_matrix(X))
    ld_r, ld_c = ds.ld()
    Wt = torch.zeros((4, ld_r), dtype=torch.float32, device="cuda:0")
    H = torch.zeros((4, ld_c), dtype=torch.float32, device="cuda:0")
    with pytest.raises(CnmfError, match="sparse"):
        ds.nndsvd_init_dev([4], [1], "nndsvd", Wt.data_ptr(), H.data_ptr())


# ------------------------------------------------------------------------------------ solves from device starts
@pytest.mark.parametrize("precision", ["f16x2", "tf32x3-general"])
def test_factorize_without_host_matrix_matches_reference_fixture(eng, precision):
    """`--init nndsvd` entirely on the device: the reference's own run (fixture sim_nndsvd), every restart: same
    n_iter, spectra within 1e-4 (median 1e-5), reported error = ||X - WH||_F."""
    from oracle import nmf_ref
    g = load_golden("sim_nndsvd")
    ds = eng.dataset(g["X"], precision=precision)
    kw = dict(solver=g["solver"], tol=1e-4, max_iter=1000, alpha_W=0.0, alpha_H=0.0, l1_ratio=0.0,
              beta_loss=2.0 if g["solver"] == "mu" else "frobenius", init=g["init"])
    table = g["table"]
    sp, us, n_iter, err = ds.factorize(table[:, 0], table[:, 2], kw, return_usages=True)
    errs = []
    for r, (k, it, seed) in enumerate(table):
        ref = g["merged_k%d" % k][it * k:(it + 1) * k]
        e = rel(sp[r], ref)
        errs.append(e)
        assert e < 1e-4, (precision, k, it, e)
        _, _, n_o = nmf_ref.nmf(g["X"], int(k), int(seed), solver=g["solver"], init=g["init"])
        assert n_o == int(n_iter[r]), (precision, k, it, n_o, int(n_iter[r]))
        e_true = nmf_ref.frobenius_error(g["X"], us[r].astype(np.float64), sp[r].astype(np.float64))
        assert abs(err[r] - e_true) / e_true < 1e-5
    assert np.median(errs) < 1e-5, errs


def test_factorize_seeds_dev_with_nndsvd_agrees_with_factorize(eng):
    import torch
    g = load_golden("sim_nndsvd")
    ds = eng.dataset(g["X"])
    kw = dict(solver="mu", tol=1e-4, max_iter=1000, init="nndsvda")
    table = g["table"]
    ks, seeds = table[:, 0], table[:, 2]
    sp, _, n_iter, _ = ds.factorize(ks, seeds, kw)
    _, ld = ds.ld()
    out = torch.zeros((int(ks.sum()), ld), dtype=torch.float32, device="cuda:0")
    n_iter_d, _ = ds.factorize_seeds_dev(ks, seeds, out.data_ptr(), ld, kw)
    assert np.array_equal(n_iter, n_iter_d)
    got = out.cpu().numpy()[:, :ds.shape[1]]
    assert rel(got, np.vstack(sp)) < 1e-6


def test_atlas_sized_starts_against_host(eng):
    """50 000 x 2 000 (BASELINE c3's shape), K = 5, 9, 13: device starts against the host on the fp32 matrix."""
    from cnmf_b200.nndsvd import nndsvd_init
    X = _counts(50000, 2000, 11, k_true=12)
    ds = eng.dataset(X)
    ks, seeds = [5, 9, 13], [101, 102, 103]
    Ws, Hs = device_starts(ds, ks, seeds, "nndsvd")
    X64 = X.astype(np.float64)
    for r, (k, seed) in enumerate(zip(ks, seeds)):
        W0, H0 = nndsvd_init(X64, k, seed, "nndsvd")
        assert rel(Ws[r], W0) < 1e-7 and rel(Hs[r], H0) < 1e-7
