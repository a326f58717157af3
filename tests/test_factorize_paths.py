"""GPU (`-m gpu`): the factorize entry points are one solve behind different ways of supplying the starting factors and
taking out the results.  Fed the same starts they must return the same bits: spectra, n_iter and err.

  cnmf_factorize (device RNG)  ==  cnmf_random_init_dev + cnmf_factorize_dev
                               ==  cnmf_factorize_init on the host copy of those starts
                               ==  cnmf_factorize_seeds_dev
  cnmf_factorize (NNDSVD)      ==  cnmf_nndsvd_init_dev + cnmf_factorize_dev

Batches mix restarts of different K; one list stays at K <= 16 and one reaches K > 16, so both packed-width classes
of the update kernels run."""
import numpy as np
import pytest

from cnmf_golden import load_golden

pytestmark = pytest.mark.gpu

KS = {"k_le16": [3, 7, 12, 5], "k_gt16": [5, 20, 9]}


@pytest.fixture(scope="module")
def eng():
    from cnmf_b200.engine import Engine
    return Engine(0)


@pytest.fixture(scope="module")
def X():
    return load_golden("sim_mu")["X"]


def same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def _device_paths(ds, ks, kw, starts):
    """(spectra, n_iter, err) of factorize_dev from the device starts `starts` (Wt, H as torch tensors); checks that
    factorize_dev writes whole padded rows, the padding columns as zeros."""
    import torch
    Wt, H = starts
    g = ds.shape[1]
    out = torch.full_like(H, float("nan"))
    n_iter, err = ds.factorize_dev(ks, Wt.data_ptr(), H.data_ptr(), out.data_ptr(), kw)
    o = out.cpu().numpy()
    assert not o[:, g:].any(), "factorize_dev: padding columns of the spectra slab are not zero"
    return o[:, :g], n_iter, err


def _starts(ds, ks, seeds, init):
    import torch
    ld_r, ld_c = ds.ld()
    SK = int(np.sum(ks))
    Wt = torch.full((SK, ld_r), 7.0, dtype=torch.float32, device="cuda:0")
    H = torch.full((SK, ld_c), 7.0, dtype=torch.float32, device="cuda:0")
    if init == "random":
        ds.random_init_dev(ks, seeds, Wt.data_ptr(), H.data_ptr())
    else:
        ds.nndsvd_init_dev(ks, seeds, init, Wt.data_ptr(), H.data_ptr())
    return Wt, H


def _assert_same(ref, got, what):
    sp_ref, it_ref, err_ref = ref
    sp, it, err = got
    assert same_bits(np.asarray(sp, np.float32), sp_ref), what + ": spectra differ"
    assert np.array_equal(it, it_ref), (what, it, it_ref)
    assert same_bits(np.asarray(err, np.float64), np.asarray(err_ref, np.float64)), (what, err, err_ref)


@pytest.mark.parametrize("ks_tag", sorted(KS))
@pytest.mark.parametrize("solver", ["mu", "cd"])
@pytest.mark.parametrize("precision", ["f16x2", "tf32x3", "tf32x3-general", "fp32"])
def test_random_start_paths_agree(eng, X, precision, solver, ks_tag):
    import torch
    ks = np.array(KS[ks_tag], np.int32)
    seeds = np.array([11, 2 ** 31 - 2, 59886188, 7][:len(ks)], np.uint32)
    ds = eng.dataset(X, precision=precision)
    n, g = ds.shape
    kw = dict(solver=solver, tol=1e-4, max_iter=300)
    sp, _, n_iter, err = ds.factorize(ks, seeds, kw)
    ref = (np.vstack(sp), n_iter, err)

    Wt, H = _starts(ds, ks, seeds, "random")
    _assert_same(ref, _device_paths(ds, ks, kw, (Wt, H)), "random_init_dev + factorize_dev")

    W0, H0 = Wt.cpu().numpy()[:, :n], H.cpu().numpy()[:, :g]
    sp_i, _, it_i, err_i = ds.factorize(ks, seeds, kw, W0=W0, H0=H0)
    _assert_same(ref, (np.vstack(sp_i), it_i, err_i), "factorize_init")

    ld_out = g + 3                                  # any row stride >= n_cols; the columns past n_cols stay untouched
    slab = torch.full((int(ks.sum()), ld_out), float("nan"), dtype=torch.float32, device="cuda:0")
    it_s, err_s = ds.factorize_seeds_dev(ks, seeds, slab.data_ptr(), ld_out, kw)
    s = slab.cpu().numpy()
    assert np.isnan(s[:, g:]).all()
    _assert_same(ref, (s[:, :g], it_s, err_s), "factorize_seeds_dev")


@pytest.mark.parametrize("solver", ["mu", "cd"])
@pytest.mark.parametrize("precision", ["f16x2", "tf32x3-general"])
def test_nndsvd_start_paths_agree(eng, X, precision, solver):
    ks = np.array([4, 18, 6], np.int32)
    seeds = np.array([59886188, 1812018521, 3], np.uint32)
    ds = eng.dataset(X, precision=precision)
    kw = dict(solver=solver, tol=1e-4, max_iter=300, init="nndsvd")
    sp, _, n_iter, err = ds.factorize(ks, seeds, kw)
    ref = (np.vstack(sp), n_iter, err)
    starts = _starts(ds, ks, seeds, "nndsvd")
    _assert_same(ref, _device_paths(ds, ks, kw, starts), "nndsvd_init_dev + factorize_dev")


def test_kl_start_paths_agree(eng):
    """KL on a tf32x3 dataset: the streaming beta-divergence solve reads no operand pieces."""
    X = load_golden("sim_kl")["X"]
    ks = np.array([4, 20, 5], np.int32)
    seeds = np.array([59886188, 1812018521, 1173234957], np.uint32)
    ds = eng.dataset(X, precision="tf32x3")
    n, g = ds.shape
    kw = dict(solver="mu", tol=1e-4, max_iter=200, beta_loss="kullback-leibler")
    sp, _, n_iter, err = ds.factorize(ks, seeds, kw)
    ref = (np.vstack(sp), n_iter, err)
    Wt, H = _starts(ds, ks, seeds, "random")
    _assert_same(ref, _device_paths(ds, ks, kw, (Wt, H)), "random_init_dev + factorize_dev")
    sp_i, _, it_i, err_i = ds.factorize(ks, seeds, kw, W0=Wt.cpu().numpy()[:, :n], H0=H.cpu().numpy()[:, :g])
    _assert_same(ref, (np.vstack(sp_i), it_i, err_i), "factorize_init")
