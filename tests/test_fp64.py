"""precision='fp64': float64 datasets, factorize and refits in float64 on the fp64 tensor cores.

CPU tests (unmarked): the precision code, the CLI option, and the refusals of what fp64 does not cover, all raised
before any device work.  GPU tests (`-m gpu`) hold the float64 path to float64 references: the oracle's solvers after
1 and 10 iterations (1e-12), the reference's own fixtures (1e-9, with no exemption) and its sampled BASELINE runs
(1e-7: the stored spectra are the float64 result rounded to float32).
"""
import os

import numpy as np
import pytest

from cnmf_golden import load_golden

gpu = pytest.mark.gpu


def rel(a, b):
    a = np.asarray(a, dtype=np.float64)
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


# ------------------------------------------------------------------------------------ CPU
def test_precision_code_fp64():
    from cnmf_b200 import _lib
    from cnmf_b200.engine import make_params, precision_code
    assert precision_code("fp64") == _lib.PRECISION_FP64 == 4
    assert precision_code(4) == 4
    p = make_params(dict(solver="cd"), 100, 50, "fp64")
    assert p.precision == 4


def test_cli_accepts_precision_fp64():
    from cnmf_b200.pipeline import build_parser
    args = build_parser().parse_args(["factorize", "--output-dir", "x", "--name", "y", "--precision", "fp64"])
    assert args.precision == "fp64"


@pytest.mark.parametrize("beta_loss", ["kullback-leibler", "itakura-saito", 1, 0])
def test_fp64_refuses_kl_is(beta_loss):
    from cnmf_b200.engine import make_params
    with pytest.raises(NotImplementedError, match="fp64"):
        make_params(dict(solver="mu", beta_loss=beta_loss), 100, 50, "fp64")


def test_fp64_refuses_host_rng():
    from cnmf_b200.engine import make_params
    with pytest.raises(NotImplementedError, match="fp64"):
        make_params(dict(solver="mu", rng="host"), 100, 50, "fp64")


class _NoDeviceEngine:
    """Stands in for an Engine: any device work fails the test; the dense-size query answers 'does not fit'."""

    def mem_info(self):
        return 0, 0, 0

    def dense_dataset_bytes(self, n_rows, n_cols, precision):
        return 1

    def dataset(self, *a, **k):
        raise AssertionError("device work before the refusal")

    sparse_dataset = dataset


def test_fp64_refusals_before_device_work(tmp_path):
    """Each combination fp64 does not cover raises where the user states it, before any device work."""
    from cnmf_b200 import cNMF, parallel
    from cnmf_b200.engine import Engine
    from cnmf_b200.pipeline import tpm_dataset
    with pytest.raises(NotImplementedError, match="fp64"):            # sparse datasets
        Engine.sparse_dataset(None, np.zeros((2, 2)), precision="fp64")
    with pytest.raises(NotImplementedError, match="fp64"):            # a TPM that does not fit dense
        tpm_dataset(_NoDeviceEngine(), np.zeros((4, 3)), "fp64")
    c = cNMF(output_dir=str(tmp_path), name="run", precision="fp64")
    c._engine = _NoDeviceEngine()
    missing = str(tmp_path / "no_such_counts.npz")                    # refused before the counts are read
    with pytest.raises(NotImplementedError, match="fp64"):            # KL / IS
        c.prepare(missing, components=[3], beta_loss="kullback-leibler")
    with pytest.raises(NotImplementedError, match="fp64"):            # device-side prepare
        c.prepare(missing, components=[3], on_device=True)

    class _Ds:
        fp64 = True
    with pytest.raises(NotImplementedError, match="fp64"):            # the torchrun sharded path
        parallel.factorize_sharded(_Ds(), [3], [1], dict(solver="cd"))


def test_fp64_dense_sizes():
    """fits_dense / plan_groups see 8 bytes per entry of a float64 dataset (X64 only, no transposed copy)."""
    from cnmf_b200.engine import Engine
    eng = Engine.__new__(Engine)
    from cnmf_b200 import _lib
    eng.lib = _lib.load()
    assert eng.dense_dataset_bytes(1000, 500, "fp64") == 8 * 1000 * 512
    assert eng.dense_dataset_bytes(1000, 500, "fp32") == 4 * 1000 * 512 + 4 * 500 * 1024


# ------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def eng():
    from cnmf_b200.engine import Engine
    return Engine(0)


def _packed_starts(X, ks, seeds):
    """The oracle's float64 random starts of every restart, packed (W^T rows, H rows)."""
    from oracle import nmf_ref
    Ws, Hs = [], []
    for k, seed in zip(ks, seeds):
        W, H = nmf_ref.init_random(X.mean(), X.shape[0], X.shape[1], int(k), int(seed))
        Ws.append(W.T)
        Hs.append(H)
    return np.vstack(Ws), np.vstack(Hs)


@gpu
@pytest.mark.parametrize("solver", ["mu", "cd"])
@pytest.mark.parametrize("max_iter", [1, 10])
@pytest.mark.parametrize("reg", [False, True])
def test_half_steps_every_k_against_oracle(eng, solver, max_iter, reg):
    """factorize_init from the oracle's starts, K = 1..32 in one batch: each restart within 1e-12 of the float64
    oracle after 1 and 10 iterations, identical n_iter."""
    from oracle import nmf_ref
    g = load_golden("sim_mu")
    X = g["X"]
    n, G = X.shape
    ks = np.arange(1, 33)
    seeds = 1000 + ks
    W0, H0 = _packed_starts(X, ks, seeds)
    kw = dict(solver=solver, tol=1e-4, max_iter=max_iter)
    if reg:
        kw.update(alpha_W=0.02, alpha_H=0.01, l1_ratio=0.3)
    l1W, l2W, l1H, l2H = nmf_ref.reg_terms(n, G, kw.get("alpha_W", 0.0), kw.get("alpha_H", 0.0),
                                           kw.get("l1_ratio", 0.0))
    ds = eng.dataset(X, precision="fp64")
    sp, us, n_iter, err = ds.factorize(ks, seeds, kw, return_usages=True, W0=W0, H0=H0)
    assert sp[0].dtype == np.float64
    fn = nmf_ref.mu_frobenius if solver == "mu" else nmf_ref.cd_frobenius
    o = 0
    for r, k in enumerate(ks):
        W, H, it = fn(X, W0[o:o + k].T.copy(), H0[o:o + k].copy(), tol=1e-4, max_iter=max_iter, l1_reg_W=l1W,
                      l2_reg_W=l2W, l1_reg_H=l1H, l2_reg_H=l2H)
        o += k
        assert it == int(n_iter[r]), (k, it, int(n_iter[r]))
        assert rel(sp[r], H) < 1e-12, (k, rel(sp[r], H))
        assert rel(us[r], W) < 1e-12, (k, rel(us[r], W))


def _fixture_run(eng, tag, device_starts=True):
    g = load_golden(tag)
    ds = eng.dataset(g["X"], precision="fp64")
    kw = dict(solver=g["solver"], tol=1e-4, max_iter=1000, beta_loss=2.0 if g["solver"] == "mu" else "frobenius",
              init=g["init"])
    t = g["table"]
    out = ds.factorize(t[:, 0], t[:, 2], kw, return_usages=True, X_host=None if device_starts else g["X"])
    return g, out


@gpu
@pytest.mark.parametrize("tag,device_starts", [("sim_mu", True), ("sim_cd", True), ("sim_nndsvd", True),
                                               ("sim_nndsvd", False), ("c1_mu", True), ("c1_cd", True)])
def test_factorize_matches_reference_fixture_fp64(eng, tag, device_starts):
    """Every restart of the reference's own factorize(): identical n_iter and spectra within 1e-9 -- sim_mu K = 4
    iter 0 included, which the float precisions cannot hold to 1e-4.  err = ||X - WH||_F of the returned factors."""
    from oracle import nmf_ref
    g, (sp, us, n_iter, err) = _fixture_run(eng, tag, device_starts)
    for r, (k, it, seed) in enumerate(g["table"]):
        ref = g["merged_k%d" % k][it * k:(it + 1) * k]
        e = rel(sp[r], ref)
        assert e < 1e-9, (tag, k, it, e)
        _, _, n_o = nmf_ref.nmf(g["X"], int(k), int(seed), solver=g["solver"], init=g["init"])
        assert n_o == int(n_iter[r]), (tag, k, it, n_o, int(n_iter[r]))
        e_true = nmf_ref.frobenius_error(g["X"], us[r], sp[r])
        assert abs(err[r] - e_true) / e_true < 1e-12, (tag, k, it, err[r], e_true)


def _big_samples():
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "big_samples.npz"))
    return {key[2:]: (z[key], int(z["it_" + key[2:]]), z["meta_" + key[2:]]) for key in z.files if key.startswith("H_")}


@gpu
@pytest.mark.parametrize("case", ["c2", "c3", "k20", "k30"])
def test_factorize_baseline_configs_sampled_fp64(eng, case):
    """The sampled BASELINE restarts, each in a mixed batch with neighbours from its job table: identical n_iter,
    spectra within 1e-7 of the reference's float64 result (stored rounded to float32: 6e-8)."""
    from oracle.make_golden_big import case_inputs
    X, table = case_inputs(case)
    lookup = {(k, it): seed for k, it, seed in table}
    samples = {t: v for t, v in _big_samples().items() if t.startswith(case + "_")}
    assert samples
    ds = eng.dataset(X, precision="fp64")
    for solver in ("mu", "cd"):
        want = [(t, v) for t, v in samples.items() if t.endswith("_" + solver)]
        if not want:
            continue
        jobs = [(int(v[2][2]), int(v[2][3])) for _, v in want]
        extra = [(k, it) for (k, it, _) in table[1::max(1, len(table) // 6)] if (k, it) not in jobs][:5]
        batch = jobs + extra
        kw = dict(solver=solver, tol=1e-4, max_iter=1000, beta_loss=2.0 if solver == "mu" else "frobenius")
        sp, _, n_iter, _ = ds.factorize([k for k, _ in batch], [lookup[j] for j in batch], kw)
        for i, (t, (H, it_ref, meta)) in enumerate(want):
            assert meta[4] == lookup[jobs[i]]
            assert int(n_iter[i]) == it_ref, (t, int(n_iter[i]), it_ref)
            assert rel(sp[i], H) < 1e-7, (t, rel(sp[i], H))


@gpu
@pytest.mark.parametrize("solver", ["mu", "cd"])
def test_batch_invariance_fp64(eng, solver):
    """A restart alone, in a 6-restart batch, and among neighbours that converge first and force compaction:
    bit-identical spectra and n_iter."""
    g = load_golden("sim_mu")
    ds = eng.dataset(g["X"], precision="fp64")
    t = g["table"]
    kw = dict(solver=solver, tol=1e-4, max_iter=400)
    sp1, _, it1, _ = ds.factorize(t[3:4, 0], t[3:4, 2], kw)
    sp6, _, it6, _ = ds.factorize(t[:6, 0], t[:6, 2], kw)
    assert it1[0] == it6[3] and np.array_equal(sp1[0], sp6[3])
    # neighbours with a loose tolerance stop at iteration 10 / 4 and leave the packed arrays; ours keeps going
    ks = [int(t[3, 0])] + [32] * 8
    seeds = [int(t[3, 2])] + list(range(50, 58))
    spm, _, itm, _ = ds.factorize(ks, seeds, dict(kw, max_iter=400))
    assert itm[0] == it1[0] and np.array_equal(spm[0], sp1[0])
    spc, _, itc, _ = ds.factorize([int(t[3, 0]), 32, 32, 32], [int(t[3, 2]), 7, 8, 9], dict(kw, max_iter=400))
    assert itc[0] == it1[0] and np.array_equal(spc[0], sp1[0])


@gpu
@pytest.mark.parametrize("solver", ["mu", "cd"])
@pytest.mark.parametrize("k", [1, 9, 32])
def test_refit_and_projection_fp64(eng, solver, k):
    """refit (both orientations) against the oracle's float64 refit; project_rows and col_stats against numpy."""
    from oracle import nmf_ref
    g = load_golden("sim_mu")
    X = g["X"]
    n, G = X.shape
    ds = eng.dataset(X, precision="fp64")
    rng = np.random.RandomState(k)
    H = np.abs(rng.randn(k, G))
    W, it, err = ds.refit(H, dict(solver=solver, tol=1e-4, max_iter=1000))
    assert W.dtype == np.float64
    W_ref, it_ref = nmf_ref.refit(X, H, solver=solver)
    assert it == it_ref and rel(W, W_ref) < 1e-9, (it, it_ref, rel(W, W_ref))
    Wt = np.abs(rng.randn(k, n))
    Ht, it, _ = ds.refit(Wt, dict(solver=solver, tol=1e-4, max_iter=1000), transposed=True)
    Ht_ref, it_ref = nmf_ref.refit(X.T, Wt, solver=solver)
    assert it == it_ref and rel(Ht, Ht_ref) < 1e-9, (it, it_ref, rel(Ht, Ht_ref))
    Ut = rng.randn(k, n)
    assert rel(ds.project_rows(Ut), Ut @ X) < 1e-13
    mean, var = ds.col_stats()
    assert rel(mean, X.mean(axis=0)) < 1e-13 and rel(var, X.var(axis=0)) < 1e-13
    s, q = ds.sums()
    assert abs(s - X.sum()) / X.sum() < 1e-13 and abs(q - (X ** 2).sum()) / (X ** 2).sum() < 1e-13


@gpu
def test_from_columns_f64_is_host_division(eng):
    g = load_golden("sim_mu")
    tpm = g["tpm"]
    ds = eng.dataset(tpm, precision="fp64")
    idx = np.ascontiguousarray(g["hvg_idx"], dtype=np.int32)
    std = tpm[:, idx].std(axis=0, ddof=0)
    sub = ds.from_columns_div(idx, std)
    Ut = np.eye(sub.shape[0])
    assert np.array_equal(sub.project_rows(Ut), tpm[:, idx] / std)


@gpu
def test_nndsvd_starts_fp64_match_host(eng):
    """The device NNDSVD starts of a float64 dataset against cnmf_b200.nndsvd on the host: one MU step from each
    agrees within 1e-10."""
    from cnmf_b200.engine import nndsvd_starts
    g = load_golden("sim_nndsvd")
    X = g["X"]
    ds = eng.dataset(X, precision="fp64")
    t = g["table"]
    for init in ("nndsvd", "nndsvda", "nndsvdar"):
        kw = dict(solver="mu", tol=1e-4, max_iter=1, init=init)
        sp_d, us_d, _, _ = ds.factorize(t[:, 0], t[:, 2], kw, return_usages=True)
        W0, H0 = nndsvd_starts(X, t[:, 0], t[:, 2], init, dtype=np.float64)
        sp_h, us_h, _, _ = ds.factorize(t[:, 0], t[:, 2], kw, return_usages=True, W0=W0, H0=H0)
        for r in range(len(t)):
            assert rel(sp_d[r], sp_h[r]) < 1e-10, (init, r, rel(sp_d[r], sp_h[r]))
            assert rel(us_d[r], us_h[r]) < 1e-10, (init, r, rel(us_d[r], us_h[r]))


@gpu
def test_entry_points_refuse_the_other_dataset_kind(eng):
    from cnmf_b200._lib import CnmfError
    g = load_golden("sim_mu")
    d32 = eng.dataset(g["X"])
    d64 = eng.dataset(g["X"], precision="fp64")
    H = np.abs(np.random.RandomState(0).randn(3, g["X"].shape[1]))
    with pytest.raises(CnmfError, match="cnmf_refit_f64"):
        _call_refit32(d64, H)
    with pytest.raises(CnmfError, match="cnmf_project_rows"):
        _call_project64(d32, np.ones((3, g["X"].shape[0])))


def _call_refit32(ds, H):
    import ctypes
    from cnmf_b200 import _lib
    from cnmf_b200.engine import make_params
    H = _lib.f32c(H)
    p = make_params(dict(solver="mu"), ds.shape[0], ds.shape[1], "tf32x3", for_refit=True)
    out = np.empty((ds.shape[0], H.shape[0]), np.float32)
    _lib.check(ds.lib.cnmf_refit(ds._d, 0, H.shape[0], _lib.ptr(H), ctypes.byref(p), _lib.ptr(out), None, None, None))


def _call_project64(ds, Ut):
    from cnmf_b200 import _lib
    Ut = _lib.f64c(Ut)
    out = np.empty((Ut.shape[0], ds.shape[1]))
    _lib.check(ds.lib.cnmf_project_rows_f64(ds._d, Ut.shape[0], _lib.ptr(Ut), _lib.ptr(out), None))


@gpu
@pytest.mark.parametrize("tag", ["sim_mu", "sim_cd", "c1_cd"])
def test_pipeline_fp64_matches_reference_outputs(tmp_path, tag):
    """cNMF(precision='fp64'): prepare -> factorize -> combine -> consensus.  Merged spectra within 1e-9 of the
    reference's; every consensus file within 1e-5 -- sim_mu K = 4 included.  The consensus kernels (distances, KMeans,
    medians) compare the spectra in float32, which is what bounds these files."""
    import warnings
    import pandas as pd
    from cnmf_b200 import cNMF, load_df_from_npz, save_df_to_npz
    g = load_golden(tag)
    counts = g["counts"].astype(np.float64)
    df = pd.DataFrame(counts, index=["c%d" % i for i in range(counts.shape[0])],
                      columns=["g%d" % i for i in range(counts.shape[1])])
    fn = str(tmp_path / "counts.df.npz")
    save_df_to_npz(df, fn)
    obj = cNMF(output_dir=str(tmp_path), name="run", precision="fp64")
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        obj.prepare(fn, components=list(g["ks"]), n_iter=int(g["n_iter"]), seed=int(g["seed"]), densify=True,
                    beta_loss=g["beta_loss_arg"], num_highvar_genes=len(g["hvg_idx"]), init=g["init"])
        obj.factorize()
        obj.combine()
        dt = float(g["dt"])
        for k in g["ks"]:
            k = int(k)
            merged = load_df_from_npz(obj.paths["merged_spectra"] % k)
            e = rel(merged.values, g["merged_k%d" % k])
            assert e < 1e-9, (tag, k, e)
            obj.consensus(k, density_threshold=dt, show_clustering=False)
            dts = str(dt).replace(".", "_")
            for key, name in (("consensus_spectra", "cspectra"), ("consensus_usages", "cusages"),
                              ("gene_spectra_tpm", "tpmspec"), ("gene_spectra_score", "score"),
                              ("starcat_spectra", "starcat")):
                got = load_df_from_npz(obj.paths[key] % (k, dts)).values
                e = rel(got, g["%s_k%d" % (name, k)])
                assert e < 1e-5, (tag, k, key, e)
