"""The NMF step's kernels one launch at a time (`-m gpu`), through the cnmf_update_step_host / cnmf_gemm_abt_host test
hooks, against the float64 references of oracle/kernel_ref.py -- at every K from 1 to 32, in both register classes
(kp = 16: every K <= 16; kp = 32: a K > 16 restart in the batch), ragged n, split-K products, both operand-piece forms
-- and bit for bit where the solver's batch independence rests on equal bits (DESIGN.md section 2).

u = 2^-24 is the unit roundoff of fp32.
"""
import numpy as np
import pytest

from oracle import kernel_ref as kr

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
TOL_GEMM = 2e-6          # fp32-class GEMM vs float64, as in test_gpu_parity.py
SENTINEL = -12345.0

KP16_ALL = list(range(1, 17))
KP32_ALL = list(range(1, 33))
MIXED = [1, 17, 32, 3, 12, 16, 21, 28]


@pytest.fixture(scope="module")
def eng():
    from cnmf_b200.engine import Engine
    return Engine(0)


def ld_of(n):
    return -(-n // 32) * 32


def offsets(ks):
    return np.concatenate([[0], np.cumsum(ks)]).astype(int)


def gram_blocks(rng, n_rids, symmetric=True, m=48):
    """Per rid a 32 x 32 positive Gram-like block: unit diagonal plus coupling of about 1/32 per pair (enough that a
    Jacobi order of the CD sweep moves every coordinate after the first by far more than the tolerance)."""
    out = np.zeros((n_rids, 32, 32))
    for r in range(n_rids):
        P = rng.uniform(0, 1, (32, m))
        Q = P if symmetric else rng.uniform(0, 1, (32, m))
        out[r] = np.eye(32) + (P @ Q.T) / (8 * m)
    return out


def make_batch(ks, n, nsplit, solver, seed, rids=None, symmetric=True, piece_scale=False):
    """Packed fp32 data of one launch.  Product columns >= n hold garbage (the GEMM leaves them undefined); factor
    padding is zero (the layout's invariant)."""
    rng = np.random.RandomState(seed)
    ks = list(ks)
    R, SK, ld = len(ks), sum(ks), ld_of(n)
    rids = np.arange(R) if rids is None else np.asarray(rids)
    n_rids = int(rids.max()) + 1
    off = offsets(ks)
    F = np.zeros((SK, ld), np.float32)
    F[:, :n] = rng.uniform(0.1, 2.0, (SK, n))
    gin = gram_blocks(rng, n_rids, symmetric)
    num = np.zeros((nsplit, SK, ld), np.float32)
    w = rng.dirichlet(np.ones(nsplit), size=(SK, n)).transpose(2, 0, 1)       # positive split-K slices
    if solver == "mu":
        num[:, :, :n] = w * rng.uniform(0.05, 1.5, (SK, n))
    else:
        F[:, :n][rng.rand(SK, n) < 0.1] = 0.0                                  # the projected gradient's min(0, g)
        for s, (k, r) in enumerate(zip(ks, rids)):
            target = rng.uniform(-0.3, 1.5, (k, n))                            # negative targets: clipped at 0
            num[:, off[s]:off[s + 1], :n] = w[:, off[s]:off[s + 1]] * (gin[r, :k, :k] @ target)
    num[:, :, n:] = 7.0
    ps = None
    if piece_scale:
        ps = np.zeros(ld, np.float32)
        ps[:n] = 2.0 ** rng.randint(-3, 4, n) * rng.uniform(1, 2, n)
    return dict(ks=ks, rids=rids, n_rids=n_rids, off=off, n=n, F=F, num=num, gin=gin, ps=ps)


def run(eng, b, solver, done=None, **kw):
    done = np.zeros(b["n_rids"], np.int32) if done is None else done
    return eng.update_step(b["ks"], b["rids"], done, b["n"], b["F"], b["num"], b["gin"], solver=solver,
                           piece_scale=b["ps"], **kw)


def kp_of(ks):
    return 16 if max(ks) <= 16 else 32


def check_padding(b, out):
    n = b["n"]
    assert not out["F"][:, n:].any(), "factor padding columns must stay exactly 0"
    for p in ("hi", "lo"):
        if out[p] is not None:
            assert not out[p][:, n:].astype(np.float32).any(), "piece padding columns must stay exactly 0"


# ------------------------------------------------------------------------------------------------ MU
# l1, l2 are fp32-representable: the kernels take them as floats, the references as given
MU_CASES = [  # n, nsplit, pieces, piece_scale, (l1, l2), symmetric Gram, cpb_tiles
    (1, 1, None, False, (0.0, 0.0), True, 1),
    (3, 3, "tf32", True, (0.125, 0.25), False, 2),
    (511, 1, "f16", True, (0.0, 0.0), True, 1),
    (513, 3, "tf32", False, (0.0625, 0.0), False, 4),
    (2049, 1, None, False, (0.0, 0.375), False, 2),
    (2049, 3, "f16", False, (0.25, 0.125), True, 4),
]


def mu_check(b, out, l1, l2, nsplit):
    """MU per entry: den is a chain of K fp32 FMAs over non-negative terms (K roundings) plus l1 and l2 F (2), the
    product is the fp32 sum of nsplit non-negative slices (nsplit - 1), the Newton quotient is within 2 ulp (2), and the
    final multiply rounds once (1): |F - ref| <= (K + nsplit + 4) u |ref| to first order, with no cancellation
    anywhere.  (A factor 1 + 1e-6 covers the second-order terms.)"""
    num64 = b["num"].astype(np.float64).sum(axis=0)
    for s, (k, r) in enumerate(zip(b["ks"], b["rids"])):
        rows = slice(b["off"][s], b["off"][s + 1])
        G = kr.gram_fp32(b["gin"][r], k)
        ref = kr.mu_half_step(b["F"][rows, :b["n"]], num64[rows, :b["n"]], G, l1, l2)
        got = out["F"][rows, :b["n"]].astype(np.float64)
        bound = (k + nsplit + 4) * U * (1 + 1e-6) * np.abs(ref)
        bad = np.abs(got - ref) > bound
        assert not bad.any(), ("MU", k, int(bad.sum()), float((np.abs(got - ref) / np.maximum(ref, 1e-300)).max()))


@pytest.mark.parametrize("case", MU_CASES, ids=lambda c: "n%d-s%d-%s" % (c[0], c[1], c[2]))
def test_mu_update_against_float64_every_k(eng, case):
    n, nsplit, pieces, ps, (l1, l2), sym, cpb = case
    for ks, gram in ((KP16_ALL, "fused"), (KP16_ALL, None), (KP32_ALL, "standalone"), (MIXED, None)):
        b = make_batch(ks, n, nsplit, "mu", seed=n + nsplit + len(ks), symmetric=sym, piece_scale=ps)
        out = run(eng, b, "mu", pieces=pieces, gram=gram, want_scalar=True, cpb_tiles=cpb, l1=l1, l2=l2)
        mu_check(b, out, l1, l2, nsplit)
        check_padding(b, out)


def test_mu_zero_denominator_takes_eps(eng):
    """A zero Gram row with l1 = l2 = 0 gives den = 0 exactly: the kernel divides by float32 eps, like scikit-learn."""
    for ks, gram in ((MIXED, None), ([3, 12, 16], "fused")):
        bb = make_batch(ks, 513, 1, "mu", seed=5)
        bb["gin"][:, 2, :] = 0.0
        out = run(eng, bb, "mu", gram=gram)
        mu_check(bb, out, 0.0, 0.0, 1)


# ------------------------------------------------------------------------------------------------ CD
CD_CASES = [  # n, nsplit, pieces, piece_scale, (l1, l2), cpb_tiles
    (1, 1, None, False, (0.0, 0.0), 1),
    (3, 3, "tf32", True, (0.125, 0.25), 2),
    (511, 1, "f16", False, (0.0, 0.5), 1),
    (513, 3, None, False, (0.0625, 0.0), 4),
    (2049, 1, "tf32", False, (0.25, 0.125), 2),
]


def cd_check(b, out, l1, l2, vec_of_kp, nsplit=1, viol=True):
    """CD, per restart: rel-L2 <= 1e-6, and every entry within the bound of its own arithmetic.  The gradient g of
    coordinate t is l1 - num (num: fp32 sum of nsplit same-signed slices) plus a chain of K fp32 FMAs, so its error is
    <= (K + 1 + nsplit) u mag (mag = |num - l1| + sum |G F|) plus sum_{r<t} |G[t, r]| |dF_r| from the coordinates the
    device already moved differently; the Newton quotient by h = G[t, t] adds 2 u |g / h| <= 2 u mag / h and
    F - g / h one rounding, u (|F| + mag / h):
        |dF_t| <= ((K + 4 + nsplit) u mag + sum_{r<t} |G[t, r]| |dF_r|) / h + u |F_old|   (doubled: second order).
    (An entry-relative bound cannot work: F - g / h cancels for coordinates the sweep drives towards 0.)  h = 0 leaves
    the coordinate alone: dF = 0.  The violation adds |projected gradient| over coordinates in fp32 over the K VEC terms
    of a thread's items and in fp64 beyond: |viol - ref| <= (K + 2 + K VEC) u sum mag + sum |G| |dF|, doubled."""
    num64 = b["num"].astype(np.float64).sum(axis=0)
    n = b["n"]
    for s, (k, r) in enumerate(zip(b["ks"], b["rids"])):
        rows = slice(b["off"][s], b["off"][s + 1])
        G = kr.gram_fp32(b["gin"][r], k, diag_add=l2)
        F0 = b["F"][rows, :n].astype(np.float64)
        ref, vref, mag = kr.cd_sweep(F0, num64[rows, :n], G, l1, 0.0)
        got = out["F"][rows, :n].astype(np.float64)
        d = np.abs(got - ref)
        if np.linalg.norm(ref) > 0:
            assert np.linalg.norm(d) <= 1e-6 * np.linalg.norm(ref), ("CD rel-L2", k, np.linalg.norm(d) / np.linalg.norm(ref))
        lower = np.tril(np.abs(G), -1)                              # |G[t, r]| for r < t
        h = np.abs(np.diag(G))[:, None]
        with np.errstate(divide="ignore", invalid="ignore"):
            bound = np.where(h > 0, 2 * (((k + 4 + nsplit) * U * mag + lower @ d) / h + U * np.abs(F0)), 0.0)
        assert (d <= bound).all(), ("CD entry", k, float(np.max(d - bound)))
        if viol:
            vec = vec_of_kp
            bound = 2 * ((k + 2 + k * vec) * U * mag.sum() + (lower @ d).sum())
            assert abs(out["scal"][r] - vref) <= bound, ("CD violation", k, out["scal"][r], vref, bound)


@pytest.mark.parametrize("case", CD_CASES, ids=lambda c: "n%d-s%d-%s" % (c[0], c[1], c[2]))
def test_cd_update_against_float64_every_k(eng, case):
    n, nsplit, pieces, ps, (l1, l2), cpb = case
    for ks, gram in ((KP16_ALL, "fused"), (KP16_ALL, None), (KP32_ALL, "standalone"), (MIXED, None)):
        b = make_batch(ks, n, nsplit, "cd", seed=3 * n + nsplit + len(ks), piece_scale=ps)
        out = run(eng, b, "cd", pieces=pieces, gram=gram, want_scalar=True, cpb_tiles=cpb, l1=l1, l2=l2)
        cd_check(b, out, l1, l2, 4 if kp_of(ks) == 16 else 2, nsplit)
        check_padding(b, out)


def test_cd_is_gauss_seidel_and_zero_diagonal_is_left_alone(eng):
    """The fixtures couple the coordinates strongly enough that a Jacobi order of the sweep lands far outside the
    tolerance; a zero Gram diagonal (l2 = 0) leaves its coordinate bitwise unchanged."""
    for ks in (KP16_ALL, MIXED):
        b = make_batch(ks, 2049, 1, "cd", seed=11)
        b["gin"][:, 5, 5] = 0.0
        out = run(eng, b, "cd", want_scalar=True)
        cd_check(b, out, 0.0, 0.0, 4 if kp_of(ks) == 16 else 2)
        num64 = b["num"].astype(np.float64).sum(axis=0)
        for s, (k, r) in enumerate(zip(b["ks"], b["rids"])):
            rows = slice(b["off"][s], b["off"][s + 1])
            if k > 5:
                assert np.array_equal(out["F"][b["off"][s] + 5], b["F"][b["off"][s] + 5])
            if k >= 4:
                G = kr.gram_fp32(b["gin"][r], k)
                gs, _, _ = kr.cd_sweep(b["F"][rows, :b["n"]], num64[rows, :b["n"]], G)
                jac, _, _ = kr.cd_sweep(b["F"][rows, :b["n"]], num64[rows, :b["n"]], G, jacobi=True)
                assert np.linalg.norm(jac - gs) > 100 * 1e-6 * np.linalg.norm(gs)


# ------------------------------------------------------------------------------------------------ exact bits
def test_streamed_and_rolled_mu_bodies_give_the_same_bits(eng):
    """A MU refit alternates between the streamed body (Gram-fused launches) and the rolled one (no Gram)."""
    for n, nsplit, pieces in ((2049, 1, None), (513, 3, "tf32"), (3, 1, "tf32")):
        b = make_batch(KP16_ALL, n, nsplit, "mu", seed=n, piece_scale=True)
        a = run(eng, b, "mu", pieces=pieces, gram="fused", want_scalar=True)
        c = run(eng, b, "mu", pieces=pieces, gram=None, want_scalar=True)
        assert np.array_equal(a["F"], c["F"])
        if pieces:
            assert np.array_equal(a["hi"], c["hi"]) and np.array_equal(a["lo"], c["lo"])


def test_cd_with_and_without_fused_gram_gives_the_same_bits(eng):
    b = make_batch(KP16_ALL, 2049, 3, "cd", seed=2, piece_scale=True)
    a = run(eng, b, "cd", pieces="tf32", gram="fused", want_scalar=True)
    c = run(eng, b, "cd", pieces="tf32", gram=None, want_scalar=True)
    assert np.array_equal(a["F"], c["F"]) and np.array_equal(a["hi"], c["hi"]) and np.array_equal(a["lo"], c["lo"])
    assert np.array_equal(a["scal"], c["scal"])


@pytest.mark.parametrize("solver", ["mu", "cd"])
def test_restart_update_does_not_depend_on_its_batch_class(eng, solver):
    """The same restarts in a kp = 16 batch (Gram-fused, as the solver runs them) and beside a K = 20 restart (kp = 32:
    two items per thread, no fused Gram): the same bits."""
    small = [1, 4, 7, 9, 12, 16]
    b16 = make_batch(small, 2049, 3, solver, seed=4, piece_scale=True)
    b32 = dict(b16)
    extra = make_batch([20], 2049, 3, solver, seed=5)
    b32["ks"] = small + [20]
    b32["off"] = offsets(b32["ks"])
    b32["rids"] = np.arange(len(b32["ks"]))
    b32["n_rids"] = len(b32["ks"])
    b32["F"] = np.vstack([b16["F"], extra["F"]])
    b32["num"] = np.concatenate([b16["num"], extra["num"]], axis=1)
    b32["gin"] = np.concatenate([b16["gin"], extra["gin"][:1]])
    a = run(eng, b16, solver, pieces="tf32", gram="fused", want_scalar=True)
    c = run(eng, b32, solver, pieces="tf32", gram="standalone", want_scalar=True)
    SK = sum(small)
    assert np.array_equal(a["F"], c["F"][:SK])
    assert np.array_equal(a["hi"], c["hi"][:SK]) and np.array_equal(a["lo"], c["lo"][:SK])


@pytest.mark.parametrize("solver", ["mu", "cd"])
def test_blocks_of_one_two_four_tiles_give_the_same_bits(eng, solver):
    """F and pieces are per item: equal bits for any block size.  Gram and scalar are fp64 sums of per-block partials:
    equal up to the fp64 reordering."""
    for ks, pieces, gram in ((KP16_ALL, "f16", "fused"), (MIXED, "tf32", "standalone")):
        b = make_batch(ks, 50003, 1, solver, seed=6, piece_scale=True)
        outs = [run(eng, b, solver, pieces=pieces, gram=gram, want_scalar=True, cpb_tiles=t) for t in (1, 2, 4)]
        for o in outs[1:]:
            assert np.array_equal(o["F"], outs[0]["F"])
            assert np.array_equal(o["hi"], outs[0]["hi"]) and np.array_equal(o["lo"], outs[0]["lo"])
            if pieces == "f16":
                assert np.array_equal(o["tile_scale"], outs[0]["tile_scale"])
            assert np.allclose(o["gram"], outs[0]["gram"], rtol=1e-12, atol=0)
            assert np.allclose(o["scal"], outs[0]["scal"], rtol=1e-12, atol=0)


def test_consecutive_calls_reset_their_tickets(eng):
    """The last-block tickets are never zeroed between calls: the second launch finds the Gram and the scalar only if
    the first one's last block reset them."""
    for solver in ("mu", "cd"):
        b = make_batch(MIXED[:1] + [3, 12, 16], 50003, 1, solver, seed=8)
        first = run(eng, b, solver, gram="fused", want_scalar=True)
        g0 = np.full((b["n_rids"], 32, 32), SENTINEL)
        s0 = np.full(b["n_rids"], SENTINEL)
        second = run(eng, b, solver, gram="fused", want_scalar=True, gram_out=g0, scal_out=s0)
        for key in ("F", "scal"):
            assert np.array_equal(first[key], second[key])
        for s, k in enumerate(b["ks"]):
            kp = -(-k // 4) * 4
            assert np.array_equal(first["gram"][s, :kp, :kp], second["gram"][s, :kp, :kp])


# ------------------------------------------------------------------------------------------------ pieces
def piece_batch(ks, n, seed):
    """MU data whose new factor has rows with 512-column groups 2^40 apart and rows at / below the 2^-111 floor of the
    group scale: F_new = F num / den scales with num."""
    b = make_batch(ks, n, 1, "mu", seed=seed, piece_scale=True)
    SK = sum(ks)
    rows = np.arange(SK)
    b["num"][0, rows % 5 == 1, 512:1024] *= np.float32(2.0 ** -40)
    b["num"][0, rows % 5 == 2, :n] *= np.float32(2.0 ** -113)
    b["num"][0, rows % 5 == 3, :n] *= np.float32(2.0 ** -135)
    return b


@pytest.mark.parametrize("ks", [KP16_ALL, MIXED], ids=["kp16", "kp32"])
def test_pieces_equal_the_numpy_restatement(eng, ks):
    n = 2049
    b = piece_batch(ks, n, seed=9)
    for pieces in ("tf32", "f16"):
        for solver in ("mu", "cd"):
            gram = "fused" if kp_of(ks) == 16 else "standalone"
            out = run(eng, b, solver, pieces=pieces, gram=gram)
            F = out["F"]
            if pieces == "tf32":
                hi, lo = kr.tf32_pieces(F, b["ps"])
                assert np.array_equal(out["hi"].view(np.uint32), hi.view(np.uint32))
                assert np.array_equal(out["lo"].view(np.uint32), lo.view(np.uint32))
            else:
                hi, mid, ts = kr.f16_pieces(F, b["ps"])
                assert np.array_equal(out["tile_scale"], ts)
                assert np.array_equal(out["hi"].view(np.uint16), hi.view(np.uint16))
                assert np.array_equal(out["lo"].view(np.uint16), mid.view(np.uint16))
                # the stand-alone emission (initial factors, compaction, K > 16) on the same F: the same bits
                bb = dict(b, F=F)
                st = run(eng, bb, None, pieces="f16")
                assert np.array_equal(st["F"], F)
                for key in ("hi", "lo", "tile_scale"):
                    assert np.array_equal(st[key], out[key])
            check_padding(b, out)
            if solver == "mu":          # MU keeps the scaled rows small (CD moves them back to O(1))
                ts = kr.f16_pieces(out["F"], b["ps"])[2]
                assert (ts == np.float32(2.0 ** -126)).any()                   # the floor was exercised
                assert (ts[1::5, 0] / ts[1::5, 1] >= 2.0 ** 36).all()          # groups about 2^40 apart


# ------------------------------------------------------------------------------------------------ Gram and scalars
def gram_L(kp, fused):
    """fp32 partial length of one Gram entry: fused (update-kernel tile, 128 threads) -- a lane sums 1, 2 or 4 quads
    of 4 columns at KP 4, 8, 12-16 (the symmetric plan at 12 / 16 gives every warp all 128 quads of the tile); stand-alone
    gram_body -- a thread walks at most 8192 columns in steps of 256 / TPC, TPC = 1, 2, 4, 8 threads per column
    group at KP <= 8, 16, 24, 32, i.e. <= 32 TPC terms."""
    if fused:
        return {4: 4, 8: 8, 12: 16, 16: 16}[kp]
    tpc = 1 if kp <= 8 else 2 if kp <= 16 else 4 if kp <= 24 else 8
    return 32 * tpc


def gram_check(b, out, F, fused):
    for s, (k, r) in enumerate(zip(b["ks"], b["rids"])):
        kp = -(-k // 4) * 4
        Fr = F[b["off"][s]:b["off"][s + 1]].astype(np.float64)
        ref = Fr @ Fr.T
        mag = np.abs(Fr) @ np.abs(Fr).T
        g = out["gram"][r]
        assert np.array_equal(g, g.T), "Gram must be exactly symmetric"
        assert not g[k:kp, :kp].any() and not g[:kp, k:kp].any()
        L = gram_L(kp, fused)
        assert (np.abs(g[:k, :k] - ref) <= (L + 1) * U * mag).all(), ("Gram", k, fused)


@pytest.mark.parametrize("solver", ["mu", "cd"])
def test_fused_and_standalone_gram_against_float64(eng, solver):
    for ks, n in ((KP16_ALL, 2049), ([4, 8, 12, 16], 50003), ([1, 2, 3], 3)):
        b = make_batch(ks, n, 1, solver, seed=12)
        out = run(eng, b, solver, gram="fused")
        gram_check(b, out, out["F"], True)
    for ks, n in ((KP32_ALL, 2049), (MIXED, 50003), ([20, 24, 28, 32], 100003)):
        b = make_batch(ks, n, 1, solver, seed=13)
        out = run(eng, b, solver, gram="standalone")
        gram_check(b, out, out["F"], False)
        st = run(eng, b, None, gram="standalone")               # stand-alone Gram of the initial factors
        gram_check(b, st, b["F"], False)


def test_cross_and_update_scalars_against_float64(eng):
    """<NUM, F> from cross_kernel (fp32 slice sum, fp64 products and sums: (nsplit + 1) u) and from the MU update
    (per thread fp32 over K VEC terms of num * F_new, F_new itself within (K + nsplit + 4) u: all non-negative)."""
    for ks in (KP16_ALL, MIXED):
        vec = 4 if kp_of(ks) == 16 else 2
        for nsplit in (1, 3):
            b = make_batch(ks, 50003, nsplit, "mu", seed=14 + nsplit)
            num64 = b["num"].astype(np.float64).sum(axis=0)
            st = run(eng, b, None, want_scalar=True)
            out = run(eng, b, "mu", want_scalar=True, gram="fused" if vec == 4 else None)
            for s, (k, r) in enumerate(zip(b["ks"], b["rids"])):
                rows = slice(b["off"][s], b["off"][s + 1])
                nn = num64[rows, :b["n"]]
                cref = float((nn * b["F"][rows, :b["n"]]).sum())
                assert abs(st["scal"][r] - cref) <= (nsplit + 1) * U * cref
                Fn = kr.mu_half_step(b["F"][rows, :b["n"]], nn, kr.gram_fp32(b["gin"][r], k))
                uref = float((nn * Fn).sum())
                assert abs(out["scal"][r] - uref) <= (k * vec + k + 2 * nsplit + 6) * U * uref


# ------------------------------------------------------------------------------------------------ bookkeeping
@pytest.mark.parametrize("solver", ["mu", "cd"])
@pytest.mark.parametrize("ks,pieces,gram", [([5, 16, 1, 9, 12], "f16", "fused"), (MIXED, "tf32", "standalone"),
                                            ([5, 16, 1, 9, 12], "tf32", None)], ids=["kp16-f16", "kp32-tf32", "kp16-nogram"])
def test_slots_rids_done_and_sentinels(eng, solver, ks, pieces, gram):
    """Slots permuted against rids, one rid absent from the batch, two restarts frozen: live restarts match the
    reference and put their Gram and scalar at their rid; frozen ones and every entry no launch owns keep the sentinel
    bit for bit."""
    R = len(ks)
    perm = np.random.RandomState(R).permutation(R + 1)
    rids = perm[perm != 2]                                     # rid 2 is not in the batch
    b = make_batch(ks, 2049, 3, solver, seed=15, rids=rids, piece_scale=True)
    done = np.zeros(b["n_rids"], np.int32)
    frozen = [int(rids[1]), int(rids[-1])]
    done[frozen] = 1
    SK, ld = b["F"].shape
    pdt = np.float16 if pieces == "f16" else np.float32
    init = dict(pieces_hi=np.full((SK, ld), -3.0, pdt), pieces_lo=np.full((SK, ld), -3.0, pdt),
                tile_scale=np.full((SK, (ld + 511) // 512), SENTINEL, np.float32),
                gram_out=np.full((b["n_rids"], 32, 32), SENTINEL), scal_out=np.full(b["n_rids"], SENTINEL))
    out = run(eng, b, solver, done=done, pieces=pieces, gram=gram, want_scalar=True, **init)
    live = [s for s in range(R) if int(rids[s]) not in frozen]
    sub = dict(b, ks=[ks[s] for s in live], rids=rids[live], off=None)
    # reference checks of the live restarts, slot by slot
    rows_live = np.concatenate([np.arange(b["off"][s], b["off"][s + 1]) for s in live])
    sub["off"] = offsets(sub["ks"])
    sub["F"] = b["F"][rows_live]
    sub["num"] = b["num"][:, rows_live]
    o2 = dict(out, F=out["F"][rows_live])
    if solver == "mu":
        mu_check(sub, o2, 0.0, 0.0, 3)
    else:
        cd_check(sub, o2, 0.0, 0.0, 4 if kp_of(ks) == 16 else 2, 3)
    for s in range(R):
        rows = slice(b["off"][s], b["off"][s + 1])
        r, k = int(rids[s]), ks[s]
        kp = -(-k // 4) * 4
        if r in frozen:
            assert np.array_equal(out["F"][rows], b["F"][rows])
            assert np.array_equal(out["hi"][rows], init["pieces_hi"][rows])
            assert np.array_equal(out["lo"][rows], init["pieces_lo"][rows])
            if pieces == "f16":
                assert np.array_equal(out["tile_scale"][rows], init["tile_scale"][rows])
            assert (out["gram"][r] == SENTINEL).all() and out["scal"][r] == SENTINEL
        else:
            assert not np.array_equal(out["F"][rows], b["F"][rows])
            assert (out["hi"][rows][:, :b["n"]] != -3.0).all()
            if gram:
                assert (out["gram"][r][:kp, :kp] != SENTINEL).all()
            blk = out["gram"][r].copy()
            if gram:
                blk[:kp, :kp] = SENTINEL
            assert (blk == SENTINEL).all(), "Gram entries outside the restart's KP x KP block are not the launch's"
            assert out["scal"][r] != SENTINEL
    absent = sorted(set(range(b["n_rids"])) - set(int(x) for x in rids))
    for r in absent:
        assert (out["gram"][r] == SENTINEL).all() and out["scal"][r] == SENTINEL


# ------------------------------------------------------------------------------------------------ GEMM, exact forms
GEMM_SHAPES = [(37, n, 2600, 1 + n % 3) for n in range(1, 10)] + [(130, 127, 1500, 1), (129, 129, 3000, 4),
                                                                   (7, 257, 1100, 2), (200, 129, 700, 1)]


@pytest.mark.parametrize("precision", ["tf32x3", "f16x2"])
@pytest.mark.parametrize("shape", GEMM_SHAPES, ids=lambda s: "%dx%dx%d-s%d" % s)
def test_gemm_exact_forms_with_scales(eng, precision, shape):
    """C = A diag(s) B^T diag(c) with B integer counts (exact in tf32 and fp16), s spanning 2^-60..2^60 from one
    512-element group to the next (a misplaced group scale is off by 2^40 or more), c in 1e-6..1e6, signed A rows (the
    OLS projection's centred rows).  Per row within 4 TOL_GEMM of the magnitude product |A| diag(s) |B|^T diag(c)."""
    M, N, Kd, sp = shape
    rng = np.random.RandomState(M * N + Kd)
    A = rng.uniform(0.05, 1.0, (M, Kd)).astype(np.float32)
    A[::3] *= np.where(rng.rand(Kd) < 0.5, -1, 1).astype(np.float32)
    B = rng.poisson(1.5, (N, Kd)).astype(np.float32)
    B[0, 0] = 2048.0
    groups = -(-Kd // 512)
    ge = rng.randint(-60, 61, groups)
    s = (2.0 ** np.repeat(ge, 512)[:Kd] * rng.uniform(1, 2, Kd)).astype(np.float32)
    c = (10.0 ** rng.uniform(-6, 6, N)).astype(np.float32)
    C, _ = eng.gemm_abt(A, B, precision=precision, splits=sp, b_exact=True, k_scale=s, out_col_scale=c)
    As = A.astype(np.float64) * s.astype(np.float64)
    ref = (As @ B.astype(np.float64).T) * c.astype(np.float64)
    mag = (np.abs(As) @ B.astype(np.float64).T) * c.astype(np.float64)
    assert np.isfinite(C).all()
    err = np.linalg.norm(C - ref, axis=1) / np.linalg.norm(mag, axis=1)
    assert err.max() <= 4 * TOL_GEMM, err.max()


def test_gemm_f16_rows_at_and_below_the_scale_floor(eng):
    """Rows whose group maxima sit at and below 2^-111 keep the floor scale 2^-126: each fp16 piece pair then represents
    an entry to within half an fp16 subnormal step of the scaled value, 2^-25 * 2^-126 = 2^-151, so a product entry is
    off by at most 2^-151 sum_k |B[n, k]| from the pieces plus fp32 rounding of the chain and output sums (relative,
    4 TOL_GEMM of the magnitude, and 2^-149 absolute per rounding of a subnormal partial, at most Kd / 128 + splits + 2
    of them).  Every output must be finite."""
    rng = np.random.RandomState(3)
    M, N, Kd = 6, 9, 1600
    A = rng.uniform(0.5, 1.0, (M, Kd))
    A *= (2.0 ** np.array([-111, -112, -118, -126, -135, -60]))[:, None]
    A = A.astype(np.float32)
    B = rng.poisson(2.0, (N, Kd)).astype(np.float32)
    for sp in (1, 3):
        C, _ = eng.gemm_abt(A, B, precision="f16x2", splits=sp)
        assert np.isfinite(C).all()
        ref = A.astype(np.float64) @ B.astype(np.float64).T
        bound = 4 * TOL_GEMM * np.abs(ref) + 2.0 ** -151 * B.sum(axis=1)[None, :] + (Kd / 128 + sp + 2) * 2.0 ** -149
        assert (np.abs(C - ref) <= bound).all()
        assert (np.abs(C[0] - ref[0]) <= 4 * TOL_GEMM * ref[0]).all()     # 2^-111 still scales to [2^14, 2^15)


def test_gemm_scales_need_an_exact_form(eng):
    from cnmf_b200._lib import CnmfError
    A = np.ones((4, 8), np.float32)
    with pytest.raises(CnmfError):
        eng.gemm_abt(A, A, precision="tf32x3", k_scale=np.ones(8, np.float32))
    with pytest.raises(CnmfError):
        eng.gemm_abt(A, A, precision="fp32", b_exact=True)
