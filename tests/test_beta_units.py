"""The KL / IS solver's kernels (nmf_beta.cu) one launch at a time (`-m gpu`), through the cnmf_beta_step_host test
hook, against the float64 references of oracle/kernel_ref.py -- at every K from 1 to 32 in each KPMAX instantiation
(8, 16, 32), both halves, both losses, item counts around the 256-item block and contraction lengths around the 4-row
unroll and the 128-row tile -- and bit for bit where the solver's batch independence rests on equal bits.

Layout as in the kernels: F_own (K x items) is updated, F_other (K x n_contract) is the other factor, D (n_contract x
items) is the data with the item index contiguous (X^T for the W half, X for the H half).  u = 2^-24.
"""
import numpy as np
import pytest

from oracle import kernel_ref as kr

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
EPS32 = np.float32(kr.EPSILON)
SENTINEL = -12345.0
CC = 128                 # contraction rows per shared-memory tile

KP8_ALL = list(range(1, 9))
KP16_ALL = list(range(1, 17))
KP32_ALL = list(range(1, 33))
MIXED = [1, 17, 32, 3, 12, 16, 21, 28]
LOSSES = {"kl": ("kullback-leibler", 1), "is": ("itakura-saito", 0)}


@pytest.fixture(scope="module")
def eng():
    from cnmf_b200.engine import Engine
    return Engine(0)


def ld_of(n):
    return -(-n // 32) * 32


def offsets(ks):
    return np.concatenate([[0], np.cumsum(ks)]).astype(int)


def make_batch(ks, n_items, n_contract, seed, rids=None):
    """Packed fp32 data of one launch with NaN in the padding columns of D and F_other (no launch may read them) and
    zeros in those of F_own (the layout's invariant).  Entries of order 1: WH is of order K, far above the eps floor."""
    rng = np.random.RandomState(seed)
    ks = list(ks)
    SK = sum(ks)
    rids = np.arange(len(ks)) if rids is None else np.asarray(rids)
    ldi, ldk = ld_of(n_items), ld_of(n_contract)
    D = np.full((n_contract, ldi), np.nan, np.float32)
    D[:, :n_items] = rng.uniform(0.2, 2.0, (n_contract, n_items))
    F = np.zeros((SK, ldi), np.float32)
    F[:, :n_items] = rng.uniform(0.1, 1.5, (SK, n_items))
    Fo = np.full((SK, ldk), np.nan, np.float32)
    Fo[:, :n_contract] = rng.uniform(0.1, 1.5, (SK, n_contract))
    return dict(ks=ks, rids=rids, n_rids=int(rids.max()) + 1, off=offsets(ks), ni=n_items, nk=n_contract, D=D, F=F, Fo=Fo)


def run(eng, b, side, loss, op="update", done=None, **kw):
    done = np.zeros(b["n_rids"], np.int32) if done is None else done
    return eng.beta_step(b["ks"], b["rids"], done, side, loss, b["D"], b["F"], b["Fo"], b["ni"], b["nk"], op=op, **kw)


def slot_rows(b, s):
    return slice(b["off"][s], b["off"][s + 1])


def check_extents(b, out):
    assert np.isfinite(out["F"]).all(), "NaN padding of D / F_other leaked into the factor"
    assert not out["F"][:, b["ni"]:].any(), "factor padding columns must stay exactly 0"


def update_bound(k, n_contract, beta):
    """Relative error of one updated entry, in units of u, to first order.  Every term is non-negative, so no sum
    cancels and each rounding contributes at most u of the value it rounds:
      WH: a chain of k FMAs (k); the quotient div_nr / reciprocal rcp_nr (Newton step after rcp.approx: 2).
      numerator / IS denominator: a chain of <= 128 FMAs per tile (min(n, 128)), then ceil(n / 128) tile partials
        summed in fp32 (ceil(n / 128) - 1), each term carrying the relative error of its factor q:
        KL q = X / WH: k + 2;  IS q = X (WH^-1)^2: 2 (k + 2) + 2;  IS denominator term WH^-1: k + 2.
      denominator: KL row sum rounded from fp64 (1), + l1 (1), + l2 F (2);  division (1).
      IS: gamma = 1/2 halves the relative error of the quotient and sqrtf rounds once (1).
      final multiply by the old entry (1)."""
    chain = min(n_contract, CC) + (-(-n_contract // CC) - 1)
    if beta == 1:
        return (k + 2) + chain + 4 + 1 + 1
    num = 2 * (k + 2) + 2 + chain
    den = (k + 2) + chain + 3
    return (num + den + 1) / 2 + 1 + 1


def update_check(b, out, loss, side, l1, l2):
    beta = LOSSES[loss][1]
    n, m = b["ni"], b["nk"]
    D = b["D"][:, :n]
    for s, k in enumerate(b["ks"]):
        rows = slot_rows(b, s)
        ref = kr.beta_half_step(b["F"][rows, :n], D, b["Fo"][rows, :m], beta, side, l1, l2)
        got = out["F"][rows, :n].astype(np.float64)
        bound = update_bound(k, m, beta) * U * (1 + 1e-3) * np.abs(ref)
        bad = np.abs(got - ref) > bound
        assert not bad.any(), (loss, side, k, n, m, int(bad.sum()),
                               float(np.max(np.abs(got - ref) / np.maximum(np.abs(ref), 1e-300))))
    if loss == "kl":             # the denominators the launch used: fp64 row sums of F_other
        ref = b["Fo"][:, :m].astype(np.float64).sum(axis=1)
        assert np.allclose(out["oth_sum"], ref, rtol=m * 2.0 ** -52, atol=0)


# ------------------------------------------------------------------------------------------------ updates
UPDATE_CASES = [  # n_items, n_contract, (l1, l2)
    (1, 1, (0.0, 0.0)),
    (255, 3, (0.125, 0.0)),
    (256, 4, (0.0, 0.25)),
    (257, 5, (0.0625, 0.5)),
    (513, 127, (0.0, 0.0)),
    (255, 128, (0.25, 0.125)),
    (257, 129, (0.0, 0.0)),
    (513, 1031, (0.5, 0.0)),
]


@pytest.mark.parametrize("side", ["W", "H"])
@pytest.mark.parametrize("loss", ["kl", "is"])
@pytest.mark.parametrize("case", UPDATE_CASES, ids=lambda c: "i%d-c%d" % (c[0], c[1]))
def test_beta_update_against_float64_every_k(eng, case, loss, side):
    n, m, (l1, l2) = case
    for ks in (KP8_ALL, KP16_ALL, KP32_ALL, MIXED):
        b = make_batch(ks, n, m, seed=n + 7 * m + len(ks))
        out = run(eng, b, side, LOSSES[loss][0], l1=l1, l2=l2)
        update_check(b, out, loss, side, l1, l2)
        check_extents(b, out)


@pytest.mark.parametrize("loss", ["kl", "is"])
def test_beta_update_long_contraction(eng, loss):
    """50 003 contraction rows: 391 tile partials summed in fp32 after the 128-row chains."""
    for ks, side in ((MIXED, "W"), (KP8_ALL, "H")):
        b = make_batch(ks, 257, 50003, seed=21)
        out = run(eng, b, side, LOSSES[loss][0], l1=0.125)
        update_check(b, out, loss, side, 0.125, 0.0)
        check_extents(b, out)


@pytest.mark.parametrize("side", ["W", "H"])
@pytest.mark.parametrize("loss", ["kl", "is"])
def test_beta_floors_dead_components_and_flush(eng, loss, side):
    """Every value at least a factor 4 from the threshold it tests:
    - items whose factor column is zero (WH = 0) or 1e-10 (WH <= 5e-9, floored to eps = 1.2e-7): the floor decides
      the quotient of the whole column;
    - a zero component row of F_other: its KL row sum is 0 and IS has a zero numerator and a zero denominator: the
      output row is exactly 0 and finite, the other components unaffected.  (The KL numerator is 0 whenever that row
      sum is, so the result is 0 whether the sum becomes eps (W half) or 1 (H half): on non-negative data the H half's
      zero-sum rule changes no value, and no test can tell it from the W half's.)
    - entries of 1e-30 beside entries of order 1 (their update stays near 1e-30, far below 2^-52 = 2.2e-16): flushed
      to 0 in the H half for both losses and in the W half for IS, kept in the KL W half."""
    for ks in (KP8_ALL, MIXED):
        b = make_batch(ks, 300, 140, seed=31 + len(ks))
        n = b["ni"]
        b["F"][:, 5] = 0.0
        b["F"][:, 10:20] *= np.float32(1e-10)
        dead = [int(b["off"][s]) + k - 1 for s, k in enumerate(ks)]          # last component of every restart
        b["Fo"][dead, :b["nk"]] = 0.0
        tiny = np.zeros_like(b["F"], bool)
        tiny[::2, 40:n:7] = True                     # every other component: WH and the quotient stay of order 1
        b["F"][tiny] = np.float32(1e-30)
        out = run(eng, b, side, LOSSES[loss][0])
        update_check(b, out, loss, side, 0.0, 0.0)
        check_extents(b, out)
        assert not out["F"][:, 5].any() and not out["F"][dead].any()
        live_tiny = tiny.copy()
        live_tiny[dead] = False
        if side == "H" or loss == "is":
            assert not out["F"][live_tiny].any(), "values below float64 eps must be flushed"
        else:
            v = out["F"][live_tiny]
            assert (v > 0).all() and (v < kr.EPS64 / 4).all(), "the KL W half does not flush"
        WH = b["Fo"][:, :b["nk"]].astype(np.float64).T @ b["F"][:, :n].astype(np.float64)
        assert WH[:, 10:20].max() < EPS32 / 4


# ------------------------------------------------------------------------------------------------ divergences
def divergence_bound(D, F, Foth, k, ct, mode):
    """|t - t_ref|, |s - s_ref| bounds of one restart, to first order.  A thread sums the terms of <= 128 rows x ct
    items of one tile into one fp32 accumulator (chain M = ct * min(n, 128): (M - 1) u sum |term|), then fp64 across
    tiles and blocks (1e-12 relative covers it).  Each term's own error, with WH a chain of k FMAs over non-negative
    products (|dWH| <= k u WH), div_nr within 2u, logf within 1 ulp (2u |log div|), 1 - div and div - 1 rounded once
    (exact for div in [0.5, 2]) and the term's last operation rounded once (u |term|):
      KL  T = WH' (div log div - div + 1): dT/dWH' = 1 - div and dT/ddiv = WH' log div, so
          (k + 1) u WH' |1 - div| + 2u x |log div| (div) + 2u x |log div| (logf) + u T;
          s: k u WH over the dropped entries, k u WH + u |WH - eps| where the floor applies;
      IS  T = (div - 1) - log div: dT/ddiv = 1 - 1/div, so (k + 3) u |div - 1| + 2u |log div| + u T;  s is an exact
          count;
      Frobenius: d = x - WH with |d err| <= k u WH + u |d|, squared: 2 |d| (k u WH + u |d|).
    Both divergence terms are flat in WH and div where div = 1, so the bound shrinks with the residual r like
    r (u / r relative to res), where a sum X log div - (sum X - sum WH) or sum div - log div - N G loses all of it as
    u / r^2."""
    D = np.asarray(D, np.float64)
    WH = np.asarray(Foth, np.float64).T @ np.asarray(F, np.float64)
    M = ct * min(D.shape[0], CC)
    if mode == 2:
        d = D - WH
        terms = d * d
        own = 2 * np.abs(d) * (k * U * WH + U * np.abs(d))
        return (M - 1) * U * terms.sum() + own.sum() + 1e-12 * terms.sum(), 0.0
    keep = D > kr.EPSILON
    x = D[keep]
    whr = WH[keep]
    whf = np.maximum(whr, kr.EPSILON)
    div = x / whf
    lg = np.abs(np.log(div))
    if mode == 1:
        terms = x * np.log(div) - x + whf
        own = (k + 1) * U * whf * np.abs(1 - div) + 4 * U * x * lg + U * np.abs(terms)
        floored = whr < kr.EPSILON
        sterms = np.concatenate([WH[~keep], whr[floored] - kr.EPSILON])
        sown = k * U * WH[~keep].sum() + (k * U * whr[floored] + U * np.abs(whr[floored] - kr.EPSILON)).sum()
        sxb = (M - 1) * U * np.abs(sterms).sum() + sown + 1e-12 * np.abs(sterms).sum()
    else:
        terms = (div - 1) - np.log(div)
        own = (k + 3) * U * np.abs(div - 1) + 2 * U * lg + U * np.abs(terms)
        sxb = 0.0
    return (M - 1) * U * np.abs(terms).sum() + own.sum() + 1e-12 * np.abs(terms).sum(), sxb


MODES = {"kl": ("kullback-leibler", 1), "is": ("itakura-saito", 0), "frob": ("frobenius", 2)}


def divergence_check(b, out, mode_name, side):
    loss, beta = MODES[mode_name]
    n, m = b["ni"], b["nk"]
    D = b["D"][:, :n]
    for s, (k, r) in enumerate(zip(b["ks"], b["rids"])):
        rows = slot_rows(b, s)
        F, Fo = b["F"][rows, :n], b["Fo"][rows, :m]
        t, sx, res, err = kr.beta_terms(D, F, Fo, beta)
        ct = 2 if -(-k // 4) * 4 <= 16 else 1            # items per thread of the error kernel's body
        tb, sxb = divergence_bound(D, F, Fo, k, ct, beta)
        gt, gsx = out["totals"][r]
        assert abs(gt - t) <= tb, (mode_name, side, k, gt, t, tb)
        assert abs(gsx - sx) <= sxb, (mode_name, side, k, gsx, sx, sxb)
        resb = tb + sxb + 1e-12 * abs(res)
        errb = resb / err if beta != 2 else resb / (2 * err)
        assert abs(out["last"][r] - err) <= errb * (1 + 1e-3), (mode_name, side, k, out["last"][r], err, errb)


@pytest.mark.parametrize("side", ["W", "H"])
@pytest.mark.parametrize("mode", ["kl", "is", "frob"])
def test_beta_divergence_against_float64(eng, mode, side):
    """Mixed batch, every KPMAX, with X holding exact zeros, entries equal to float32 eps (dropped: the test is a
    strict x > eps) and entries just above it (kept)."""
    for ks, n, m in ((MIXED, 513, 1031), (KP8_ALL, 257, 129), (KP16_ALL, 300, 5)):
        b = make_batch(ks, n, m, seed=41 + n)
        rng = np.random.RandomState(n)
        sel = rng.rand(m, n)
        D = b["D"][:, :n]
        D[sel < 0.05] = 0.0
        D[(sel >= 0.05) & (sel < 0.08)] = EPS32
        D[(sel >= 0.08) & (sel < 0.1)] = np.nextafter(EPS32, np.float32(1))
        b["D"][:, :n] = D
        out = run(eng, b, side, MODES[mode][0], op="divergence")
        divergence_check(b, out, mode, side)


def near_converged(ks, n_items, n_contract, rel, seed):
    """W, H of order 1 and X = WH (1 + rel * noise) in fp32: the divergence a solve sees near convergence."""
    rng = np.random.RandomState(seed)
    b = make_batch(ks, n_items, n_contract, seed)
    k0 = slot_rows(b, 0)
    WH = b["Fo"][k0, :n_contract].astype(np.float64).T @ b["F"][k0, :n_items].astype(np.float64)
    b["D"][:, :n_items] = (WH * (1 + rel * rng.uniform(-1, 1, WH.shape))).astype(np.float32)
    return b


@pytest.mark.parametrize("mode", ["kl", "is"])
def test_beta_divergence_near_convergence(eng, mode):
    """4 000 x 600 entries, WH within 0.1 %, 1 % and 10 % of X (the fit of the first restart; the others see the same X
    with their own factors).  The stopping rule compares (prev - err) / err0 with tol = 1e-4, so err must be right to
    well under tol / 10 = 1e-5 relative.  Holds err to divergence_bound (worst case: every rounding of the 2.4 million
    entries in the same direction; about 1.3e-3 at r = 0.1 %, 1.4e-4 at 1 %, 2.1e-5 at 10 % relative) and, since the
    per-entry roundings are independent and add as a random walk rather than in one direction, the measured error to
    1e-6, a tenth of the stopping rule's resolution."""
    loss, beta = MODES[mode]
    for rel in (0.001, 0.01, 0.1):
        b = near_converged([10, 3, 7], 4000, 600, rel, seed=int(10000 * rel))
        out = run(eng, b, "W", loss, op="divergence")
        r = int(b["rids"][0])
        rows = slot_rows(b, 0)
        D, F, Fo = b["D"][:, :4000], b["F"][rows, :4000], b["Fo"][rows, :600]
        t, sx, res, err = kr.beta_terms(D, F, Fo, beta)
        tb, sxb = divergence_bound(D, F, Fo, 10, 2, beta)
        got = out["last"][r]
        print("\n%s r %.3f: err %.9g, float64 %.9g, relative error %.2e, worst-case bound %.2e"
              % (mode, rel, got, err, abs(got - err) / err, (tb + sxb) / err ** 2))
        divergence_check(b, out, mode, "W")
        assert abs(got - err) <= 1e-6 * err, (mode, rel, got, err)


# ------------------------------------------------------------------------------------------------ exact bits
@pytest.mark.parametrize("loss", ["kl", "is"])
def test_restart_bits_do_not_depend_on_the_batch(eng, loss):
    """The same restarts alone (KPMAX 8), beside a K = 12 restart (KPMAX 16) and beside a K = 20 one (KPMAX 32), at
    other slots and rids: the same bits for both halves and for every divergence output."""
    small = [1, 3, 5, 8]
    base = make_batch(small, 513, 300, seed=51)
    outs = []
    for extra, perm in ((None, [0, 1, 2, 3]), (12, [3, 0, 2, 1]), (20, [2, 3, 1, 0])):
        ks = [small[i] for i in perm]
        rows = np.concatenate([np.arange(base["off"][i], base["off"][i + 1]) for i in perm])
        b = dict(base, ks=ks, F=base["F"][rows], Fo=base["Fo"][rows])
        rids = np.array(perm) + 2                              # restart p sits at rid p + 2 in every batch
        if extra is not None:
            e = make_batch([extra], 513, 300, seed=52)
            b = dict(b, ks=[extra] + ks, F=np.vstack([e["F"], b["F"]]), Fo=np.vstack([e["Fo"], b["Fo"]]))
            rids = np.concatenate([[0], rids])
        b.update(rids=rids, n_rids=int(rids.max()) + 1, off=offsets(b["ks"]))
        first = 0 if extra is None else 1
        got = {}
        for side in ("W", "H"):
            o = run(eng, b, side, LOSSES[loss][0])
            for j, p in enumerate(perm):
                got[(side, p)] = o["F"][slot_rows(b, j + first)].tobytes()
        for mode in (loss, "frob"):
            o = run(eng, b, "W", MODES[mode][0], op="divergence")
            for p in perm:
                got[(mode, p)] = np.concatenate([[o["last"][p + 2]], o["totals"][p + 2]]).tobytes()
        outs.append(got)
    for o in outs[1:]:
        assert o.keys() == outs[0].keys()
        for key in o:
            assert o[key] == outs[0][key], key


@pytest.mark.parametrize("loss", ["kl", "is"])
def test_frozen_and_absent_restarts_keep_their_sentinels(eng, loss):
    ks = [5, 16, 1, 9, 12, 30]
    R = len(ks)
    perm = np.random.RandomState(R).permutation(R + 1)
    rids = perm[perm != 2]                                     # rid 2 is not in the batch
    b = make_batch(ks, 300, 200, seed=61, rids=rids)
    done = np.zeros(b["n_rids"], np.int32)
    frozen = [int(rids[1]), int(rids[-1])]
    done[frozen] = 1
    live = [s for s in range(R) if int(rids[s]) not in frozen]
    for side in ("W", "H"):
        out = run(eng, b, side, LOSSES[loss][0], done=done)
        for s in range(R):
            same = np.array_equal(out["F"][slot_rows(b, s)], b["F"][slot_rows(b, s)])
            assert same == (s not in live), (side, s)
        sub = dict(b, ks=[ks[s] for s in live], F=np.vstack([b["F"][slot_rows(b, s)] for s in live]),
                   Fo=np.vstack([b["Fo"][slot_rows(b, s)] for s in live]))
        sub["off"] = offsets(sub["ks"])
        update_check(sub, dict(out, F=np.vstack([out["F"][slot_rows(b, s)] for s in live]),
                               oth_sum=np.concatenate([out["oth_sum"][slot_rows(b, s)] for s in live])),
                     loss, side, 0.0, 0.0)
    for mode in (loss, "frob"):
        last0 = np.full(b["n_rids"], SENTINEL)
        tot0 = np.full((b["n_rids"], 2), SENTINEL)
        out = run(eng, b, "W", MODES[mode][0], op="divergence", done=done, last=last0, totals=tot0)
        for r in range(b["n_rids"]):
            keep = r in frozen or r == 2
            assert (out["last"][r] == SENTINEL) == keep and (out["totals"][r] == SENTINEL).all() == keep, (mode, r)


@pytest.mark.parametrize("loss", ["kl", "is"])
def test_hook_halves_equal_one_solver_iteration(eng, loss):
    """The hook's W half then its H half, from the same starts, give the bits of Dataset.factorize(max_iter=1) -- the
    solver's own BetaSides -- for usages and spectra, and the hook's Frobenius divergence is the solve's err bit for
    bit.  KL also with regularisation on both halves."""
    from cnmf_b200.engine import make_params
    rng = np.random.RandomState(71)
    n, g = 700, 333
    X = rng.uniform(0.1, 3.0, (n, g)).astype(np.float32)
    X[rng.rand(n, g) < 0.2] = 0.0 if loss == "kl" else np.float32(0.05)
    ds = eng.dataset(X, precision="fp32")
    ks = [4, 17, 9]
    SK = sum(ks)
    W0 = rng.uniform(0.1, 1.0, (SK, n)).astype(np.float32)
    H0 = rng.uniform(0.1, 1.0, (SK, g)).astype(np.float32)
    regs = [dict()] + ([dict(alpha_W=0.001, alpha_H=0.002, l1_ratio=0.25)] if loss == "kl" else [])
    for reg in regs:
        kw = dict(solver="mu", beta_loss=LOSSES[loss][0], max_iter=1, tol=1e-4, **reg)
        sp, us, _, err = ds.factorize(ks, [1, 2, 3], kw, return_usages=True, W0=W0, H0=H0)
        p = make_params(kw, n, g, "fp32")
        ldr, ldc = ld_of(n), ld_of(g)
        Xt = np.zeros((g, ldr), np.float32)
        Xt[:, :n] = X.T
        Xp = np.zeros((n, ldc), np.float32)
        Xp[:, :g] = X
        Wt = np.zeros((SK, ldr), np.float32)
        Wt[:, :n] = W0
        H = np.zeros((SK, ldc), np.float32)
        H[:, :g] = H0
        done = np.zeros(len(ks), np.int32)
        rids = np.arange(len(ks))
        a = eng.beta_step(ks, rids, done, "W", LOSSES[loss][0], Xt, Wt, H, n, g,
                          l1=np.float32(p.l1_reg_W), l2=np.float32(p.l2_reg_W))
        c = eng.beta_step(ks, rids, done, "H", LOSSES[loss][0], Xp, H, a["F"], g, n,
                          l1=np.float32(p.l1_reg_H), l2=np.float32(p.l2_reg_H))
        e = eng.beta_step(ks, rids, done, "W", "frobenius", Xt, a["F"], c["F"], n, g, op="divergence")
        off = offsets(ks)
        for r in range(len(ks)):
            assert np.array_equal(sp[r], c["F"][off[r]:off[r + 1], :g]), (loss, reg, r)
            assert np.array_equal(us[r], a["F"][off[r]:off[r + 1], :n].T), (loss, reg, r)
        assert np.array_equal(err, e["last"]), (loss, reg, err, e["last"])


# ------------------------------------------------------------------------------------------------ minimum
def test_dataset_min_is_exact(eng):
    """Dataset.min() (what refuses IS data with zeros) equals X.min() bit for bit: minimum in the last row and column,
    more rows than the NUM_SMS * 8 blocks, negative values, a single row, a single column."""
    rng = np.random.RandomState(81)
    cases = []
    X = rng.uniform(1, 2, (2500, 37)).astype(np.float32)
    X[-1, -1] = np.float32(0.5)
    cases.append(X)
    X = rng.uniform(1, 2, (1500, 300)).astype(np.float32)
    X[1499, 7] = np.float32(0.75)
    cases.append(X)
    X = rng.uniform(-1, 2, (300, 257)).astype(np.float32)
    X[0, 256] = np.float32(-3.25)
    cases.append(X)
    X = rng.uniform(1, 2, (1, 1000)).astype(np.float32)
    X[0, 999] = np.float32(0.125)
    cases.append(X)
    X = rng.uniform(1, 2, (3000, 1)).astype(np.float32)
    X[2999, 0] = np.float32(0.0625)
    cases.append(X)
    X = rng.uniform(1e-3, 2, (2000, 65)).astype(np.float32)
    X[2000 - 1, 64] = 0.0                                       # a zero IS must refuse
    cases.append(X)
    for X in cases:
        ds = eng.dataset(X, precision="fp32")
        assert ds.min() == float(X.min()), (X.shape, ds.min(), X.min())
    with pytest.raises(ValueError):
        ds.factorize([2], [1], dict(solver="mu", beta_loss="itakura-saito", max_iter=1))
