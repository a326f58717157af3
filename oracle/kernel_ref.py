"""ORACLE (test infrastructure) -- float64 references of ONE launch of the batched solver's kernels
(cnmf_b200/csrc/nmf_kernels.cu, and nmf_f64.cu for the float64 solver), the stopping decision of the solver loops, and
bit-exact numpy restatements of the operand pieces the GEMM reads.

Layout as in the kernels: a factor is K x n (components x items); `num` is the product the update divides by
(X H^T for W, W^T X for H) summed over its split-K slices; `G` is the K x K Gram of the other factor.  The update
references take the fp32 inputs the kernel takes: G already rounded to fp32 (load_gram_smem), everything else exact.
Pinned to scikit-learn's own update functions by tests/test_oracle_golden.py.
"""
import numpy as np

EPSILON = float(np.finfo(np.float32).eps)      # SK/decomposition/_nmf.py:32
FLT_MIN = float(np.finfo(np.float32).tiny)


def gram_fp32(gram_in, K, diag_add=0.0):
    """The K x K Gram as the update kernel holds it in shared memory (load_gram_smem): each fp64 entry rounded to fp32,
    then `diag_add` (CD: l2) added to the diagonal in fp32.  Returned as float64 holding those fp32 values."""
    G = np.asarray(gram_in, np.float64)[:K, :K].astype(np.float32)
    if diag_add:
        idx = np.arange(K)
        G[idx, idx] = G[idx, idx] + np.float32(diag_add)
    return G.astype(np.float64)


def mu_half_step(F, num, G, l1=0.0, l2=0.0, eps_rule="floor", dtype=np.float64):
    """One multiplicative update of F (SK/decomposition/_nmf.py:535-549,610-624 for W; :633-635,696-721 for H):
        den = G F + l1 + l2 F;   den -> float32 eps by eps_rule;   F_new = F * num / den.
    eps_rule "floor" (the default) is the fp32 kernels' rule: den < FLT_MIN -> eps (their Newton quotient needs a normal
    denominator).  "zero" is scikit-learn's own rule, which the float64 solver keeps: only den == 0 -> eps, a positive
    denominator below FLT_MIN is used as it is.  The two agree on every denominator that is 0 or >= FLT_MIN.  dtype:
    the arithmetic (np.longdouble gives a reference whose own rounding is far below float64's)."""
    F = np.asarray(F, dtype)
    den = np.asarray(G, dtype) @ F + dtype(l1) + dtype(l2) * F
    if eps_rule == "floor":
        den = np.where(den < FLT_MIN, dtype(EPSILON), den)
    elif eps_rule == "zero":
        den = np.where(den == 0, dtype(EPSILON), den)
    else:
        raise ValueError("eps_rule must be 'floor' or 'zero'")
    return F * np.asarray(num, dtype) / den


def cd_sweep(F, num, G, l1=0.0, l2=0.0, jacobi=False, dtype=np.float64):
    """One coordinate-descent sweep over the K coordinates of every item (SK/decomposition/_cdnmf_fast.pyx:8-37 with
    shuffle=False; l1 subtracted from the product and l2 added to the Gram diagonal, SK/decomposition/_nmf.py:
    379-385), in dtype (float64 by default).  G must be the Gram WITHOUT l2 (gram_fp32(..., diag_add=l2) gives the
    kernel's form; pass l2=0 then).  Returns (F_new, violation, magnitude): violation = sum |projected gradient| over
    items and coordinates (a Python float), magnitude[t, j] = |num - l1| + sum_r |G[t, r] F[r, j]| of each gradient
    (what its rounding error scales with).  jacobi=True evaluates every gradient from the OLD F (a wrong order, for
    tests that must tell Gauss-Seidel from it)."""
    F = np.array(F, dtype)
    num = np.asarray(num, dtype)
    G = np.asarray(G, dtype) + dtype(l2) * np.eye(len(G), dtype=dtype)
    l1 = dtype(l1)
    K = F.shape[0]
    F0 = F.copy()
    viol = dtype(0.0)
    mag = np.zeros_like(F)
    for t in range(K):
        src = F0 if jacobi else F
        grad = l1 - num[t] + G[t] @ src
        mag[t] = np.abs(l1 - num[t]) + np.abs(G[t]) @ np.abs(src)
        pg = np.where(src[t] == 0.0, np.minimum(dtype(0.0), grad), grad)
        viol += np.abs(pg).sum()
        h = G[t, t]
        if h != 0.0:
            F[t] = np.maximum(src[t] - grad / h, dtype(0.0))
    return F, float(viol), mag


# ---------------------------------------------------------------------------------------- stopping decisions
def mu_stop(it, err, err0, prev, tol, max_iter):
    """The MU loop's decision after iteration it >= 1 (oracle/nmf_ref.py mu_frobenius, SK/decomposition/_nmf.py:
    867-888): the error is looked at only when tol > 0 and it % 10 == 0; the restart stops when (prev - err) / err0 <
    tol -- strict, and with numpy's IEEE quotient, so err0 == 0 gives NaN (never stops) or -inf (stops) -- and prev
    advances to err only when it continues.  The loop ends after max_iter whatever the error.  err is not read at the
    other iterations.  Returns (stop, prev)."""
    if tol > 0 and it % 10 == 0:
        with np.errstate(divide="ignore", invalid="ignore"):
            q = (np.float64(prev) - np.float64(err)) / np.float64(err0)
        if q < tol:
            return True, prev
        prev = err
    return it >= max_iter, prev


def cd_stop(it, viol, viol0, tol, max_iter):
    """The CD loop's decision after iteration it >= 1 (oracle/nmf_ref.py cd_frobenius, SK/decomposition/_nmf.py:
    504-516): iteration 1's violation becomes viol0; the restart stops when viol0 == 0 or viol / viol0 <= tol (not
    strict), and after max_iter.  Returns (stop, viol0)."""
    if it == 1:
        viol0 = viol
    return bool(viol0 == 0 or viol / viol0 <= tol or it >= max_iter), viol0


# ---------------------------------------------------------------------------------------- operand pieces
def to_tf32(x):
    """cvt.rna.tf32.f32 on finite fp32 values (to_tf32 of common.cuh): add half an ulp of tf32, clear 13 bits."""
    u = np.ascontiguousarray(x, np.float32).view(np.uint32)
    return ((u + np.uint32(0x1000)) & np.uint32(0xffffe000)).view(np.float32)


def tf32_pieces(F, scale=None):
    """(hi, lo) tf32 pieces of F * scale (fp32 product), as split_scaled_kernel and the update kernels' store_items
    write them: hi = tf32(x), lo = tf32(x - hi)."""
    x = np.ascontiguousarray(F, np.float32)
    if scale is not None:
        x = x * np.asarray(scale, np.float32)
    hi = to_tf32(x)
    lo = to_tf32(x - hi)
    return hi, lo


def f16_group_scale(m):
    """f16_group_scale of common.cuh: the power of two 2^max(e - 15, -126) for a group maximum m = f 2^e (f in
    [0.5, 1)), which puts m in [2^14, 2^15); 1 for m = 0 or m >= 3e38.  Maxima below 2^-111 get the floor 2^-126."""
    m = np.ascontiguousarray(m, np.float32)
    b = (m.view(np.uint32) >> np.uint32(23)).astype(np.int64)
    sc = (np.maximum(b - 14, 1).astype(np.uint32) << np.uint32(23)).view(np.float32)
    return np.where((m > 0) & (m < np.float32(3.0e38)), sc, np.float32(1.0)).astype(np.float32)


def f16_pieces(F, scale=None, group=512):
    """fp16 pieces of the rows of F * scale (fp32 product) as emit_f16_kernel / emit_tile_f16 write them: per row and
    group of `group` columns sc = f16_group_scale(max |x|), hi = fp16(x / sc), mid = fp16(x / sc - hi) (division by a
    power of two is exact).  F is rows x ld, ld the padded row stride.  Returns (hi, mid, tile_scale)."""
    x = np.ascontiguousarray(F, np.float32)
    if scale is not None:
        x = x * np.asarray(scale, np.float32)
    rows, ld = x.shape
    nt = (ld + group - 1) // group
    pad = np.zeros((rows, nt * group), np.float32)
    pad[:, :ld] = x
    m = np.abs(pad).reshape(rows, nt, group).max(axis=2)
    ts = f16_group_scale(m)
    y = (pad.reshape(rows, nt, group) / ts[:, :, None]).reshape(rows, nt * group)[:, :ld].astype(np.float32)
    hi = y.astype(np.float16)
    mid = (y - hi.astype(np.float32)).astype(np.float16)
    return hi, mid, ts


# ---------------------------------------------------------------------------------------- KL / IS (nmf_beta.cu)
EPS64 = float(np.finfo(np.float64).eps)


def beta_half_step(F, D, Foth, beta, half, l1=0.0, l2=0.0):
    """One multiplicative half-step of the KL (beta = 1) or IS (beta = 0) loss in the kernels' layout, float64:
    F (K x items) is updated, Foth (K x n_contract) is the other factor, D (n_contract x items) the data with the item
    index contiguous (X^T for the W half, X for the H half), so WH = Foth^T F in D's layout.  scikit-learn's rules
    (SK/decomposition/_nmf.py:551-624 for W, :637-721 for H, :845-865 for the flush):
        WH floored at float32 eps;  KL: num = Foth (D / WH), den = row sums of Foth (a zero sum -> 1 in the H half only);
        IS: num = Foth (D WH^-2), den = Foth WH^-1;  den += l1, + l2 F;  den == 0 -> float32 eps;
        F_new = F (num / den)^gamma, gamma = 1/2 for IS;  values below float64 eps -> 0 after the H half for beta <= 1
        and after the W half for beta < 1."""
    F = np.asarray(F, np.float64)
    Foth = np.asarray(Foth, np.float64)
    D = np.asarray(D, np.float64)
    WH = np.maximum(Foth.T @ F, EPSILON)
    if beta == 1:
        num = Foth @ (D / WH)
        den = np.repeat(Foth.sum(axis=1)[:, None], F.shape[1], axis=1)
        if half == "H":
            den[den == 0] = 1.0
    elif beta == 0:
        num = Foth @ (D / WH ** 2)
        den = Foth @ (1.0 / WH)
    else:
        raise ValueError("beta must be 0 or 1")
    if l1 > 0:
        den = den + l1
    if l2 > 0:
        den = den + l2 * F
    den = np.where(den == 0, EPSILON, den)
    delta = num / den
    if beta == 0:
        delta = np.sqrt(delta)
    out = F * delta
    if half == "H" or beta < 1:
        out[out < EPS64] = 0.0
    return out


def beta_terms(D, F, Foth, beta):
    """(t, s, res, err) of SK/decomposition/_nmf.py:_beta_divergence (dense branch, square_root=True) for X = D,
    WH = Foth^T F (either orientation: the divergence is the same for X^T), split as beta_error_kernel splits it: each
    entry's share of the divergence, which vanishes as WH -> X, so nothing large cancels.  Entries with x <= float32 eps
    are dropped; WH' = max(WH, eps) on the rest, div = x / WH'.
      KL: t = sum x log div - x + WH',  s = sum(WH) over the dropped entries + sum(WH - WH') over the rest,  res = t + s
          (= sum x log div + sum(WH) - sum x, scikit-learn's form);
      IS: t = sum (div - 1) - log div,  s = number of entries kept,  res = t - (entries - s)
          (= sum div - sum log div - entries);
      beta = 2: t = res = sum (x - WH)^2 over every entry, s = 0.
    err = sqrt(2 max(res, 0)), or sqrt(res) for beta = 2 (the kernel's ||X - WH||_F, which scikit-learn's formula
    sqrt(2 * res / 2) equals)."""
    D = np.asarray(D, np.float64)
    WHr = np.asarray(Foth, np.float64).T @ np.asarray(F, np.float64)
    if beta == 2:
        t = float(((D - WHr) ** 2).sum())
        return t, 0.0, t, float(np.sqrt(max(t, 0.0)))
    keep = D > EPSILON
    x = D[keep]
    whf = np.maximum(WHr[keep], EPSILON)
    div = x / whf
    if beta == 1:
        t = float(np.sum(x * np.log(div) - x + whf))
        s = float(WHr[~keep].sum() + (WHr[keep] - whf).sum())
        res = t + s
    elif beta == 0:
        t = float(np.sum((div - 1.0) - np.log(div)))
        s = float(keep.sum())
        res = t - (D.size - s)
    else:
        raise ValueError("beta must be 0, 1 or 2")
    return t, s, res, float(np.sqrt(2.0 * max(res, 0.0)))
