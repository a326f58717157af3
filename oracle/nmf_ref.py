"""ORACLE (test infrastructure) -- numpy restatement of the NMF solvers the reference
reaches through ``cNMF._nmf`` (cnmf.py:661-674 -> sklearn.decomposition.non_negative_factorization).

The arithmetic lives in scikit-learn 1.9.0 (third-party, NOT part of the reference;
``SK/`` below = site-packages/sklearn).  Each function cites the lines it restates.
Pinned by tests/test_oracle_golden.py against fixtures produced by the reference itself
(oracle/make_golden.py) and against live sklearn calls.
"""
import numpy as np

EPSILON = np.finfo(np.float32).eps  # SK/decomposition/_nmf.py:32


def init_random(X_mean, n_samples, n_features, k, seed, dtype=np.float64):
    """SK/decomposition/_nmf.py:296-307: H is drawn FIRST, then W, from the legacy
    RandomState(seed) (SK/utils/validation.py check_random_state); cast, then abs."""
    avg = np.sqrt(X_mean / k)
    rng = np.random.RandomState(seed)
    H = avg * rng.standard_normal(size=(k, n_features)).astype(dtype, copy=False)
    W = avg * rng.standard_normal(size=(n_samples, k)).astype(dtype, copy=False)
    np.abs(H, out=H)
    np.abs(W, out=W)
    return W, H


def frobenius_error(X, W, H):
    """SK/decomposition/_nmf.py:113-127 (dense branch) with square_root=True."""
    return np.sqrt(((X - W @ H) ** 2).sum())


def frobenius_error_trace(X, W, H, norm_X_sq=None):
    """SK/decomposition/_nmf.py:116-120 (sparse branch; the reference's default X is CSR):
    ||X||^2 + <W^T W H, H> - 2 <X H^T, W>.  This is the identity the CUDA path uses."""
    if norm_X_sq is None:
        norm_X_sq = float((X.astype(np.float64) ** 2).sum())
    norm_WH = np.sum((W.T @ W) * (H @ H.T))
    cross = np.sum((X @ H.T) * W)
    return np.sqrt(max(norm_X_sq + norm_WH - 2.0 * cross, 0.0))


def mu_frobenius(X, W, H, tol=1e-4, max_iter=1000, l1_reg_W=0.0, l2_reg_W=0.0,
                 l1_reg_H=0.0, l2_reg_H=0.0, update_H=True, error_fn=frobenius_error):
    """Multiplicative-update NMF, beta=2.
    SK/decomposition/_nmf.py:726-888 (loop), :535-549,610-624 (W), :633-635,696-721 (H)."""
    W = W.copy()
    H = H.copy()
    err0 = prev = error_fn(X, W, H)
    XHt = HHt = None
    n_iter = 0
    for n_iter in range(1, max_iter + 1):
        if XHt is None:
            XHt = X @ H.T
        num = XHt if update_H else XHt.copy()
        if HHt is None:
            HHt = H @ H.T
        den = W @ HHt
        if l1_reg_W > 0:
            den += l1_reg_W
        if l2_reg_W > 0:
            den = den + l2_reg_W * W
        den[den == 0] = EPSILON
        num /= den
        W *= num
        if update_H:
            num = W.T @ X
            den = np.linalg.multi_dot([W.T, W, H])
            if l1_reg_H > 0:
                den += l1_reg_H
            if l2_reg_H > 0:
                den = den + l2_reg_H * H
            den[den == 0] = EPSILON
            num /= den
            H *= num
            XHt = HHt = None
        if tol > 0 and n_iter % 10 == 0:
            err = error_fn(X, W, H)
            if (prev - err) / err0 < tol:
                break
            prev = err
    return W, H, n_iter


def beta_divergence(X, W, H, beta):
    """SK/decomposition/_nmf.py:77-175 (dense branch), square_root=True, for beta in {1: generalized
    Kullback-Leibler, 0: Itakura-Saito}.  Entries with X <= EPSILON are dropped (:140-142), WH is
    floored at EPSILON (:145); the result is sqrt(2 * max(res, 0)) (:170-175)."""
    WH = (W @ H).ravel()
    Xd = X.ravel()
    keep = Xd > EPSILON
    WH = WH[keep]
    Xd = Xd[keep]
    WH[WH < EPSILON] = EPSILON
    if beta == 1:
        sum_WH = np.dot(W.sum(axis=0), H.sum(axis=1))
        div = Xd / WH
        res = np.dot(Xd, np.log(div)) + sum_WH - Xd.sum()
    elif beta == 0:
        div = Xd / WH
        res = div.sum() - np.prod(X.shape) - np.log(div).sum()
    else:
        raise ValueError("oracle restates beta in {0, 1} (and 2 via mu_frobenius)")
    return np.sqrt(2.0 * max(res, 0.0))


def mu_beta(X, W, H, beta, tol=1e-4, max_iter=1000, l1_reg_W=0.0, l2_reg_W=0.0,
            l1_reg_H=0.0, l2_reg_H=0.0, update_H=True):
    """Multiplicative-update NMF for beta_loss 'kullback-leibler' (1) / 'itakura-saito' (0), dense X.
    SK/decomposition/_nmf.py:726-888 (loop; gamma :813-818; clipping :845-846, :863-865),
    :551-608 (W numerator / denominator), :637-694 (H), :610-624 / :696-721 (regularisation, guard).
    Asymmetries kept: the H half replaces a zero W_sum by 1 (:669), the W half does not; with beta=1
    only H is clipped below float64 eps (:864), with beta<1 both are (:845)."""
    W = W.copy()
    H = H.copy()
    gamma = 1.0 / (2.0 - beta) if beta < 1 else 1.0
    eps64 = np.finfo(np.float64).eps
    err0 = prev = beta_divergence(X, W, H, beta)
    H_sum = None
    n_iter = 0
    for n_iter in range(1, max_iter + 1):
        WH = W @ H
        WHs = WH.copy()
        if beta < 1:
            WH[WH < EPSILON] = EPSILON
        WHs[WHs < EPSILON] = EPSILON
        if beta == 1:
            Q = X / WHs
            num = Q @ H.T
            if H_sum is None:
                H_sum = H.sum(axis=1)
            den = np.repeat(H_sum[None, :], W.shape[0], axis=0)
        else:
            Q = X * (1.0 / WHs) ** 2
            num = Q @ H.T
            den = (WH ** (beta - 1.0)) @ H.T
        if l1_reg_W > 0:
            den = den + l1_reg_W
        if l2_reg_W > 0:
            den = den + l2_reg_W * W
        den[den == 0] = EPSILON
        delta = num / den
        if gamma != 1:
            delta **= gamma
        W *= delta
        if beta < 1:
            W[W < eps64] = 0.0
        if update_H:
            WH = W @ H
            WHs = WH.copy()
            if beta < 1:
                WH[WH < EPSILON] = EPSILON
            WHs[WHs < EPSILON] = EPSILON
            if beta == 1:
                num = W.T @ (X / WHs)
                W_sum = W.sum(axis=0)
                W_sum[W_sum == 0] = 1.0
                den = np.repeat(W_sum[:, None], H.shape[1], axis=1)
            else:
                num = W.T @ (X * (1.0 / WHs) ** 2)
                den = W.T @ (WH ** (beta - 1.0))
            if l1_reg_H > 0:
                den = den + l1_reg_H
            if l2_reg_H > 0:
                den = den + l2_reg_H * H
            den[den == 0] = EPSILON
            delta = num / den
            if gamma != 1:
                delta **= gamma
            H *= delta
            H_sum = None
            if beta <= 1:
                H[H < eps64] = 0.0
        if tol > 0 and n_iter % 10 == 0:
            err = beta_divergence(X, W, H, beta)
            if (prev - err) / err0 < tol:
                break
            prev = err
    return W, H, n_iter


def _cd_sweep(A, Gram, B):
    """SK/decomposition/_cdnmf_fast.pyx:8-37 restated row-outer (rows are independent,
    verified identical to the t-outer Cython order; SURVEY.md appendix C).
    Vectorised over rows; sequential over the K coordinates."""
    K = A.shape[1]
    viol = 0.0
    for t in range(K):
        g = -B[:, t] + A @ Gram[t, :]
        pg = np.where(A[:, t] == 0, np.minimum(0.0, g), g)
        viol += np.abs(pg).sum()
        if Gram[t, t] != 0:
            A[:, t] = np.maximum(A[:, t] - g / Gram[t, t], 0.0)
    return viol


def cd_frobenius(X, W, H, tol=1e-4, max_iter=1000, l1_reg_W=0.0, l2_reg_W=0.0,
                 l1_reg_H=0.0, l2_reg_H=0.0, update_H=True):
    """Coordinate-descent NMF (the reference's DEFAULT for beta_loss='frobenius',
    cnmf.py:629-631).  SK/decomposition/_nmf.py:399-518 (loop, shuffle=False),
    :369-396 (one half-step)."""
    W = W.copy()
    Ht = np.ascontiguousarray(H.T.copy())
    viol0 = 1.0
    n_iter = 0
    for n_iter in range(1, max_iter + 1):
        HHt = Ht.T @ Ht
        XHt = X @ Ht
        if l2_reg_W != 0:
            HHt = HHt.copy()
            HHt.flat[:: HHt.shape[0] + 1] += l2_reg_W
        if l1_reg_W != 0:
            XHt = XHt - l1_reg_W
        viol = _cd_sweep(W, HHt, XHt)
        if update_H:
            WtW = W.T @ W
            XtW = X.T @ W
            if l2_reg_H != 0:
                WtW = WtW.copy()
                WtW.flat[:: WtW.shape[0] + 1] += l2_reg_H
            if l1_reg_H != 0:
                XtW = XtW - l1_reg_H
            viol += _cd_sweep(Ht, WtW, XtW)
        if n_iter == 1:
            viol0 = viol
        if viol0 == 0:
            break
        if viol / viol0 <= tol:
            break
    return W, Ht.T.copy(), n_iter


def nmf(X, k, seed, solver="mu", tol=1e-4, max_iter=1000, dtype=np.float64,
        alpha_W=0.0, alpha_H=0.0, l1_ratio=0.0, beta=2, init="random"):
    """One restart as cNMF.factorize issues it (cnmf.py:738-741): init + solver.  init != 'random' (`--init nndsvd`,
    cnmf.py:1252): the starting factors come from scikit-learn's own `_initialize_nmf` -- the third-party code the
    reference's call runs -- not from a restatement."""
    X = np.asarray(X, dtype=dtype)
    n, g = X.shape
    if init == "random":
        W, H = init_random(X.mean(), n, g, k, seed, dtype=dtype)
    else:
        from sklearn.decomposition._nmf import _initialize_nmf
        W, H = _initialize_nmf(X, k, init=init, random_state=seed)
    l1W, l2W, l1H, l2H = reg_terms(n, g, alpha_W, alpha_H, l1_ratio)
    if solver == "mu" and beta != 2:
        return mu_beta(X, W, H, beta, tol, max_iter, l1W, l2W, l1H, l2H)
    if solver == "mu":
        return mu_frobenius(X, W, H, tol, max_iter, l1W, l2W, l1H, l2H)
    return cd_frobenius(X, W, H, tol, max_iter, l1W, l2W, l1H, l2H)


def reg_terms(n_samples, n_features, alpha_W, alpha_H, l1_ratio):
    """SK/decomposition/_nmf.py:1249-1260 (alpha_H='same' never reaches here: cNMF always
    passes a float, cnmf.py:619-620)."""
    l1W = n_features * alpha_W * l1_ratio
    l1H = n_samples * alpha_H * l1_ratio
    l2W = n_features * alpha_W * (1.0 - l1_ratio)
    l2H = n_samples * alpha_H * (1.0 - l1_ratio)
    return l1W, l2W, l1H, l2H


def refit(X, H, solver="mu", tol=1e-4, max_iter=1000, dtype=np.float64, beta=2):
    """cNMF.refit_usage (cnmf.py:776-802): NMF with H fixed (update_H=False).
    W0: SK/decomposition/_nmf.py:1223-1228 -- 'mu': constant sqrt(X.mean()/k); 'cd': zeros."""
    X = np.asarray(X, dtype=dtype)
    H = np.asarray(H, dtype=dtype)
    n = X.shape[0]
    k = H.shape[0]
    if solver == "mu":
        W0 = np.full((n, k), np.sqrt(X.mean() / k), dtype=dtype)
        if beta != 2:
            W, _, it = mu_beta(X, W0, H, beta, tol, max_iter, update_H=False)
        else:
            W, _, it = mu_frobenius(X, W0, H, tol, max_iter, update_H=False)
    else:
        W0 = np.zeros((n, k), dtype=dtype)
        W, _, it = cd_frobenius(X, W0, H, tol, max_iter, update_H=False)
    return W, it
