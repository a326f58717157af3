"""numpy restatement of the device NNDSVD starts (cnmf_b200/csrc/nndsvd.cu), step for step in float64: the range
finder with CholeskyQR2 in place of scikit-learn's LU normaliser and QR, B's SVD as CholeskyQR of B^T followed by a
one-sided Jacobi SVD of the small triangular factor, svd_flip on the vector over the cells, the NNDSVD composition
and the fills.  Tests hold it against cnmf_b200.nndsvd.nndsvd_init (scikit-learn's algorithm) and the device
against both."""
import numpy as np

PIVOT_TOL = 1e-12
JACOBI_TOL = 1e-14
EPS = 1e-6


def cholesky_dropping(G):
    """Right-looking Cholesky of a Gram matrix; a pivot at or below PIVOT_TOL of its row's original squared norm
    marks the row dependent: zero row and column in L."""
    G = np.tril(G).astype(np.float64)
    d0 = np.diag(G).copy()
    P = G.shape[0]
    for j in range(P):
        dd = G[j, j]
        piv = np.sqrt(dd) if dd > PIVOT_TOL * d0[j] else 0.0
        G[j, j] = piv
        G[j + 1:, j] = G[j + 1:, j] / piv if piv > 0 else 0.0
        for i in range(j + 1, P):
            G[i, j + 1:i + 1] -= G[i, j] * G[j + 1:i + 1, j]
    return np.tril(G)


def forward(L, A):
    """L^-1 A row by row; rows with a zero pivot come out zero."""
    Y = np.zeros_like(A)
    for i in range(A.shape[0]):
        if L[i, i] != 0.0:
            Y[i] = (A[i] - L[i, :i] @ Y[:i]) / L[i, i]
    return Y


def orth_rows(A):
    """CholeskyQR2 of the rows of A (P x n): returns (Q, L) with A = L Q on the rows that are not dropped."""
    L1 = cholesky_dropping(A @ A.T)
    Q = forward(L1, A)
    L2 = cholesky_dropping(Q @ Q.T)
    return forward(L2, Q), L1 @ L2


def jacobi_svd(A):
    """One-sided Jacobi: A = U diag(S) V^T, S descending (stable), U column of S = 0 set to zero."""
    A = A.copy()
    P = A.shape[1]
    V = np.eye(P)
    for _ in range(60):
        rotated = False
        for p in range(P - 1):
            for q in range(p + 1, P):
                a, b, g = A[:, p] @ A[:, p], A[:, q] @ A[:, q], A[:, p] @ A[:, q]
                if not abs(g) > JACOBI_TOL * np.sqrt(a * b):
                    continue
                rotated = True
                zeta = (b - a) / (2.0 * g)
                t = (1.0 if zeta >= 0 else -1.0) / (abs(zeta) + np.sqrt(1.0 + zeta * zeta))
                cs = 1.0 / np.sqrt(1.0 + t * t)
                sn = cs * t
                A[:, [p, q]] = np.stack([cs * A[:, p] - sn * A[:, q], sn * A[:, p] + cs * A[:, q]], axis=1)
                V[:, [p, q]] = np.stack([cs * V[:, p] - sn * V[:, q], sn * V[:, p] + cs * V[:, q]], axis=1)
        if not rotated:
            break
    S = np.sqrt((A * A).sum(axis=0))
    order = np.argsort(-S, kind="stable")
    S = S[order]
    U = np.zeros_like(A)
    nz = S > 0
    U[:, nz] = A[:, order][:, nz] / S[nz]
    return U, S, V[:, order]


def device_randomized_svd(X, k, seed):
    """(U n x k, S, V k x g): the k leading triplets as the device computes them, cells-vector sign convention."""
    X = np.asarray(X, dtype=np.float64)
    N, G = X.shape
    mn = min(N, G)
    P = min(k + 10, mn)
    n_iter = 7 if k < 0.1 * mn else 4
    M = X if N >= G else X.T
    Qa = np.random.RandomState(seed).normal(size=(M.shape[1], k + 10))[:, :P].T.copy()    # rows over M's columns
    for _ in range(n_iter):
        Qb, _ = orth_rows(Qa @ M.T)
        Qa, _ = orth_rows(Qb @ M)
    Qb, _ = orth_rows(Qa @ M.T)
    QB, L = orth_rows(Qb @ M)                       # B = L QB
    Us, S, Vs = jacobi_svd(L)
    Ub = Us[:, :k].T @ Qb                           # rows over M's rows
    Va = Vs[:, :k].T @ QB                           # rows over M's columns
    cells, genes = (Ub, Va) if N >= G else (Va, Ub)
    idx = np.argmax(np.abs(cells), axis=1)
    signs = np.sign(cells[np.arange(k), idx])
    return (cells * signs[:, None]).T, S[:k], genes * signs[:, None]


def device_nndsvd_init(X, k, seed, init="nndsvd"):
    """(W n x k, H k x g) as cnmf_nndsvd_init_dev computes them, in float64."""
    X = np.asarray(X, dtype=np.float64)
    U, S, V = device_randomized_svd(X, k, seed)
    W = np.zeros_like(U)
    H = np.zeros_like(V)
    W[:, 0] = np.sqrt(S[0]) * np.abs(U[:, 0])
    H[0, :] = np.sqrt(S[0]) * np.abs(V[0, :])
    for j in range(1, k):
        x, y = U[:, j], V[j, :]
        xp, yp, xn, yn = np.maximum(x, 0), np.maximum(y, 0), np.abs(np.minimum(x, 0)), np.abs(np.minimum(y, 0))
        xpn, ypn = np.sqrt(xp @ xp), np.sqrt(yp @ yp)
        xnn, ynn = np.sqrt(xn @ xn), np.sqrt(yn @ yn)
        mp, mn = xpn * ypn, xnn * ynn
        if mp > mn:
            u, v, sigma, nu, nv = xp, yp, mp, xpn, ypn
        else:
            u, v, sigma, nu, nv = xn, yn, mn, xnn, ynn
        lbd = np.sqrt(S[j] * sigma)
        W[:, j] = lbd * (u / nu if nu > 0 else 0.0 * u)
        H[j, :] = lbd * (v / nv if nv > 0 else 0.0 * v)
    W[W < EPS] = 0
    H[H < EPS] = 0
    avg = X.mean()
    if init == "nndsvda":
        W[W == 0] = avg
        H[H == 0] = avg
    elif init == "nndsvdar":
        zw, zh = np.flatnonzero(W == 0), np.flatnonzero(H == 0)      # row-major: W's zeros first, then H's
        z = np.random.RandomState(seed).standard_normal(size=len(zw) + len(zh))
        W.flat[zw] = np.abs(avg * z[:len(zw)] / 100)
        H.flat[zh] = np.abs(avg * z[len(zw):] / 100)
    return W, H
