"""CPU emulation: does a 2-piece fp16 factor split (per-row power-of-two normalisation) keep the MU iteration within
the parity budget?  Compared with the current 2-piece tf32 split.  Products accumulate in float64 here (the operand
representation is what is being tested)."""
import os, sys, numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cnmf_b200.synth import make_counts, normalise, restart_table
EPS = np.finfo(np.float32).eps

def tf32_round(x):
    u = x.astype(np.float32).view(np.uint32)
    u = (u + np.uint32(0x1000)) & np.uint32(0xffffe000)
    return u.view(np.float32)

def split_tf32(A):
    A = A.astype(np.float32)
    hi = tf32_round(A); lo = tf32_round(A - hi)
    return hi.astype(np.float64) + lo.astype(np.float64)

def split_fp16(A, pieces=2):
    A = A.astype(np.float32).astype(np.float64)
    rowmax = np.maximum(A.max(axis=1, keepdims=True), 1e-30)
    s = 2.0 ** np.ceil(np.log2(rowmax))
    Ap = A / s
    rep = np.zeros_like(Ap); res = Ap.copy()
    for _ in range(pieces):
        p = res.astype(np.float16).astype(np.float64)
        rep += p; res = res - p
    return rep * s

def mu(X, k, seed, rep, max_iter=1000, tol=1e-4):
    rng = np.random.RandomState(seed)
    avg = np.sqrt(X.mean() / k)
    H = np.abs(avg * rng.standard_normal((k, X.shape[1]))).astype(np.float32).astype(np.float64)
    W = np.abs(avg * rng.standard_normal((X.shape[0], k))).astype(np.float32).astype(np.float64)
    def err(W, H): return np.linalg.norm(X - W @ H)
    e0 = prev = err(W, H)
    for it in range(1, max_iter + 1):
        num = X @ rep(H).T                     # A operand = H (SK x G), B = X
        den = W @ (H @ H.T); den[den == 0] = EPS
        W = (W * num / den).astype(np.float32).astype(np.float64)
        num = rep(W.T) @ X                     # A operand = W^T
        den = (W.T @ W) @ H; den[den == 0] = EPS
        H = (H * num / den).astype(np.float32).astype(np.float64)
        if it % 10 == 0:
            e = err(W, H)
            if (prev - e) / e0 < tol: break
            prev = e
    return H, it

def rel(a, b): return np.linalg.norm(a - b) / np.linalg.norm(b)
X, _ = normalise(make_counts(3000, 600, k_true=8, seed=3), np.float64)
rows = restart_table([6, 9], 4, seed=14)
ident = lambda A: A.astype(np.float32).astype(np.float64)
for (k, _, seed) in rows:
    Href, itref = mu(X, k, seed, lambda A: A)          # fp64 operands, fp32-stored factors
    out = []
    for name, rep in (("fp32", ident), ("tf32x2", split_tf32), ("fp16x2", lambda A: split_fp16(A, 2)), ("fp16x3", lambda A: split_fp16(A, 3))):
        H, it = mu(X, k, seed, rep)
        out.append("%s: it %d rel %.2e" % (name, it, rel(H, Href)))
    print("K=%d seed %d ref it %d | " % (k, seed, itref) + " | ".join(out), flush=True)
# representation error on a heavy-tailed factor
rng = np.random.RandomState(0)
A = np.abs(rng.standard_cauchy((50, 20000))) * 0.1
for name, rep in (("tf32x2", split_tf32), ("fp16x2", lambda A: split_fp16(A, 2))):
    R = rep(A); A32 = A.astype(np.float32).astype(np.float64)
    Xc = rng.poisson(0.5, size=(20000, 64)).astype(np.float64)
    P = A32 @ Xc; Pr = R @ Xc
    print(name, "heavy-tailed rows: max rel product error %.2e, median %.2e" % (np.abs(Pr - P).max() / np.abs(P).max(), np.median(np.abs(Pr - P) / np.abs(P))))

def split_fp16_hi(A, pieces=2):
    A = A.astype(np.float32).astype(np.float64)
    rowmax = np.maximum(A.max(axis=1, keepdims=True), 1e-30)
    s = 2.0 ** (np.ceil(np.log2(rowmax)) - 15)       # row maximum lands in [2^14, 2^15]: far from fp16's subnormals
    Ap = A / s
    rep = np.zeros_like(Ap); res = Ap.copy()
    for _ in range(pieces):
        p = res.astype(np.float16).astype(np.float64)
        rep += p; res = res - p
    return rep * s
R = split_fp16_hi(A, 2); A32 = A.astype(np.float32).astype(np.float64)
P = A32 @ Xc; Pr = R @ Xc
print("fp16x2 scaled to 2^15", "heavy-tailed rows: max rel product error %.2e, median %.2e, max entry rel err %.2e" % (np.abs(Pr - P).max() / np.abs(P).max(), np.median(np.abs(Pr - P) / np.abs(P)), np.max(np.abs(R - A32) / np.maximum(A32, 1e-300))))
R = split_tf32(A)
print("tf32x2 max entry rel err %.2e" % np.max(np.abs(R - A32) / np.maximum(A32, 1e-300)))
