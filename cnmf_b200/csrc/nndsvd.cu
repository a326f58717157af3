// NNDSVD starting factors on the device (init = 'nndsvd' / 'nndsvda' / 'nndsvdar'): scikit-learn's
// randomized_svd(X, k, random_state=seed) followed by the NNDSVD composition of `_initialize_nmf`
// (SK/utils/extmath.py, SK/decomposition/_nmf.py:309-369), for every restart of a call at once.
//
// Layout: restart r owns P_r = min(k + 10, min(N, G)) consecutive rows of two packed fp64 arrays, Qc over the cells
// (row stride ld_r) and Qg over the genes (ld_c), exactly like the solver's factors.  The products with X of all
// restarts are then ONE fp64 GEMM each (gemm_f64.cu, M = sum P_r).  M is X when N >= G and X^T otherwise (sklearn's
// transpose='auto'); Omega lives on M's columns ("space a"), M Q on its rows ("space b").
//
//   Qa <- Omega^T                         RandomState(seed).normal(size=(n_a, k + 10)), first P_r columns
//   n_iter times: Qb <- rows of (M Qa), orth;  Qa <- rows of (M^T Qb), orth     (7 if k < 0.1 min(N, G), else 4)
//   Qb <- rows of (M Qa), orth            the range basis Q
//   Qa <- rows of B = Q^T M, orth with the triangular factors accumulated: B = L Q_B^T
//   L = U_s S V_s^T                       one-sided Jacobi, one warp per restart, descending order
//   U = Q U_s (over space b), V = Q_B V_s (over space a), first k triplets only
//   svd_flip on the vector over the cells (u-based without the transpose, v-based with it), NNDSVD composition,
//   entries below 1e-6 -> 0 / mean(X) / |mean(X) z / 100| with z from a fresh RandomState(seed) (W's zeros in W's
//   row-major order, then H's).
//
// Orthonormalisation ("orth") is CholeskyQR2: Gram (fixed-order partial sums per item split), Cholesky, forward
// substitution of every item, twice.  Every normaliser multiplies on the right by an invertible matrix, so the
// subspace -- and hence the SVD -- is the one scikit-learn's LU-normalised iteration and QR give, in exact
// arithmetic.  A Gram that is not numerically positive definite (X of rank < P, duplicated columns) has a pivot
// that cancels to rounding noise; the Cholesky then drops that row (its pivot is below 1e-12 of the row's own squared
// norm): the row comes out zero and stays zero, the others stay orthonormal.  A zero row carries singular value 0,
// so it can reach the k leading triplets only when rank(X) < k, and then with S = 0, i.e. an all-zero component
// before the fill, as scikit-learn's own result is up to rounding.  This was chosen over a shifted first pass, which
// keeps full-rank inputs of any condition number but cannot make an exactly rank-deficient block orthonormal
// either, and over a Householder fallback, which needs a second code path over all items for inputs that do not
// occur in practice.
//
// Every reduction runs in an order fixed by the shape (N, G, P_r) alone, so a restart's starts are bit-identical
// whatever other restarts share its call or its chunk.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <vector>

#include "common.cuh"
#include "engine.h"
#include "legacy_gauss.cuh"

namespace cnmf {

namespace {

constexpr int PMAX = KMAX + 10;                 // largest P_r
constexpr int LSTRIDE = PMAX * PMAX;            // per-restart P x P matrices (row-major, stride PMAX)
constexpr int GRAM_CHUNK = 4096;                // items per Gram partial sum
constexpr int TILE = 64;                        // items per block of the Gram / apply kernels
constexpr double PIVOT_TOL = 1e-12;             // Cholesky pivot below this share of the row's squared norm: dependent
constexpr double JACOBI_TOL = 1e-14;            // rotate while |a_p . a_q| > tol * |a_p| |a_q|
constexpr int JACOBI_MAX_SWEEPS = 60;
constexpr double NNDSVD_EPS = 1e-6;             // sklearn _initialize_nmf eps

struct Meta {             // per restart of a chunk (device arrays)
  const int* poff;        // first row in Qc / Qg
  const int* P;           // rows
  const int* k;           // components
  const int* koff;        // first row in the output Wt / H
  const uint32_t* seed;
  const int* comp_r;      // per component row of the chunk (sum k entries): its restart ...
  const int* comp_j;      // ... and its index within the restart
};

__host__ __device__ inline int gram_splits(int n) { return (n + GRAM_CHUNK - 1) / GRAM_CHUNK; }

// Omega^T: normal t = (item, column) of the row-major n_a x P_full matrix -> Qa[poff + column][item]
__global__ void __launch_bounds__(LEGACY_GAUSS_THREADS)
omega_kernel(Meta m, int n_a, double* __restrict__ Qa, int lda) {
  __shared__ LegacyGaussShared sh;
  const int r = blockIdx.x;
  const int P = m.P[r], p_full = m.k[r] + 10;
  double* q = Qa + (long long)m.poff[r] * lda;
  legacy_gauss_block(m.seed[r], (long long)n_a * p_full, sh, [&](long long t, double z) {
    const long long item = t / p_full;
    const int col = (int)(t % p_full);
    if (col < P) q[(long long)col * lda + item] = z;
  });
}

// part[r][s] (lower triangle) = sum over the items of split s of Q_r[i] * Q_r[j]
__global__ void __launch_bounds__(256)
gram_kernel(Meta m, const double* __restrict__ Q, int ld, int n, double* __restrict__ part) {
  __shared__ double T[TILE][PMAX + 1];
  const int r = blockIdx.y, s = blockIdx.x, S = gridDim.x;
  const int P = m.P[r];
  const double* q = Q + (long long)m.poff[r] * ld;
  const int ne = P * (P + 1) / 2;
  int ei[4], ej[4];
  double acc[4];
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int e = threadIdx.x + 256 * u;
    int i = (int)((sqrt(8.0 * e + 1.0) - 1.0) * 0.5);
    while (i * (i + 1) / 2 > e) --i;
    while ((i + 1) * (i + 2) / 2 <= e) ++i;
    ei[u] = e < ne ? i : -1;
    ej[u] = e - i * (i + 1) / 2;
    acc[u] = 0.0;
  }
  const int c0 = s * GRAM_CHUNK, c1 = min(n, c0 + GRAM_CHUNK);
  for (int cb = c0; cb < c1; cb += TILE) {
    __syncthreads();
    for (int idx = threadIdx.x; idx < P * TILE; idx += 256) {
      const int p = idx / TILE, c = idx % TILE;
      T[c][p] = (cb + c < c1) ? q[(long long)p * ld + cb + c] : 0.0;
    }
    __syncthreads();
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (ei[u] < 0) continue;
      double a = acc[u];
      for (int c = 0; c < TILE; ++c) a = fma(T[c][ei[u]], T[c][ej[u]], a);
      acc[u] = a;
    }
  }
  double* out = part + ((long long)r * S + s) * LSTRIDE;
#pragma unroll
  for (int u = 0; u < 4; ++u)
    if (ei[u] >= 0) out[ei[u] * PMAX + ej[u]] = acc[u];
}

// Right-looking Cholesky of the summed Gram; dependent rows get a zero row and column in L.
// mode 0: L only; 1: also Lacc = L; 2: also Lacc = Lacc * L.
__global__ void __launch_bounds__(64)
chol_kernel(Meta m, const double* __restrict__ part, int S, double* __restrict__ L, double* __restrict__ Lacc, int mode) {
  __shared__ double Gs[PMAX][PMAX + 1];
  __shared__ double Ao[PMAX][PMAX + 1];
  __shared__ double d0[PMAX];
  const int r = blockIdx.x, tid = threadIdx.x;
  const int P = m.P[r];
  for (int e = tid; e < P * P; e += 64) {
    const int i = e / P, j = e % P;
    double v = 0.0;
    if (j <= i)
      for (int s = 0; s < S; ++s) v += part[((long long)r * S + s) * LSTRIDE + i * PMAX + j];
    Gs[i][j] = v;
  }
  __syncthreads();
  if (tid < P) d0[tid] = Gs[tid][tid];
  __syncthreads();
  for (int j = 0; j < P; ++j) {
    if (tid == 0) {
      const double dd = Gs[j][j];
      Gs[j][j] = dd > PIVOT_TOL * d0[j] ? sqrt(dd) : 0.0;
    }
    __syncthreads();
    const double piv = Gs[j][j];
    for (int i = j + 1 + tid; i < P; i += 64) Gs[i][j] = piv > 0.0 ? Gs[i][j] / piv : 0.0;
    __syncthreads();
    const int w = P - j - 1;
    for (int e = tid; e < w * w; e += 64) {
      const int i = j + 1 + e / w, c = j + 1 + e % w;
      if (c <= i) Gs[i][c] -= Gs[i][j] * Gs[c][j];
    }
    __syncthreads();
  }
  double* Lr = L + (long long)r * LSTRIDE;
  for (int e = tid; e < P * P; e += 64) {
    const int i = e / P, j = e % P;
    Lr[i * PMAX + j] = j <= i ? Gs[i][j] : 0.0;
  }
  if (mode == 0) return;
  double* Ar = Lacc + (long long)r * LSTRIDE;
  if (mode == 1) {
    for (int e = tid; e < P * P; e += 64) {
      const int i = e / P, j = e % P;
      Ar[i * PMAX + j] = j <= i ? Gs[i][j] : 0.0;
    }
    return;
  }
  for (int e = tid; e < P * P; e += 64) Ao[e / P][e % P] = Ar[(e / P) * PMAX + e % P];
  __syncthreads();
  for (int e = tid; e < P * P; e += 64) {
    const int i = e / P, j = e % P;
    double v = 0.0;
    for (int c = j; c <= i; ++c) v = fma(Ao[i][c], Gs[c][j], v);
    Ar[i * PMAX + j] = j <= i ? v : 0.0;
  }
}

// FULL = false: rows of restart r <- L^-1 rows (forward substitution per item; a zero pivot gives a zero row).
// FULL = true:  rows j < k of restart r <- sum_p F[p][j] row p (F = U_s or V_s).  In place: a block stages all P
// rows of its items before it writes.
template <bool FULL>
__global__ void __launch_bounds__(TILE)
apply_kernel(Meta m, double* __restrict__ Q, int ld, int n, const double* __restrict__ F) {
  __shared__ double Fs[PMAX][PMAX + 1];
  __shared__ double T[PMAX][TILE];
  const int r = blockIdx.y, c = threadIdx.x;
  const int P = m.P[r];
  double* q = Q + (long long)m.poff[r] * ld;
  const int item = blockIdx.x * TILE + c;
  const double* Fr = F + (long long)r * LSTRIDE;
  for (int e = c; e < P * P; e += TILE) Fs[e / P][e % P] = Fr[(e / P) * PMAX + e % P];
  for (int p = 0; p < P; ++p) T[p][c] = item < n ? q[(long long)p * ld + item] : 0.0;
  __syncthreads();
  if (item >= n) return;
  if (!FULL) {
    for (int i = 0; i < P; ++i) {
      const double piv = Fs[i][i];
      double y = 0.0;
      if (piv != 0.0) {
        double v = T[i][c];
        for (int j = 0; j < i; ++j) v = fma(-Fs[i][j], T[j][c], v);
        y = v / piv;
      }
      T[i][c] = y;
      q[(long long)i * ld + item] = y;
    }
  } else {
    const int k = m.k[r];
    for (int j = 0; j < k; ++j) {
      double v = 0.0;
      for (int p = 0; p < P; ++p) v = fma(Fs[p][j], T[p][c], v);
      q[(long long)j * ld + item] = v;
    }
  }
}

__device__ __forceinline__ double warp_sum_bcast(double v) { return __shfl_sync(0xffffffffu, warp_sum(v), 0); }

// One-sided (Hestenes) Jacobi SVD of the accumulated P x P factor, one warp per restart:
// Lacc = U_s diag(S) V_s^T with S descending (stable in the column index); U_s column of a zero S is zero.
__global__ void __launch_bounds__(32)
jacobi_kernel(Meta m, const double* __restrict__ Lacc, double* __restrict__ Us, double* __restrict__ Vs,
              double* __restrict__ Sv) {
  __shared__ double A[PMAX][PMAX + 1];    // A[col][row]
  __shared__ double V[PMAX][PMAX + 1];
  __shared__ double nrm[PMAX];
  __shared__ int perm[PMAX];
  const int r = blockIdx.x, lane = threadIdx.x;
  const int P = m.P[r];
  const double* Lr = Lacc + (long long)r * LSTRIDE;
  for (int e = lane; e < P * P; e += 32) {
    const int i = e / P, j = e % P;
    A[j][i] = Lr[i * PMAX + j];
    V[j][i] = i == j ? 1.0 : 0.0;
  }
  __syncwarp();
  for (int sweep = 0; sweep < JACOBI_MAX_SWEEPS; ++sweep) {
    bool rotated = false;
    for (int p = 0; p < P - 1; ++p)
      for (int q = p + 1; q < P; ++q) {
        double a = 0.0, b = 0.0, g = 0.0;
        for (int i = lane; i < P; i += 32) {
          a = fma(A[p][i], A[p][i], a);
          b = fma(A[q][i], A[q][i], b);
          g = fma(A[p][i], A[q][i], g);
        }
        a = warp_sum_bcast(a);
        b = warp_sum_bcast(b);
        g = warp_sum_bcast(g);
        if (!(fabs(g) > JACOBI_TOL * sqrt(a * b))) continue;
        rotated = true;
        const double zeta = (b - a) / (2.0 * g);
        const double t = (zeta >= 0.0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
        const double cs = 1.0 / sqrt(1.0 + t * t), sn = cs * t;
        for (int i = lane; i < P; i += 32) {
          const double x = A[p][i], y = A[q][i];
          A[p][i] = cs * x - sn * y;
          A[q][i] = sn * x + cs * y;
          const double vx = V[p][i], vy = V[q][i];
          V[p][i] = cs * vx - sn * vy;
          V[q][i] = sn * vx + cs * vy;
        }
        __syncwarp();
      }
    if (!rotated) break;
  }
  for (int j = 0; j < P; ++j) {
    double s = 0.0;
    for (int i = lane; i < P; i += 32) s = fma(A[j][i], A[j][i], s);
    s = warp_sum_bcast(s);
    if (lane == 0) nrm[j] = sqrt(s);
  }
  __syncwarp();
  if (lane == 0) {
    for (int j = 0; j < P; ++j) perm[j] = j;
    for (int j = 0; j < P; ++j) {          // stable selection of the largest remaining value
      int best = j;
      for (int c = j + 1; c < P; ++c)
        if (nrm[perm[c]] > nrm[perm[best]]) best = c;
      const int v = perm[best];
      for (int c = best; c > j; --c) perm[c] = perm[c - 1];
      perm[j] = v;
    }
  }
  __syncwarp();
  double* U = Us + (long long)r * LSTRIDE;
  double* Vo = Vs + (long long)r * LSTRIDE;
  for (int e = lane; e < P * P; e += 32) {
    const int i = e / P, j = e % P;
    const int src = perm[j];
    const double s = nrm[src];
    U[i * PMAX + j] = s > 0.0 ? A[src][i] / s : 0.0;
    Vo[i * PMAX + j] = V[src][i];
  }
  for (int j = lane; j < P; j += 32) Sv[(long long)r * PMAX + j] = nrm[perm[j]];
}

// Per (restart, component j < k): the svd_flip sign from the vector over the cells (largest |entry|, first index on
// ties, numpy's sign) and the squared norms of the positive / negative parts of both vectors.
// stats[(r * KMAX + j) * 8 + {0: sign, 1, 2: cells +/-, 3, 4: genes +/-}]
__global__ void __launch_bounds__(256)
stats_kernel(Meta m, const double* __restrict__ Qcell, int ldc, int n_cells, const double* __restrict__ Qgene, int ldg,
             int n_genes, double* __restrict__ stats) {
  __shared__ double s_abs[256], s_val[256], s_sum[4][256];
  __shared__ int s_idx[256];
  const int r = m.comp_r[blockIdx.x], j = m.comp_j[blockIdx.x], tid = threadIdx.x;
  const double* xc = Qcell + (long long)(m.poff[r] + j) * ldc;
  const double* xg = Qgene + (long long)(m.poff[r] + j) * ldg;
  double best = -1.0, bval = 0.0, cp = 0.0, cn = 0.0, gp = 0.0, gn = 0.0;
  int bidx = 0x7fffffff;
  for (int i = tid; i < n_cells; i += 256) {
    const double v = xc[i], a = fabs(v);
    if (a > best) { best = a; bval = v; bidx = i; }
    if (v > 0.0) cp = fma(v, v, cp); else cn = fma(v, v, cn);
  }
  for (int i = tid; i < n_genes; i += 256) {
    const double v = xg[i];
    if (v > 0.0) gp = fma(v, v, gp); else gn = fma(v, v, gn);
  }
  s_abs[tid] = best; s_val[tid] = bval; s_idx[tid] = bidx;
  s_sum[0][tid] = cp; s_sum[1][tid] = cn; s_sum[2][tid] = gp; s_sum[3][tid] = gn;
  __syncthreads();
  for (int w = 128; w > 0; w >>= 1) {
    if (tid < w) {
      const int o = tid + w;
      if (s_abs[o] > s_abs[tid] || (s_abs[o] == s_abs[tid] && s_idx[o] < s_idx[tid])) {
        s_abs[tid] = s_abs[o]; s_val[tid] = s_val[o]; s_idx[tid] = s_idx[o];
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) s_sum[u][tid] += s_sum[u][o];
    }
    __syncthreads();
  }
  if (tid == 0) {
    double* o = stats + ((long long)r * KMAX + j) * 8;
    o[0] = s_val[0] > 0.0 ? 1.0 : (s_val[0] < 0.0 ? -1.0 : 0.0);
    o[1] = s_sum[0][0]; o[2] = s_sum[1][0]; o[3] = s_sum[2][0]; o[4] = s_sum[3][0];
  }
}

// W^T rows (cells = true) or H rows of restart r, component j: sklearn's NNDSVD composition, eps zeroing and the
// 'nndsvda' fill (the 'nndsvdar' fill follows in ar_fill_kernel), rounded to fp32 once (T = float) or kept in fp64
// (T = double, float64 datasets).
template <typename T>
__global__ void __launch_bounds__(256)
compose_kernel(Meta m, const double* __restrict__ Qv, int ldq, int n, bool cells, const double* __restrict__ stats,
               const double* __restrict__ Sv, T* __restrict__ out, int ldo, double fill) {
  const int r = m.comp_r[blockIdx.y], j = m.comp_j[blockIdx.y];
  const int item = blockIdx.x * 256 + threadIdx.x;
  if (item >= n) return;
  const double v = Qv[(long long)(m.poff[r] + j) * ldq + item];
  const double S = Sv[(long long)r * PMAX + j];
  double w;
  if (j == 0) {
    w = sqrt(S) * fabs(v);
  } else {
    const double* st = stats + ((long long)r * KMAX + j) * 8;
    const double sg = st[0];
    // squared norms of the positive / negative parts after the flip x = sg * u
    const double cp = sg > 0.0 ? st[1] : (sg < 0.0 ? st[2] : 0.0), cn = sg > 0.0 ? st[2] : (sg < 0.0 ? st[1] : 0.0);
    const double gp = sg > 0.0 ? st[3] : (sg < 0.0 ? st[4] : 0.0), gn = sg > 0.0 ? st[4] : (sg < 0.0 ? st[3] : 0.0);
    const double cpn = sqrt(cp), cnn = sqrt(cn), gpn = sqrt(gp), gnn = sqrt(gn);
    const double mp = cpn * gpn, mn = cnn * gnn;
    const double x = sg * v;
    const bool pos = mp > mn;
    const double part = pos ? fmax(x, 0.0) : fabs(fmin(x, 0.0));
    const double nrm = pos ? (cells ? cpn : gpn) : (cells ? cnn : gnn);
    const double u = nrm > 0.0 ? part / nrm : 0.0;
    const double lbd = sqrt(S * (pos ? mp : mn));
    w = lbd * u;
  }
  if (w < NNDSVD_EPS) w = fill;
  out[(long long)(m.koff[r] + j) * ldo + item] = (T)w;
}

// block-wide exclusive scan of one flag per thread; returns this thread's slot, *total = number of set flags
__device__ __forceinline__ int block_rank(bool flag, int* warp_tot, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned bal = __ballot_sync(0xffffffffu, flag);
  if (lane == 0) warp_tot[warp] = __popc(bal);
  __syncthreads();
  int base = 0, tot = 0;
#pragma unroll
  for (int w = 0; w < 8; ++w) {
    if (w < warp) base += warp_tot[w];
    tot += warp_tot[w];
  }
  __syncthreads();
  *total = tot;
  return base + __popc(bal & ((1u << lane) - 1u));
}

// 'nndsvdar': the zeros of W (n x k, row-major) then of H (k x g) take |avg * z / 100| for the normals z of a fresh
// RandomState(seed), in that order.  The zeros' positions are listed in the restart's (no longer needed) rows of
// Qc / Qg first.
template <typename T>
__global__ void __launch_bounds__(LEGACY_GAUSS_THREADS)
ar_fill_kernel(Meta m, T* __restrict__ Wt, int ldw, int n_cells, T* __restrict__ H, int ldh, int n_genes,
               double* Qc, int ld_r, double* Qg, int ld_c, double avg) {
  __shared__ LegacyGaussShared sh;
  __shared__ int warp_tot[8];
  const int r = blockIdx.x, tid = threadIdx.x;
  const int k = m.k[r], koff = m.koff[r];
  long long* posW = reinterpret_cast<long long*>(Qc + (long long)m.poff[r] * ld_r);
  long long* posH = reinterpret_cast<long long*>(Qg + (long long)m.poff[r] * ld_c);
  const long long nW = (long long)n_cells * k, nH = (long long)k * n_genes;
  long long zW = 0, zH = 0;
  for (long long b = 0; b < nW; b += LEGACY_GAUSS_THREADS) {
    const long long t = b + tid;
    const bool z = t < nW && Wt[(long long)(koff + t % k) * ldw + t / k] == T(0);
    int tot;
    const int slot = block_rank(z, warp_tot, &tot);
    if (z) posW[zW + slot] = t;
    zW += tot;
  }
  for (long long b = 0; b < nH; b += LEGACY_GAUSS_THREADS) {
    const long long t = b + tid;
    const bool z = t < nH && H[(long long)(koff + t / n_genes) * ldh + t % n_genes] == T(0);
    int tot;
    const int slot = block_rank(z, warp_tot, &tot);
    if (z) posH[zH + slot] = t;
    zH += tot;
  }
  __syncthreads();
  legacy_gauss_block(m.seed[r], zW + zH, sh, [&](long long t, double z) {
    const T v = (T)fabs(__ddiv_rn(__dmul_rn(avg, z), 100.0));
    if (t < zW) {
      const long long p = posW[t];
      Wt[(long long)(koff + p % k) * ldw + p / k] = v;
    } else {
      const long long p = posH[t - zW];
      H[(long long)(koff + p / n_genes) * ldh + p % n_genes] = v;
    }
  });
}

struct DevBuf {          // cudaMalloc'd for one call: the solve that follows gets the memory back
  void* p = nullptr;
  ~DevBuf() { if (p) cudaFree(p); }
};

// TX: element type of the dataset's X (float, or double on float64 datasets); T: element type of the starts
template <typename TX, typename T>
int nndsvd_starts(cnmf_dataset_s* d, const TX* X, int R, const int* ks, const uint32_t* seeds, int init, T* Wt, T* H,
                  cudaStream_t s) {
  CNMF_REQUIRE(R > 0 && ks && seeds && Wt && H && X, "nndsvd_init_dev: bad arguments");
  CNMF_REQUIRE(init == CNMF_INIT_NNDSVD || init == CNMF_INIT_NNDSVDA || init == CNMF_INIT_NNDSVDAR,
               "nndsvd_init_dev: init must be CNMF_INIT_NNDSVD, _NNDSVDA or _NNDSVDAR");
  cnmf_handle_s* h = d->h;
  const int N = d->n_rows, G = d->n_cols, ld_r = d->ld_r, ld_c = d->ld_c;
  const int mn = std::min(N, G);
  const bool a_genes = N >= G;           // sklearn transposes M when N < G
  std::vector<int> P(R), koff(R), n_iter(R);
  int SK = 0;
  for (int r = 0; r < R; ++r) {
    CNMF_REQUIRE(ks[r] >= 1 && ks[r] <= KMAX, "nndsvd_init_dev: n_components must be in [1, 32]");
    CNMF_REQUIRE(ks[r] <= mn, "nndsvd_init_dev: init='nndsvd' can only be used when n_components <= "
                              "min(n_samples, n_features)");
    P[r] = std::min(ks[r] + 10, mn);
    n_iter[r] = ks[r] < 0.1 * mn ? 7 : 4;
    koff[r] = SK;
    SK += ks[r];
  }
  CNMF_CUDA_CHECK(cudaMemsetAsync(Wt, 0, (size_t)SK * ld_r * sizeof(T), s));
  CNMF_CUDA_CHECK(cudaMemsetAsync(H, 0, (size_t)SK * ld_c * sizeof(T), s));
  const double avg = d->sum / ((double)N * (double)G);

  // ---- chunk capacity from the free device memory: rows of Qc + Qg and the per-restart small matrices
  const int S_c = gram_splits(N), S_g = gram_splits(G), S_max = std::max(S_c, S_g);
  const size_t row_bytes = 8 * ((size_t)ld_r + ld_c);
  const size_t restart_bytes = 8 * ((size_t)LSTRIDE * (S_max + 4) + PMAX + KMAX * 8) + (5 + 2 * KMAX) * sizeof(int);
  size_t fr = 0, tot = 0;
  CNMF_CUDA_CHECK(cudaMemGetInfo(&fr, &tot));
  const size_t budget = fr / 2;
  const int max_p = *std::max_element(P.begin(), P.end());
  long long sum_p = 0;
  for (int r = 0; r < R; ++r) sum_p += P[r];
  const size_t per_max = max_p * row_bytes + restart_bytes;
  CNMF_REQUIRE(budget >= per_max, "nndsvd_init_dev: not enough free device memory for one restart");
  // compose_kernel's grid.y is the chunk's sum of k <= cap_R * KMAX; h->nndsvd_chunk_restarts caps it further
  int cap_R = (int)std::min<size_t>(std::min(R, 65535 / KMAX), budget / per_max);
  if (h->nndsvd_chunk_restarts > 0) cap_R = std::min(cap_R, h->nndsvd_chunk_restarts);
  // at least the largest restart's rows: budget >= per_max guarantees they fit
  const long long cap_rows = std::max<long long>(
      max_p, std::min<long long>(sum_p, (long long)((budget - (size_t)cap_R * restart_bytes) / row_bytes)));
  DevBuf b_qc, b_qg, b_small;
  CNMF_CUDA_CHECK(cudaMalloc(&b_qc.p, (size_t)cap_rows * ld_r * 8));
  CNMF_CUDA_CHECK(cudaMalloc(&b_qg.p, (size_t)cap_rows * ld_c * 8));
  CNMF_CUDA_CHECK(cudaMalloc(&b_small.p, (size_t)cap_R * restart_bytes + 256));
  double* Qc = static_cast<double*>(b_qc.p);
  double* Qg = static_cast<double*>(b_qg.p);
  double* part = static_cast<double*>(b_small.p);
  double* Lb = part + (size_t)cap_R * S_max * LSTRIDE;
  double* Lacc = Lb + (size_t)cap_R * LSTRIDE;
  double* Us = Lacc + (size_t)cap_R * LSTRIDE;
  double* Vs = Us + (size_t)cap_R * LSTRIDE;
  double* Sv = Vs + (size_t)cap_R * LSTRIDE;
  double* stats = Sv + (size_t)cap_R * PMAX;
  int* imeta = reinterpret_cast<int*>(stats + (size_t)cap_R * KMAX * 8);
  const int cap_K = cap_R * KMAX;
  Meta m{imeta, imeta + cap_R, imeta + 2 * cap_R, imeta + 3 * cap_R,
         reinterpret_cast<const uint32_t*>(imeta + 4 * cap_R), imeta + 5 * cap_R, imeta + 5 * cap_R + cap_K};
  std::vector<int> hmeta(5 * (size_t)cap_R + 2 * (size_t)cap_K);

  double* Qa = a_genes ? Qg : Qc;
  double* Qb = a_genes ? Qc : Qg;
  const int n_a = a_genes ? G : N, ld_a = a_genes ? ld_c : ld_r;
  const int n_b = a_genes ? N : G, ld_b = a_genes ? ld_r : ld_c;

  for (int cls : {7, 4}) {
    std::vector<int> todo;
    for (int r = 0; r < R; ++r)
      if (n_iter[r] == cls) todo.push_back(r);
    size_t i0 = 0;
    while (i0 < todo.size()) {
      // ---- one chunk
      size_t i1 = i0;
      int rows = 0;
      while (i1 < todo.size() && (int)(i1 - i0) < cap_R && rows + P[todo[i1]] <= cap_rows) rows += P[todo[i1++]];
      const int Rc = (int)(i1 - i0);
      int Kc = 0;
      for (int c = 0; c < Rc; ++c) {
        const int r = todo[i0 + c];
        hmeta[c] = c == 0 ? 0 : hmeta[c - 1] + P[todo[i0 + c - 1]];
        hmeta[cap_R + c] = P[r];
        hmeta[2 * cap_R + c] = ks[r];
        hmeta[3 * cap_R + c] = koff[r];
        hmeta[4 * cap_R + c] = (int)seeds[r];
        for (int j = 0; j < ks[r]; ++j, ++Kc) {
          hmeta[5 * cap_R + Kc] = c;
          hmeta[5 * cap_R + cap_K + Kc] = j;
        }
      }
      CNMF_CUDA_CHECK(cudaMemcpyAsync(imeta, hmeta.data(), hmeta.size() * sizeof(int), cudaMemcpyHostToDevice, s));
      CNMF_CUDA_CHECK(cudaMemsetAsync(Qc, 0, (size_t)rows * ld_r * 8, s));
      CNMF_CUDA_CHECK(cudaMemsetAsync(Qg, 0, (size_t)rows * ld_c * 8, s));

      auto gemm = [&](bool to_genes) -> int {
        const double* A = to_genes ? Qc : Qg;
        double* C = to_genes ? Qg : Qc;
        h->launches += 1;
        const int slot = h->prof_begin(s, 2.0 * rows * (double)N * G, 3);
        CNMF_TRY(launch_gemm_f64(A, to_genes ? ld_r : ld_c, rows, X, N, G, ld_c, to_genes, C, to_genes ? ld_c : ld_r, s));
        h->prof_end(s, slot);
        return 0;
      };
      // M Q: space a -> space b (cells when a is the genes); M^T Q: back
      auto mul_M = [&]() { return gemm(!a_genes); };
      auto mul_Mt = [&]() { return gemm(a_genes); };
      auto orth = [&](double* Q, int n, int ld, bool accumulate) -> int {
        const int S = gram_splits(n);
        for (int pass = 0; pass < 2; ++pass) {
          gram_kernel<<<dim3(S, Rc), 256, 0, s>>>(m, Q, ld, n, part);
          chol_kernel<<<Rc, 64, 0, s>>>(m, part, S, Lb, Lacc, accumulate ? pass + 1 : 0);
          apply_kernel<false><<<dim3((n + TILE - 1) / TILE, Rc), TILE, 0, s>>>(m, Q, ld, n, Lb);
          CNMF_CUDA_CHECK(cudaGetLastError());
          h->launches += 3;
        }
        return 0;
      };

      omega_kernel<<<Rc, LEGACY_GAUSS_THREADS, 0, s>>>(m, n_a, Qa, ld_a);
      CNMF_CUDA_CHECK(cudaGetLastError());
      h->launches += 1;
      for (int it = 0; it < cls; ++it) {
        CNMF_TRY(mul_M());
        CNMF_TRY(orth(Qb, n_b, ld_b, false));
        CNMF_TRY(mul_Mt());
        CNMF_TRY(orth(Qa, n_a, ld_a, false));
      }
      CNMF_TRY(mul_M());
      CNMF_TRY(orth(Qb, n_b, ld_b, false));         // Q
      CNMF_TRY(mul_Mt());                           // B^T as rows over space a
      CNMF_TRY(orth(Qa, n_a, ld_a, true));          // B = Lacc Q_B^T
      jacobi_kernel<<<Rc, 32, 0, s>>>(m, Lacc, Us, Vs, Sv);
      apply_kernel<true><<<dim3((n_b + TILE - 1) / TILE, Rc), TILE, 0, s>>>(m, Qb, ld_b, n_b, Us);
      apply_kernel<true><<<dim3((n_a + TILE - 1) / TILE, Rc), TILE, 0, s>>>(m, Qa, ld_a, n_a, Vs);
      stats_kernel<<<Kc, 256, 0, s>>>(m, Qc, ld_r, N, Qg, ld_c, G, stats);
      const double fill = init == CNMF_INIT_NNDSVDA ? avg : 0.0;
      compose_kernel<T><<<dim3((N + 255) / 256, Kc), 256, 0, s>>>(m, Qc, ld_r, N, true, stats, Sv, Wt, ld_r, fill);
      compose_kernel<T><<<dim3((G + 255) / 256, Kc), 256, 0, s>>>(m, Qg, ld_c, G, false, stats, Sv, H, ld_c, fill);
      h->launches += 6;
      if (init == CNMF_INIT_NNDSVDAR) {
        ar_fill_kernel<T><<<Rc, LEGACY_GAUSS_THREADS, 0, s>>>(m, Wt, ld_r, N, H, ld_c, G, Qc, ld_r, Qg, ld_c, avg);
        h->launches += 1;
      }
      CNMF_CUDA_CHECK(cudaGetLastError());
      CNMF_CUDA_CHECK(cudaStreamSynchronize(s));     // hmeta is rewritten by the next chunk
      i0 = i1;
    }
  }
  return 0;
}

}  // namespace

int nndsvd_starts_dev(cnmf_dataset_s* d, int R, const int* ks, const uint32_t* seeds, int init, float* Wt, float* H,
                      cudaStream_t s) {
  CNMF_TRY(require_dense(d, "nndsvd_init_dev"));
  return nndsvd_starts(d, d->X, R, ks, seeds, init, Wt, H, s);
}

int nndsvd_starts_dev(cnmf_dataset_s* d, int R, const int* ks, const uint32_t* seeds, int init, double* Wt, double* H,
                      cudaStream_t s) {
  CNMF_TRY(require_f64(d, "nndsvd_init_dev"));
  return nndsvd_starts(d, d->X64, R, ks, seeds, init, Wt, H, s);
}

}  // namespace cnmf

using namespace cnmf;

extern "C" {

int cnmf_nndsvd_init_dev(cnmf_dataset_t d, int n_restarts, const int32_t* ks, const uint32_t* seeds, int init,
                         float* Wt_dev, float* H_dev, void* stream) {
  CNMF_REQUIRE(d, "nndsvd_init_dev: NULL dataset");
  CNMF_CUDA_CHECK(cudaSetDevice(d->h->device));
  return nndsvd_starts_dev(d, n_restarts, ks, seeds, init, Wt_dev, H_dev, as_stream(stream));
}

int cnmf_nndsvd_chunk_limit(cnmf_handle_t h, int max_restarts) {
  CNMF_REQUIRE(h && max_restarts >= 0, "nndsvd_chunk_limit: bad arguments");
  h->nndsvd_chunk_restarts = max_restarts;
  return 0;
}

int cnmf_nndsvd_gemm_host(cnmf_dataset_t d, int to_genes, int M, const double* A_host, double* C_host, void* stream) {
  CNMF_REQUIRE(d && A_host && C_host && M > 0, "nndsvd_gemm_host: bad arguments");
  if (d->sparse) CNMF_TRY(require_dense(d, "nndsvd_gemm_host"));
  CNMF_CUDA_CHECK(cudaSetDevice(d->h->device));
  cudaStream_t s = as_stream(stream);
  const int n_in = to_genes ? d->n_rows : d->n_cols, ld_in = to_genes ? d->ld_r : d->ld_c;
  const int n_out = to_genes ? d->n_cols : d->n_rows, ld_out = to_genes ? d->ld_c : d->ld_r;
  DevBuf a, c;
  CNMF_CUDA_CHECK(cudaMalloc(&a.p, (size_t)M * ld_in * 8));
  CNMF_CUDA_CHECK(cudaMalloc(&c.p, (size_t)M * ld_out * 8));
  CNMF_CUDA_CHECK(cudaMemsetAsync(a.p, 0, (size_t)M * ld_in * 8, s));
  CNMF_CUDA_CHECK(cudaMemsetAsync(c.p, 0xff, (size_t)M * ld_out * 8, s));   // NaN pattern: unwritten outputs show up
  CNMF_CUDA_CHECK(cudaMemcpy2DAsync(a.p, (size_t)ld_in * 8, A_host, (size_t)n_in * 8, (size_t)n_in * 8, M,
                                    cudaMemcpyHostToDevice, s));
  const double* A = static_cast<double*>(a.p);
  double* C = static_cast<double*>(c.p);
  if (d->form == Form::FP64)     // float64 dataset: the <*, double> instantiation the float64 solver runs, on X64
    CNMF_TRY(launch_gemm_f64(A, ld_in, M, d->X64, d->n_rows, d->n_cols, d->ld_c, to_genes != 0, C, ld_out, s));
  else
    CNMF_TRY(launch_gemm_f64(A, ld_in, M, d->X, d->n_rows, d->n_cols, d->ld_c, to_genes != 0, C, ld_out, s));
  d->h->launches += 1;
  CNMF_CUDA_CHECK(cudaMemcpy2DAsync(C_host, (size_t)n_out * 8, c.p, (size_t)ld_out * 8, (size_t)n_out * 8, M,
                                    cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
  return 0;
}

}  // extern "C"
