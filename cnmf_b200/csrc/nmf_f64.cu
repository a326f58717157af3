// Kernels and ops of the batched solve on float64 datasets (precision "fp64"): the Frobenius MU and CD iterations of
// solve_frobenius (nmf_engine.cu) with every value in fp64 -- factors, products, Grams, scalars -- as scikit-learn
// computes on the reference's float64 X.
//
// One outer iteration, all restarts together (packed slot layout of nmf_kernels.cuh, factors as doubles):
//   NUM_r = Fc * X^T            gemm_f64 (DMMA), M = sum k, reduction over n_c in ascending K tiles
//   Fr   <- update(Fr, NUM_r, Gram(Fc))         mu64_kernel / cd64_kernel, one thread per item
//   Gram(Fr)                                    gram64_kernel + finalize
//   NUM_c = Fr * X              gemm_f64 in the other orientation (same X, no transposed copy)
//   Fc   <- update(Fc, NUM_c, Gram(Fr)), Gram(Fc)
// The convergence kernels are the fp32 solver's (launch_mu_check / launch_cd_check on fp64 Grams and scalars).
//
// Determinism: every block of the update, cross and Gram kernels covers a fixed range of items whose size depends on
// the item count only (F64_ITEMS, F64_GRAM_COLS), its partial sums are reduced in a fixed tree, and finalize adds the
// partials in chunk order.  The GEMM sums a row's K tiles in ascending order wherever the row sits.  A restart's result
// is therefore bit-identical whether it is solved alone or beside any other restarts, compacted or not.
#include <algorithm>
#include <cmath>
#include <cstring>

#include "nmf_f64.h"

namespace cnmf {

namespace {

constexpr int F64_THREADS = F64_ITEMS;      // one item per thread in the update / cross kernels
constexpr int F64_GRAM_TILE = 64;           // items staged in shared memory per pass of the Gram kernel
constexpr double EPSILON_F32_D = 1.1920928955078125e-07;   // np.finfo(np.float32).eps, sklearn _nmf.py:32

// fixed-tree block sum of one value per thread (F64_THREADS threads); the result is valid in thread 0
__device__ __forceinline__ double block_sum(double v, double* red) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) red[warp] = v;
  __syncthreads();
  double a = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < F64_THREADS / 32; ++w) a += red[w];
  return a;
}

// gram_partial[(rid * gridDim.x + chunk) * kp*kp + c*KP + i] = sum over the chunk's items of F[c, j] F[i, j]
// (KP = K rounded up to 4, entries with c or i >= K written as 0: the layout finalize_kernel reads)
__global__ void __launch_bounds__(F64_THREADS)
gram64_kernel(F64View f, BatchMeta b, double* __restrict__ gram_partial) {
  const int slot = blockIdx.y;
  const int r = b.rid[slot];
  if (b.done[r]) return;
  const int K = b.k[slot], o = b.off[slot];
  const int KP = round_up(K, 4);
  __shared__ double tile[KMAX][F64_GRAM_TILE + 1];
  const int j0 = blockIdx.x * F64_GRAM_COLS, j1 = min(f.n, j0 + F64_GRAM_COLS);
  constexpr int PER = (KMAX * KMAX + F64_THREADS - 1) / F64_THREADS;
  double acc[PER];
#pragma unroll
  for (int q = 0; q < PER; ++q) acc[q] = 0.0;
  for (int t0 = j0; t0 < j1; t0 += F64_GRAM_TILE) {
    __syncthreads();
    for (int e = threadIdx.x; e < K * F64_GRAM_TILE; e += F64_THREADS) {
      const int c = e / F64_GRAM_TILE, j = e % F64_GRAM_TILE;
      tile[c][j] = t0 + j < j1 ? f.F[(long long)(o + c) * f.ld + t0 + j] : 0.0;
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < PER; ++q) {
      const int e = threadIdx.x + q * F64_THREADS;
      if (e < K * K) {
        const int c = e / K, i = e % K;
        double a = acc[q];
        for (int j = 0; j < F64_GRAM_TILE; ++j) a = fma(tile[c][j], tile[i][j], a);
        acc[q] = a;
      }
    }
  }
  double* out = gram_partial + ((long long)r * gridDim.x + blockIdx.x) * (b.kp * b.kp);
#pragma unroll
  for (int q = 0; q < PER; ++q) {
    const int e = threadIdx.x + q * F64_THREADS;
    if (e < K * K) out[(e / K) * KP + e % K] = acc[q];
  }
  for (int e = threadIdx.x; e < KP * KP; e += F64_THREADS)
    if (e / KP >= K || e % KP >= K) out[e] = 0.0;
}

// scal_partial[rid * gridDim.x + chunk] = sum over the chunk's items j and c < K of NUM[c, j] F[c, j]
__global__ void __launch_bounds__(F64_THREADS)
cross64_kernel(F64View f, const double* __restrict__ NUM, BatchMeta b, double* __restrict__ scal_partial) {
  const int slot = blockIdx.y;
  const int r = b.rid[slot];
  if (b.done[r]) return;
  __shared__ double red[F64_THREADS / 32];
  const int K = b.k[slot], o = b.off[slot];
  const int j = blockIdx.x * F64_ITEMS + threadIdx.x;
  double a = 0.0;
  if (j < f.n)
    for (int c = 0; c < K; ++c) {
      const long long e = (long long)(o + c) * f.ld + j;
      a = fma(NUM[e], f.F[e], a);
    }
  a = block_sum(a, red);
  if (threadIdx.x == 0) scal_partial[(long long)r * gridDim.x + blockIdx.x] = a;
}

// the restart's K x K Gram (fp64, [c * KMAX + i]) into shared memory, l2 added on the diagonal
__device__ __forceinline__ void load_gram(const double* __restrict__ gram_in, int r, int K, double l2, double* G) {
  for (int e = threadIdx.x; e < K * K; e += F64_THREADS) {
    const int c = e / K, i = e % K;
    G[c * KMAX + i] = gram_in[(long long)r * KMAX * KMAX + c * KMAX + i] + (c == i ? l2 : 0.0);
  }
  __syncthreads();
}

// Multiplicative update of one item (sklearn _nmf.py:535-549,610-624 / :633-635,696-721):
//   F[c] <- F[c] * (NUM[c] / den),  den = sum_i G[c, i] F[i] + l1 + l2 F[c],  den == 0 -> float32 eps
// every component from the old values; returns <NUM, F_new> over the item
template <int KP>
__device__ __forceinline__ double mu64_item(double* F, const double* __restrict__ NUM, unsigned ld, const double* G,
                                            int K, double l1, double l2) {
  double fv[KP];
#pragma unroll
  for (int i = 0; i < KP; ++i) fv[i] = i < K ? F[i * ld] : 0.0;
  double s = 0.0;
#pragma unroll
  for (int c = 0; c < KP; ++c) {
    if (c < K) {
      double den = 0.0;
#pragma unroll
      for (int i = 0; i < KP; ++i)
        if (i < K) den = fma(G[c * KMAX + i], fv[i], den);
      den = den + l1;
      den = den + l2 * fv[c];
      if (den == 0.0) den = EPSILON_F32_D;
      const double num = NUM[c * ld];
      const double out = fv[c] * (num / den);
      F[c * ld] = out;
      s = fma(num, out, s);
    }
  }
  return s;
}

// One coordinate-descent sweep over the K coordinates of one item (sklearn _cdnmf_fast.pyx:8-37, shuffle=False):
// G carries l2 on its diagonal, B = NUM - l1; returns sum |projected gradient|
template <int KP>
__device__ __forceinline__ double cd64_item(double* F, const double* __restrict__ NUM, unsigned ld, const double* G,
                                            int K, double l1) {
  double fv[KP];
#pragma unroll
  for (int i = 0; i < KP; ++i) fv[i] = i < K ? F[i * ld] : 0.0;
  double viol = 0.0;
#pragma unroll
  for (int t = 0; t < KP; ++t) {
    if (t < K) {
      double grad = -(NUM[t * ld] - l1);
#pragma unroll
      for (int i = 0; i < KP; ++i)
        if (i < K) grad = fma(G[t * KMAX + i], fv[i], grad);
      const double pg = fv[t] == 0.0 ? fmin(0.0, grad) : grad;
      viol += fabs(pg);
      const double hess = G[t * KMAX + t];
      if (hess != 0.0) fv[t] = fmax(fv[t] - grad / hess, 0.0);
    }
  }
#pragma unroll
  for (int i = 0; i < KP; ++i)
    if (i < K) F[i * ld] = fv[i];
  return viol;
}

// one update launch: grid (ceil(n / F64_ITEMS), live slots).  scal_partial (optional): MU <NUM, F_new>, CD sum
// |projected gradient| per block, [rid * gridDim.x + chunk]
template <bool CD>
__global__ void __launch_bounds__(F64_THREADS)
update64_kernel(F64View f, const double* __restrict__ NUM, const double* __restrict__ gram_in, BatchMeta b, double l1,
                double l2, double* __restrict__ scal_partial) {
  const int slot = blockIdx.y;
  const int r = b.rid[slot];
  if (b.done[r]) return;
  __shared__ double G[KMAX * KMAX];
  __shared__ double red[F64_THREADS / 32];
  const int K = b.k[slot], o = b.off[slot];
  load_gram(gram_in, r, K, CD ? l2 : 0.0, G);
  const int j = blockIdx.x * F64_ITEMS + threadIdx.x;
  double s = 0.0;
  if (j < f.n) {
    double* F = f.F + (long long)o * f.ld + j;
    const double* N = NUM + (long long)o * f.ld + j;
    const unsigned ld = (unsigned)f.ld;
    if (CD) {
      if (K <= 8) s = cd64_item<8>(F, N, ld, G, K, l1);
      else if (K <= 16) s = cd64_item<16>(F, N, ld, G, K, l1);
      else s = cd64_item<32>(F, N, ld, G, K, l1);
    } else {
      if (K <= 8) s = mu64_item<8>(F, N, ld, G, K, l1, l2);
      else if (K <= 16) s = mu64_item<16>(F, N, ld, G, K, l1, l2);
      else s = mu64_item<32>(F, N, ld, G, K, l1, l2);
    }
  }
  if (scal_partial) {
    s = block_sum(s, red);
    if (threadIdx.x == 0) scal_partial[(long long)r * gridDim.x + blockIdx.x] = s;
  }
}

__global__ void fill64_kernel(double* p, double v, int rows, int n, int ld) {
  const long long total = (long long)rows * n;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
    p[(i / n) * ld + (i % n)] = v;
}

// sum and sum of squares of the valid region, one block per strip of rows, then the strips in order
__global__ void __launch_bounds__(F64_THREADS)
sums64_kernel(const double* __restrict__ X, int rows, int cols, int ld, int rows_per_block, double* __restrict__ part) {
  __shared__ double red[F64_THREADS / 32];
  const int r0 = blockIdx.x * rows_per_block, r1 = min(rows, r0 + rows_per_block);
  double s = 0.0, q = 0.0;
  for (int r = r0; r < r1; ++r)
    for (int c = threadIdx.x; c < cols; c += F64_THREADS) {
      const double v = X[(long long)r * ld + c];
      s += v;
      q = fma(v, v, q);
    }
  const double ts = block_sum(s, red);
  __syncthreads();
  const double tq = block_sum(q, red);
  if (threadIdx.x == 0) {
    part[2 * blockIdx.x] = ts;
    part[2 * blockIdx.x + 1] = tq;
  }
}

__global__ void sums64_final_kernel(const double* __restrict__ part, int nblocks, double* __restrict__ out2) {
  double s = 0.0, q = 0.0;
  for (int i = 0; i < nblocks; ++i) {
    s += part[2 * i];
    q += part[2 * i + 1];
  }
  out2[0] = s;
  out2[1] = q;
}

}  // namespace

int f64_gram(const F64Launch& L, const F64View& f, const BatchMeta& b, double* part, double* gram) {
  const int gch = f64_gram_chunks(f.n);
  gram64_kernel<<<dim3(gch, b.R), F64_THREADS, 0, L.s>>>(f, b, part);
  CNMF_CUDA_CHECK(cudaGetLastError());
  L.h->launches += 2;
  return launch_finalize(part, gram, nullptr, nullptr, gch, b, L.s);
}

int f64_cross(const F64Launch& L, const F64View& f, const double* NUM, const BatchMeta& b, double* part, double* out) {
  const int ch = f64_chunks(f.n);
  cross64_kernel<<<dim3(ch, b.R), F64_THREADS, 0, L.s>>>(f, NUM, b, part);
  CNMF_CUDA_CHECK(cudaGetLastError());
  L.h->launches += 2;
  return launch_finalize(nullptr, nullptr, part, out, ch, b, L.s);
}

int f64_update(const F64Launch& L, bool cd, const F64View& f, const double* NUM, const double* gram_in,
               const BatchMeta& b, double l1, double l2, double* part, double* scal) {
  const int ch = f64_chunks(f.n);
  if (!scal) part = nullptr;
  L.h->launches += 1;
  const int slot = L.h->prof_begin(L.s, 8.0 * (double)L.SK * (double)f.n * 3.0, 1);
  if (!cd) update64_kernel<false><<<dim3(ch, b.R), F64_THREADS, 0, L.s>>>(f, NUM, gram_in, b, l1, l2, part);
  else update64_kernel<true><<<dim3(ch, b.R), F64_THREADS, 0, L.s>>>(f, NUM, gram_in, b, l1, l2, part);
  L.h->prof_end(L.s, slot);
  CNMF_CUDA_CHECK(cudaGetLastError());
  if (!scal) return 0;
  L.h->launches += 1;
  return launch_finalize(nullptr, nullptr, part, scal, ch, b, L.s);
}

int matrix_sums_f64(cnmf_handle_s* h, const double* X, int rows, int cols, int ld, double* out_host, cudaStream_t s) {
  const int rpb = 64;
  const int nb = (rows + rpb - 1) / rpb;
  double* part = static_cast<double*>(h->dev_buf("dataset.sums64", sizeof(double) * (2 * (size_t)nb + 2)));
  if (!part) return -2;
  sums64_kernel<<<nb, F64_THREADS, 0, s>>>(X, rows, cols, ld, rpb, part);
  sums64_final_kernel<<<1, 1, 0, s>>>(part, nb, part + 2 * nb);
  CNMF_CUDA_CHECK(cudaGetLastError());
  h->launches += 2;
  CNMF_CUDA_CHECK(cudaMemcpyAsync(out_host, part + 2 * nb, 2 * sizeof(double), cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
  return 0;
}

int fill_f64(double* p, double v, int rows, int n, int ld, cudaStream_t s) {
  fill64_kernel<<<NUM_SMS * 4, 256, 0, s>>>(p, v, rows, n, ld);
  CNMF_CUDA_CHECK(cudaGetLastError());
  return 0;
}

F64Ops::F64Ops(FroSolve<double>& b_, const cnmf_nmf_params& p) : b(b_), cd(p.solver == CNMF_SOLVER_CD) {
  l1[0] = p.l1_reg_W; l2[0] = p.l2_reg_W; l1[1] = p.l1_reg_H; l2[1] = p.l2_reg_H;
  chunks[0] = f64_chunks(b.v.n_r);
  chunks[1] = f64_chunks(b.v.n_c);
  chunks_cap = std::max(chunks[0], chunks[1]);
  gram_part_elems = (size_t)b.R0 * std::max(f64_gram_chunks(b.v.n_r), f64_gram_chunks(b.v.n_c)) * b.kp * b.kp;
}

int F64Ops::alloc() {
  b.NUM[0] = static_cast<double*>(b.h->dev_buf("solve.NUMr64", sizeof(double) * (size_t)b.SK0 * b.v.ld_r));
  b.NUM[1] = b.io.update_cols ? static_cast<double*>(b.h->dev_buf("solve.NUMc64", sizeof(double) * (size_t)b.SK0 * b.v.ld_c))
                              : nullptr;
  return !b.NUM[0] || (b.io.update_cols && !b.NUM[1]) ? -2 : 0;
}

// NUM_r = Fc * X^T over the row items (reduction over n_c); NUM_c = Fr * X over the column items
int F64Ops::gemm(int side) {
  const DataView& v = b.v;
  const bool rows = side == 0;
  // untransposed: rows = cells, X^T products run over the genes (to_genes = false)
  const bool to_genes = rows ? v.transposed : !v.transposed;
  b.h->launches += 1;
  const int slot = b.h->prof_begin(b.s, 2.0 * (double)b.SK * (double)v.n_r * (double)v.n_c, 4);
  const int nrow_x = v.transposed ? v.n_c : v.n_r, ncol_x = v.transposed ? v.n_r : v.n_c;
  const int ldx = v.transposed ? v.ld_r : v.ld_c;
  const int rc = launch_gemm_f64(b.F[1 - side], b.ld(1 - side), b.SK, v.X64, nrow_x, ncol_x, ldx, to_genes, b.NUM[side],
                                 b.ld(side), b.s);
  b.h->prof_end(b.s, slot);
  return rc;
}

int F64Ops::gram(int side, const BatchMeta& m) {
  return f64_gram(F64Launch{b.h, b.s, b.SK}, F64View{b.F[side], b.n(side), b.ld(side)}, m, b.gram_part[side], b.gram[side]);
}

int F64Ops::grams(const BatchMeta& m) {
  CNMF_TRY(gram(0, m));
  return gram(1, m);
}

int F64Ops::cross(int side, const BatchMeta& m, double* out) {
  return f64_cross(F64Launch{b.h, b.s, b.SK}, F64View{b.F[side], b.n(side), b.ld(side)}, b.NUM[side], m,
                   b.scal_part[side], out);
}

int F64Ops::update(int side, bool /* want_gram: the driver runs gram() after every update */, bool want_scal,
                   double* scal) {
  return f64_update(F64Launch{b.h, b.s, b.SK}, cd, F64View{b.F[side], b.n(side), b.ld(side)}, b.NUM[side],
                    b.gram[1 - side], b.bm(), l1[side], l2[side], b.scal_part[side], want_scal ? scal : nullptr);
}

}  // namespace cnmf
