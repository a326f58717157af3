// Batched NMF solver of float64 datasets (precision "fp64"): the Frobenius MU and CD iterations of nmf_engine.cu with
// every value in fp64 -- factors, products, Grams, scalars -- as scikit-learn computes on the reference's float64 X.
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

int solve_batched_f64(cnmf_handle_s* h, const DataView& v, SolveIO& io, const cnmf_nmf_params& p, cudaStream_t s) {
  const int R0 = io.R;
  CNMF_REQUIRE(v.form == Form::FP64 && v.X64, "solve: the float64 solver needs a float64 dataset");
  CNMF_REQUIRE(p.beta_loss == CNMF_LOSS_FROBENIUS, "solve: float64 datasets support beta_loss = frobenius only");
  CNMF_REQUIRE(R0 > 0 && (int)io.ks.size() == R0, "solve: bad restart list");
  CNMF_REQUIRE(p.solver == CNMF_SOLVER_MU || p.solver == CNMF_SOLVER_CD, "solve: unknown solver");
  CNMF_REQUIRE(p.max_iter >= 1, "solve: max_iter must be >= 1");
  CNMF_REQUIRE(io.Fr64 && io.Fc64, "solve: float64 factors missing");
  const bool mu = p.solver == CNMF_SOLVER_MU;

  // ---- slot tables (host mirrors); slot s holds restart rid[s] at packed rows [off[s], off[s]+k[s])
  std::vector<int> off0(R0), s_off(R0), s_k(io.ks), s_rid(R0);
  int SK0 = 0, kmax = 0;
  for (int r = 0; r < R0; ++r) {
    CNMF_REQUIRE(io.ks[r] >= 1 && io.ks[r] <= KMAX, "solve: n_components must be in [1, 32] on the CUDA path");
    off0[r] = s_off[r] = SK0;
    s_rid[r] = r;
    SK0 += io.ks[r];
    kmax = std::max(kmax, io.ks[r]);
  }
  int R = R0, SK = SK0;
  const int kp = round_up(kmax, 4);      // partial Gram stride kp * kp (finalize_kernel)
  auto pack_offsets = [&](const std::vector<int>& kk, std::vector<int>& offs) -> int {
    int pos = 0;
    offs.clear();
    for (int k : kk) {
      offs.push_back(pos);
      pos += k;
    }
    return pos;
  };
  const int chunks_r = f64_chunks(v.n_r), chunks_c = f64_chunks(v.n_c);
  const int gchunks_r = f64_gram_chunks(v.n_r), gchunks_c = f64_gram_chunks(v.n_c);
  const int chunks_cap = std::max(chunks_r, chunks_c), gchunks_cap = std::max(gchunks_r, gchunks_c);

  // ---- workspace
  int* d_meta = static_cast<int*>(h->dev_buf("solve.meta", sizeof(int) * 8 * R0));
  double* d_state = static_cast<double*>(h->dev_buf("solve.state", sizeof(double) * 8 * R0));
  double* d_gram = static_cast<double*>(h->dev_buf("solve.gram", sizeof(double) * 2 * R0 * KMAX * KMAX));
  const size_t gpart_elems = (size_t)R0 * gchunks_cap * kp * kp;
  double* d_gram_part = static_cast<double*>(h->dev_buf("solve.gram_part", sizeof(double) * 2 * gpart_elems));
  double* d_scal_part = static_cast<double*>(h->dev_buf("solve.scal_part", sizeof(double) * 2 * (size_t)R0 * chunks_cap));
  double* NUMr = static_cast<double*>(h->dev_buf("solve.NUMr64", sizeof(double) * (size_t)SK0 * v.ld_r));
  double* NUMc = io.update_cols ? static_cast<double*>(h->dev_buf("solve.NUMc64", sizeof(double) * (size_t)SK0 * v.ld_c))
                                : nullptr;
  if (!d_meta || !d_state || !d_gram || !d_gram_part || !d_scal_part || !NUMr || (io.update_cols && !NUMc)) return -2;

  int* d_off = d_meta;
  int* d_k = d_meta + R0;
  int* d_rid = d_meta + 2 * R0;
  int* d_done = d_meta + 3 * R0;
  int* d_niter = d_meta + 4 * R0;
  auto upload_slots = [&]() -> int {
    std::vector<int> hm(3 * R0, 0);
    std::memcpy(hm.data(), s_off.data(), sizeof(int) * R);
    std::memcpy(hm.data() + R0, s_k.data(), sizeof(int) * R);
    std::memcpy(hm.data() + 2 * R0, s_rid.data(), sizeof(int) * R);
    CNMF_CUDA_CHECK(cudaMemcpyAsync(d_meta, hm.data(), sizeof(int) * 3 * R0, cudaMemcpyHostToDevice, s));
    CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
    return 0;
  };
  CNMF_TRY(upload_slots());
  CNMF_CUDA_CHECK(cudaMemsetAsync(d_done, 0, sizeof(int) * 2 * R0, s));   // done, n_iter
  CNMF_CUDA_CHECK(cudaMemsetAsync(d_state, 0, sizeof(double) * 8 * R0, s));
  ConvState st{d_state, d_state + R0, d_state + 2 * R0, d_done, d_niter};
  double* d_crossA = d_state + 3 * R0;
  double* d_crossB = d_state + 4 * R0;
  double* d_gramR = d_gram;
  double* d_gramC = d_gram + (size_t)R0 * KMAX * KMAX;
  double* d_scalA = d_scal_part;
  double* d_scalB = d_scal_part + (size_t)R0 * chunks_cap;
  double* d_gpartR = d_gram_part;
  double* d_gpartC = d_gram_part + gpart_elems;

  double *wFr = io.Fr64, *wFc = io.Fc64;
  double *aFr = nullptr, *aFc = nullptr, *resFr = nullptr, *resFc = nullptr;
  bool compacted = false;

  auto bm = [&]() { return BatchMeta{d_off, d_k, d_rid, d_done, R, kp}; };
  auto fr = [&]() { return F64View{wFr, v.n_r, v.ld_r}; };
  auto fc = [&]() { return F64View{wFc, v.n_c, v.ld_c}; };

  auto L = [&]() { return F64Launch{h, s, SK}; };

  auto gram = [&](const F64View& f, int side_is_c, const BatchMeta& b) -> int {
    return f64_gram(L(), f, b, side_is_c ? d_gpartC : d_gpartR, side_is_c ? d_gramC : d_gramR);
  };
  auto cross = [&](const F64View& f, const double* NUM, int side_is_c, double* out, const BatchMeta& b) -> int {
    return f64_cross(L(), f, NUM, b, side_is_c ? d_scalB : d_scalA, out);
  };
  // update of one factor; scal (optional) receives MU <NUM, F_new> / CD sum |projected gradient| per restart
  auto update = [&](const F64View& f, const double* NUM, int side_is_c, const double* gram_in, double l1, double l2,
                    double* scal) -> int {
    return f64_update(L(), !mu, f, NUM, gram_in, bm(), l1, l2, side_is_c ? d_scalB : d_scalA, scal);
  };
  // NUM_r = Fc * X^T over the row items (reduction over n_c); NUM_c = Fr * X over the column items
  auto gemm = [&](bool rows) -> int {
    const double* A = rows ? wFc : wFr;
    const int lda = rows ? v.ld_c : v.ld_r;
    double* C = rows ? NUMr : NUMc;
    const int ldc = rows ? v.ld_r : v.ld_c;
    // untransposed: rows = cells, X^T products run over the genes (to_genes = false)
    const bool to_genes = rows ? v.transposed : !v.transposed;
    h->launches += 1;
    const int slot = h->prof_begin(s, 2.0 * (double)SK * (double)v.n_r * (double)v.n_c, 4);
    const int nrow_x = v.transposed ? v.n_c : v.n_r, ncol_x = v.transposed ? v.n_r : v.n_c;
    const int ldx = v.transposed ? v.ld_r : v.ld_c;
    const int rc = launch_gemm_f64(A, lda, SK, v.X64, nrow_x, ncol_x, ldx, to_genes, C, ldc, s);
    h->prof_end(s, slot);
    return rc;
  };

  constexpr int GATHER_SLOTS = 12;
  int* h_gidx = static_cast<int*>(h->host_buf("solve.gather_idx", sizeof(int) * 3 * (size_t)R0 * GATHER_SLOTS));
  int* d_gidx = static_cast<int*>(h->dev_buf("solve.gather_didx", sizeof(int) * 3 * (size_t)R0 * GATHER_SLOTS));
  if (!h_gidx || !d_gidx) return -2;
  int gslot = 0;
  // fp64 rows gathered as rows of 2 * ld floats: a bit copy
  auto gather = [&](const double* src, double* dst, const std::vector<int>& so, const std::vector<int>& dof,
                    const std::vector<int>& kk, int ld) -> int {
    const int cnt = (int)kk.size();
    if (cnt == 0) return 0;
    if (gslot == GATHER_SLOTS) {
      CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
      gslot = 0;
    }
    int* hm = h_gidx + (size_t)gslot * 3 * R0;
    int* dm = d_gidx + (size_t)gslot * 3 * R0;
    ++gslot;
    std::memcpy(hm, so.data(), sizeof(int) * cnt);
    std::memcpy(hm + R0, dof.data(), sizeof(int) * cnt);
    std::memcpy(hm + 2 * R0, kk.data(), sizeof(int) * cnt);
    CNMF_CUDA_CHECK(cudaMemcpyAsync(dm, hm, sizeof(int) * 3 * R0, cudaMemcpyHostToDevice, s));
    h->launches += 1;
    return launch_gather_rows(reinterpret_cast<const float*>(src), dm, reinterpret_cast<float*>(dst), dm + R0, dm + 2 * R0,
                              cnt, 2 * ld, s);
  };

  const double normX2 = v.sum_sq;
  double* d_cd_err = d_state + 7 * R0;
  // CD: ||X - Fr^T Fc||_F of the restarts still packed, in the trace form, into d_cd_err
  auto cd_final_error = [&]() -> int {
    int* d_zero = static_cast<int*>(h->dev_buf("solve.zero", sizeof(int) * 2 * R0));
    if (!d_zero) return -2;
    CNMF_CUDA_CHECK(cudaMemsetAsync(d_zero, 0, sizeof(int) * 2 * R0, s));
    BatchMeta bm0{d_off, d_k, d_rid, d_zero, R, kp};
    CNMF_TRY(gram(fr(), 0, bm0));
    CNMF_TRY(gram(fc(), 1, bm0));
    if (io.update_cols) CNMF_TRY(cross(fc(), NUMc, 1, d_crossB, bm0));
    else CNMF_TRY(cross(fr(), NUMr, 0, d_crossB, bm0));
    ConvState scratch{d_state + 5 * R0, d_state + 6 * R0, d_cd_err, d_zero, d_zero + R0};
    h->launches += 1;
    return launch_mu_check(scratch, d_crossB, d_gramR, d_gramC, normX2, bm0, 0, 0.0, p.max_iter, s);
  };

  std::vector<int> h_done(R0, 0);
  // drop converged restarts from the packed arrays when that saves a 64-row GEMM tile (or >= 1/8 of the rows)
  auto maybe_compact = [&]() -> int {
    if (!io.update_cols) return 0;
    std::vector<int> lk, lo;
    for (int sl = 0; sl < R; ++sl)
      if (!h_done[s_rid[sl]]) lk.push_back(s_k[sl]);
    const int new_rows = pack_offsets(lk, lo);
    if (new_rows == SK || new_rows == 0) return 0;
    const bool saves_tile = (new_rows + 63) / 64 < (SK + 63) / 64;
    if (!saves_tile && new_rows > SK - SK / 8) return 0;
    if (!mu) CNMF_TRY(cd_final_error());    // restarts leaving the packed arrays get their ||X - WH||_F now
    if (!aFr) {
      const size_t nr = (size_t)SK0 * v.ld_r * 8, nc = (size_t)SK0 * v.ld_c * 8;
      aFr = static_cast<double*>(h->dev_buf("solve.alt.Fr64", nr));
      aFc = static_cast<double*>(h->dev_buf("solve.alt.Fc64", nc));
      resFr = static_cast<double*>(h->dev_buf("solve.res.Fr64", nr));
      resFc = static_cast<double*>(h->dev_buf("solve.res.Fc64", nc));
      if (!aFr || !aFc || !resFr || !resFc) return -2;
    }
    std::vector<int> f_src, f_dst, f_k, l_src, l_dst, l_k, n_rid;
    for (int sl = 0; sl < R; ++sl) {
      const int rid = s_rid[sl];
      if (h_done[rid]) {
        f_src.push_back(s_off[sl]); f_dst.push_back(off0[rid]); f_k.push_back(s_k[sl]);
      } else {
        l_src.push_back(s_off[sl]); l_k.push_back(s_k[sl]); n_rid.push_back(rid);
      }
    }
    const int pos = pack_offsets(l_k, l_dst);
    CNMF_TRY(gather(wFr, resFr, f_src, f_dst, f_k, v.ld_r));
    CNMF_TRY(gather(wFc, resFc, f_src, f_dst, f_k, v.ld_c));
    CNMF_TRY(gather(wFr, aFr, l_src, l_dst, l_k, v.ld_r));
    CNMF_TRY(gather(wFc, aFc, l_src, l_dst, l_k, v.ld_c));
    std::swap(wFr, aFr);
    std::swap(wFc, aFc);
    R = (int)l_k.size();
    SK = pos;
    std::copy(l_dst.begin(), l_dst.end(), s_off.begin());
    std::copy(l_k.begin(), l_k.end(), s_k.begin());
    std::copy(n_rid.begin(), n_rid.end(), s_rid.begin());
    CNMF_TRY(upload_slots());
    gslot = 0;
    compacted = true;
    return 0;
  };
  auto poll_all_done = [&]() -> int {   // 1 = all done, 0 = not yet, <0 error
    CNMF_CUDA_CHECK(cudaMemcpyAsync(h_done.data(), d_done, sizeof(int) * R0, cudaMemcpyDeviceToHost, s));
    CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
    for (int sl = 0; sl < R; ++sl)
      if (!h_done[s_rid[sl]]) return maybe_compact();
    return 1;
  };

  const double l1W = p.l1_reg_W, l2W = p.l2_reg_W, l1H = p.l1_reg_H, l2H = p.l2_reg_H;
  if (mu) {
    // ---------------- multiplicative update (sklearn _nmf.py:726-888) ----------------
    CNMF_TRY(gram(fc(), 1, bm()));
    CNMF_TRY(gram(fr(), 0, bm()));
    if (io.update_cols) {
      CNMF_TRY(gemm(false));
      CNMF_TRY(cross(fc(), NUMc, 1, d_crossB, bm()));
    } else {
      CNMF_TRY(gemm(true));             // H fixed: X H^T is formed once (sklearn caches XHt, _nmf.py:537-548)
      CNMF_TRY(cross(fr(), NUMr, 0, d_crossB, bm()));
    }
    h->launches += 1;
    CNMF_TRY(launch_mu_check(st, d_crossB, d_gramR, d_gramC, normX2, bm(), 0, p.tol, p.max_iter, s));
    for (int it = 1; it <= p.max_iter; ++it) {
      const bool check = (p.tol > 0 && it % 10 == 0) || it == p.max_iter;
      if (io.update_cols) {
        CNMF_TRY(gemm(true));
        CNMF_TRY(update(fr(), NUMr, 0, d_gramC, l1W, l2W, nullptr));
        CNMF_TRY(gram(fr(), 0, bm()));
        CNMF_TRY(gemm(false));
        CNMF_TRY(update(fc(), NUMc, 1, d_gramR, l1H, l2H, check ? d_crossB : nullptr));
        CNMF_TRY(gram(fc(), 1, bm()));
      } else {
        CNMF_TRY(update(fr(), NUMr, 0, d_gramC, l1W, l2W, check ? d_crossB : nullptr));
        if (check) CNMF_TRY(gram(fr(), 0, bm()));
      }
      if (check) {
        h->launches += 1;
        const double tol_eff = (p.tol > 0 && it % 10 == 0) ? p.tol : -1.0;
        CNMF_TRY(launch_mu_check(st, d_crossB, d_gramR, d_gramC, normX2, bm(), it, tol_eff, p.max_iter, s));
        const int all = poll_all_done();
        if (all < 0) return all;
        if (all) break;
      }
    }
  } else {
    // ---------------- coordinate descent (sklearn _nmf.py:399-518, shuffle=False) ----------------
    const int poll_every = 4;
    for (int it = 1; it <= p.max_iter; ++it) {
      if (it == 1) CNMF_TRY(gram(fc(), 1, bm()));
      if (io.update_cols || it == 1) CNMF_TRY(gemm(true));
      CNMF_TRY(update(fr(), NUMr, 0, d_gramC, l1W, l2W, d_crossA));
      if (io.update_cols) {
        CNMF_TRY(gram(fr(), 0, bm()));
        CNMF_TRY(gemm(false));
        CNMF_TRY(update(fc(), NUMc, 1, d_gramR, l1H, l2H, d_crossB));
        CNMF_TRY(gram(fc(), 1, bm()));
      }
      h->launches += 1;
      CNMF_TRY(launch_cd_check(st, d_crossA, io.update_cols ? d_crossB : nullptr, bm(), it, p.tol, p.max_iter, s));
      if (it % poll_every == 0 || it == p.max_iter) {
        const int all = poll_all_done();
        if (all < 0) return all;
        if (all) break;
      }
    }
  }

  double* d_err = st.last;
  if (!mu) {
    CNMF_TRY(cd_final_error());
    d_err = d_cd_err;
  }
  if (compacted) {
    std::vector<int> so(s_off.begin(), s_off.begin() + R), ko(s_k.begin(), s_k.begin() + R), dof(R);
    for (int sl = 0; sl < R; ++sl) dof[sl] = off0[s_rid[sl]];
    CNMF_TRY(gather(wFr, resFr, so, dof, ko, v.ld_r));
    CNMF_TRY(gather(wFc, resFc, so, dof, ko, v.ld_c));
    CNMF_CUDA_CHECK(cudaMemcpyAsync(io.Fr64, resFr, (size_t)SK0 * v.ld_r * 8, cudaMemcpyDeviceToDevice, s));
    CNMF_CUDA_CHECK(cudaMemcpyAsync(io.Fc64, resFc, (size_t)SK0 * v.ld_c * 8, cudaMemcpyDeviceToDevice, s));
  }
  io.n_iter.assign(R0, 0);
  io.last.assign(R0, 0.0);
  io.err.assign(R0, 0.0);
  CNMF_CUDA_CHECK(cudaMemcpyAsync(io.n_iter.data(), d_niter, sizeof(int) * R0, cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaMemcpyAsync(io.last.data(), st.last, sizeof(double) * R0, cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaMemcpyAsync(io.err.data(), d_err, sizeof(double) * R0, cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
  return 0;
}

}  // namespace cnmf
