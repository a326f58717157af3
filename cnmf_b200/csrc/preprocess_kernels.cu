// Preprocessing before `cnmf prepare`: Harmony's mixture-of-experts ridge correction of a cells x genes matrix and
// the variance scaling with a quantile ceiling (cnmf_moe_grams, cnmf_moe_correct, cnmf_scale_quantile_ceiling).
//
// Ridge correction.  X: N cells x G genes; R: K x N soft cluster assignments; Phi: B1 x N design (row 0 the intercept);
// P (K*B1 x N): P[i*B1 + b, n] = Phi[b, n] R[i, n].  Every cluster's W_i is computed from the uncorrected X, so the
// correction is two products and an epilogue:
//   A_i = P_i Phi^T + lambda         (cnmf_moe_grams; inverted by the caller)
//   C   = P X                        (fp64 tensor cores, gemm_f64 in fixed split-K slices summed in slice order)
//   W_i = inv(A_i) C_i, row 0 zeroed
//   X_corr = X - sum_i P_i^T W_i     one cluster at a time per element, the cluster's term in fp64, rounded to X's
//                                    element type after each cluster (what `Z_corr -= term` does to a float32 array)
// No floating-point atomics anywhere: two calls give the same bits.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstring>

#include "engine.h"

namespace cnmf {

namespace {

constexpr int MOE_TILE = 64;      // apply kernel: 64 cells x 64 genes per block, 4 x 4 per thread
constexpr int MOE_ROWS = 32;      // rows of P / W staged in shared memory per step
constexpr int SEL_THREADS = 256;
constexpr int MOM_LOADS = 12;     // column moments: rows each staging lane loads per step
constexpr int MOM_ROWS = 7 * MOM_LOADS;   // rows of a 32-column strip staged per step by warps 1-7

// split-K plan of the products over cells: slices of a fixed length that depends on N only
int moe_chunk(int n) {
  const int splits = std::min((n + 4095) / 4096, 32);
  return round_up((n + splits - 1) / splits, 16);
}

__global__ void moe_form_p_kernel(const double* __restrict__ R, const double* __restrict__ Phi, int K, int B1, int N,
                                  double* __restrict__ P) {
  const long long total = (long long)K * B1 * N;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total;
       e += (long long)gridDim.x * blockDim.x) {
    const long long row = e / N;
    const int n = (int)(e - row * N);
    const int i = (int)(row / B1), b = (int)(row - (long long)i * B1);
    P[e] = Phi[(long long)b * N + n] * R[(long long)i * N + n];
  }
}

// A[i][b][c] = sum over slices (in order) + lambda[b][c]
__global__ void moe_gram_reduce_kernel(const double* __restrict__ Cs, int splits, long long stride, int ldc, int K,
                                       int B1, const double* __restrict__ lamb, double* __restrict__ A) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= K * B1 * B1) return;
  const int row = e / B1, c = e - row * B1, b = row % B1;
  double v = 0.0;
  for (int z = 0; z < splits; ++z) v += Cs[z * stride + (long long)row * ldc + c];
  A[e] = v + lamb[b * B1 + c];
}

// W[i*B1 + b][g] = sum_c Ainv[i][b][c] * C[i*B1 + c][g] (C summed over slices in order); row b = 0 is zero
__global__ void moe_w_kernel(const double* __restrict__ Cs, int splits, long long stride, int ldg, int G, int K, int B1,
                             const double* __restrict__ Ainv, double* __restrict__ W) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  const int i = blockIdx.y;
  if (g >= G) return;
  double c[64];
  for (int cc = 0; cc < B1; ++cc) {
    double v = 0.0;
    for (int z = 0; z < splits; ++z) v += Cs[z * stride + (long long)(i * B1 + cc) * ldg + g];
    c[cc] = v;
  }
  W[(long long)i * B1 * ldg + g] = 0.0;
  for (int b = 1; b < B1; ++b) {
    const double* a = Ainv + ((long long)i * B1 + b) * B1;
    double v = 0.0;
    for (int cc = 0; cc < B1; ++cc) v += a[cc] * c[cc];
    W[((long long)i * B1 + b) * ldg + g] = v;
  }
}

// X (in place, N x ld) -= sum_i P_i^T W_i, cluster by cluster; optional clamp at zero; per (cell, gene tile) partial
// sums of squares of the unclamped result into sq (gridDim.x x N)
template <typename T>
__global__ void __launch_bounds__(256) moe_apply_kernel(T* __restrict__ X, int ld, int N, int G,
                                                        const double* __restrict__ P, const double* __restrict__ W,
                                                        int ldw, int M, int B1, int clamp, double* __restrict__ sq) {
  __shared__ double Ps[MOE_ROWS][MOE_TILE];
  __shared__ double Ws[MOE_ROWS][MOE_TILE];
  __shared__ double red[16][MOE_TILE + 1];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int g0 = blockIdx.x * MOE_TILE, n0 = blockIdx.y * MOE_TILE;
  double z[4][4], term[4][4];
#pragma unroll
  for (int j = 0; j < 4; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int n = n0 + ty + 16 * j, g = g0 + tx + 16 * e;
      z[j][e] = (n < N && g < G) ? (double)X[(long long)n * ld + g] : 0.0;
      term[j][e] = 0.0;
    }
  for (int r0 = 0; r0 < M; r0 += MOE_ROWS) {
    __syncthreads();
    for (int q = tid; q < MOE_ROWS * MOE_TILE; q += 256) {
      const int r = q / MOE_TILE, c = q % MOE_TILE;
      const bool ok = r0 + r < M;
      Ps[r][c] = (ok && n0 + c < N) ? P[(long long)(r0 + r) * N + n0 + c] : 0.0;
      Ws[r][c] = (ok && g0 + c < G) ? W[(long long)(r0 + r) * ldw + g0 + c] : 0.0;
    }
    __syncthreads();
    const int rn = min(MOE_ROWS, M - r0);
    for (int r = 0; r < rn; ++r) {
      const int b = (r0 + r) % B1;
      if (b == 0) continue;          // W's intercept row is zero
      double p[4], w[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) p[j] = Ps[r][ty + 16 * j];
#pragma unroll
      for (int e = 0; e < 4; ++e) w[e] = Ws[r][tx + 16 * e];
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) term[j][e] = fma(p[j], w[e], term[j][e]);
      if (b == B1 - 1) {
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            z[j][e] = (double)(T)(z[j][e] - term[j][e]);
            term[j][e] = 0.0;
          }
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    double s = 0.0;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int n = n0 + ty + 16 * j, g = g0 + tx + 16 * e;
      if (n < N && g < G) {
        s += z[j][e] * z[j][e];
        const double v = (clamp && z[j][e] < 0.0) ? 0.0 : z[j][e];
        X[(long long)n * ld + g] = (T)v;
      }
    }
    red[tx][ty + 16 * j] = s;
  }
  if (!sq) return;
  __syncthreads();
  if (tid < MOE_TILE && n0 + tid < N) {
    double s = 0.0;
    for (int t = 0; t < 16; ++t) s += red[t][tid];
    sq[(long long)blockIdx.x * N + n0 + tid] = s;
  }
}

// Xcos[n, g] = X[n, g] / norm_n, with norm_n the square root of the gene-tile partials summed in order, rounded to T
template <typename T>
__global__ void moe_cos_kernel(const T* __restrict__ X, int ld, int N, int G, const double* __restrict__ sq, int tiles,
                               T* __restrict__ Xc) {
  const int n = blockIdx.x;
  __shared__ T nrm;
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int t = 0; t < tiles; ++t) s += sq[(long long)t * N + n];
    nrm = (T)sqrt(s);
  }
  __syncthreads();
  for (int g = threadIdx.x; g < G; g += blockDim.x) Xc[(long long)n * ld + g] = X[(long long)n * ld + g] / nrm;
}

// ---- variance scaling with a quantile ceiling

// per column sum(x) and sum(x^2) in fp64, each one sequential chain in row order with every square rounded before it is
// added: the order of numpy's axis-0 sum of a 2-D array, so that mean, mean(x^2) and the std that cancels between them
// are the reference's bit for bit.  The chains of a 32-column strip run in warp 0 while warps 1-7 stage the next
// MOM_ROWS rows of the strip in shared memory, each lane issuing all its MOM_LOADS loads before it stores any.
template <typename T>
__global__ void __launch_bounds__(256) col_moments_kernel(const T* __restrict__ X, int ld, int N, int G,
                                                          double* __restrict__ sum, double* __restrict__ sumsq) {
  __shared__ T tile[2][MOM_ROWS][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + lane;
  const int tiles = (N + MOM_ROWS - 1) / MOM_ROWS;
  auto stage = [&](int t) {
    T v[MOM_LOADS];
#pragma unroll
    for (int j = 0; j < MOM_LOADS; ++j) {
      const int r = t * MOM_ROWS + (warp - 1) + 7 * j;
      v[j] = (r < N && c < G) ? X[(long long)r * ld + c] : T(0);
    }
#pragma unroll
    for (int j = 0; j < MOM_LOADS; ++j) tile[t & 1][(warp - 1) + 7 * j][lane] = v[j];
  };
  if (warp > 0) stage(0);
  __syncthreads();
  double a = 0.0, q = 0.0;
  for (int t = 0; t < tiles; ++t) {
    if (warp > 0) {
      if (t + 1 < tiles) stage(t + 1);
    } else {
      const int rn = min(MOM_ROWS, N - t * MOM_ROWS);
      for (int r = 0; r < rn; ++r) {
        const double v = (double)tile[t & 1][r][lane];
        a = __dadd_rn(a, v);
        q = __dadd_rn(q, __dmul_rn(v, v));
      }
    }
    __syncthreads();
  }
  if (warp == 0 && c < G) {
    sum[c] = a;
    sumsq[c] = q;
  }
}

// std of each column from its moments as the reference forms it, sqrt((msq - mean^2) * (N / (N - 1))) with every
// operation rounded on its own (no contraction); a zero std maps to 1
__global__ void col_std_kernel(const double* __restrict__ sum, const double* __restrict__ sumsq, int N, int G,
                               double* __restrict__ sd) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= G) return;
  const double mean = sum[c] / (double)N, msq = sumsq[c] / (double)N;
  const double var = __dmul_rn(__dsub_rn(msq, __dmul_rn(mean, mean)), (double)N / (double)(N - 1));
  double s = sqrt(var);
  if (s == 0.0) s = 1.0;
  sd[c] = s;
}

// X / std rounded to T, clipped at max_value; *nan_seen = 1 when a result is NaN
template <typename T>
__global__ void scale_clip_kernel(T* __restrict__ X, int ld, int N, int G, const double* __restrict__ sd, int clip,
                                  double max_value, int* __restrict__ nan_seen) {
  const long long total = (long long)N * G;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total;
       e += (long long)gridDim.x * blockDim.x) {
    const long long r = e / G;
    const int c = (int)(e - r * G);
    T v = (T)((double)X[r * ld + c] / sd[c]);
    if (clip && (double)v > max_value) v = (T)max_value;
    if (v != v) *nan_seen = 1;
    X[r * ld + c] = v;
  }
}

template <typename T> struct KeyOf;
template <> struct KeyOf<float> {
  using K = unsigned int;
  static constexpr int BITS = 32;
  __device__ static K key(float v) {
    const K u = __float_as_uint(v);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  }
};
template <> struct KeyOf<double> {
  using K = unsigned long long;
  static constexpr int BITS = 64;
  __device__ static K key(double v) {
    const K u = (K)__double_as_longlong(v);
    return (u & 0x8000000000000000ull) ? ~u : (u | 0x8000000000000000ull);
  }
};

// 256-bin histogram of the digit at `shift` of the order-preserving keys whose bits above it equal `prefix`
template <typename T>
__global__ void __launch_bounds__(SEL_THREADS) radix_hist_kernel(const T* __restrict__ X, int ld, int N, int G,
                                                                 typename KeyOf<T>::K prefix, int shift,
                                                                 unsigned long long* __restrict__ hist) {
  using K = typename KeyOf<T>::K;
  __shared__ unsigned int h[256];
  for (int i = threadIdx.x; i < 256; i += SEL_THREADS) h[i] = 0;
  __syncthreads();
  const int top = shift + 8;
  const long long total = (long long)N * G;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total;
       e += (long long)gridDim.x * blockDim.x) {
    const long long r = e / G;
    const int c = (int)(e - r * G);
    const K k = KeyOf<T>::key(X[r * ld + c]);
    if (top >= KeyOf<T>::BITS || (k >> top) == prefix) atomicAdd(&h[(unsigned)(k >> shift) & 255u], 1u);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 256; i += SEL_THREADS)
    if (h[i]) atomicAdd(&hist[i], (unsigned long long)h[i]);
}

template <typename T>
__global__ void ceiling_kernel(T* __restrict__ X, int ld, int N, int G, T thresh) {
  const long long total = (long long)N * G;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total;
       e += (long long)gridDim.x * blockDim.x) {
    const long long r = e / G;
    const int c = (int)(e - r * G);
    if (X[r * ld + c] > thresh) X[r * ld + c] = thresh;
  }
}

template <typename T>
T key_value(typename KeyOf<T>::K k);
template <>
float key_value<float>(unsigned int k) {
  const unsigned int u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
  float v;
  memcpy(&v, &u, 4);
  return v;
}
template <>
double key_value<double>(unsigned long long k) {
  const unsigned long long u = (k & 0x8000000000000000ull) ? (k & 0x7fffffffffffffffull) : ~k;
  double v;
  memcpy(&v, &u, 8);
  return v;
}

// the value of rank `rank` (0-based, ascending) among the N x G entries: one histogram pass per 8-bit digit
template <typename T>
int radix_select(cnmf_handle_s* h, const T* X, int ld, int N, int G, long long rank, unsigned long long* hist_dev,
                 T* out, cudaStream_t s) {
  using K = typename KeyOf<T>::K;
  K prefix = 0;
  unsigned long long hist[256];
  const int blocks = 4 * h->sm_count;
  for (int shift = KeyOf<T>::BITS - 8; shift >= 0; shift -= 8) {
    CNMF_CUDA_CHECK(cudaMemsetAsync(hist_dev, 0, sizeof(hist), s));
    radix_hist_kernel<T><<<blocks, SEL_THREADS, 0, s>>>(X, ld, N, G, prefix, shift, hist_dev);
    CNMF_CUDA_CHECK(cudaGetLastError());
    h->launches += 1;
    CNMF_CUDA_CHECK(cudaMemcpyAsync(hist, hist_dev, sizeof(hist), cudaMemcpyDeviceToHost, s));
    CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
    int d = 0;
    while (d < 255 && rank >= (long long)hist[d]) rank -= (long long)hist[d++];
    prefix = (prefix << 8) | (K)d;
  }
  *out = key_value<T>(prefix);
  return 0;
}

// numpy's _lerp in the array's element type: a + (b - a) t, or b - (b - a)(1 - t) when t >= 0.5
template <typename T>
T numpy_lerp(T a, T b, T t) {
  volatile T diff = b - a;
  volatile T lo = diff * t;
  T r = a + lo;
  if (t >= (T)0.5) {
    volatile T om = (T)1 - t;
    volatile T hi = diff * om;
    r = b - hi;
  }
  return r;
}

int grid_for(long long total, int threads, int sm) {
  return (int)std::max(1LL, std::min((total + threads - 1) / threads, (long long)sm * 8));
}

// X (host or device, row stride ld, rows may be CSR values) -> zero-padded device matrix at stride ldp
template <typename T>
int stage_matrix(const void* X, int N, int G, long long ld, int src_is_device, const long long* csr_row_ptr,
                 const int* csr_col_idx, long long nnz, T* dst, int ldp, DeviceTemp* csr_tmp, cudaStream_t s) {
  CNMF_CUDA_CHECK(cudaMemsetAsync(dst, 0, (size_t)N * ldp * sizeof(T), s));
  if (csr_row_ptr) {
    CNMF_REQUIRE(!src_is_device, "CSR input is host memory");
    CNMF_TRY(check_csr("CSR input", N, G, nnz, reinterpret_cast<const int64_t*>(csr_row_ptr), csr_col_idx));
    const size_t rp = (size_t)(N + 1) * 8, ci = (size_t)nnz * 4, va = (size_t)nnz * sizeof(T);
    CNMF_TRY(csr_tmp->alloc(rp + round_up_ll(ci, 16) + va, "CSR input"));
    char* base = csr_tmp->as<char>();
    long long* d_rp = reinterpret_cast<long long*>(base);
    int* d_ci = reinterpret_cast<int*>(base + rp);
    T* d_va = reinterpret_cast<T*>(base + rp + round_up_ll(ci, 16));
    CNMF_CUDA_CHECK(cudaMemcpyAsync(d_rp, csr_row_ptr, rp, cudaMemcpyHostToDevice, s));
    if (nnz) {
      CNMF_CUDA_CHECK(cudaMemcpyAsync(d_ci, csr_col_idx, ci, cudaMemcpyHostToDevice, s));
      CNMF_CUDA_CHECK(cudaMemcpyAsync(d_va, X, va, cudaMemcpyHostToDevice, s));
    }
    return csr_scatter_rows(d_rp, 0, d_ci, d_va, 0, N, dst, ldp, s);
  }
  CNMF_REQUIRE(ld >= G, "row stride smaller than the number of columns");
  CNMF_CUDA_CHECK(cudaMemcpy2DAsync(dst, (size_t)ldp * sizeof(T), X, (size_t)ld * sizeof(T), (size_t)G * sizeof(T), N,
                                    src_is_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, s));
  return 0;
}

template <typename T>
int copy_out(const T* src, int ldp, int N, int G, void* dst, long long ld_out, int dst_is_device, cudaStream_t s) {
  CNMF_REQUIRE(ld_out >= G, "output row stride smaller than the number of columns");
  CNMF_CUDA_CHECK(cudaMemcpy2DAsync(dst, (size_t)ld_out * sizeof(T), src, (size_t)ldp * sizeof(T),
                                    (size_t)G * sizeof(T), N,
                                    dst_is_device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, s));
  return 0;
}

// device copies of R (K x N) and P (K*B1 x N) from the host R and Phi
int moe_upload_p(cnmf_handle_s* h, const double* R, const double* Phi, int K, int B1, int N, double* Rd, double* Phid,
                 double* P, cudaStream_t s) {
  CNMF_CUDA_CHECK(cudaMemcpyAsync(Rd, R, (size_t)K * N * 8, cudaMemcpyHostToDevice, s));
  CNMF_CUDA_CHECK(cudaMemcpyAsync(Phid, Phi, (size_t)B1 * N * 8, cudaMemcpyHostToDevice, s));
  moe_form_p_kernel<<<grid_for((long long)K * B1 * N, 256, h->sm_count), 256, 0, s>>>(Rd, Phid, K, B1, N, P);
  CNMF_CUDA_CHECK(cudaGetLastError());
  h->launches += 1;
  return 0;
}

template <typename T>
int moe_correct(cnmf_handle_s* h, const void* X, int N, int G, long long ld, int src_is_device, const double* R,
                const double* Phi, const double* Ainv, int K, int B1, int clamp, void* X_out, long long ld_out,
                int dst_is_device, void* Xcos_out, double* W_last, cudaStream_t s) {
  const int ldp = pad_ld(G);
  const int M = K * B1;
  const int chunk = moe_chunk(N);
  const int splits = (N + chunk - 1) / chunk;
  const long long cstride = (long long)M * ldp;
  const int tiles_g = (G + MOE_TILE - 1) / MOE_TILE, tiles_n = (N + MOE_TILE - 1) / MOE_TILE;
  DeviceTemp xb, pb, rb, cb, wb, ab, sqb, xc, csr;
  CNMF_TRY(xb.alloc((size_t)N * ldp * sizeof(T), "moe_correct X"));
  CNMF_TRY(pb.alloc((size_t)M * N * 8, "moe_correct P"));
  CNMF_TRY(rb.alloc((size_t)(K + B1) * N * 8, "moe_correct R, Phi"));
  CNMF_TRY(cb.alloc((size_t)splits * cstride * 8, "moe_correct C slices"));
  CNMF_TRY(wb.alloc((size_t)M * ldp * 8, "moe_correct W"));
  CNMF_TRY(ab.alloc((size_t)M * B1 * 8, "moe_correct inv(A)"));
  CNMF_TRY(sqb.alloc((size_t)tiles_g * N * 8, "moe_correct norms"));
  T* Xd = xb.as<T>();
  CNMF_TRY(stage_matrix<T>(X, N, G, ld, src_is_device, nullptr, nullptr, 0, Xd, ldp, &csr, s));
  CNMF_TRY(moe_upload_p(h, R, Phi, K, B1, N, rb.as<double>(), rb.as<double>() + (size_t)K * N, pb.as<double>(), s));
  CNMF_CUDA_CHECK(cudaMemcpyAsync(ab.p, Ainv, (size_t)M * B1 * 8, cudaMemcpyHostToDevice, s));

  h->launches += 1;
  const int slot = h->prof_begin(s, 2.0 * (double)M * (double)N * (double)G, 5);
  CNMF_TRY(launch_gemm_f64_split(pb.as<double>(), N, M, Xd, N, G, ldp, true, chunk, cb.as<double>(), ldp, cstride, s));
  h->prof_end(s, slot);

  moe_w_kernel<<<dim3((G + 127) / 128, K), 128, 0, s>>>(cb.as<double>(), splits, cstride, ldp, G, K, B1,
                                                        ab.as<double>(), wb.as<double>());
  CNMF_CUDA_CHECK(cudaGetLastError());
  h->launches += 1;

  moe_apply_kernel<T><<<dim3(tiles_g, tiles_n), 256, 0, s>>>(Xd, ldp, N, G, pb.as<double>(), wb.as<double>(), ldp, M,
                                                             B1, clamp, sqb.as<double>());
  CNMF_CUDA_CHECK(cudaGetLastError());
  h->launches += 1;
  CNMF_TRY(copy_out<T>(Xd, ldp, N, G, X_out, ld_out, dst_is_device, s));
  if (Xcos_out) {
    CNMF_TRY(xc.alloc((size_t)N * ldp * sizeof(T), "moe_correct Z_cos"));
    moe_cos_kernel<T><<<N, 256, 0, s>>>(Xd, ldp, N, G, sqb.as<double>(), tiles_g, xc.as<T>());
    CNMF_CUDA_CHECK(cudaGetLastError());
    h->launches += 1;
    CNMF_TRY(copy_out<T>(xc.as<T>(), ldp, N, G, Xcos_out, ld_out, dst_is_device, s));
  }
  if (W_last)
    CNMF_CUDA_CHECK(cudaMemcpy2DAsync(W_last, (size_t)G * 8, wb.as<double>() + (size_t)(K - 1) * B1 * ldp,
                                      (size_t)ldp * 8, (size_t)G * 8, B1, cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
  return 0;
}

template <typename T>
int scale_quantile(cnmf_handle_s* h, const void* X, int N, int G, long long ld, int src_is_device,
                   const long long* csr_row_ptr, const int* csr_col_idx, long long nnz, double max_value, int clip,
                   long long k_lo, long long k_hi, double gamma, void* X_out, long long ld_out, int dst_is_device,
                   double* thresh_out, cudaStream_t s) {
  const int ldp = pad_ld(G);
  DeviceTemp xb, mom, sd, hist, flag, csr;
  CNMF_TRY(xb.alloc((size_t)N * ldp * sizeof(T), "scale_quantile_ceiling X"));
  CNMF_TRY(mom.alloc((size_t)2 * G * 8, "scale_quantile_ceiling moments"));
  CNMF_TRY(sd.alloc((size_t)G * 8, "scale_quantile_ceiling std"));
  CNMF_TRY(hist.alloc(256 * 8, "scale_quantile_ceiling histogram"));
  CNMF_TRY(flag.alloc(sizeof(int), "scale_quantile_ceiling NaN flag"));
  T* Xd = xb.as<T>();
  CNMF_TRY(stage_matrix<T>(X, N, G, ld, src_is_device, csr_row_ptr, csr_col_idx, nnz, Xd, ldp, &csr, s));
  CNMF_CUDA_CHECK(cudaMemsetAsync(flag.p, 0, sizeof(int), s));
  col_moments_kernel<T><<<(G + 31) / 32, 256, 0, s>>>(Xd, ldp, N, G, mom.as<double>(), mom.as<double>() + G);
  CNMF_CUDA_CHECK(cudaGetLastError());
  col_std_kernel<<<(G + 255) / 256, 256, 0, s>>>(mom.as<double>(), mom.as<double>() + G, N, G, sd.as<double>());
  CNMF_CUDA_CHECK(cudaGetLastError());
  const long long total = (long long)N * G;
  scale_clip_kernel<T><<<grid_for(total, 256, h->sm_count), 256, 0, s>>>(Xd, ldp, N, G, sd.as<double>(), clip,
                                                                         max_value, flag.as<int>());
  CNMF_CUDA_CHECK(cudaGetLastError());
  h->launches += 3;
  if (k_lo >= 0) {
    CNMF_REQUIRE(k_lo < total && k_hi >= k_lo && k_hi < total, "scale_quantile_ceiling: rank out of range");
    int nan_seen = 0;
    CNMF_CUDA_CHECK(cudaMemcpyAsync(&nan_seen, flag.p, sizeof(int), cudaMemcpyDeviceToHost, s));
    CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
    if (nan_seen) {
      // np.quantile of values that include a NaN is NaN, and nothing compares above NaN: X stays as scaled
      if (thresh_out) *thresh_out = std::nan("");
    } else {
      T a, b;
      auto* hd = hist.as<unsigned long long>();
      CNMF_TRY(radix_select<T>(h, Xd, ldp, N, G, k_lo, hd, &a, s));
      b = a;
      if (k_hi != k_lo) CNMF_TRY(radix_select<T>(h, Xd, ldp, N, G, k_hi, hd, &b, s));
      const T thresh = numpy_lerp<T>(a, b, (T)gamma);
      if (thresh_out) *thresh_out = (double)thresh;
      ceiling_kernel<T><<<grid_for(total, 256, h->sm_count), 256, 0, s>>>(Xd, ldp, N, G, thresh);
      CNMF_CUDA_CHECK(cudaGetLastError());
      h->launches += 1;
    }
  }
  CNMF_TRY(copy_out<T>(Xd, ldp, N, G, X_out, ld_out, dst_is_device, s));
  CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
  return 0;
}

}  // namespace

}  // namespace cnmf

using namespace cnmf;

extern "C" {

int cnmf_moe_grams(cnmf_handle_t h, const double* R, const double* Phi, const double* lamb, int K, int n_phi,
                   int n_cells, double* A_out, void* stream) {
  CNMF_REQUIRE(h && R && Phi && lamb && A_out, "moe_grams: NULL argument");
  CNMF_REQUIRE(K > 0 && n_phi > 0 && n_phi <= 64 && n_cells > 0, "moe_grams: bad shape (1 <= n_phi <= 64)");
  CNMF_CUDA_CHECK(cudaSetDevice(h->device));
  cudaStream_t s = as_stream(stream);
  const int N = n_cells, B1 = n_phi, M = K * B1;
  const int ldphi = pad_ld(N), ldc = round_up(B1, 8);
  const int chunk = moe_chunk(N);
  const int splits = (N + chunk - 1) / chunk;
  const long long cstride = (long long)M * ldc;
  DeviceTemp pb, rb, phib, cb, lb, ab;
  CNMF_TRY(pb.alloc((size_t)M * N * 8, "moe_grams P"));
  CNMF_TRY(rb.alloc((size_t)(K + B1) * N * 8, "moe_grams R, Phi"));
  CNMF_TRY(phib.alloc((size_t)B1 * ldphi * 8, "moe_grams Phi"));
  CNMF_TRY(cb.alloc((size_t)splits * cstride * 8, "moe_grams slices"));
  CNMF_TRY(lb.alloc((size_t)B1 * B1 * 8, "moe_grams lambda"));
  CNMF_TRY(ab.alloc((size_t)M * B1 * 8, "moe_grams A"));
  CNMF_TRY(moe_upload_p(h, R, Phi, K, B1, N, rb.as<double>(), rb.as<double>() + (size_t)K * N, pb.as<double>(), s));
  // Phi as the gemm's X operand: rows zero padded to the stride it reads whole K tiles from
  CNMF_CUDA_CHECK(cudaMemsetAsync(phib.p, 0, (size_t)B1 * ldphi * 8, s));
  CNMF_CUDA_CHECK(cudaMemcpy2DAsync(phib.p, (size_t)ldphi * 8, Phi, (size_t)N * 8, (size_t)N * 8, B1,
                                    cudaMemcpyHostToDevice, s));
  CNMF_CUDA_CHECK(cudaMemcpyAsync(lb.p, lamb, (size_t)B1 * B1 * 8, cudaMemcpyHostToDevice, s));
  h->launches += 1;
  const int slot = h->prof_begin(s, 2.0 * (double)M * (double)B1 * (double)N, 5);
  CNMF_TRY(launch_gemm_f64_split(pb.as<double>(), N, M, phib.as<double>(), B1, N, ldphi, false, chunk,
                                 cb.as<double>(), ldc, cstride, s));
  h->prof_end(s, slot);
  moe_gram_reduce_kernel<<<(M * B1 + 255) / 256, 256, 0, s>>>(cb.as<double>(), splits, cstride, ldc, K, B1,
                                                              lb.as<double>(), ab.as<double>());
  CNMF_CUDA_CHECK(cudaGetLastError());
  h->launches += 1;
  CNMF_CUDA_CHECK(cudaMemcpyAsync(A_out, ab.p, (size_t)M * B1 * 8, cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
  return 0;
}

int cnmf_moe_correct(cnmf_handle_t h, const void* X, int dtype, int n_cells, int n_genes, long long ld,
                     int src_is_device, const double* R, const double* Phi, const double* A_inv, int K, int n_phi,
                     int clamp_zero, void* X_out, long long ld_out, int dst_is_device, void* X_cos_out,
                     double* W_last, void* stream) {
  CNMF_REQUIRE(h && X && R && Phi && A_inv && X_out, "moe_correct: NULL argument");
  CNMF_REQUIRE(dtype == 0 || dtype == 1, "moe_correct: dtype must be 0 (float32) or 1 (float64)");
  CNMF_REQUIRE(K > 0 && n_phi > 0 && n_phi <= 64 && n_cells > 0 && n_genes > 0, "moe_correct: bad shape");
  CNMF_CUDA_CHECK(cudaSetDevice(h->device));
  cudaStream_t s = as_stream(stream);
  if (dtype == 0)
    return moe_correct<float>(h, X, n_cells, n_genes, ld, src_is_device, R, Phi, A_inv, K, n_phi, clamp_zero, X_out,
                              ld_out, dst_is_device, X_cos_out, W_last, s);
  return moe_correct<double>(h, X, n_cells, n_genes, ld, src_is_device, R, Phi, A_inv, K, n_phi, clamp_zero, X_out,
                             ld_out, dst_is_device, X_cos_out, W_last, s);
}

int cnmf_scale_quantile_ceiling(cnmf_handle_t h, const void* X, int dtype, int n_rows, int n_cols, long long ld,
                                int src_is_device, const long long* csr_row_ptr, const int* csr_col_idx,
                                long long nnz, double max_value, int clip, long long k_lo, long long k_hi,
                                double gamma, void* X_out, long long ld_out, int dst_is_device, double* thresh_out,
                                void* stream) {
  CNMF_REQUIRE(h && X && X_out, "scale_quantile_ceiling: NULL argument");
  CNMF_REQUIRE(dtype == 0 || dtype == 1, "scale_quantile_ceiling: dtype must be 0 (float32) or 1 (float64)");
  CNMF_REQUIRE(n_rows > 1 && n_cols > 0, "scale_quantile_ceiling: bad shape");
  CNMF_CUDA_CHECK(cudaSetDevice(h->device));
  cudaStream_t s = as_stream(stream);
  if (dtype == 0)
    return scale_quantile<float>(h, X, n_rows, n_cols, ld, src_is_device, csr_row_ptr, csr_col_idx, nnz, max_value,
                                 clip, k_lo, k_hi, gamma, X_out, ld_out, dst_is_device, thresh_out, s);
  return scale_quantile<double>(h, X, n_rows, n_cols, ld, src_is_device, csr_row_ptr, csr_col_idx, nnz, max_value,
                                clip, k_lo, k_hi, gamma, X_out, ld_out, dst_is_device, thresh_out, s);
}

}  // extern "C"
