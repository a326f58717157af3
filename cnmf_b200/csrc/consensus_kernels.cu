// Consensus-stage kernels: the numeric steps of cNMF.consensus (cnmf.py:882-916) on the stacked
// spectra matrix S (R x G, row stride ld).  R <= ~6000, G <= ~5000 at the BASELINE configs, so
// S (<= 120 MB) lives in L2 and every kernel here is a streaming / reduction kernel:
//   C1  l2_normalize_rows          cnmf.py:882
//   C2  pairwise distances         cnmf.py:891  (direct sum (x-y)^2: no ||x||^2+||y||^2-2xy cancellation)
//   C3  k-NN local density         cnmf.py:893-896 (exact radix select of the n+1 smallest per row)
//   C5  Lloyd E+M step             sklearn _k_means_lloyd.pyx:168-219 (k-means++ draws stay on the host)
//   C6  per-cluster median         cnmf.py:913-916
// Every kernel is templated on the element type T of S: float for the fp32-class precisions, double for
// precision="fp64" (the reference's own float64).  Where the float kernel already accumulates in double, T changes the
// storage type and nothing else; the distance tile has a separate fp64 body because its fp32 one runs on add2 / fma2.
#include <algorithm>
#include <type_traits>
#include <vector>

#include "engine.h"

using namespace cnmf;

namespace {

template <typename T>
__device__ __forceinline__ T block_sum_all(T v, T* smem /* >= 33 entries */) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) smem[warp] = v;
  __syncthreads();
  const int nw = (blockDim.x + 31) >> 5;
  T r = (threadIdx.x < nw) ? smem[threadIdx.x] : T(0);
  if (warp == 0) {
    r = warp_sum(r);
    if (lane == 0) smem[32] = r;
  }
  __syncthreads();
  return smem[32];   // broadcast to every thread
}

// Bit patterns of an element type for the radix selects (C3, C6): the values selected are non-negative, so their
// order is the order of the patterns below the sign bit, walked MSB first from bit kTop.
template <typename T> struct Bits;
template <> struct Bits<float> {
  using U = uint32_t;
  static constexpr int kTop = 30;
  static __device__ __forceinline__ U of(float v) { return __float_as_uint(v); }
  static __device__ __forceinline__ float value(U u) { return __uint_as_float(u); }
  static __device__ __forceinline__ float nan() { return __int_as_float(0x7fc00000); }
  static __device__ __forceinline__ float inf() { return __int_as_float(0x7f800000); }
};
template <> struct Bits<double> {
  using U = unsigned long long;
  static constexpr int kTop = 62;
  static __device__ __forceinline__ U of(double v) { return (U)__double_as_longlong(v); }
  static __device__ __forceinline__ double value(U u) { return __longlong_as_double((long long)u); }
  static __device__ __forceinline__ double nan() { return __longlong_as_double(0x7ff8000000000000ll); }
  static __device__ __forceinline__ double inf() { return __longlong_as_double(0x7ff0000000000000ll); }
};

// bits above `bit`, sign bit excluded
template <typename U>
__device__ __forceinline__ U radix_mask_hi(int bit) {
  return ~((U(1) << (bit + 1)) - U(1)) & (~U(0) >> 1);
}

// four consecutive elements as one load (cand_dist_kernel, kmeans_batched.cu row_dists)
template <typename T> struct Vec4;
template <> struct Vec4<float> { using type = float4; };
struct __align__(32) double4a { double x, y, z, w; };
template <> struct Vec4<double> { using type = double4a; };

// ---------------------------------------------------------------- C1
template <typename T>
__global__ void l2_normalize_kernel(T* __restrict__ S, int R, int G, int ld) {
  __shared__ double sm[33];
  const int r = blockIdx.x;
  T* row = S + (long long)r * ld;
  double q = 0.0;
  for (int g = threadIdx.x; g < G; g += blockDim.x) {
    const double v = row[g];
    q += v * v;
  }
  q = block_sum_all(q, sm);
  const double inv = 1.0 / sqrt(q);
  for (int g = threadIdx.x; g < G; g += blockDim.x) row[g] = (T)((double)row[g] * inv);
}

// ---------------------------------------------------------------- C2: D[i][j] = sqrt(sum_g (A_i - B_j)^2)
// 64 x 64 output tile per block, 16 x 16 threads, 4 x 4 per thread, k-tiles of 16 through smem.  The fp32 inner product
// runs on element pairs (add2 / fma2 of common.cuh: two round-to-nearest fp32 instructions per pair) -- this kernel
// is FP32-issue bound, not HBM-bound (3 R^2 G FLOPs against R G 4 bytes).  The fp64 tile forms the same direct
// difference and square, one DFMA per entry.  SYM (A == B, the R x R matrix of cnmf.py:891): only tiles on or above the
// diagonal are computed, each is also written transposed, so the matrix is exactly symmetric with an exactly zero
// diagonal at half the work.
template <typename T, bool SQRT, bool SYM>
__global__ void __launch_bounds__(256)
pair_dist_kernel(const T* __restrict__ A, int RA, int lda, const T* __restrict__ B, int RB, int ldb, int G,
                 T* __restrict__ D, int ldd) {
  constexpr int TT = 64, TK = 16;
  if (SYM && blockIdx.x < blockIdx.y) return;
  __shared__ __align__(16) T As[TK][TT + 4];
  __shared__ __align__(16) T Bs[TK][TT + 4];
  const int i0 = blockIdx.y * TT, j0 = blockIdx.x * TT;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int lrow = threadIdx.x >> 2, lk = (threadIdx.x & 3) * 4;
  // fp32: element pairs through add2 / fma2; fp64: one DSUB + DFMA per entry (the unused one is never touched)
  float2 acc[4][2];
  double accd[4][4];
  if constexpr (std::is_same<T, float>::value) {
#pragma unroll
    for (int i = 0; i < 4; ++i) acc[i][0] = acc[i][1] = make_float2(0.f, 0.f);
  } else {
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) accd[i][j] = 0.0;
  }
  for (int k0 = 0; k0 < G; k0 += TK) {
    {
      T va[4] = {T(0), T(0), T(0), T(0)}, vb[4] = {T(0), T(0), T(0), T(0)};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int g = k0 + lk + e;
        if (g < G) {
          if (i0 + lrow < RA) va[e] = A[(long long)(i0 + lrow) * lda + g];
          if (j0 + lrow < RB) vb[e] = B[(long long)(j0 + lrow) * ldb + g];
        }
      }
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        As[lk + e][lrow] = va[e];
        Bs[lk + e][lrow] = vb[e];
      }
    }
    __syncthreads();
    if constexpr (std::is_same<T, float>::value) {
#pragma unroll
      for (int k = 0; k < TK; ++k) {
        const float4 a = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
        const float4 b = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
        const float av[4] = {a.x, a.y, a.z, a.w};
        const float2 nb0 = make_float2(-b.x, -b.y), nb1 = make_float2(-b.z, -b.w);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 d0 = add2(bcast2(av[i]), nb0), d1 = add2(bcast2(av[i]), nb1);
          acc[i][0] = fma2(d0, d0, acc[i][0]);
          acc[i][1] = fma2(d1, d1, acc[i][1]);
        }
      }
    } else {
#pragma unroll
      for (int k = 0; k < TK; ++k) {
        const double2 a01 = *reinterpret_cast<const double2*>(&As[k][ty * 4]);
        const double2 a23 = *reinterpret_cast<const double2*>(&As[k][ty * 4 + 2]);
        const double2 b01 = *reinterpret_cast<const double2*>(&Bs[k][tx * 4]);
        const double2 b23 = *reinterpret_cast<const double2*>(&Bs[k][tx * 4 + 2]);
        const double av[4] = {a01.x, a01.y, a23.x, a23.y}, bv[4] = {b01.x, b01.y, b23.x, b23.y};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const double d = __dsub_rn(av[i], bv[j]);
            accd[i][j] = __fma_rn(d, d, accd[i][j]);
          }
      }
    }
    __syncthreads();
  }
  T o[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    if constexpr (std::is_same<T, float>::value) {
      o[i][0] = acc[i][0].x; o[i][1] = acc[i][0].y; o[i][2] = acc[i][1].x; o[i][3] = acc[i][1].y;
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) o[i][j] = accd[i][j];
    }
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (SQRT) o[i][j] = sqrt(o[i][j]);
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = i0 + ty * 4 + i;
    if (r >= RA) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int c = j0 + tx * 4 + j;
      if (c < RB) D[(long long)r * ldd + c] = o[i][j];
    }
  }
  if (SYM && blockIdx.x != blockIdx.y) {             // mirror image of an off-diagonal tile
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int c = j0 + tx * 4 + j;
      if (c >= RB) continue;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int r = i0 + ty * 4 + i;
        if (r < RA) D[(long long)c * ldd + r] = o[i][j];
      }
    }
  }
}

// k-means++ candidate scoring (sklearn _kmeans.py:231-262): squared distances from every row of S to a handful of
// candidate rows of S.  HBM-bound form: one warp per row streams it once with 16-byte (fp32) / 32-byte (fp64) loads
// against the (L1-hot) candidate rows, differences in T, squares accumulated in fp64 (sklearn scores candidates in
// float64).  The 64 x 64-tile kernel above is latency-bound for this shape (a few dozen blocks), and it runs once per
// candidate round of every init.
template <typename T, int NC>
__global__ void __launch_bounds__(256)
cand_dist_kernel(const T* __restrict__ S, int R, int G, int ld, const int32_t* __restrict__ idx, int n_c,
                 T* __restrict__ out /* n_c x R */) {
  using V4 = typename Vec4<T>::type;
  const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (r >= R) return;
  const V4* row = reinterpret_cast<const V4*>(S + (long long)r * ld);
  const V4* cand[NC];
#pragma unroll
  for (int c = 0; c < NC; ++c) cand[c] = reinterpret_cast<const V4*>(S + (long long)idx[c < n_c ? c : 0] * ld);
  double acc[NC];
#pragma unroll
  for (int c = 0; c < NC; ++c) acc[c] = 0.0;
  const int g4 = G / 4;
  for (int q = lane; q < g4; q += 32) {
    const V4 x = row[q];
#pragma unroll
    for (int c = 0; c < NC; ++c) {
      const V4 y = cand[c][q];
      const T d0 = x.x - y.x, d1 = x.y - y.y, d2 = x.z - y.z, d3 = x.w - y.w;
      acc[c] += (double)d0 * d0 + (double)d1 * d1 + (double)d2 * d2 + (double)d3 * d3;
    }
  }
  for (int g = 4 * g4 + lane; g < G; g += 32) {      // ragged tail
    const T x = S[(long long)r * ld + g];
#pragma unroll
    for (int c = 0; c < NC; ++c) {
      const T d = x - S[(long long)idx[c < n_c ? c : 0] * ld + g];
      acc[c] += (double)d * d;
    }
  }
#pragma unroll
  for (int c = 0; c < NC; ++c) {
    const double v = warp_sum(acc[c]);
    if (lane == 0 && c < n_c) out[(long long)c * R + r] = (T)v;
  }
}

// ---------------------------------------------------------------- C3: sum of the m smallest entries of each row
// Exact MSB-first radix select on the (non-negative) bit patterns, one block per row.
template <typename T>
__global__ void __launch_bounds__(256)
knn_density_kernel(const T* __restrict__ D, int R, int ldd, int m /* n_neighbors + 1 */, int n_neighbors,
                   T* __restrict__ density) {
  using U = typename Bits<T>::U;
  __shared__ int smi[33];
  __shared__ double smd[33];
  const int r = blockIdx.x;
  const T* row = D + (long long)r * ldd;
  U prefix = 0;
  int k = m - 1;   // 0-based rank of the threshold element
  for (int bit = Bits<T>::kTop; bit >= 0; --bit) {
    const U mask_hi = radix_mask_hi<U>(bit);
    int cnt = 0;
    for (int j = threadIdx.x; j < R; j += blockDim.x) {
      const U u = Bits<T>::of(row[j]);
      cnt += ((u & mask_hi) == prefix) && !((u >> bit) & U(1));
    }
    cnt = block_sum_all(cnt, smi);
    if (k >= cnt) {
      k -= cnt;
      prefix |= (U(1) << bit);
    }
  }
  const T tau = Bits<T>::value(prefix);   // the m-th smallest value
  double s = 0.0;
  int less = 0;
  for (int j = threadIdx.x; j < R; j += blockDim.x) {
    const T v = row[j];
    if (v < tau) {
      s += (double)v;
      ++less;
    }
  }
  s = block_sum_all(s, smd);
  less = block_sum_all(less, smi);
  if (threadIdx.x == 0) density[r] = (T)((s + (double)(m - less) * (double)tau) / (double)n_neighbors);
}

// ---------------------------------------------------------------- C5: Lloyd E step
// one warp per row: direct squared distances to the K centres held in shared memory (K*G*sizeof(T) bytes may
// exceed smem for large G, so centres are read through L1/L2 instead; they are tiny and hot).
template <typename T>
__global__ void __launch_bounds__(256)
kmeans_assign_kernel(const T* __restrict__ S, int R, int G, int ld, const T* __restrict__ C, int K, int ldc,
                     int32_t* __restrict__ labels, T* __restrict__ mind, int* __restrict__ n_changed) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= R) return;
  const T* x = S + (long long)warp * ld;
  T best = T(0);
  int bl = 0;
  for (int c = 0; c < K; ++c) {
    const T* cc = C + (long long)c * ldc;
    T a = T(0);
    for (int g = lane; g < G; g += 32) {
      const T d = x[g] - cc[g];
      a = fma(d, d, a);
    }
    a = warp_sum(a);
    if (c == 0 || a < best) {   // strict '<': first minimum wins (sklearn _k_means_lloyd.pyx:205-209)
      best = a;
      bl = c;
    }
  }
  if (lane == 0) {
    if (labels[warp] != bl) atomicAdd(n_changed, 1);
    labels[warp] = bl;
    mind[warp] = best;
  }
}

// stable counting sort of row indices by label: thread c lists the members of cluster c in row order
__global__ void members_kernel(const int32_t* __restrict__ labels, int R, int K, int32_t* __restrict__ counts,
                               int32_t* __restrict__ order /* K x R */) {
  const int c = threadIdx.x;
  if (c >= K) return;
  int n = 0;
  for (int i = 0; i < R; ++i)
    if (labels[i] == c) order[(long long)c * R + n++] = i;
  counts[c] = n;
}

// M step: per-cluster column sums in fp64, members visited in row order (deterministic)
template <typename T>
__global__ void __launch_bounds__(128)
cluster_sums_kernel(const T* __restrict__ S, int G, int ld, const int32_t* __restrict__ counts,
                    const int32_t* __restrict__ order, int R, double* __restrict__ sums /* K x G */) {
  const int c = blockIdx.y;
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= G) return;
  const int n = counts[c];
  const int32_t* mem = order + (long long)c * R;
  double a = 0.0;
  for (int i = 0; i < n; ++i) a += (double)S[(long long)mem[i] * ld + g];
  sums[(long long)c * G + g] = a;
}

// M step, second half, on the device: new centre = sums * (1 / count) (sklearn _k_means_common.pyx:274-298),
// squared shift against the current centre; with T = float also the fp32 copy CT_new for the next E step (with
// T = double the E step reads C64_new itself).  One block per cluster; a cluster without members raises `any_empty`
// and is left to the host's relocation rule (the caller keeps the old centres).
template <typename T>
__global__ void __launch_bounds__(256)
centre_update_kernel(const double* __restrict__ sums, const int32_t* __restrict__ counts, int G,
                     const double* __restrict__ C64_cur, double* __restrict__ C64_new, T* __restrict__ CT_new,
                     double* __restrict__ shift_part, int* __restrict__ any_empty) {
  __shared__ double sm[33];
  const int j = blockIdx.x;
  const int w = counts[j];
  if (w == 0) {
    if (threadIdx.x == 0) {
      atomicExch(any_empty, 1);
      shift_part[j] = 0.0;
    }
    return;
  }
  const double inv = 1.0 / (double)w;
  double acc = 0.0;
  for (int g = threadIdx.x; g < G; g += blockDim.x) {
    const double nv = sums[(long long)j * G + g] * inv;
    const double d = nv - C64_cur[(long long)j * G + g];
    acc += d * d;
    C64_new[(long long)j * G + g] = nv;
    if constexpr (!std::is_same<T, double>::value) CT_new[(long long)j * G + g] = (T)nv;
  }
  acc = block_sum_all(acc, sm);
  if (threadIdx.x == 0) shift_part[j] = acc;
}

template <typename T>
__global__ void sum_kernel(const T* __restrict__ v, int n, double* __restrict__ out) {
  __shared__ double sm[33];
  double a = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) a += (double)v[i];
  a = block_sum_all(a, sm);
  if (threadIdx.x == 0) *out = a;
}

// ---------------------------------------------------------------- C6: per-(cluster, gene) median by radix select
template <typename T>
__device__ __forceinline__ T select_kth(const T* __restrict__ S, int ld, int g, const int32_t* mem, int n, int k) {
  using U = typename Bits<T>::U;
  U prefix = 0;
  for (int bit = Bits<T>::kTop; bit >= 0; --bit) {
    const U mask_hi = radix_mask_hi<U>(bit);
    int cnt = 0;
    for (int i = 0; i < n; ++i) {
      const U u = Bits<T>::of(S[(long long)mem[i] * ld + g]);
      cnt += ((u & mask_hi) == prefix) && !((u >> bit) & U(1));
    }
    if (k >= cnt) {
      k -= cnt;
      prefix |= (U(1) << bit);
    }
  }
  return Bits<T>::value(prefix);
}

template <typename T>
__global__ void __launch_bounds__(128)
cluster_median_kernel(const T* __restrict__ S, int G, int ld, const int32_t* __restrict__ counts,
                      const int32_t* __restrict__ order, int R, T* __restrict__ M, int ldm) {
  const int c = blockIdx.y;
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= G) return;
  const int n = counts[c];
  const int32_t* mem = order + (long long)c * R;
  T med = Bits<T>::nan();                  // NaN for an empty cluster (pandas drops the group)
  if (n > 0) {
    if (n & 1) {
      med = select_kth(S, ld, g, mem, n, n / 2);
    } else {
      const T v1 = select_kth(S, ld, g, mem, n, n / 2 - 1);
      int le = 0;
      T nxt = Bits<T>::inf();
      for (int i = 0; i < n; ++i) {
        const T v = S[(long long)mem[i] * ld + g];
        le += (v <= v1);
        if (v > v1) nxt = fmin(nxt, v);
      }
      const T v2 = (le >= n / 2 + 1) ? v1 : nxt;
      med = T(0.5) * (v1 + v2);             // pandas: (a + b) / 2 of the two middle values
    }
  }
  M[(long long)c * ldm + g] = med;
}

template <typename T>
__global__ void row_normalize_sum_kernel(T* __restrict__ M, int G, int ldm) {
  __shared__ double sm[33];
  T* row = M + (long long)blockIdx.x * ldm;
  double s = 0.0;
  for (int g = threadIdx.x; g < G; g += blockDim.x) s += (double)row[g];
  s = block_sum_all(s, sm);
  for (int g = threadIdx.x; g < G; g += blockDim.x) row[g] = (T)((double)row[g] / s);
}

// per-row sums of distances to the members of every cluster (silhouette_score, cnmf.py:923):
// one block per row; per-warp cluster bins in shared memory, folded in warp order (deterministic)
template <typename T>
__global__ void __launch_bounds__(256)
cluster_dist_sums_kernel(const T* __restrict__ D, int R, const int32_t* __restrict__ labels, int K,
                         double* __restrict__ out /* R x K */) {
  extern __shared__ double bins[];        // 8 warps x K
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < 8 * K; i += blockDim.x) bins[i] = 0.0;
  __syncthreads();
  const T* row = D + (long long)blockIdx.x * R;
  // each warp owns a contiguous slice of columns and walks it in order, lane by lane
  const int per = (R + 7) / 8;
  const int j0 = warp * per, j1 = min(R, j0 + per);
  for (int jb = j0; jb < j1; jb += 32) {
    const int j = jb + lane;
    const double v = (j < j1) ? (double)row[j] : 0.0;
    const int lab = (j < j1) ? labels[j] : -1;
    for (int l = 0; l < 32; ++l) {        // serialise the lanes: fixed summation order
      const double vl = __shfl_sync(0xffffffffu, v, l);
      const int ll = __shfl_sync(0xffffffffu, lab, l);
      if (lane == 0 && ll >= 0) bins[warp * K + ll] += vl;
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < K; c += blockDim.x) {
    double s = 0.0;
    for (int w = 0; w < 8; ++w) s += bins[w * K + c];
    out[(long long)blockIdx.x * K + c] = s;
  }
}

template <typename T>
__global__ void col_stats_dev_kernel(const T* __restrict__ X, int rows, int cols, int ld, double* __restrict__ sum,
                                    double* __restrict__ sq) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= cols) return;
  double s = 0.0, q = 0.0;
  for (int r = 0; r < rows; ++r) {           // fixed order: deterministic
    const double v = X[(long long)r * ld + c];
    s += v;
    q += v * v;
  }
  sum[c] = s;
  sq[c] = q;
}

template <typename T>
__global__ void gather_rows_idx_kernel(const T* __restrict__ src, int ld_src, const int32_t* __restrict__ idx,
                                       int G, T* __restrict__ dst, int ld_dst) {
  const T* s = src + (long long)idx[blockIdx.x] * ld_src;
  T* d = dst + (long long)blockIdx.x * ld_dst;
  for (int g = threadIdx.x; g < G; g += blockDim.x) d[g] = s[g];
}

// ---------------------------------------------------------------- entry points, one body per element type
template <typename T>
int l2_normalize_rows(cnmf_handle_t h, T* S, int R, int G, int ld, void* stream) {
  CNMF_REQUIRE(h && S && R > 0 && G > 0 && ld >= G, "l2_normalize_rows: bad arguments");
  CNMF_CUDA_CHECK(cudaSetDevice(h->device));
  l2_normalize_kernel<T><<<R, 256, 0, as_stream(stream)>>>(S, R, G, ld);
  CNMF_CUDA_CHECK(cudaGetLastError());
  h->launches += 1;
  return 0;
}

template <typename T>
int local_density(cnmf_handle_t h, const T* S, int R, int G, int ld, int n_neighbors, T* density_dev, T* D_dev,
                  void* stream) {
  CNMF_REQUIRE(h && S && density_dev && R > 0 && G > 0 && ld >= G, "local_density: bad arguments");
  CNMF_REQUIRE(n_neighbors >= 1 && n_neighbors + 1 <= R, "local_density: need 1 <= n_neighbors < R");
  cudaStream_t s = as_stream(stream);
  CNMF_CUDA_CHECK(cudaSetDevice(h->device));
  T* D = D_dev ? D_dev : static_cast<T*>(h->dev_buf("consensus.D", (size_t)R * R * sizeof(T)));
  if (!D) return -2;
  dim3 grid((R + 63) / 64, (R + 63) / 64);
  pair_dist_kernel<T, true, true><<<grid, 256, 0, s>>>(S, R, ld, S, R, ld, G, D, R);
  CNMF_CUDA_CHECK(cudaGetLastError());
  knn_density_kernel<T><<<R, 256, 0, s>>>(D, R, R, n_neighbors + 1, n_neighbors, density_dev);
  CNMF_CUDA_CHECK(cudaGetLastError());
  h->launches += 2;
  return 0;
}

template <typename T>
int col_stats_dev(cnmf_handle_t h, const T* S, int R, int G, int ld, double* mean_host, double* var_host,
                  void* stream) {
  CNMF_REQUIRE(h && S && mean_host && var_host && R > 0 && G > 0, "col_stats_dev: bad arguments");
  cudaStream_t s = as_stream(stream);
  CNMF_CUDA_CHECK(cudaSetDevice(h->device));
  double* buf = static_cast<double*>(h->dev_buf("consensus.colstats", sizeof(double) * 2 * G));
  if (!buf) return -2;
  col_stats_dev_kernel<T><<<(G + 127) / 128, 128, 0, s>>>(S, R, G, ld, buf, buf + G);
  CNMF_CUDA_CHECK(cudaGetLastError());
  h->launches += 1;
  CNMF_CUDA_CHECK(cudaMemcpyAsync(mean_host, buf, sizeof(double) * G, cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaMemcpyAsync(var_host, buf + G, sizeof(double) * G, cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
  for (int c = 0; c < G; ++c) {
    const double m = mean_host[c] / R;
    mean_host[c] = m;
    var_host[c] = std::max(var_host[c] / R - m * m, 0.0);
  }
  return 0;
}

template <typename T>
int cluster_dist_sums(cnmf_handle_t h, const T* S, int R, int G, int ld, const int32_t* labels_dev, int K,
                      double* sums_host, void* stream) {
  CNMF_REQUIRE(h && S && labels_dev && sums_host && R > 0 && K >= 1 && K <= 512, "cluster_dist_sums: bad arguments");
  cudaStream_t s = as_stream(stream);
  CNMF_CUDA_CHECK(cudaSetDevice(h->device));
  T* D = static_cast<T*>(h->dev_buf("consensus.D", (size_t)R * R * sizeof(T)));
  double* out = static_cast<double*>(h->dev_buf("consensus.dsums", sizeof(double) * (size_t)R * K));
  if (!D || !out) return -2;
  dim3 grid((R + 63) / 64, (R + 63) / 64);
  pair_dist_kernel<T, true, true><<<grid, 256, 0, s>>>(S, R, ld, S, R, ld, G, D, R);
  cluster_dist_sums_kernel<T><<<R, 256, sizeof(double) * 8 * K, s>>>(D, R, labels_dev, K, out);
  CNMF_CUDA_CHECK(cudaGetLastError());
  h->launches += 2;
  CNMF_CUDA_CHECK(cudaMemcpyAsync(sums_host, out, sizeof(double) * (size_t)R * K, cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
  return 0;
}

template <typename T>
int gather_rows(cnmf_handle_t h, const T* src_dev, int ld_src, const int32_t* idx_host, int n, int G, T* dst_dev,
                int ld_dst, void* stream) {
  CNMF_REQUIRE(h && src_dev && idx_host && dst_dev && n > 0 && G > 0, "gather_rows: bad arguments");
  cudaStream_t s = as_stream(stream);
  CNMF_CUDA_CHECK(cudaSetDevice(h->device));
  int32_t* d_idx = static_cast<int32_t*>(h->dev_buf("consensus.idx", sizeof(int32_t) * n));
  if (!d_idx) return -2;
  CNMF_CUDA_CHECK(cudaMemcpyAsync(d_idx, idx_host, sizeof(int32_t) * n, cudaMemcpyHostToDevice, s));
  gather_rows_idx_kernel<T><<<n, 256, 0, s>>>(src_dev, ld_src, d_idx, G, dst_dev, ld_dst);
  CNMF_CUDA_CHECK(cudaGetLastError());
  CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
  h->launches += 1;
  return 0;
}

template <typename T>
int sq_dists_to_rows(cnmf_handle_t h, const T* S, int R, int G, int ld, const int32_t* idx_host, int n_c, T* out_host,
                     void* stream) {
  CNMF_REQUIRE(h && S && idx_host && out_host && n_c > 0 && R > 0, "sq_dists_to_rows: bad arguments");
  cudaStream_t s = as_stream(stream);
  CNMF_CUDA_CHECK(cudaSetDevice(h->device));
  T* C = static_cast<T*>(h->dev_buf("consensus.cand", (size_t)n_c * ld * sizeof(T)));
  T* out = static_cast<T*>(h->dev_buf("consensus.cand_out", (size_t)n_c * R * sizeof(T)));
  int32_t* d_idx = static_cast<int32_t*>(h->dev_buf("consensus.idx", sizeof(int32_t) * std::max(n_c, 1)));
  if (!C || !out || !d_idx) return -2;
  CNMF_CUDA_CHECK(cudaMemcpyAsync(d_idx, idx_host, sizeof(int32_t) * n_c, cudaMemcpyHostToDevice, s));
  if (n_c <= 8 && ld % 4 == 0) {
    const int blocks = (R * 32 + 255) / 256;
    if (n_c <= 2) cand_dist_kernel<T, 2><<<blocks, 256, 0, s>>>(S, R, G, ld, d_idx, n_c, out);
    else if (n_c <= 4) cand_dist_kernel<T, 4><<<blocks, 256, 0, s>>>(S, R, G, ld, d_idx, n_c, out);
    else cand_dist_kernel<T, 8><<<blocks, 256, 0, s>>>(S, R, G, ld, d_idx, n_c, out);
  } else {
    gather_rows_idx_kernel<T><<<n_c, 256, 0, s>>>(S, ld, d_idx, G, C, ld);
    dim3 grid((R + 63) / 64, (n_c + 63) / 64);
    pair_dist_kernel<T, false, false><<<grid, 256, 0, s>>>(C, n_c, ld, S, R, ld, G, out, R);
  }
  CNMF_CUDA_CHECK(cudaGetLastError());
  CNMF_CUDA_CHECK(cudaMemcpyAsync(out_host, out, (size_t)n_c * R * sizeof(T), cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
  h->launches += 2;
  return 0;
}

template <typename T>
int kmeans_assign(cnmf_handle_t h, const T* S, int R, int G, int ld, const T* centers_host, int K, int32_t* labels_dev,
                  double* sums_host, int32_t* counts_host, T* mind_dev, int32_t* n_changed_host, double* inertia_host,
                  void* stream) {
  CNMF_REQUIRE(h && S && centers_host && labels_dev && mind_dev && K >= 1 && K <= 1024 && R > 0,
               "kmeans_assign: bad arguments");
  cudaStream_t s = as_stream(stream);
  CNMF_CUDA_CHECK(cudaSetDevice(h->device));
  T* C = static_cast<T*>(h->dev_buf("kmeans.C", (size_t)K * G * sizeof(T)));
  int32_t* cnt = static_cast<int32_t*>(h->dev_buf("kmeans.cnt", sizeof(int32_t) * (K + 2)));
  int32_t* order = static_cast<int32_t*>(h->dev_buf("kmeans.order", sizeof(int32_t) * (size_t)K * R));
  double* sums = static_cast<double*>(h->dev_buf("kmeans.sums", sizeof(double) * ((size_t)K * G + 1)));
  if (!C || !cnt || !order || !sums) return -2;
  int* n_changed = cnt + K;
  CNMF_CUDA_CHECK(cudaMemcpyAsync(C, centers_host, (size_t)K * G * sizeof(T), cudaMemcpyHostToDevice, s));
  CNMF_CUDA_CHECK(cudaMemsetAsync(n_changed, 0, sizeof(int), s));
  kmeans_assign_kernel<T><<<(R * 32 + 255) / 256, 256, 0, s>>>(S, R, G, ld, C, K, G, labels_dev, mind_dev, n_changed);
  CNMF_CUDA_CHECK(cudaGetLastError());
  h->launches += 1;
  if (sums_host) {
    members_kernel<<<1, 1024, 0, s>>>(labels_dev, R, K, cnt, order);
    dim3 grid((G + 127) / 128, K);
    cluster_sums_kernel<T><<<grid, 128, 0, s>>>(S, G, ld, cnt, order, R, sums);
    CNMF_CUDA_CHECK(cudaGetLastError());
    h->launches += 2;
    CNMF_CUDA_CHECK(cudaMemcpyAsync(sums_host, sums, sizeof(double) * (size_t)K * G, cudaMemcpyDeviceToHost, s));
    if (counts_host) CNMF_CUDA_CHECK(cudaMemcpyAsync(counts_host, cnt, sizeof(int32_t) * K, cudaMemcpyDeviceToHost, s));
  }
  if (inertia_host) {
    sum_kernel<T><<<1, 1024, 0, s>>>(mind_dev, R, sums + (size_t)K * G);
    CNMF_CUDA_CHECK(cudaGetLastError());
    h->launches += 1;
    CNMF_CUDA_CHECK(cudaMemcpyAsync(inertia_host, sums + (size_t)K * G, sizeof(double), cudaMemcpyDeviceToHost, s));
  }
  if (n_changed_host) CNMF_CUDA_CHECK(cudaMemcpyAsync(n_changed_host, n_changed, sizeof(int), cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
  return 0;
}

// CE_cur: the centres the E step reads (the fp32 copy for T = float, C64_cur itself for T = double); CE_new receives
// the copy of C64_new for the next E step (T = float only)
template <typename T>
int kmeans_step(cnmf_handle_t h, const T* S, int R, int G, int ld, int K, const T* CE_cur, const double* C64_cur,
                double* C64_new, T* CE_new, int32_t* labels_dev, T* mind_dev, double* sums_dev, int32_t* counts_dev,
                int32_t* n_changed_host, int32_t* any_empty_host, double* shift_host, void* stream) {
  cudaStream_t s = as_stream(stream);
  CNMF_CUDA_CHECK(cudaSetDevice(h->device));
  int32_t* order = static_cast<int32_t*>(h->dev_buf("kmeans.order", sizeof(int32_t) * (size_t)K * R));
  int32_t* flags = static_cast<int32_t*>(h->dev_buf("kmeans.flags", sizeof(int32_t) * 2));
  double* shift_part = static_cast<double*>(h->dev_buf("kmeans.shift", sizeof(double) * K));
  struct HostOut { int32_t flags[2]; double shift[1024]; };
  HostOut* ho = static_cast<HostOut*>(h->host_buf("kmeans.step_out", sizeof(HostOut)));
  if (!order || !flags || !shift_part || !ho) return -2;
  CNMF_CUDA_CHECK(cudaMemsetAsync(flags, 0, sizeof(int32_t) * 2, s));
  kmeans_assign_kernel<T><<<(R * 32 + 255) / 256, 256, 0, s>>>(S, R, G, ld, CE_cur, K, G, labels_dev, mind_dev, flags);
  members_kernel<<<1, 1024, 0, s>>>(labels_dev, R, K, counts_dev, order);
  dim3 grid((G + 127) / 128, K);
  cluster_sums_kernel<T><<<grid, 128, 0, s>>>(S, G, ld, counts_dev, order, R, sums_dev);
  centre_update_kernel<T><<<K, 256, 0, s>>>(sums_dev, counts_dev, G, C64_cur, C64_new, CE_new, shift_part, flags + 1);
  CNMF_CUDA_CHECK(cudaGetLastError());
  h->launches += 4;
  CNMF_CUDA_CHECK(cudaMemcpyAsync(ho->flags, flags, sizeof(int32_t) * 2, cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaMemcpyAsync(ho->shift, shift_part, sizeof(double) * K, cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
  *n_changed_host = ho->flags[0];
  *any_empty_host = ho->flags[1];
  double tot = 0.0;
  for (int j = 0; j < K; ++j) tot += ho->shift[j];      // fixed order
  *shift_host = tot;
  return 0;
}

template <typename T>
int cluster_median(cnmf_handle_t h, const T* S, int R, int G, int ld, const int32_t* labels_dev, int K, T* M_dev,
                   int ldm, void* stream) {
  CNMF_REQUIRE(h && S && labels_dev && M_dev && K >= 1 && K <= 1024 && R > 0 && ldm >= G, "cluster_median: bad arguments");
  cudaStream_t s = as_stream(stream);
  CNMF_CUDA_CHECK(cudaSetDevice(h->device));
  int32_t* cnt = static_cast<int32_t*>(h->dev_buf("kmeans.cnt", sizeof(int32_t) * (K + 2)));
  int32_t* order = static_cast<int32_t*>(h->dev_buf("kmeans.order", sizeof(int32_t) * (size_t)K * R));
  if (!cnt || !order) return -2;
  members_kernel<<<1, 1024, 0, s>>>(labels_dev, R, K, cnt, order);
  dim3 grid((G + 127) / 128, K);
  cluster_median_kernel<T><<<grid, 128, 0, s>>>(S, G, ld, cnt, order, R, M_dev, ldm);
  row_normalize_sum_kernel<T><<<K, 256, 0, s>>>(M_dev, G, ldm);
  CNMF_CUDA_CHECK(cudaGetLastError());
  h->launches += 3;
  return 0;
}

}  // namespace

extern "C" {

int cnmf_l2_normalize_rows(cnmf_handle_t h, float* S, int R, int G, int ld, void* stream) {
  return l2_normalize_rows(h, S, R, G, ld, stream);
}
int cnmf_l2_normalize_rows_f64(cnmf_handle_t h, double* S, int R, int G, int ld, void* stream) {
  return l2_normalize_rows(h, S, R, G, ld, stream);
}

int cnmf_local_density(cnmf_handle_t h, const float* S, int R, int G, int ld, int n_neighbors, float* density_dev,
                       float* D_dev, void* stream) {
  return local_density(h, S, R, G, ld, n_neighbors, density_dev, D_dev, stream);
}
int cnmf_local_density_f64(cnmf_handle_t h, const double* S, int R, int G, int ld, int n_neighbors,
                           double* density_dev, double* D_dev, void* stream) {
  return local_density(h, S, R, G, ld, n_neighbors, density_dev, D_dev, stream);
}

int cnmf_col_stats_dev(cnmf_handle_t h, const float* S, int R, int G, int ld, double* mean_host, double* var_host,
                       void* stream) {
  return col_stats_dev(h, S, R, G, ld, mean_host, var_host, stream);
}
int cnmf_col_stats_dev_f64(cnmf_handle_t h, const double* S, int R, int G, int ld, double* mean_host, double* var_host,
                           void* stream) {
  return col_stats_dev(h, S, R, G, ld, mean_host, var_host, stream);
}

int cnmf_cluster_dist_sums(cnmf_handle_t h, const float* S, int R, int G, int ld, const int32_t* labels_dev, int K,
                           double* sums_host, void* stream) {
  return cluster_dist_sums(h, S, R, G, ld, labels_dev, K, sums_host, stream);
}
int cnmf_cluster_dist_sums_f64(cnmf_handle_t h, const double* S, int R, int G, int ld, const int32_t* labels_dev, int K,
                               double* sums_host, void* stream) {
  return cluster_dist_sums(h, S, R, G, ld, labels_dev, K, sums_host, stream);
}

int cnmf_gather_rows(cnmf_handle_t h, const float* src_dev, int ld_src, const int32_t* idx_host, int n, int G,
                     float* dst_dev, int ld_dst, void* stream) {
  return gather_rows(h, src_dev, ld_src, idx_host, n, G, dst_dev, ld_dst, stream);
}
int cnmf_gather_rows_f64(cnmf_handle_t h, const double* src_dev, int ld_src, const int32_t* idx_host, int n, int G,
                         double* dst_dev, int ld_dst, void* stream) {
  return gather_rows(h, src_dev, ld_src, idx_host, n, G, dst_dev, ld_dst, stream);
}

int cnmf_sq_dists_to_rows(cnmf_handle_t h, const float* S, int R, int G, int ld, const int32_t* idx_host, int n_c,
                          float* out_host, void* stream) {
  return sq_dists_to_rows(h, S, R, G, ld, idx_host, n_c, out_host, stream);
}
int cnmf_sq_dists_to_rows_f64(cnmf_handle_t h, const double* S, int R, int G, int ld, const int32_t* idx_host, int n_c,
                              double* out_host, void* stream) {
  return sq_dists_to_rows(h, S, R, G, ld, idx_host, n_c, out_host, stream);
}

int cnmf_kmeans_assign(cnmf_handle_t h, const float* S, int R, int G, int ld, const float* centers_host, int K,
                       int32_t* labels_dev, double* sums_host, int32_t* counts_host, float* mind_dev,
                       int32_t* n_changed_host, double* inertia_host, void* stream) {
  return kmeans_assign(h, S, R, G, ld, centers_host, K, labels_dev, sums_host, counts_host, mind_dev, n_changed_host,
                       inertia_host, stream);
}
int cnmf_kmeans_assign_f64(cnmf_handle_t h, const double* S, int R, int G, int ld, const double* centers_host, int K,
                           int32_t* labels_dev, double* sums_host, int32_t* counts_host, double* mind_dev,
                           int32_t* n_changed_host, double* inertia_host, void* stream) {
  return kmeans_assign(h, S, R, G, ld, centers_host, K, labels_dev, sums_host, counts_host, mind_dev, n_changed_host,
                       inertia_host, stream);
}

int cnmf_kmeans_step(cnmf_handle_t h, const float* S, int R, int G, int ld, int K, const float* C32_cur,
                     const double* C64_cur, double* C64_new, float* C32_new, int32_t* labels_dev, float* mind_dev,
                     double* sums_dev, int32_t* counts_dev, int32_t* n_changed_host, int32_t* any_empty_host,
                     double* shift_host, void* stream) {
  CNMF_REQUIRE(h && S && C32_cur && C64_cur && C64_new && C32_new && labels_dev && mind_dev && sums_dev && counts_dev &&
                   n_changed_host && any_empty_host && shift_host && K >= 1 && K <= 1024 && R > 0,
               "kmeans_step: bad arguments");
  return kmeans_step(h, S, R, G, ld, K, C32_cur, C64_cur, C64_new, C32_new, labels_dev, mind_dev, sums_dev, counts_dev,
                     n_changed_host, any_empty_host, shift_host, stream);
}
int cnmf_kmeans_step_f64(cnmf_handle_t h, const double* S, int R, int G, int ld, int K, const double* C64_cur,
                         double* C64_new, int32_t* labels_dev, double* mind_dev, double* sums_dev, int32_t* counts_dev,
                         int32_t* n_changed_host, int32_t* any_empty_host, double* shift_host, void* stream) {
  CNMF_REQUIRE(h && S && C64_cur && C64_new && labels_dev && mind_dev && sums_dev && counts_dev && n_changed_host &&
                   any_empty_host && shift_host && K >= 1 && K <= 1024 && R > 0,
               "kmeans_step_f64: bad arguments");
  return kmeans_step<double>(h, S, R, G, ld, K, C64_cur, C64_cur, C64_new, nullptr, labels_dev, mind_dev, sums_dev,
                             counts_dev, n_changed_host, any_empty_host, shift_host, stream);
}

int cnmf_cluster_median(cnmf_handle_t h, const float* S, int R, int G, int ld, const int32_t* labels_dev, int K,
                        float* M_dev, int ldm, void* stream) {
  return cluster_median(h, S, R, G, ld, labels_dev, K, M_dev, ldm, stream);
}
int cnmf_cluster_median_f64(cnmf_handle_t h, const double* S, int R, int G, int ld, const int32_t* labels_dev, int K,
                            double* M_dev, int ldm, void* stream) {
  return cluster_median(h, S, R, G, ld, labels_dev, K, M_dev, ldm, stream);
}

}  // extern "C"
