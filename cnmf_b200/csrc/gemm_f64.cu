// float64 tensor-core GEMM: packed fp64 rows times the dataset's X, in either orientation, on the fp64 MMA
// (mma.sync m16n8k16 .f64 -> DMMA.16x8x16; Hopper has no fp64 wgmma).  X is the fp32 matrix of an ordinary dataset
// (the NNDSVD range finder, nndsvd.cu) or the fp64 matrix of a float64 dataset (its NNDSVD starts and the float64
// solver's two products, nmf_f64.cu); the element type only changes how a tile is loaded.
//
//   to_genes = false:  C[m, i] = sum_g A[m, g] X[i, g]     (A over genes, output over cells; X read K-major)
//   to_genes = true:   C[m, g] = sum_i A[m, i] X[i, g]     (A over cells, output over genes; X read MN-major)
//
// An fp32 X is converted to fp64 on its way into shared memory: no fp64 or transposed copy of it exists.  Every output
// element accumulates its K tiles in ascending order, one MMA per 16-deep tile, whatever M is and wherever its row
// sits in the tile: a restart's products do not depend on the other restarts of the call.
#include <cuda_runtime.h>

#include "common.cuh"
#include "engine.h"

namespace cnmf {

namespace {

constexpr int F64_BM = 64, F64_BN = 128, F64_BK = 16;
constexpr int F64_PAD = F64_BK + 4;      // smem row stride (doubles): fragment reads take the minimum 2 wavefronts
constexpr int F64_THREADS = 256;         // 8 warps: 2 along M x 4 along N, 32 x 32 outputs each

__device__ __forceinline__ void mma_f64_16816(double (&d)[4], const double (&a)[8], const double (&b)[4]) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
      "{%12,%13,%14,%15}, {%0,%1,%2,%3};"
      : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
      : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]),
        "d"(b[2]), "d"(b[3]));
}

// 8 consecutive elements of X (16-byte aligned for float, 64-byte for double) into registers
__device__ __forceinline__ void load8(const float* p, float (&r)[8]) {
  const float4* src = reinterpret_cast<const float4*>(p);
  const float4 v0 = src[0], v1 = src[1];
  r[0] = v0.x; r[1] = v0.y; r[2] = v0.z; r[3] = v0.w;
  r[4] = v1.x; r[5] = v1.y; r[6] = v1.z; r[7] = v1.w;
}
__device__ __forceinline__ void load8(const double* p, double (&r)[8]) {
  const double2* src = reinterpret_cast<const double2*>(p);
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const double2 v = src[e];
    r[2 * e] = v.x; r[2 * e + 1] = v.y;
  }
}

template <bool TO_GENES, typename TX>
__global__ void __launch_bounds__(F64_THREADS)
gemm_f64_kernel(const double* __restrict__ A, int lda, int M, int K, const TX* __restrict__ X, int ldx, int n_rows,
                double* __restrict__ C, int ldc, int n_out, int k_chunk, long long c_split_stride) {
  // split-K slice blockIdx.z: reduction elements [z * k_chunk, (z + 1) * k_chunk), its own C slice.  One slice (the
  // solver's products) is the whole reduction.
  {
    const int kz0 = blockIdx.z * k_chunk;
    const int kn = min(k_chunk, K - kz0);
    A += kz0;
    X += TO_GENES ? (long long)kz0 * ldx : (long long)kz0;
    if (TO_GENES) n_rows = kn;
    K = kn;
    C += blockIdx.z * c_split_stride;
  }
  __shared__ double As[F64_BM][F64_PAD];
  __shared__ double Bs[F64_BN][F64_PAD];      // [output item][k]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int wm = (warp & 1) * 32, wn = (warp >> 1) * 32;
  const int m0 = blockIdx.y * F64_BM, n0 = blockIdx.x * F64_BN;

  // global -> register staging of one K tile
  const int a_row = tid >> 2, a_k = (tid & 3) * 4;
  double ra[4];
  TX rb[8];
  auto load_tile = [&](int k0) {
    const long long am = m0 + a_row;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int k = k0 + a_k + e;
      ra[e] = (am < M && k < K) ? A[am * lda + k] : 0.0;
    }
    if (!TO_GENES) {        // Bs[n][k] = X[n0 + n][k0 + k]: 8 consecutive k of one cell (zero padded up to ldx)
      const int n = tid >> 1, kh = (tid & 1) * 8;
      const long long i = n0 + n;
      if (i < n_rows) {
        load8(X + i * ldx + k0 + kh, rb);
      } else {
#pragma unroll
        for (int e = 0; e < 8; ++e) rb[e] = TX(0);
      }
    } else {                // Bs[n][k] = X[k0 + k][n0 + n]: 8 consecutive genes of one cell
      const int k = tid >> 4, nq = (tid & 15) * 8;
      const long long i = k0 + k;
      if (i < n_rows && n0 + nq + 8 <= ldx) {
        load8(X + i * ldx + n0 + nq, rb);
      } else {
#pragma unroll
        for (int e = 0; e < 8; ++e) rb[e] = TX(0);
      }
    }
  };
  auto store_tile = [&]() {
#pragma unroll
    for (int e = 0; e < 4; ++e) As[a_row][a_k + e] = ra[e];
    if (!TO_GENES) {
      const int n = tid >> 1, kh = (tid & 1) * 8;
#pragma unroll
      for (int e = 0; e < 8; ++e) Bs[n][kh + e] = (double)rb[e];
    } else {
      const int k = tid >> 4, nq = (tid & 15) * 8;
#pragma unroll
      for (int e = 0; e < 8; ++e) Bs[nq + e][k] = (double)rb[e];
    }
  };

  double acc[2][4][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.0;

  load_tile(0);
  for (int k0 = 0; k0 < K; k0 += F64_BK) {
    __syncthreads();                  // previous tile's fragment reads are done
    store_tile();
    __syncthreads();
    if (k0 + F64_BK < K) load_tile(k0 + F64_BK);      // next tile's global loads in flight under the MMAs
    double af[2][8], bf[4][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int i = 0; i < 8; ++i) af[mt][i] = As[wm + mt * 16 + g + 8 * (i & 1)][t + 4 * (i >> 1)];
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int i = 0; i < 4; ++i) bf[nt][i] = Bs[wn + nt * 8 + g][t + 4 * i];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) mma_f64_16816(acc[mt][nt], af[mt], bf[nt]);
  }

#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const long long row = m0 + wm + mt * 16 + g + 8 * h;
        const int col = n0 + wn + nt * 8 + 2 * t;
        if (row >= M) continue;
        double* dst = C + row * ldc + col;
        if (col + 1 < n_out) {
          *reinterpret_cast<double2*>(dst) = make_double2(acc[mt][nt][2 * h], acc[mt][nt][2 * h + 1]);
        } else if (col < n_out) {
          dst[0] = acc[mt][nt][2 * h];
        }
      }
}

template <typename TX>
int gemm_f64_launch(const double* A, int lda, int M, const TX* X, int n_rows, int n_cols, int ldx, bool to_genes,
                    double* C, int ldc, int k_chunk, long long c_split_stride, cudaStream_t s) {
  if (M <= 0) return 0;
  const int n_out = to_genes ? n_cols : n_rows;
  const int K = to_genes ? n_rows : n_cols;
  if (k_chunk <= 0) k_chunk = K;
  const int splits = K > 0 ? (K + k_chunk - 1) / k_chunk : 1;
  dim3 grid((n_out + F64_BN - 1) / F64_BN, (M + F64_BM - 1) / F64_BM, splits);
  CNMF_REQUIRE(grid.y <= 65535 && grid.z <= 65535, "fp64 GEMM: too many rows or slices");
  if (to_genes)
    gemm_f64_kernel<true, TX><<<grid, F64_THREADS, 0, s>>>(A, lda, M, K, X, ldx, n_rows, C, ldc, n_out, k_chunk,
                                                           c_split_stride);
  else
    gemm_f64_kernel<false, TX><<<grid, F64_THREADS, 0, s>>>(A, lda, M, K, X, ldx, n_rows, C, ldc, n_out, k_chunk,
                                                            c_split_stride);
  CNMF_CUDA_CHECK(cudaGetLastError());
  return 0;
}

}  // namespace

int launch_gemm_f64(const double* A, int lda, int M, const float* X, int n_rows, int n_cols, int ldx, bool to_genes,
                    double* C, int ldc, cudaStream_t s) {
  return gemm_f64_launch(A, lda, M, X, n_rows, n_cols, ldx, to_genes, C, ldc, 0, 0, s);
}

int launch_gemm_f64(const double* A, int lda, int M, const double* X, int n_rows, int n_cols, int ldx, bool to_genes,
                    double* C, int ldc, cudaStream_t s) {
  return gemm_f64_launch(A, lda, M, X, n_rows, n_cols, ldx, to_genes, C, ldc, 0, 0, s);
}

int launch_gemm_f64_split(const double* A, int lda, int M, const float* X, int n_rows, int n_cols, int ldx,
                          bool to_genes, int k_chunk, double* C, int ldc, long long c_split_stride, cudaStream_t s) {
  CNMF_REQUIRE(k_chunk > 0 && k_chunk % F64_BK == 0, "fp64 GEMM: split-K slices must be whole K tiles");
  return gemm_f64_launch(A, lda, M, X, n_rows, n_cols, ldx, to_genes, C, ldc, k_chunk, c_split_stride, s);
}

int launch_gemm_f64_split(const double* A, int lda, int M, const double* X, int n_rows, int n_cols, int ldx,
                          bool to_genes, int k_chunk, double* C, int ldc, long long c_split_stride, cudaStream_t s) {
  CNMF_REQUIRE(k_chunk > 0 && k_chunk % F64_BK == 0, "fp64 GEMM: split-K slices must be whole K tiles");
  return gemm_f64_launch(A, lda, M, X, n_rows, n_cols, ldx, to_genes, C, ldc, k_chunk, c_split_stride, s);
}

}  // namespace cnmf
