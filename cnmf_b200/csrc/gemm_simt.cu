// Plain fp32 FFMA GEMM with the same contract as gemm_tf32x3 (precision mode "fp32"):
//   C[z] (M x N) = A[:, Kz] (M x Kd, K-major) * B[:, Kz]^T (N x Kd, K-major)
// Used for small problems, for the fp32 precision mode and as the on-device cross-check of the
// tensor-core kernel in tests.  128x128x16 tiles, 256 threads, 8x8 micro-tile per thread.
#include <cuda_runtime.h>

#include "common.cuh"
#include "gemm.h"

namespace cnmf {

namespace {

constexpr int TM = 128, TN = 128, TK = 16;

__global__ void __launch_bounds__(256)
gemm_fp32_simt_kernel(const float* __restrict__ A, const float* __restrict__ B, float* __restrict__ C, int M, int N,
                      int Kd, int lda, int ldb, int ldc, long long c_split_stride, int k_per_split) {
  __shared__ float As[TK][TM + 4];
  __shared__ float Bs[TK][TN + 4];

  const int m0 = blockIdx.y * TM;
  const int n0 = blockIdx.x * TN;
  const int z = blockIdx.z;
  const int k_begin = z * k_per_split;
  const int k_end = min(Kd, k_begin + k_per_split);

  const int tid = threadIdx.x;
  const int tx = tid & 15;    // 16 threads across N
  const int ty = tid >> 4;    // 16 threads across M
  const int lrow = tid >> 2;  // 0..63: row loaded (and +64)
  const int lk = (tid & 3) * 4;

  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  for (int k0 = k_begin; k0 < k_end; k0 += TK) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = lrow + h * 64;
      float4 va = make_float4(0.f, 0.f, 0.f, 0.f), vb = va;
      const int gk = k0 + lk;
      if (m0 + r < M) {
        const float* p = A + static_cast<long long>(m0 + r) * lda + gk;
        if (gk + 3 < k_end) va = *reinterpret_cast<const float4*>(p);
        else {
          if (gk < k_end) va.x = p[0];
          if (gk + 1 < k_end) va.y = p[1];
          if (gk + 2 < k_end) va.z = p[2];
        }
      }
      if (n0 + r < N) {
        const float* p = B + static_cast<long long>(n0 + r) * ldb + gk;
        if (gk + 3 < k_end) vb = *reinterpret_cast<const float4*>(p);
        else {
          if (gk < k_end) vb.x = p[0];
          if (gk + 1 < k_end) vb.y = p[1];
          if (gk + 2 < k_end) vb.z = p[2];
        }
      }
      As[lk + 0][r] = va.x; As[lk + 1][r] = va.y; As[lk + 2][r] = va.z; As[lk + 3][r] = va.w;
      Bs[lk + 0][r] = vb.x; Bs[lk + 1][r] = vb.y; Bs[lk + 2][r] = vb.z; Bs[lk + 3][r] = vb.w;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < TK; ++k) {
      float a[8], b[8];
      const float4 a0 = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[k][ty * 4 + 64]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Bs[k][tx * 4 + 64]);
      a[0] = a0.x; a[1] = a0.y; a[2] = a0.z; a[3] = a0.w; a[4] = a1.x; a[5] = a1.y; a[6] = a1.z; a[7] = a1.w;
      b[0] = b0.x; b[1] = b0.y; b[2] = b0.z; b[3] = b0.w; b[4] = b1.x; b[5] = b1.y; b[6] = b1.z; b[7] = b1.w;
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }

  float* Cz = C + static_cast<long long>(z) * c_split_stride;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int m = m0 + ty * 4 + (i & 3) + (i >> 2) * 64;
    if (m >= M) continue;
#pragma unroll
    for (int jh = 0; jh < 2; ++jh) {
      const int n = n0 + tx * 4 + jh * 64;
      if (n + 3 < ldc && n < round_up(N, 4)) {
        *reinterpret_cast<float4*>(Cz + static_cast<long long>(m) * ldc + n) =
            make_float4(acc[i][jh * 4], acc[i][jh * 4 + 1], acc[i][jh * 4 + 2], acc[i][jh * 4 + 3]);
      }
    }
  }
}

}  // namespace

int gemm_fp32_simt(const GemmArgs& g, cudaStream_t stream) {
  CNMF_REQUIRE(g.M > 0 && g.N > 0 && g.Kd > 0, "gemm: empty problem");
  CNMF_REQUIRE(g.lda % 4 == 0 && g.ldb % 4 == 0 && g.ldc % 4 == 0, "gemm: leading dimensions must be multiples of 4 floats");
  const int splits = gemm_effective_splits(g.Kd, g.splits);
  CNMF_REQUIRE(splits == g.splits_effective, "gemm: splits_effective mismatch");
  const int total_kb = (g.Kd + 31) / 32;
  const int kb_per_split = (total_kb + splits - 1) / splits;
  dim3 grid((g.N + TN - 1) / TN, (g.M + TM - 1) / TM, splits);
  gemm_fp32_simt_kernel<<<grid, 256, 0, stream>>>(g.A_hi, g.B_hi, g.C, g.M, g.N, g.Kd, g.lda, g.ldb, g.ldc,
                                                   g.c_split_stride, kb_per_split * 32);
  CNMF_CUDA_CHECK(cudaGetLastError());
  return 0;
}

}  // namespace cnmf
