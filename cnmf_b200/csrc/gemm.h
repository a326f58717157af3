// Internal GEMM interface: C[z] (M x N) = A[:, Kz] (M x Kd, K-major) * B[:, Kz]^T (N x Kd, K-major).
#pragma once
#include <cuda_runtime.h>

namespace cnmf {

struct GemmArgs {
  const float* A_hi;   // M x Kd, row stride lda   (tf32x3: tf32 "hi" piece; fp32 path: the full matrix)
  const float* A_lo;   // tf32 "lo" piece (unused by the fp32 path)
  const float* B_hi;   // N x Kd, row stride ldb
  const float* B_lo;
  float* C;            // splits_effective x (M x ldc)
  int M, N, Kd;
  int lda, ldb, ldc;
  long long c_split_stride;   // elements between consecutive split-K slices of C
  int splits;                 // requested split-K factor
  int splits_effective;       // gemm_effective_splits(Kd, splits): what the kernel will actually write
  int b_exact;                // tf32x3: B_hi holds B exactly (tf32-representable values); B_lo unused -> 2 passes
  const float* out_col_scale; // optional: C[:, n] *= out_col_scale[n] (length >= ldc, 16-byte aligned, zero padded)
  // f16 = 1 (tensor-core path, b_exact only): A_hi / A_lo / B_hi point to __half arrays (two fp16 pieces of the row-
  // normalised A, the integer matrix B), lda / ldb are in half elements, k-blocks hold 64 elements; f16 MMAs run
  // at twice the tf32 rate and carry the same 11-bit significand per piece
  int f16;
  // f16: the A pieces were divided by a power of two per (row, group of 512 reduction elements); the consumers
  // multiply each finished MMA chain (128 elements, never straddling a group) by a_tile_scale[m * a_tiles + group]
  const float* a_tile_scale;
  int a_tiles;                // groups per row = ceil(Kd / 512)
  // columns of C per output tile: 0 = the launcher's choice by shape; 128, or with b_exact 168 / 192, forces that width
  // (tests and micro-benchmarks: every element is formed by the same chains in the same order whatever the width)
  int tile_n;
};

// number of non-empty split-K slices for a reduction length Kd (k-blocks of 32 fp32 / 64 fp16 elements = 128 B)
int gemm_effective_splits(int Kd, int splits, int f16 = 0);

// split-K factor used by the solver: a function of the reduction length only (slices of 64 k-blocks, <= 16), so that a
// restart's result does not depend on the batch it is solved in
int gemm_fixed_splits(int Kd, int f16 = 0);

// wgmma / TMA path (gemm_tf32x3.cu), 128- or 192-row and 128- to 192-column output tiles
int gemm_tf32x3(const GemmArgs& g, cudaStream_t stream);

// plain fp32 FFMA path (gemm_simt.cu): A = A_hi, B = B_hi exactly; same split-K contract
int gemm_fp32_simt(const GemmArgs& g, cudaStream_t stream);

}  // namespace cnmf
