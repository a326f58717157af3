// Split-operand tensor-core GEMM for sm_90a (wgmma + TMA + mbarrier), hand-written PTX.
//
//   C[z] (M x N, row-major, ldc) = A[:, Kz] * B[:, Kz]^T          z = split-K slice
//
// A (M x Kd) and B (N x Kd) are both K-major (row-major with the reduction index contiguous),
// each given as two tf32-representable pieces  A = A_hi + A_lo,  B = B_hi + B_lo  and the
// product is accumulated in fp32 as  A_hi*B_hi + A_lo*B_hi + A_hi*B_lo
// (the dropped A_lo*B_lo term is <= 2^-22 relative): fp32-class accuracy from tf32 MMAs.
// With an exact B (integer counts) the A_hi*B_lo term vanishes (2 passes), and with f16 = 1 the two A pieces
// are fp16 (row-normalised per 512-element group) against an fp16 B: the same 2 passes at twice the tf32 rate.
//
// This is the shape of both big products of an NMF multiplicative-update / coordinate-descent
// iteration once the restarts are batched (SURVEY.md section 8a rows A2/A3):
//   M = sum of K over live restarts (rows of H_batch or W^T_batch),  N = cells or genes.
//   X H^T   (sklearn _nmf.py:538, :380)  ->  A = H_batch (SK x G),   B = X   (cells x G)
//   W^T X   (sklearn _nmf.py:634, :380)  ->  A = W^T_batch (SK x N), B = X^T (G x cells), split-K
//
// Structure (one CTA per SM, persistent over a static tile schedule, 384 threads = 3 warpgroups):
//   warpgroup 0     TMA producer (one thread): cp.async.bulk.tensor 2D, 128B-swizzled tiles, mbarrier full/empty ring
//   warpgroups 1-2  consumers: rows [0, 64) / [64, 128) of the 128 x 128 tile, wgmma.mma_async m64n128 from shared
//                   memory descriptors, fp32 fragment in registers, float2 stores
//
// Accumulation accuracy.  The tensor core does not round its running sum to nearest: a long chain of MMAs on
// non-negative data is biased low by about 3e-8 relative per MMA (2.3e-5 at K = 2048), far outside the 1e-4 parity
// budget of an NMF run.  So the wgmma accumulator only ever holds SHORT chains (`chain_kb` k-blocks, at most 16 MMAs:
// 1 k-block of 12 MMAs in the general 3-pass form, 2 k-blocks of 8 MMAs in the exact-B 2-pass forms): every chain
// starts from zero (scale-d = 0) and is then added into a second set of round-to-nearest fp32 register accumulators.
// Result: ~4e-7 relative, the same class as an FFMA fp32 GEMM.
//
// FUSE (gemm_fused_w_kernel): NUM = F_other * X^T with the multiplicative update of the row factor applied to the tile
// before it leaves the SM (struct FuseW in gemm.h): the consumers pass their sums through shared memory into row layout
// and run fused_w_epilogue instead of storing the product.
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <algorithm>
#include <cstdlib>
#include <map>
#include <mutex>
#include <tuple>

#include "common.cuh"
#include "gemm.h"

namespace cnmf {

namespace {

constexpr int BM = 128;          // rows of A per tile: two consumer warpgroups of 64
constexpr int BN = 128;          // rows of B per tile (wgmma N)
constexpr int BK = 32;           // fp32 elements per k-block = 128 B = one swizzle row
constexpr int NUM_THREADS = 384;
constexpr long long WAIT_TIMEOUT_CYCLES = 4000000000LL;   // ~2 s: a dead pipeline traps instead of hanging

// BEXACT: the B operand is exactly representable in tf32 / fp16 (e.g. integer counts), so it needs no "lo" piece:
// 2 MMAs per k-step instead of 3, 48 KB stages (4 of them) instead of 64 KB (3).
template <int STAGES, bool BEXACT, int EPI_BYTES = 0>
struct SmemLayout {
  static constexpr int A_BYTES = BM * BK * 4;              // 16 KB
  static constexpr int B_BYTES = BN * BK * 4;              // 16 KB
  static constexpr int STAGE_BYTES = 2 * A_BYTES + (BEXACT ? 1 : 2) * B_BYTES;
  static constexpr int BAR_OFFSET = STAGES * STAGE_BYTES;  // full[STAGES], empty[STAGES]
  static constexpr int EPI_OFFSET = BAR_OFFSET + 2 * STAGES * 8;
  static constexpr int TOTAL = EPI_OFFSET + EPI_BYTES;
  static constexpr int DYN_BYTES = TOTAL + 1024;           // slack for manual 1024 B alignment
  static_assert(DYN_BYTES <= 227 * 1024, "pipeline stages do not fit the shared memory of an SM");
};

// ------------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// No printf on timeout: any call in the kernel makes ptxas serialise the wgmma pipeline.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > WAIT_TIMEOUT_CYCLES) __trap();
  }
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}

// K-major, 128B-swizzled operand tile: rows of 128 B, 8-row groups 1024 B apart (wgmma matrix descriptor:
// start address >> 4 in bits [0,14), leading offset (unused for swizzled K-major) [16,30), stride offset [32,46),
// swizzle mode in bits [62,64): 1 = 128B).  Tiles are 1024 B aligned, so the base offset field stays 0.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D (64 x 128 fp32, warpgroup fragment) (+)= A (64 x k, smem) * B (128 x k, smem)^T, both K-major; acc = 0: D = A * B^T
template <bool F16>
__device__ __forceinline__ void wgmma_m64n128(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t acc) {
  if constexpr (F16) {
    asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63 "
      "}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(acc));
  } else {
    asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63 "
      "}, %64, %65, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(acc));
  }
}

// ------------------------------------------------------------------ fused W-half epilogue
__device__ __forceinline__ void named_bar(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid) {
  const int sz = valid ? 16 : 0;                       // src-size 0: the 16 bytes are zero-filled
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// shared memory of the fused epilogue (after the pipeline stages and barriers): the 128 x 128 product tile in row layout
// (rows of 136 floats; the wgmma fragments are written into it, then every thread reads its row half), reused as the
// staging area of 128 rows x 36 floats per column half; per consumer thread its row of the other factor's Gram
// (16 floats) and of the new Gram (16 doubles); the group maxima of the two column halves
constexpr int FUSE_XROW = 136;                                       // floats per product row (128 + pad)
constexpr int FUSE_SROW = 36;                                        // floats per staging row (32 items + pad: conflict-free)
constexpr int FUSE_STAGING_BYTES = 128 * FUSE_XROW * 4;              // 69 632 (>= 2 * 128 * FUSE_SROW * 4)
constexpr int FUSE_G_BYTES = 16 * 256 * 4;                           // 16 384
constexpr int FUSE_GD_BYTES = 16 * 256 * 8;                          // 32 768
constexpr int FUSE_MAX_BYTES = 256 * 4;
constexpr int FUSE_EPI_BYTES = FUSE_STAGING_BYTES + FUSE_G_BYTES + FUSE_GD_BYTES + FUSE_MAX_BYTES;

// The multiplicative update of the row factor, applied to the product tile while it is still in registers (struct
// FuseW in gemm.h).  Thread = packed row (o + c) of a restart x 64 items, one column half of the tile's 128-item scale
// group; acc[] holds the numerators on entry and the new factor values on exit.  The 128 threads that share a column half exchange rows
// through a shared-memory staging area: per 32-item chunk every thread publishes the OLD values of its row (cp.async
// straight from global memory), reads the K rows of its restart (den = sum_i Gram[c, i] F[o + i, item]), publishes the
// NEW values, accumulates its row of the restart's K x K Gram of the new values (fp32 over 16 items, fp64 beyond: the
// summation granularity of the stand-alone update kernel) and the warp stores its 32 rows of the chunk coalesced.
// Restarts never straddle a 128-row tile (the engine packs them that way), so every row a thread needs is in the
// staging area.  All per-thread state that is indexed by the component lives in shared memory, the component loops are
// rolled (small code, no local memory: with ~200 KB of shared memory per CTA the L1 is too small to hold spills).
// Afterwards the two halves of a row agree on the group maximum and each emits the two fp16 operand pieces of its 64
// values with the power-of-two scale of the group: the same bits emit_f16_kernel would produce from F_out.
template <int HALF>
__device__ __forceinline__ void fused_w_epilogue(float (&acc)[HALF], const FuseW& fz, int M, int mt, int nt, int n_tiles,
                                                 int q, int half, int lane, const float* __restrict__ out_scale,
                                                 uint8_t* epi) {
  static_assert(HALF == 64, "two threads (column halves) own one 128-item scale group");
  constexpr float EPS32 = 1.1920928955078125e-07f;     // np.finfo(np.float32).eps, sklearn _nmf.py:32
  constexpr float FMIN = 1.17549435e-38f;
  constexpr int SR = FUSE_SROW;
  const int r = q * 32 + lane;                          // row inside the 128-row tile
  const int tid = half * 128 + r;                       // consumer-thread index 0..255
  const int grow = mt * BM + r;
  const int col0 = nt * 128 + half * HALF;              // first item of this thread's half (tile width 128)
  float* S = reinterpret_cast<float*>(epi) + half * (128 * SR);     // staging of this column half
  float* Sr = S + r * SR;
  float* gs = reinterpret_cast<float*>(epi + FUSE_STAGING_BYTES) + tid;                       // gs[i * 256]
  double* gd = reinterpret_cast<double*>(epi + FUSE_STAGING_BYTES + FUSE_G_BYTES) + tid;      // gd[i * 256]
  const int bar_id = 1 + half;
  const int ld = fz.ld;

  int slot = -1;
  if (grow < M) slot = __ldg(fz.row_slot + grow);
  int K = 0, o = grow, rid = 0;
  bool upd = false, cpy = false;
  if (slot >= 0) {
    rid = __ldg(fz.rid + slot);
    K = __ldg(fz.k + slot);
    o = __ldg(fz.off + slot);
    if (__ldg(fz.done + rid)) cpy = true; else upd = true;
  }
  const int c = grow - o;
  const int lr0 = o - mt * BM;                          // tile-local row of the restart's first component
  const int Kl = upd ? K : 0;
  const bool want_gram = fz.gram_part != nullptr;
  const bool row_ok = grow < M;
  const float* pin = fz.F_in + static_cast<long long>(row_ok ? grow : 0) * ld + col0;
  const uint32_t sr_addr = smem_u32(Sr);

  // old values of the first chunk on their way while the per-thread state is set up
#pragma unroll
  for (int t = 0; t < 8; ++t) cp_async16(sr_addr + 16 * t, pin + 4 * t, row_ok && col0 + 4 * t + 3 < ld);
  for (int i = 0; i < 16; ++i) {
    gs[i * 256] = (i < Kl) ? static_cast<float>(fz.gram_in[static_cast<long long>(rid) * (KMAX * KMAX) + c * KMAX + i]) : 0.f;
    gd[i * 256] = 0.0;
  }
  if (out_scale) {                                      // per-item scale of the product (exact-count datasets)
#pragma unroll
    for (int j = 0; j < HALF; j += 4) {
      if (col0 + j + 3 < ld) {
        const float4 sc = *reinterpret_cast<const float4*>(out_scale + col0 + j);
        acc[j] *= sc.x; acc[j + 1] *= sc.y; acc[j + 2] *= sc.z; acc[j + 3] *= sc.w;
      }
    }
  }
  float* pout = fz.F_out;
  const int sub_r = lane >> 3, sub_c = (lane & 7) * 4;  // coalesced store: 4 rows x 128 B per instruction

#pragma unroll
  for (int ch = 0; ch < HALF / 32; ++ch) {              // 32 items per chunk
    cp_async_wait_all();
    named_bar(bar_id, 128);                             // old rows of the chunk are published
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {                    // 16 items at a time (register budget)
      float2 den[8];
#pragma unroll
      for (int t = 0; t < 8; ++t) den[t] = make_float2(0.f, 0.f);
#pragma unroll 2
      for (int i = 0; i < Kl; ++i) {                    // summed in component order, like the reference's W @ HHt row
        const float2 gi = bcast2(gs[i * 256]);
        const float4* sp = reinterpret_cast<const float4*>(S + (lr0 + i) * SR + hh * 16);
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const float4 w = sp[t];
          den[2 * t] = fma2(gi, make_float2(w.x, w.y), den[2 * t]);
          den[2 * t + 1] = fma2(gi, make_float2(w.z, w.w), den[2 * t + 1]);
        }
      }
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const float4 own = *reinterpret_cast<const float4*>(Sr + hh * 16 + 4 * t);
        const int j = ch * 32 + hh * 16 + 4 * t;
        const float2 own0 = make_float2(own.x, own.y), own1 = make_float2(own.z, own.w);
        const float2 num0 = make_float2(acc[j], acc[j + 1]), num1 = make_float2(acc[j + 2], acc[j + 3]);
        // regularisation terms unconditionally (adding 0 is exact); zero denominators -> eps (sklearn _nmf.py:615)
        float2 d0 = fma2(bcast2(fz.l2), own0, add2(den[2 * t], bcast2(fz.l1)));
        float2 d1 = fma2(bcast2(fz.l2), own1, add2(den[2 * t + 1], bcast2(fz.l1)));
        d0.x = (d0.x < FMIN) ? EPS32 : d0.x; d0.y = (d0.y < FMIN) ? EPS32 : d0.y;
        d1.x = (d1.x < FMIN) ? EPS32 : d1.x; d1.y = (d1.y < FMIN) ? EPS32 : d1.y;
        float2 o0 = mul2(own0, div_nr2(num0, d0));
        float2 o1 = mul2(own1, div_nr2(num1, d1));
        if (!upd) {                                     // converged restart: carried over unchanged; padding row: zero
          o0 = cpy ? own0 : make_float2(0.f, 0.f);
          o1 = cpy ? own1 : make_float2(0.f, 0.f);
        }
        acc[j] = o0.x; acc[j + 1] = o0.y; acc[j + 2] = o1.x; acc[j + 3] = o1.y;
      }
    }
    named_bar(bar_id, 128);                             // everybody has read the old rows
#pragma unroll
    for (int t = 0; t < 8; ++t)
      *reinterpret_cast<float4*>(Sr + 4 * t) = make_float4(acc[ch * 32 + 4 * t], acc[ch * 32 + 4 * t + 1],
                                                           acc[ch * 32 + 4 * t + 2], acc[ch * 32 + 4 * t + 3]);
    named_bar(bar_id, 128);                             // new rows of the chunk are published
    if (want_gram) {
#pragma unroll 2
      for (int i = 0; i < Kl; ++i) {
        const float4* sp = reinterpret_cast<const float4*>(S + (lr0 + i) * SR);
        float2 sa = make_float2(0.f, 0.f), sb = make_float2(0.f, 0.f);   // two 16-item partial sums
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const float4 w = sp[t], w2 = sp[t + 4];
          const int j = ch * 32 + 4 * t;
          sa = fma2(make_float2(acc[j], acc[j + 1]), make_float2(w.x, w.y), sa);
          sa = fma2(make_float2(acc[j + 2], acc[j + 3]), make_float2(w.z, w.w), sa);
          sb = fma2(make_float2(acc[j + 16], acc[j + 17]), make_float2(w2.x, w2.y), sb);
          sb = fma2(make_float2(acc[j + 18], acc[j + 19]), make_float2(w2.z, w2.w), sb);
        }
        gd[i * 256] += static_cast<double>(sa.x + sa.y) + static_cast<double>(sb.x + sb.y);
      }
    }
    {                                                   // this warp's 32 rows x 32 items, 4 rows x 128 B per instruction
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int rr = q * 32 + sub_r + 4 * j;
        const float4 v = *reinterpret_cast<const float4*>(S + rr * SR + sub_c);
        const int grow2 = mt * BM + rr, gcol = col0 + ch * 32 + sub_c;
        if (grow2 < M && gcol + 3 < ld) *reinterpret_cast<float4*>(pout + static_cast<long long>(grow2) * ld + gcol) = v;
      }
    }
    named_bar(bar_id, 128);                             // staging free for the next chunk
    if (ch < HALF / 32 - 1) {
#pragma unroll
      for (int t = 0; t < 8; ++t) {
        const int cc = (ch + 1) * 32 + 4 * t;
        cp_async16(sr_addr + 16 * t, pin + cc, row_ok && col0 + cc + 3 < ld);
      }
    }
  }

  if (want_gram) {                                      // the two column halves of a row meet in shared memory
    named_bar(3, 256);
    if (half == 0 && upd) {
      const int KP = (K + 3) & ~3;                      // layout finalize_kernel reads: [c * KP + i]
      double* dst = fz.gram_part + (static_cast<long long>(rid) * n_tiles + nt) * 256 + c * KP;
      for (int i = 0; i < KP; ++i) dst[i] = (i < K) ? gd[i * 256] + gd[i * 256 + 128] : 0.0;
    }
    named_bar(3, 256);
  }

  // ---- fp16 operand pieces of the new values, group scale = power of two from the group maximum
  float m = 0.f;
  if (fz.piece_scale) {
#pragma unroll
    for (int j = 0; j < HALF; j += 4) {
      float4 ps = make_float4(1.f, 1.f, 1.f, 1.f);
      if (col0 + j + 3 < ld) ps = *reinterpret_cast<const float4*>(fz.piece_scale + col0 + j);
      acc[j] *= ps.x; acc[j + 1] *= ps.y; acc[j + 2] *= ps.z; acc[j + 3] *= ps.w;
    }
  }
#pragma unroll
  for (int j = 0; j < HALF; ++j) m = fmaxf(m, acc[j]);
  float* gmax = reinterpret_cast<float*>(epi + FUSE_STAGING_BYTES + FUSE_G_BYTES + FUSE_GD_BYTES);
  gmax[tid] = m;
  named_bar(3, 256);
  m = fmaxf(m, gmax[tid ^ 128]);                        // the other column half of the row
  const float sc = f16_group_scale(m);
  const float inv = 1.f / sc;                           // power of two: exact
  if (half == 0 && row_ok && col0 < ld) fz.tile_scale[static_cast<long long>(grow) * fz.n_groups + (col0 >> 7)] = sc;
  __half* ph = static_cast<__half*>(fz.P_hi);
  __half* pm = static_cast<__half*>(fz.P_mid);
  uint32_t* Su = reinterpret_cast<uint32_t*>(Sr);
  const int sub_r8 = lane >> 2, sub_q = lane & 3;       // 8 rows x 64 B per instruction
#pragma unroll
  for (int cc = 0; cc < HALF / 32; ++cc) {              // 32 items = 64 B of halves per row and piece
#pragma unroll
    for (int pc = 0; pc < 2; ++pc) {
      __syncwarp();
#pragma unroll
      for (int e = 0; e < 16; e += 4) {
        uint32_t u[4];
#pragma unroll
        for (int k2 = 0; k2 < 4; ++k2) {
          const float x0 = acc[cc * 32 + 2 * (e + k2)] * inv, x1 = acc[cc * 32 + 2 * (e + k2) + 1] * inv;
          const __half2 h = __floats2half2_rn(x0, x1);
          if (pc == 0) {
            u[k2] = *reinterpret_cast<const uint32_t*>(&h);
          } else {
            const float2 hf = __half22float2(h);
            const __half2 md = __floats2half2_rn(x0 - hf.x, x1 - hf.y);
            u[k2] = *reinterpret_cast<const uint32_t*>(&md);
          }
        }
        *reinterpret_cast<uint4*>(Su + e) = make_uint4(u[0], u[1], u[2], u[3]);
      }
      __syncwarp();
      __half* dstp = pc == 0 ? ph : pm;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int rr = q * 32 + sub_r8 + 8 * j;
        const uint4 v = *reinterpret_cast<const uint4*>(reinterpret_cast<const uint32_t*>(S + rr * SR) + sub_q * 4);
        const int grow2 = mt * BM + rr, gcol = col0 + cc * 32 + sub_q * 8;
        if (grow2 < M && gcol + 7 < ld) *reinterpret_cast<uint4*>(dstp + static_cast<long long>(grow2) * ld + gcol) = v;
      }
    }
  }
  __syncwarp();
}

// ------------------------------------------------------------------ the kernel
// F16 (with BEXACT): operands are fp16 (two pieces of A, one exact B); a k-block is still 128 B per row = 64 elements,
// a k-step still 32 B = 16 elements (wgmma K of f16), so the smem / TMA / descriptor byte geometry is unchanged.
//
// Fragment of consumer thread (warp w of its warpgroup, lane l): d[4j + e] is row 16w + l/4 (+8 for e >= 2),
// column 8j + 2(l%4) + (e & 1) of the warpgroup's 64 x 128 block.
template <int STAGES, bool BEXACT, bool F16, bool FUSE>
__device__ __forceinline__ void
gemm_body(const CUtensorMap& tmA_hi, const CUtensorMap& tmA_lo, const CUtensorMap& tmB_hi, const CUtensorMap& tmB_lo,
          float* __restrict__ C, int M, int ldc, long long c_split_stride,
          int m_tiles, int n_tiles, int splits, int total_kb, int kb_per_split, int chain_kb,
          const float* __restrict__ out_scale, const float* __restrict__ a_tile_scale, int a_tiles, int a_gshift,
          const FuseW* __restrict__ fz) {
  static_assert(!F16 || BEXACT, "the fp16 path exists for exact integer B operands only");
  static_assert(!FUSE || (F16 && STAGES == 2), "the fused W-half epilogue is built for the 2-stage f16 kernel");
  constexpr int BKE = F16 ? 2 * BK : BK;                        // elements per k-block
  constexpr int KSTEP_BYTES = 32;                               // wgmma K: 8 tf32 or 16 fp16 elements
  using L = SmemLayout<STAGES, BEXACT, FUSE ? FUSE_EPI_BYTES : 0>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;     // SWIZZLE_128B needs 1024 B alignment
  uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));

  const uint32_t bar_base = smem_base + L::BAR_OFFSET;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };

  const int wg = threadIdx.x >> 7;
  const int warp = (threadIdx.x >> 5) & 3;                      // warp inside its warpgroup
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 8);                               // one arrival per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int items = m_tiles * n_tiles * splits;

  if constexpr (FUSE) {     // the epilogue's state needs more than 168 registers: move them from the producer warpgroup
    if (wg == 0) asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    else asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
  }
  if (wg == 0) {
    // ===================== TMA producer =====================
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      constexpr uint32_t stage_tx = static_cast<uint32_t>(L::STAGE_BYTES);
      for (int w = blockIdx.x; w < items; w += gridDim.x) {
        const int mt = w % m_tiles;
        const int nt = (w / m_tiles) % n_tiles;
        const int z = w / (m_tiles * n_tiles);
        const int kb0 = z * kb_per_split;
        const int kb1 = min(total_kb, kb0 + kb_per_split);
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(empty_bar(stage), phase ^ 1u);
          const uint32_t st = smem_base + stage * L::STAGE_BYTES;
          mbar_arrive_expect_tx(full_bar(stage), stage_tx);
          tma_load_2d(st, &tmA_hi, full_bar(stage), kb * BKE, mt * BM);
          tma_load_2d(st + L::A_BYTES, &tmA_lo, full_bar(stage), kb * BKE, mt * BM);
          tma_load_2d(st + 2 * L::A_BYTES, &tmB_hi, full_bar(stage), kb * BKE, nt * BN);
          if constexpr (!BEXACT) tma_load_2d(st + 2 * L::A_BYTES + L::B_BYTES, &tmB_lo, full_bar(stage), kb * BKE, nt * BN);
          if (++stage == STAGES) { stage = 0; phase ^= 1u; }
        }
      }
    }
  } else {
    // ===================== consumers: MMA chains + drain + epilogue =====================
    const int cw = wg - 1;                                      // rows [64 cw, 64 cw + 64) of the tile
    const uint32_t a_off = static_cast<uint32_t>(cw * 64 * 128);
    int stage = 0;
    uint32_t phase = 0;
    for (int w = blockIdx.x; w < items; w += gridDim.x) {
      const int mt = w % m_tiles;
      const int nt = (w / m_tiles) % n_tiles;
      const int z = w / (m_tiles * n_tiles);
      const int kb0 = z * kb_per_split;
      const int kb1 = min(total_kb, kb0 + kb_per_split);
      const int row0 = mt * BM + cw * 64 + warp * 16 + (lane >> 2);   // and row0 + 8
      float acc[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = 0.f;
      // f16: power-of-two scale of this thread's two A rows for the scale group (2^a_gshift k-blocks) of a chain
      const float* sc_row0 = (F16 && a_tile_scale && row0 < M) ? a_tile_scale + static_cast<long long>(row0) * a_tiles : nullptr;
      const float* sc_row1 = (F16 && a_tile_scale && row0 + 8 < M) ? a_tile_scale + static_cast<long long>(row0 + 8) * a_tiles : nullptr;
      for (int c0 = kb0; c0 < kb1; c0 += chain_kb) {            // one short accumulation chain
        const int c1 = min(kb1, c0 + chain_kb);
        float d[64];
        int prev = -1;
        for (int kb = c0; kb < c1; ++kb) {
          mbar_wait(full_bar(stage), phase);
          const uint32_t st = smem_base + stage * L::STAGE_BYTES;
          const uint64_t a_hi = make_smem_desc(st + a_off);
          const uint64_t a_lo = make_smem_desc(st + L::A_BYTES + a_off);
          const uint64_t b_hi = make_smem_desc(st + 2 * L::A_BYTES);
          const uint64_t b_lo = make_smem_desc(st + 2 * L::A_BYTES + L::B_BYTES);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < BK * 4 / KSTEP_BYTES; ++k) {
            const uint64_t koff = static_cast<uint64_t>((k * KSTEP_BYTES) >> 4);   // +32 B per k-step inside the swizzle row
            const uint32_t acc0 = (kb > c0 || k > 0) ? 1u : 0u;
            wgmma_m64n128<F16>(d, a_lo + koff, b_hi + koff, acc0);     // small terms first
            if constexpr (!BEXACT) wgmma_m64n128<F16>(d, a_hi + koff, b_lo + koff, 1u);
            wgmma_m64n128<F16>(d, a_hi + koff, b_hi + koff, 1u);
          }
          wgmma_commit();
          if (prev >= 0) {                                      // the previous k-block's MMAs have read their slot
            wgmma_wait<1>();
            if (lane == 0) mbar_arrive(empty_bar(prev));
          }
          prev = stage;
          if (++stage == STAGES) { stage = 0; phase ^= 1u; }
        }
        wgmma_wait<0>();
        if (lane == 0) mbar_arrive(empty_bar(prev));
        if constexpr (F16) {                                    // exact power-of-two scaling, one rounding
          const float s0 = sc_row0 ? sc_row0[c0 >> a_gshift] : 1.f;
          const float s1 = sc_row1 ? sc_row1[c0 >> a_gshift] : 1.f;
#pragma unroll
          for (int i = 0; i < 64; i += 4) {
            acc[i] = fmaf(d[i], s0, acc[i]);
            acc[i + 1] = fmaf(d[i + 1], s0, acc[i + 1]);
            acc[i + 2] = fmaf(d[i + 2], s1, acc[i + 2]);
            acc[i + 3] = fmaf(d[i + 3], s1, acc[i + 3]);
          }
        } else {
#pragma unroll
          for (int i = 0; i < 64; ++i) acc[i] += d[i];          // round-to-nearest fp32
        }
      }
      if constexpr (FUSE) {
        // fragments -> row layout: consumer thread ct owns tile row ct % 128, items [64 (ct / 128), +64)
        const int ct = static_cast<int>(threadIdx.x) - 128;
        float* X = reinterpret_cast<float*>(smem_gen + L::EPI_OFFSET);
        named_bar(4, 256);                                      // the previous tile's epilogue is done with X
        const int lr = cw * 64 + warp * 16 + (lane >> 2);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int lc = 8 * j + 2 * (lane & 3);
          *reinterpret_cast<float2*>(X + lr * FUSE_XROW + lc) = make_float2(acc[4 * j], acc[4 * j + 1]);
          *reinterpret_cast<float2*>(X + (lr + 8) * FUSE_XROW + lc) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
        }
        named_bar(4, 256);
        float rowv[64];
        const float4* src = reinterpret_cast<const float4*>(X + (ct & 127) * FUSE_XROW + (ct >> 7) * 64);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const float4 v = src[j];
          rowv[4 * j] = v.x; rowv[4 * j + 1] = v.y; rowv[4 * j + 2] = v.z; rowv[4 * j + 3] = v.w;
        }
        named_bar(4, 256);                                      // X is reused as the epilogue's staging area
        fused_w_epilogue<64>(rowv, *fz, M, mt, nt, n_tiles, (ct & 127) >> 5, ct >> 7, lane, out_scale,
                             smem_gen + L::EPI_OFFSET);
        continue;
      }
      // Epilogue: a quad of lanes writes 32 contiguous bytes of a row per instruction (whole sectors)
      float* cbase = C + static_cast<long long>(z) * c_split_stride;
      const int colq = nt * BN + 2 * (lane & 3);
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int col = colq + 8 * j;
        if (col >= ldc) continue;                               // ldc % 4 == 0 and col even: col + 1 < ldc too
        float2 sc = make_float2(1.f, 1.f);
        if (out_scale) sc = *reinterpret_cast<const float2*>(out_scale + col);   // length >= ldc, zero padded
        if (row0 < M)
          *reinterpret_cast<float2*>(cbase + static_cast<long long>(row0) * ldc + col) =
              make_float2(acc[4 * j] * sc.x, acc[4 * j + 1] * sc.y);
        if (row0 + 8 < M)
          *reinterpret_cast<float2*>(cbase + static_cast<long long>(row0 + 8) * ldc + col) =
              make_float2(acc[4 * j + 2] * sc.x, acc[4 * j + 3] * sc.y);
      }
    }
  }
}

template <int STAGES, bool BEXACT, bool F16>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_tf32x3_kernel(const __grid_constant__ CUtensorMap tmA_hi, const __grid_constant__ CUtensorMap tmA_lo,
                   const __grid_constant__ CUtensorMap tmB_hi, const __grid_constant__ CUtensorMap tmB_lo,
                   float* __restrict__ C, int M, int ldc, long long c_split_stride,
                   int m_tiles, int n_tiles, int splits, int total_kb, int kb_per_split, int chain_kb,
                   const float* __restrict__ out_scale, const float* __restrict__ a_tile_scale, int a_tiles, int a_gshift) {
  gemm_body<STAGES, BEXACT, F16, false>(tmA_hi, tmA_lo, tmB_hi, tmB_lo, C, M, ldc, c_split_stride, m_tiles, n_tiles, splits,
                                        total_kb, kb_per_split, chain_kb, out_scale, a_tile_scale, a_tiles, a_gshift,
                                        nullptr);
}

// NUM = F_other * X^T with the multiplicative update of the row factor in the epilogue (f16, 128-wide tiles, no split-K)
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_fused_w_kernel(const __grid_constant__ CUtensorMap tmA_hi, const __grid_constant__ CUtensorMap tmA_lo,
                    const __grid_constant__ CUtensorMap tmB_hi, int M, int m_tiles, int n_tiles, int total_kb,
                    const float* __restrict__ out_scale, const float* __restrict__ a_tile_scale, int a_tiles, int a_gshift,
                    const __grid_constant__ FuseW fz) {
  gemm_body<2, true, true, true>(tmA_hi, tmA_lo, tmB_hi, tmB_hi, nullptr, M, 0, 0, m_tiles, n_tiles, 1, total_kb,
                                 total_kb + (total_kb & 1), 2, out_scale, a_tile_scale, a_tiles, a_gshift, &fz);
}

// ------------------------------------------------------------------ host side
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  });
  return fn;
}

// 2D fp32 / fp16 tensor (rows x cols, row stride ld elements), box = 128 B x box_rows rows, 128B swizzle, zero OOB fill.
// Encoded maps are cached by (pointer, shape, box): the solver relaunches the same few operand views a thousand
// times per solve, and the driver call costs more than the launch itself.
struct MapKey {
  const void* ptr; int rows, cols, ld, box_rows, f16;
  bool operator<(const MapKey& o) const {
    return std::tie(ptr, rows, cols, ld, box_rows, f16) < std::tie(o.ptr, o.rows, o.cols, o.ld, o.box_rows, o.f16);
  }
};

int make_map(CUtensorMap* map, const float* ptr, int rows, int cols, int ld, int box_rows, bool f16 = false) {
  static std::mutex mu;
  static std::map<MapKey, CUtensorMap> cache;
  const MapKey key{ptr, rows, cols, ld, box_rows, f16 ? 1 : 0};
  {
    std::lock_guard<std::mutex> lock(mu);
    auto it = cache.find(key);
    if (it != cache.end()) { *map = it->second; return 0; }
  }
  PFN_encodeTiled enc = get_encode_fn();
  if (!enc) { set_last_error("cuTensorMapEncodeTiled entry point not available"); return -2; }
  const int esize = f16 ? 2 : 4;                      // a box row is always 128 B: 32 fp32 or 64 fp16 elements
  cuuint64_t dims[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
  cuuint64_t strides[1] = {static_cast<cuuint64_t>(ld) * esize};
  cuuint32_t box[2] = {static_cast<cuuint32_t>(128 / esize), static_cast<cuuint32_t>(box_rows)};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled failed with CUresult " + std::to_string(static_cast<int>(r)));
    return -2;
  }
  std::lock_guard<std::mutex> lock(mu);
  if (cache.size() >= 512) cache.clear();             // views are few; a runaway caller just re-encodes
  cache.emplace(key, *map);
  return 0;
}

static int env_int(const char* name, int dflt) {
  const char* e = std::getenv(name);
  return e ? std::atoi(e) : dflt;
}

// k-blocks per accumulation chain: at most 16 MMAs between drains (general: 1 k-block = 12 MMAs,
// exact-B: 2 k-blocks = 16 MMAs)
template <bool BEXACT, bool F16>
static int pick_chain_kb(const GemmArgs& g) {
  int chain_kb = g.chain_kb;
  if (chain_kb <= 0) {
    static const int env_chain = [] { const int v = env_int("CNMF_CHAIN_KB", 0); return v >= 1 ? v : 0; }();   // tuning knob
    chain_kb = env_chain > 0 ? env_chain : (BEXACT ? 2 : 1);
  }
  if (F16) chain_kb = 2;     // scale groups of 512 elements = 8 k-blocks: chains of 2 never straddle one
  return chain_kb;
}

template <int STAGES, bool BEXACT, bool F16>
int launch(const GemmArgs& g, cudaStream_t stream) {
  using L = SmemLayout<STAGES, BEXACT>;
  constexpr int BKE = F16 ? 2 * BK : BK;
  CUtensorMap mAh, mAl, mBh, mBl;
  int rc;
  if ((rc = make_map(&mAh, g.A_hi, g.M, g.Kd, g.lda, BM, F16))) return rc;
  if ((rc = make_map(&mAl, g.A_lo, g.M, g.Kd, g.lda, BM, F16))) return rc;
  if ((rc = make_map(&mBh, g.B_hi, g.N, g.Kd, g.ldb, BN, F16))) return rc;
  if ((rc = make_map(&mBl, BEXACT ? g.B_hi : g.B_lo, g.N, g.Kd, g.ldb, BN, F16))) return rc;
  int dev = 0, sms = 0;
  CNMF_CUDA_CHECK(cudaGetDevice(&dev));
  CNMF_CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const int m_tiles = (g.M + BM - 1) / BM;
  const int n_tiles = (g.N + BN - 1) / BN;
  const int total_kb = (g.Kd + BKE - 1) / BKE;
  int splits = g.splits < 1 ? 1 : g.splits;
  if (splits > total_kb) splits = total_kb;
  int kb_per_split = (total_kb + splits - 1) / splits;
  if (F16 && (kb_per_split & 1)) ++kb_per_split;             // chains (2 k-blocks) must not straddle a 512-element scale group
  splits = (total_kb + kb_per_split - 1) / kb_per_split;      // no empty slices
  if (splits != g.splits_effective) { set_last_error("gemm: splits_effective mismatch (use gemm_effective_splits)"); return -1; }

  auto kern = gemm_tf32x3_kernel<STAGES, BEXACT, F16>;
  static bool attr_set[64] = {};              // per device: a second GPU in the same process needs its own call
  if (dev < 0 || dev >= 64 || !attr_set[dev]) {
    CNMF_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::DYN_BYTES));
    if (dev >= 0 && dev < 64) attr_set[dev] = true;
  }
  const int items = m_tiles * n_tiles * splits;
  const int grid = items < sms ? items : sms;
  const int chain_kb = pick_chain_kb<BEXACT, F16>(g);
  kern<<<grid, NUM_THREADS, L::DYN_BYTES, stream>>>(mAh, mAl, mBh, mBl, g.C, g.M, g.ldc, g.c_split_stride,
                                                    m_tiles, n_tiles, splits, total_kb, kb_per_split, chain_kb,
                                                    g.out_col_scale, g.a_tile_scale, g.a_tiles,
                                                    g.a_group_kb_shift > 0 ? g.a_group_kb_shift : 3);
  CNMF_CUDA_CHECK(cudaGetLastError());
  return 0;
}

// fused W-half launch: 128 x 128 tiles, the whole reduction in one item (no split-K), f16
int launch_fused_w(const GemmArgs& g, cudaStream_t stream) {
  using L = SmemLayout<2, true, FUSE_EPI_BYTES>;     // 2 stages of 48 KB leave room for the epilogue's state
  CUtensorMap mAh, mAl, mBh;
  int rc;
  if ((rc = make_map(&mAh, g.A_hi, g.M, g.Kd, g.lda, BM, true))) return rc;
  if ((rc = make_map(&mAl, g.A_lo, g.M, g.Kd, g.lda, BM, true))) return rc;
  if ((rc = make_map(&mBh, g.B_hi, g.N, g.Kd, g.ldb, BN, true))) return rc;
  int dev = 0, sms = 0;
  CNMF_CUDA_CHECK(cudaGetDevice(&dev));
  CNMF_CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const int m_tiles = (g.M + BM - 1) / BM, n_tiles = (g.N + BN - 1) / BN;
  const int total_kb = (g.Kd + 2 * BK - 1) / (2 * BK);
  static bool attr_set[64] = {};
  if (dev < 0 || dev >= 64 || !attr_set[dev]) {
    CNMF_CUDA_CHECK(cudaFuncSetAttribute(gemm_fused_w_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, L::DYN_BYTES));
    if (dev >= 0 && dev < 64) attr_set[dev] = true;
  }
  const int items = m_tiles * n_tiles;
  const int grid = items < sms ? items : sms;
  gemm_fused_w_kernel<<<grid, NUM_THREADS, L::DYN_BYTES, stream>>>(mAh, mAl, mBh, g.M, m_tiles, n_tiles, total_kb,
                                                                   g.out_col_scale, g.a_tile_scale, g.a_tiles,
                                                                   g.a_group_kb_shift > 0 ? g.a_group_kb_shift : 3, g.fuse);
  CNMF_CUDA_CHECK(cudaGetLastError());
  return 0;
}

}  // namespace

// Split-K factor as a function of the reduction length ONLY: slices of 64 k-blocks (4 096 fp16 / 2 048 fp32
// elements), at most 16 of them.  The partition of a restart's reduction -- and with it every rounding of its
// products -- is then the same whatever else shares the batch and however far the batch has been compacted:
// a (k, seed) restart gives the same spectra alone, in a worker's shard or in the full K-sweep, which is the
// reference's semantics (independent sklearn calls, cnmf.py:735-745).
int gemm_fixed_splits(int Kd, int f16) {
  const int bke = f16 ? 2 * BK : BK;
  const int total_kb = (Kd + bke - 1) / bke;
  const int s = std::max(1, std::min(16, (total_kb + 63) / 64));
  return gemm_effective_splits(Kd, s, f16);
}

int gemm_effective_splits(int Kd, int splits, int f16) {
  const int bke = f16 ? 2 * BK : BK;
  const int total_kb = (Kd + bke - 1) / bke;
  if (splits < 1) splits = 1;
  if (splits > total_kb) splits = total_kb;
  int kb_per_split = (total_kb + splits - 1) / splits;
  if (f16 && (kb_per_split & 1)) ++kb_per_split;   // same rule as the launcher: slices start on even k-blocks
  return (total_kb + kb_per_split - 1) / kb_per_split;
}

int gemm_tf32x3(const GemmArgs& g, cudaStream_t stream) {
  CNMF_REQUIRE(g.M > 0 && g.N > 0 && g.Kd > 0, "gemm: empty problem");
  CNMF_REQUIRE(g.lda % 4 == 0 && g.ldb % 4 == 0 && g.ldc % 4 == 0, "gemm: leading dimensions must be multiples of 4 floats");
  CNMF_REQUIRE((reinterpret_cast<uintptr_t>(g.A_hi) | reinterpret_cast<uintptr_t>(g.A_lo) |
                reinterpret_cast<uintptr_t>(g.B_hi) | reinterpret_cast<uintptr_t>(g.B_lo) |
                reinterpret_cast<uintptr_t>(g.C) | reinterpret_cast<uintptr_t>(g.out_col_scale)) % 16 == 0,
               "gemm: pointers must be 16-byte aligned");
  if (g.f16) {
    CNMF_REQUIRE(g.b_exact, "gemm: the fp16 path needs an exact B operand");
    CNMF_REQUIRE(g.lda % 8 == 0 && g.ldb % 8 == 0, "gemm: fp16 leading dimensions must be multiples of 8 halves");
    CNMF_REQUIRE(!g.a_tile_scale || g.a_tiles * 512 >= g.Kd, "gemm: a_tiles does not cover the reduction length");
    CNMF_REQUIRE(g.chain_kb == 0 || g.chain_kb == 2, "gemm: the fp16 path drains chains of 2 k-blocks");
    if (g.fuse.active) {
      CNMF_REQUIRE(g.fuse.F_in && g.fuse.F_out && g.fuse.F_in != g.fuse.F_out && g.fuse.P_hi && g.fuse.P_mid &&
                       g.fuse.tile_scale && g.fuse.gram_in && g.fuse.row_slot && g.fuse.ld % 32 == 0,
                   "gemm: incomplete fused-update arguments");
      return launch_fused_w(g, stream);
    }
    return launch<4, true, true>(g, stream);
  }
  if (g.b_exact) return launch<4, true, false>(g, stream);
  return launch<3, false, false>(g, stream);
}

}  // namespace cnmf
