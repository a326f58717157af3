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
// Structure (one CTA per SM, persistent over a static tile schedule of 128 x BN tiles, BN = 128, 168 or 192; 384
// threads = 3 warpgroups; the CTAs run in clusters of 2 whose tiles share an m-tile, and each CTA loads half of the
// shared A panel and multicasts it to both):
//   warpgroup 0     TMA producer (one thread): cp.async.bulk.tensor 2D, 128B-swizzled tiles, mbarrier full/empty ring,
//                   a stage refilled only once both CTAs of the pair have released it
//   warpgroups 1-2  consumers: rows [64 (w - 1), 64 w) of the tile, wgmma.mma_async m64nBN from shared memory
//                   descriptors, fp32 fragment in registers, float2 stores.  Named barriers make them take turns in a
//                   ring issuing one k-block of MMAs each (ping-pong), so one warpgroup's chain drain and tile stores
//                   run while the others' MMAs keep the tensor pipe busy.
//   At BN > 128 setmaxnreg moves the producer to 40 registers and the consumers to 232.  The launcher picks BN by
//   shape (pick_tile_n below); measured on one H100 SXM (700 W), DESIGN.md section 4.1.
//
// Accumulation accuracy.  The tensor core does not round its running sum to nearest: a long chain of MMAs on
// non-negative data is biased low by about 3e-8 relative per MMA (2.3e-5 at K = 2048), far outside the 1e-4 parity
// budget of an NMF run.  So the wgmma accumulator only ever holds SHORT chains (`chain_kb` k-blocks, at most 16 MMAs:
// 1 k-block of 12 MMAs in the general 3-pass form, 2 k-blocks of 8 MMAs in the exact-B 2-pass forms): every chain
// starts from zero (scale-d = 0) and is then added into a second set of round-to-nearest fp32 register accumulators.
// Result: ~4e-7 relative, the same class as an FFMA fp32 GEMM.
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <algorithm>
#include <map>
#include <mutex>
#include <tuple>

#include "common.cuh"
#include "gemm.h"

namespace cnmf {

namespace {

// BN (rows of B per tile, the wgmma N) is a template parameter.  BM rows of A per tile: one consumer warpgroup per 64.
constexpr int BM = 128;
constexpr int NUM_THREADS = 128 * (1 + BM / 64);
constexpr int BK = 32;           // fp32 elements per k-block = 128 B = one swizzle row
constexpr long long WAIT_TIMEOUT_CYCLES = 4000000000LL;   // ~2 s: a dead pipeline traps instead of hanging

// BEXACT: the B operand is exactly representable in tf32 / fp16 (e.g. integer counts), so it needs no "lo" piece:
// 2 MMAs per k-step instead of 3.  Stages: 4 of 32 KB + BN * 128 B (48-56 KB) for the exact-B forms, 3 of 64 KB for
// the general form (BN = 128 only).
template <int BN, int STAGES, bool BEXACT>
struct SmemLayout {
  static constexpr int A_BYTES = BM * BK * 4;              // 16 KB
  static constexpr int B_BYTES = BN * BK * 4;              // 16 KB (BN = 128) to 24 KB (BN = 192), a multiple of 1 KB
  static constexpr int STAGE_BYTES = 2 * A_BYTES + (BEXACT ? 1 : 2) * B_BYTES;
  static constexpr int BAR_OFFSET = STAGES * STAGE_BYTES;  // full[STAGES], empty[STAGES], peer_free[STAGES]
  static constexpr int TOTAL = BAR_OFFSET + 3 * STAGES * 8;
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
// No printf on timeout: any call in the kernel makes ptxas serialise the wgmma pipeline.  Only the producer's waits
// trap: a trap in code after setmaxnreg.inc makes ptxas allocate that code at the launch-wide register count (and
// spill).  A stalled consumer still ends in a trap, because the producer waits (with the timeout) for every stage to be
// released before it leaves, and a consumer that stops releasing stages stalls it.
template <bool TRAP>
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (TRAP && clock64() - t0 > WAIT_TIMEOUT_CYCLES) __trap();
  }
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
// The same box written to the same CTA-relative `dst` in every CTA of `mask`, each CTA's copy signalling its own
// mbarrier at the CTA-relative address `bar`.
__device__ __forceinline__ void tma_load_2d_multicast(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1,
                                                      uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "h"(mask)
      : "memory");
}

// Arrive on the mbarrier at the same offset in the CTA of cluster rank `rank`.  Default (CTA-scope) semantics, as for
// the local arrivals: the arrival only signals that this CTA's consumers have finished reading a stage, and what follows
// it is a TMA write, not a generic load.  With .release.cluster (and .acquire.cluster on the wait) ptxas emits
// MEMBAR.ALL.GPU and an L1 invalidate around every k-block of the producer, which made the kernel slower than unpaired.
__device__ __forceinline__ void mbar_arrive_remote(uint32_t bar, uint32_t rank) {
  asm volatile(
      "{\n\t.reg .b32 remote;\n\t"
      "mapa.shared::cluster.u32 remote, %0, %1;\n\t"
      "mbarrier.arrive.shared::cluster.b64 _, [remote];\n\t}"
      ::"r"(bar), "r"(rank)
      : "memory");
}
// All threads of both CTAs: release what this CTA did before, acquire what the peer did before its arrival.  Not
// .aligned: the producer warp's lanes may reach it diverged.
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release;\n\tbarrier.cluster.wait.acquire;" ::: "memory");
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

// Named barriers (id 0 is __syncthreads): bar.sync blocks until `count` threads have reached the barrier, bar.arrive
// counts this warp without waiting.  Here 128 threads sync and the other warpgroup's 128 arrive.
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}
__device__ __forceinline__ void named_bar_arrive(uint32_t id, uint32_t count) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// Hand registers between warpgroups (all threads of the warpgroup, converged): the producer gives up what it never
// uses so that the consumers can hold more than the launch-wide share.
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D (64 x N fp32, warpgroup fragment) (+)= A (64 x k, smem) * B (N x k, smem)^T, both K-major; acc = 0: D = A * B^T.
// One wrapper per N: the fragment's N / 2 registers are the asm outputs %0 .. %(N/2 - 1), then the two descriptors and
// the accumulate flag (at IA, IB, IACC).
#define CNMF_R64                                                                      \
  "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "            \
  "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "  \
  "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "  \
  "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
#define CNMF_R84 CNMF_R64 ", %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, " \
  "%80, %81, %82, %83"
#define CNMF_R96 CNMF_R84 ", %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95"
#define CNMF_D4(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3])
#define CNMF_D8(i) CNMF_D4(i), CNMF_D4(i + 4)
#define CNMF_D64 CNMF_D8(0), CNMF_D8(8), CNMF_D8(16), CNMF_D8(24), CNMF_D8(32), CNMF_D8(40), CNMF_D8(48), CNMF_D8(56)
#define CNMF_D84 CNMF_D64, CNMF_D8(64), CNMF_D8(72), CNMF_D4(80)
#define CNMF_D96 CNMF_D64, CNMF_D8(64), CNMF_D8(72), CNMF_D8(80), CNMF_D8(88)
#define CNMF_WGMMA(N, REGS, IA, IB, IACC, ...)                                                                        \
  template <bool F16>                                                                                                 \
  __device__ __forceinline__ void wgmma_m64n##N(float (&d)[N / 2], uint64_t adesc, uint64_t bdesc, uint32_t acc) {    \
    if constexpr (F16)                                                                                                \
      asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" IACC ", 0;\n\t"                                          \
                   "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32.f16.f16 {" REGS "}, %" IA ", %" IB                 \
                   ", p, 1, 1, 0, 0;\n\t}"                                                                            \
                   : __VA_ARGS__ : "l"(adesc), "l"(bdesc), "r"(acc));                                                 \
    else                                                                                                              \
      asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" IACC ", 0;\n\t"                                          \
                   "wgmma.mma_async.sync.aligned.m64n" #N "k8.f32.tf32.tf32 {" REGS "}, %" IA ", %" IB ", p, 1, 1;\n\t}" \
                   : __VA_ARGS__ : "l"(adesc), "l"(bdesc), "r"(acc));                                                 \
  }
CNMF_WGMMA(128, CNMF_R64, "64", "65", "66", CNMF_D64)
CNMF_WGMMA(168, CNMF_R84, "84", "85", "86", CNMF_D84)
CNMF_WGMMA(192, CNMF_R96, "96", "97", "98", CNMF_D96)

template <int BN, bool F16>
__device__ __forceinline__ void wgmma_tile(float (&d)[BN / 2], uint64_t adesc, uint64_t bdesc, uint32_t acc) {
  if constexpr (BN == 128) wgmma_m64n128<F16>(d, adesc, bdesc, acc);
  else if constexpr (BN == 168) wgmma_m64n168<F16>(d, adesc, bdesc, acc);
  else wgmma_m64n192<F16>(d, adesc, bdesc, acc);
}

// ------------------------------------------------------------------ tile order
// The CTAs run in clusters of 2 (a pair), and a pair's work item is an m-tile and two adjacent n-tiles: the CTA of
// cluster rank r computes n-tile 2 * n-pair + r, and the two share the m-tile's A panel (multicast, see gemm_body).
// Pair item w -> (m-tile, n-pair, split-K slice z).  The slice is outermost.  Inside a slice the items run in groups of
// `group` consecutive m-tiles (n-pairs if group_n), the grouped index fastest, and each group sweeps every tile of the
// other dimension: the group's operand panels stay in the L2 while the other operand streams past them (DESIGN.md
// section 4.1; pick_tile_order chooses the group).  group = m_tiles, group_n = 0 is the plain m-tile-fastest order.
// The producer and the consumers both decode through this function, so they always agree on a CTA's tiles.
struct TileOrder {
  int m_tiles, n_pairs, group, group_n;
};

__host__ __device__ __forceinline__ void decode_item(int w, const TileOrder& o, int& mt, int& np, int& z) {
  const int per_slice = o.m_tiles * o.n_pairs;
  z = w / per_slice;
  int r = w - z * per_slice;
  const int q_tiles = o.group_n ? o.n_pairs : o.m_tiles;      // grouped dimension
  const int p_tiles = o.group_n ? o.m_tiles : o.n_pairs;      // swept dimension
  const int g0 = r / (o.group * p_tiles) * o.group;           // first grouped tile of w's group (earlier groups are full)
  r -= g0 * p_tiles;
  const int gq = q_tiles - g0 < o.group ? q_tiles - g0 : o.group;   // the last group may be partial
  const int p = r / gq, q = g0 + r % gq;
  mt = o.group_n ? p : q;
  np = o.group_n ? q : p;
}

// ------------------------------------------------------------------ the kernel
// F16 (with BEXACT): operands are fp16 (two pieces of A, one exact B); a k-block is still 128 B per row = 64 elements,
// a k-step still 32 B = 16 elements (wgmma K of f16), so the smem / TMA / descriptor byte geometry is unchanged.
//
// Fragment of consumer thread (warp w of its warpgroup, lane l): d[4j + e] is row 16w + l/4 (+8 for e >= 2),
// column 8j + 2(l%4) + (e & 1) of the warpgroup's 64 x BN block.
template <int BN, int STAGES, bool BEXACT, bool F16>
__device__ __forceinline__ void
gemm_body(const CUtensorMap& tmA_hi, const CUtensorMap& tmA_lo, const CUtensorMap& tmB_hi, const CUtensorMap& tmB_lo,
          float* __restrict__ C, int M, int ldc, long long c_split_stride,
          const TileOrder& ord, int n_tiles, int splits, int total_kb, int kb_per_split, int chain_kb,
          const float* __restrict__ out_scale, const float* __restrict__ a_tile_scale, int a_tiles, int a_gshift) {
  static_assert(!F16 || BEXACT, "the fp16 path exists for exact integer B operands only");
  static_assert(BN == 128 || (BEXACT && (BN == 168 || BN == 192)), "wide n-tiles in the exact-B forms only");
  constexpr int NC = BM / 64;                                   // consumer warpgroups
  constexpr int BKE = F16 ? 2 * BK : BK;                        // elements per k-block
  constexpr int KSTEP_BYTES = 32;                               // wgmma K: 8 tf32 or 16 fp16 elements
  using L = SmemLayout<BN, STAGES, BEXACT>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;     // SWIZZLE_128B needs 1024 B alignment

  const uint32_t bar_base = smem_base + L::BAR_OFFSET;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };
  auto peer_free_bar = [&](int s) { return bar_base + 8u * (2 * STAGES + s); };

  const int wg = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 7), 0);   // warp-uniform, as setmaxnreg needs
  const int warp = (threadIdx.x >> 5) & 3;                      // warp inside its warpgroup
  const int lane = threadIdx.x & 31;
  // __cluster_dims__(2, 1, 1): blocks 2c and 2c + 1 form cluster c, with ranks 0 and 1.
  const int rank = blockIdx.x & 1, cluster = blockIdx.x >> 1, clusters = gridDim.x >> 1;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 4 * NC);                          // one arrival per consumer warp
      mbar_init(peer_free_bar(s), 1);                           // the peer's producer
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  cluster_sync();                                               // both CTAs' barriers exist before any remote use

  const int items = ord.m_tiles * ord.n_pairs * splits;

  // 384 threads get 168 registers each at launch, enough for BN = 128.  A wider tile's fragment and sums (2 x BN / 2
  // floats) do not fit that, so the producer drops to 40 and the consumers rise to 232 (128 * 40 + 256 * 232 = 64 512,
  // what the launch allocates).
  constexpr bool REBALANCE = BN > 128;
  if (wg == 0) {
    if constexpr (REBALANCE) setmaxnreg_dec<40>();
    // ===================== TMA producer =====================
    // Both CTAs of the pair need the whole BM-row A panel of the m-tile: each loads its BM/2-row half of A_hi and A_lo
    // once from L2 and multicasts it to the same stage offset in both CTAs; B is the CTA's own n-tile, a local load.
    // So a stage of this CTA is written by both producers, and may be refilled only once the consumers of BOTH CTAs
    // have released it: after its local `empty` wait, the producer tells the peer (remote arrival on the peer's
    // `peer_free`) and waits for the peer to say the same.  `full` still expects the whole stage; the peer's half may
    // land before the local expect_tx, which the transaction count allows.  Both CTAs walk the same k-blocks.
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      constexpr uint32_t stage_tx = static_cast<uint32_t>(L::STAGE_BYTES);
      constexpr uint32_t HALF_A = L::A_BYTES / 2;
      for (int w = cluster; w < items; w += clusters) {
        int mt, np, z;
        decode_item(w, ord, mt, np, z);
        const int nt = 2 * np + rank;                           // past the last n-tile: B is zero-filled
        const int kb0 = z * kb_per_split;
        const int kb1 = min(total_kb, kb0 + kb_per_split);
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait<true>(empty_bar(stage), phase ^ 1u);
          mbar_arrive_remote(peer_free_bar(stage), rank ^ 1);
          mbar_wait<true>(peer_free_bar(stage), phase);
          const uint32_t st = smem_base + stage * L::STAGE_BYTES;
          mbar_arrive_expect_tx(full_bar(stage), stage_tx);
          tma_load_2d_multicast(st + rank * HALF_A, &tmA_hi, full_bar(stage), kb * BKE, mt * BM + rank * (BM / 2), 0x3);
          tma_load_2d_multicast(st + L::A_BYTES + rank * HALF_A, &tmA_lo, full_bar(stage), kb * BKE,
                                mt * BM + rank * (BM / 2), 0x3);
          tma_load_2d(st + 2 * L::A_BYTES, &tmB_hi, full_bar(stage), kb * BKE, nt * BN);
          if constexpr (!BEXACT) tma_load_2d(st + 2 * L::A_BYTES + L::B_BYTES, &tmB_lo, full_bar(stage), kb * BKE, nt * BN);
          if (++stage == STAGES) { stage = 0; phase ^= 1u; }
        }
      }
      for (int s = 0; s < STAGES; ++s) {                        // every stage released: the consumers are through
        mbar_wait<true>(empty_bar(stage), phase ^ 1u);
        if (++stage == STAGES) { stage = 0; phase ^= 1u; }
      }
    }
  } else {
    // ===================== consumers: MMA chains + drain + epilogue =====================
    // The NC warpgroups take turns issuing one k-block of MMAs each, in a ring (warpgroup 1 first, then 2, ..., then 1
    // again): barrier TURN_BAR + cw is this warpgroup's turn, and it hands the turn to the next one right after its
    // commit.  Each chain's drain, sums and tile stores then run while the other warpgroups' k-blocks are still in the
    // tensor pipe.  All walk the same items, so they take the same number of turns; the last warpgroup's hand-off
    // before the first turn and warpgroup 1's sync after the last one pair the ends.  Only the issue time changes, not
    // which MMAs form a chain or the order of the sums.
    if constexpr (REBALANCE) setmaxnreg_inc<232>();
    constexpr uint32_t TURN_BAR = 1, TURN_THREADS = 256;
    const int cw = wg - 1;                                      // rows [64 cw, 64 cw + 64) of the tile
    const uint32_t a_off = static_cast<uint32_t>(cw * 64 * 128);
    const uint32_t next_bar = TURN_BAR + (cw + 1 == NC ? 0 : cw + 1);
    if (cw == NC - 1) named_bar_arrive(TURN_BAR, TURN_THREADS);
    int stage = 0;
    uint32_t phase = 0;
    for (int w = cluster; w < items; w += clusters) {
      int mt, np, z;
      decode_item(w, ord, mt, np, z);
      const int nt = 2 * np + rank;
      const int kb0 = z * kb_per_split;
      const int kb1 = min(total_kb, kb0 + kb_per_split);
      const int row0 = mt * BM + cw * 64 + warp * 16 + (lane >> 2);   // and row0 + 8
      float acc[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      // f16: power-of-two scale of this thread's two A rows for the scale group (2^a_gshift k-blocks) of a chain
      const float* sc_row0 = (F16 && a_tile_scale && row0 < M) ? a_tile_scale + static_cast<long long>(row0) * a_tiles : nullptr;
      const float* sc_row1 = (F16 && a_tile_scale && row0 + 8 < M) ? a_tile_scale + static_cast<long long>(row0 + 8) * a_tiles : nullptr;
      for (int c0 = kb0; c0 < kb1; c0 += chain_kb) {            // one short accumulation chain
        const int c1 = min(kb1, c0 + chain_kb);
        float d[BN / 2];
        int prev = -1;
        for (int kb = c0; kb < c1; ++kb) {
          mbar_wait<false>(full_bar(stage), phase);
          named_bar_sync(TURN_BAR + cw, TURN_THREADS);
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
            wgmma_tile<BN, F16>(d, a_lo + koff, b_hi + koff, acc0);     // small terms first
            if constexpr (!BEXACT) wgmma_tile<BN, F16>(d, a_hi + koff, b_lo + koff, 1u);
            wgmma_tile<BN, F16>(d, a_hi + koff, b_hi + koff, 1u);
          }
          wgmma_commit();
          named_bar_arrive(next_bar, TURN_THREADS);
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
          for (int i = 0; i < BN / 2; i += 4) {
            acc[i] = fmaf(d[i], s0, acc[i]);
            acc[i + 1] = fmaf(d[i + 1], s0, acc[i + 1]);
            acc[i + 2] = fmaf(d[i + 2], s1, acc[i + 2]);
            acc[i + 3] = fmaf(d[i + 3], s1, acc[i + 3]);
          }
        } else {
#pragma unroll
          for (int i = 0; i < BN / 2; ++i) acc[i] += d[i];          // round-to-nearest fp32
        }
      }
      if (nt >= n_tiles) continue;                              // second CTA of a pair past the last n-tile
      // Epilogue: a quad of lanes writes 32 contiguous bytes of a row per instruction (whole sectors).  The column
      // scales are loaded EPI_J at a time ahead of their stores, so the epilogue waits for 3 or fewer load latencies,
      // not for BN / 8 in a row, and fits better under the other warpgroup's last k-block (all 16 of a 128-column tile
      // at once would need 168 registers and spill).  EPI_J divides BN / 8: 8 (BN = 128, 192) or 7 (BN = 168).
      constexpr int EPI_J = (BN / 8) % 8 == 0 ? 8 : 7;
      static_assert((BN / 8) % EPI_J == 0, "column groups in whole batches");
      float* cbase = C + static_cast<long long>(z) * c_split_stride;
      const int colq = nt * BN + 2 * (lane & 3);
#pragma unroll
      for (int j0 = 0; j0 < BN / 8; j0 += EPI_J) {
        float2 sc[EPI_J];
#pragma unroll
        for (int j = 0; j < EPI_J; ++j) {                       // length >= ldc, zero padded
          const int col = colq + 8 * (j0 + j);
          sc[j] = out_scale && col < ldc ? *reinterpret_cast<const float2*>(out_scale + col) : make_float2(1.f, 1.f);
        }
#pragma unroll
        for (int j = 0; j < EPI_J; ++j) {
          const int col = colq + 8 * (j0 + j);
          if (col >= ldc) continue;                             // ldc % 4 == 0 and col even: col + 1 < ldc too
          const float* a = acc + 4 * (j0 + j);
          if (row0 < M)
            *reinterpret_cast<float2*>(cbase + static_cast<long long>(row0) * ldc + col) =
                make_float2(a[0] * sc[j].x, a[1] * sc[j].y);
          if (row0 + 8 < M)
            *reinterpret_cast<float2*>(cbase + static_cast<long long>(row0 + 8) * ldc + col) =
                make_float2(a[2] * sc[j].x, a[3] * sc[j].y);
        }
      }
    }
    if (cw == 0) named_bar_sync(TURN_BAR, TURN_THREADS);
  }
  cluster_sync();                 // neither CTA exits while the peer may still write its shared memory or barriers
}

template <int BN, int STAGES, bool BEXACT, bool F16>
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(NUM_THREADS, 1)
gemm_tf32x3_kernel(const __grid_constant__ CUtensorMap tmA_hi, const __grid_constant__ CUtensorMap tmA_lo,
                   const __grid_constant__ CUtensorMap tmB_hi, const __grid_constant__ CUtensorMap tmB_lo,
                   float* __restrict__ C, int M, int ldc, long long c_split_stride,
                   const TileOrder ord, int n_tiles, int splits, int total_kb, int kb_per_split, int chain_kb,
                   const float* __restrict__ out_scale, const float* __restrict__ a_tile_scale, int a_tiles, int a_gshift) {
  gemm_body<BN, STAGES, BEXACT, F16>(tmA_hi, tmA_lo, tmB_hi, tmB_lo, C, M, ldc, c_split_stride, ord, n_tiles, splits,
                                     total_kb, kb_per_split, chain_kb, out_scale, a_tile_scale, a_tiles, a_gshift);
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

// Modelled HBM bytes of one split-K slice in a grouped tile order (tools/probe_gemm.py restates this model): the
// `group` panels of the grouped operand q are read once if they fit the L2 budget, else once per wave of the grid that
// passes over them; every panel of the swept operand p is read once per group (its readers run side by side).
static double order_bytes(int q_tiles, int p_tiles, double q_panel, double p_panel, int group, int grid, double budget) {
  const long long waves = (static_cast<long long>(group) * p_tiles + grid - 1) / grid;
  const double q_reads = group * q_panel <= budget ? 1.0 : static_cast<double>(std::min<long long>(p_tiles, waves));
  return q_tiles * q_panel * q_reads + static_cast<double>((q_tiles + group - 1) / group) * p_tiles * p_panel;
}

// The tile order with the least modelled traffic, over both orientations and every balanced group size, with half of
// the L2 as the budget of the resident panels (the other half holds the streamed operand and the output lines).
// a_panel: bytes of one BM-row A panel of a slice, b_panel: of the 2 BN rows of B one n-pair covers, all pieces;
// grid: the number of pairs (clusters) that run at once.  Ties keep the m-tile-fastest order, which is what a problem
// whose factor operand fits the L2 gets.  The order decides only which CTA computes a tile when: every output element
// is still formed by the same chains in the same order.
static TileOrder pick_tile_order(int m_tiles, int n_pairs, double a_panel, double b_panel, int grid, long long l2_bytes) {
  const double budget = 0.5 * static_cast<double>(l2_bytes);
  TileOrder best{m_tiles, n_pairs, m_tiles, 0};
  double best_bytes = order_bytes(m_tiles, n_pairs, a_panel, b_panel, m_tiles, grid, budget);
  for (int gn = 0; gn < 2; ++gn) {
    const int q = gn ? n_pairs : m_tiles, p = gn ? m_tiles : n_pairs;
    const double qb = gn ? b_panel : a_panel, pb = gn ? a_panel : b_panel;
    int prev = 0;
    for (int ng = 1; ng <= q; ++ng) {                 // groups of ceil(q / ng) tiles, the last one possibly shorter
      const int g = (q + ng - 1) / ng;
      if (g == prev) continue;
      prev = g;
      const double b = order_bytes(q, p, qb, pb, g, grid, budget);
      if (b < best_bytes) { best_bytes = b; best = TileOrder{m_tiles, n_pairs, g, gn}; }
    }
  }
  return best;
}

template <int BN, int STAGES, bool BEXACT, bool F16>
int launch(const GemmArgs& g, cudaStream_t stream) {
  using L = SmemLayout<BN, STAGES, BEXACT>;
  constexpr int BKE = F16 ? 2 * BK : BK;
  CUtensorMap mAh, mAl, mBh, mBl;
  int rc;
  if ((rc = make_map(&mAh, g.A_hi, g.M, g.Kd, g.lda, BM / 2, F16))) return rc;     // each CTA of a pair loads half
  if ((rc = make_map(&mAl, g.A_lo, g.M, g.Kd, g.lda, BM / 2, F16))) return rc;
  if ((rc = make_map(&mBh, g.B_hi, g.N, g.Kd, g.ldb, BN, F16))) return rc;
  if ((rc = make_map(&mBl, BEXACT ? g.B_hi : g.B_lo, g.N, g.Kd, g.ldb, BN, F16))) return rc;
  int dev = 0, l2 = 0;
  CNMF_CUDA_CHECK(cudaGetDevice(&dev));
  CNMF_CUDA_CHECK(cudaDeviceGetAttribute(&l2, cudaDevAttrL2CacheSize, dev));
  const int m_tiles = (g.M + BM - 1) / BM;
  // The tiles cover the columns up to the next multiple of 32 (ldc permitting) whatever BN is: a 128-column tile
  // grid always reaches that far, and the padding columns of a row-stride-padded output then hold zeros.
  const int n_tiles = (std::min(g.ldc, (g.N + 31) / 32 * 32) + BN - 1) / BN;
  const int n_pairs = (n_tiles + 1) / 2;
  const int total_kb = (g.Kd + BKE - 1) / BKE;
  int splits = g.splits < 1 ? 1 : g.splits;
  if (splits > total_kb) splits = total_kb;
  int kb_per_split = (total_kb + splits - 1) / splits;
  if (F16 && (kb_per_split & 1)) ++kb_per_split;             // chains (2 k-blocks) must not straddle a 512-element scale group
  splits = (total_kb + kb_per_split - 1) / kb_per_split;      // no empty slices
  if (splits != g.splits_effective) { set_last_error("gemm: splits_effective mismatch (use gemm_effective_splits)"); return -1; }

  auto kern = gemm_tf32x3_kernel<BN, STAGES, BEXACT, F16>;
  // Per device (a second GPU in the same process needs its own calls): the shared-memory attribute, then how many
  // pairs fit at once (66 on a 132-SM H100 SXM).
  static int max_clusters[64] = {};
  int clusters_cap = dev >= 0 && dev < 64 ? max_clusters[dev] : 0;
  if (clusters_cap == 0) {
    CNMF_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::DYN_BYTES));
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(2, 1, 1);
    cfg.blockDim = dim3(NUM_THREADS, 1, 1);
    cfg.dynamicSmemBytes = L::DYN_BYTES;
    CNMF_CUDA_CHECK(cudaOccupancyMaxActiveClusters(&clusters_cap, kern, &cfg));
    if (clusters_cap < 1) { set_last_error("gemm: no 2-CTA cluster of this kernel fits the device"); return -1; }
    if (dev >= 0 && dev < 64) max_clusters[dev] = clusters_cap;
  }
  const int items = m_tiles * n_pairs * splits;
  const int clusters = items < clusters_cap ? items : clusters_cap;
  const double kslice_row = static_cast<double>(kb_per_split) * BK * 4;       // bytes of one slice row, one piece
  const TileOrder ord = pick_tile_order(m_tiles, n_pairs, BM * kslice_row * 2, 2 * BN * kslice_row * (BEXACT ? 1 : 2),
                                        clusters, l2);
  // chain_kb: at most 16 MMAs between drains (3-pass form: 1 k-block = 12 MMAs, exact-B forms: 2 k-blocks = 16; f16
  // chains of 2 never straddle a scale group).  a_gshift = 3: f16 scale groups of 8 k-blocks = 512 elements.
  kern<<<2 * clusters, NUM_THREADS, L::DYN_BYTES, stream>>>(mAh, mAl, mBh, mBl, g.C, g.M, g.ldc, g.c_split_stride,
                                                            ord, n_tiles, splits, total_kb, kb_per_split, BEXACT ? 2 : 1,
                                                    g.out_col_scale, g.a_tile_scale, g.a_tiles, 3);
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

// Output-tile width of an exact-B product (the general 3-pass form has 128-column tiles only).  The persistent grid
// runs its pair items in ceil(items / pairs) rounds, and a pair item of a BN-column tile takes about 1.25 (BN = 168)
// or 1.42 (BN = 192) times as long as a 128-column one, measured on the c3 products (DESIGN.md section 4.1), against
// the 1.31 and 1.5 of their FLOPs, because the MMAs read less shared memory per FLOP the wider the tile.  So a width
// costs its rounds times that; a wide width is taken when it saves at least 2 % (near-ties keep 128 columns).
static int pick_tile_n(const GemmArgs& g) {
  if (!g.b_exact) return 128;
  int dev = 0, sms = 0;
  CNMF_CUDA_CHECK(cudaGetDevice(&dev));
  CNMF_CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const long long pairs = std::max(1, sms / 2);
  const long long m_items = static_cast<long long>((g.M + BM - 1) / BM) * g.splits_effective;
  const int cols = std::min(g.ldc, (g.N + 31) / 32 * 32);      // what launch() covers
  auto cost = [&](int bn, int per_item) {
    const long long items = m_items * (((cols + bn - 1) / bn + 1) / 2);
    return (items + pairs - 1) / pairs * per_item;
  };
  const long long narrow = cost(128, 100);
  int best = 128;
  long long best_cost = narrow * 98 / 100;
  for (const auto& [bn, per_item] : {std::pair<int, int>{168, 125}, std::pair<int, int>{192, 142}}) {
    const long long c = cost(bn, per_item);
    if (c <= best_cost) { best_cost = c; best = bn; }
  }
  return best;
}

int gemm_tf32x3(const GemmArgs& g, cudaStream_t stream) {
  CNMF_REQUIRE(g.M > 0 && g.N > 0 && g.Kd > 0, "gemm: empty problem");
  CNMF_REQUIRE(g.lda % 4 == 0 && g.ldb % 4 == 0 && g.ldc % 4 == 0, "gemm: leading dimensions must be multiples of 4 floats");
  CNMF_REQUIRE((reinterpret_cast<uintptr_t>(g.A_hi) | reinterpret_cast<uintptr_t>(g.A_lo) |
                reinterpret_cast<uintptr_t>(g.B_hi) | reinterpret_cast<uintptr_t>(g.B_lo) |
                reinterpret_cast<uintptr_t>(g.C) | reinterpret_cast<uintptr_t>(g.out_col_scale)) % 16 == 0,
               "gemm: pointers must be 16-byte aligned");
  // Results do not depend on the tile width: every element is formed by the same chains in the same order.
  CNMF_REQUIRE(g.tile_n == 0 || g.tile_n == 128 || (g.b_exact && (g.tile_n == 168 || g.tile_n == 192)),
               "gemm: tile_n must be 0 (the launcher's choice), 128, or 168 / 192 with an exact B");
  const int bn = g.tile_n ? g.tile_n : pick_tile_n(g);
  if (g.f16) {
    CNMF_REQUIRE(g.b_exact, "gemm: the fp16 path needs an exact B operand");
    CNMF_REQUIRE(g.lda % 8 == 0 && g.ldb % 8 == 0, "gemm: fp16 leading dimensions must be multiples of 8 halves");
    CNMF_REQUIRE(!g.a_tile_scale || g.a_tiles * 512 >= g.Kd, "gemm: a_tiles does not cover the reduction length");
    if (bn == 168) return launch<168, 4, true, true>(g, stream);
    if (bn == 192) return launch<192, 4, true, true>(g, stream);
    return launch<128, 4, true, true>(g, stream);
  }
  if (g.b_exact) {
    if (bn == 168) return launch<168, 4, true, false>(g, stream);
    if (bn == 192) return launch<192, 4, true, false>(g, stream);
    return launch<128, 4, true, false>(g, stream);
  }
  return launch<128, 3, false, false>(g, stream);
}

}  // namespace cnmf
