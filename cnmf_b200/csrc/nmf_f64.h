// Launches of the float64 solver (nmf_f64.cu), shared by its ops in the batched solve (solve.h) and the
// cnmf_update_step_f64_host test hook (capi_units.cu), so that the hook runs exactly the launches the solver runs.
#pragma once
#include "engine.h"
#include "nmf_kernels.cuh"
#include "solve.h"

namespace cnmf {

constexpr int F64_ITEMS = 256;        // items per block of the update / cross kernels (one per thread)
constexpr int F64_GRAM_COLS = 2048;   // items per block of the Gram kernel

// chunkings: functions of the item count only
inline int f64_chunks(int n) { return (n + F64_ITEMS - 1) / F64_ITEMS; }
inline int f64_gram_chunks(int n) { return (n + F64_GRAM_COLS - 1) / F64_GRAM_COLS; }

struct F64View {
  double* F;       // SK x ld
  int n, ld;
};

struct F64Launch {      // what every launch of one batch shares
  cnmf_handle_s* h;     // counts the launches, times the updates
  cudaStream_t s;
  int SK;               // packed rows (the updates' profiled work)
};

// Gram of every live restart: gram64_kernel into part ([rid][chunk] kp x kp blocks, f64_gram_chunks(f.n) chunks),
// then finalize_kernel into gram ([rid] 32 x 32)
int f64_gram(const F64Launch& L, const F64View& f, const BatchMeta& b, double* part, double* gram);
// <NUM, F> of every live restart: cross64_kernel into part ([rid][chunk], f64_chunks(f.n) chunks), then finalize into out
int f64_cross(const F64Launch& L, const F64View& f, const double* NUM, const BatchMeta& b, double* part, double* out);
// one MU (cd = false) or CD update of every live restart with the other factor's Gram gram_in; scal (optional, then part
// is its [rid][chunk] partials) receives MU <NUM, F_new> / CD sum |projected gradient| through finalize
int f64_update(const F64Launch& L, bool cd, const F64View& f, const double* NUM, const double* gram_in,
               const BatchMeta& b, double l1, double l2, double* part, double* scal);

// The FP64 ops of the batched solve: products through gemm_f64 (one slice), the update then a stand-alone Gram, block
// plans fixed by the item counts, no operand pieces.  Compaction saves 64-row GEMM tiles.
struct F64Ops {
  using T = double;
  static constexpr int tile_rows = 64;
  static constexpr const char* buf_tag = "64";     // suffix of the workspace buffer names
  static constexpr bool fused_gram = false;
  static int pick_kp(int kmax) { return round_up(kmax, 4); }

  FroSolve<double>& b;
  bool cd;
  double l1[2], l2[2];
  int chunks[2];
  int chunks_cap;            // partial scalars per restart and side
  size_t gram_part_elems;    // Gram partials per side

  F64Ops(FroSolve<double>& b, const cnmf_nmf_params& p);
  int alloc();                                            // product buffers
  int start() { return 0; }
  int gemm(int side);                                     // NUM[side]
  int gram(int side, const BatchMeta& m);                 // Gram of F[side]
  int grams(const BatchMeta& m);                          // both Grams
  int cross(int side, const BatchMeta& m, double* out);   // <NUM[side], F[side]>
  int update(int side, bool want_gram, bool want_scal, double* scal);
  int compact(const std::vector<int>&, const std::vector<int>&, const std::vector<int>&) { return 0; }
  int repack() { return 0; }
};

}  // namespace cnmf
