// Batched NMF solver: all (k, seed) restarts of cNMF.factorize (cnmf.py:735-745) advance together.
//
// One outer iteration of sklearn's solvers (MU: _nmf.py:826-879, CD: _nmf.py:491-516) becomes
//   NUM_r = Fc * X^T            tensor-core GEMM, M = sum k (all restarts), N = n_r, reduce over n_c
//   Fr   <- update(Fr, NUM_r, Gram(Fc))       elementwise, K x K Gram from smem
//   NUM_c = Fr * X              tensor-core GEMM, split-K over n_r
//   Fc   <- update(Fc, NUM_c, Gram(Fr))
// with Fr = W^T (SK x cells) and Fc = H (SK x genes), so the data matrix is streamed once per
// product for ALL restarts.  Convergence is evaluated on the device per restart (trace-form
// Frobenius error for MU, projected-gradient violation for CD); converged restarts are frozen
// (their blocks exit) and the host only polls the flags.
#include <algorithm>
#include <cmath>
#include <cstring>

#include "engine.h"
#include "gemm.h"
#include "nmf_f64.h"
#include "nmf_kernels.cuh"
#include "solve.h"

namespace cnmf {

DataView make_view(const cnmf_dataset_s* d, bool transposed) {
  const bool f16 = d->form == Form::F16_EXACT;
  Operand X{d->X, f16 ? static_cast<const float*>(d->X_h16) : d->X_hi, d->X_lo, d->n_rows, d->n_cols, d->ld_c};
  Operand Xt{d->Xt, f16 ? static_cast<const float*>(d->Xt_h16) : d->Xt_hi, d->Xt_lo, d->n_cols, d->n_rows, d->ld_r};
  DataView v;
  if (!transposed) {
    v.B_rows = X; v.B_cols = Xt;
    v.n_r = d->n_rows; v.n_c = d->n_cols; v.ld_r = d->ld_r; v.ld_c = d->ld_c;
  } else {
    v.B_rows = Xt; v.B_cols = X;
    v.n_r = d->n_cols; v.n_c = d->n_rows; v.ld_r = d->ld_c; v.ld_c = d->ld_r;
  }
  v.sum = d->sum;
  v.sum_sq = d->sum_sq;
  // a sparse dataset keeps its detected form and scales for cnmf_dataset_from_columns; its solves (refits) take the
  // one product from csc_project and run the fp32 solver code: no GEMM, no pieces, no scales
  v.form = d->sparse ? Form::FP32 : d->form;
  v.scale_r = d->sparse ? nullptr : transposed ? d->col_scale : d->row_scale;
  v.scale_c = d->sparse ? nullptr : transposed ? d->row_scale : d->col_scale;
  v.X64 = d->X64;
  v.transposed = transposed;
  return v;
}

int form_gemm(Form form, GemmArgs g, const float* A, const float* A_hi, const float* A_lo, const float* a_tile_scale,
              const Operand& B, const float* out_scale, cudaStream_t s) {
  switch (form) {
    case Form::FP32:
      g.A_hi = A; g.B_hi = B.full;
      return gemm_fp32_simt(g, s);
    case Form::TF32:
      g.B_lo = B.lo;
      break;
    case Form::F16_EXACT:      // A_hi / A_lo hold the two fp16 pieces of the row-normalised factor, B.hi fp16 C
      g.f16 = 1; g.a_tile_scale = a_tile_scale; g.a_tiles = (g.lda + 511) / 512;
      [[fallthrough]];
    case Form::TF32_EXACT:
      g.b_exact = 1; g.out_col_scale = out_scale;
      break;
    case Form::FP64:
      set_last_error("float64 datasets run their products through gemm_f64");
      return -3;
  }
  g.A_hi = A_hi; g.A_lo = A_lo; g.B_hi = B.hi;
  return gemm_tf32x3(g, s);
}

int make_pieces(Form form, const float* F, int rows, int n, int ld, const float* scale, float* hi, float* lo,
                float* tile_scale, cudaStream_t s) {
  switch (form) {
    case Form::FP32:
    case Form::FP64: return 0;
    case Form::F16_EXACT: return launch_emit_f16(F, rows, n, ld, scale, hi, lo, tile_scale, (ld + 511) / 512, s);
    default: return launch_split_scaled(F, hi, lo, rows, ld, scale, s);
  }
}

GemmPlan view_gemm_plan(const DataView& v, int side, int SK) {
  const int f16 = v.form == Form::F16_EXACT ? 1 : 0;
  return side == 0 ? GemmPlan{gemm_fixed_splits(v.n_c, f16), (long long)SK * v.ld_r}
                   : GemmPlan{gemm_fixed_splits(v.n_r, f16), (long long)SK * v.ld_c};
}

int view_gemm(cnmf_handle_s* h, const DataView& v, int side, const float* F, const float* F_hi, const float* F_lo,
              const float* tile_scale, int SK, float* C, const GemmPlan& plan, cudaStream_t s) {
  const Operand& B = side == 0 ? v.B_rows : v.B_cols;
  GemmArgs g{};
  g.M = SK; g.N = B.rows; g.Kd = B.cols;
  g.lda = side == 0 ? v.ld_c : v.ld_r;
  g.ldb = B.ld;
  g.ldc = side == 0 ? v.ld_r : v.ld_c;
  g.C = C;
  g.c_split_stride = plan.split_stride;
  g.splits = plan.splits;
  g.splits_effective = plan.splits;
  h->launches += 1;
  const int slot = h->prof_begin(s, 2.0 * (double)g.M * (double)g.N * (double)g.Kd);
  const int rc = form_gemm(v.form, g, F, F_hi, F_lo, tile_scale, B, side == 0 ? v.scale_r : v.scale_c, s);
  h->prof_end(s, slot);
  return rc;
}

// gather member of the batched solve's state (solve.h): rows of E go through launch_gather_rows as ld * sizeof(E) / 4
// floats, a bit copy
template <class T>
template <class E>
int FroSolve<T>::gather(const E* src, E* dst, const std::vector<int>& so, const std::vector<int>& dof,
                        const std::vector<int>& kk, int ld_e) {
  const int cnt = (int)kk.size();
  if (cnt == 0 || !src || !dst) return 0;
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
                            cnt, ld_e * (int)(sizeof(E) / sizeof(float)), s);
}

namespace {

// The float forms' ops of the batched solve: products through view_gemm with the split-K plan of view_gemm_plan, the
// update kernels with their fused outputs (Gram when kp == 16, otherwise a stand-alone Gram follows), and the factors'
// operand pieces -- tf32 hi / lo written by the update kernels, or on f16 datasets the two fp16 pieces (same buffers).
// Block plans follow the live restart count.  Compaction saves 128-row GEMM tiles.
struct F32Ops {
  using T = float;
  static constexpr int tile_rows = 128;
  static constexpr const char* buf_tag = "";
  static int pick_kp(int kmax) { return kmax <= 16 ? 16 : 32; }

  FroSolve<float>& b;
  const DataView& v;
  bool cd;
  float l1[2], l2[2];
  const bool tf32, f16;     // the factors have operand pieces; they are fp16 pieces
  bool fused_gram;          // the update kernels emit the Gram of the factor they write (nmf_kernels.cu)
  // tf32 pieces are written by the update kernels; the fp16 pieces need the row maximum first and come from
  // emit_pieces() after the update (the hi / lo buffers then hold halves)
  bool upd_pieces;
  // f16: the Gram-fused update kernels (K <= 16, factor being iterated) emit the fp16 pieces themselves, per 512-column
  // tile; everything else (initial factors, compaction, K > 16) goes through emit_pieces(), which normalises the same
  // 512-column groups and writes the same bits
  bool emit_in_update;
  int cpb[2] = {}, gcpb[2] = {}, chunks[2] = {}, ktiles[2] = {};
  int chunks_cap;           // finest chunking possible
  size_t gram_part_elems;
  GemmPlan plan[2];         // plan[0]: NUM_r = Fc * B_rows^T (reduce over n_c); plan[1]: NUM_c = Fr * B_cols^T
  float *hi[2] = {}, *lo[2] = {}, *alt_hi[2] = {}, *alt_lo[2] = {};
  float* tile_scale[2] = {};   // f16: power-of-two scales of the pieces, [packed row][512-element group]

  const float* scale(int side) const { return side ? v.scale_c : v.scale_r; }

  F32Ops(FroSolve<float>& b_, const cnmf_nmf_params& p)
      : b(b_), v(b_.v), cd(p.solver == CNMF_SOLVER_CD), tf32(v.form != Form::FP32), f16(v.form == Form::F16_EXACT) {
    l1[0] = (float)p.l1_reg_W; l2[0] = (float)p.l2_reg_W; l1[1] = (float)p.l1_reg_H; l2[1] = (float)p.l2_reg_H;
    fused_gram = b.kp == 16;
    upd_pieces = tf32 && !f16;
    emit_in_update = f16 && b.kp == 16 && b.io.update_cols;
    // block granularity of the streaming kernels: update kernels 3 blocks of 128 threads per SM resident, a block walks
    // 1-4 tiles -> aim for >= 8 blocks per SM; stand-alone Gram kernel: 1 block/SM resident and a fixed-cost block
    // reduction -> long blocks, about two waves
    const int tile = upd_tile_cols(b.kp);
    for (int side = 0; side < 2; ++side) {
      gcpb[side] = pick_cols_per_block(b.n(side), b.R0, 8192, 1024, b.h->sm_count * 2);
      ktiles[side] = (b.ld(side) + 511) / 512;
    }
    chunks_cap = std::max((v.n_r + tile - 1) / tile, (v.n_c + tile - 1) / tile);
    const int gchunks_max = std::max((v.n_r + gcpb[0] - 1) / gcpb[0], (v.n_c + gcpb[1] - 1) / gcpb[1]);
    size_t fused_part_slots = 0;   // slot-indexed partials of the fused kernels: max over live counts of R * chunks
    for (int r = 1; r <= b.R0; ++r) {
      plan_blocks(r);
      fused_part_slots = std::max(fused_part_slots, (size_t)r * std::max(chunks[0], chunks[1]));
    }
    plan_blocks(b.R0);
    gram_part_elems = std::max((size_t)b.R0 * std::max(gchunks_max, std::max((v.n_r + 1023) / 1024, (v.n_c + 1023) / 1024)),
                               fused_part_slots) * b.kp * b.kp;
    plan_gemms();
  }
  // the update kernels' chunking follows the number of LIVE restarts (re-planned after every compaction): with few
  // restarts left a block should hold one tile, so that the work spreads over many SMs
  void plan_blocks(int r_live) {
    const int tile = upd_tile_cols(b.kp);
    for (int side = 0; side < 2; ++side) {
      cpb[side] = pick_cols_per_block(b.n(side), r_live, 4 * tile, tile, b.h->sm_count * 8);
      chunks[side] = (b.n(side) + cpb[side] - 1) / cpb[side];
    }
  }
  // the split-K factor is a function of the reduction length only (gemm_fixed_splits)
  void plan_gemms() {
    plan[0] = view_gemm_plan(v, 0, b.SK);
    if (b.io.num_rows) plan[0].splits = 1;
    plan[1] = view_gemm_plan(v, 1, b.SK);
  }

  int alloc() {
    // the rows never exceed SK0
    const size_t need_r = (size_t)plan[0].splits * (size_t)b.SK0 * v.ld_r;
    const size_t need_c = (size_t)plan[1].splits * (size_t)b.SK0 * v.ld_c;
    b.NUM[0] = b.io.num_rows ? const_cast<float*>(b.io.num_rows)
                             : static_cast<float*>(b.h->dev_buf("solve.NUMr", sizeof(float) * need_r));
    b.NUM[1] = b.io.update_cols ? static_cast<float*>(b.h->dev_buf("solve.NUMc", sizeof(float) * need_c)) : nullptr;
    if (!b.NUM[0] || (b.io.update_cols && !b.NUM[1])) return -2;
    if (tf32) {
      const size_t nr = (size_t)b.SK0 * v.ld_r, nc = (size_t)b.SK0 * v.ld_c;
      hi[0] = static_cast<float*>(b.h->dev_buf("solve.Fr_hi", nr * 4));
      lo[0] = static_cast<float*>(b.h->dev_buf("solve.Fr_lo", nr * 4));
      hi[1] = static_cast<float*>(b.h->dev_buf("solve.Fc_hi", nc * 4));
      lo[1] = static_cast<float*>(b.h->dev_buf("solve.Fc_lo", nc * 4));
      if (!hi[0] || !lo[0] || !hi[1] || !lo[1]) return -2;
    }
    if (f16) {
      tile_scale[0] = static_cast<float*>(b.h->dev_buf("solve.rowscale_r", sizeof(float) * (size_t)b.SK0 * ktiles[0]));
      tile_scale[1] = static_cast<float*>(b.h->dev_buf("solve.rowscale_c", sizeof(float) * (size_t)b.SK0 * ktiles[1]));
      if (!tile_scale[0] || !tile_scale[1]) return -2;
    }
    return 0;
  }

  FactorView view(int side) const {
    FactorView f{};
    f.F = b.F[side];
    // the fixed factor of a refit is never rewritten
    const bool pieces = upd_pieces && (side == 0 || b.io.update_cols);
    f.F_hi = pieces ? hi[side] : nullptr;
    f.F_lo = pieces ? lo[side] : nullptr;
    f.n = b.n(side); f.ld = b.ld(side); f.piece_scale = scale(side);
    if (emit_in_update) { f.P_hi = hi[side]; f.P_mid = lo[side]; f.tile_scale = tile_scale[side]; f.n_ktiles = ktiles[side]; }
    f.cpb = cpb[side]; f.gcpb = gcpb[side];
    return f;
  }
  int pieces(int side) {
    return make_pieces(v.form, b.F[side], b.SK, b.n(side), b.ld(side), scale(side), hi[side], lo[side], tile_scale[side], b.s);
  }
  int emit_pieces(int side) {   // fp16 pieces + row scales of a factor that was just (re)written
    if (!f16) return 0;
    b.h->launches += 1;
    const int slot = b.h->prof_begin(b.s, 8.0 * (double)b.SK * (double)b.n(side), 1);   // fp32 in, two fp16 pieces out
    const int rc = pieces(side);
    b.h->prof_end(b.s, slot);
    return rc;
  }
  int start() {
    if (upd_pieces) {              // tf32 pieces of the starting factors; afterwards the update kernels write them
      CNMF_TRY(pieces(0));
      CNMF_TRY(pieces(1));
      b.h->launches += 2;
    }
    CNMF_TRY(emit_pieces(0));      // f16: fp16 pieces of the starting factors
    return emit_pieces(1);
  }

  int gemm(int side) {
    if (side == 0 && b.io.num_rows) return 0;   // computed by the caller
    const int o = 1 - side;                     // the factor multiplied
    return view_gemm(b.h, v, side, b.F[o], hi[o], lo[o], tile_scale[o], b.SK, b.NUM[side], plan[side], b.s);
  }
  // stand-alone Gram: partial launch + finalize (initial factors, fixed factors of a refit, batches with K > 16)
  int gram(int side, const BatchMeta& m) {
    b.h->launches += 2;
    const FactorView f = view(side);
    CNMF_TRY(launch_gram_partial(f, m, b.gram_part[side], b.s));
    return launch_finalize(b.gram_part[side], b.gram[side], nullptr, nullptr, gram_chunks(f), m, b.s);
  }
  int grams(const BatchMeta& m) {
    b.h->launches += 4;
    CNMF_TRY(launch_gram_partial(view(0), m, b.gram_part[0], b.s));
    CNMF_TRY(launch_gram_partial(view(1), m, b.gram_part[1], b.s));
    CNMF_TRY(launch_finalize(b.gram_part[0], b.gram[0], nullptr, nullptr, gram_chunks(view(0)), m, b.s));
    return launch_finalize(b.gram_part[1], b.gram[1], nullptr, nullptr, gram_chunks(view(1)), m, b.s);
  }
  int cross(int side, const BatchMeta& m, double* out) {
    b.h->launches += 2;
    CNMF_TRY(launch_cross(view(side), b.NUM[side], plan[side].splits, plan[side].split_stride, m, b.scal_part[side], b.s));
    return launch_finalize(nullptr, nullptr, b.scal_part[side], out, chunks[side], m, b.s);
  }
  int update(int side, bool want_gram, bool want_scal, double* scal) {
    const FactorView f = view(side);
    FusedOut out{};
    if (want_gram && fused_gram) {
      out.gram_part = b.gram_part[side];
      out.gram = b.gram[side];
    }
    out.scal_part = want_scal ? b.scal_part[side] : nullptr;
    out.scal = scal;
    out.counter = b.d_ticket;
    const GemmPlan& pl = plan[side];
    // algorithmic bytes: factor read, product slices read, factor (+ pieces: two tf32 pieces = 2 floats per element,
    // two fp16 pieces = 1) written
    const int piece_floats = f.F_hi ? 2 : ((f.P_hi && out.gram_part) ? 1 : 0);
    b.h->launches += 1;
    const int slot = b.h->prof_begin(b.s, 4.0 * (double)b.SK * (double)f.n * (double)(2 + pl.splits + piece_floats), 1);
    const double* gram_in = b.gram[1 - side];
    const int rc = cd ? launch_cd_update(f, b.NUM[side], pl.splits, pl.split_stride, gram_in, b.bm(), l1[side], l2[side], out, b.s)
                      : launch_mu_update(f, b.NUM[side], pl.splits, pl.split_stride, gram_in, b.bm(), l1[side], l2[side], out, b.s);
    b.h->prof_end(b.s, slot);
    if (rc != 0 || !b.io.update_cols) return rc;   // a refit never multiplies by the factor it updates
    if (f.P_hi && out.gram_part) return 0;         // the Gram-fused kernel emitted the pieces of every tile it wrote
    return emit_pieces(side);
  }

  // the live restarts' pieces follow their factors to the packed front of the alternates (tf32; f16 pieces are
  // emitted again by repack)
  int compact(const std::vector<int>& src, const std::vector<int>& dst, const std::vector<int>& k) {
    if (tf32 && !alt_hi[0]) {
      const size_t nr = (size_t)b.SK0 * v.ld_r, nc = (size_t)b.SK0 * v.ld_c;
      alt_hi[0] = static_cast<float*>(b.h->dev_buf("solve.alt.Fr_hi", nr * 4));
      alt_lo[0] = static_cast<float*>(b.h->dev_buf("solve.alt.Fr_lo", nr * 4));
      alt_hi[1] = static_cast<float*>(b.h->dev_buf("solve.alt.Fc_hi", nc * 4));
      alt_lo[1] = static_cast<float*>(b.h->dev_buf("solve.alt.Fc_lo", nc * 4));
      if (!alt_hi[0] || !alt_lo[0] || !alt_hi[1] || !alt_lo[1]) return -2;
    }
    if (upd_pieces)
      for (int side = 0; side < 2; ++side) {
        CNMF_TRY(b.gather(hi[side], alt_hi[side], src, dst, k, b.ld(side)));
        CNMF_TRY(b.gather(lo[side], alt_lo[side], src, dst, k, b.ld(side)));
      }
    for (int side = 0; side < 2; ++side) {
      std::swap(hi[side], alt_hi[side]);
      std::swap(lo[side], alt_lo[side]);
    }
    return 0;
  }
  // after a compaction: plans and f16 pieces follow the new packing
  int repack() {
    plan_gemms();
    plan_blocks(b.R);
    CNMF_TRY(emit_pieces(0));
    return emit_pieces(1);
  }
};

// One Frobenius batched solve (MU or CD, factorize or refit) on the ops of the factor element type.
//
// One outer iteration of sklearn's solvers (MU: _nmf.py:826-879, CD: _nmf.py:491-516) becomes
//   NUM_r = Fc * X^T,  Fr <- update(Fr, NUM_r, Gram(Fc)),  NUM_c = Fr * X,  Fc <- update(Fc, NUM_c, Gram(Fr)).
// Convergence is evaluated on the device per restart; converged restarts are frozen and the host only polls the flags,
// dropping them from the packed arrays (compaction) when that saves a GEMM tile.
template <class Ops>
int solve_frobenius(cnmf_handle_s* h, const DataView& v, SolveIO<typename Ops::T>& io, const cnmf_nmf_params& p,
                    cudaStream_t s) {
  using T = typename Ops::T;
  const int R0 = io.R;
  CNMF_REQUIRE(R0 > 0 && (int)io.ks.size() == R0, "solve: bad restart list");
  CNMF_REQUIRE(p.solver == CNMF_SOLVER_MU || p.solver == CNMF_SOLVER_CD, "solve: unknown solver");
  CNMF_REQUIRE(p.max_iter >= 1, "solve: max_iter must be >= 1");
  CNMF_REQUIRE(!io.num_rows || !io.update_cols, "solve: a caller-computed row product needs update_cols = false");
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
  FroSolve<T> b{h, v, io, s};
  b.R0 = b.R = R0;
  b.SK0 = b.SK = SK0;
  b.kp = Ops::pick_kp(kmax);
  b.F[0] = io.Fr;
  b.F[1] = io.Fc;
  // packed layout of a list of restarts: each one's rows follow the previous one's
  auto pack_offsets = [&](const std::vector<int>& kk, std::vector<int>& offs) -> int {
    int pos = 0;
    offs.clear();
    for (int k : kk) {
      offs.push_back(pos);
      pos += k;
    }
    return pos;
  };
  Ops ops(b, p);

  // ---- workspace
  int* d_meta = static_cast<int*>(h->dev_buf("solve.meta", sizeof(int) * 8 * R0));
  double* d_state = static_cast<double*>(h->dev_buf("solve.state", sizeof(double) * 8 * R0));
  double* d_gram = static_cast<double*>(h->dev_buf("solve.gram", sizeof(double) * 2 * R0 * KMAX * KMAX));
  double* d_gram_part = static_cast<double*>(h->dev_buf("solve.gram_part", sizeof(double) * 2 * ops.gram_part_elems));
  double* d_scal_part =
      static_cast<double*>(h->dev_buf("solve.scal_part", sizeof(double) * 2 * (size_t)R0 * ops.chunks_cap));
  if (!d_meta || !d_state || !d_gram || !d_gram_part || !d_scal_part) return -2;
  CNMF_TRY(ops.alloc());

  b.d_off = d_meta;                // [slots]
  b.d_k = d_meta + R0;             // [slots]
  b.d_rid = d_meta + 2 * R0;       // [slots]
  b.d_done = d_meta + 3 * R0;      // [rid]
  int* d_niter = d_meta + 4 * R0;  // [rid]
  b.d_ticket = d_meta + 5 * R0;    // [rid] last-block tickets of the fused update kernels (self-resetting)
  auto upload_slots = [&]() -> int {
    std::vector<int> hm(3 * R0, 0);
    std::memcpy(hm.data(), s_off.data(), sizeof(int) * b.R);
    std::memcpy(hm.data() + R0, s_k.data(), sizeof(int) * b.R);
    std::memcpy(hm.data() + 2 * R0, s_rid.data(), sizeof(int) * b.R);
    CNMF_CUDA_CHECK(cudaMemcpyAsync(d_meta, hm.data(), sizeof(int) * 3 * R0, cudaMemcpyHostToDevice, s));
    CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
    return 0;
  };
  CNMF_TRY(upload_slots());
  CNMF_CUDA_CHECK(cudaMemsetAsync(b.d_done, 0, sizeof(int) * 3 * R0, s));   // done, n_iter, tickets
  CNMF_CUDA_CHECK(cudaMemsetAsync(d_state, 0, sizeof(double) * 8 * R0, s));
  ConvState st{d_state, d_state + R0, d_state + 2 * R0, b.d_done, d_niter};
  double* d_crossA = d_state + 3 * R0;   // finalised scalars: cross / violation of the row half
  double* d_crossB = d_state + 4 * R0;   // ... of the column half
  b.gram[0] = d_gram;                                // Gram of Fr (e.g. W^T W), by rid
  b.gram[1] = d_gram + (size_t)R0 * KMAX * KMAX;     // Gram of Fc (e.g. H H^T), by rid
  b.scal_part[0] = d_scal_part;
  b.scal_part[1] = d_scal_part + (size_t)R0 * ops.chunks_cap;
  b.gram_part[0] = d_gram_part;
  b.gram_part[1] = d_gram_part + ops.gram_part_elems;

  b.h_gidx = static_cast<int*>(h->host_buf("solve.gather_idx", sizeof(int) * 3 * (size_t)R0 * b.GATHER_SLOTS));
  b.d_gidx = static_cast<int*>(h->dev_buf("solve.gather_didx", sizeof(int) * 3 * (size_t)R0 * b.GATHER_SLOTS));
  if (!b.h_gidx || !b.d_gidx) return -2;

  // working factors start in the caller's buffers; compaction ping-pongs them with the alternates and parks the
  // final factors of the restarts it removes in the result slabs (original offsets)
  T* alt[2] = {};
  T* res[2] = {};
  bool compacted = false;
  auto gram_after = [&](int side) -> int {   // Gram of a factor the update kernel just wrote
    return ops.fused_gram ? 0 : ops.gram(side, b.bm());
  };

  const double normX2 = v.sum_sq;
  double* d_cd_err = d_state + 7 * R0;
  // CD: ||X - Fr^T Fc||_F of the restarts still packed, in the trace form, into d_cd_err
  auto cd_final_error = [&]() -> int {
    int* d_zero = static_cast<int*>(h->dev_buf("solve.zero", sizeof(int) * 2 * R0));
    if (!d_zero) return -2;
    CNMF_CUDA_CHECK(cudaMemsetAsync(d_zero, 0, sizeof(int) * 2 * R0, s));
    BatchMeta bm0{b.d_off, b.d_k, b.d_rid, d_zero, b.R, b.kp};
    CNMF_TRY(ops.grams(bm0));
    CNMF_TRY(ops.cross(io.update_cols ? 1 : 0, bm0, d_crossB));
    ConvState scratch{d_state + 5 * R0, d_state + 6 * R0, d_cd_err, d_zero, d_zero + R0};
    h->launches += 1;
    return launch_mu_check(scratch, d_crossB, b.gram[0], b.gram[1], normX2, bm0, 0, 0.0, p.max_iter, s);
  };

  std::vector<int> h_done(R0, 0);
  // Drop converged restarts from the packed arrays when that saves a GEMM tile (or >= 1/8 of the rows).
  auto maybe_compact = [&]() -> int {
    if (!io.update_cols) return 0;
    std::vector<int> f_src, f_dst, f_k, l_src, l_dst, l_k, n_rid;
    for (int sl = 0; sl < b.R; ++sl) {
      const int rid = s_rid[sl];
      if (h_done[rid]) {
        f_src.push_back(s_off[sl]); f_dst.push_back(off0[rid]); f_k.push_back(s_k[sl]);
      } else {
        l_src.push_back(s_off[sl]); l_k.push_back(s_k[sl]); n_rid.push_back(rid);
      }
    }
    const int new_rows = pack_offsets(l_k, l_dst);   // rows of the packed live set
    const int SK = b.SK, tr = Ops::tile_rows;
    if (new_rows == SK || new_rows == 0) return 0;
    const bool saves_tile = (new_rows + tr - 1) / tr < (SK + tr - 1) / tr;
    if (!saves_tile && new_rows > SK - SK / 8) return 0;
    if (!mu) CNMF_TRY(cd_final_error());    // restarts leaving the packed arrays get their ||X - WH||_F now
    if (!alt[0]) {
      const std::string tag = Ops::buf_tag;
      const size_t nr = (size_t)SK0 * v.ld_r * sizeof(T), nc = (size_t)SK0 * v.ld_c * sizeof(T);
      alt[0] = static_cast<T*>(h->dev_buf("solve.alt.Fr" + tag, nr));
      alt[1] = static_cast<T*>(h->dev_buf("solve.alt.Fc" + tag, nc));
      res[0] = static_cast<T*>(h->dev_buf("solve.res.Fr" + tag, nr));
      res[1] = static_cast<T*>(h->dev_buf("solve.res.Fc" + tag, nc));
      if (!alt[0] || !alt[1] || !res[0] || !res[1]) return -2;
    }
    CNMF_TRY(b.gather(b.F[0], res[0], f_src, f_dst, f_k, v.ld_r));    // finished restarts -> result slabs
    CNMF_TRY(b.gather(b.F[1], res[1], f_src, f_dst, f_k, v.ld_c));
    CNMF_TRY(b.gather(b.F[0], alt[0], l_src, l_dst, l_k, v.ld_r));    // live restarts -> packed front of the alternates
    CNMF_TRY(b.gather(b.F[1], alt[1], l_src, l_dst, l_k, v.ld_c));
    CNMF_TRY(ops.compact(l_src, l_dst, l_k));
    std::swap(b.F[0], alt[0]);
    std::swap(b.F[1], alt[1]);
    b.R = (int)l_k.size();
    b.SK = new_rows;
    std::copy(l_dst.begin(), l_dst.end(), s_off.begin());
    std::copy(l_k.begin(), l_k.end(), s_k.begin());
    std::copy(n_rid.begin(), n_rid.end(), s_rid.begin());
    CNMF_TRY(upload_slots());      // synchronises the stream: the gather ring can be reused
    b.gslot = 0;
    CNMF_TRY(ops.repack());
    compacted = true;
    return 0;
  };

  auto poll_all_done = [&]() -> int {   // 1 = all done, 0 = not yet, <0 error
    CNMF_CUDA_CHECK(cudaMemcpyAsync(h_done.data(), b.d_done, sizeof(int) * R0, cudaMemcpyDeviceToHost, s));
    CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
    for (int sl = 0; sl < b.R; ++sl)
      if (!h_done[s_rid[sl]]) return maybe_compact();
    return 1;
  };

  CNMF_TRY(ops.start());
  if (mu) {
    // ---------------- multiplicative update (sklearn _nmf.py:726-888) ----------------
    CNMF_TRY(ops.gram(1, b.bm()));
    CNMF_TRY(ops.gram(0, b.bm()));
    // the starting error from <NUM_c, Fc>, or on a refit from <NUM_r, Fr>: H fixed, X H^T is computed once (sklearn
    // caches XHt, _nmf.py:537-548)
    const int first = io.update_cols ? 1 : 0;
    CNMF_TRY(ops.gemm(first));
    CNMF_TRY(ops.cross(first, b.bm(), d_crossB));
    h->launches += 1;
    CNMF_TRY(launch_mu_check(st, d_crossB, b.gram[0], b.gram[1], normX2, b.bm(), 0, p.tol, p.max_iter, s));

    // one iteration = GEMM, update(+Gram), GEMM, update(+Gram): the float update kernels leave the finalised Gram of
    // the factor they wrote (and, at check iterations, <NUM, F>) behind, so nothing else sits between the GEMMs
    for (int it = 1; it <= p.max_iter; ++it) {
      const bool check = (p.tol > 0 && it % 10 == 0) || it == p.max_iter;
      if (io.update_cols) {
        CNMF_TRY(ops.gemm(0));
        CNMF_TRY(ops.update(0, true, false, nullptr));
        CNMF_TRY(gram_after(0));
        CNMF_TRY(ops.gemm(1));
        CNMF_TRY(ops.update(1, true, check, d_crossB));
        CNMF_TRY(gram_after(1));
      } else {
        CNMF_TRY(ops.update(0, check, check, d_crossB));
        if (check) CNMF_TRY(gram_after(0));
      }
      if (check) {
        h->launches += 1;
        // at it == max_iter with it % 10 != 0 sklearn does not test; tol = -1 makes the test never fire
        const double tol_eff = (p.tol > 0 && it % 10 == 0) ? p.tol : -1.0;
        CNMF_TRY(launch_mu_check(st, d_crossB, b.gram[0], b.gram[1], normX2, b.bm(), it, tol_eff, p.max_iter, s));
        const int all = poll_all_done();
        if (all < 0) return all;
        if (all) break;
      }
    }
  } else {
    // ---------------- coordinate descent (sklearn _nmf.py:399-518, shuffle=False) ----------------
    const int poll_every = 4;
    for (int it = 1; it <= p.max_iter; ++it) {
      if (it == 1) CNMF_TRY(ops.gram(1, b.bm()));     // afterwards: left behind by the sweep over Fc
      if (io.update_cols || it == 1) CNMF_TRY(ops.gemm(0));
      CNMF_TRY(ops.update(0, io.update_cols, true, d_crossA));
      if (io.update_cols) {
        CNMF_TRY(gram_after(0));
        CNMF_TRY(ops.gemm(1));
        CNMF_TRY(ops.update(1, true, true, d_crossB));
        CNMF_TRY(gram_after(1));
      }
      h->launches += 1;
      CNMF_TRY(launch_cd_check(st, d_crossA, io.update_cols ? d_crossB : nullptr, b.bm(), it, p.tol, p.max_iter, s));
      if (it % poll_every == 0 || it == p.max_iter) {
        const int all = poll_all_done();
        if (all < 0) return all;
        if (all) break;
      }
    }
  }

  // final ||X - Fr^T Fc||_F: MU holds it in st.last from each restart's last check; CD tracks the
  // projected-gradient violation instead, so the trace form is evaluated here for the restarts still
  // packed (those compacted away earlier were evaluated just before they left)
  double* d_err = st.last;
  if (!mu) {
    CNMF_TRY(cd_final_error());
    d_err = d_cd_err;
  }

  // ---- put every restart's final factors back at its original rows of the caller's buffers
  if (compacted) {
    const int R = b.R;
    std::vector<int> so(s_off.begin(), s_off.begin() + R), ko(s_k.begin(), s_k.begin() + R), dof(R);
    for (int sl = 0; sl < R; ++sl) dof[sl] = off0[s_rid[sl]];
    CNMF_TRY(b.gather(b.F[0], res[0], so, dof, ko, v.ld_r));
    CNMF_TRY(b.gather(b.F[1], res[1], so, dof, ko, v.ld_c));
    CNMF_CUDA_CHECK(cudaMemcpyAsync(io.Fr, res[0], (size_t)SK0 * v.ld_r * sizeof(T), cudaMemcpyDeviceToDevice, s));
    CNMF_CUDA_CHECK(cudaMemcpyAsync(io.Fc, res[1], (size_t)SK0 * v.ld_c * sizeof(T), cudaMemcpyDeviceToDevice, s));
  }

  io.n_iter.assign(R0, 0);
  io.last.assign(R0, 0.0);
  io.err.assign(R0, 0.0);
  CNMF_CUDA_CHECK(cudaMemcpyAsync(io.n_iter.data(), d_niter, sizeof(int) * R0, cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaMemcpyAsync(io.last.data(), st.last, sizeof(double) * R0, cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaMemcpyAsync(io.err.data(), d_err, sizeof(double) * R0, cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
  // per-launch event pairs are folded into the totals lazily (cnmf_profile_get*), not inside the solve
  return 0;
}

}  // namespace

int solve_batched(cnmf_handle_s* h, const DataView& v, SolveIO<float>& io, const cnmf_nmf_params& p, cudaStream_t s) {
  CNMF_REQUIRE(v.form != Form::FP64, "solve: float64 datasets solve with float64 factors");
  if (p.beta_loss != CNMF_LOSS_FROBENIUS) return solve_batched_beta(h, v, io, p, s);
  return solve_frobenius<F32Ops>(h, v, io, p, s);
}

int solve_batched(cnmf_handle_s* h, const DataView& v, SolveIO<double>& io, const cnmf_nmf_params& p, cudaStream_t s) {
  CNMF_REQUIRE(v.form == Form::FP64 && v.X64, "solve: the float64 solver needs a float64 dataset");
  CNMF_REQUIRE(p.beta_loss == CNMF_LOSS_FROBENIUS, "solve: float64 datasets support beta_loss = frobenius only");
  return solve_frobenius<F64Ops>(h, v, io, p, s);
}

}  // namespace cnmf
