// The Frobenius batched solve (MU and CD): what its driver (solve_frobenius, nmf_engine.cu) shares with the ops of the
// factor element type -- F32Ops (nmf_engine.cu) for the float forms, F64Ops (nmf_f64.cu) for FP64.
//
// The driver owns the schedule: slot tables, convergence checks and polls, compaction, the final error and the
// copy-back.  The ops own what differs by precision: the products, the update, Gram and cross launches, their block
// plans, and the float forms' operand pieces.  Side 0 is the row factor Fr, side 1 the column factor Fc; NUM[side] is
// the product its update reads (NUM_r = Fc * X^T, NUM_c = Fr * X).
#pragma once
#include <vector>

#include "engine.h"
#include "nmf_kernels.cuh"

namespace cnmf {

template <class T>
struct FroSolve {
  cnmf_handle_s* h;
  const DataView& v;
  SolveIO<T>& io;
  cudaStream_t s;
  int R0 = 0, SK0 = 0, kp = 0;     // restarts / packed rows of the whole batch; Gram stride
  int R = 0, SK = 0;               // live slots / live packed rows
  int *d_off = nullptr, *d_k = nullptr, *d_rid = nullptr, *d_done = nullptr, *d_ticket = nullptr;
  double* gram[2] = {};            // finalised K x K Gram of each factor, by rid
  double* gram_part[2] = {};       // per-block Gram partials of each factor
  double* scal_part[2] = {};       // per-block partials of the cross / violation scalar of each side's update
  T* F[2] = {};                    // working factors: the caller's buffers, or the compaction alternates
  T* NUM[2] = {};

  int n(int side) const { return side ? v.n_c : v.n_r; }
  int ld(int side) const { return side ? v.ld_c : v.ld_r; }
  BatchMeta bm() const { return BatchMeta{d_off, d_k, d_rid, d_done, R, kp}; }

  // gathers kk.size() restarts' rows of ld elements E: dst[dst_off[i] ..] <- src[src_off[i] ..]; nothing when src or dst
  // is null.  Index triples go through a pinned ring of GATHER_SLOTS entries so that consecutive gathers need no host
  // synchronisation in between; the ring is reset (gslot = 0) after each synchronisation of the stream.
  static constexpr int GATHER_SLOTS = 12;
  int* h_gidx = nullptr;
  int* d_gidx = nullptr;
  int gslot = 0;
  template <class E>
  int gather(const E* src, E* dst, const std::vector<int>& so, const std::vector<int>& dof, const std::vector<int>& kk,
             int ld);
};

}  // namespace cnmf
