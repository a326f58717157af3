// Test hooks of the C ABI: one launch of the batched solver's update / Gram / <NUM, F> / piece kernels on host data
// (cnmf_update_step_host, include/cnmf_b200.h).  It builds the FactorView / BatchMeta / FusedOut the solver builds
// (nmf_engine.cu) and calls the same launch_* functions; no kernel code of its own.  cnmf_beta_step_host does the same
// for the KL / IS solver (nmf_beta.cu), cnmf_update_step_f64_host for the float64 solver (nmf_f64.cu), and
// cnmf_conv_check_host runs the convergence kernels every solver shares.  cnmf_dataset_form / cnmf_dataset_operand_host
// read what dataset creation left resident, and cnmf_dataset_gemm_host runs one of the solver's products (view_gemm)
// on a dataset, or on a sparse one the transposed refit's product (stage_rows + csc_project).
#include <algorithm>
#include <vector>

#include "engine.h"
#include "nmf_beta.h"
#include "nmf_f64.h"
#include "nmf_kernels.cuh"

using namespace cnmf;

extern "C" int cnmf_update_step_host(cnmf_handle_t h, const cnmf_update_step_args* a, void* stream) {
  CNMF_REQUIRE(h && a && a->ks && a->rids && a->done && a->F && a->gram_in, "update_step: NULL argument");
  CNMF_REQUIRE(a->n_slots >= 1 && a->n_rids >= 1 && a->n >= 1 && a->nsplit >= 1, "update_step: bad sizes");
  CNMF_REQUIRE(a->cpb_tiles == 1 || a->cpb_tiles == 2 || a->cpb_tiles == 4, "update_step: cpb_tiles must be 1, 2 or 4");
  CNMF_REQUIRE(a->solver == CNMF_SOLVER_MU || a->solver == CNMF_SOLVER_CD || a->solver == CNMF_UNIT_SOLVER_NONE,
               "update_step: unknown solver");
  CNMF_REQUIRE(a->pieces >= CNMF_UNIT_PIECES_NONE && a->pieces <= CNMF_UNIT_PIECES_F16, "update_step: unknown pieces mode");
  CNMF_REQUIRE(a->gram >= CNMF_UNIT_GRAM_NONE && a->gram <= CNMF_UNIT_GRAM_STANDALONE, "update_step: unknown Gram mode");
  CNMF_REQUIRE(a->pieces == CNMF_UNIT_PIECES_NONE || (a->pieces_hi && a->pieces_lo), "update_step: pieces buffers missing");
  CNMF_REQUIRE(a->pieces != CNMF_UNIT_PIECES_F16 || a->tile_scale, "update_step: tile_scale missing");
  CNMF_REQUIRE(a->gram == CNMF_UNIT_GRAM_NONE || a->gram_out, "update_step: gram_out missing");
  CNMF_REQUIRE(!a->want_scalar || a->scal_out, "update_step: scal_out missing");
  const bool none = a->solver == CNMF_UNIT_SOLVER_NONE;
  CNMF_REQUIRE(!none || a->gram != CNMF_UNIT_GRAM_FUSED, "update_step: no update launch to fuse the Gram into");
  CNMF_REQUIRE(a->num || (none && !a->want_scalar), "update_step: num missing");
  const int R = a->n_slots, NR = a->n_rids;
  std::vector<int> meta(3 * R + NR, 0);         // off | k | rid per slot, done per rid
  std::vector<char> seen(NR, 0);
  int SK = 0, kmax = 0;
  for (int s = 0; s < R; ++s) {
    CNMF_REQUIRE(a->ks[s] >= 1 && a->ks[s] <= KMAX, "update_step: ks must be in [1, 32]");
    CNMF_REQUIRE(a->rids[s] >= 0 && a->rids[s] < NR && !seen[a->rids[s]], "update_step: rids must be distinct and < n_rids");
    seen[a->rids[s]] = 1;
    meta[s] = SK;
    meta[R + s] = a->ks[s];
    meta[2 * R + s] = a->rids[s];
    SK += a->ks[s];
    kmax = std::max(kmax, a->ks[s]);
  }
  for (int r = 0; r < NR; ++r) meta[3 * R + r] = a->done[r];
  const int kp = kmax <= 16 ? 16 : 32;
  CNMF_REQUIRE(a->gram != CNMF_UNIT_GRAM_FUSED || kp == 16, "update_step: the fused Gram exists for kp == 16 batches only");

  cudaStream_t s = as_stream(stream);
  CNMF_CUDA_CHECK(cudaSetDevice(h->device));
  const int n = a->n, ld = pad_ld(n), n_ktiles = (ld + 511) / 512;
  const int tile = upd_tile_cols(kp);
  const int cpb = a->cpb_tiles * tile;
  const int gcpb = pick_cols_per_block(n, R, 8192, 1024, h->sm_count * 2);     // as solve_batched
  const int chunks = (n + cpb - 1) / cpb, gchunks = (n + gcpb - 1) / gcpb;
  const size_t nf = (size_t)SK * ld;
  const int RR = std::max(R, NR);              // partials: slot-indexed (update launches) or rid-indexed (the others)
  const size_t piece_bytes = a->pieces == CNMF_UNIT_PIECES_F16 ? 2 : 4;

  int* d_meta = static_cast<int*>(h->dev_buf("unit.meta", sizeof(int) * meta.size()));
  float* d_F = static_cast<float*>(h->dev_buf("unit.F", nf * 4));
  float* d_num = static_cast<float*>(h->dev_buf("unit.num", (size_t)a->nsplit * nf * 4));
  double* d_gin = static_cast<double*>(h->dev_buf("unit.gram_in", sizeof(double) * (size_t)NR * KMAX * KMAX));
  double* d_gout = static_cast<double*>(h->dev_buf("unit.gram_out", sizeof(double) * (size_t)NR * KMAX * KMAX));
  double* d_scal = static_cast<double*>(h->dev_buf("unit.scal", sizeof(double) * NR));
  double* d_gpart = static_cast<double*>(h->dev_buf("unit.gram_part", sizeof(double) * (size_t)RR * std::max(chunks, gchunks) * kp * kp));
  double* d_spart = static_cast<double*>(h->dev_buf("unit.scal_part", sizeof(double) * (size_t)RR * chunks));
  float* d_ps = static_cast<float*>(h->dev_buf("unit.piece_scale", (size_t)ld * 4));
  float* d_hi = static_cast<float*>(h->dev_buf("unit.pieces_hi", nf * piece_bytes));
  float* d_lo = static_cast<float*>(h->dev_buf("unit.pieces_lo", nf * piece_bytes));
  float* d_ts = static_cast<float*>(h->dev_buf("unit.tile_scale", sizeof(float) * (size_t)SK * n_ktiles));
  if (!d_meta || !d_F || !d_num || !d_gin || !d_gout || !d_scal || !d_gpart || !d_spart || !d_ps || !d_hi || !d_lo || !d_ts)
    return -2;
  // tickets: zeroed when first allocated, never again (the fused launches leave them at zero themselves)
  const size_t tbytes = sizeof(int) * (size_t)std::max(NR, 64);
  auto tk = h->ws.find("unit.tickets");
  const bool fresh = tk == h->ws.end() || !tk->second.first || tk->second.second < tbytes;
  int* d_ticket = static_cast<int*>(h->dev_buf("unit.tickets", tbytes));
  if (!d_ticket) return -2;
  if (fresh) CNMF_CUDA_CHECK(cudaMemsetAsync(d_ticket, 0, tbytes, s));

  CNMF_CUDA_CHECK(cudaMemcpyAsync(d_meta, meta.data(), sizeof(int) * meta.size(), cudaMemcpyHostToDevice, s));
  CNMF_CUDA_CHECK(cudaMemcpyAsync(d_F, a->F, nf * 4, cudaMemcpyHostToDevice, s));
  if (a->num) CNMF_CUDA_CHECK(cudaMemcpyAsync(d_num, a->num, (size_t)a->nsplit * nf * 4, cudaMemcpyHostToDevice, s));
  CNMF_CUDA_CHECK(cudaMemcpyAsync(d_gin, a->gram_in, sizeof(double) * (size_t)NR * KMAX * KMAX, cudaMemcpyHostToDevice, s));
  if (a->gram_out)
    CNMF_CUDA_CHECK(cudaMemcpyAsync(d_gout, a->gram_out, sizeof(double) * (size_t)NR * KMAX * KMAX, cudaMemcpyHostToDevice, s));
  if (a->want_scalar) CNMF_CUDA_CHECK(cudaMemcpyAsync(d_scal, a->scal_out, sizeof(double) * NR, cudaMemcpyHostToDevice, s));
  if (a->piece_scale) CNMF_CUDA_CHECK(cudaMemcpyAsync(d_ps, a->piece_scale, (size_t)ld * 4, cudaMemcpyHostToDevice, s));
  if (a->pieces != CNMF_UNIT_PIECES_NONE) {
    CNMF_CUDA_CHECK(cudaMemcpyAsync(d_hi, a->pieces_hi, nf * piece_bytes, cudaMemcpyHostToDevice, s));
    CNMF_CUDA_CHECK(cudaMemcpyAsync(d_lo, a->pieces_lo, nf * piece_bytes, cudaMemcpyHostToDevice, s));
  }
  if (a->pieces == CNMF_UNIT_PIECES_F16)
    CNMF_CUDA_CHECK(cudaMemcpyAsync(d_ts, a->tile_scale, sizeof(float) * (size_t)SK * n_ktiles, cudaMemcpyHostToDevice, s));

  const BatchMeta b{d_meta, d_meta + R, d_meta + 2 * R, d_meta + 3 * R, R, kp};
  const float* pscale = a->piece_scale ? d_ps : nullptr;
  const bool fused = a->gram == CNMF_UNIT_GRAM_FUSED;
  // the dataset form whose pieces the mode names
  const Form form = a->pieces == CNMF_UNIT_PIECES_TF32 ? Form::TF32
                  : a->pieces == CNMF_UNIT_PIECES_F16 ? Form::F16_EXACT : Form::FP32;
  FactorView f{};
  f.F = d_F;
  f.n = n; f.ld = ld; f.piece_scale = pscale;
  if (a->pieces == CNMF_UNIT_PIECES_TF32) { f.F_hi = d_hi; f.F_lo = d_lo; }
  if (a->pieces == CNMF_UNIT_PIECES_F16 && fused) { f.P_hi = d_hi; f.P_mid = d_lo; f.tile_scale = d_ts; f.n_ktiles = n_ktiles; }
  f.cpb = cpb; f.gcpb = gcpb;
  const long long sstride = (long long)nf;

  if (none) {
    // start of a solve: pieces of the initial factors (solve_batched: split or emit_pieces), stand-alone Gram, <NUM, F>
    CNMF_TRY(make_pieces(form, d_F, SK, n, ld, pscale, d_hi, d_lo, d_ts, s));
    if (a->gram == CNMF_UNIT_GRAM_STANDALONE) {
      CNMF_TRY(launch_gram_partial(f, b, d_gpart, s));
      CNMF_TRY(launch_finalize(d_gpart, d_gout, nullptr, nullptr, gchunks, b, s));
    }
    if (a->want_scalar) {
      CNMF_TRY(launch_cross(f, d_num, a->nsplit, sstride, b, d_spart, s));
      CNMF_TRY(launch_finalize(nullptr, nullptr, d_spart, d_scal, chunks, b, s));
    }
  } else {
    FusedOut o{};
    if (fused) { o.gram_part = d_gpart; o.gram = d_gout; }
    if (a->want_scalar) { o.scal_part = d_spart; o.scal = d_scal; }
    o.counter = d_ticket;
    const bool cd = a->solver == CNMF_SOLVER_CD;
    CNMF_TRY(cd ? launch_cd_update(f, d_num, a->nsplit, sstride, d_gin, b, a->l1, a->l2, o, s)
                : launch_mu_update(f, d_num, a->nsplit, sstride, d_gin, b, a->l1, a->l2, o, s));
    if (a->gram == CNMF_UNIT_GRAM_STANDALONE) {          // gram_after() of the solver for batches without the fused Gram
      CNMF_TRY(launch_gram_partial(f, b, d_gpart, s));
      CNMF_TRY(launch_finalize(d_gpart, d_gout, nullptr, nullptr, gchunks, b, s));
    }
    // f16 pieces: emitted by the Gram-fused launch itself, else by the stand-alone kernel after it (update() of the solver)
    if (a->pieces == CNMF_UNIT_PIECES_F16 && !fused)
      CNMF_TRY(make_pieces(form, d_F, SK, n, ld, pscale, d_hi, d_lo, d_ts, s));
  }
  h->launches += 1;

  CNMF_CUDA_CHECK(cudaMemcpyAsync(a->F, d_F, nf * 4, cudaMemcpyDeviceToHost, s));
  if (a->pieces != CNMF_UNIT_PIECES_NONE) {
    CNMF_CUDA_CHECK(cudaMemcpyAsync(a->pieces_hi, d_hi, nf * piece_bytes, cudaMemcpyDeviceToHost, s));
    CNMF_CUDA_CHECK(cudaMemcpyAsync(a->pieces_lo, d_lo, nf * piece_bytes, cudaMemcpyDeviceToHost, s));
  }
  if (a->pieces == CNMF_UNIT_PIECES_F16)
    CNMF_CUDA_CHECK(cudaMemcpyAsync(a->tile_scale, d_ts, sizeof(float) * (size_t)SK * n_ktiles, cudaMemcpyDeviceToHost, s));
  if (a->gram_out)
    CNMF_CUDA_CHECK(cudaMemcpyAsync(a->gram_out, d_gout, sizeof(double) * (size_t)NR * KMAX * KMAX, cudaMemcpyDeviceToHost, s));
  if (a->want_scalar) CNMF_CUDA_CHECK(cudaMemcpyAsync(a->scal_out, d_scal, sizeof(double) * NR, cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
  return 0;
}

// cnmf_beta_step_host: one half-step or one divergence evaluation of the KL / IS solver.  The BetaSide comes from
// beta_side on a view whose data operand is D, so the half's flags are the solver's; the launches are the solver's
// beta_row_sums / beta_update / beta_check.
extern "C" int cnmf_beta_step_host(cnmf_handle_t h, const cnmf_beta_step_args* a, void* stream) {
  CNMF_REQUIRE(h && a && a->ks && a->rids && a->done && a->D && a->F_own && a->F_other, "beta_step: NULL argument");
  CNMF_REQUIRE(a->n_slots >= 1 && a->n_rids >= 1 && a->n_items >= 1 && a->n_contract >= 1, "beta_step: bad sizes");
  CNMF_REQUIRE(a->op == CNMF_UNIT_BETA_UPDATE || a->op == CNMF_UNIT_BETA_DIVERGENCE, "beta_step: unknown op");
  CNMF_REQUIRE(a->side == CNMF_UNIT_SIDE_W || a->side == CNMF_UNIT_SIDE_H, "beta_step: unknown side");
  const bool update = a->op == CNMF_UNIT_BETA_UPDATE;
  CNMF_REQUIRE(a->loss == CNMF_LOSS_KULLBACK_LEIBLER || a->loss == CNMF_LOSS_ITAKURA_SAITO ||
                   (!update && a->loss == CNMF_LOSS_FROBENIUS), "beta_step: unknown loss");
  CNMF_REQUIRE(!update || a->loss != CNMF_LOSS_KULLBACK_LEIBLER || a->oth_sum, "beta_step: oth_sum missing");
  CNMF_REQUIRE(update || (a->last && a->totals), "beta_step: last / totals missing");
  const int R = a->n_slots, NR = a->n_rids;
  std::vector<int> meta(3 * R + NR, 0);         // off | k | rid per slot, done per rid
  std::vector<char> seen(NR, 0);
  int SK = 0, kmax = 0;
  for (int s = 0; s < R; ++s) {
    CNMF_REQUIRE(a->ks[s] >= 1 && a->ks[s] <= KMAX, "beta_step: ks must be in [1, 32]");
    CNMF_REQUIRE(a->rids[s] >= 0 && a->rids[s] < NR && !seen[a->rids[s]], "beta_step: rids must be distinct and < n_rids");
    seen[a->rids[s]] = 1;
    meta[s] = SK;
    meta[R + s] = a->ks[s];
    meta[2 * R + s] = a->rids[s];
    SK += a->ks[s];
    kmax = std::max(kmax, a->ks[s]);
  }
  for (int r = 0; r < NR; ++r) meta[3 * R + r] = a->done[r];

  cudaStream_t s = as_stream(stream);
  CNMF_CUDA_CHECK(cudaSetDevice(h->device));
  const int ld_i = pad_ld(a->n_items), ld_k = pad_ld(a->n_contract);
  const size_t n_d = (size_t)a->n_contract * ld_i, n_own = (size_t)SK * ld_i, n_oth = (size_t)SK * ld_k;
  int* d_meta = static_cast<int*>(h->dev_buf("unit.meta", sizeof(int) * meta.size()));
  float* d_D = static_cast<float*>(h->dev_buf("unit.beta_D", n_d * 4));
  float* d_own = static_cast<float*>(h->dev_buf("unit.F", n_own * 4));
  float* d_oth = static_cast<float*>(h->dev_buf("unit.beta_F_other", n_oth * 4));
  double* d_sums = static_cast<double*>(h->dev_buf("unit.beta_sums", sizeof(double) * 2 * SK));
  double* d_state = static_cast<double*>(h->dev_buf("unit.beta_state", sizeof(double) * 3 * NR));
  int* d_niter = static_cast<int*>(h->dev_buf("unit.beta_niter", sizeof(int) * NR));
  if (!d_meta || !d_D || !d_own || !d_oth || !d_sums || !d_state || !d_niter) return -2;
  CNMF_CUDA_CHECK(cudaMemcpyAsync(d_meta, meta.data(), sizeof(int) * meta.size(), cudaMemcpyHostToDevice, s));
  CNMF_CUDA_CHECK(cudaMemcpyAsync(d_D, a->D, n_d * 4, cudaMemcpyHostToDevice, s));
  CNMF_CUDA_CHECK(cudaMemcpyAsync(d_own, a->F_own, n_own * 4, cudaMemcpyHostToDevice, s));
  CNMF_CUDA_CHECK(cudaMemcpyAsync(d_oth, a->F_other, n_oth * 4, cudaMemcpyHostToDevice, s));
  CNMF_CUDA_CHECK(cudaMemsetAsync(d_sums, 0, sizeof(double) * 2 * SK, s));
  if (!update) CNMF_CUDA_CHECK(cudaMemcpyAsync(d_state + 2 * NR, a->last, sizeof(double) * NR, cudaMemcpyHostToDevice, s));

  // the view the solver would hold: the data operand of the half is D, the factors are F_own and F_other
  const bool w = a->side == CNMF_UNIT_SIDE_W;
  DataView v{};
  v.n_r = w ? a->n_items : a->n_contract;
  v.n_c = w ? a->n_contract : a->n_items;
  v.ld_r = pad_ld(v.n_r);
  v.ld_c = pad_ld(v.n_c);
  (w ? v.B_cols : v.B_rows) = Operand{d_D, nullptr, nullptr, a->n_contract, a->n_items, ld_i};
  cnmf_nmf_params p{};
  p.solver = CNMF_SOLVER_MU;
  p.beta_loss = a->loss;
  p.l1_reg_W = p.l1_reg_H = a->l1;
  p.l2_reg_W = p.l2_reg_H = a->l2;
  float* Fr = w ? d_own : d_oth;
  float* Fc = w ? d_oth : d_own;
  const BetaSide sd = beta_side(v, p, w ? BetaHalf::W : BetaHalf::H, Fr, Fc, d_sums + SK);
  const BatchMeta b{d_meta, d_meta + R, d_meta + 2 * R, d_meta + 3 * R, R, 32};
  const BetaLaunch L{h, s, SK, kmax};
  const int chunks = beta_chunks(sd);
  double* d_part = static_cast<double*>(h->dev_buf("unit.beta_part", sizeof(double) * 2 * (size_t)NR * chunks));
  if (!d_part) return -2;

  if (update) {
    const bool is = a->loss == CNMF_LOSS_ITAKURA_SAITO;
    if (!is) CNMF_TRY(beta_row_sums(L, sd.Foth, sd.n_contract, sd.ld_oth, d_sums + SK));
    CNMF_TRY(beta_update(L, is, sd, b));
    CNMF_CUDA_CHECK(cudaMemcpyAsync(a->F_own, d_own, n_own * 4, cudaMemcpyDeviceToHost, s));
    if (!is) CNMF_CUDA_CHECK(cudaMemcpyAsync(a->oth_sum, d_sums + SK, sizeof(double) * SK, cudaMemcpyDeviceToHost, s));
    CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
    return 0;
  }
  const int mode = a->loss == CNMF_LOSS_KULLBACK_LEIBLER ? ERR_KL : a->loss == CNMF_LOSS_ITAKURA_SAITO ? ERR_IS : ERR_FROB;
  const ConvState st{d_state, d_state + NR, d_state + 2 * NR, d_meta + 3 * R, d_niter};
  CNMF_TRY(beta_check(L, mode, sd, b, st, d_part, 0, 0.0, 1));
  std::vector<double> part(2 * (size_t)NR * chunks);
  CNMF_CUDA_CHECK(cudaMemcpyAsync(part.data(), d_part, sizeof(double) * part.size(), cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaMemcpyAsync(a->last, d_state + 2 * NR, sizeof(double) * NR, cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
  for (int sl = 0; sl < R; ++sl) {
    const int r = a->rids[sl];
    if (a->done[r]) continue;
    double t = 0.0, sx = 0.0;                    // beta_check_kernel's order
    for (int c = 0; c < chunks; ++c) {
      t += part[((size_t)r * chunks + c) * 2];
      sx += part[((size_t)r * chunks + c) * 2 + 1];
    }
    a->totals[2 * r] = t;
    a->totals[2 * r + 1] = sx;
  }
  return 0;
}

// the slot tables of a unit launch: meta = off | k | rid per slot, done per rid; returns SK and kmax
static int unit_slots(const int32_t* ks, const int32_t* rids, const int32_t* done, int R, int NR, const char* what,
                      std::vector<int>& meta, int* SK, int* kmax) {
  meta.assign(3 * R + NR, 0);
  std::vector<char> seen(NR, 0);
  *SK = *kmax = 0;
  for (int s = 0; s < R; ++s) {
    if (ks[s] < 1 || ks[s] > KMAX) {
      set_last_error(std::string("invalid argument: ") + what + ": ks must be in [1, 32]");
      return -1;
    }
    if (rids[s] < 0 || rids[s] >= NR || seen[rids[s]]) {
      set_last_error(std::string("invalid argument: ") + what + ": rids must be distinct and < n_rids");
      return -1;
    }
    seen[rids[s]] = 1;
    meta[s] = *SK;
    meta[R + s] = ks[s];
    meta[2 * R + s] = rids[s];
    *SK += ks[s];
    *kmax = std::max(*kmax, ks[s]);
  }
  for (int r = 0; r < NR; ++r) meta[3 * R + r] = done ? done[r] : 0;
  return 0;
}

// cnmf_update_step_f64_host: one launch of the float64 solver through its own f64_update / f64_gram / f64_cross, with
// the partial-Gram stride the solver sets (kp = kmax rounded up to 4)
extern "C" int cnmf_update_step_f64_host(cnmf_handle_t h, const cnmf_update_step_f64_args* a, void* stream) {
  CNMF_REQUIRE(h && a && a->ks && a->rids && a->done && a->F, "update_step_f64: NULL argument");
  CNMF_REQUIRE(a->n_slots >= 1 && a->n_rids >= 1 && a->n >= 1, "update_step_f64: bad sizes");
  CNMF_REQUIRE(a->op == CNMF_UNIT_F64_UPDATE || a->op == CNMF_UNIT_F64_GRAM || a->op == CNMF_UNIT_F64_CROSS,
               "update_step_f64: unknown op");
  const bool upd = a->op == CNMF_UNIT_F64_UPDATE;
  CNMF_REQUIRE(!upd || a->solver == CNMF_SOLVER_MU || a->solver == CNMF_SOLVER_CD, "update_step_f64: unknown solver");
  CNMF_REQUIRE(!upd || (a->num && a->gram_in), "update_step_f64: num / gram_in missing");
  CNMF_REQUIRE(a->op != CNMF_UNIT_F64_CROSS || (a->num && a->scal_out), "update_step_f64: num / scal_out missing");
  CNMF_REQUIRE(a->op != CNMF_UNIT_F64_GRAM || a->gram_out, "update_step_f64: gram_out missing");
  CNMF_REQUIRE(!(upd && a->want_scalar) || a->scal_out, "update_step_f64: scal_out missing");
  const int R = a->n_slots, NR = a->n_rids;
  std::vector<int> meta;
  int SK = 0, kmax = 0;
  CNMF_TRY(unit_slots(a->ks, a->rids, a->done, R, NR, "update_step_f64", meta, &SK, &kmax));
  const int kp = round_up(kmax, 4);

  cudaStream_t s = as_stream(stream);
  CNMF_CUDA_CHECK(cudaSetDevice(h->device));
  const int n = a->n, ld = pad_ld(n);
  const size_t nf = (size_t)SK * ld, gsz = (size_t)NR * KMAX * KMAX;
  const int chunks = f64_chunks(n), gchunks = f64_gram_chunks(n);
  int* d_meta = static_cast<int*>(h->dev_buf("unit.meta", sizeof(int) * meta.size()));
  double* d_F = static_cast<double*>(h->dev_buf("unit.F64", nf * 8));
  double* d_num = static_cast<double*>(h->dev_buf("unit.num64", nf * 8));
  double* d_gin = static_cast<double*>(h->dev_buf("unit.gram_in", sizeof(double) * gsz));
  double* d_gout = static_cast<double*>(h->dev_buf("unit.gram_out", sizeof(double) * gsz));
  double* d_scal = static_cast<double*>(h->dev_buf("unit.scal", sizeof(double) * NR));
  double* d_gpart = static_cast<double*>(h->dev_buf("unit.gram_part", sizeof(double) * (size_t)NR * gchunks * kp * kp));
  double* d_spart = static_cast<double*>(h->dev_buf("unit.scal_part", sizeof(double) * (size_t)NR * chunks));
  if (!d_meta || !d_F || !d_num || !d_gin || !d_gout || !d_scal || !d_gpart || !d_spart) return -2;
  CNMF_CUDA_CHECK(cudaMemcpyAsync(d_meta, meta.data(), sizeof(int) * meta.size(), cudaMemcpyHostToDevice, s));
  CNMF_CUDA_CHECK(cudaMemcpyAsync(d_F, a->F, nf * 8, cudaMemcpyHostToDevice, s));
  if (a->num) CNMF_CUDA_CHECK(cudaMemcpyAsync(d_num, a->num, nf * 8, cudaMemcpyHostToDevice, s));
  if (a->gram_in) CNMF_CUDA_CHECK(cudaMemcpyAsync(d_gin, a->gram_in, sizeof(double) * gsz, cudaMemcpyHostToDevice, s));
  if (a->gram_out) CNMF_CUDA_CHECK(cudaMemcpyAsync(d_gout, a->gram_out, sizeof(double) * gsz, cudaMemcpyHostToDevice, s));
  if (a->scal_out) CNMF_CUDA_CHECK(cudaMemcpyAsync(d_scal, a->scal_out, sizeof(double) * NR, cudaMemcpyHostToDevice, s));

  const BatchMeta b{d_meta, d_meta + R, d_meta + 2 * R, d_meta + 3 * R, R, kp};
  const F64Launch L{h, s, SK};
  const F64View f{d_F, n, ld};
  if (upd)
    CNMF_TRY(f64_update(L, a->solver == CNMF_SOLVER_CD, f, d_num, d_gin, b, a->l1, a->l2, d_spart,
                        a->want_scalar ? d_scal : nullptr));
  else if (a->op == CNMF_UNIT_F64_GRAM)
    CNMF_TRY(f64_gram(L, f, b, d_gpart, d_gout));
  else
    CNMF_TRY(f64_cross(L, f, d_num, b, d_spart, d_scal));

  CNMF_CUDA_CHECK(cudaMemcpyAsync(a->F, d_F, nf * 8, cudaMemcpyDeviceToHost, s));
  if (a->gram_out) CNMF_CUDA_CHECK(cudaMemcpyAsync(a->gram_out, d_gout, sizeof(double) * gsz, cudaMemcpyDeviceToHost, s));
  if (a->scal_out) CNMF_CUDA_CHECK(cudaMemcpyAsync(a->scal_out, d_scal, sizeof(double) * NR, cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
  return 0;
}

// cnmf_conv_check_host: one mu_check_kernel / cd_check_kernel launch (launch_mu_check / launch_cd_check) on host state;
// the state's done array is also the batch's, as in the solvers
extern "C" int cnmf_conv_check_host(cnmf_handle_t h, const cnmf_conv_check_args* a, void* stream) {
  CNMF_REQUIRE(h && a && a->ks && a->rids && a->done && a->n_iter && a->err0 && a->prev && a->last,
               "conv_check: NULL argument");
  CNMF_REQUIRE(a->n_slots >= 1 && a->n_rids >= 1, "conv_check: bad sizes");
  CNMF_REQUIRE(a->solver == CNMF_SOLVER_MU || a->solver == CNMF_SOLVER_CD, "conv_check: unknown solver");
  const bool mu = a->solver == CNMF_SOLVER_MU;
  CNMF_REQUIRE(!mu || (a->cross && a->gramA && a->gramB), "conv_check: cross / gramA / gramB missing");
  CNMF_REQUIRE(mu || a->violA, "conv_check: violA missing");
  const int R = a->n_slots, NR = a->n_rids;
  std::vector<int> meta;
  int SK = 0, kmax = 0;
  CNMF_TRY(unit_slots(a->ks, a->rids, nullptr, R, NR, "conv_check", meta, &SK, &kmax));
  meta.resize(3 * R + 2 * NR);
  for (int r = 0; r < NR; ++r) {
    meta[3 * R + r] = a->done[r];
    meta[3 * R + NR + r] = a->n_iter[r];
  }

  cudaStream_t s = as_stream(stream);
  CNMF_CUDA_CHECK(cudaSetDevice(h->device));
  const size_t gsz = (size_t)NR * KMAX * KMAX;
  int* d_meta = static_cast<int*>(h->dev_buf("unit.meta", sizeof(int) * meta.size()));
  double* d_state = static_cast<double*>(h->dev_buf("unit.conv_state", sizeof(double) * 6 * NR));
  double* d_gram = static_cast<double*>(h->dev_buf("unit.conv_gram", sizeof(double) * 2 * gsz));
  if (!d_meta || !d_state || !d_gram) return -2;
  double *d_err0 = d_state, *d_prev = d_state + NR, *d_last = d_state + 2 * NR;
  double *d_x = d_state + 3 * NR, *d_vb = d_state + 4 * NR;
  CNMF_CUDA_CHECK(cudaMemcpyAsync(d_meta, meta.data(), sizeof(int) * meta.size(), cudaMemcpyHostToDevice, s));
  CNMF_CUDA_CHECK(cudaMemcpyAsync(d_err0, a->err0, sizeof(double) * NR, cudaMemcpyHostToDevice, s));
  CNMF_CUDA_CHECK(cudaMemcpyAsync(d_prev, a->prev, sizeof(double) * NR, cudaMemcpyHostToDevice, s));
  CNMF_CUDA_CHECK(cudaMemcpyAsync(d_last, a->last, sizeof(double) * NR, cudaMemcpyHostToDevice, s));
  CNMF_CUDA_CHECK(cudaMemcpyAsync(d_x, mu ? a->cross : a->violA, sizeof(double) * NR, cudaMemcpyHostToDevice, s));
  if (mu) {
    CNMF_CUDA_CHECK(cudaMemcpyAsync(d_gram, a->gramA, sizeof(double) * gsz, cudaMemcpyHostToDevice, s));
    CNMF_CUDA_CHECK(cudaMemcpyAsync(d_gram + gsz, a->gramB, sizeof(double) * gsz, cudaMemcpyHostToDevice, s));
  } else if (a->violB) {
    CNMF_CUDA_CHECK(cudaMemcpyAsync(d_vb, a->violB, sizeof(double) * NR, cudaMemcpyHostToDevice, s));
  }

  int* d_done = d_meta + 3 * R;
  const BatchMeta b{d_meta, d_meta + R, d_meta + 2 * R, d_done, R, round_up(kmax, 4)};
  const ConvState st{d_err0, d_prev, d_last, d_done, d_done + NR};
  h->launches += 1;
  if (mu) CNMF_TRY(launch_mu_check(st, d_x, d_gram, d_gram + gsz, a->normX2, b, a->it, a->tol, a->max_iter, s));
  else CNMF_TRY(launch_cd_check(st, d_x, a->violB ? d_vb : nullptr, b, a->it, a->tol, a->max_iter, s));

  CNMF_CUDA_CHECK(cudaMemcpyAsync(meta.data(), d_meta, sizeof(int) * meta.size(), cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaMemcpyAsync(a->err0, d_err0, sizeof(double) * NR, cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaMemcpyAsync(a->prev, d_prev, sizeof(double) * NR, cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaMemcpyAsync(a->last, d_last, sizeof(double) * NR, cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
  for (int r = 0; r < NR; ++r) {
    a->done[r] = meta[3 * R + r];
    a->n_iter[r] = meta[3 * R + NR + r];
  }
  return 0;
}

static_assert((int)Form::FP32 == CNMF_FORM_FP32 && (int)Form::TF32 == CNMF_FORM_TF32 &&
                  (int)Form::TF32_EXACT == CNMF_FORM_TF32_EXACT && (int)Form::F16_EXACT == CNMF_FORM_F16_EXACT &&
                  (int)Form::FP64 == CNMF_FORM_FP64,
              "CNMF_FORM_* mirror cnmf::Form");

extern "C" int cnmf_dataset_form(cnmf_dataset_t d) {
  CNMF_REQUIRE(d, "dataset_form: NULL dataset");
  return (int)d->form;
}

extern "C" int cnmf_dataset_operand_host(cnmf_dataset_t d, int which, void* out_host, long long bytes) {
  CNMF_REQUIRE(d && out_host, "dataset_operand: NULL argument");
  const long long nx = (long long)d->n_rows * d->ld_c, nxt = (long long)d->n_cols * d->ld_r;
  const void* src = nullptr;
  long long size = 0;
  switch (which) {
    case CNMF_OPERAND_X: src = d->X; size = 4 * nx; break;
    case CNMF_OPERAND_XT: src = d->Xt; size = 4 * nxt; break;
    case CNMF_OPERAND_X_HI: src = d->X_hi; size = 4 * nx; break;
    case CNMF_OPERAND_X_LO: src = d->X_lo; size = 4 * nx; break;
    case CNMF_OPERAND_XT_HI: src = d->Xt_hi; size = 4 * nxt; break;
    case CNMF_OPERAND_XT_LO: src = d->Xt_lo; size = 4 * nxt; break;
    case CNMF_OPERAND_X_H16: src = d->X_h16; size = 2 * nx; break;
    case CNMF_OPERAND_XT_H16: src = d->Xt_h16; size = 2 * nxt; break;
    case CNMF_OPERAND_ROW_SCALE: src = d->row_scale; size = 4LL * d->ld_r; break;
    case CNMF_OPERAND_COL_SCALE: src = d->col_scale; size = 4LL * d->ld_c; break;
    case CNMF_OPERAND_CSC_COL_PTR: src = d->col_ptr; size = 8LL * (d->n_cols + 1); break;
    case CNMF_OPERAND_CSC_ROW_IDX: src = d->row_idx; size = 4LL * d->nnz; break;
    case CNMF_OPERAND_CSC_VALUES: src = d->vals; size = 4LL * d->nnz; break;
    default: CNMF_REQUIRE(false, "dataset_operand: unknown array");
  }
  if (!src) {
    set_last_error("dataset_operand: this dataset does not hold that array");
    return -3;
  }
  CNMF_REQUIRE(bytes == size, "dataset_operand: bytes must be the array's size");
  CNMF_CUDA_CHECK(cudaSetDevice(d->h->device));
  CNMF_CUDA_CHECK(cudaMemcpy(out_host, src, (size_t)size, cudaMemcpyDeviceToHost));
  return 0;
}

extern "C" int cnmf_dataset_gemm_host(cnmf_dataset_t d, int transposed, int side, int SK, const float* F_host,
                                      float* out_host, int* splits_out) {
  CNMF_REQUIRE(d && splits_out && (side == 0 || side == 1) && SK >= 1, "dataset_gemm: bad arguments");
  cnmf_handle_s* h = d->h;
  if (d->sparse) {
    // the one product of the transposed refit on a CSC dataset, issued as cnmf_refit issues it: the factor in a zeroed
    // SK x ld_c buffer, staged as rows (stage_rows), csc_project into a zeroed NUM_r at stride ld_r, one slice
    if (!transposed || side != 0 || SK > KMAX) {
      set_last_error("dataset_gemm: a sparse (CSC) dataset runs only the transposed refit's product (transposed = 1, "
                     "side = 0, SK <= 32)");
      return -3;
    }
    *splits_out = 1;
    if (!out_host) return 0;
    CNMF_REQUIRE(F_host, "dataset_gemm: NULL factor");
    const DataView v = make_view(d, true);
    cudaStream_t s = nullptr;
    CNMF_CUDA_CHECK(cudaSetDevice(h->device));
    const int kp = round_up(SK, 4);
    const size_t nf = (size_t)SK * v.ld_c, nr = (size_t)SK * v.ld_r;
    float* F = static_cast<float*>(h->dev_buf("unit.gemm_F", nf * 4));
    float* U = static_cast<float*>(h->dev_buf("unit.gemm_U", (size_t)v.n_c * kp * 4));
    float* NUM = static_cast<float*>(h->dev_buf("unit.gemm_C", nr * 4));
    if (!F || !U || !NUM) return -2;
    CNMF_CUDA_CHECK(cudaMemsetAsync(F, 0, nf * 4, s));
    CNMF_CUDA_CHECK(cudaMemcpy2DAsync(F, (size_t)v.ld_c * 4, F_host, (size_t)v.n_c * 4, (size_t)v.n_c * 4, SK,
                                      cudaMemcpyHostToDevice, s));
    CNMF_CUDA_CHECK(cudaMemsetAsync(NUM, 0, nr * 4, s));
    CNMF_TRY(stage_rows(h, F, SK, v.n_c, v.ld_c, kp, U, s));
    CNMF_TRY(csc_project(d, U, SK, kp, NUM, v.ld_r, s));
    CNMF_CUDA_CHECK(cudaMemcpy2DAsync(out_host, (size_t)v.n_r * 4, NUM, (size_t)v.ld_r * 4, (size_t)v.n_r * 4, SK,
                                      cudaMemcpyDeviceToHost, s));
    CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
    return 0;
  }
  CNMF_TRY(require_dense(d, "dataset_gemm"));
  const DataView v = make_view(d, transposed != 0);
  const GemmPlan plan = view_gemm_plan(v, side, SK);
  *splits_out = plan.splits;
  if (!out_host) return 0;
  CNMF_REQUIRE(F_host, "dataset_gemm: NULL factor");
  // the factor is the other side's: Fc (n_c items, scale_c) for NUM_r, Fr (n_r items, scale_r) for NUM_c
  const int n_in = side == 0 ? v.n_c : v.n_r, ld_in = side == 0 ? v.ld_c : v.ld_r;
  const int n_out = side == 0 ? v.n_r : v.n_c, ld_out = side == 0 ? v.ld_r : v.ld_c;
  const float* piece_scale = side == 0 ? v.scale_c : v.scale_r;
  cudaStream_t s = nullptr;
  CNMF_CUDA_CHECK(cudaSetDevice(h->device));
  const size_t nf = (size_t)SK * ld_in, nc = (size_t)plan.splits * SK * ld_out;
  const int ktiles = (ld_in + 511) / 512;
  float* F = static_cast<float*>(h->dev_buf("unit.gemm_F", nf * 4));
  float* F_hi = static_cast<float*>(h->dev_buf("unit.gemm_F_hi", nf * 4));
  float* F_lo = static_cast<float*>(h->dev_buf("unit.gemm_F_lo", nf * 4));
  float* ts = static_cast<float*>(h->dev_buf("unit.gemm_tile_scale", sizeof(float) * (size_t)SK * ktiles));
  float* C = static_cast<float*>(h->dev_buf("unit.gemm_C", nc * 4));
  if (!F || !F_hi || !F_lo || !ts || !C) return -2;
  CNMF_CUDA_CHECK(cudaMemsetAsync(F, 0, nf * 4, s));
  CNMF_CUDA_CHECK(cudaMemcpy2DAsync(F, (size_t)ld_in * 4, F_host, (size_t)n_in * 4, (size_t)n_in * 4, SK,
                                    cudaMemcpyHostToDevice, s));
  CNMF_TRY(make_pieces(v.form, F, SK, n_in, ld_in, piece_scale, F_hi, F_lo, ts, s));
  h->launches += v.form == Form::FP32 ? 0 : 1;
  CNMF_TRY(view_gemm(h, v, side, F, F_hi, F_lo, ts, SK, C, plan, s));
  CNMF_CUDA_CHECK(cudaMemcpy2DAsync(out_host, (size_t)n_out * 4, C, (size_t)ld_out * 4, (size_t)n_out * 4,
                                    (size_t)plan.splits * SK, cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
  return 0;
}
