// Launches of the beta-divergence (KL / IS) solver (nmf_beta.cu), shared by solve_batched_beta and the
// cnmf_beta_step_host test hook (capi_units.cu), so that the hook runs exactly the launches the solver runs.
#pragma once
#include "engine.h"
#include "nmf_kernels.cuh"

namespace cnmf {

// One half of a beta-divergence iteration: the factor Fown (SK x ld_own) whose items are updated, walking the
// contraction dimension of the item-contiguous data D (n_contract x ldD) with the other factor Foth (SK x ld_oth).
struct BetaSide {
  const float* D;        // data, n_contract x ldD, item index contiguous
  long long ldD;
  int n_items, n_contract;
  float* Fown;           // SK x ld_own, updated in place
  int ld_own;
  const float* Foth;     // SK x ld_oth
  int ld_oth;
  const double* oth_sum; // [SK] row sums of Foth (KL denominators)
  float l1, l2;
  int zero_sum_to_one;   // H half of KL: W_sum == 0 -> 1
  int clip;              // flush values < float64 eps to zero after the update
};

// W: Fr is updated, items are the rows of the view and the data is read as X^T; H: Fc, the columns, X.
enum class BetaHalf { W, H };
// The BetaSide of one half on view v (loss, l1 / l2 of that half from p).  It decides sklearn's asymmetries: only the
// H half maps a zero KL sum to 1, and the W half flushes values below float64 eps only for IS (_nmf.py:669, 845-865).
BetaSide beta_side(const DataView& v, const cnmf_nmf_params& p, BetaHalf half, float* Fr, float* Fc,
                   const double* oth_sum);

// divergence modes of beta_error_kernel / beta_check_kernel.  FROB: plain squared residual sum over every entry.
enum { ERR_KL = 0, ERR_IS = 1, ERR_FROB = 2 };

struct BetaLaunch {     // what every launch of one batch shares
  cnmf_handle_s* h;     // counts the launches
  cudaStream_t s;
  int SK;               // packed rows
  int kpmax;            // largest K of the batch: selects the KPMAX = 8 / 16 / 32 instantiation
};

// fp64 per-block partials of the divergence: chunks per restart of a side
int beta_chunks(const BetaSide& sd);
// out[row] = sum_j F[row, j], fp64, for the SK packed rows of F (n valid columns, row stride ld)
int beta_row_sums(const BetaLaunch& L, const float* F, int n, int ld, double* out);
// one multiplicative half-step of every live restart (beta_update_kernel); KL reads sd.oth_sum
int beta_update(const BetaLaunch& L, bool is, const BetaSide& sd, const BatchMeta& b);
// divergence of every live restart: beta_error_kernel (part: [rid][chunk] {t, s}, res = t + s for KL, t - (N G - s) for
// IS, t for FROB) then beta_check_kernel at iteration it into st
int beta_check(const BetaLaunch& L, int mode, const BetaSide& sd, const BatchMeta& b, const ConvState& st, double* part,
               int it, double tol, int max_iter);

}  // namespace cnmf
