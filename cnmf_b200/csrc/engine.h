// Host-side engine objects behind the C ABI (handle, dataset, workspace).
#pragma once
#include <cuda_runtime.h>

#include <map>
#include <string>
#include <vector>

#include "../../include/cnmf_b200.h"
#include "common.cuh"
#include "gemm.h"

namespace cnmf {

// How a dense dataset feeds the tensor cores, decided once per dataset (dataset_resolve_form):
//   FP32        X, Xt                        factor used as is        gemm_fp32_simt
//   TF32        X, X_hi / X_lo, Xt_hi / lo   tf32 hi / lo pieces      gemm_tf32x3, 3 passes
//   TF32_EXACT  X, C = X_hi, C^T = Xt_hi     tf32 pieces of F * scale gemm_tf32x3, exact B, 2 passes
//   F16_EXACT   X, C, C^T as fp16            fp16 pieces of F * scale gemm_tf32x3, f16 = 1
//   FP64        X64 only (fp64, row-major)    factor in fp64            gemm_f64 (DMMA), both orientations
// The exact forms hold X = diag(row_scale) C diag(col_scale) with C small non-negative integers.
enum class Form { FP32, TF32, TF32_EXACT, F16_EXACT, FP64 };
inline bool form_exact(Form f) { return f == Form::TF32_EXACT || f == Form::F16_EXACT; }

}  // namespace cnmf

struct cnmf_handle_s {
  int device = 0;
  int sm_count = cnmf::NUM_SMS;
  long long launches = 0;                       // kernels launched by this library (bench: gpu_launches)
  // optional per-launch timing of the hot kernels (batched GEMM, fused update) with CUDA events on the
  // launching stream; read back by bench.py for the roofline lines
  bool profile = false;
  std::vector<cudaEvent_t> ev_pool;
  struct Pending { int begin; int end; int cls; double work; };   // indices of the start / end events in ev_pool
  // a profiled launch that directly follows another profiled launch (no other counted launch in between, same
  // stream) takes the predecessor's end event as its start: one event record per kernel boundary instead of two
  int prof_last_end = -1;
  long long prof_last_launches = -1;
  cudaStream_t prof_last_stream = nullptr;
  std::vector<Pending> ev_pending;
  size_t ev_used = 0;
  // kernel classes: 0 = batched GEMM (work = algorithmic FLOPs), 1 = fused update kernels (work = algorithmic bytes),
  // 2 = sparse products csc_project (work = algorithmic bytes), 3 = fp64 GEMM of the NNDSVD starts (work = FLOPs),
  // 4 = fp64 GEMM of the float64 solver (work = FLOPs), 5 = fp64 GEMMs of the Harmony ridge correction (work = FLOPs)
  static constexpr int PROF_CLASSES = 6;
  double prof_ms[PROF_CLASSES] = {}, prof_work[PROF_CLASSES] = {};
  long long prof_launches[PROF_CLASSES] = {};
  int nndsvd_chunk_restarts = 0;                // > 0: at most this many restarts per chunk of the NNDSVD starts
  double t_rng_ms = 0, t_h2d_ms = 0, t_solve_ms = 0, t_d2h_ms = 0;   // host wall-clock phases of the last factorize
  int prof_begin(cudaStream_t s, double work, int cls = 0);    // start event (recorded or shared); returns slot or -1
  void prof_end(cudaStream_t s, int slot);
  void prof_collect();                              // after a stream sync: fold pending pairs into the totals
  std::map<std::string, std::pair<void*, size_t>> ws;   // named grow-only device buffers
  std::map<std::string, std::pair<void*, size_t>> pinned;  // named grow-only pinned host buffers

  // size-keyed pool of dataset buffers: cudaMalloc / cudaFree of several 160 MB arrays per dataset
  // cost tens of ms (cudaFree synchronises); datasets of a repeated shape reuse their buffers
  std::multimap<size_t, void*> pool;
  size_t pool_bytes = 0;
  void* pool_take(size_t bytes);
  void pool_give(void* p, size_t bytes);
  void* dev_buf(const std::string& name, size_t bytes);      // nullptr on failure (error set)
  void* host_buf(const std::string& name, size_t bytes);
  void release_all();
};

// A cells x genes matrix resident on the device in the forms the two GEMM orientations need.
//   X   (n_rows x ld_c)  : K-major over columns  -> B operand of  NUM_rows = F_cols * X^T
//   Xt  (n_cols x ld_r)  : K-major over rows     -> B operand of  NUM_cols = F_rows * X
// The resident operands follow the dataset's form (cnmf::Form); X is always kept (column operations, derived datasets).
struct cnmf_dataset_s {
  cnmf_handle_s* h = nullptr;
  int n_rows = 0, n_cols = 0;
  int ld_c = 0;   // row stride of X  (>= n_cols)
  int ld_r = 0;   // row stride of Xt (>= n_rows)
  int precision = 0;                        // CNMF_PRECISION_* the dataset was created with
  cnmf::Form form = cnmf::Form::FP32;
  float *X = nullptr, *Xt = nullptr;
  float *X_hi = nullptr, *X_lo = nullptr, *Xt_hi = nullptr, *Xt_lo = nullptr;
  // exact forms (what HVG-normalised counts and TPM are): X_hi / Xt_hi hold C / C^T -- exactly representable in tf32, no
  // lo piece -- and the scales are folded into the factor pieces / applied to the GEMM output.  On F16_EXACT, X_h16 /
  // Xt_h16 hold C / C^T as fp16 (same shapes and element strides) and the fp32 copies are released.  Either scale may
  // be nullptr (= 1); both are nullptr on the other forms.
  void *X_h16 = nullptr, *Xt_h16 = nullptr;
  float *row_scale = nullptr, *col_scale = nullptr;    // lengths ld_r / ld_c, zero padded
  double sum = 0.0, sum_sq = 0.0;
  // sparse datasets (cnmf_dataset_create_csc): X stays canonical CSC and none of the dense forms above exist
  // (X == nullptr).  The form and the scales are still detected, so that cnmf_dataset_from_columns builds the same
  // dense dataset from it as from the dense form of the matrix.  col_sums: per column sum(x) then sum(x^2), fp64.
  // Columns are cut into chunks of at most CSC_CHUNK entries (item_ptr: first chunk of each column, n_cols + 1):
  // csc_project_kernel gives one warp to a chunk.
  bool sparse = false;
  long long nnz = 0;
  long long* col_ptr = nullptr;
  int* row_idx = nullptr;
  float* vals = nullptr;
  double* col_sums = nullptr;
  int* item_ptr = nullptr;
  int n_items = 0;
  // float64 datasets (precision CNMF_PRECISION_FP64, form FP64): X64 is the only resident form, n_rows x ld_c, padding
  // zeroed; X and every other array above stay nullptr
  double* X64 = nullptr;
  std::vector<std::pair<void*, size_t>> owned;

  // every creator starts here: shape, padded strides and the creation precision
  cnmf_dataset_s(cnmf_handle_s* h_, int rows, int cols, int precision_)
      : h(h_), n_rows(rows), n_cols(cols), ld_c(cnmf::pad_ld(cols)), ld_r(cnmf::pad_ld(rows)), precision(precision_) {}
};

namespace cnmf {

inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

struct Operand {     // a K-major matrix as the GEMM sees it
  const float* full;
  const float* hi;     // tf32 hi piece, or the exact integer matrix C (as fp16 on F16_EXACT)
  const float* lo;
  int rows, cols, ld;
};

// View of a dataset for one solve: "rows" are the items of the row factor (Fr: SK x n_r),
// "cols" the items of the column factor (Fc: SK x n_c).  transposed swaps the roles.
struct DataView {
  Operand B_rows;   // n_r x n_c : B operand when updating Fr (reduction over n_c)
  Operand B_cols;   // n_c x n_r : B operand when updating Fc (reduction over n_r)
  int n_r, n_c, ld_r, ld_c;
  double sum, sum_sq;
  Form form;                // FP32 on sparse datasets: their solves run no GEMM and make no pieces
  const float* scale_r;     // per row-item scale (length ld_r) or nullptr
  const float* scale_c;     // per column-item scale (length ld_c) or nullptr
  const double* X64;        // FP64: the dataset's fp64 X (n_rows x ld_c); both products read it through gemm_f64
  bool transposed;          // rows are the dataset's columns
};

DataView make_view(const cnmf_dataset_s* d, bool transposed);

// C = A * B^T in the given form: g holds the shape, C and split-K; this fills the operands (factor A in fp32, its pieces
// and tile scales from make_pieces; out_scale on the output columns of the exact forms) and launches the GEMM
int form_gemm(Form form, GemmArgs g, const float* A, const float* A_hi, const float* A_lo, const float* a_tile_scale,
              const Operand& B, const float* out_scale, cudaStream_t s);
// split-K plan of one of the solver's two products on a view: splits from gemm_fixed_splits (a function of the
// reduction length only), slices of SK rows at the output's row stride
struct GemmPlan {
  int splits;
  long long split_stride;   // elements
};
GemmPlan view_gemm_plan(const DataView& v, int side, int SK);
// one of the solver's two products on a view, counted and profiled as a batched GEMM:
//   side 0: NUM_r = Fc * B_rows^T (SK x ld_r per slice, output scale scale_r); F = Fc (SK x ld_c)
//   side 1: NUM_c = Fr * B_cols^T (SK x ld_c per slice, output scale scale_c); F = Fr (SK x ld_r)
// F_hi / F_lo / tile_scale: F's pieces for the view's form (make_pieces with the other side's scale)
int view_gemm(cnmf_handle_s* h, const DataView& v, int side, const float* F, const float* F_hi, const float* F_lo,
              const float* tile_scale, int SK, float* C, const GemmPlan& plan, cudaStream_t s);
// operand pieces of F diag(scale) (rows x ld, n valid columns) for the form: none, tf32 split, or two fp16 pieces with
// tile scales (rows x ceil(ld / 512)); at most one launch
int make_pieces(Form form, const float* F, int rows, int n, int ld, const float* scale, float* hi, float* lo,
                float* tile_scale, cudaStream_t s);

// ---- datasets: capi.cu
int dataset_alloc(cnmf_dataset_s* d, float** p, size_t elems);   // owned by d, from the handle's pool if one fits
// form, operands and sums from d->X (resident, padding zeroed); exact: inherited (scales set), no detection
int dataset_finish(cnmf_dataset_s* d, cudaStream_t s, bool exact = false);
// d->form from the creation precision and, where it allows an exact form and `exact` is not yet known, exact-count
// detection on the dense or CSC matrix (synchronises)
int dataset_resolve_form(cnmf_dataset_s* d, bool exact, cudaStream_t s);
// params.precision must be FP32, FP64 on a float64 dataset or, for every tensor-core precision, TF32X3
int check_params_precision(const cnmf_dataset_s* d, const cnmf_nmf_params* p);
// -3 with a message naming the float64 entry point `what`_f64 when d is a float64 dataset (float entry points)
int require_f32(const cnmf_dataset_s* d, const char* what);
// -3 with a message naming the float entry point `what` when d is not a float64 dataset (_f64 entry points)
int require_f64(const cnmf_dataset_s* d, const char* what);

// one batched solve: T = float on the float forms, double on FP64
template <class T>
struct SolveIO {
  int R = 0;
  std::vector<int> ks;      // per restart
  // packed device factors (SK x ld) in the dataset's element type: row factor Fr (e.g. W^T), column factor Fc (e.g. H).
  // The solver makes their operand pieces itself.
  T *Fr = nullptr, *Fc = nullptr;
  bool update_cols = true;  // false: Fc fixed (refit)
  // the row product, computed by the caller (refits of sparse datasets: NUM_r = Fc * X^T, SK x ld_r, one split).
  // Requires update_cols = false; the solver then runs no GEMM and reads no B operand.  Float forms only.
  const float* num_rows = nullptr;
  std::vector<int> n_iter;  // out
  std::vector<double> last; // out: last convergence statistic (mu: error, cd: violation)
  std::vector<double> err;  // out: final ||X - Fr^T Fc||_F
};

// Runs the batched solver in place on io.Fr / io.Fc: float factors on the float forms (beta_loss KL / IS go to
// solve_batched_beta), double factors on FP64 (Frobenius only).  The Frobenius solves of both share one driver (solve.h).
int solve_batched(cnmf_handle_s* h, const DataView& v, SolveIO<float>& io, const cnmf_nmf_params& p, cudaStream_t s);
int solve_batched(cnmf_handle_s* h, const DataView& v, SolveIO<double>& io, const cnmf_nmf_params& p, cudaStream_t s);
// beta_loss = kullback-leibler / itakura-saito (nmf_beta.cu); reached through solve_batched
int solve_batched_beta(cnmf_handle_s* h, const DataView& v, SolveIO<float>& io, const cnmf_nmf_params& p,
                       cudaStream_t s);
// out[0] = sum(X), out[1] = sum(X^2) of a float64 dataset matrix, fp64 in an order fixed by the shape (synchronises)
int matrix_sums_f64(cnmf_handle_s* h, const double* X, int rows, int cols, int ld, double* out_host, cudaStream_t s);
// p[r, j] = v for r < rows, j < n (row stride ld); does not synchronise
int fill_f64(double* p, double v, int rows, int n, int ld, cudaStream_t s);
int matrix_min(cnmf_handle_s* h, const float* X, int rows, int cols, int ld, float* out_host, cudaStream_t s);
// the streaming beta-divergence kernels read X in both orientations in full fp32: builds d->Xt if the dataset
// (tf32x3 mode) only holds the pieces
int dataset_ensure_full_transpose(cnmf_dataset_s* d, cudaStream_t s);

// ---- sparse (CSC) datasets: sparse_kernels.cu
constexpr int CSC_CHUNK = 4096;     // most entries of a column one warp of csc_project_kernel reduces
// -3 with a message naming the entry point when d is sparse or float64
int require_dense(const cnmf_dataset_s* d, const char* what);
// out (k x ld, first n_cols columns written) = U^T * X with U staged on the device as n_rows x kp floats
// (kp = k rounded up to 4, zero padded); fp64 products and sums in a fixed order, rounded to fp32 once
int csc_project(const cnmf_dataset_s* d, const float* U, int k, int kp, float* out, int ld, cudaStream_t s);
// U (n x kp) <- F^T for a device matrix F (k x ld), zero in the columns k..kp-1: the layout csc_project reads
int stage_rows(cnmf_handle_s* h, const float* F, int k, int n, int ld, int kp, float* U, cudaStream_t s);
// per column sum(x), sum(x^2) into d->col_sums and the dataset totals into d->sum / d->sum_sq (synchronises)
int csc_col_stats(cnmf_dataset_s* d, cudaStream_t s);
// exact-count detection on the stored entries: the test dataset_resolve_form runs on the dense form; sets the scale of
// an exact matrix (synchronises)
int csc_detect_exact(cnmf_dataset_s* d, cudaStream_t s, bool* exact);
// dst (n_rows x ld_dst, zeroed by the caller)[:, c] = X[:, cols[c]] * scale[c]
int csc_gather_cols(const cnmf_dataset_s* d, const int* cols, const float* scale, int n_cols, float* dst, int ld_dst,
                    cudaStream_t s);
// device totals (n_rows): fp64 row sums; col_sums (2 x n_cols): per column sum(v), sum(v^2) of v = x * target_sum /
// (row total), 0 for a row without counts.  Fixed reduction order, no floating-point atomics.  Does not synchronise.
int csc_tpm_sums(const cnmf_dataset_s* d, double target_sum, double* totals, double* col_sums, cudaStream_t s);
// a temporary device array outside the handle's pool, freed when it goes out of scope: the owner synchronises the
// stream that uses it first
struct DeviceTemp {
  void* p = nullptr;
  DeviceTemp() = default;
  DeviceTemp(const DeviceTemp&) = delete;
  DeviceTemp& operator=(const DeviceTemp&) = delete;
  ~DeviceTemp() {
    if (p) cudaFree(p);
  }
  int alloc(size_t bytes, const std::string& what) {
    const cudaError_t e = cudaMalloc(&p, bytes < 256 ? 256 : bytes);
    if (e != cudaSuccess) {
      p = nullptr;
      set_last_error(what + ": cudaMalloc(" + std::to_string(bytes) + " bytes) failed: " + cudaGetErrorString(e));
      return -2;
    }
    return 0;
  }
  template <class T>
  T* as() const { return static_cast<T*>(p); }
};
// a host CSR matrix (row_ptr from 0 to nnz, col_idx strictly increasing within each row and in [0, n_cols)) checked
// before any device work: the device kernels below rely on it
int check_csr(const char* what, int n_rows, int n_cols, long long nnz, const int64_t* row_ptr, const int32_t* col_idx);
// A sparse dataset d (shape, precision, nnz and sparse set) from a canonical CSR matrix in device arrays: the canonical
// CSC arrays of d (owned by d) by a column histogram per block of CSR_ROW_BLOCK rows, a per-column scan over the
// blocks, a 64-bit scan of the column totals into d->col_ptr, and a scatter in which each row block walks its rows in
// order -- no atomic decides a position, so the row indices of a column come out increasing -- then the chunk table,
// column sums and form as cnmf_dataset_create_csc makes them.  The row block grows when the per-block count table
// (blocks x n_cols ints, freed before return) would exceed CSR_COUNT_BUDGET ints.  Synchronises.
constexpr int CSR_ROW_BLOCK = 256;
constexpr long long CSR_COUNT_BUDGET = 1LL << 25;
int csr_to_csc(cnmf_dataset_s* d, const long long* row_ptr, const int* col_idx, const float* vals, cudaStream_t s);
// rows [r0, r1) of a canonical CSR matrix into a zeroed dense matrix: X[r][col_idx[j]] = vals[j], with row_ptr[r] -
// base indexing col_idx / vals (a staged slice).  Does not synchronise.
int csr_scatter_rows(const long long* row_ptr, long long base, const int* col_idx, const float* vals, int r0, int r1,
                     float* X, int ld, cudaStream_t s);
int csr_scatter_rows(const long long* row_ptr, long long base, const int* col_idx, const double* vals, int r0, int r1,
                     double* X, int ld, cudaStream_t s);

// ---- NNDSVD starts on the device: gemm_f64.cu, nndsvd.cu
// C (M x n_out, row stride ldc) = A (M x K, row stride lda) * op(X) in fp64 for the dataset matrix X (n_rows x n_cols,
// fp32, row stride ldx): to_genes = false -> C = A X^T (K = n_cols, n_out = n_rows); true -> C = A X (K = n_rows,
// n_out = n_cols).  Reduction order depends on the shape only.  Does not synchronise.
int launch_gemm_f64(const double* A, int lda, int M, const float* X, int n_rows, int n_cols, int ldx, bool to_genes,
                    double* C, int ldc, cudaStream_t s);
// the same product for a float64 dataset matrix X (the float64 solver's NUM_r / NUM_c and the NNDSVD starts of a
// float64 dataset): same tiles, same reduction order
int launch_gemm_f64(const double* A, int lda, int M, const double* X, int n_rows, int n_cols, int ldx, bool to_genes,
                    double* C, int ldc, cudaStream_t s);
// the same product cut along its reduction into slices of k_chunk elements (a multiple of 16): slice z accumulates
// reduction elements [z * k_chunk, (z + 1) * k_chunk) in ascending order into C + z * c_split_stride.  The caller sums
// the slices in a fixed order.  Does not synchronise.
int launch_gemm_f64_split(const double* A, int lda, int M, const float* X, int n_rows, int n_cols, int ldx,
                          bool to_genes, int k_chunk, double* C, int ldc, long long c_split_stride, cudaStream_t s);
int launch_gemm_f64_split(const double* A, int lda, int M, const double* X, int n_rows, int n_cols, int ldx,
                          bool to_genes, int k_chunk, double* C, int ldc, long long c_split_stride, cudaStream_t s);
// scikit-learn's NNDSVD starting factors of every restart (ks[r], seeds[r]) for init = CNMF_INIT_NNDSVD / NNDSVDA /
// NNDSVDAR into packed padded Wt (sum ks x ld_r) and H (sum ks x ld_c); synchronises
int nndsvd_starts_dev(cnmf_dataset_s* d, int R, const int* ks, const uint32_t* seeds, int init, float* Wt, float* H,
                      cudaStream_t s);
// the same starts of a float64 dataset into fp64 Wt / H: no rounding to fp32
int nndsvd_starts_dev(cnmf_dataset_s* d, int R, const int* ks, const uint32_t* seeds, int init, double* Wt, double* H,
                      cudaStream_t s);

}  // namespace cnmf
