/* cnmf_b200 -- C ABI of the H100-native consensus-NMF hot path.
 *
 * Plain C, plain pointers and sizes, no torch / C++ types.  This is the boundary a reference
 * maintainer binds instead of scikit-learn at the seam
 *
 *     cNMF._nmf(X, nmf_kwargs) -> (spectra, usages)          cnmf.py:661-674
 *
 * which the reference calls from cNMF.factorize (cnmf.py:735-745, one call per (k, seed)
 * restart) and cNMF.refit_usage (cnmf.py:776-802, update_H=False), plus the numeric steps of
 * cNMF.consensus (cnmf.py:882-975).  INTEGRATION.md shows the ctypes stub.
 *
 * Conventions
 *   - every function returns 0 on success, <0 on error; cnmf_last_error() gives the message
 *     (thread-local).  -1 = invalid argument, -2 = CUDA error, -3 = unsupported.
 *   - "host" pointers are ordinary (ideally pinned) host memory; "dev" pointers are device
 *     memory of the device the handle was created on (e.g. torch.Tensor.data_ptr()).
 *   - matrices are dense row-major fp32; `ld` = row stride in elements.
 *   - `stream` is a cudaStream_t passed as void* (NULL = default stream).  Calls are
 *     synchronous with respect to the host on return unless stated otherwise.
 *   - there is NO CPU fallback: without a CUDA device every compute entry point fails.
 */
#ifndef CNMF_B200_H
#define CNMF_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CNMF_B200_ABI_VERSION 19     /* 19: cnmf_moe_grams, cnmf_moe_correct, cnmf_scale_quantile_ceiling; profile
                                      * class 5 */
#define CNMF_MAX_COMPONENTS 32          /* largest n_components per restart on the CUDA path */

typedef struct cnmf_handle_s* cnmf_handle_t;
typedef struct cnmf_dataset_s* cnmf_dataset_t;

enum { CNMF_SOLVER_MU = 0, CNMF_SOLVER_CD = 1 };            /* yaml 'solver': cnmf.py:618-631 */
/* FFMA | wgmma 3xTF32 with exact-count detection (default: 2 passes when X is scaled integers, else 3) |
 * wgmma 3xTF32 always in the general 3-pass form.  Params for a dataset created with 2 use precision 1. */
enum { CNMF_PRECISION_FP32 = 0, CNMF_PRECISION_TF32X3 = 1, CNMF_PRECISION_TF32X3_GENERAL = 2,
       /* dataset_create only: like TF32X3, but when X is recognised as scaled integer counts the big products run as
        * 2 f16 tensor-core passes (integer operand exact in fp16, factor = two fp16 pieces of its row-normalised
        * values: the same 22 significant bits as the tf32 pair at twice the MMA rate); params.precision stays TF32X3 */
       CNMF_PRECISION_F16X2 = 3,
       /* float64 datasets (cnmf_dataset_create_f64 / cnmf_dataset_from_columns_f64) and their params: X, factors,
        * products and every sum in fp64 (fp64 tensor-core GEMM), Frobenius loss with MU or CD, as scikit-learn computes
        * on a float64 X.  Reached through the _f64 entry points only. */
       CNMF_PRECISION_FP64 = 4 };

/* yaml 'beta_loss' (cnmf.py:622, CLI --beta-loss cnmf.py:1251).  'frobenius' (or 2) runs the tensor-core path with
 * either solver; 'kullback-leibler' (1) and 'itakura-saito' (0) run the multiplicative updates of sklearn
 * _nmf.py:551-608, 637-694 as fused streaming kernels (solver must be CNMF_SOLVER_MU, as in sklearn). */
enum { CNMF_LOSS_FROBENIUS = 0, CNMF_LOSS_KULLBACK_LEIBLER = 1, CNMF_LOSS_ITAKURA_SAITO = 2 };

/* yaml 'init' (cnmf.py:335, CLI --init cnmf.py:1252): scikit-learn's seeded random init or one of its NNDSVD starts */
enum { CNMF_INIT_RANDOM = 0, CNMF_INIT_NNDSVD = 1, CNMF_INIT_NNDSVDA = 2, CNMF_INIT_NNDSVDAR = 3 };

/* Mirrors the nmf_kwargs dict of cnmf.py:618-627 after sklearn's own scaling of the
 * regularisation (sklearn/decomposition/_nmf.py:1249-1260): l1_reg_W = n_features*alpha_W*l1_ratio ... */
typedef struct cnmf_nmf_params {
  int32_t solver;        /* CNMF_SOLVER_* */
  int32_t precision;     /* CNMF_PRECISION_* */
  int32_t max_iter;      /* 'max_iter' (cnmf.py:625) */
  int32_t reserved;      /* flags: bit 0 = draw the random init on the host (bit-exact numpy stream) instead of the GPU;
                          * bits 1-2 = CNMF_INIT_* of cnmf_factorize / cnmf_factorize_seeds_dev (0 = random) */
  double tol;            /* 'tol' (cnmf.py:624) */
  double l1_reg_W, l2_reg_W, l1_reg_H, l2_reg_H;
  int32_t beta_loss;     /* CNMF_LOSS_* ('beta_loss', cnmf.py:622); 0 = frobenius */
  int32_t reserved2;     /* must be 0 */
} cnmf_nmf_params;

/* ---- library / handle -------------------------------------------------------------- */
int cnmf_abi_version(void);
const char* cnmf_last_error(void);
int cnmf_create(cnmf_handle_t* out, int device);
int cnmf_destroy(cnmf_handle_t h);
/* number of kernels this library has launched through the handle since creation */
long long cnmf_launch_count(cnmf_handle_t h);
/* free / total bytes of the handle's device (cudaMemGetInfo) plus the bytes parked in the handle's own buffer
 * pool and workspace (reusable by the next call): what the facade sizes its restart groups from, so that a
 * K-sweep larger than HBM is factorized in several batched solves instead of failing in cudaMalloc */
int cnmf_mem_info(cnmf_handle_t h, long long* free_bytes, long long* total_bytes, long long* cached_bytes);
/* device bytes one packed factor row (one component of one restart) costs in a batched solve on this dataset:
 * factors, operand pieces, compaction ping-pong and result slabs, product slices */
long long cnmf_solve_bytes_per_row(cnmf_dataset_t d);

/* per-launch CUDA-event timing of the dominant kernel (the batched GEMM) on its launching stream:
 * enable (resets the counters), run, then read total device ms, launches and algorithmic FLOPs
 * (2*M*N*K per launch, counted once -- not 3x for the 3xTF32 passes) */
int cnmf_profile_enable(cnmf_handle_t h, int on);
int cnmf_profile_get(cnmf_handle_t h, double* gemm_ms, long long* gemm_launches, double* gemm_flops);
/* same counters per kernel class: 0 = batched GEMM (work = algorithmic FLOPs), 1 = fused update kernels
 * (work = algorithmic bytes: factor read + product slices read + factor and tf32 pieces written), 2 = the product
 * of a sparse dataset, both of its kernels (work = algorithmic bytes: 8 per entry, col_ptr, staged U, output),
 * 3 = the fp64 GEMM of cnmf_nndsvd_init_dev (work = algorithmic FLOPs, 2*M*N*K per launch), 4 = the fp64 GEMM of
 * the float64 solver (work = algorithmic FLOPs, 2*M*N*K per launch), 5 = the fp64 GEMMs of cnmf_moe_grams and
 * cnmf_moe_correct (work = algorithmic FLOPs, 2*M*N*K per launch) */
int cnmf_profile_get_class(cnmf_handle_t h, int kernel_class, double* ms, long long* launches, double* work);

/* host wall-clock phases (ms) of the last cnmf_factorize, cnmf_factorize_seeds_dev, cnmf_factorize_init or
 * cnmf_factorize_dev on this handle: starting factors (host RNG, device RNG enqueue or NNDSVD), H2D of host initial
 * factors, batched solve, copy-out of the results.  A phase the call does not have reads 0. */
int cnmf_last_timing(cnmf_handle_t h, double* rng_ms, double* h2d_ms, double* solve_ms, double* d2h_ms);

/* ---- dataset: a cells x genes matrix made resident on the device ------------------- */
/* Replaces `norm_counts.X` / `tpm.X` handed to _nmf (cnmf.py:726,741,873,919,950-952).
 * Builds the device-side forms both GEMM orientations need (X, X^T, tf32 pieces) and
 * sum(X), sum(X^2).  `src_is_device` = 0: X is host memory (copied H2D inside the call). */
int cnmf_dataset_create(cnmf_handle_t h, const float* X, int n_rows, int n_cols, long long ld,
                        int src_is_device, int precision, void* stream, cnmf_dataset_t* out);
/* cnmf_dataset_create of the dense form of a canonical host CSR matrix (row_ptr[n_rows + 1] int64 from 0 to nnz;
 * col_idx int32 in [0, n_cols), strictly increasing within a row -- checked; values fp32) without forming it on the
 * host: the zeroed device matrix receives the stored entries, which cross PCIe in slices of at most 2^24 entries, then
 * the form and the operands are built as cnmf_dataset_create builds them -- the dataset is bit-identical to the one
 * cnmf_dataset_create makes of the dense matrix.  The staged slices are freed before the operands are built. */
int cnmf_dataset_create_from_csr(cnmf_handle_t h, int n_rows, int n_cols, long long nnz, const int64_t* row_ptr,
                                 const int32_t* col_idx, const float* values, int precision, void* stream,
                                 cnmf_dataset_t* out);
/* A cells x genes matrix kept sparse on the device: canonical CSC from the host (col_ptr[n_cols + 1] int64, monotone,
 * from 0 to nnz; row_idx int32 in [0, n_rows), increasing and unique within a column -- scipy.sparse tocsc() gives
 * exactly that; the order is not checked; values fp32), 8 bytes per stored entry.  For the TPM matrix of the consensus
 * step (cnmf.py:950-969), or the raw counts of prepare, when its dense forms do not fit.  Supported on such a dataset:
 * shape, ld, sums, col_stats, tpm_stats, from_columns (the result is an ordinary dense dataset), destroy, project_rows
 * and refit with transposed = 1 and beta_loss = frobenius (MU and CD; the one product X^T W is formed in fp64).  Every
 * other entry point returns -3.
 * cnmf_dataset_is_exact reports 0 (no tensor-core product runs on it). */
int cnmf_dataset_create_csc(cnmf_handle_t h, int n_rows, int n_cols, long long nnz, const int64_t* col_ptr,
                            const int32_t* row_idx, const float* values, int precision, void* stream,
                            cnmf_dataset_t* out);
/* The same sparse dataset from a canonical host CSR matrix (row_ptr[n_rows + 1] int64 from 0 to nnz; col_idx int32 in
 * [0, n_cols), strictly increasing within a row -- checked; values fp32), transposed on the device: the CSC arrays
 * are bit-identical to what cnmf_dataset_create_csc gets from scipy's tocsc() of the same matrix, and every result on
 * the dataset is too.  Only the stored entries cross PCIe (12 bytes each).  The CSR upload (12 bytes per entry) and a
 * count table of at most 128 MB are freed before the call returns. */
int cnmf_dataset_create_csr(cnmf_handle_t h, int n_rows, int n_cols, long long nnz, const int64_t* row_ptr,
                            const int32_t* col_idx, const float* values, int precision, void* stream,
                            cnmf_dataset_t* out);
/* worst-case device bytes cnmf_dataset_create of an n_rows x n_cols matrix at `precision` needs while the dataset is
 * built, over the forms it can take (exact f16, exact tf32, general): what a caller compares with free memory to
 * choose between the dense and the CSC dataset */
int cnmf_dataset_dense_bytes(int n_rows, int n_cols, int precision, long long* peak);
/* new dataset = src[:, cols] * col_scale (cnmf.py:965-969: tpm[:, hvgs] / std) */
int cnmf_dataset_from_columns(cnmf_dataset_t src, const int32_t* cols_host, const float* col_scale_host,
                              int n_cols, void* stream, cnmf_dataset_t* out);
int cnmf_dataset_destroy(cnmf_dataset_t d);
int cnmf_dataset_shape(cnmf_dataset_t d, int* n_rows, int* n_cols);
/* padded row strides of the packed factor layout: W^T rows (ld_rows >= n_rows), H rows (ld_cols >= n_cols) */
int cnmf_dataset_ld(cnmf_dataset_t d, int* ld_rows, int* ld_cols);
int cnmf_dataset_sums(cnmf_dataset_t d, double* sum, double* sum_sq);
/* smallest entry of X (sklearn refuses beta_loss <= 0 when X.min() == 0, _nmf.py:1675-1680; the caller raises) */
int cnmf_dataset_min(cnmf_dataset_t d, float* min_host, void* stream);
/* 1 when the dataset was recognised as (row scale) x (integer counts <= 2048) x (column scale) -- what
 * HVG-normalised counts (cnmf.py:542) and TPM (cnmf.py:245-251) are -- and therefore runs the 2-pass
 * tensor-core products (the integer operand needs no tf32 "lo" piece); 0 = general 3-pass 3xTF32.
 * Returns 2 when, in addition, the dataset was created with CNMF_PRECISION_F16X2 and the 2 passes therefore run on
 * f16 MMAs. */
int cnmf_dataset_is_exact(cnmf_dataset_t d);
/* per-column mean and population variance (StandardScaler(with_mean=False), cnmf.py:131-134) */
int cnmf_dataset_col_stats(cnmf_dataset_t d, double* mean_host, double* var_host, void* stream);

/* ---- device-side `prepare` numerics (cnmf.py:131-251, 487-556) on a resident counts matrix ------------- */
/* per-row (cell) totals, fp64: the TPM denominators of compute_tpm / sc.pp.normalize_total (cnmf.py:245-251) */
int cnmf_dataset_row_sums(cnmf_dataset_t d, double* row_sums_host, void* stream);
/* per-column mean and population variance of diag(row_scale) * X accumulated in fp64 from the stored values:
 * with X = raw counts and row_scale = 1e6 / cell total these are the TPM gene statistics that drive the
 * over-dispersion ranking (get_highvar_genes, cnmf.py:192-242) and `tpm_stats` (cnmf.py:436-445), without
 * materialising TPM */
int cnmf_dataset_scaled_col_stats(cnmf_dataset_t d, const double* row_scale_host, double* mean_host, double* var_host,
                                  void* stream);
/* sparse (CSC) counts datasets only -- a dense one gets -3 and has row_sums / scaled_col_stats instead: per-row totals
 * (fp64 sums of the stored values) and the per-column mean and population variance of diag(target_sum / total) * X,
 * the row scale being 0 for a row whose total is 0.  The TPM totals and gene statistics of prepare (cnmf.py:245-251,
 * 436-445) for counts that stay sparse on the device; fixed reduction order, so two calls are bit-identical. */
int cnmf_dataset_tpm_stats(cnmf_dataset_t d, double target_sum, double* totals_host, double* mean_host,
                           double* var_host, void* stream);
/* new dataset = diag(row_scale) * src (TPM from counts, cnmf.py:245-251); the exact-count detection runs again */
int cnmf_dataset_scale_rows(cnmf_dataset_t src, const float* row_scale_host, void* stream, cnmf_dataset_t* out);

/* ---- random init (sklearn _nmf.py:296-307; host RNG, bit-exact numpy legacy stream) -- */
/* Writes |avg*z| as fp32: H (k x n_features, row stride ldH) first, then W stored transposed
 * Wt (k x n_samples, row stride ldW).  Pure host code (no CUDA). */
int cnmf_random_init_host(uint32_t seed, double avg, int n_samples, int n_features, int k,
                          float* Wt, long long ldW, float* H, long long ldH);

/* Same stream generated ON THE DEVICE (one thread block per restart; see csrc/rng_device.cu for the one
 * caveat: log() may differ from glibc in the last fp64 bit, visible in ~1 fp32 value per 10^8) into packed,
 * padded device buffers: Wt_dev (sum ks) x ld_rows, H_dev (sum ks) x ld_cols (cnmf_dataset_ld), avg =
 * sqrt(mean(X) / k) as sklearn.  This is what cnmf_factorize uses unless params.reserved bit 0 is set. */
int cnmf_random_init_dev(cnmf_dataset_t d, int n_restarts, const int32_t* ks, const uint32_t* seeds, float* Wt_dev,
                         float* H_dev, void* stream);

/* NNDSVD starting factors (sklearn _nmf.py:309-369 after randomized_svd(X, k, random_state=seed), SK/utils/extmath.py)
 * of every restart, computed on the device from the dataset's fp32 X with float64 arithmetic (fp64 tensor-core
 * products, CholeskyQR2 in place of the LU / QR normalisers, Jacobi SVD of the small factor) into the same packed,
 * padded buffers as cnmf_random_init_dev.  init = CNMF_INIT_NNDSVD / _NNDSVDA / _NNDSVDAR; every ks[r] must be
 * <= min(n_rows, n_cols) (sklearn's condition).  The work space (about 8 * sum(ks + 10) * (n_rows + n_cols) bytes)
 * is allocated and freed inside the call, in chunks of restarts sized from the free device memory; a restart's
 * result does not depend on the chunking or on the other restarts.  Sparse datasets: -3. */
int cnmf_nndsvd_init_dev(cnmf_dataset_t d, int n_restarts, const int32_t* ks, const uint32_t* seeds, int init,
                         float* Wt_dev, float* H_dev, void* stream);
/* test hook: at most max_restarts restarts per chunk of cnmf_nndsvd_init_dev on this handle (0 = sized from the free
 * device memory only, the default) -- chunkings can then be compared without starving the device */
int cnmf_nndsvd_chunk_limit(cnmf_handle_t h, int max_restarts);
/* test hook: the fp64 GEMM of cnmf_nndsvd_init_dev and of the float64 solver, on the dataset's own X: the fp32 X of an
 * ordinary dataset, the fp64 X of a float64 one.  to_genes = 0: C_host (M x n_rows) = A_host (M x n_cols) X^T;
 * 1: C_host (M x n_cols) = A_host (M x n_rows) X.  Host arrays dense row-major fp64.  The device output starts as NaN
 * bytes, so an output the kernel does not write shows.  Sparse datasets: -3. */
int cnmf_nndsvd_gemm_host(cnmf_dataset_t d, int to_genes, int M, const double* A_host, double* C_host, void* stream);

/* ---- float64 datasets (CNMF_PRECISION_FP64) -------------------------------------------------------------------- */
/* X (n_rows x n_cols, row stride ld, fp64) resident as one fp64 row-major copy, 8 bytes per entry, no transposed copy
 * and no operand pieces.  Entry points that take or return floats refuse such a dataset (-3) and name their _f64
 * form; the _f64 entry points refuse any other dataset.  Also supported on it: destroy, shape, ld, sums, col_stats,
 * solve_bytes_per_row.  Supported: beta_loss = frobenius, MU and CD, random (device generator) and NNDSVD starts. */
int cnmf_dataset_create_f64(cnmf_handle_t h, const double* X, int n_rows, int n_cols, long long ld, int src_is_device,
                            void* stream, cnmf_dataset_t* out);
/* cnmf_dataset_create_from_csr for float64 datasets: fp64 values, scattered into the zeroed fp64 X; bit-identical to
 * cnmf_dataset_create_f64 of the dense matrix */
int cnmf_dataset_create_from_csr_f64(cnmf_handle_t h, int n_rows, int n_cols, long long nnz, const int64_t* row_ptr,
                                     const int32_t* col_idx, const double* values, void* stream, cnmf_dataset_t* out);
/* new float64 dataset = src[:, cols] / divisor (cnmf.py:542, 967-969: X /= std), each entry one IEEE fp64 division */
int cnmf_dataset_from_columns_f64(cnmf_dataset_t src, const int32_t* cols_host, const double* divisor_host, int n_cols,
                                  void* stream, cnmf_dataset_t* out);
/* cnmf_factorize, cnmf_factorize_init, cnmf_refit and cnmf_project_rows of a float64 dataset: the same arguments with
 * fp64 factors and outputs; params.precision = CNMF_PRECISION_FP64.  The starting factors of cnmf_factorize_f64 are
 * scikit-learn's random init drawn on the device (params.reserved bit 0 must be 0) or its NNDSVD starts (bits 1-2),
 * both kept in fp64. */
int cnmf_factorize_f64(cnmf_dataset_t d, int n_restarts, const int32_t* ks, const uint32_t* seeds,
                       const cnmf_nmf_params* params, double* spectra_host, double* usages_host, int32_t* n_iter_host,
                       double* err_host, void* stream);
int cnmf_factorize_init_f64(cnmf_dataset_t d, int n_restarts, const int32_t* ks, const double* Wt0_host,
                            const double* H0_host, const cnmf_nmf_params* params, double* spectra_host,
                            double* usages_host, int32_t* n_iter_host, double* err_host, void* stream);
int cnmf_refit_f64(cnmf_dataset_t d, int transposed, int k, const double* fixed_host, const cnmf_nmf_params* params,
                   double* out_host, int32_t* n_iter_host, double* err_host, void* stream);
int cnmf_project_rows_f64(cnmf_dataset_t d, int k, const double* Ut_host, double* out_host, void* stream);

/* ---- batched factorize: replaces the restart loop of cNMF.factorize ---------------- */
/* For r in [0, n_restarts): one NMF of the dataset with n_components = ks[r] and
 * random_state = seeds[r] (cnmf.py:738-741), all restarts advanced together on the GPU.  The starting factors are
 * sklearn's random init, or its NNDSVD starts (cnmf_nndsvd_init_dev) when params.reserved bits 1-2 name one.
 *   spectra_host : packed (sum ks) x n_cols, row stride n_cols; restart r owns rows
 *                  [sum ks[0..r), +ks[r])  -- what factorize saves per restart (cnmf.py:742-745)
 *   usages_host  : optional (may be NULL; the reference discards W) packed (sum ks) x n_rows,
 *                  i.e. W^T per restart
 *   n_iter_host  : optional [n_restarts] iterations run;  err_host: optional [n_restarts]
 *                  ||X - WH||_F of the returned factors (every solver and loss) */
int cnmf_factorize(cnmf_dataset_t d, int n_restarts, const int32_t* ks, const uint32_t* seeds,
                   const cnmf_nmf_params* params, float* spectra_host, float* usages_host,
                   int32_t* n_iter_host, double* err_host, void* stream);

/* Same restarts, same seeds, but the spectra stay on the device: spectra_dev is (sum ks) x ld_out (ld_out >= n_cols).
 * This is the per-rank half of the multi-GPU path: the slab goes straight into cnmf_allgather_spectra / an NCCL
 * all-gather without touching the host (cnmf.py:748-773 `combine` meets on disk instead). */
int cnmf_factorize_seeds_dev(cnmf_dataset_t d, int n_restarts, const int32_t* ks, const uint32_t* seeds,
                             const cnmf_nmf_params* params, float* spectra_dev, long long ld_out,
                             int32_t* n_iter_host, double* err_host, void* stream);

/* ---- the one collective of the path: all-gather of the per-rank spectra slabs (SURVEY.md 8b/8e) ---------------- */
/* merged_dev (world x rows_per_rank x ld) <- every rank's local_dev (rows_per_rank x ld; ranks with fewer rows pad),
 * asynchronous on `stream`.  `nccl_comm` is an ncclComm_t -- the host application's own, or one made by
 * cnmf_comm_create.  libnccl.so.2 is bound at run time (no link-time dependency; CNMF_NCCL_LIB overrides the path). */
int cnmf_allgather_spectra(void* nccl_comm, const float* local_dev, long long rows_per_rank, long long ld,
                           float* merged_dev, void* stream);
/* communicator bootstrap for hosts without one: rank 0 calls cnmf_comm_unique_id and ships the 128 bytes to every
 * rank over whatever channel it has (MPI, a TCP store, torch.distributed ...); every rank then calls
 * cnmf_comm_create with its rank (collective: blocks until all ranks arrive) */
int cnmf_comm_unique_id(char* id_out_128);
int cnmf_comm_create(cnmf_handle_t h, const char* id_128, int rank, int world, void** comm_out);
int cnmf_comm_destroy(void* nccl_comm);

/* Same, but initial factors are supplied (host, packed like the outputs) instead of seeds. */
int cnmf_factorize_init(cnmf_dataset_t d, int n_restarts, const int32_t* ks, const float* Wt0_host,
                        const float* H0_host, const cnmf_nmf_params* params, float* spectra_host,
                        float* usages_host, int32_t* n_iter_host, double* err_host, void* stream);

/* Device-resident form: initial factors and the output stay on the GPU (packed, padded strides from
 * cnmf_dataset_ld): Wt0_dev (sum ks) x ld_rows, H0_dev / spectra_dev (sum ks) x ld_cols. */
int cnmf_factorize_dev(cnmf_dataset_t d, int n_restarts, const int32_t* ks, const float* Wt0_dev,
                       const float* H0_dev, const cnmf_nmf_params* params, float* spectra_dev,
                       int32_t* n_iter_host, double* err_host, void* stream);

/* ---- NNLS refit: replaces cNMF.refit_usage / refit_spectra (cnmf.py:776-820) ------- */
/* NMF with one factor fixed (sklearn update_H=False), same solver as factorize (cnmf.py:792).
 * transposed = 0 (refit_usage,  cnmf.py:798):  fixed_host = H   (k x n_cols), out_host = W (n_rows x k)
 * transposed = 1 (refit_spectra, cnmf.py:820): fixed_host = W^T (k x n_rows), out_host = H^T (n_cols x k)
 * W0 follows sklearn _nmf.py:1223-1228 ('mu': sqrt(X.mean()/k) constant, 'cd': zeros).
 * err_host (optional): final ||X - W H||_F (its square is the prediction error of cnmf.py:926-930). */
int cnmf_refit(cnmf_dataset_t d, int transposed, int k, const float* fixed_host, const cnmf_nmf_params* params,
               float* out_host, int32_t* n_iter_host, double* err_host, void* stream);

/* out (k x n_cols) = Ut (k x n_rows) * X : the X^T Y accumulator of efficient_ols_all_cols
 * (cnmf.py:98-119) as one tensor-core GEMM; the caller centres U (see cnmf_b200/consensus.py).
 * On a sparse dataset (k <= 32): fp64 products and sums in a fixed order, bit-identical from call to call. */
int cnmf_project_rows(cnmf_dataset_t d, int k, const float* Ut_host, float* out_host, void* stream);

/* test / micro-benchmark hook: C (M x N) = A (M x Kd) * B (N x Kd)^T through the same GEMM kernels the
 * solver uses (precision selects FFMA or wgmma 3xTF32); reps > 1 reports mean device ms per launch.
 * The exact-count forms the solver runs on scaled-integer datasets: b_exact = 1 (tf32x3; implied by f16x2) takes B as
 * exact tf32 values (2 passes, no lo piece of B); then k_scale (length Kd, or NULL) is folded into the A pieces as the
 * solver folds the dataset's scale, A diag(k_scale), and out_col_scale (length N, or NULL) multiplies column n of C:
 * C = A diag(k_scale) B^T diag(out_col_scale).  The scales are refused without the exact form.
 * tile_n: columns per output tile, 0 = chosen by shape as in the solver; 128, or 168 / 192 in the exact forms, forces
 * that width (the result does not depend on it). */
int cnmf_gemm_abt_host(cnmf_handle_t h, int precision, const float* A, const float* B, int M, int N, int Kd,
                       int splits, int b_exact, const float* k_scale, const float* out_col_scale, int tile_n, float* C,
                       int reps, float* ms_out, void* stream);

/* test hook: ONE update launch of the batched solver (or the stand-alone Gram / <NUM, F> / piece launches that start a
 * solve) on host-supplied packed data, issued exactly as the solver issues it.  Slot s holds restart rids[s] with
 * ks[s] components at packed rows [sum ks[0..s), +ks[s]); every per-restart output is indexed by rid.  Host arrays are
 * dense row-major with the padded row stride ld = ceil(n / 32) * 32; every array marked in/out is uploaded before the
 * launch and downloaded after it, so entries the launch must not touch can be pre-filled and checked. */
enum { CNMF_UNIT_SOLVER_NONE = -1 };                               /* or CNMF_SOLVER_MU / CNMF_SOLVER_CD */
enum { CNMF_UNIT_PIECES_NONE = 0, CNMF_UNIT_PIECES_TF32 = 1, CNMF_UNIT_PIECES_F16 = 2 };
enum { CNMF_UNIT_GRAM_NONE = 0, CNMF_UNIT_GRAM_FUSED = 1, CNMF_UNIT_GRAM_STANDALONE = 2 };
typedef struct cnmf_update_step_args {
  int32_t n_slots;              /* restarts in the batch */
  int32_t n_rids;               /* length of done / scal_out, and of gram_in / gram_out in 32 x 32 blocks */
  const int32_t* ks;            /* [n_slots], 1..32; kp = 16 when every K <= 16, else 32 (as the solver decides) */
  const int32_t* rids;          /* [n_slots], distinct, < n_rids */
  const int32_t* done;          /* [n_rids] 1 = frozen restart: the launches skip it */
  int32_t n;                    /* valid columns of the factor */
  int32_t cpb_tiles;            /* columns per block of the update / cross launches, in update tiles: 1, 2 or 4 */
  int32_t solver;               /* CNMF_SOLVER_MU / CNMF_SOLVER_CD: one update launch; CNMF_UNIT_SOLVER_NONE: no update
                                 * (initial factors): stand-alone Gram, <NUM, F> and pieces of F as it stands */
  int32_t pieces;               /* CNMF_UNIT_PIECES_*: tf32 hi / lo of F * piece_scale, or fp16 hi / mid + group scales */
  int32_t gram;                 /* CNMF_UNIT_GRAM_*: Gram of the new F fused into the update (kp == 16 only), or the
                                 * stand-alone gram_partial + finalize launches after it */
  int32_t want_scalar;          /* MU: <NUM, F_new>; CD: sum |projected gradient|; NONE: <NUM, F> */
  int32_t nsplit;               /* split-K slices of the product */
  float l1, l2;
  float* F;                     /* in/out: (sum ks) x ld */
  const float* num;             /* nsplit x (sum ks) x ld */
  const double* gram_in;        /* n_rids x 32 x 32: finalised Gram of the other factor */
  const float* piece_scale;     /* ld, or NULL */
  void* pieces_hi;              /* in/out (pieces != NONE): (sum ks) x ld floats (tf32) or fp16 halves (f16) */
  void* pieces_lo;
  float* tile_scale;            /* in/out (f16 pieces): (sum ks) x ceil(ld / 512) */
  double* gram_out;             /* in/out (gram != NONE): n_rids x 32 x 32 */
  double* scal_out;             /* in/out (want_scalar): n_rids */
} cnmf_update_step_args;
/* The last-block tickets of the fused launches are zeroed once per handle, when first allocated: a second call relies
 * on the kernel's own reset. */
int cnmf_update_step_host(cnmf_handle_t h, const cnmf_update_step_args* args, void* stream);

/* test hook: ONE half-step or ONE divergence evaluation of the KL / IS solver on host-supplied packed data, issued
 * through the launch functions the solver uses (batch layout, rids and done as for cnmf_update_step_host).  side names
 * the half whose BetaSide the solver would build: W (items = cells, D = X^T) or H (items = genes, D = X); the half
 * decides the KL zero-sum rule and the clip.  Strides are the dataset's: ld_items = ceil(n_items / 32) * 32,
 * ld_contract = ceil(n_contract / 32) * 32.
 *   op UPDATE (loss KL or IS): KL first computes the fp64 row sums of F_other (row_sum_kernel) into oth_sum, then one
 *     beta_update_kernel launch updates F_own in place with l1 / l2.
 *   op DIVERGENCE (loss KL, IS or FROBENIUS): one beta_error_kernel pass, then beta_check_kernel at iteration 0.
 *     last[rid] = sqrt(2 max(res, 0)), or ||D - F_own^T F_other||_F for FROBENIUS; totals[2 rid + {0, 1}] = the fp64
 *     sums (t, s) of the per-block partials, in the order beta_check_kernel adds them: KL t = sum over x > eps of
 *     x log(x / WH') - x + WH' (WH' = max(WH, eps)), s = sum(WH) over x <= eps plus sum(WH - WH') over x > eps,
 *     res = t + s;  IS t = sum over x > eps of (x / WH' - 1) - log(x / WH'), s = number of entries x > eps,
 *     res = t - (entries - s);  FROBENIUS t = sum (x - WH)^2, s = 0. */
enum { CNMF_UNIT_BETA_UPDATE = 0, CNMF_UNIT_BETA_DIVERGENCE = 1 };
enum { CNMF_UNIT_SIDE_W = 0, CNMF_UNIT_SIDE_H = 1 };
typedef struct cnmf_beta_step_args {
  int32_t n_slots;              /* restarts in the batch */
  int32_t n_rids;               /* length of done / last, and of totals in pairs */
  const int32_t* ks;            /* [n_slots], 1..32 */
  const int32_t* rids;          /* [n_slots], distinct, < n_rids */
  const int32_t* done;          /* [n_rids] 1 = frozen restart: the launches skip it */
  int32_t op;                   /* CNMF_UNIT_BETA_* */
  int32_t side;                 /* CNMF_UNIT_SIDE_* */
  int32_t loss;                 /* CNMF_LOSS_* */
  int32_t n_items, n_contract;
  float l1, l2;                 /* regularisation of the updated half */
  const float* D;               /* n_contract x ld_items: the data, item index contiguous */
  float* F_own;                 /* in/out: (sum ks) x ld_items */
  const float* F_other;         /* (sum ks) x ld_contract */
  double* oth_sum;              /* out (update, KL): sum ks */
  double* last;                 /* in/out (divergence): n_rids */
  double* totals;               /* in/out (divergence): n_rids x 2 */
} cnmf_beta_step_args;
int cnmf_beta_step_host(cnmf_handle_t h, const cnmf_beta_step_args* args, void* stream);

/* test hook: ONE launch of the float64 solver (nmf_f64.cu) on host-supplied packed fp64 data, through the launch
 * functions the solver uses (batch layout, rids and done as for cnmf_update_step_host; ld = ceil(n / 32) * 32; the
 * partial Grams use the solver's stride kp = max ks rounded up to 4).
 *   op UPDATE: one MU or CD update of F with the other factor's Gram gram_in, l1 / l2; with want_scalar, MU <NUM, F_new>
 *     or CD sum |projected gradient| per restart into scal_out, through finalize.
 *   op GRAM: the Gram of F (gram64 + finalize) into gram_out.
 *   op CROSS: <NUM, F> per restart (cross64 + finalize) into scal_out.
 * Every array marked in/out is uploaded before the launch and downloaded after it. */
enum { CNMF_UNIT_F64_UPDATE = 0, CNMF_UNIT_F64_GRAM = 1, CNMF_UNIT_F64_CROSS = 2 };
typedef struct cnmf_update_step_f64_args {
  int32_t n_slots;              /* restarts in the batch */
  int32_t n_rids;               /* length of done / scal_out, and of gram_in / gram_out in 32 x 32 blocks */
  const int32_t* ks;            /* [n_slots], 1..32 */
  const int32_t* rids;          /* [n_slots], distinct, < n_rids */
  const int32_t* done;          /* [n_rids] 1 = frozen restart: the launches skip it */
  int32_t n;                    /* valid columns of the factor */
  int32_t op;                   /* CNMF_UNIT_F64_* */
  int32_t solver;               /* op UPDATE: CNMF_SOLVER_MU / CNMF_SOLVER_CD */
  int32_t want_scalar;          /* op UPDATE: also the per-restart scalar */
  double l1, l2;
  double* F;                    /* in/out: (sum ks) x ld */
  const double* num;            /* (sum ks) x ld (UPDATE, CROSS) */
  const double* gram_in;        /* n_rids x 32 x 32 (UPDATE) */
  double* gram_out;             /* in/out (GRAM): n_rids x 32 x 32 */
  double* scal_out;             /* in/out (UPDATE with want_scalar, CROSS): n_rids */
} cnmf_update_step_f64_args;
int cnmf_update_step_f64_host(cnmf_handle_t h, const cnmf_update_step_f64_args* args, void* stream);

/* test hook: ONE launch of the convergence kernel every solver shares, on host state (batch layout and rids as for
 * cnmf_update_step_host; the state's done is also the batch's, as in the solvers).  it, tol and max_iter are what the
 * solvers pass: MU it = 0 initialises err0 / prev, a check at it with tol > 0 and it % 10 == 0 passes tol, a forced check
 * at it = max_iter passes -1; CD passes tol at every iteration.
 *   MU: err = sqrt(max(normX2 - 2 cross + <gramA, gramB>, 0)) over the K x K block of each rid (32 x 32 blocks).
 *   CD: viol = violA (+ violB when given).
 * Frozen restarts (done = 1) are left alone. */
typedef struct cnmf_conv_check_args {
  int32_t n_slots;              /* restarts in the batch */
  int32_t n_rids;               /* length of every per-restart array */
  const int32_t* ks;            /* [n_slots], 1..32 */
  const int32_t* rids;          /* [n_slots], distinct, < n_rids */
  int32_t solver;               /* CNMF_SOLVER_MU / CNMF_SOLVER_CD */
  int32_t it, max_iter;
  double tol, normX2;
  const double* cross;          /* MU: n_rids */
  const double* gramA;          /* MU: n_rids x 32 x 32 */
  const double* gramB;
  const double* violA;          /* CD: n_rids */
  const double* violB;          /* CD: n_rids, or NULL */
  int32_t* done;                /* in/out: n_rids */
  int32_t* n_iter;              /* in/out: n_rids */
  double* err0;                 /* in/out: n_rids */
  double* prev;
  double* last;
} cnmf_conv_check_args;
int cnmf_conv_check_host(cnmf_handle_t h, const cnmf_conv_check_args* args, void* stream);

/* test hooks: what a dataset holds and the solver's two products on it.
 * cnmf_dataset_form returns the operand form decided at creation (CNMF_FORM_*; >= 0) or < 0 on error.  Sparse (CSC)
 * datasets report the form their detection chose, which cnmf_dataset_from_columns passes on; they hold none of the
 * dense operands themselves (cnmf_dataset_is_exact reports 0 for them). */
enum { CNMF_FORM_FP32 = 0, CNMF_FORM_TF32 = 1, CNMF_FORM_TF32_EXACT = 2, CNMF_FORM_F16_EXACT = 3, CNMF_FORM_FP64 = 4 };
int cnmf_dataset_form(cnmf_dataset_t d);
/* copies one resident array, padding included, to out_host; bytes must be its exact size:
 *   X, X_HI, X_LO (n_rows x ld_cols floats), XT, XT_HI, XT_LO (n_cols x ld_rows floats), X_H16 / XT_H16 (the same
 *   shapes as fp16), ROW_SCALE (ld_rows floats), COL_SCALE (ld_cols floats); on sparse (CSC) datasets CSC_COL_PTR
 *   (n_cols + 1 int64), CSC_ROW_IDX (nnz int32), CSC_VALUES (nnz floats), nnz being the last entry of CSC_COL_PTR.
 * The exact forms hold their integer matrix C in X_HI and C^T in XT_HI (F16_EXACT: only as fp16, X_H16 / XT_H16).
 * Returns -3 for an array this dataset does not hold. */
enum { CNMF_OPERAND_X = 0, CNMF_OPERAND_XT = 1, CNMF_OPERAND_X_HI = 2, CNMF_OPERAND_X_LO = 3, CNMF_OPERAND_XT_HI = 4,
       CNMF_OPERAND_XT_LO = 5, CNMF_OPERAND_X_H16 = 6, CNMF_OPERAND_XT_H16 = 7, CNMF_OPERAND_ROW_SCALE = 8,
       CNMF_OPERAND_COL_SCALE = 9, CNMF_OPERAND_CSC_COL_PTR = 10, CNMF_OPERAND_CSC_ROW_IDX = 11,
       CNMF_OPERAND_CSC_VALUES = 12 };
int cnmf_dataset_operand_host(cnmf_dataset_t d, int which, void* out_host, long long bytes);
/* one of the batched solver's two products on the dataset's view (transposed as cnmf_refit's), through the solver's own
 * launch: the factor's operand pieces for the dataset's form, then the split-K GEMM with the solver's split plan.
 *   side 0: NUM_r = F * B_rows^T, F the column factor (SK x n_c of the view), out SK x n_r per slice
 *   side 1: NUM_c = F * B_cols^T, F the row factor (SK x n_r of the view), out SK x n_c per slice
 * (untransposed: n_r = n_rows, n_c = n_cols).  F_host is dense row-major; out_host receives the raw split-K slices,
 * splits x SK x n_out, their sum being the product.  *splits_out = the number of slices; out_host may be NULL to ask
 * for it alone.  Dense float datasets, and sparse (CSC) ones for the one product their transposed refit runs
 * (transposed = 1, side 0, SK <= 32): the factor staged as rows, then csc_project into the zeroed NUM_r, as cnmf_refit
 * issues it, one slice; any other combination on a sparse dataset returns -3. */
int cnmf_dataset_gemm_host(cnmf_dataset_t d, int transposed, int side, int SK, const float* F_host, float* out_host,
                           int* splits_out);

/* ---- consensus kernels (cnmf.py:882-916) on a stacked-spectra matrix S (R x G, device, row stride ld) -- */
/* rows / ||row||_2 in place (cnmf.py:882) */
int cnmf_l2_normalize_rows(cnmf_handle_t h, float* S_dev, int R, int G, int ld, void* stream);
/* local density (cnmf.py:891-896): density[i] = (sum of the n_neighbors+1 smallest entries of row i of the
 * Euclidean distance matrix, self-distance 0 included) / n_neighbors.  D_dev: optional R x R output
 * (ld = R) for the clustergram; NULL keeps it in the library's workspace. Asynchronous on `stream`. */
int cnmf_local_density(cnmf_handle_t h, const float* S_dev, int R, int G, int ld, int n_neighbors,
                       float* density_dev, float* D_dev, void* stream);
/* per-column mean and population variance of a device matrix (KMeans tolerance, sklearn _kmeans.py:285-293) */
int cnmf_col_stats_dev(cnmf_handle_t h, const float* S_dev, int R, int G, int ld, double* mean_host,
                       double* var_host, void* stream);
/* dst row i = src row idx[i] (density filter compaction, cnmf.py:903-904) */
int cnmf_gather_rows(cnmf_handle_t h, const float* src_dev, int ld_src, const int32_t* idx_host, int n, int G,
                     float* dst_dev, int ld_dst, void* stream);
/* squared Euclidean distances from rows idx[0..n_c) of S to every row of S -> out_host (n_c x R):
 * candidate scoring of k-means++ (sklearn _kmeans.py:231-262; the random draws stay on the host) */
int cnmf_sq_dists_to_rows(cnmf_handle_t h, const float* S_dev, int R, int G, int ld, const int32_t* idx_host,
                          int n_c, float* out_host, void* stream);
/* one Lloyd E+M step (sklearn _k_means_lloyd.pyx:168-219): labels_dev updated in place (first minimum wins),
 * mind_dev[i] = squared distance to the assigned centre; optional host outputs: per-cluster fp64 column
 * sums (K x G) + counts, number of labels that changed, inertia = sum(mind). */
int cnmf_kmeans_assign(cnmf_handle_t h, const float* S_dev, int R, int G, int ld, const float* centers_host, int K,
                       int32_t* labels_dev, double* sums_host, int32_t* counts_host, float* mind_dev,
                       int32_t* n_changed_host, double* inertia_host, void* stream);
/* one full Lloyd iteration with the centres resident on the device (the loop of sklearn _kmeans.py:630-758 without a
 * K x G round trip per iteration): E step against C32_cur (labels_dev / mind_dev updated), fp64 per-cluster sums and
 * counts (sums_dev K x G, counts_dev K), new centres = sums / count into C64_new (fp64) and C32_new (their fp32 copy
 * for the next E step).  Host outputs: labels that changed, whether a cluster came out empty (then C*_new are not
 * valid for it: the caller applies the relocation rule of _k_means_common.pyx:167-211 from sums_dev / counts_dev and
 * the current centres, which this call leaves untouched), and sum((C64_new - C64_cur)^2) over the non-empty clusters. */
int cnmf_kmeans_step(cnmf_handle_t h, const float* S_dev, int R, int G, int ld, int K, const float* C32_cur_dev,
                     const double* C64_cur_dev, double* C64_new_dev, float* C32_new_dev, int32_t* labels_dev,
                     float* mind_dev, double* sums_dev, int32_t* counts_dev, int32_t* n_changed_host,
                     int32_t* any_empty_host, double* shift_host, void* stream);
/* The whole KMeans(n_clusters=K, n_init, random_state) fit of the consensus step (cnmf.py:908-910) with every
 * initialisation resident and advancing together on the device: k-means++ for all runs (2 launches per centre, no
 * host round trip), Lloyd for all runs (one small flag read per iteration), final E step + inertia.  The random
 * draws are data-independent in count and order, so the caller draws them from numpy's legacy RandomState exactly
 * as sklearn would and passes them in: first_idx_host[n_init] (rng.choice per run) and uniforms_host
 * [n_init][K-1][n_trials] (rng.uniform(size=n_trials) per further centre, n_trials = 2 + int(log(K))), in sklearn's
 * order of consumption (run by run).  tol_abs = mean feature variance * tol (sklearn _kmeans.py:285-293).
 * Outputs per run: labels (n_init x R), inertia, iterations; the caller applies sklearn's best-run rule
 * (_kmeans.py:1534-1541).  *needs_host_path = 1 when a cluster came out empty (sklearn's relocation rule,
 * _k_means_common.pyx:167-211): outputs are then undefined and the caller falls back to cnmf_kmeans_step. */
int cnmf_kmeans_fit(cnmf_handle_t h, const float* S_dev, int R, int G, int ld, int K, int n_init, int max_iter,
                    double tol_abs, const int32_t* first_idx_host, const double* uniforms_host, int n_trials,
                    int32_t* labels_host, double* inertia_host, int32_t* n_iter_host, int32_t* needs_host_path,
                    void* stream);
/* sums_host[i*K + c] = sum over rows j with label c of ||S_i - S_j||_2 : the per-sample cluster distance sums
 * from which sklearn.metrics.silhouette_score(metric='euclidean') is formed (cnmf.py:923, k_selection) */
int cnmf_cluster_dist_sums(cnmf_handle_t h, const float* S_dev, int R, int G, int ld, const int32_t* labels_dev,
                           int K, double* sums_host, void* stream);
/* per-cluster per-gene median (pandas groupby().median(), cnmf.py:913), rows then divided by their sum
 * (cnmf.py:916) -> M_dev (K x ldm). Asynchronous on `stream`. */
int cnmf_cluster_median(cnmf_handle_t h, const float* S_dev, int R, int G, int ld, const int32_t* labels_dev, int K,
                        float* M_dev, int ldm, void* stream);

/* ---- the same consensus kernels on a float64 S (precision="fp64"): S, distances, densities, centres and medians are
 * double, every argument is otherwise that of the float entry point above.  Distances keep the direct sum (x - y)^2
 * form (fp64 FMA), the radix selects of the density and the medians run over the 64-bit patterns, and the KMeans E step
 * reads the fp64 centres themselves (cnmf_kmeans_step_f64 has no fp32 centre copy). */
int cnmf_l2_normalize_rows_f64(cnmf_handle_t h, double* S_dev, int R, int G, int ld, void* stream);
int cnmf_local_density_f64(cnmf_handle_t h, const double* S_dev, int R, int G, int ld, int n_neighbors,
                           double* density_dev, double* D_dev, void* stream);
int cnmf_col_stats_dev_f64(cnmf_handle_t h, const double* S_dev, int R, int G, int ld, double* mean_host,
                           double* var_host, void* stream);
int cnmf_gather_rows_f64(cnmf_handle_t h, const double* src_dev, int ld_src, const int32_t* idx_host, int n, int G,
                         double* dst_dev, int ld_dst, void* stream);
int cnmf_sq_dists_to_rows_f64(cnmf_handle_t h, const double* S_dev, int R, int G, int ld, const int32_t* idx_host,
                              int n_c, double* out_host, void* stream);
int cnmf_kmeans_assign_f64(cnmf_handle_t h, const double* S_dev, int R, int G, int ld, const double* centers_host,
                           int K, int32_t* labels_dev, double* sums_host, int32_t* counts_host, double* mind_dev,
                           int32_t* n_changed_host, double* inertia_host, void* stream);
int cnmf_kmeans_step_f64(cnmf_handle_t h, const double* S_dev, int R, int G, int ld, int K, const double* C64_cur_dev,
                         double* C64_new_dev, int32_t* labels_dev, double* mind_dev, double* sums_dev,
                         int32_t* counts_dev, int32_t* n_changed_host, int32_t* any_empty_host, double* shift_host,
                         void* stream);
int cnmf_kmeans_fit_f64(cnmf_handle_t h, const double* S_dev, int R, int G, int ld, int K, int n_init, int max_iter,
                        double tol_abs, const int32_t* first_idx_host, const double* uniforms_host, int n_trials,
                        int32_t* labels_host, double* inertia_host, int32_t* n_iter_host, int32_t* needs_host_path,
                        void* stream);
int cnmf_cluster_dist_sums_f64(cnmf_handle_t h, const double* S_dev, int R, int G, int ld, const int32_t* labels_dev,
                               int K, double* sums_host, void* stream);
int cnmf_cluster_median_f64(cnmf_handle_t h, const double* S_dev, int R, int G, int ld, const int32_t* labels_dev,
                            int K, double* M_dev, int ldm, void* stream);

/* ---- preprocessing: Harmony's ridge correction and variance scaling (preprocess.py:9-29) ------ */
/* Harmony's mixture-of-experts ridge correction of a cells x genes matrix X (moe_correct_ridge on Z_orig = X^T).
 * Host inputs: R (K x n_cells) soft cluster assignments, Phi (n_phi x n_cells) design with row 0 the intercept of
 * ones, lamb (n_phi x n_phi) ridge penalty; all row-major fp64, 1 <= n_phi <= 64.  With P_i = Phi * R[i, :] (per cell):
 *   cnmf_moe_grams:   A_out (K x n_phi x n_phi, host) = P_i Phi^T + lamb, fp64 on the fp64 tensor cores in a fixed
 *                     split-K order.  The caller inverts the K small systems.
 *   cnmf_moe_correct: W_i = A_inv_i (P_i X) with row 0 zeroed, then X_out = X - sum_i W_i^T P_i, subtracted one
 *                     cluster at a time per element with the cluster's term in fp64 and rounded to X's element type
 *                     after each cluster.  dtype 0 = float32, 1 = float64 (X, X_out and X_cos_out).  X (row stride ld)
 *                     and X_out / X_cos_out (row stride ld_out) are host or device memory as the flags say.
 *                     clamp_zero != 0 writes max(x, 0).  X_cos_out (optional) = each cell's row of X_out divided by
 *                     its L2 norm (Z_cos; meaningful with clamp_zero = 0).  W_last (optional, host, n_phi x n_genes)
 *                     = W of the last cluster.
 * No floating-point atomics: repeated calls give identical bits.  Both synchronise. */
int cnmf_moe_grams(cnmf_handle_t h, const double* R, const double* Phi, const double* lamb, int K, int n_phi,
                   int n_cells, double* A_out, void* stream);
int cnmf_moe_correct(cnmf_handle_t h, const void* X, int dtype, int n_cells, int n_genes, long long ld,
                     int src_is_device, const double* R, const double* Phi, const double* A_inv, int K, int n_phi,
                     int clamp_zero, void* X_out, long long ld_out, int dst_is_device, void* X_cos_out,
                     double* W_last, void* stream);
/* stdscale_quantile_celing: X / std per column (ddof = 1, a zero std maps to 1, the division in fp64 rounded to the
 * element type), clipped at max_value when clip != 0; then, when k_lo >= 0, every value above the quantile threshold
 * is set to it.  The moments are summed in row order (numpy's axis-0 order), so that the std is the reference's bit
 * for bit.  A NaN anywhere in the scaled matrix makes the threshold NaN and leaves the matrix as scaled.  The threshold is numpy's linear-method lerp in the element type of the values of ranks k_lo and k_hi
 * (ascending over all n_rows * n_cols entries, found exactly by a radix select on the float bits) with weight gamma;
 * the caller derives k_lo, k_hi and gamma from the quantile as np.quantile does.  thresh_out (optional) receives it.
 * csr_row_ptr != NULL: X is the values array (nnz) of a host CSR matrix (csr_row_ptr: n_rows + 1 entries from 0,
 * csr_col_idx: nnz), densified on the device.  dtype as for cnmf_moe_correct.  Synchronises. */
int cnmf_scale_quantile_ceiling(cnmf_handle_t h, const void* X, int dtype, int n_rows, int n_cols, long long ld,
                                int src_is_device, const long long* csr_row_ptr, const int* csr_col_idx,
                                long long nnz, double max_value, int clip, long long k_lo, long long k_hi,
                                double gamma, void* X_out, long long ld_out, int dst_is_device, double* thresh_out,
                                void* stream);

#ifdef __cplusplus
}
#endif
#endif /* CNMF_B200_H */
