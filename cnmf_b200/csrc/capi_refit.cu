// extern "C": NNLS refits (cNMF.refit_usage / refit_spectra, cnmf.py:776-820), prediction error
// (cnmf.py:926-930), left projections for the OLS step (cnmf.py:98-119), column statistics,
// column-subset datasets (cnmf.py:965-969) and a raw GEMM hook used by tests / micro-benchmarks.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <vector>

#include "engine.h"
#include "gemm.h"
#include "nmf_kernels.cuh"

using namespace cnmf;

namespace {

__global__ void fill_kernel(float* p, float v, int rows, int n, int ld) {
  const long long total = (long long)rows * n;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
    p[(i / n) * ld + (i % n)] = v;
}

// column sums of v and v^2 with v = X[r, c] * (row_scale ? row_scale[r] : 1), fp64.  Threads own columns (coalesced),
// blockIdx.y owns a fixed strip of rows: partial[y][c], reduced in strip order by col_stats_reduce_kernel
// (deterministic: the HVG ranking of prepare() is a sort of these numbers).
template <typename T>
__global__ void col_stats_kernel(const T* __restrict__ X, int rows, int cols, int ld,
                                 const double* __restrict__ row_scale, double* __restrict__ part) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= cols) return;
  const int per = (rows + gridDim.y - 1) / gridDim.y;
  const int r0 = blockIdx.y * per, r1 = min(rows, r0 + per);
  double s = 0.0, q = 0.0;
  for (int r = r0; r < r1; ++r) {
    double v = X[(long long)r * ld + c];
    if (row_scale) v *= row_scale[r];
    s += v;
    q += v * v;
  }
  part[((long long)blockIdx.y * 2) * cols + c] = s;
  part[((long long)blockIdx.y * 2 + 1) * cols + c] = q;
}

// float64 datasets: dst[r, c] = src[r, cols[c]] / divisor[c] (one IEEE division, as numpy's X /= std)
__global__ void gather_cols_div_kernel(const double* __restrict__ src, int rows, int ld_src, const int* __restrict__ cols,
                                       const double* __restrict__ divisor, int n_cols, double* __restrict__ dst,
                                       int ld_dst) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_cols) return;
  const int sc = cols[c];
  const double f = divisor[c];
  for (int r = blockIdx.y; r < rows; r += gridDim.y)
    dst[(long long)r * ld_dst + c] = __ddiv_rn(src[(long long)r * ld_src + sc], f);
}

// out (n x k, dense) = F^T for F (k x ld, n valid columns)
__global__ void transpose64_kernel(const double* __restrict__ F, int k, int n, int ld, double* __restrict__ out) {
  const long long total = (long long)n * k;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
    out[i] = F[(i % k) * ld + i / k];
}

__global__ void col_stats_reduce_kernel(const double* __restrict__ part, int strips, int cols, double* __restrict__ out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= cols) return;
  double s = 0.0, q = 0.0;
  for (int y = 0; y < strips; ++y) {
    s += part[((long long)y * 2) * cols + c];
    q += part[((long long)y * 2 + 1) * cols + c];
  }
  out[c] = s;
  out[cols + c] = q;
}

// one warp per row: fp64 sum of the row (cell totals: the TPM denominators of cnmf.py:245-251)
__global__ void row_sums_kernel(const float* __restrict__ X, int rows, int cols, int ld, double* __restrict__ out) {
  const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (r >= rows) return;
  const float* row = X + (long long)r * ld;
  double s = 0.0;
  for (int c = lane; c < cols; c += 32) s += (double)row[c];
  s = warp_sum(s);
  if (lane == 0) out[r] = s;
}

__global__ void scale_rows_kernel(const float* __restrict__ src, int rows, int cols, int ld, const float* __restrict__ rs,
                                  float* __restrict__ dst) {
  const long long total = (long long)rows * (ld / 4);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(i / (ld / 4));
    float4 v = reinterpret_cast<const float4*>(src)[i];
    const float f = rs[r];
    v.x *= f; v.y *= f; v.z *= f; v.w *= f;
    reinterpret_cast<float4*>(dst)[i] = v;
  }
}

__global__ void combine_scale_kernel(const float* __restrict__ scale, const float* __restrict__ src_cs,
                                     const int* __restrict__ cols, int n, int n_pad, float* __restrict__ out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_pad) return;
  out[c] = (c < n) ? scale[c] * (src_cs ? src_cs[cols[c]] : 1.f) : 0.f;
}

__global__ void gather_cols_kernel(const float* __restrict__ src, int rows, int ld_src, const int* __restrict__ cols,
                                   const float* __restrict__ scale, int n_cols, float* __restrict__ dst, int ld_dst) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_cols) return;
  const int sc = cols[c];
  const float f = scale[c];
  for (int r = blockIdx.y; r < rows; r += gridDim.y) dst[(long long)r * ld_dst + c] = src[(long long)r * ld_src + sc] * f;
}

}  // namespace

extern "C" {

// column sums (mean_host) and sums of squares (var_host) over n rows -> mean and population variance, in place
static void finish_col_stats(double n, int n_cols, double* mean_host, double* var_host) {
  for (int c = 0; c < n_cols; ++c) {
    const double m = mean_host[c] / n;
    mean_host[c] = m;
    var_host[c] = std::max(var_host[c] / n - m * m, 0.0);
  }
}

static int col_stats_impl(cnmf_dataset_t d, const double* row_scale_host, double* mean_host, double* var_host, void* stream) {
  CNMF_REQUIRE(d && mean_host && var_host, "col_stats: NULL argument");
  cnmf_handle_s* h = d->h;
  cudaStream_t s = as_stream(stream);
  CNMF_CUDA_CHECK(cudaSetDevice(h->device));
  if (row_scale_host) CNMF_TRY(require_dense(d, "scaled_col_stats"));
  const bool f64 = d->precision == CNMF_PRECISION_FP64;
  double* buf = d->col_sums;        // sparse datasets: csc_col_stats_kernel ran at creation
  if (!d->sparse) {
    const int strips = std::max(1, std::min(64, d->n_rows / 64));
    double* part = static_cast<double*>(h->dev_buf("colstats.part", sizeof(double) * 2 * (size_t)strips * d->n_cols));
    buf = static_cast<double*>(h->dev_buf("colstats", sizeof(double) * 2 * d->n_cols));
    double* d_rs = nullptr;
    if (row_scale_host) {
      d_rs = static_cast<double*>(h->dev_buf("colstats.rs", sizeof(double) * d->n_rows));
      if (!d_rs) return -2;
      CNMF_CUDA_CHECK(cudaMemcpyAsync(d_rs, row_scale_host, sizeof(double) * d->n_rows, cudaMemcpyHostToDevice, s));
    }
    if (!part || !buf) return -2;
    dim3 grid((d->n_cols + 127) / 128, strips);
    if (f64) col_stats_kernel<<<grid, 128, 0, s>>>(d->X64, d->n_rows, d->n_cols, d->ld_c, d_rs, part);
    else col_stats_kernel<<<grid, 128, 0, s>>>(d->X, d->n_rows, d->n_cols, d->ld_c, d_rs, part);
    col_stats_reduce_kernel<<<(d->n_cols + 127) / 128, 128, 0, s>>>(part, strips, d->n_cols, buf);
    CNMF_CUDA_CHECK(cudaGetLastError());
    h->launches += 2;
  }
  CNMF_CUDA_CHECK(cudaMemcpyAsync(mean_host, buf, sizeof(double) * d->n_cols, cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaMemcpyAsync(var_host, buf + d->n_cols, sizeof(double) * d->n_cols, cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
  finish_col_stats(d->n_rows, d->n_cols, mean_host, var_host);
  return 0;
}

int cnmf_dataset_col_stats(cnmf_dataset_t d, double* mean_host, double* var_host, void* stream) {
  return col_stats_impl(d, nullptr, mean_host, var_host, stream);
}

int cnmf_dataset_scaled_col_stats(cnmf_dataset_t d, const double* row_scale_host, double* mean_host, double* var_host,
                                  void* stream) {
  CNMF_REQUIRE(row_scale_host, "scaled_col_stats: NULL row scale");
  return col_stats_impl(d, row_scale_host, mean_host, var_host, stream);
}

int cnmf_dataset_row_sums(cnmf_dataset_t d, double* row_sums_host, void* stream) {
  CNMF_REQUIRE(d && row_sums_host, "row_sums: NULL argument");
  CNMF_TRY(require_dense(d, "row_sums"));
  cnmf_handle_s* h = d->h;
  cudaStream_t s = as_stream(stream);
  CNMF_CUDA_CHECK(cudaSetDevice(h->device));
  double* buf = static_cast<double*>(h->dev_buf("rowsums", sizeof(double) * d->n_rows));
  if (!buf) return -2;
  row_sums_kernel<<<(d->n_rows + 7) / 8, 256, 0, s>>>(d->X, d->n_rows, d->n_cols, d->ld_c, buf);
  CNMF_CUDA_CHECK(cudaGetLastError());
  h->launches += 1;
  CNMF_CUDA_CHECK(cudaMemcpyAsync(row_sums_host, buf, sizeof(double) * d->n_rows, cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
  return 0;
}

int cnmf_dataset_tpm_stats(cnmf_dataset_t d, double target_sum, double* totals_host, double* mean_host,
                           double* var_host, void* stream) {
  CNMF_REQUIRE(d && totals_host && mean_host && var_host, "tpm_stats: NULL argument");
  if (!d->sparse) {
    set_last_error("tpm_stats is implemented for sparse (CSC) datasets only: a dense dataset gives the same numbers "
                   "through row_sums and scaled_col_stats");
    return -3;
  }
  cnmf_handle_s* h = d->h;
  cudaStream_t s = as_stream(stream);
  CNMF_CUDA_CHECK(cudaSetDevice(h->device));
  double* tot = static_cast<double*>(h->dev_buf("rowsums", sizeof(double) * d->n_rows));
  double* sums = static_cast<double*>(h->dev_buf("colstats", sizeof(double) * 2 * d->n_cols));
  if (!tot || !sums) return -2;
  CNMF_TRY(csc_tpm_sums(d, target_sum, tot, sums, s));
  CNMF_CUDA_CHECK(cudaMemcpyAsync(totals_host, tot, sizeof(double) * d->n_rows, cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaMemcpyAsync(mean_host, sums, sizeof(double) * d->n_cols, cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaMemcpyAsync(var_host, sums + d->n_cols, sizeof(double) * d->n_cols, cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
  finish_col_stats(d->n_rows, d->n_cols, mean_host, var_host);
  return 0;
}

int cnmf_dataset_from_columns(cnmf_dataset_t src, const int32_t* cols_host, const float* col_scale_host, int n_cols,
                              void* stream, cnmf_dataset_t* out) {
  CNMF_REQUIRE(src && cols_host && col_scale_host && out && n_cols > 0, "dataset_from_columns: bad arguments");
  CNMF_TRY(require_f32(src, "dataset_from_columns"));
  for (int c = 0; c < n_cols; ++c)
    CNMF_REQUIRE(cols_host[c] >= 0 && cols_host[c] < src->n_cols, "dataset_from_columns: column index out of range");
  cnmf_handle_s* h = src->h;
  cudaStream_t s = as_stream(stream);
  CNMF_CUDA_CHECK(cudaSetDevice(h->device));
  int* d_cols = static_cast<int*>(h->dev_buf("fromcols.idx", sizeof(int) * n_cols));
  float* d_scale = static_cast<float*>(h->dev_buf("fromcols.scale", sizeof(float) * n_cols));
  if (!d_cols || !d_scale) return -2;
  CNMF_CUDA_CHECK(cudaMemcpyAsync(d_cols, cols_host, sizeof(int) * n_cols, cudaMemcpyHostToDevice, s));
  CNMF_CUDA_CHECK(cudaMemcpyAsync(d_scale, col_scale_host, sizeof(float) * n_cols, cudaMemcpyHostToDevice, s));
  auto* d = new cnmf_dataset_s(h, src->n_rows, n_cols, src->precision);
  int rc = dataset_alloc(d, &d->X, (size_t)d->n_rows * d->ld_c);
  if (rc == 0) {
    cudaError_t e = cudaMemsetAsync(d->X, 0, (size_t)d->n_rows * d->ld_c * sizeof(float), s);
    if (e != cudaSuccess) rc = -2;
  }
  if (rc == 0 && src->sparse) {
    rc = csc_gather_cols(src, d_cols, d_scale, n_cols, d->X, d->ld_c, s);
  } else if (rc == 0) {
    dim3 grid((n_cols + 127) / 128, std::min(d->n_rows, 16384));
    gather_cols_kernel<<<grid, 128, 0, s>>>(src->X, d->n_rows, src->ld_c, d_cols, d_scale, n_cols, d->X, d->ld_c);
    h->launches += 1;
    if (cudaGetLastError() != cudaSuccess) rc = -2;
  }
  const bool exact = form_exact(src->form);
  if (rc == 0 && exact) {
    // an exact-count source stays exact: same integer matrix (the selected columns), same row scale, and the
    // column scale becomes scale[c] * src.col_scale[cols[c]]; finish() rebuilds C from the scaled values
    rc = dataset_alloc(d, &d->col_scale, (size_t)d->ld_c);
    if (rc == 0) {
      combine_scale_kernel<<<(d->ld_c + 255) / 256, 256, 0, s>>>(d_scale, src->col_scale, d_cols, n_cols, d->ld_c, d->col_scale);
      h->launches += 1;
      if (cudaGetLastError() != cudaSuccess) rc = -2;
    }
    if (rc == 0 && src->row_scale) {
      rc = dataset_alloc(d, &d->row_scale, (size_t)d->ld_r);
      if (rc == 0 && cudaMemcpyAsync(d->row_scale, src->row_scale, sizeof(float) * d->ld_r, cudaMemcpyDeviceToDevice, s) != cudaSuccess)
        rc = -2;
    }
  }
  if (rc == 0) rc = dataset_finish(d, s, exact);
  if (rc != 0) {
    cnmf_dataset_destroy(d);
    return rc;
  }
  *out = d;
  return 0;
}

int cnmf_dataset_scale_rows(cnmf_dataset_t src, const float* row_scale_host, void* stream, cnmf_dataset_t* out) {
  CNMF_REQUIRE(src && row_scale_host && out, "dataset_scale_rows: bad arguments");
  CNMF_TRY(require_dense(src, "scale_rows"));
  cnmf_handle_s* h = src->h;
  cudaStream_t s = as_stream(stream);
  CNMF_CUDA_CHECK(cudaSetDevice(h->device));
  float* d_rs = static_cast<float*>(h->dev_buf("scalerows.rs", sizeof(float) * src->n_rows));
  if (!d_rs) return -2;
  CNMF_CUDA_CHECK(cudaMemcpyAsync(d_rs, row_scale_host, sizeof(float) * src->n_rows, cudaMemcpyHostToDevice, s));
  auto* d = new cnmf_dataset_s(h, src->n_rows, src->n_cols, src->precision);
  int rc = dataset_alloc(d, &d->X, (size_t)d->n_rows * d->ld_c);
  if (rc == 0) {
    scale_rows_kernel<<<NUM_SMS * 8, 256, 0, s>>>(src->X, d->n_rows, d->n_cols, d->ld_c, d_rs, d->X);
    h->launches += 1;
    if (cudaGetLastError() != cudaSuccess) rc = -2;
  }
  // exact-count detection runs from scratch in finish(): counts x (1e6 / cell total) is again scaled integers
  if (rc == 0) rc = dataset_finish(d, s);
  if (rc != 0) {
    cnmf_dataset_destroy(d);
    return rc;
  }
  *out = d;
  return 0;
}

// --------------------------------------------------------------------------------- refit
int cnmf_refit(cnmf_dataset_t d, int transposed, int k, const float* fixed_host, const cnmf_nmf_params* p,
               float* out_host, int32_t* n_iter_host, double* err_host, void* stream) {
  CNMF_REQUIRE(d && fixed_host && p && out_host, "refit: NULL argument");
  CNMF_TRY(require_f32(d, "refit"));
  CNMF_TRY(check_params_precision(d, p));
  CNMF_REQUIRE(k >= 1 && k <= KMAX, "refit: n_components must be in [1, 32] on the CUDA path");
  if (d->sparse && !transposed) CNMF_TRY(require_dense(d, "refit with transposed = 0"));
  if (d->sparse && p->beta_loss != CNMF_LOSS_FROBENIUS) CNMF_TRY(require_dense(d, "refit with a KL / IS beta_loss"));
  const auto t_enter = std::chrono::steady_clock::now();
  cnmf_handle_s* h = d->h;
  cudaStream_t s = as_stream(stream);
  CNMF_CUDA_CHECK(cudaSetDevice(h->device));
  // sparse datasets: the one product X^T W is formed by csc_project_kernel in fp64 before the solve, which then
  // iterates on K x K Grams only -- no GEMM runs, so no operand pieces are made (make_view: FP32 form)
  if (p->beta_loss != CNMF_LOSS_FROBENIUS) CNMF_TRY(dataset_ensure_full_transpose(d, s));
  const DataView v = make_view(d, transposed != 0);

  const size_t nr = (size_t)k * v.ld_r, nc = (size_t)k * v.ld_c;
  float* Fr = static_cast<float*>(h->dev_buf("refit.Fr", nr * 4));
  float* Fc = static_cast<float*>(h->dev_buf("refit.Fc", nc * 4));
  if (!Fr || !Fc) return -2;
  CNMF_CUDA_CHECK(cudaMemsetAsync(Fr, 0, nr * 4, s));
  CNMF_CUDA_CHECK(cudaMemsetAsync(Fc, 0, nc * 4, s));
  CNMF_CUDA_CHECK(cudaMemcpy2DAsync(Fc, (size_t)v.ld_c * 4, fixed_host, (size_t)v.n_c * 4, (size_t)v.n_c * 4, k,
                                    cudaMemcpyHostToDevice, s));
  if (p->solver == CNMF_SOLVER_MU) {
    // sklearn _nmf.py:1223-1226: W = full(sqrt(X.mean() / k))
    const double mean = v.sum / ((double)v.n_r * (double)v.n_c);
    fill_kernel<<<NUM_SMS * 4, 256, 0, s>>>(Fr, (float)std::sqrt(mean / k), k, v.n_r, v.ld_r);
    CNMF_CUDA_CHECK(cudaGetLastError());
    h->launches += 1;
  }  // 'cd': zeros (sklearn _nmf.py:1227-1228)
  SolveIO<float> io;
  io.R = 1;
  io.ks = {k};
  io.Fr = Fr;
  io.Fc = Fc;
  io.update_cols = false;
  if (d->sparse) {
    const int kp = round_up(k, 4);
    float* U = static_cast<float*>(h->dev_buf("refit.U", (size_t)v.n_c * kp * 4));
    float* NUM = static_cast<float*>(h->dev_buf("refit.NUM", nr * 4));
    if (!U || !NUM) return -2;
    CNMF_CUDA_CHECK(cudaMemsetAsync(NUM, 0, nr * 4, s));
    CNMF_TRY(stage_rows(h, Fc, k, v.n_c, v.ld_c, kp, U, s));
    CNMF_TRY(csc_project(d, U, k, kp, NUM, v.ld_r, s));
    io.num_rows = NUM;
  }
  auto t_solve = std::chrono::steady_clock::now();
  if (h->profile) {
    CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
    h->t_h2d_ms = std::chrono::duration<double, std::milli>(t_solve - t_enter).count();
    t_solve = std::chrono::steady_clock::now();
  }
  CNMF_TRY(solve_batched(h, v, io, *p, s));
  if (h->profile) h->t_solve_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_solve).count();

  // Fr is k x n_r; the caller wants n_r x k (row-major).  Transposed on the device into a COMPACT n_r x k array and
  // copied back in one contiguous transfer through pinned memory: a pitched 2-D copy of 50 000 rows of ~40 bytes to
  // pageable memory can take longer than the solve itself.
  float* T = static_cast<float*>(h->dev_buf("refit.T", (size_t)v.n_r * k * 4));
  float* T_host = static_cast<float*>(h->host_buf("refit.T_host", (size_t)v.n_r * k * 4));
  if (!T || !T_host) return -2;
  CNMF_TRY(launch_transpose(Fr, k, v.n_r, v.ld_r, T, nullptr, nullptr, k, s));
  h->launches += 1;
  CNMF_CUDA_CHECK(cudaMemcpyAsync(T_host, T, (size_t)v.n_r * k * 4, cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
  std::memcpy(out_host, T_host, (size_t)v.n_r * k * 4);
  if (n_iter_host) *n_iter_host = io.n_iter[0];
  if (err_host) *err_host = io.err[0];
  return 0;
}

// --------------------------------------------------------------------------------- projections
// out (k x n_cols) = Ut (k x n_rows) * X  -- the X^T Y accumulator of efficient_ols_all_cols (cnmf.py:119)
int cnmf_project_rows(cnmf_dataset_t d, int k, const float* Ut_host, float* out_host, void* stream) {
  CNMF_REQUIRE(d && Ut_host && out_host && k >= 1, "project_rows: bad arguments");
  CNMF_TRY(require_f32(d, "project_rows"));
  cnmf_handle_s* h = d->h;
  cudaStream_t s = as_stream(stream);
  CNMF_CUDA_CHECK(cudaSetDevice(h->device));
  if (d->sparse) {       // fp64 products and sums in a fixed order (csc_project_kernel), one rounding to fp32
    CNMF_REQUIRE(k <= KMAX, "project_rows: k must be <= 32 on a sparse dataset");
    const int kp = round_up(k, 4);
    float* Ut = static_cast<float*>(h->dev_buf("proj.Ut", (size_t)k * d->n_rows * 4));
    float* U = static_cast<float*>(h->dev_buf("proj.U", (size_t)d->n_rows * kp * 4));
    float* C = static_cast<float*>(h->dev_buf("proj.C", (size_t)k * d->ld_c * 4));
    if (!Ut || !U || !C) return -2;
    CNMF_CUDA_CHECK(cudaMemcpyAsync(Ut, Ut_host, (size_t)k * d->n_rows * 4, cudaMemcpyHostToDevice, s));
    CNMF_TRY(stage_rows(h, Ut, k, d->n_rows, d->n_rows, kp, U, s));
    CNMF_TRY(csc_project(d, U, k, kp, C, d->ld_c, s));
    CNMF_CUDA_CHECK(cudaMemcpy2DAsync(out_host, (size_t)d->n_cols * 4, C, (size_t)d->ld_c * 4, (size_t)d->n_cols * 4, k,
                                      cudaMemcpyDeviceToHost, s));
    CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
    return 0;
  }
  const DataView v = make_view(d, false);     // out = the solver's NUM_c product of the rows Ut
  const size_t nr = (size_t)k * d->ld_r;
  float* A = static_cast<float*>(h->dev_buf("proj.A", nr * 4));
  float *A_hi = nullptr, *A_lo = nullptr, *A_rs = nullptr;
  if (!A) return -2;
  CNMF_CUDA_CHECK(cudaMemsetAsync(A, 0, nr * 4, s));
  CNMF_CUDA_CHECK(cudaMemcpy2DAsync(A, (size_t)d->ld_r * 4, Ut_host, (size_t)d->n_rows * 4, (size_t)d->n_rows * 4, k,
                                    cudaMemcpyHostToDevice, s));
  if (v.form != Form::FP32) {     // pieces of the (signed) rows; on f16 datasets two fp16 pieces with group scales
    A_hi = static_cast<float*>(h->dev_buf("proj.A_hi", nr * 4));
    A_lo = static_cast<float*>(h->dev_buf("proj.A_lo", nr * 4));
    if (!A_hi || !A_lo) return -2;
    if (v.form == Form::F16_EXACT) {
      A_rs = static_cast<float*>(h->dev_buf("proj.A_rs", sizeof(float) * (size_t)k * ((d->ld_r + 511) / 512)));
      if (!A_rs) return -2;
    }
    CNMF_TRY(make_pieces(v.form, A, k, d->n_rows, d->ld_r, v.scale_r, A_hi, A_lo, A_rs, s));
    h->launches += 1;
  }
  GemmArgs g{};
  g.M = k; g.N = d->n_cols; g.Kd = d->n_rows;
  g.lda = d->ld_r; g.ldb = d->ld_r; g.ldc = d->ld_c;
  int splits = 1;
  {
    const int tiles = ((k + 127) / 128) * ((d->n_cols + 255) / 256);
    if (tiles < 2 * h->sm_count) splits = (2 * h->sm_count + tiles - 1) / tiles;
    splits = std::min(splits, std::max(1, ((d->n_rows + 31) / 32) / 8));
    splits = std::min(splits, 32);
    splits = gemm_effective_splits(d->n_rows, splits, v.form == Form::F16_EXACT ? 1 : 0);
  }
  g.splits = g.splits_effective = splits;
  g.c_split_stride = (long long)k * d->ld_c;
  float* C = static_cast<float*>(h->dev_buf("proj.C", (size_t)splits * k * d->ld_c * 4));
  if (!C) return -2;
  g.C = C;
  CNMF_TRY(form_gemm(v.form, g, A, A_hi, A_lo, A_rs, v.B_cols, v.scale_c, s));
  h->launches += 1;
  std::vector<float> tmp((size_t)splits * k * d->ld_c);
  CNMF_CUDA_CHECK(cudaMemcpyAsync(tmp.data(), C, tmp.size() * 4, cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
  for (int c = 0; c < k; ++c)
    for (int j = 0; j < d->n_cols; ++j) {
      double a = 0.0;
      for (int z = 0; z < splits; ++z) a += tmp[(size_t)z * k * d->ld_c + (size_t)c * d->ld_c + j];
      out_host[(size_t)c * d->n_cols + j] = (float)a;
    }
  return 0;
}

// --------------------------------------------------------------------------------- float64 datasets
int cnmf_dataset_from_columns_f64(cnmf_dataset_t src, const int32_t* cols_host, const double* divisor_host, int n_cols,
                                  void* stream, cnmf_dataset_t* out) {
  CNMF_REQUIRE(src && cols_host && divisor_host && out && n_cols > 0, "dataset_from_columns_f64: bad arguments");
  CNMF_TRY(require_f64(src, "dataset_from_columns"));
  for (int c = 0; c < n_cols; ++c)
    CNMF_REQUIRE(cols_host[c] >= 0 && cols_host[c] < src->n_cols, "dataset_from_columns_f64: column index out of range");
  cnmf_handle_s* h = src->h;
  cudaStream_t s = as_stream(stream);
  CNMF_CUDA_CHECK(cudaSetDevice(h->device));
  int* d_cols = static_cast<int*>(h->dev_buf("fromcols.idx", sizeof(int) * n_cols));
  double* d_div = static_cast<double*>(h->dev_buf("fromcols.div64", sizeof(double) * n_cols));
  if (!d_cols || !d_div) return -2;
  CNMF_CUDA_CHECK(cudaMemcpyAsync(d_cols, cols_host, sizeof(int) * n_cols, cudaMemcpyHostToDevice, s));
  CNMF_CUDA_CHECK(cudaMemcpyAsync(d_div, divisor_host, sizeof(double) * n_cols, cudaMemcpyHostToDevice, s));
  auto* d = new cnmf_dataset_s(h, src->n_rows, n_cols, CNMF_PRECISION_FP64);
  d->form = Form::FP64;
  const size_t nx = (size_t)d->n_rows * d->ld_c;
  float* buf = nullptr;
  int rc = dataset_alloc(d, &buf, 2 * nx);
  if (rc == 0) {
    d->X64 = reinterpret_cast<double*>(buf);
    if (cudaMemsetAsync(d->X64, 0, nx * sizeof(double), s) != cudaSuccess) rc = -2;
  }
  if (rc == 0) {
    dim3 grid((n_cols + 127) / 128, std::min(d->n_rows, 16384));
    gather_cols_div_kernel<<<grid, 128, 0, s>>>(src->X64, d->n_rows, src->ld_c, d_cols, d_div, n_cols, d->X64, d->ld_c);
    h->launches += 1;
    if (cudaGetLastError() != cudaSuccess) rc = -2;
  }
  double sums[2] = {0.0, 0.0};
  if (rc == 0) rc = matrix_sums_f64(h, d->X64, d->n_rows, d->n_cols, d->ld_c, sums, s);
  if (rc != 0) {
    cnmf_dataset_destroy(d);
    return rc;
  }
  d->sum = sums[0];
  d->sum_sq = sums[1];
  *out = d;
  return 0;
}

int cnmf_refit_f64(cnmf_dataset_t d, int transposed, int k, const double* fixed_host, const cnmf_nmf_params* p,
                   double* out_host, int32_t* n_iter_host, double* err_host, void* stream) {
  CNMF_REQUIRE(d && fixed_host && p && out_host, "refit_f64: NULL argument");
  CNMF_TRY(require_f64(d, "refit"));
  CNMF_TRY(check_params_precision(d, p));
  CNMF_REQUIRE(k >= 1 && k <= KMAX, "refit_f64: n_components must be in [1, 32] on the CUDA path");
  if (p->beta_loss != CNMF_LOSS_FROBENIUS) {
    set_last_error("cnmf_refit_f64: float64 datasets support beta_loss = frobenius only");
    return -3;
  }
  cnmf_handle_s* h = d->h;
  cudaStream_t s = as_stream(stream);
  CNMF_CUDA_CHECK(cudaSetDevice(h->device));
  const DataView v = make_view(d, transposed != 0);
  const size_t nr = (size_t)k * v.ld_r, nc = (size_t)k * v.ld_c;
  double* Fr = static_cast<double*>(h->dev_buf("refit.Fr64", nr * 8));
  double* Fc = static_cast<double*>(h->dev_buf("refit.Fc64", nc * 8));
  double* T = static_cast<double*>(h->dev_buf("refit.T64", (size_t)v.n_r * k * 8));
  if (!Fr || !Fc || !T) return -2;
  CNMF_CUDA_CHECK(cudaMemsetAsync(Fr, 0, nr * 8, s));
  CNMF_CUDA_CHECK(cudaMemsetAsync(Fc, 0, nc * 8, s));
  CNMF_CUDA_CHECK(cudaMemcpy2DAsync(Fc, (size_t)v.ld_c * 8, fixed_host, (size_t)v.n_c * 8, (size_t)v.n_c * 8, k,
                                    cudaMemcpyHostToDevice, s));
  if (p->solver == CNMF_SOLVER_MU) {
    // sklearn _nmf.py:1223-1226: W = full(sqrt(X.mean() / k))
    const double mean = v.sum / ((double)v.n_r * (double)v.n_c);
    CNMF_TRY(fill_f64(Fr, std::sqrt(mean / k), k, v.n_r, v.ld_r, s));
    h->launches += 1;
  }  // 'cd': zeros (sklearn _nmf.py:1227-1228)
  SolveIO<double> io;
  io.R = 1;
  io.ks = {k};
  io.Fr = Fr;
  io.Fc = Fc;
  io.update_cols = false;
  CNMF_TRY(solve_batched(h, v, io, *p, s));
  transpose64_kernel<<<NUM_SMS * 4, 256, 0, s>>>(Fr, k, v.n_r, v.ld_r, T);
  CNMF_CUDA_CHECK(cudaGetLastError());
  h->launches += 1;
  CNMF_CUDA_CHECK(cudaMemcpyAsync(out_host, T, (size_t)v.n_r * k * 8, cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
  if (n_iter_host) *n_iter_host = io.n_iter[0];
  if (err_host) *err_host = io.err[0];
  return 0;
}

int cnmf_project_rows_f64(cnmf_dataset_t d, int k, const double* Ut_host, double* out_host, void* stream) {
  CNMF_REQUIRE(d && Ut_host && out_host && k >= 1, "project_rows_f64: bad arguments");
  CNMF_TRY(require_f64(d, "project_rows"));
  cnmf_handle_s* h = d->h;
  cudaStream_t s = as_stream(stream);
  CNMF_CUDA_CHECK(cudaSetDevice(h->device));
  const size_t na = (size_t)k * d->ld_r, nc = (size_t)k * d->ld_c;
  double* A = static_cast<double*>(h->dev_buf("proj.A64", na * 8));
  double* C = static_cast<double*>(h->dev_buf("proj.C64", nc * 8));
  if (!A || !C) return -2;
  CNMF_CUDA_CHECK(cudaMemsetAsync(A, 0, na * 8, s));
  CNMF_CUDA_CHECK(cudaMemcpy2DAsync(A, (size_t)d->ld_r * 8, Ut_host, (size_t)d->n_rows * 8, (size_t)d->n_rows * 8, k,
                                    cudaMemcpyHostToDevice, s));
  h->launches += 1;
  CNMF_TRY(launch_gemm_f64(A, d->ld_r, k, d->X64, d->n_rows, d->n_cols, d->ld_c, true, C, d->ld_c, s));
  CNMF_CUDA_CHECK(cudaMemcpy2DAsync(out_host, (size_t)d->n_cols * 8, C, (size_t)d->ld_c * 8, (size_t)d->n_cols * 8, k,
                                    cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
  return 0;
}

// --------------------------------------------------------------------------------- raw GEMM hook
// C (M x N) = A (M x Kd) * B (N x Kd)^T on host buffers; reps > 1 re-runs the kernel and reports the
// mean device time per launch in *ms_out (CUDA events).  Used by tests and by the roofline micro-bench.
// Exact forms (b_exact, f16x2): A diag(k_scale) goes into the A pieces and out_col_scale onto C, as in the solver.
int cnmf_gemm_abt_host(cnmf_handle_t h, int precision, const float* A, const float* B, int M, int N, int Kd, int splits,
                       int b_exact, const float* k_scale, const float* out_col_scale, int tile_n, float* C, int reps,
                       float* ms_out, void* stream) {
  CNMF_REQUIRE(h && A && B && C && M > 0 && N > 0 && Kd > 0, "gemm_abt_host: bad arguments");
  const bool f16 = precision == CNMF_PRECISION_F16X2;    // B must hold integers <= 2048 (exact in fp16)
  CNMF_REQUIRE(!b_exact || f16 || precision == CNMF_PRECISION_TF32X3, "gemm_abt_host: b_exact needs tf32x3 or f16x2");
  const bool exact = f16 || b_exact;
  CNMF_REQUIRE(exact || (!k_scale && !out_col_scale), "gemm_abt_host: k_scale / out_col_scale need an exact form");
  // the dataset form whose GEMM this runs; precisions other than tf32x3 and f16x2 run the fp32 path
  const Form form = f16 ? Form::F16_EXACT
                  : precision != CNMF_PRECISION_TF32X3 ? Form::FP32
                  : b_exact ? Form::TF32_EXACT : Form::TF32;
  cudaStream_t s = as_stream(stream);
  CNMF_CUDA_CHECK(cudaSetDevice(h->device));
  const int lda = pad_ld(Kd), ldc = pad_ld(N);
  const size_t na = (size_t)M * lda, nb = (size_t)N * lda;
  float* dA = static_cast<float*>(h->dev_buf("gemmtest.A", na * 4));
  float* dB = static_cast<float*>(h->dev_buf("gemmtest.B", nb * 4));
  float* dAh = static_cast<float*>(h->dev_buf("gemmtest.Ah", na * 4));
  float* dAl = static_cast<float*>(h->dev_buf("gemmtest.Al", na * 4));
  float* dBh = static_cast<float*>(h->dev_buf("gemmtest.Bh", nb * 4));
  float* dBl = static_cast<float*>(h->dev_buf("gemmtest.Bl", nb * 4));
  const int se = gemm_effective_splits(Kd, splits, f16 ? 1 : 0);
  float* dC = static_cast<float*>(h->dev_buf("gemmtest.C", (size_t)se * M * ldc * 4));
  float* dRs = static_cast<float*>(h->dev_buf("gemmtest.rs", sizeof(float) * (size_t)M * ((lda + 511) / 512)));
  if (!dA || !dB || !dAh || !dAl || !dBh || !dBl || !dC || !dRs) return -2;
  CNMF_CUDA_CHECK(cudaMemsetAsync(dA, 0, na * 4, s));
  CNMF_CUDA_CHECK(cudaMemsetAsync(dB, 0, nb * 4, s));
  CNMF_CUDA_CHECK(cudaMemcpy2DAsync(dA, (size_t)lda * 4, A, (size_t)Kd * 4, (size_t)Kd * 4, M, cudaMemcpyHostToDevice, s));
  CNMF_CUDA_CHECK(cudaMemcpy2DAsync(dB, (size_t)lda * 4, B, (size_t)Kd * 4, (size_t)Kd * 4, N, cudaMemcpyHostToDevice, s));
  // the scales as the solver holds a dataset's: zero-padded to the row stride, 16-byte aligned (dev_buf)
  float* dKs = nullptr;
  float* dCs = nullptr;
  if (k_scale) {
    dKs = static_cast<float*>(h->dev_buf("gemmtest.kscale", (size_t)lda * 4));
    if (!dKs) return -2;
    CNMF_CUDA_CHECK(cudaMemsetAsync(dKs, 0, (size_t)lda * 4, s));
    CNMF_CUDA_CHECK(cudaMemcpyAsync(dKs, k_scale, (size_t)Kd * 4, cudaMemcpyHostToDevice, s));
  }
  if (out_col_scale) {
    dCs = static_cast<float*>(h->dev_buf("gemmtest.cscale", (size_t)ldc * 4));
    if (!dCs) return -2;
    CNMF_CUDA_CHECK(cudaMemsetAsync(dCs, 0, (size_t)ldc * 4, s));
    CNMF_CUDA_CHECK(cudaMemcpyAsync(dCs, out_col_scale, (size_t)N * 4, cudaMemcpyHostToDevice, s));
  }
  // B as a dataset of that form holds it: fp16 (integers <= 2048), tf32 pieces (exact forms read only hi), or as is
  if (f16) CNMF_TRY(launch_to_half(dB, dBh, (long long)nb, s));
  else if (form != Form::FP32) CNMF_TRY(launch_split_tf32(dB, dBh, dBl, (long long)nb, s));
  CNMF_TRY(make_pieces(form, dA, M, Kd, lda, dKs, dAh, dAl, dRs, s));
  CNMF_CUDA_CHECK(cudaMemsetAsync(dC, 0xff, (size_t)se * M * ldc * 4, s));   // NaN pattern: unwritten outputs show up
  GemmArgs g{};
  g.M = M; g.N = N; g.Kd = Kd; g.lda = lda; g.ldb = lda; g.ldc = ldc;
  g.C = dC; g.c_split_stride = (long long)M * ldc; g.splits = splits; g.splits_effective = se;
  g.tile_n = tile_n;
  const Operand Bop{dB, dBh, dBl, N, Kd, lda};
  cudaEvent_t e0, e1;
  CNMF_CUDA_CHECK(cudaEventCreate(&e0));
  CNMF_CUDA_CHECK(cudaEventCreate(&e1));
  if (reps < 1) reps = 1;
  int rc = form_gemm(form, g, dA, dAh, dAl, dRs, Bop, dCs, s);   // warm-up + result
  if (rc == 0 && reps > 1) {
    cudaEventRecord(e0, s);
    for (int i = 0; i < reps && rc == 0; ++i) rc = form_gemm(form, g, dA, dAh, dAl, dRs, Bop, dCs, s);
    cudaEventRecord(e1, s);
  }
  h->launches += reps;
  if (rc != 0) return rc;
  std::vector<float> tmp((size_t)se * M * ldc);
  CNMF_CUDA_CHECK(cudaMemcpyAsync(tmp.data(), dC, tmp.size() * 4, cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
  if (ms_out) {
    float ms = 0.f;
    if (reps > 1) cudaEventElapsedTime(&ms, e0, e1);
    *ms_out = reps > 1 ? ms / reps : 0.f;
  }
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  for (int m = 0; m < M; ++m)
    for (int n = 0; n < N; ++n) {
      double a = 0.0;
      for (int z = 0; z < se; ++z) a += tmp[(size_t)z * M * ldc + (size_t)m * ldc + n];
      C[(size_t)m * N + n] = (float)a;
    }
  return 0;
}

}  // extern "C"
