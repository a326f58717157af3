// Sparse (CSC) datasets: the TPM matrix of the consensus step (cnmf.py:950-969) kept as canonical CSC on the device
// instead of the dense forms, for matrices whose dense forms do not fit.  Every use of the TPM in consensus touches it
// in a single product or a column pass, so three kernels cover them:
//   csc_project_kernel     out (k x G) = U^T X : the OLS accumulator (cnmf.py:119) and the one product X^T W of
//                          refit_spectra (cnmf.py:952), after which the refit iterates on K x K Grams only
//   csc_col_stats_kernel   per-column sum(x), sum(x^2) in fp64: col_stats and the refit's ||X||^2 and mean(X)
//   csc_gather_cols_kernel X[:, cols] * scale into a dense matrix: the HVG dataset of cnmf.py:965-969
// The same CSC form holds raw counts for prepare (cnmf.py:245-251, 436-445) when their dense dataset does not fit:
//   csc_row_partials_kernel + csc_row_totals_kernel   cell totals and the TPM row scale
//   csc_scaled_col_sums_kernel                         per-column sums of the TPM, formed entry by entry
// Products and sums run in fp64 in a fixed order, without floating-point atomics: two runs are bit-identical.
#include <algorithm>
#include <string>
#include <type_traits>
#include <vector>

#include "engine.h"
#include "nmf_kernels.cuh"

using namespace cnmf;

namespace {

constexpr int WARPS = 8;    // warps per block of the warp-per-column / warp-per-chunk kernels
constexpr int TPM_SLABS = 128;   // most column slabs of the cell-total reduction (csc_row_partials_kernel)

// One warp per chunk item (at most CSC_CHUNK entries of one column).  The kp / 4 lanes of a strand share one entry:
// lane q of the strand gathers float4 number q of the entry's U row, so an entry costs one contiguous kp-float read.
// The 32 / (kp / 4) strands take the chunk's entries round robin; their fp64 partials are added in strand order.
__global__ void __launch_bounds__(WARPS * 32) csc_project_kernel(const long long* __restrict__ col_ptr,
                                                                 const int* __restrict__ row_idx,
                                                                 const float* __restrict__ vals,
                                                                 const int* __restrict__ item_ptr, int n_cols,
                                                                 int n_items, const float4* __restrict__ U, int kp,
                                                                 double* __restrict__ part) {
  __shared__ double acc_s[WARPS][32 * 4];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int G = kp >> 2;             // lanes per strand
  const int P = 32 / G;              // strands per warp
  const int strand = lane / G, q = lane - strand * G;
  double* acc_w = acc_s[warp];
  for (int item = blockIdx.x * WARPS + warp; item < n_items; item += gridDim.x * WARPS) {
    // column of the item: last c with item_ptr[c] <= item
    int lo = 0, hi = n_cols;
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (item_ptr[mid] <= item) lo = mid; else hi = mid;
    }
    const long long beg = col_ptr[lo] + (long long)(item - item_ptr[lo]) * CSC_CHUNK;
    const long long end = min(beg + CSC_CHUNK, col_ptr[lo + 1]);
    double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;
    if (strand < P) {
#pragma unroll 4
      for (long long j = beg + strand; j < end; j += P) {
        const double v = vals[j];
        const float4 u = U[(long long)row_idx[j] * G + q];
        // fp32 x fp32 is exact in fp64: the fma rounds once, like the separate add
        a0 = fma((double)u.x, v, a0);
        a1 = fma((double)u.y, v, a1);
        a2 = fma((double)u.z, v, a2);
        a3 = fma((double)u.w, v, a3);
      }
    }
    // lane = strand * G + q holds components 4q..4q+3 of its strand: acc_w[strand * kp + c]
    acc_w[lane * 4 + 0] = a0;
    acc_w[lane * 4 + 1] = a1;
    acc_w[lane * 4 + 2] = a2;
    acc_w[lane * 4 + 3] = a3;
    __syncwarp();
    if (lane < kp) {
      double t = 0.0;
      for (int s = 0; s < P; ++s) t += acc_w[s * kp + lane];
      part[(long long)item * kp + lane] = t;
    }
    __syncwarp();
  }
}

// out[c][col] = sum of the column's chunk partials in chunk order, rounded to fp32 once
__global__ void csc_project_reduce_kernel(const double* __restrict__ part, const int* __restrict__ item_ptr, int n_cols,
                                          int k, int kp, float* __restrict__ out, int ld) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)k * n_cols) return;
  const int c = (int)(i / n_cols), col = (int)(i % n_cols);
  double t = 0.0;
  for (int it = item_ptr[col]; it < item_ptr[col + 1]; ++it) t += part[(long long)it * kp + c];
  out[(long long)c * ld + col] = (float)t;
}

// U (n x kp) <- F^T for F (k x ld, first n columns), zero beyond k
__global__ void stage_rows_kernel(const float* __restrict__ F, int k, int n, int ld, int kp, float* __restrict__ U) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)n * kp) return;
  const int r = (int)(i / kp), c = (int)(i % kp);
  U[i] = c < k ? F[(long long)c * ld + r] : 0.f;
}

// one warp per column: sum(x), sum(x^2) in fp64 (lane strides, then the xor tree of warp_sum: a fixed order)
__global__ void __launch_bounds__(WARPS * 32) csc_col_stats_kernel(const long long* __restrict__ col_ptr,
                                                                   const float* __restrict__ vals, int n_cols,
                                                                   double* __restrict__ col_sums) {
  const int col = blockIdx.x * WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (col >= n_cols) return;
  double s = 0.0, q = 0.0;
  for (long long j = col_ptr[col] + lane; j < col_ptr[col + 1]; j += 32) {
    const double v = vals[j];
    s += v;
    q = fma(v, v, q);
  }
  s = warp_sum(s);
  q = warp_sum(q);
  if (lane == 0) {
    col_sums[col] = s;
    col_sums[n_cols + col] = q;
  }
}

// dataset totals from the column sums: one block, fixed strides, fixed tree
__global__ void csc_totals_kernel(const double* __restrict__ col_sums, int n_cols, double* __restrict__ out) {
  __shared__ double sh[2][256];
  double s = 0.0, q = 0.0;
  for (int c = threadIdx.x; c < n_cols; c += 256) {
    s += col_sums[c];
    q += col_sums[n_cols + c];
  }
  sh[0][threadIdx.x] = s;
  sh[1][threadIdx.x] = q;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      sh[0][threadIdx.x] += sh[0][threadIdx.x + o];
      sh[1][threadIdx.x] += sh[1][threadIdx.x + o];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    out[0] = sh[0][0];
    out[1] = sh[1][0];
  }
}

// smallest positive stored value per column and per row, as int bit patterns (positive floats order like them);
// both arrays start at 0x7f7f7f7f.  Integer atomics: the result does not depend on the order.
__global__ void csc_min_positive_kernel(const long long* __restrict__ col_ptr, const int* __restrict__ row_idx,
                                        const float* __restrict__ vals, int n_cols, int* __restrict__ col_min,
                                        int* __restrict__ row_min) {
  const int col = blockIdx.x * WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (col >= n_cols) return;
  int cm = 0x7f7f7f7f;
  for (long long j = col_ptr[col] + lane; j < col_ptr[col + 1]; j += 32) {
    const float v = vals[j];
    if (v > 0.f) {
      cm = min(cm, __float_as_int(v));
      atomicMin(&row_min[row_idx[j]], __float_as_int(v));
    }
  }
  for (int o = 16; o > 0; o >>= 1) cm = min(cm, __shfl_xor_sync(0xffffffffu, cm, o));
  if (lane == 0) col_min[col] = cm;
}

// entries that are not an integer multiple of their column scale (n_bad[0]) / row scale (n_bad[1])
__global__ void csc_check_scaled_int_kernel(const long long* __restrict__ col_ptr, const int* __restrict__ row_idx,
                                            const float* __restrict__ vals, int n_cols, const float* __restrict__ cs,
                                            const float* __restrict__ rs, int* __restrict__ n_bad) {
  const int col = blockIdx.x * WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (col >= n_cols) return;
  int bad_c = 0, bad_r = 0;
  for (long long j = col_ptr[col] + lane; j < col_ptr[col + 1]; j += 32) {
    const float v = vals[j];
    if (v == 0.f) continue;
    bad_c += !is_scaled_int(v, cs[col]);
    bad_r += !is_scaled_int(v, rs[row_idx[j]]);
  }
  bad_c = warp_sum(bad_c);
  bad_r = warp_sum(bad_r);
  if (lane == 0 && bad_c) atomicAdd(&n_bad[0], bad_c);
  if (lane == 0 && bad_r) atomicAdd(&n_bad[1], bad_r);
}

// Cell totals, pass 1 (prepare on sparse counts): slab s, one block, owns the columns whose entries start in
// [nnz * s / S, nnz * (s + 1) / S) and adds them into its own fp64 row vector part[s], one column at a time.  The row
// indices of a canonical CSC column are distinct, so the threads of one column never touch the same row, and the
// barrier orders the columns: the result is a function of the matrix alone.  Four entries per thread are loaded
// before their partials are written back (distinct rows: no aliasing), so each thread keeps four gathers in flight.
constexpr int TPM_THREADS = 512;
__global__ void __launch_bounds__(TPM_THREADS) csc_row_partials_kernel(const long long* __restrict__ col_ptr,
                                                                      const int* __restrict__ row_idx,
                                                                      const float* __restrict__ vals, int n_rows,
                                                                      int n_cols, double* __restrict__ part) {
  const int S = gridDim.x, s = blockIdx.x;
  const long long nnz = col_ptr[n_cols];
  // first column whose entries start at or after `target` (col_ptr is monotone)
  auto first_col = [&](long long target) {
    int lo = 0, hi = n_cols;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (col_ptr[mid] < target) lo = mid + 1; else hi = mid;
    }
    return lo;
  };
  const int c0 = s == 0 ? 0 : first_col(nnz * s / S);
  const int c1 = s == S - 1 ? n_cols : first_col(nnz * (s + 1) / S);
  double* p = part + (long long)s * n_rows;
  constexpr int B = TPM_THREADS;
  for (int c = c0; c < c1; ++c) {
    const long long end = col_ptr[c + 1];
    long long j = col_ptr[c] + threadIdx.x;
    for (; j + 3 * B < end; j += 4 * B) {
      int r[4];
      double v[4], a[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        r[u] = row_idx[j + u * B];
        v[u] = vals[j + u * B];
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) a[u] = p[r[u]];
#pragma unroll
      for (int u = 0; u < 4; ++u) p[r[u]] = a[u] + v[u];
    }
    for (; j < end; j += B) p[row_idx[j]] += (double)vals[j];
    __syncthreads();
  }
}

// Cell totals, pass 2: totals[r] = the slab partials added in slab order; row scale target / total, 0 for a row
// without counts (scanpy's normalize_total leaves such a row at zero)
__global__ void csc_row_totals_kernel(const double* __restrict__ part, int slabs, int n_rows, double target,
                                      double* __restrict__ totals, double* __restrict__ scale) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_rows) return;
  double t = 0.0;
  for (int s = 0; s < slabs; ++s) t += part[(long long)s * n_rows + r];
  totals[r] = t;
  scale[r] = t != 0.0 ? target / t : 0.0;
}

// csc_col_stats_kernel with every entry times its row scale: sum(x * rs), sum((x * rs)^2) per column in fp64
__global__ void __launch_bounds__(WARPS * 32) csc_scaled_col_sums_kernel(const long long* __restrict__ col_ptr,
                                                                         const int* __restrict__ row_idx,
                                                                         const float* __restrict__ vals, int n_cols,
                                                                         const double* __restrict__ rs,
                                                                         double* __restrict__ col_sums) {
  const int col = blockIdx.x * WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (col >= n_cols) return;
  double s = 0.0, q = 0.0;
  for (long long j = col_ptr[col] + lane; j < col_ptr[col + 1]; j += 32) {
    const double v = (double)vals[j] * rs[row_idx[j]];
    s += v;
    q = fma(v, v, q);
  }
  s = warp_sum(s);
  q = warp_sum(q);
  if (lane == 0) {
    col_sums[col] = s;
    col_sums[n_cols + col] = q;
  }
}

// one warp per selected column: dst[row][c] = X[row][cols[c]] * scale[c] (the product gather_cols_kernel forms)
__global__ void __launch_bounds__(WARPS * 32) csc_gather_cols_kernel(const long long* __restrict__ col_ptr,
                                                                     const int* __restrict__ row_idx,
                                                                     const float* __restrict__ vals,
                                                                     const int* __restrict__ cols,
                                                                     const float* __restrict__ scale, int n_sel,
                                                                     float* __restrict__ dst, int ld_dst) {
  const int c = blockIdx.x * WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (c >= n_sel) return;
  const int src = cols[c];
  const float f = scale[c];
  for (long long j = col_ptr[src] + lane; j < col_ptr[src + 1]; j += 32) dst[(long long)row_idx[j] * ld_dst + c] = vals[j] * f;
}

// CSR -> CSC (csr_to_csc).  Row block b holds rows [b * rb, min((b + 1) * rb, n_rows)); its entries are one contiguous
// range of the CSR arrays.  cnt[b * n_cols + c]: entries of column c in block b.
// Pass 1: the counts.  Integer atomics only count; no position depends on their order.
__global__ void csr_block_hist_kernel(const long long* __restrict__ row_ptr, const int* __restrict__ col_idx, int n_rows,
                                      int n_cols, int rb, int* __restrict__ cnt) {
  const long long r0 = (long long)blockIdx.x * rb, r1 = min(r0 + rb, (long long)n_rows);
  int* c = cnt + (long long)blockIdx.x * n_cols;
  for (long long j = row_ptr[r0] + threadIdx.x; j < row_ptr[r1]; j += blockDim.x) atomicAdd(&c[col_idx[j]], 1);
}

// Pass 2, one thread per column: the counts become exclusive prefixes over the blocks (where block b's entries of the
// column start within it) and col_tot[c] the column's length
__global__ void csr_block_scan_kernel(int* __restrict__ cnt, int n_blocks, int n_cols, long long* __restrict__ col_tot) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_cols) return;
  int run = 0;
  for (int b = 0; b < n_blocks; ++b) {
    int* p = cnt + (long long)b * n_cols + c;
    const int t = *p;
    *p = run;
    run += t;
  }
  col_tot[c] = run;
}

// Pass 3, one block: out[0..n] = exclusive prefix sums of in[0..n-1], 64-bit (col_ptr from the column lengths)
constexpr int SCAN_THREADS = 1024;
__global__ void __launch_bounds__(SCAN_THREADS) exclusive_scan_ll_kernel(const long long* __restrict__ in, int n,
                                                                         long long* __restrict__ out) {
  __shared__ long long part[SCAN_THREADS];
  const long long per = (n + SCAN_THREADS - 1) / SCAN_THREADS;
  const long long beg = threadIdx.x * per, end = min(beg + per, (long long)n);
  long long s = 0;
  for (long long i = beg; i < end; ++i) s += in[i];
  part[threadIdx.x] = s;
  __syncthreads();
  for (int o = 1; o < SCAN_THREADS; o <<= 1) {      // inclusive scan of the thread totals
    const long long v = threadIdx.x >= o ? part[threadIdx.x - o] : 0;
    __syncthreads();
    part[threadIdx.x] += v;
    __syncthreads();
  }
  long long run = threadIdx.x > 0 ? part[threadIdx.x - 1] : 0;
  for (long long i = beg; i < end; ++i) {
    out[i] = run;
    run += in[i];
  }
  if (threadIdx.x == SCAN_THREADS - 1) out[n] = part[SCAN_THREADS - 1];
}

// Pass 4: block b walks its rows in order; the entries of one canonical row have distinct columns, so the threads of a
// row never share a cursor (next[b * n_cols + c], block b's next slot in column c), and the barrier orders the rows:
// each column receives its rows in increasing order.
__global__ void csr_block_scatter_kernel(const long long* __restrict__ row_ptr, const int* __restrict__ col_idx,
                                         const float* __restrict__ vals, int n_rows, int n_cols, int rb,
                                         const long long* __restrict__ col_ptr, int* next, int* __restrict__ row_out,
                                         float* __restrict__ val_out) {
  const int r0 = (int)min((long long)blockIdx.x * rb, (long long)n_rows);
  const int r1 = (int)min((long long)r0 + rb, (long long)n_rows);
  int* nx = next + (long long)blockIdx.x * n_cols;
  for (int r = r0; r < r1; ++r) {
    for (long long j = row_ptr[r] + threadIdx.x; j < row_ptr[r + 1]; j += blockDim.x) {
      const int c = col_idx[j];
      const long long p = col_ptr[c] + nx[c];
      nx[c] += 1;
      row_out[p] = r;
      val_out[p] = vals[j];
    }
    __syncthreads();
  }
}

// one warp per row of [r0, r1): X[r][col_idx[j]] = vals[j] (a canonical row: no two lanes write one element)
template <class T>
__global__ void __launch_bounds__(WARPS * 32) csr_scatter_rows_kernel(const long long* __restrict__ row_ptr,
                                                                      long long base, const int* __restrict__ col_idx,
                                                                      const T* __restrict__ vals, int r0, int r1,
                                                                      T* __restrict__ X, int ld) {
  const long long r = r0 + (long long)blockIdx.x * WARPS + (threadIdx.x >> 5);
  if (r >= r1) return;
  T* row = X + r * ld;
  const long long end = row_ptr[r + 1] - base;
  for (long long j = row_ptr[r] - base + (threadIdx.x & 31); j < end; j += 32) row[col_idx[j]] = vals[j];
}

template <class T>
int launch_csr_scatter_rows(const long long* row_ptr, long long base, const int* col_idx, const T* vals, int r0, int r1,
                            T* X, int ld, cudaStream_t s) {
  if (r1 <= r0) return 0;
  const unsigned blocks = (unsigned)((r1 - r0 + WARPS - 1) / WARPS);
  csr_scatter_rows_kernel<T><<<blocks, WARPS * 32, 0, s>>>(row_ptr, base, col_idx, vals, r0, r1, X, ld);
  CNMF_CUDA_CHECK(cudaGetLastError());
  return 0;
}

// device arrays owned by d (from the handle's pool when one fits), typed
template <class T>
int alloc_owned(cnmf_dataset_s* d, T** p, size_t count) {
  float* q = nullptr;
  const int rc = dataset_alloc(d, &q, (count * sizeof(T) + 3) / 4);
  *p = reinterpret_cast<T*>(q);
  return rc;
}

// chunk table of csc_project_kernel from a host col_ptr, which is checked monotone on the way
int csc_item_table(const int64_t* col_ptr, int n_cols, std::vector<int>* item_ptr) {
  item_ptr->assign(n_cols + 1, 0);
  long long items = 0;
  for (int c = 0; c < n_cols; ++c) {
    CNMF_REQUIRE(col_ptr[c + 1] >= col_ptr[c], "CSC dataset: col_ptr is not monotone");
    (*item_ptr)[c] = (int)items;
    items += (col_ptr[c + 1] - col_ptr[c] + CSC_CHUNK - 1) / CSC_CHUNK;
    CNMF_REQUIRE(items < (1LL << 31), "CSC dataset: too many entries");
  }
  (*item_ptr)[n_cols] = (int)items;
  return 0;
}

// the rest of every CSC dataset creation once its three arrays are resident: chunk table, column sums, form
int csc_finish(cnmf_dataset_s* d, const std::vector<int>& item_ptr, cudaStream_t s) {
  d->n_items = item_ptr[d->n_cols];
  CNMF_TRY(alloc_owned(d, &d->item_ptr, (size_t)d->n_cols + 1));
  CNMF_TRY(alloc_owned(d, &d->col_sums, 2 * (size_t)d->n_cols));
  CNMF_CUDA_CHECK(cudaMemcpyAsync(d->item_ptr, item_ptr.data(), sizeof(int) * (d->n_cols + 1), cudaMemcpyHostToDevice, s));
  CNMF_TRY(csc_col_stats(d, s));    // synchronises: item_ptr may go out of scope afterwards
  return dataset_resolve_form(d, false, s);
}

}  // namespace

namespace cnmf {

int require_dense(const cnmf_dataset_s* d, const char* what) {
  if (d && d->sparse) {
    set_last_error(std::string(what) + " is not implemented for sparse (CSC) datasets: they serve the consensus "
                   "step only (col_stats, project_rows, from_columns, transposed Frobenius refit)");
    return -3;
  }
  if (d && d->precision == CNMF_PRECISION_FP64) {
    set_last_error(std::string(what) + " is not available on float64 datasets: they support shape, ld, sums, "
                   "col_stats, solve_bytes_per_row and the _f64 entry points");
    return -3;
  }
  return 0;
}

int csc_project(const cnmf_dataset_s* d, const float* U, int k, int kp, float* out, int ld, cudaStream_t s) {
  cnmf_handle_s* h = d->h;
  double* part = static_cast<double*>(h->dev_buf("csc.part", sizeof(double) * std::max(1, d->n_items) * (size_t)kp));
  if (!part) return -2;
  h->launches += 2;
  // algorithmic bytes: the entries (row index + value), col_ptr, U and the output
  const double bytes = 8.0 * d->nnz + 8.0 * (d->n_cols + 1) + 4.0 * d->n_rows * kp + 4.0 * k * d->n_cols;
  const int slot = h->prof_begin(s, bytes, 2);
  if (d->n_items > 0) {
    const int blocks = std::min((d->n_items + WARPS - 1) / WARPS, h->sm_count * 16);
    csc_project_kernel<<<blocks, WARPS * 32, 0, s>>>(d->col_ptr, d->row_idx, d->vals, d->item_ptr, d->n_cols, d->n_items,
                                                      reinterpret_cast<const float4*>(U), kp, part);
  }
  const long long n_out = (long long)k * d->n_cols;
  csc_project_reduce_kernel<<<(unsigned)((n_out + 255) / 256), 256, 0, s>>>(part, d->item_ptr, d->n_cols, k, kp, out, ld);
  h->prof_end(s, slot);
  CNMF_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int csc_col_stats(cnmf_dataset_s* d, cudaStream_t s) {
  cnmf_handle_s* h = d->h;
  double* tot = static_cast<double*>(h->dev_buf("csc.totals", sizeof(double) * 2));
  if (!tot) return -2;
  csc_col_stats_kernel<<<(d->n_cols + WARPS - 1) / WARPS, WARPS * 32, 0, s>>>(d->col_ptr, d->vals, d->n_cols, d->col_sums);
  csc_totals_kernel<<<1, 256, 0, s>>>(d->col_sums, d->n_cols, tot);
  h->launches += 2;
  CNMF_CUDA_CHECK(cudaGetLastError());
  double out2[2];
  CNMF_CUDA_CHECK(cudaMemcpyAsync(out2, tot, sizeof(out2), cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
  d->sum = out2[0];
  d->sum_sq = out2[1];
  return 0;
}

int csc_detect_exact(cnmf_dataset_s* d, cudaStream_t s, bool* exact) {
  cnmf_handle_s* h = d->h;
  float *cmin = nullptr, *rmin = nullptr;
  CNMF_TRY(dataset_alloc(d, &cmin, (size_t)d->ld_c));
  CNMF_TRY(dataset_alloc(d, &rmin, (size_t)d->ld_r));
  int* n_bad = static_cast<int*>(h->dev_buf("dataset.nbad", sizeof(int) * 2));
  if (!n_bad) return -2;
  CNMF_CUDA_CHECK(cudaMemsetAsync(cmin, 0x7f, sizeof(float) * d->n_cols, s));   // 0x7f7f7f7f: a huge finite float
  CNMF_CUDA_CHECK(cudaMemsetAsync(rmin, 0x7f, sizeof(float) * d->n_rows, s));
  CNMF_CUDA_CHECK(cudaMemsetAsync(n_bad, 0, sizeof(int) * 2, s));
  const int blocks = (d->n_cols + WARPS - 1) / WARPS;
  csc_min_positive_kernel<<<blocks, WARPS * 32, 0, s>>>(d->col_ptr, d->row_idx, d->vals, d->n_cols,
                                                        reinterpret_cast<int*>(cmin), reinterpret_cast<int*>(rmin));
  CNMF_CUDA_CHECK(cudaGetLastError());
  CNMF_TRY(launch_fix_scale(cmin, d->n_cols, d->ld_c, s));
  CNMF_TRY(launch_fix_scale(rmin, d->n_rows, d->ld_r, s));
  csc_check_scaled_int_kernel<<<blocks, WARPS * 32, 0, s>>>(d->col_ptr, d->row_idx, d->vals, d->n_cols, cmin, rmin, n_bad);
  CNMF_CUDA_CHECK(cudaGetLastError());
  h->launches += 4;
  int bad[2] = {1, 1};
  CNMF_CUDA_CHECK(cudaMemcpyAsync(bad, n_bad, sizeof(int) * 2, cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
  if (bad[0] == 0) { *exact = true; d->col_scale = cmin; }
  else if (bad[1] == 0) { *exact = true; d->row_scale = rmin; }
  return 0;
}

int csc_gather_cols(const cnmf_dataset_s* d, const int* cols, const float* scale, int n_cols, float* dst, int ld_dst,
                    cudaStream_t s) {
  csc_gather_cols_kernel<<<(n_cols + WARPS - 1) / WARPS, WARPS * 32, 0, s>>>(d->col_ptr, d->row_idx, d->vals, cols, scale,
                                                                              n_cols, dst, ld_dst);
  d->h->launches += 1;
  CNMF_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int csc_tpm_sums(const cnmf_dataset_s* d, double target_sum, double* totals, double* col_sums, cudaStream_t s) {
  cnmf_handle_s* h = d->h;
  // a function of the shape alone, so the reduction order is too; the partial vectors stay within 256 MB
  const int slabs = (int)std::max(1LL, std::min({(long long)TPM_SLABS, (long long)d->n_cols, (1LL << 25) / d->n_rows}));
  const size_t part_bytes = sizeof(double) * (size_t)slabs * d->n_rows;
  double* part = static_cast<double*>(h->dev_buf("tpm.part", part_bytes));
  double* scale = static_cast<double*>(h->dev_buf("tpm.scale", sizeof(double) * d->n_rows));
  if (!part || !scale) return -2;
  CNMF_CUDA_CHECK(cudaMemsetAsync(part, 0, part_bytes, s));
  csc_row_partials_kernel<<<slabs, TPM_THREADS, 0, s>>>(d->col_ptr, d->row_idx, d->vals, d->n_rows, d->n_cols, part);
  csc_row_totals_kernel<<<(d->n_rows + 255) / 256, 256, 0, s>>>(part, slabs, d->n_rows, target_sum, totals, scale);
  csc_scaled_col_sums_kernel<<<(d->n_cols + WARPS - 1) / WARPS, WARPS * 32, 0, s>>>(d->col_ptr, d->row_idx, d->vals,
                                                                                    d->n_cols, scale, col_sums);
  h->launches += 3;
  CNMF_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int stage_rows(cnmf_handle_s* h, const float* F, int k, int n, int ld, int kp, float* U, cudaStream_t s) {
  const long long total = (long long)n * kp;
  stage_rows_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(F, k, n, ld, kp, U);
  h->launches += 1;
  CNMF_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int check_csr(const char* what, int n_rows, int n_cols, long long nnz, const int64_t* row_ptr, const int32_t* col_idx) {
  const std::string w(what);
  CNMF_REQUIRE(row_ptr[0] == 0 && row_ptr[n_rows] == nnz, w + ": row_ptr must start at 0 and end at nnz");
  for (int r = 0; r < n_rows; ++r) {
    CNMF_REQUIRE(row_ptr[r + 1] >= row_ptr[r], w + ": row_ptr is not monotone");
    for (long long j = row_ptr[r]; j < row_ptr[r + 1]; ++j) {
      CNMF_REQUIRE(col_idx[j] >= 0 && col_idx[j] < n_cols, w + ": column index out of range");
      CNMF_REQUIRE(j == row_ptr[r] || col_idx[j] > col_idx[j - 1],
                   w + ": column indices must increase within a row (canonical CSR: sorted, no duplicates)");
    }
  }
  return 0;
}

int csr_to_csc(cnmf_dataset_s* d, const long long* row_ptr, const int* col_idx, const float* vals, cudaStream_t s) {
  cnmf_handle_s* h = d->h;
  const int n_rows = d->n_rows, n_cols = d->n_cols;
  const long long max_blocks = std::max(1LL, CSR_COUNT_BUDGET / n_cols);
  long long rb = CSR_ROW_BLOCK;
  if ((n_rows + rb - 1) / rb > max_blocks) rb = (n_rows + max_blocks - 1) / max_blocks;
  const int n_blocks = (int)((n_rows + rb - 1) / rb);
  CNMF_TRY(alloc_owned(d, &d->col_ptr, (size_t)n_cols + 1));
  CNMF_TRY(alloc_owned(d, &d->row_idx, (size_t)d->nnz));
  CNMF_TRY(alloc_owned(d, &d->vals, (size_t)d->nnz));
  DeviceTemp cnt, col_tot;
  CNMF_TRY(cnt.alloc(sizeof(int) * (size_t)n_blocks * n_cols, "dataset_create_csr: block counts"));
  CNMF_TRY(col_tot.alloc(sizeof(long long) * (size_t)n_cols, "dataset_create_csr: column lengths"));
  CNMF_CUDA_CHECK(cudaMemsetAsync(cnt.p, 0, sizeof(int) * (size_t)n_blocks * n_cols, s));
  csr_block_hist_kernel<<<n_blocks, 256, 0, s>>>(row_ptr, col_idx, n_rows, n_cols, (int)rb, cnt.as<int>());
  csr_block_scan_kernel<<<(n_cols + 255) / 256, 256, 0, s>>>(cnt.as<int>(), n_blocks, n_cols, col_tot.as<long long>());
  exclusive_scan_ll_kernel<<<1, SCAN_THREADS, 0, s>>>(col_tot.as<long long>(), n_cols, d->col_ptr);
  csr_block_scatter_kernel<<<n_blocks, 256, 0, s>>>(row_ptr, col_idx, vals, n_rows, n_cols, (int)rb, d->col_ptr,
                                                     cnt.as<int>(), d->row_idx, d->vals);
  h->launches += 4;
  CNMF_CUDA_CHECK(cudaGetLastError());
  std::vector<int64_t> col_ptr(n_cols + 1);
  CNMF_CUDA_CHECK(cudaMemcpyAsync(col_ptr.data(), d->col_ptr, sizeof(long long) * (n_cols + 1), cudaMemcpyDeviceToHost,
                                  s));
  CNMF_CUDA_CHECK(cudaStreamSynchronize(s));      // the count table is released on return
  std::vector<int> item_ptr;
  CNMF_TRY(csc_item_table(col_ptr.data(), n_cols, &item_ptr));
  return csc_finish(d, item_ptr, s);
}

int csr_scatter_rows(const long long* row_ptr, long long base, const int* col_idx, const float* vals, int r0, int r1,
                     float* X, int ld, cudaStream_t s) {
  return launch_csr_scatter_rows(row_ptr, base, col_idx, vals, r0, r1, X, ld, s);
}

int csr_scatter_rows(const long long* row_ptr, long long base, const int* col_idx, const double* vals, int r0, int r1,
                     double* X, int ld, cudaStream_t s) {
  return launch_csr_scatter_rows(row_ptr, base, col_idx, vals, r0, r1, X, ld, s);
}

}  // namespace cnmf

extern "C" {

int cnmf_dataset_create_csc(cnmf_handle_t h, int n_rows, int n_cols, long long nnz, const int64_t* col_ptr,
                            const int32_t* row_idx, const float* values, int precision, void* stream,
                            cnmf_dataset_t* out) {
  CNMF_REQUIRE(h && col_ptr && out && (nnz == 0 || (row_idx && values)), "dataset_create_csc: NULL argument");
  CNMF_REQUIRE(n_rows > 0 && n_cols > 0 && nnz >= 0, "dataset_create_csc: bad shape");
  CNMF_REQUIRE(precision == CNMF_PRECISION_FP32 || precision == CNMF_PRECISION_TF32X3 ||
                   precision == CNMF_PRECISION_TF32X3_GENERAL || precision == CNMF_PRECISION_F16X2,
               "dataset_create_csc: bad precision");
  CNMF_REQUIRE(col_ptr[0] == 0 && col_ptr[n_cols] == nnz, "dataset_create_csc: col_ptr must start at 0 and end at nnz");
  std::vector<int> item_ptr;
  CNMF_TRY(csc_item_table(col_ptr, n_cols, &item_ptr));
  for (long long j = 0; j < nnz; ++j)
    CNMF_REQUIRE(row_idx[j] >= 0 && row_idx[j] < n_rows, "dataset_create_csc: row index out of range");
  cudaStream_t s = as_stream(stream);
  CNMF_CUDA_CHECK(cudaSetDevice(h->device));
  auto* d = new cnmf_dataset_s(h, n_rows, n_cols, precision);
  d->sparse = true;
  d->nnz = nnz;
  auto upload = [&](void* dst, const void* src, size_t bytes) {
    if (bytes == 0) return 0;
    const cudaError_t e = cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, s);
    if (e != cudaSuccess) {
      set_last_error(std::string("dataset_create_csc: upload failed: ") + cudaGetErrorString(e));
      return -2;
    }
    return 0;
  };
  int rc = alloc_owned(d, &d->col_ptr, (size_t)n_cols + 1);
  if (rc == 0) rc = alloc_owned(d, &d->row_idx, (size_t)nnz);
  if (rc == 0) rc = alloc_owned(d, &d->vals, (size_t)nnz);
  if (rc == 0) rc = upload(d->col_ptr, col_ptr, sizeof(long long) * (n_cols + 1));
  if (rc == 0) rc = upload(d->row_idx, row_idx, sizeof(int) * (size_t)nnz);
  if (rc == 0) rc = upload(d->vals, values, sizeof(float) * (size_t)nnz);
  if (rc == 0) rc = csc_finish(d, item_ptr, s);
  if (rc != 0) {
    cudaStreamSynchronize(s);
    cnmf_dataset_destroy(d);
    return rc;
  }
  *out = d;
  return 0;
}

}  // extern "C"
