// extern "C" entry points declared in include/cnmf_b200.h (handle, dataset, factorize, refit).
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstring>
#include <functional>
#include <string>
#include <thread>
#include <vector>

#include "engine.h"
#include "gemm.h"
#include "legacy_rng.h"
#include "nmf_kernels.cuh"

namespace cnmf {

int launch_rng_init(const uint32_t* seeds_host, const int* ks_host, const int* offs_host, const double* avgs_host, int R,
                    int n_samples, int n_features, float* Wt, long long ldW, float* H, long long ldH, cnmf_handle_s* h,
                    cudaStream_t s);
int launch_rng_init(const uint32_t* seeds_host, const int* ks_host, const int* offs_host, const double* avgs_host, int R,
                    int n_samples, int n_features, double* Wt, long long ldW, double* H, long long ldH, cnmf_handle_s* h,
                    cudaStream_t s);

static thread_local std::string g_last_error;
void set_last_error(const std::string& msg) { g_last_error = msg; }

}  // namespace cnmf

using namespace cnmf;

// ----------------------------------------------------------------------------- handle
void* cnmf_handle_s::dev_buf(const std::string& name, size_t bytes) {
  auto& e = ws[name];
  if (e.second >= bytes && e.first) return e.first;
  if (e.first) cudaFree(e.first);
  e.first = nullptr;
  e.second = 0;
  const size_t want = std::max<size_t>(bytes, 256);
  cudaError_t err = cudaMalloc(&e.first, want);
  if (err != cudaSuccess) {
    set_last_error("cudaMalloc(" + name + ", " + std::to_string(want) + " bytes) failed: " + cudaGetErrorString(err));
    e.first = nullptr;
    return nullptr;
  }
  e.second = want;
  return e.first;
}

void* cnmf_handle_s::host_buf(const std::string& name, size_t bytes) {
  auto& e = pinned[name];
  if (e.second >= bytes && e.first) return e.first;
  if (e.first) cudaFreeHost(e.first);
  e.first = nullptr;
  e.second = 0;
  const size_t want = std::max<size_t>(bytes, 256);
  cudaError_t err = cudaMallocHost(&e.first, want);
  if (err != cudaSuccess) {
    set_last_error("cudaMallocHost(" + name + ", " + std::to_string(want) + " bytes) failed: " + cudaGetErrorString(err));
    e.first = nullptr;
    return nullptr;
  }
  e.second = want;
  return e.first;
}

int cnmf_handle_s::prof_begin(cudaStream_t s, double work, int cls) {
  if (!profile) return -1;
  while (ev_pool.size() < ev_used + 2) {
    cudaEvent_t e;
    if (cudaEventCreate(&e) != cudaSuccess) return -1;
    ev_pool.push_back(e);
  }
  int begin;
  // call sites count their launch (launches += 1) before prof_begin: exactly one more than at the last prof_end
  // means nothing else was enqueued by the library in between
  if (prof_last_end >= 0 && prof_last_stream == s && launches == prof_last_launches + 1) {
    begin = prof_last_end;
  } else {
    begin = (int)ev_used++;
    cudaEventRecord(ev_pool[begin], s);
  }
  const int end = (int)ev_used++;
  ev_pending.push_back(Pending{begin, end, cls, work});
  return (int)ev_pending.size() - 1;
}

void cnmf_handle_s::prof_end(cudaStream_t s, int slot) {
  if (slot < 0) return;
  const int end = ev_pending[slot].end;
  cudaEventRecord(ev_pool[end], s);
  prof_last_end = end;
  prof_last_launches = launches;
  prof_last_stream = s;
}

void cnmf_handle_s::prof_collect() {
  for (auto& pr : ev_pending) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, ev_pool[pr.begin], ev_pool[pr.end]) == cudaSuccess) {
      prof_ms[pr.cls] += ms;
      prof_work[pr.cls] += pr.work;
      prof_launches[pr.cls] += 1;
    }
  }
  ev_pending.clear();
  ev_used = 0;
  prof_last_end = -1;
}

void* cnmf_handle_s::pool_take(size_t bytes) {
  auto it = pool.find(bytes);
  if (it == pool.end()) return nullptr;
  void* p = it->second;
  pool.erase(it);
  pool_bytes -= bytes;
  return p;
}

void cnmf_handle_s::pool_give(void* p, size_t bytes) {
  constexpr size_t POOL_CAP = (size_t)16 << 30;     // keep at most 16 GB parked
  if (pool_bytes + bytes > POOL_CAP) {
    cudaFree(p);
    return;
  }
  pool.emplace(bytes, p);
  pool_bytes += bytes;
}

void cnmf_handle_s::release_all() {
  for (auto& kv : pool) cudaFree(kv.second);
  pool.clear();
  pool_bytes = 0;
  for (auto e : ev_pool) cudaEventDestroy(e);
  ev_pool.clear();
  for (auto& kv : ws)
    if (kv.second.first) cudaFree(kv.second.first);
  ws.clear();
  for (auto& kv : pinned)
    if (kv.second.first) cudaFreeHost(kv.second.first);
  pinned.clear();
}

extern "C" {

int cnmf_abi_version(void) { return CNMF_B200_ABI_VERSION; }
const char* cnmf_last_error(void) { return g_last_error.c_str(); }

int cnmf_create(cnmf_handle_t* out, int device) {
  CNMF_REQUIRE(out != nullptr, "cnmf_create: out is NULL");
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) {
    set_last_error(std::string("no CUDA device available (") + cudaGetErrorString(e) +
                   "); cnmf_b200 has no CPU fallback");
    return -2;
  }
  CNMF_REQUIRE(device >= 0 && device < n, "cnmf_create: bad device index");
  CNMF_CUDA_CHECK(cudaSetDevice(device));
  cudaDeviceProp prop;
  CNMF_CUDA_CHECK(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {
    set_last_error("cnmf_b200 is built for sm_90a only; device reports sm_" + std::to_string(prop.major) +
                   std::to_string(prop.minor));
    return -3;
  }
  auto* h = new cnmf_handle_s();
  h->device = device;
  h->sm_count = prop.multiProcessorCount;
  *out = h;
  return 0;
}

int cnmf_destroy(cnmf_handle_t h) {
  if (!h) return 0;
  cudaSetDevice(h->device);
  h->release_all();
  delete h;
  return 0;
}

long long cnmf_launch_count(cnmf_handle_t h) { return h ? h->launches : 0; }

int cnmf_mem_info(cnmf_handle_t h, long long* free_bytes, long long* total_bytes, long long* cached_bytes) {
  CNMF_REQUIRE(h, "mem_info: NULL handle");
  CNMF_CUDA_CHECK(cudaSetDevice(h->device));
  size_t fr = 0, tot = 0;
  CNMF_CUDA_CHECK(cudaMemGetInfo(&fr, &tot));
  size_t cached = h->pool_bytes;
  for (auto& kv : h->ws) cached += kv.second.second;
  if (free_bytes) *free_bytes = (long long)fr;
  if (total_bytes) *total_bytes = (long long)tot;
  if (cached_bytes) *cached_bytes = (long long)cached;
  return 0;
}

long long cnmf_solve_bytes_per_row(cnmf_dataset_t d) {
  if (!d) return 0;
  // float64 solve: the factor, its compaction alternate and result slab and one product, each side, 8 bytes an entry
  if (d->precision == CNMF_PRECISION_FP64) return 8LL * 4 * ((long long)d->ld_r + d->ld_c);
  // factorize / solve_batched: Fr + 2 piece buffers, their 3 compaction alternates, the result slab and the
  // product NUM_r along the cells; the same along the genes with one product slice per split-K slice
  const int f16 = make_view(d, false).form == Form::F16_EXACT ? 1 : 0;
  const long long splits_c = gemm_fixed_splits(d->n_rows, f16);
  const long long splits_r = gemm_fixed_splits(d->n_cols, f16);
  return 4LL * ((7 + splits_r) * (long long)d->ld_r + (7 + splits_c) * (long long)d->ld_c);
}

int cnmf_profile_enable(cnmf_handle_t h, int on) {
  CNMF_REQUIRE(h, "profile_enable: NULL handle");
  h->profile = on != 0;
  for (int c = 0; c < cnmf_handle_s::PROF_CLASSES; ++c) {
    h->prof_ms[c] = h->prof_work[c] = 0.0;
    h->prof_launches[c] = 0;
  }
  h->ev_pending.clear();
  h->ev_used = 0;
  h->prof_last_end = -1;
  if (on) {       // event creation is kept out of the timed region: a pool for ~32 000 launches up front
    while (h->ev_pool.size() < 65536) {
      cudaEvent_t e;
      if (cudaEventCreate(&e) != cudaSuccess) break;
      h->ev_pool.push_back(e);
    }
  }
  return 0;
}

int cnmf_profile_get(cnmf_handle_t h, double* gemm_ms, long long* gemm_launches, double* gemm_flops) {
  CNMF_REQUIRE(h, "profile_get: NULL handle");
  return cnmf_profile_get_class(h, 0, gemm_ms, gemm_launches, gemm_flops);
}

int cnmf_profile_get_class(cnmf_handle_t h, int cls, double* ms, long long* launches, double* work) {
  CNMF_REQUIRE(h, "profile_get_class: NULL handle");
  CNMF_REQUIRE(cls >= 0 && cls < cnmf_handle_s::PROF_CLASSES, "profile_get_class: unknown kernel class");
  CNMF_CUDA_CHECK(cudaDeviceSynchronize());     // every recorded event has completed
  h->prof_collect();
  if (ms) *ms = h->prof_ms[cls];
  if (launches) *launches = h->prof_launches[cls];
  if (work) *work = h->prof_work[cls];
  return 0;
}

}  // extern "C"

// ----------------------------------------------------------------------------- dataset
namespace cnmf {

int dataset_alloc(cnmf_dataset_s* d, float** p, size_t elems) {
  const size_t bytes = std::max<size_t>(elems, 64) * sizeof(float);
  void* q = d->h->pool_take(bytes);
  if (!q) {
    cudaError_t e = cudaMalloc(&q, bytes);
    if (e != cudaSuccess) {
      set_last_error(std::string("dataset cudaMalloc failed: ") + cudaGetErrorString(e));
      return -2;
    }
  }
  d->owned.emplace_back(q, bytes);
  *p = static_cast<float*>(q);
  return 0;
}

int dataset_resolve_form(cnmf_dataset_s* d, bool exact, cudaStream_t s) {
  // exact-count detection: is X = diag(r) C diag(s) with C integer <= 2048 ?  (column scale first, then row scale).
  // The same condition for dense and CSC matrices, so that both give the same dataset.
  const bool may_be_exact = d->precision == CNMF_PRECISION_TF32X3 || d->precision == CNMF_PRECISION_F16X2;
  if (may_be_exact && !exact) {
    if (d->sparse) {
      CNMF_TRY(csc_detect_exact(d, s, &exact));
    } else {
      cnmf_handle_s* h = d->h;
      float* cmin = nullptr;
      float* rmin = nullptr;
      CNMF_TRY(dataset_alloc(d, &cmin, (size_t)d->ld_c));
      CNMF_TRY(dataset_alloc(d, &rmin, (size_t)d->ld_r));
      int* n_bad = static_cast<int*>(h->dev_buf("dataset.nbad", sizeof(int) * 2));
      if (!n_bad) return -2;
      CNMF_TRY(launch_min_positive(d->X, d->n_rows, d->n_cols, d->ld_c, cmin, rmin, s));
      CNMF_TRY(launch_fix_scale(cmin, d->n_cols, d->ld_c, s));
      CNMF_TRY(launch_fix_scale(rmin, d->n_rows, d->ld_r, s));
      CNMF_CUDA_CHECK(cudaMemsetAsync(n_bad, 0, sizeof(int) * 2, s));
      CNMF_TRY(launch_check_scaled_int(d->X, d->n_rows, d->n_cols, d->ld_c, nullptr, cmin, n_bad, s));
      CNMF_TRY(launch_check_scaled_int(d->X, d->n_rows, d->n_cols, d->ld_c, rmin, nullptr, n_bad + 1, s));
      h->launches += 5;
      int bad[2] = {1, 1};
      CNMF_CUDA_CHECK(cudaMemcpyAsync(bad, n_bad, sizeof(int) * 2, cudaMemcpyDeviceToHost, s));
      CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
      if (bad[0] == 0) { exact = true; d->col_scale = cmin; d->row_scale = nullptr; }
      else if (bad[1] == 0) { exact = true; d->row_scale = rmin; d->col_scale = nullptr; }
    }
  }
  if (d->precision == CNMF_PRECISION_FP32) d->form = Form::FP32;
  else if (!exact) d->form = Form::TF32;
  else d->form = d->precision == CNMF_PRECISION_F16X2 ? Form::F16_EXACT : Form::TF32_EXACT;
  return 0;
}

int dataset_finish(cnmf_dataset_s* d, cudaStream_t s, bool exact) {
  cnmf_handle_s* h = d->h;
  const size_t nx = (size_t)d->n_rows * d->ld_c, nxt = (size_t)d->n_cols * d->ld_r;
  CNMF_TRY(dataset_resolve_form(d, exact, s));
  if (d->form == Form::FP32) {
    CNMF_TRY(dataset_alloc(d, &d->Xt, nxt));
    CNMF_CUDA_CHECK(cudaMemsetAsync(d->Xt, 0, nxt * sizeof(float), s));
    CNMF_TRY(launch_transpose(d->X, d->n_rows, d->n_cols, d->ld_c, d->Xt, nullptr, nullptr, d->ld_r, s));
    h->launches += 1;
  } else if (d->form == Form::TF32) {
    CNMF_TRY(dataset_alloc(d, &d->X_hi, nx));
    CNMF_TRY(dataset_alloc(d, &d->X_lo, nx));
    CNMF_TRY(dataset_alloc(d, &d->Xt_hi, nxt));
    CNMF_TRY(dataset_alloc(d, &d->Xt_lo, nxt));
    CNMF_CUDA_CHECK(cudaMemsetAsync(d->Xt_hi, 0, nxt * sizeof(float), s));
    CNMF_CUDA_CHECK(cudaMemsetAsync(d->Xt_lo, 0, nxt * sizeof(float), s));
    CNMF_TRY(launch_split_tf32(d->X, d->X_hi, d->X_lo, (long long)nx, s));
    CNMF_TRY(launch_transpose(d->X, d->n_rows, d->n_cols, d->ld_c, nullptr, d->Xt_hi, d->Xt_lo, d->ld_r, s));
    h->launches += 2;
  } else {
    CNMF_TRY(dataset_alloc(d, &d->X_hi, nx));
    CNMF_TRY(dataset_alloc(d, &d->Xt_hi, nxt));
    CNMF_CUDA_CHECK(cudaMemsetAsync(d->X_hi, 0, nx * sizeof(float), s));
    CNMF_CUDA_CHECK(cudaMemsetAsync(d->Xt_hi, 0, nxt * sizeof(float), s));
    CNMF_TRY(launch_build_counts(d->X, d->n_rows, d->n_cols, d->ld_c, d->row_scale, d->col_scale, d->X_hi, s));
    CNMF_TRY(launch_transpose(d->X_hi, d->n_rows, d->n_cols, d->ld_c, d->Xt_hi, nullptr, nullptr, d->ld_r, s));
    h->launches += 2;
    if (d->form == Form::F16_EXACT) {       // counts <= 2048 are exact in fp16: the B operands of the f16 products
      float *xh = nullptr, *xth = nullptr;
      CNMF_TRY(dataset_alloc(d, &xh, (nx + 1) / 2));
      CNMF_TRY(dataset_alloc(d, &xth, (nxt + 1) / 2));
      d->X_h16 = xh;
      d->Xt_h16 = xth;
      CNMF_TRY(launch_to_half(d->X_hi, d->X_h16, (long long)nx, s));
      CNMF_TRY(launch_to_half(d->Xt_hi, d->Xt_h16, (long long)nxt, s));
      h->launches += 2;
    }
  }
  const int scratch_len = 2 * cnmf::NUM_SMS * 8 + 2;
  double* scratch = static_cast<double*>(h->dev_buf("dataset.sums", sizeof(double) * (scratch_len + 2)));
  if (!scratch) return -2;
  CNMF_TRY(launch_matrix_sums(d->X, d->n_rows, d->n_cols, d->ld_c, scratch + scratch_len, scratch, scratch_len, s));
  h->launches += 2;
  double out2[2];
  CNMF_CUDA_CHECK(cudaMemcpyAsync(out2, scratch + scratch_len, 2 * sizeof(double), cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
  d->sum = out2[0];
  d->sum_sq = out2[1];
  // every product of an f16 dataset reads the fp16 count matrices: the fp32 copies of C / C^T were scaffolding.
  // Resident forms are then X (fp32, column operations and derived datasets) + C and C^T as fp16: 2 x the bytes of X
  // instead of 4 x.  Released only now, after the synchronisation above: the conversions have completed.
  if (d->form == Form::F16_EXACT) {
    for (float** pp : {&d->X_hi, &d->Xt_hi}) {
      for (auto it = d->owned.begin(); it != d->owned.end(); ++it)
        if (it->first == *pp) {
          h->pool_give(it->first, it->second);
          d->owned.erase(it);
          break;
        }
      *pp = nullptr;
    }
  }
  return 0;
}

int check_params_precision(const cnmf_dataset_s* d, const cnmf_nmf_params* p) {
  const int want = d->precision == CNMF_PRECISION_FP32 || d->precision == CNMF_PRECISION_FP64 ? d->precision
                                                                                                : CNMF_PRECISION_TF32X3;
  CNMF_REQUIRE(p->precision == want, "params.precision must match the precision the dataset was created with");
  return 0;
}

int require_f32(const cnmf_dataset_s* d, const char* what) {
  if (d && d->precision == CNMF_PRECISION_FP64) {
    set_last_error(std::string("cnmf_") + what + " takes float data; this dataset is float64: call cnmf_" + what + "_f64");
    return -3;
  }
  return 0;
}

int require_f64(const cnmf_dataset_s* d, const char* what) {
  if (d && d->precision != CNMF_PRECISION_FP64) {
    set_last_error(std::string("cnmf_") + what + "_f64 needs a float64 dataset (cnmf_dataset_create_f64); this one "
                   "holds float data: call cnmf_" + what);
    return -3;
  }
  return 0;
}

}  // namespace cnmf

extern "C" {

}  // extern "C"

namespace {

bool float_precision(int precision) {
  return precision == CNMF_PRECISION_FP32 || precision == CNMF_PRECISION_TF32X3 ||
         precision == CNMF_PRECISION_TF32X3_GENERAL || precision == CNMF_PRECISION_F16X2;
}

// Every dense dataset creator: the staging array (X, or X64 for CNMF_PRECISION_FP64; n_rows x ld_c) is zero-filled,
// fill(d, X) writes the matrix into it on stream s, then the forms and sums are built from it.  cudaError_t from fill
// is reported as an upload failure; a library status is passed on.
template <class T, class Fill>
int create_dense(cnmf_handle_t h, int n_rows, int n_cols, int precision, cudaStream_t s, cnmf_dataset_t* out, Fill fill) {
  CNMF_CUDA_CHECK(cudaSetDevice(h->device));
  auto* d = new cnmf_dataset_s(h, n_rows, n_cols, precision);
  const size_t nx = (size_t)n_rows * d->ld_c;
  float* buf = nullptr;
  int rc = dataset_alloc(d, &buf, nx * sizeof(T) / sizeof(float));
  T* X = reinterpret_cast<T*>(buf);
  if (rc == 0) {
    const cudaError_t e = cudaMemsetAsync(X, 0, nx * sizeof(T), s);
    if (e != cudaSuccess) {
      set_last_error(std::string("dataset upload failed: ") + cudaGetErrorString(e));
      rc = -2;
    }
  }
  if (rc == 0) rc = fill(d, X);
  if (rc == 0 && precision == CNMF_PRECISION_FP64) {
    d->form = Form::FP64;
    d->X64 = reinterpret_cast<double*>(buf);
    double sums[2] = {0.0, 0.0};
    rc = matrix_sums_f64(h, d->X64, n_rows, n_cols, d->ld_c, sums, s);
    d->sum = sums[0];
    d->sum_sq = sums[1];
  } else if (rc == 0) {
    d->X = buf;
    rc = dataset_finish(d, s);
  }
  if (rc != 0) {
    cudaStreamSynchronize(s);
    cnmf_dataset_destroy(d);
    return rc;
  }
  *out = d;
  return 0;
}

// fill of a host or device matrix with row stride ld
template <class T>
auto copy_fill(const T* src, long long ld, int n_rows, int n_cols, bool src_is_device, cudaStream_t s) {
  return [=](cnmf_dataset_s* d, T* X) {
    const cudaError_t e = cudaMemcpy2DAsync(X, (size_t)d->ld_c * sizeof(T), src, (size_t)ld * sizeof(T),
                                            (size_t)n_cols * sizeof(T), n_rows,
                                            src_is_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, s);
    if (e != cudaSuccess) {
      set_last_error(std::string("dataset upload failed: ") + cudaGetErrorString(e));
      return -2;
    }
    return 0;
  };
}

// most stored entries staged on the device at a time while a host CSR matrix is scattered into a dense one
constexpr long long CSR_STAGE_ENTRIES = 1LL << 24;

// fill of a canonical host CSR matrix (checked by the caller): row_ptr is uploaded whole, the entries in slices of
// whole rows of at most CSR_STAGE_ENTRIES (or one row) each, each slice scattered into X (stream order keeps a slice's
// upload behind the previous scatter); the staging is freed before the dataset's other forms are built
template <class T>
auto csr_fill(const int64_t* row_ptr, const int32_t* col_idx, const T* values, const char* what, cudaStream_t s) {
  return [=](cnmf_dataset_s* d, T* X) {
    const int n = d->n_rows;
    long long stage = 0;     // entries of the largest slice
    std::vector<int> cuts{0};
    while (cuts.back() < n) {
      const int r0 = cuts.back();
      // last row end within the budget, at least one row
      const int r1 = std::max(r0 + 1, (int)(std::upper_bound(row_ptr + r0 + 1, row_ptr + n + 1,
                                                              row_ptr[r0] + CSR_STAGE_ENTRIES) - row_ptr) - 1);
      stage = std::max<long long>(stage, row_ptr[r1] - row_ptr[r0]);
      cuts.push_back(r1);
    }
    DeviceTemp rp, ci, va;
    CNMF_TRY(rp.alloc(sizeof(long long) * ((size_t)n + 1), std::string(what) + ": row_ptr"));
    CNMF_TRY(ci.alloc(sizeof(int) * (size_t)stage, std::string(what) + ": column indices"));
    CNMF_TRY(va.alloc(sizeof(T) * (size_t)stage, std::string(what) + ": values"));
    CNMF_CUDA_CHECK(cudaMemcpyAsync(rp.p, row_ptr, sizeof(long long) * ((size_t)n + 1), cudaMemcpyHostToDevice, s));
    for (size_t i = 0; i + 1 < cuts.size(); ++i) {
      const int r0 = cuts[i], r1 = cuts[i + 1];
      const long long base = row_ptr[r0], cnt = row_ptr[r1] - base;
      if (cnt == 0) continue;
      CNMF_CUDA_CHECK(cudaMemcpyAsync(ci.p, col_idx + base, sizeof(int) * cnt, cudaMemcpyHostToDevice, s));
      CNMF_CUDA_CHECK(cudaMemcpyAsync(va.p, values + base, sizeof(T) * cnt, cudaMemcpyHostToDevice, s));
      CNMF_TRY(csr_scatter_rows(rp.as<long long>(), base, ci.as<int>(), va.as<T>(), r0, r1, X, d->ld_c, s));
      d->h->launches += 1;
    }
    CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
    return 0;
  };
}

}  // namespace

extern "C" {

int cnmf_dataset_create(cnmf_handle_t h, const float* X, int n_rows, int n_cols, long long ld, int src_is_device,
                        int precision, void* stream, cnmf_dataset_t* out) {
  CNMF_REQUIRE(h && X && out, "dataset_create: NULL argument");
  CNMF_REQUIRE(n_rows > 0 && n_cols > 0 && ld >= n_cols, "dataset_create: bad shape");
  CNMF_REQUIRE(float_precision(precision), "dataset_create: bad precision");
  cudaStream_t s = as_stream(stream);
  return create_dense<float>(h, n_rows, n_cols, precision, s, out,
                             copy_fill(X, ld, n_rows, n_cols, src_is_device != 0, s));
}

int cnmf_dataset_create_from_csr(cnmf_handle_t h, int n_rows, int n_cols, long long nnz, const int64_t* row_ptr,
                                 const int32_t* col_idx, const float* values, int precision, void* stream,
                                 cnmf_dataset_t* out) {
  CNMF_REQUIRE(h && row_ptr && out && (nnz == 0 || (col_idx && values)), "dataset_create_from_csr: NULL argument");
  CNMF_REQUIRE(n_rows > 0 && n_cols > 0 && nnz >= 0, "dataset_create_from_csr: bad shape");
  CNMF_REQUIRE(float_precision(precision), "dataset_create_from_csr: bad precision");
  CNMF_TRY(check_csr("dataset_create_from_csr", n_rows, n_cols, nnz, row_ptr, col_idx));
  cudaStream_t s = as_stream(stream);
  return create_dense<float>(h, n_rows, n_cols, precision, s, out,
                             csr_fill(row_ptr, col_idx, values, "dataset_create_from_csr", s));
}

int cnmf_dataset_create_from_csr_f64(cnmf_handle_t h, int n_rows, int n_cols, long long nnz, const int64_t* row_ptr,
                                     const int32_t* col_idx, const double* values, void* stream, cnmf_dataset_t* out) {
  CNMF_REQUIRE(h && row_ptr && out && (nnz == 0 || (col_idx && values)), "dataset_create_from_csr_f64: NULL argument");
  CNMF_REQUIRE(n_rows > 0 && n_cols > 0 && nnz >= 0, "dataset_create_from_csr_f64: bad shape");
  CNMF_TRY(check_csr("dataset_create_from_csr_f64", n_rows, n_cols, nnz, row_ptr, col_idx));
  cudaStream_t s = as_stream(stream);
  return create_dense<double>(h, n_rows, n_cols, CNMF_PRECISION_FP64, s, out,
                              csr_fill(row_ptr, col_idx, values, "dataset_create_from_csr_f64", s));
}

int cnmf_dataset_create_csr(cnmf_handle_t h, int n_rows, int n_cols, long long nnz, const int64_t* row_ptr,
                            const int32_t* col_idx, const float* values, int precision, void* stream,
                            cnmf_dataset_t* out) {
  CNMF_REQUIRE(h && row_ptr && out && (nnz == 0 || (col_idx && values)), "dataset_create_csr: NULL argument");
  CNMF_REQUIRE(n_rows > 0 && n_cols > 0 && nnz >= 0, "dataset_create_csr: bad shape");
  CNMF_REQUIRE(float_precision(precision), "dataset_create_csr: bad precision");
  CNMF_TRY(check_csr("dataset_create_csr", n_rows, n_cols, nnz, row_ptr, col_idx));
  cudaStream_t s = as_stream(stream);
  CNMF_CUDA_CHECK(cudaSetDevice(h->device));
  auto* d = new cnmf_dataset_s(h, n_rows, n_cols, precision);
  d->sparse = true;
  d->nnz = nnz;
  int rc = 0;
  {
    DeviceTemp rp, ci, va;      // the CSR upload, released before return
    rc = rp.alloc(sizeof(long long) * ((size_t)n_rows + 1), "dataset_create_csr: row_ptr");
    if (rc == 0) rc = ci.alloc(sizeof(int) * (size_t)nnz, "dataset_create_csr: column indices");
    if (rc == 0) rc = va.alloc(sizeof(float) * (size_t)nnz, "dataset_create_csr: values");
    cudaError_t e = cudaSuccess;
    if (rc == 0) e = cudaMemcpyAsync(rp.p, row_ptr, sizeof(long long) * ((size_t)n_rows + 1), cudaMemcpyHostToDevice, s);
    if (rc == 0 && e == cudaSuccess && nnz > 0)
      e = cudaMemcpyAsync(ci.p, col_idx, sizeof(int) * (size_t)nnz, cudaMemcpyHostToDevice, s);
    if (rc == 0 && e == cudaSuccess && nnz > 0)
      e = cudaMemcpyAsync(va.p, values, sizeof(float) * (size_t)nnz, cudaMemcpyHostToDevice, s);
    if (e != cudaSuccess) {
      set_last_error(std::string("dataset_create_csr: upload failed: ") + cudaGetErrorString(e));
      rc = -2;
    }
    if (rc == 0) rc = csr_to_csc(d, rp.as<long long>(), ci.as<int>(), va.as<float>(), s);
    cudaStreamSynchronize(s);
  }
  if (rc != 0) {
    cnmf_dataset_destroy(d);
    return rc;
  }
  *out = d;
  return 0;
}

int cnmf_dataset_dense_bytes(int n_rows, int n_cols, int precision, long long* peak) {
  CNMF_REQUIRE(peak && n_rows > 0 && n_cols > 0, "dataset_dense_bytes: bad arguments");
  // what dataset_alloc hands out for one array of `elems` floats
  auto bytes = [](size_t elems) { return (long long)(std::max<size_t>(elems, 64) * sizeof(float)); };
  const size_t nx = (size_t)n_rows * pad_ld(n_cols), nxt = (size_t)n_cols * pad_ld(n_rows);
  if (precision == CNMF_PRECISION_FP64) {
    *peak = bytes(2 * nx);                                                 // X64
    return 0;
  }
  if (precision == CNMF_PRECISION_FP32) {
    *peak = bytes(nx) + bytes(nxt);                                        // X, Xt
    return 0;
  }
  CNMF_REQUIRE(precision == CNMF_PRECISION_TF32X3 || precision == CNMF_PRECISION_TF32X3_GENERAL ||
                   precision == CNMF_PRECISION_F16X2, "dataset_dense_bytes: bad precision");
  // dataset_finish: the general form holds X, X_hi, X_lo, Xt_hi, Xt_lo; the exact tf32 form X, C, C^T and the
  // detection's two scale vectors; the exact f16 form, while it is built, those plus C and C^T as fp16
  const long long scales = precision == CNMF_PRECISION_TF32X3_GENERAL ? 0 : bytes(pad_ld(n_cols)) + bytes(pad_ld(n_rows));
  const long long general = bytes(nx) * 3 + bytes(nxt) * 2 + scales;
  const long long exact_tf32 = bytes(nx) * 2 + bytes(nxt) + scales;
  const long long exact_f16 = exact_tf32 + bytes((nx + 1) / 2) + bytes((nxt + 1) / 2);
  *peak = std::max(general, std::max(exact_tf32, exact_f16));
  return 0;
}

int cnmf_dataset_create_f64(cnmf_handle_t h, const double* X, int n_rows, int n_cols, long long ld, int src_is_device,
                            void* stream, cnmf_dataset_t* out) {
  CNMF_REQUIRE(h && X && out, "dataset_create_f64: NULL argument");
  CNMF_REQUIRE(n_rows > 0 && n_cols > 0 && ld >= n_cols, "dataset_create_f64: bad shape");
  cudaStream_t s = as_stream(stream);
  return create_dense<double>(h, n_rows, n_cols, CNMF_PRECISION_FP64, s, out,
                              copy_fill(X, ld, n_rows, n_cols, src_is_device != 0, s));
}

int cnmf_dataset_min(cnmf_dataset_t d, float* min_host, void* stream) {
  CNMF_REQUIRE(d && min_host, "dataset_min: NULL argument");
  CNMF_TRY(require_dense(d, "dataset_min"));
  CNMF_CUDA_CHECK(cudaSetDevice(d->h->device));
  return cnmf::matrix_min(d->h, d->X, d->n_rows, d->n_cols, d->ld_c, min_host, as_stream(stream));
}

int cnmf_dataset_destroy(cnmf_dataset_t d) {
  if (!d) return 0;
  for (auto& pr : d->owned) d->h->pool_give(pr.first, pr.second);
  delete d;
  return 0;
}

int cnmf_dataset_shape(cnmf_dataset_t d, int* n_rows, int* n_cols) {
  CNMF_REQUIRE(d, "dataset_shape: NULL dataset");
  if (n_rows) *n_rows = d->n_rows;
  if (n_cols) *n_cols = d->n_cols;
  return 0;
}

int cnmf_dataset_is_exact(cnmf_dataset_t d) {
  return (d && !d->sparse && form_exact(d->form)) ? (d->form == Form::F16_EXACT ? 2 : 1) : 0;
}

int cnmf_dataset_sums(cnmf_dataset_t d, double* sum, double* sum_sq) {
  CNMF_REQUIRE(d, "dataset_sums: NULL dataset");
  if (sum) *sum = d->sum;
  if (sum_sq) *sum_sq = d->sum_sq;
  return 0;
}

// ----------------------------------------------------------------------------- random init
int cnmf_random_init_host(uint32_t seed, double avg, int n_samples, int n_features, int k, float* Wt, long long ldW,
                          float* H, long long ldH) {
  CNMF_REQUIRE(Wt && H && n_samples > 0 && n_features > 0 && k > 0, "random_init: bad arguments");
  CNMF_REQUIRE(ldW >= n_samples && ldH >= n_features, "random_init: leading dimension too small");
  nmf_random_init(seed, avg, n_samples, n_features, k, Wt, ldW, H, ldH);
  return 0;
}

}  // extern "C"

// ----------------------------------------------------------------------------- factorize
namespace {

using clk = std::chrono::steady_clock;
double ms_since(clk::time_point t0) { return std::chrono::duration<double, std::milli>(clk::now() - t0).count(); }

// the restarts of one batched solve: n_components and first packed row of each, and the packed factors
// (Fr = W^T rows, SK x ld_r; Fc = H rows, SK x ld_c) in the dataset's element type T
template <class T>
struct Batch {
  std::vector<int> ks, off;
  int SK = 0;
  T *Fr = nullptr, *Fc = nullptr;
};

template <class T>
int pack_restarts(int n_restarts, const int32_t* ks_in, const std::string& what, Batch<T>* b) {
  b->ks.assign(ks_in, ks_in + n_restarts);
  b->off.resize(n_restarts);
  b->SK = 0;
  for (int r = 0; r < n_restarts; ++r) {
    CNMF_REQUIRE(b->ks[r] >= 1 && b->ks[r] <= KMAX, what + ": n_components must be in [1, 32] on the CUDA path");
    b->off[r] = b->SK;
    b->SK += b->ks[r];
  }
  return 0;
}

void parallel_for(int n, const std::function<void(int)>& fn) {
  int nt = (int)std::thread::hardware_concurrency();
  if (nt < 1) nt = 1;
  nt = std::min(nt, n);
  if (nt <= 1) {
    for (int i = 0; i < n; ++i) fn(i);
    return;
  }
  std::atomic<int> next{0};
  std::vector<std::thread> th;
  th.reserve(nt);
  for (int t = 0; t < nt; ++t)
    th.emplace_back([&] {
      for (;;) {
        const int i = next.fetch_add(1);
        if (i >= n) break;
        fn(i);
      }
    });
  for (auto& t : th) t.join();
}

int check_params(cnmf_dataset_s* d, const cnmf_nmf_params* p) {
  CNMF_REQUIRE(d && p, "NULL dataset or params");
  CNMF_TRY(check_params_precision(d, p));
  CNMF_REQUIRE(p->reserved2 == 0, "params.reserved2 must be 0");
  CNMF_TRY(require_dense(d, "factorize"));
  if (p->beta_loss != CNMF_LOSS_FROBENIUS) CNMF_TRY(cnmf::dataset_ensure_full_transpose(d, nullptr));
  return 0;
}

// parameters of the float64 factorize entry points: float64 dataset, Frobenius loss
int check_params_f64(cnmf_dataset_s* d, const cnmf_nmf_params* p, const std::string& what) {
  CNMF_REQUIRE(d && p, "NULL dataset or params");
  CNMF_TRY(require_f64(d, what.c_str()));
  CNMF_TRY(check_params_precision(d, p));
  CNMF_REQUIRE(p->reserved2 == 0, "params.reserved2 must be 0");
  if (p->beta_loss != CNMF_LOSS_FROBENIUS) {
    set_last_error("cnmf_" + what + "_f64: float64 datasets support beta_loss = frobenius only");
    return -3;
  }
  return 0;
}

// start of every factorize entry point: parameters and arguments checked (args_ok: the entry point's own pointers),
// restarts packed, factor buffers allocated on the handle's device, phase timings reset
template <class T>
int begin_factorize(cnmf_dataset_s* d, const cnmf_nmf_params* p, int n_restarts, const int32_t* ks_in, bool args_ok,
                    const std::string& what, Batch<T>* b) {
  constexpr bool f64 = sizeof(T) == 8;
  CNMF_TRY(f64 ? check_params_f64(d, p, what) : check_params(d, p));
  CNMF_REQUIRE(args_ok && n_restarts > 0 && ks_in, what + (f64 ? "_f64" : "") + ": bad arguments");
  CNMF_TRY(pack_restarts(n_restarts, ks_in, what, b));
  cnmf_handle_s* h = d->h;
  CNMF_CUDA_CHECK(cudaSetDevice(h->device));
  b->Fr = static_cast<T*>(h->dev_buf(f64 ? "fac.Fr64" : "fac.Fr", (size_t)b->SK * d->ld_r * sizeof(T)));
  b->Fc = static_cast<T*>(h->dev_buf(f64 ? "fac.Fc64" : "fac.Fc", (size_t)b->SK * d->ld_c * sizeof(T)));
  if (!b->Fr || !b->Fc) return -2;
  h->t_rng_ms = h->t_h2d_ms = h->t_solve_ms = h->t_d2h_ms = 0;
  return 0;
}

// sklearn's random starts of every restart (the legacy MT19937 / polar-gauss stream), generated in place on the device
// into packed, padded Wt / H.  No host synchronisation: launch_rng_init stages its arguments itself.
template <class T>
int rng_starts_dev(cnmf_dataset_s* d, const Batch<T>& b, const uint32_t* seeds, T* Wt, T* H, cudaStream_t s) {
  const int R = (int)b.ks.size();
  const double mean = d->sum / ((double)d->n_rows * (double)d->n_cols);
  std::vector<double> avgs(R);
  for (int r = 0; r < R; ++r) avgs[r] = std::sqrt(mean / b.ks[r]);
  CNMF_CUDA_CHECK(cudaMemsetAsync(Wt, 0, (size_t)b.SK * d->ld_r * sizeof(T), s));
  CNMF_CUDA_CHECK(cudaMemsetAsync(H, 0, (size_t)b.SK * d->ld_c * sizeof(T), s));
  return launch_rng_init(seeds, b.ks.data(), b.off.data(), avgs.data(), R, d->n_rows, d->n_cols, Wt, d->ld_r, H, d->ld_c,
                         d->h, s);
}

// the same starts drawn on the host (bit-exact numpy legacy stream) into b.Fr / b.Fc, in groups through a pinned
// staging buffer
int rng_starts_host(cnmf_dataset_s* d, const Batch<float>& b, const uint32_t* seeds, cudaStream_t s) {
  cnmf_handle_s* h = d->h;
  const std::vector<int>& ks = b.ks;
  const std::vector<int>& off = b.off;
  const int n_restarts = (int)ks.size();
  const double mean = d->sum / ((double)d->n_rows * (double)d->n_cols);
  const size_t group_budget = (size_t)256 << 20;   // bytes of W^T staged per group
  int r0 = 0;
  while (r0 < n_restarts) {
    int r1 = r0;
    size_t bytes = 0;
    while (r1 < n_restarts && (r1 == r0 || bytes + (size_t)ks[r1] * d->ld_r * 4 <= group_budget)) {
      bytes += (size_t)ks[r1] * d->ld_r * 4;
      ++r1;
    }
    const int rows = off[r1 - 1] + ks[r1 - 1] - off[r0];
    float* stW = static_cast<float*>(h->host_buf("stage.W", (size_t)rows * d->ld_r * 4));
    float* stH = static_cast<float*>(h->host_buf("stage.H", (size_t)rows * d->ld_c * 4));
    if (!stW || !stH) return -2;
    auto t_rng = clk::now();
    parallel_for(r1 - r0, [&](int i) {
      const int r = r0 + i;
      const double avg = std::sqrt(mean / ks[r]);
      float* w = stW + (size_t)(off[r] - off[r0]) * d->ld_r;
      float* hh = stH + (size_t)(off[r] - off[r0]) * d->ld_c;
      nmf_random_init(seeds[r], avg, d->n_rows, d->n_cols, ks[r], w, d->ld_r, hh, d->ld_c);
      for (int c = 0; c < ks[r]; ++c) {                  // zero the row padding (each worker its own rows)
        std::memset(w + (size_t)c * d->ld_r + d->n_rows, 0, (size_t)(d->ld_r - d->n_rows) * 4);
        std::memset(hh + (size_t)c * d->ld_c + d->n_cols, 0, (size_t)(d->ld_c - d->n_cols) * 4);
      }
    });
    h->t_rng_ms += ms_since(t_rng);
    auto t_h2d = clk::now();
    CNMF_CUDA_CHECK(cudaMemcpyAsync(b.Fr + (size_t)off[r0] * d->ld_r, stW, (size_t)rows * d->ld_r * 4,
                                    cudaMemcpyHostToDevice, s));
    CNMF_CUDA_CHECK(cudaMemcpyAsync(b.Fc + (size_t)off[r0] * d->ld_c, stH, (size_t)rows * d->ld_c * 4,
                                    cudaMemcpyHostToDevice, s));
    CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
    h->t_h2d_ms += ms_since(t_h2d);
    r0 = r1;
  }
  return 0;
}

// float64 datasets take their starts from the device generator or the NNDSVD family only
int rng_starts_host(cnmf_dataset_s*, const Batch<double>&, const uint32_t*, cudaStream_t) {
  set_last_error("cnmf_factorize_f64: the host random generator (params.reserved bit 0) serves float datasets only");
  return -3;
}

// end of every factorize entry point: the solve from the starts in b.Fr / b.Fc, then its results out.
// Null outputs are skipped; spectra_dev gets SK rows of dev_cols elements at row stride ld_dev.
template <class T>
int solve_and_copy_out(cnmf_dataset_s* d, const Batch<T>& b, const cnmf_nmf_params& p, T* spectra_host, T* usages_host,
                       T* spectra_dev, long long ld_dev, int dev_cols, int32_t* n_iter_host, double* err_host,
                       cudaStream_t s) {
  cnmf_handle_s* h = d->h;
  constexpr size_t e = sizeof(T);
  SolveIO<T> io;
  io.R = (int)b.ks.size();
  io.ks = b.ks;
  io.Fr = b.Fr;
  io.Fc = b.Fc;
  io.update_cols = true;
  auto t_solve = clk::now();
  CNMF_TRY(solve_batched(h, make_view(d, false), io, p, s));
  h->t_solve_ms = ms_since(t_solve);
  auto t_d2h = clk::now();
  if (spectra_dev)      // result stays in HBM (multi-GPU path: the slab goes straight into the NCCL all-gather)
    CNMF_CUDA_CHECK(cudaMemcpy2DAsync(spectra_dev, (size_t)ld_dev * e, b.Fc, (size_t)d->ld_c * e, (size_t)dev_cols * e,
                                      b.SK, cudaMemcpyDeviceToDevice, s));
  if (spectra_host)
    CNMF_CUDA_CHECK(cudaMemcpy2DAsync(spectra_host, (size_t)d->n_cols * e, b.Fc, (size_t)d->ld_c * e,
                                      (size_t)d->n_cols * e, b.SK, cudaMemcpyDeviceToHost, s));
  if (usages_host)
    CNMF_CUDA_CHECK(cudaMemcpy2DAsync(usages_host, (size_t)d->n_rows * e, b.Fr, (size_t)d->ld_r * e,
                                      (size_t)d->n_rows * e, b.SK, cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
  h->t_d2h_ms = ms_since(t_d2h);
  for (int r = 0; r < io.R; ++r) {
    if (n_iter_host) n_iter_host[r] = io.n_iter[r];
    if (err_host) err_host[r] = io.err[r];
  }
  return 0;
}

template <class T>
int factorize_impl(cnmf_dataset_t d, int n_restarts, const int32_t* ks_in, const uint32_t* seeds,
                          const cnmf_nmf_params* p, T* spectra_host, T* usages_host, int32_t* n_iter_host,
                          double* err_host, void* stream, T* spectra_dev, long long ld_dev) {
  Batch<T> b;
  CNMF_TRY(begin_factorize(d, p, n_restarts, ks_in, seeds && (spectra_host || spectra_dev), "factorize", &b));
  CNMF_REQUIRE(!spectra_dev || ld_dev >= d->n_cols, "factorize: device output row stride too small");
  cudaStream_t s = as_stream(stream);
  const int init = (p->reserved >> 1) & 3;
  auto t_init = clk::now();
  if (init != CNMF_INIT_RANDOM) {
    CNMF_TRY(nndsvd_starts_dev(d, n_restarts, b.ks.data(), seeds, init, b.Fr, b.Fc, s));
    d->h->t_rng_ms = ms_since(t_init);
  } else if ((p->reserved & 1) == 0) {
    // device RNG (default): the solve is enqueued behind the generator on the same stream (t_rng_ms = enqueue time;
    // the kernel's time is part of t_solve_ms)
    CNMF_TRY(rng_starts_dev(d, b, seeds, b.Fr, b.Fc, s));
    d->h->t_rng_ms = ms_since(t_init);
  } else {
    CNMF_TRY(rng_starts_host(d, b, seeds, s));
  }
  return solve_and_copy_out(d, b, *p, spectra_host, usages_host, spectra_dev, ld_dev, d->n_cols, n_iter_host, err_host,
                            s);
}

// the starts Wt0_host / H0_host (n_rows / n_cols elements per row, SK rows each) padded into the packed factors
template <class T>
int factorize_init_impl(cnmf_dataset_t d, int n_restarts, const int32_t* ks_in, const T* Wt0_host,
                               const T* H0_host, const cnmf_nmf_params* p, T* spectra_host, T* usages_host,
                               int32_t* n_iter_host, double* err_host, void* stream) {
  Batch<T> b;
  CNMF_TRY(begin_factorize(d, p, n_restarts, ks_in, Wt0_host && H0_host && spectra_host, "factorize_init", &b));
  cudaStream_t s = as_stream(stream);
  constexpr size_t e = sizeof(T);
  auto t_h2d = clk::now();
  CNMF_CUDA_CHECK(cudaMemsetAsync(b.Fr, 0, (size_t)b.SK * d->ld_r * e, s));
  CNMF_CUDA_CHECK(cudaMemsetAsync(b.Fc, 0, (size_t)b.SK * d->ld_c * e, s));
  CNMF_CUDA_CHECK(cudaMemcpy2DAsync(b.Fr, (size_t)d->ld_r * e, Wt0_host, (size_t)d->n_rows * e, (size_t)d->n_rows * e,
                                    b.SK, cudaMemcpyHostToDevice, s));
  CNMF_CUDA_CHECK(cudaMemcpy2DAsync(b.Fc, (size_t)d->ld_c * e, H0_host, (size_t)d->n_cols * e, (size_t)d->n_cols * e,
                                    b.SK, cudaMemcpyHostToDevice, s));
  CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
  d->h->t_h2d_ms = ms_since(t_h2d);
  return solve_and_copy_out<T>(d, b, *p, spectra_host, usages_host, nullptr, 0, 0, n_iter_host, err_host, s);
}

}  // namespace

extern "C" {

int cnmf_factorize(cnmf_dataset_t d, int n_restarts, const int32_t* ks_in, const uint32_t* seeds,
                   const cnmf_nmf_params* p, float* spectra_host, float* usages_host, int32_t* n_iter_host,
                   double* err_host, void* stream) {
  CNMF_TRY(require_f32(d, "factorize"));
  CNMF_REQUIRE(spectra_host, "factorize: spectra_host is NULL");
  return factorize_impl<float>(d, n_restarts, ks_in, seeds, p, spectra_host, usages_host, n_iter_host, err_host, stream, nullptr, 0);
}

int cnmf_factorize_seeds_dev(cnmf_dataset_t d, int n_restarts, const int32_t* ks_in, const uint32_t* seeds,
                             const cnmf_nmf_params* p, float* spectra_dev, long long ld_out, int32_t* n_iter_host,
                             double* err_host, void* stream) {
  CNMF_TRY(require_dense(d, "factorize_seeds_dev"));
  CNMF_REQUIRE(spectra_dev, "factorize_seeds_dev: spectra_dev is NULL");
  return factorize_impl<float>(d, n_restarts, ks_in, seeds, p, nullptr, nullptr, n_iter_host, err_host, stream, spectra_dev,
                               ld_out);
}

int cnmf_last_timing(cnmf_handle_t h, double* rng_ms, double* h2d_ms, double* solve_ms, double* d2h_ms) {
  CNMF_REQUIRE(h, "last_timing: NULL handle");
  if (rng_ms) *rng_ms = h->t_rng_ms;
  if (h2d_ms) *h2d_ms = h->t_h2d_ms;
  if (solve_ms) *solve_ms = h->t_solve_ms;
  if (d2h_ms) *d2h_ms = h->t_d2h_ms;
  return 0;
}

int cnmf_factorize_init(cnmf_dataset_t d, int n_restarts, const int32_t* ks_in, const float* Wt0_host,
                        const float* H0_host, const cnmf_nmf_params* p, float* spectra_host, float* usages_host,
                        int32_t* n_iter_host, double* err_host, void* stream) {
  CNMF_TRY(require_f32(d, "factorize_init"));
  return factorize_init_impl(d, n_restarts, ks_in, Wt0_host, H0_host, p, spectra_host, usages_host, n_iter_host, err_host,
                             stream);
}

int cnmf_factorize_dev(cnmf_dataset_t d, int n_restarts, const int32_t* ks_in, const float* Wt0_dev,
                       const float* H0_dev, const cnmf_nmf_params* p, float* spectra_dev, int32_t* n_iter_host,
                       double* err_host, void* stream) {
  Batch<float> b;
  CNMF_TRY(begin_factorize(d, p, n_restarts, ks_in, Wt0_dev && H0_dev && spectra_dev, "factorize_dev", &b));
  cudaStream_t s = as_stream(stream);
  CNMF_CUDA_CHECK(cudaMemcpyAsync(b.Fr, Wt0_dev, (size_t)b.SK * d->ld_r * 4, cudaMemcpyDeviceToDevice, s));
  CNMF_CUDA_CHECK(cudaMemcpyAsync(b.Fc, H0_dev, (size_t)b.SK * d->ld_c * 4, cudaMemcpyDeviceToDevice, s));
  // spectra_dev has the layout of H0_dev: whole padded rows, the zero padding included
  return solve_and_copy_out<float>(d, b, *p, nullptr, nullptr, spectra_dev, d->ld_c, d->ld_c, n_iter_host, err_host, s);
}

int cnmf_factorize_f64(cnmf_dataset_t d, int n_restarts, const int32_t* ks_in, const uint32_t* seeds,
                       const cnmf_nmf_params* p, double* spectra_host, double* usages_host, int32_t* n_iter_host,
                       double* err_host, void* stream) {
  return factorize_impl<double>(d, n_restarts, ks_in, seeds, p, spectra_host, usages_host, n_iter_host, err_host, stream,
                                nullptr, 0);
}

int cnmf_factorize_init_f64(cnmf_dataset_t d, int n_restarts, const int32_t* ks_in, const double* Wt0_host,
                            const double* H0_host, const cnmf_nmf_params* p, double* spectra_host, double* usages_host,
                            int32_t* n_iter_host, double* err_host, void* stream) {
  return factorize_init_impl(d, n_restarts, ks_in, Wt0_host, H0_host, p, spectra_host, usages_host, n_iter_host, err_host,
                             stream);
}

int cnmf_random_init_dev(cnmf_dataset_t d, int n_restarts, const int32_t* ks_in, const uint32_t* seeds, float* Wt_dev,
                         float* H_dev, void* stream) {
  CNMF_REQUIRE(d && n_restarts > 0 && ks_in && seeds && Wt_dev && H_dev, "random_init_dev: bad arguments");
  CNMF_TRY(require_dense(d, "random_init_dev"));
  cudaStream_t s = as_stream(stream);
  CNMF_CUDA_CHECK(cudaSetDevice(d->h->device));
  Batch<float> b;
  CNMF_TRY(pack_restarts(n_restarts, ks_in, "random_init_dev", &b));
  CNMF_TRY(rng_starts_dev(d, b, seeds, Wt_dev, H_dev, s));
  CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
  return 0;
}

int cnmf_dataset_ld(cnmf_dataset_t d, int* ld_rows, int* ld_cols) {
  CNMF_REQUIRE(d, "dataset_ld: NULL dataset");
  if (ld_rows) *ld_rows = d->ld_r;
  if (ld_cols) *ld_cols = d->ld_c;
  return 0;
}

}  // extern "C"

namespace cnmf {

int dataset_ensure_full_transpose(cnmf_dataset_s* d, cudaStream_t s) {
  if (d->Xt) return 0;
  CNMF_CUDA_CHECK(cudaSetDevice(d->h->device));
  const size_t nxt = (size_t)d->n_cols * d->ld_r;
  CNMF_TRY(dataset_alloc(d, &d->Xt, nxt));
  CNMF_CUDA_CHECK(cudaMemsetAsync(d->Xt, 0, nxt * sizeof(float), s));
  CNMF_TRY(launch_transpose(d->X, d->n_rows, d->n_cols, d->ld_c, d->Xt, nullptr, nullptr, d->ld_r, s));
  d->h->launches += 1;
  CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
  return 0;
}

}  // namespace cnmf
