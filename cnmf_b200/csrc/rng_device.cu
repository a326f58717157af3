// Device-side random NMF initialisation: numpy's legacy RandomState(seed).standard_normal stream
// (MT19937 + polar "legacy gauss", legacy_gauss.cuh), reproduced in parallel -- one thread block per restart.
//
// What sklearn draws (sklearn/decomposition/_nmf.py:296-307, via check_random_state(int)):
//   H = |avg * N(0,1)|  (k x n_features, row-major)  FIRST, then  W = |avg * N(0,1)|  (n_samples x k).
// The values are written straight into the packed device layout (H rows, W^T rows).
//
// Exactness: see legacy_gauss.cuh -- only log() may differ from glibc in the last bit of the fp64 result; after
// |avg*z| is rounded to fp32 this is visible in about one value per 10^8.  The host generator (legacy_rng.cpp,
// bit-exact by construction) stays available (`rng="host"`) and is what the parity fixtures use.
#include <cuda_runtime.h>

#include "common.cuh"
#include "engine.h"
#include "legacy_gauss.cuh"

namespace cnmf {

namespace {

// T = float: |avg*z| rounded to fp32 (the float datasets); T = double: kept in fp64 (float64 datasets)
template <typename T>
__global__ void __launch_bounds__(LEGACY_GAUSS_THREADS)
rng_init_kernel(const uint32_t* __restrict__ seeds, const int* __restrict__ ks, const int* __restrict__ offs,
                const double* __restrict__ avgs, int n_samples, int n_features, T* __restrict__ Wt, long long ldW,
                T* __restrict__ H, long long ldH) {
  __shared__ LegacyGaussShared sh;
  const int r = blockIdx.x;
  const int k = ks[r];
  const long long row0 = offs[r];
  const double avg = avgs[r];
  const long long nH = (long long)k * n_features;
  const long long total = nH + (long long)n_samples * k;
  legacy_gauss_block(seeds[r], total, sh, [&](long long t, double z) {
    const T v = (T)fabs(__dmul_rn(avg, z));
    if (t < nH) {
      const long long c = t / n_features, g = t % n_features;
      H[(row0 + c) * ldH + g] = v;
    } else {
      const long long tt = t - nH;
      const long long j = tt / k, c = tt % k;
      Wt[(row0 + c) * ldW + j] = v;
    }
  });
}

// Fills the packed initial factors on the device.  d_meta: device scratch of >= 4 * R ints + R doubles (8-byte aligned).
template <typename T>
int rng_init(const uint32_t* seeds_host, const int* ks_host, const int* offs_host, const double* avgs_host, int R,
             int n_samples, int n_features, T* Wt, long long ldW, T* H, long long ldH, cnmf_handle_s* h, cudaStream_t s) {
  const size_t bytes = sizeof(double) * R + sizeof(int) * 3 * (size_t)R;
  unsigned char* d = static_cast<unsigned char*>(h->dev_buf("rng.meta", bytes));
  unsigned char* hp = static_cast<unsigned char*>(h->host_buf("rng.meta", bytes));
  if (!d || !hp) return -2;
  double* h_avg = reinterpret_cast<double*>(hp);
  uint32_t* h_seed = reinterpret_cast<uint32_t*>(hp + sizeof(double) * R);
  int* h_k = reinterpret_cast<int*>(hp + sizeof(double) * R + sizeof(int) * (size_t)R);
  int* h_off = h_k + R;
  for (int r = 0; r < R; ++r) {
    h_avg[r] = avgs_host[r];
    h_seed[r] = seeds_host[r];
    h_k[r] = ks_host[r];
    h_off[r] = offs_host[r];
  }
  CNMF_CUDA_CHECK(cudaMemcpyAsync(d, hp, bytes, cudaMemcpyHostToDevice, s));
  const double* d_avg = reinterpret_cast<const double*>(d);
  const uint32_t* d_seed = reinterpret_cast<const uint32_t*>(d + sizeof(double) * R);
  const int* d_k = reinterpret_cast<const int*>(d + sizeof(double) * R + sizeof(int) * (size_t)R);
  const int* d_off = d_k + R;
  rng_init_kernel<T><<<R, LEGACY_GAUSS_THREADS, 0, s>>>(d_seed, d_k, d_off, d_avg, n_samples, n_features, Wt, ldW, H, ldH);
  CNMF_CUDA_CHECK(cudaGetLastError());
  h->launches += 1;
  return 0;
}

}  // namespace

int launch_rng_init(const uint32_t* seeds_host, const int* ks_host, const int* offs_host, const double* avgs_host, int R,
                    int n_samples, int n_features, float* Wt, long long ldW, float* H, long long ldH, cnmf_handle_s* h,
                    cudaStream_t s) {
  return rng_init(seeds_host, ks_host, offs_host, avgs_host, R, n_samples, n_features, Wt, ldW, H, ldH, h, s);
}

int launch_rng_init(const uint32_t* seeds_host, const int* ks_host, const int* offs_host, const double* avgs_host, int R,
                    int n_samples, int n_features, double* Wt, long long ldW, double* H, long long ldH, cnmf_handle_s* h,
                    cudaStream_t s) {
  return rng_init(seeds_host, ks_host, offs_host, avgs_host, R, n_samples, n_features, Wt, ldW, H, ldH, h, s);
}

}  // namespace cnmf
