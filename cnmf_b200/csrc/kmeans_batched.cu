// KMeans(n_clusters=K, n_init, random_state) of the consensus step (cnmf.py:908-910 -> sklearn _kmeans.py:1436-1563) with
// every initialisation resident and advancing TOGETHER on the device:
//
//   * k-means++ (sklearn _kmeans.py:180-278) for all n_init runs at once.  The random draws are data-independent in count
//     and order, so the host draws them from the legacy RandomState exactly as sklearn would (first centre index,
//     n_local_trials uniforms per further centre) and ships them once; the device does the rest: candidate distances, the
//     potential of every candidate, argmin, and the next candidates by an exactly sequential float64 cumulative sum +
//     searchsorted (numpy's cumsum order).  2 launches per centre, no host round trip.
//   * Lloyd (sklearn _kmeans.py:630-758, _k_means_lloyd.pyx:168-219) for all runs at once: assignment, stable member
//     lists, fp64 centre sums in member order, centre update + shift, and the per-run stopping rule on the device.  The
//     host reads one small flag block per iteration (for ALL runs) instead of three scalars per run and iteration.
//   * final E step + inertia per run; the host picks the winner with sklearn's rule (_kmeans.py:1534-1541).
// An empty cluster (sklearn's relocation rule, _k_means_common.pyx:167-211) is reported to the caller, which then runs
// the per-run host-assisted path (cnmf_kmeans_step): it is rare and not worth a device implementation.
//
// The E step, the member-order centre sums, the centre update and the stopping rule have the arithmetic and summation
// orders of the per-run path (cnmf_kmeans_step), so from the same k-means++ centres every run's labels, centres and
// iteration count are those of the per-run path, and labels equal scikit-learn's on the parity fixtures.  Two sums are
// associated differently, so they agree to rounding, not bit for bit: the candidate potentials (here blocks of 8 rows,
// then the blocks in order; there host dot products) and the inertia (here 256 threads per run; there sum_kernel's one
// block of 1024).  A potential that differs in its last bits can move a k-means++ draw only when a uniform lands within
// those bits of a cumulative-sum boundary.
#include <algorithm>
#include <chrono>
#include <cstring>
#include <type_traits>
#include <vector>

#include "engine.h"

namespace cnmf {
namespace {

template <typename T>
__device__ __forceinline__ T kb_block_sum_all(T v, T* smem /* >= 33 */) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) smem[warp] = v;
  __syncthreads();
  const int nw = (blockDim.x + 31) >> 5;
  T r = (threadIdx.x < nw) ? smem[threadIdx.x] : T(0);
  if (warp == 0) {
    r = warp_sum(r);
    if (lane == 0) smem[32] = r;
  }
  __syncthreads();
  return smem[32];
}

template <typename T>
struct KmState {
  const T* S; int R, G, ld, K, n_init, n_trials, row_blocks;
  double* closest;      // [n_init][R]
  double* newd;         // [n_init][n_trials][R]
  double* part;         // [n_init][n_trials][row_blocks]
  int* cand;            // [n_init][8]
  int* centre_idx;      // [n_init][K]
  double* pot;          // [n_init]
  const double* unif;   // [n_init][K-1][n_trials]
};

// four consecutive elements as one load
template <typename T> struct KbVec4;
template <> struct KbVec4<float> { using type = float4; };
struct __align__(32) kb_double4a { double x, y, z, w; };
template <> struct KbVec4<double> { using type = kb_double4a; };

// squared distance of row r to `NC` rows: differences in T, fp64 accumulation, rounded to T (what the per-run path
// hands to the host: cand_dist_kernel)
template <typename T, int NC>
__device__ __forceinline__ void row_dists(const T* __restrict__ S, int G, int ld, int r, const int* idx, int n_c,
                                          int lane, double (&out)[NC]) {
  using V4 = typename KbVec4<T>::type;
  const V4* row = reinterpret_cast<const V4*>(S + (long long)r * ld);
  const V4* cand[NC];
#pragma unroll
  for (int c = 0; c < NC; ++c) cand[c] = reinterpret_cast<const V4*>(S + (long long)idx[c < n_c ? c : 0] * ld);
  double acc[NC];
#pragma unroll
  for (int c = 0; c < NC; ++c) acc[c] = 0.0;
  const int g4 = G / 4;
  for (int q = lane; q < g4; q += 32) {
    const V4 x = row[q];
#pragma unroll
    for (int c = 0; c < NC; ++c) {
      const V4 y = cand[c][q];
      const T d0 = x.x - y.x, d1 = x.y - y.y, d2 = x.z - y.z, d3 = x.w - y.w;
      acc[c] += (double)d0 * d0 + (double)d1 * d1 + (double)d2 * d2 + (double)d3 * d3;
    }
  }
  for (int g = 4 * g4 + lane; g < G; g += 32) {
    const T x = S[(long long)r * ld + g];
#pragma unroll
    for (int c = 0; c < NC; ++c) {
      const T d = x - S[(long long)idx[c < n_c ? c : 0] * ld + g];
      acc[c] += (double)d * d;
    }
  }
#pragma unroll
  for (int c = 0; c < NC; ++c) out[c] = (double)(T)warp_sum(acc[c]);
}

// step 0: closest = distances to the first centre.  step > 0: newd[j] = min(closest, distance to candidate j).
// Per block: fixed-order partial sums of what was written (potentials).
template <typename T, int NC>
__global__ void __launch_bounds__(256)
kpp_eval_kernel(KmState<T> st, int first) {
  __shared__ double sm[8][NC];
  const int t = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r = blockIdx.x * 8 + warp;
  const int n_c = first ? 1 : st.n_trials;
  const int* idx = first ? st.centre_idx + (long long)t * st.K : st.cand + t * 8;
  double d[NC];
#pragma unroll
  for (int c = 0; c < NC; ++c) d[c] = 0.0;
  if (r < st.R) {
    row_dists<T, NC>(st.S, st.G, st.ld, r, idx, n_c, lane, d);
    if (first) {
      if (lane == 0) st.closest[(long long)t * st.R + r] = d[0];
    } else {
      const double cl = st.closest[(long long)t * st.R + r];
#pragma unroll
      for (int c = 0; c < NC; ++c) {
        d[c] = fmin(cl, d[c]);
        if (lane == 0 && c < n_c) st.newd[((long long)t * st.n_trials + c) * st.R + r] = d[c];
      }
    }
  }
  if (lane == 0) {
#pragma unroll
    for (int c = 0; c < NC; ++c) sm[warp][c] = d[c];
  }
  __syncthreads();
  if (threadIdx.x < n_c) {
    double a = 0.0;
    for (int w = 0; w < 8; ++w) a += sm[w][threadIdx.x];
    st.part[((long long)t * st.n_trials + threadIdx.x) * st.row_blocks + blockIdx.x] = a;
  }
}

// one block per run: potentials of the candidates (fixed-order sums), argmin (first minimum wins), commit the winner,
// then the next candidates: searchsorted(cumsum(closest), uniform * pot) with numpy's sequential float64 cumsum
template <typename T>
__global__ void __launch_bounds__(256)
kpp_select_kernel(KmState<T> st, int step /* centre being committed: 0 = the first one */) {
  extern __shared__ double cl_s[];            // R doubles
  __shared__ double cpot[8];
  __shared__ int s_best;
  const int t = blockIdx.x;
  const int n_c = step == 0 ? 1 : st.n_trials;
  if (threadIdx.x < n_c) {
    double a = 0.0;
    const double* p = st.part + ((long long)t * st.n_trials + threadIdx.x) * st.row_blocks;
    for (int b = 0; b < st.row_blocks; ++b) a += p[b];
    cpot[threadIdx.x] = a;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int best = 0;
    for (int j = 1; j < n_c; ++j)
      if (cpot[j] < cpot[best]) best = j;      // np.argmin: first minimum
    s_best = best;
    st.pot[t] = cpot[best];
    if (step > 0) st.centre_idx[(long long)t * st.K + step] = st.cand[t * 8 + best];
  }
  __syncthreads();
  double* cl = st.closest + (long long)t * st.R;
  if (step > 0) {
    const double* src = st.newd + ((long long)t * st.n_trials + s_best) * st.R;
    for (int i = threadIdx.x; i < st.R; i += blockDim.x) {
      const double v = src[i];
      cl[i] = v;
      cl_s[i] = v;
    }
  } else {
    for (int i = threadIdx.x; i < st.R; i += blockDim.x) cl_s[i] = cl[i];
  }
  __syncthreads();
  if (step + 1 >= st.K || threadIdx.x != 0) return;
  // candidates for centre step + 1 (sklearn _kmeans.py:249-254)
  const double pot = st.pot[t];
  const double* u = st.unif + ((long long)t * (st.K - 1) + step) * st.n_trials;
  double rv[8];
  int found[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {                 // fixed trip count: rv / found stay in registers
    rv[j] = j < st.n_trials ? u[j] * pot : 0.0;
    found[j] = j < st.n_trials ? -1 : 0;
  }
  double c = 0.0;
  int left = st.n_trials;
  double next_rv = rv[0];                       // smallest pending value: one comparison per element in the common case
#pragma unroll
  for (int j = 1; j < 8; ++j)
    if (j < st.n_trials) next_rv = fmin(next_rv, rv[j]);
  for (int i = 0; i < st.R && left > 0; ++i) {
    c += cl_s[i];                               // np.cumsum: strictly sequential
    if (c >= next_rv) {                         // searchsorted side='left': first index with cumsum >= value
      next_rv = 1.0e308;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        if (found[j] < 0) {
          if (c >= rv[j]) {
            found[j] = i;
            --left;
          } else {
            next_rv = fmin(next_rv, rv[j]);
          }
        }
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j)
    if (j < st.n_trials) st.cand[t * 8 + j] = found[j] < 0 ? st.R - 1 : found[j];   // np.clip
}

// C64: the fp64 centres; CT: their fp32 copy for the E step (T = float only: with T = double the E step reads C64)
template <typename T>
__global__ void __launch_bounds__(256)
kpp_gather_centres_kernel(KmState<T> st, double* __restrict__ C64, T* __restrict__ CT) {
  const int k = blockIdx.x, t = blockIdx.y;
  const T* src = st.S + (long long)st.centre_idx[(long long)t * st.K + k] * st.ld;
  const long long o = ((long long)t * st.K + k) * st.G;
  for (int g = threadIdx.x; g < st.G; g += blockDim.x) {
    const T v = src[g];
    if constexpr (!std::is_same<T, double>::value) CT[o + g] = v;
    C64[o + g] = (double)v;
  }
}

// ---------------------------------------------------------------- Lloyd, all runs at once
template <typename T>
struct LloydState {
  const T* S; int R, G, ld, K, n_init;
  int* labels;        // [n_init][R]
  T* mind;            // [n_init][R]
  int* counts;        // [n_init][K]
  int* order;         // [n_init][K][R]
  double* sums;       // [n_init][K][G]
  double* shift_part; // [n_init][K]
  int* flags;         // [n_init][4]: n_changed, any_empty, done, n_iter
  double* inertia;    // [n_init]
};

// E step: one warp per row (arithmetic of kmeans_assign_kernel); `final_pass` assigns against every run's final centres.
// CEa / CEb: the two ping-pong centre buffers the E step reads (fp32 copies for T = float, the fp64 centres for double)
template <typename T>
__global__ void __launch_bounds__(256)
kmb_assign_kernel(LloydState<T> st, const T* __restrict__ CEa, const T* __restrict__ CEb, int parity, int final_pass) {
  const int t = blockIdx.y;
  int* fl = st.flags + t * 4;
  const bool done = fl[2] != 0;
  if (!final_pass && done) return;
  // centres this run reads: the live parity while iterating; after it stopped, the buffer its last step wrote
  const int buf = final_pass ? (fl[3] & 1) : parity;
  const T* C = (buf ? CEb : CEa) + (long long)t * st.K * st.G;
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= st.R) return;
  const T* x = st.S + (long long)row * st.ld;
  T best = T(0);
  int bl = 0;
  for (int c = 0; c < st.K; ++c) {
    const T* cc = C + (long long)c * st.G;
    T a = T(0);
    for (int g = lane; g < st.G; g += 32) {
      const T d = x[g] - cc[g];
      a = fma(d, d, a);
    }
    a = warp_sum(a);
    if (c == 0 || a < best) {   // strict '<': first minimum wins (sklearn _k_means_lloyd.pyx:205-209)
      best = a;
      bl = c;
    }
  }
  if (lane == 0) {
    int* lab = st.labels + (long long)t * st.R;
    if (lab[row] != bl) atomicAdd(fl, 1);
    lab[row] = bl;
    st.mind[(long long)t * st.R + row] = best;
  }
}

// stable counting sort of the row indices by label (members of cluster c in row order): 1024 rows at a time, ranks
// from warp ballots, warp offsets from a per-cluster scan over the 32 warps
template <typename T>
__global__ void __launch_bounds__(1024)
kmb_members_kernel(LloydState<T> st) {
  __shared__ int base[32];            // members of cluster c placed so far
  __shared__ int wtot[32][33];        // [cluster][warp]
  const int t = blockIdx.x;
  if (st.flags[t * 4 + 2]) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int* lab = st.labels + (long long)t * st.R;
  int* order = st.order + (long long)t * st.K * st.R;
  if (threadIdx.x < 32) base[threadIdx.x] = 0;
  __syncthreads();
  for (int r0 = 0; r0 < st.R; r0 += 1024) {
    const int r = r0 + threadIdx.x;
    const int l = r < st.R ? lab[r] : -1;
    int my_rank = 0;
    for (int c = 0; c < st.K; ++c) {
      const unsigned m = __ballot_sync(0xffffffffu, l == c);
      if (l == c) my_rank = __popc(m & ((1u << lane) - 1u));
      if (lane == 0) wtot[c][warp] = __popc(m);
    }
    __syncthreads();
    if (threadIdx.x < st.K) {         // exclusive scan over the warps, in warp order
      int a = base[threadIdx.x];
      for (int w = 0; w < 32; ++w) {
        const int n = wtot[threadIdx.x][w];
        wtot[threadIdx.x][w] = a;
        a += n;
      }
      base[threadIdx.x] = a;
    }
    __syncthreads();
    if (l >= 0) order[(long long)l * st.R + wtot[l][warp] + my_rank] = r;
    __syncthreads();
  }
  if (threadIdx.x < st.K) st.counts[t * st.K + threadIdx.x] = base[threadIdx.x];
}

// M step: per-cluster column sums in fp64, members visited in row order (arithmetic of cluster_sums_kernel)
template <typename T>
__global__ void __launch_bounds__(128)
kmb_sums_kernel(LloydState<T> st) {
  const int c = blockIdx.y, t = blockIdx.z;
  if (st.flags[t * 4 + 2]) return;
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= st.G) return;
  const int n = st.counts[t * st.K + c];
  const int* mem = st.order + ((long long)t * st.K + c) * st.R;
  double a = 0.0;
  for (int i = 0; i < n; ++i) a += (double)st.S[(long long)mem[i] * st.ld + g];
  st.sums[((long long)t * st.K + c) * st.G + g] = a;
}

// new centre = sums * (1 / count), squared shift against the current one (arithmetic of centre_update_kernel);
// CT_new: the fp32 copy for the next E step (T = float only)
template <typename T>
__global__ void __launch_bounds__(256)
kmb_centre_update_kernel(LloydState<T> st, const double* __restrict__ C64_cur, double* __restrict__ C64_new,
                         T* __restrict__ CT_new) {
  __shared__ double sm[33];
  const int j = blockIdx.x, t = blockIdx.y;
  if (st.flags[t * 4 + 2]) return;
  const int w = st.counts[t * st.K + j];
  if (w == 0) {
    if (threadIdx.x == 0) {
      atomicExch(st.flags + t * 4 + 1, 1);
      st.shift_part[t * st.K + j] = 0.0;
    }
    return;
  }
  const double inv = 1.0 / (double)w;
  const long long o = ((long long)t * st.K + j) * st.G;
  double acc = 0.0;
  for (int g = threadIdx.x; g < st.G; g += blockDim.x) {
    const double nv = st.sums[o + g] * inv;
    const double d = nv - C64_cur[o + g];
    acc += d * d;
    C64_new[o + g] = nv;
    if constexpr (!std::is_same<T, double>::value) CT_new[o + g] = (T)nv;
  }
  acc = kb_block_sum_all(acc, sm);
  if (threadIdx.x == 0) st.shift_part[t * st.K + j] = acc;
}

// the stopping rule of the per-run loop, per run: stop when no label changed or the total shift <= tol
// (sklearn _kmeans.py:700-715); flags[3] = iterations run = index of the buffer that holds the final centres (parity)
template <typename T>
__global__ void kmb_check_kernel(LloydState<T> st, double tol_abs, int max_iter) {
  const int t = threadIdx.x;
  if (t >= st.n_init) return;
  int* fl = st.flags + t * 4;
  if (fl[2]) return;
  fl[3] += 1;
  if (fl[1]) return;                      // an empty cluster: the host takes over (flags[1] stays set)
  double tot = 0.0;
  for (int j = 0; j < st.K; ++j) tot += st.shift_part[t * st.K + j];      // fixed order
  if (fl[0] == 0 || tot <= tol_abs || fl[3] >= max_iter) fl[2] = 1;
  fl[0] = 0;
}

template <typename T>
__global__ void __launch_bounds__(256)
kmb_inertia_kernel(LloydState<T> st) {
  __shared__ double sm[33];
  const int t = blockIdx.x;
  const T* v = st.mind + (long long)t * st.R;
  double a = 0.0;
  for (int i = threadIdx.x; i < st.R; i += blockDim.x) a += (double)v[i];
  a = kb_block_sum_all(a, sm);
  if (threadIdx.x == 0) st.inertia[t] = a;
}

template <typename T>
int kmeans_fit(cnmf_handle_t h, const T* S_dev, int R, int G, int ld, int K, int n_init, int max_iter, double tol_abs,
               const int32_t* first_idx_host, const double* uniforms_host, int n_trials,
               int32_t* labels_host /* n_init x R */, double* inertia_host /* n_init */, int32_t* n_iter_host /* n_init */,
               int32_t* needs_host_path, void* stream) {
  CNMF_REQUIRE(h && S_dev && first_idx_host && labels_host && inertia_host && needs_host_path, "kmeans_fit: NULL argument");
  CNMF_REQUIRE(R > 0 && G > 0 && ld >= G && ld % 4 == 0 && K >= 1 && K <= 32 && n_init >= 1 && n_init <= 32 &&
                   n_trials >= 1 && n_trials <= 8 && (K == 1 || uniforms_host) && max_iter >= 1,
               "kmeans_fit: bad arguments (K <= 32, n_init <= 32, n_trials <= 8)");
  CNMF_REQUIRE((size_t)R * sizeof(double) <= 200 * 1024, "kmeans_fit: too many rows for the in-kernel cumulative sum");
  cudaStream_t s = as_stream(stream);
  CNMF_CUDA_CHECK(cudaSetDevice(h->device));
  const int row_blocks = (R + 7) / 8;
  const size_t nR = (size_t)n_init * R, nKG = (size_t)n_init * K * G;
  KmState<T> st{};
  st.S = S_dev; st.R = R; st.G = G; st.ld = ld; st.K = K; st.n_init = n_init; st.n_trials = n_trials; st.row_blocks = row_blocks;
  st.closest = static_cast<double*>(h->dev_buf("kmb.closest", nR * 8));
  st.newd = static_cast<double*>(h->dev_buf("kmb.newd", nR * n_trials * 8));
  st.part = static_cast<double*>(h->dev_buf("kmb.part", (size_t)n_init * n_trials * row_blocks * 8));
  st.cand = static_cast<int*>(h->dev_buf("kmb.cand", (size_t)n_init * 8 * 4));
  st.centre_idx = static_cast<int*>(h->dev_buf("kmb.cidx", (size_t)n_init * K * 4));
  st.pot = static_cast<double*>(h->dev_buf("kmb.pot", (size_t)n_init * 8));
  const size_t n_unif = (size_t)n_init * (K > 1 ? K - 1 : 1) * n_trials;
  double* d_unif = static_cast<double*>(h->dev_buf("kmb.unif", n_unif * 8));
  double* C64 = static_cast<double*>(h->dev_buf("kmb.C64", 2 * nKG * 8));
  // the ping-pong centres the E step reads: an fp32 copy for T = float, the fp64 centres themselves for T = double
  T* CE = std::is_same<T, double>::value ? reinterpret_cast<T*>(C64)
                                         : static_cast<T*>(h->dev_buf("kmb.C32", 2 * nKG * sizeof(T)));
  LloydState<T> ls{};
  ls.S = S_dev; ls.R = R; ls.G = G; ls.ld = ld; ls.K = K; ls.n_init = n_init;
  ls.labels = static_cast<int*>(h->dev_buf("kmb.labels", nR * 4));
  ls.mind = static_cast<T*>(h->dev_buf("kmb.mind", nR * sizeof(T)));
  ls.counts = static_cast<int*>(h->dev_buf("kmb.counts", (size_t)n_init * K * 4));
  ls.order = static_cast<int*>(h->dev_buf("kmb.order", nR * K * 4));
  ls.sums = static_cast<double*>(h->dev_buf("kmb.sums", nKG * 8));
  ls.shift_part = static_cast<double*>(h->dev_buf("kmb.shift", (size_t)n_init * K * 8));
  ls.flags = static_cast<int*>(h->dev_buf("kmb.flags", (size_t)n_init * 4 * 4));
  ls.inertia = static_cast<double*>(h->dev_buf("kmb.inertia", (size_t)n_init * 8));
  if (!st.closest || !st.newd || !st.part || !st.cand || !st.centre_idx || !st.pot || !d_unif || !C64 || !CE ||
      !ls.labels || !ls.mind || !ls.counts || !ls.order || !ls.sums || !ls.shift_part || !ls.flags || !ls.inertia)
    return -2;
  st.unif = d_unif;
  struct HostBlock { int32_t flags[32 * 4]; double inertia[32]; };
  HostBlock* hb = static_cast<HostBlock*>(h->host_buf("kmb.host", sizeof(HostBlock)));
  if (!hb) return -2;

  using clk = std::chrono::steady_clock;
  auto ms_since = [](clk::time_point t0) { return std::chrono::duration<double, std::milli>(clk::now() - t0).count(); };
  auto t_phase = clk::now();
  // ---- k-means++ seeding, all runs together
  {
    std::vector<int> cidx((size_t)n_init * K, 0);
    for (int t = 0; t < n_init; ++t) {
      CNMF_REQUIRE(first_idx_host[t] >= 0 && first_idx_host[t] < R, "kmeans_fit: first centre index out of range");
      cidx[(size_t)t * K] = first_idx_host[t];
    }
    CNMF_CUDA_CHECK(cudaMemcpyAsync(st.centre_idx, cidx.data(), cidx.size() * 4, cudaMemcpyHostToDevice, s));
    if (K > 1) CNMF_CUDA_CHECK(cudaMemcpyAsync(d_unif, uniforms_host, n_unif * 8, cudaMemcpyHostToDevice, s));
    CNMF_CUDA_CHECK(cudaStreamSynchronize(s));          // cidx goes out of scope
  }
  // The select kernel keeps `closest` in dynamic shared memory.  Without an opt-in a launch may use at most 48 KB minus
  // the kernel's static shared memory (cpot, s_best), so the limit is read from the function rather than assumed.
  const size_t sel_smem = (size_t)R * sizeof(double);
  cudaFuncAttributes sel_fa;
  CNMF_CUDA_CHECK(cudaFuncGetAttributes(&sel_fa, kpp_select_kernel<T>));
  if (sel_smem > (size_t)sel_fa.maxDynamicSharedSizeBytes)
    CNMF_CUDA_CHECK(cudaFuncSetAttribute(kpp_select_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  // each select launch is checked at once: a refused launch raises before the next centre's eval reads candidates it
  // never wrote
  const dim3 eval_grid(row_blocks, n_init);
  kpp_eval_kernel<T, 8><<<eval_grid, 256, 0, s>>>(st, 1);
  kpp_select_kernel<T><<<n_init, 256, sel_smem, s>>>(st, 0);
  CNMF_CUDA_CHECK(cudaGetLastError());
  for (int step = 1; step < K; ++step) {
    kpp_eval_kernel<T, 8><<<eval_grid, 256, 0, s>>>(st, 0);
    kpp_select_kernel<T><<<n_init, 256, sel_smem, s>>>(st, step);
    CNMF_CUDA_CHECK(cudaGetLastError());
  }
  kpp_gather_centres_kernel<T><<<dim3(K, n_init), 256, 0, s>>>(st, C64, CE);
  CNMF_CUDA_CHECK(cudaGetLastError());
  h->launches += 2 * K + 1;

  if (h->profile) {                 // phase timing for bench / probes (cnmf_last_timing: rng = seeding, solve = Lloyd)
    CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
    h->t_rng_ms = ms_since(t_phase);
    t_phase = clk::now();
  }
  // ---- Lloyd, all runs together
  CNMF_CUDA_CHECK(cudaMemsetAsync(ls.labels, 0xff, nR * 4, s));          // -1: every label "changes" in iteration 1
  CNMF_CUDA_CHECK(cudaMemsetAsync(ls.flags, 0, (size_t)n_init * 16, s));
  const dim3 assign_grid((R * 32 + 255) / 256, n_init);
  bool all_done = false, empty = false;
  int it = 0;
  while (!all_done && it < max_iter) {
    const int cur = it & 1, nxt = cur ^ 1;
    kmb_assign_kernel<T><<<assign_grid, 256, 0, s>>>(ls, CE, CE + nKG, cur, 0);
    kmb_members_kernel<T><<<n_init, 1024, 0, s>>>(ls);
    kmb_sums_kernel<T><<<dim3((G + 127) / 128, K, n_init), 128, 0, s>>>(ls);
    kmb_centre_update_kernel<T><<<dim3(K, n_init), 256, 0, s>>>(ls, C64 + (size_t)cur * nKG, C64 + (size_t)nxt * nKG,
                                                                CE + (size_t)nxt * nKG);
    kmb_check_kernel<T><<<1, 32, 0, s>>>(ls, tol_abs, max_iter);
    h->launches += 5;
    ++it;
    CNMF_CUDA_CHECK(cudaMemcpyAsync(hb->flags, ls.flags, (size_t)n_init * 16, cudaMemcpyDeviceToHost, s));
    CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
    all_done = true;
    for (int t = 0; t < n_init; ++t) {
      if (hb->flags[t * 4 + 1]) empty = true;
      if (!hb->flags[t * 4 + 2]) all_done = false;
    }
    if (empty) break;
  }
  CNMF_CUDA_CHECK(cudaGetLastError());
  if (empty) {                       // sklearn's relocation rule: host-assisted per-run path
    *needs_host_path = 1;
    return 0;
  }
  *needs_host_path = 0;
  if (h->profile) {
    h->t_solve_ms = ms_since(t_phase);
    h->t_h2d_ms = (double)it;      // Lloyd iterations of the slowest run
    t_phase = clk::now();
  }
  // ---- final E step against every run's final centres + inertia (sklearn _kmeans.py:736-744)
  kmb_assign_kernel<T><<<assign_grid, 256, 0, s>>>(ls, CE, CE + nKG, 0, 1);
  kmb_inertia_kernel<T><<<n_init, 256, 0, s>>>(ls);
  h->launches += 2;
  CNMF_CUDA_CHECK(cudaGetLastError());
  CNMF_CUDA_CHECK(cudaMemcpyAsync(hb->inertia, ls.inertia, (size_t)n_init * 8, cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaMemcpyAsync(labels_host, ls.labels, nR * 4, cudaMemcpyDeviceToHost, s));
  CNMF_CUDA_CHECK(cudaStreamSynchronize(s));
  if (h->profile) h->t_d2h_ms = ms_since(t_phase);
  for (int t = 0; t < n_init; ++t) {
    inertia_host[t] = hb->inertia[t];
    if (n_iter_host) n_iter_host[t] = hb->flags[t * 4 + 3];
  }
  return 0;
}

}  // namespace
}  // namespace cnmf

using namespace cnmf;

extern "C" int cnmf_kmeans_fit(cnmf_handle_t h, const float* S_dev, int R, int G, int ld, int K, int n_init, int max_iter,
                               double tol_abs, const int32_t* first_idx_host, const double* uniforms_host, int n_trials,
                               int32_t* labels_host, double* inertia_host, int32_t* n_iter_host,
                               int32_t* needs_host_path, void* stream) {
  return kmeans_fit(h, S_dev, R, G, ld, K, n_init, max_iter, tol_abs, first_idx_host, uniforms_host, n_trials,
                    labels_host, inertia_host, n_iter_host, needs_host_path, stream);
}

extern "C" int cnmf_kmeans_fit_f64(cnmf_handle_t h, const double* S_dev, int R, int G, int ld, int K, int n_init,
                                   int max_iter, double tol_abs, const int32_t* first_idx_host,
                                   const double* uniforms_host, int n_trials, int32_t* labels_host,
                                   double* inertia_host, int32_t* n_iter_host, int32_t* needs_host_path, void* stream) {
  return kmeans_fit(h, S_dev, R, G, ld, K, n_init, max_iter, tol_abs, first_idx_host, uniforms_host, n_trials,
                    labels_host, inertia_host, n_iter_host, needs_host_path, stream);
}
