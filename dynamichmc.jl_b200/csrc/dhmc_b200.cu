// dhmc_b200.cu — sm_90a kernels and the C ABI (include/dhmc.h) of the
// many-chain NUTS engine.  Build: see csrc/Makefile (nvcc -fmad=false, sm_90a).
//
// Kernels (one chain group of T threads = one CTA; persistent, chains pulled
// from an atomic queue so that ragged tree depths balance across SMs):
//   k_nuts      sample_tree / warmup(::TuningNUTS) / mcmc     NUTS.jl:232-241, mcmc.jl:258-286,366-381
//   k_search    warmup(::InitialStepsizeSearch)               mcmc.jl:134-148, stepsize.jl:46-85
//   k_leapfrog  leapfrog (streaming, HBM-bound)               hamiltonian.jl:273-282
//   k_eval      evaluate_ℓ(strict) / random_position          hamiltonian.jl:202-217, mcmc.jl:108
//   k_phase     logdensity(H, z)                              hamiltonian.jl:251-256
// Logistic family, dim <= 256: k_nuts / k_search run as "packed chain groups" — 8 chains per
// CTA, one warp and state machine each, the likelihood evaluated by the whole CTA on the FP64
// tensor cores (device_backend.cuh: coop_core_tma).
//
// There is NO CPU fallback: without a CUDA device dhmc_create fails with
// DHMC_ECUDA and nothing else can be called.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <nccl.h>      // types and prototypes only: the library is bound at run time (nccl_api below)

#include <pthread.h>
#include <sched.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <fstream>
#include <memory>
#include <cstdlib>
#include <cstring>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/dhmc.h"
#include "kernels.cuh"      // KArgs, shared-memory planning helpers; the kernels themselves are instantiated in family_tu.cu

using namespace dhmc;

// kernel lookup, one function per (family, part) translation unit (family_tu.cu).  The references are WEAK: the stock
// library links every shipped family, a user-model library (`make user`, include/dhmc_models.h) links the USER family's two
// units only, and a family whose units are absent is refused by dhmc_create ("family not built into this library").
// (hidden: never bound across two copies of the library loaded into one process)
#define DHMC_TU_LINKAGE __attribute__((weak, visibility("hidden")))
#define DHMC_DECL_TU(f, p) const void* dhmc_family_kernel_##f##_##p(int W, int epl, int kernel, int dense) DHMC_TU_LINKAGE;
DHMC_DECL_TU(0, 0) DHMC_DECL_TU(1, 0) DHMC_DECL_TU(2, 0) DHMC_DECL_TU(3, 0) DHMC_DECL_TU(3, 1)
DHMC_DECL_TU(0, 3) DHMC_DECL_TU(1, 3) DHMC_DECL_TU(2, 3) DHMC_DECL_TU(3, 3)
#undef DHMC_DECL_TU
extern "C" {
const void* dhmc_user_family_kernel_0(int W, int epl, int kernel, int dense) DHMC_TU_LINKAGE;
const void* dhmc_user_family_kernel_3(int W, int epl, int kernel, int dense) DHMC_TU_LINKAGE;
const char* dhmc_user_family_name_str(void) DHMC_TU_LINKAGE;
int dhmc_user_family_min_dim(void) DHMC_TU_LINKAGE;
// generated quantities (a model with DHMC_USER_GENERATED): G(D), whether they are random (DHMC_USER_GENERATED_RNG) and
// the launch of k_generated (family_tu.cu)
int dhmc_user_family_ngq(int D) DHMC_TU_LINKAGE;
int dhmc_user_family_random(void) DHMC_TU_LINKAGE;
int dhmc_user_family_generated(const double* theta, long long n, long long n_problems, int D, int ng, const double* mparams,
                               const void* problems, long long first, const long long* chain, const unsigned* transition,
                               unsigned long long seed, double* out, int T, int grid, cudaStream_t stream) DHMC_TU_LINKAGE;
}
// part: 0 = one chain per CTA, 1 = packed chain groups (likelihood on the tensor cores),
// 3 = one chain per CTA with max_depth > 12 (persistent kernels only)
typedef const void* (*family_tu_fn)(int, int, int, int);
static family_tu_fn family_tu(int fam, int part) {
  switch (fam * 4 + part) {
    case 0: return dhmc_family_kernel_0_0;
    case 4: return dhmc_family_kernel_1_0;
    case 8: return dhmc_family_kernel_2_0;
    case 12: return dhmc_family_kernel_3_0;
    case 13: return dhmc_family_kernel_3_1;
    case 3: return dhmc_family_kernel_0_3;
    case 7: return dhmc_family_kernel_1_3;
    case 11: return dhmc_family_kernel_2_3;
    case 15: return dhmc_family_kernel_3_3;
    case 16: return dhmc_user_family_kernel_0;
    case 19: return dhmc_user_family_kernel_3;
  }
  return nullptr;
}
static const void* lookup_kernel(int fam, int part, int W, int epl, KernelId k, bool dense) {
  const family_tu_fn f = family_tu(fam, part);
  return f ? f(W, epl, k, dense) : nullptr;
}

// ------------------------------------------------------------------ Symmetric metric
// Lower Cholesky factor of the row-major symmetric A, stored transposed:
// Lt[k*D + i] = L[i][k].  One CTA; per output element the subtraction order is
// k = 0..j-1, as in the oracle (cholesky_lower).  Returns false if not positive definite.
__device__ bool chol_lower_t(const double* A, double* Lt, int D) {
  const int tid = threadIdx.x, nt = blockDim.x;
  for (int j = 0; j < D; ++j) {
    double s = A[(size_t)j * D + j];
    for (int k = 0; k < j; ++k) { const double l = Lt[(size_t)k * D + j]; s = s - l * l; }
    if (!(s > 0.0) || !dm_isfinite(s)) return false;      // uniform across the CTA
    const double d = dm_sqrt(s);
    __syncthreads();
    if (tid == 0) Lt[(size_t)j * D + j] = d;
    for (int i = j + 1 + tid; i < D; i += nt) {
      double t = A[(size_t)i * D + j];
      for (int k = 0; k < j; ++k) t = t - Lt[(size_t)k * D + i] * Lt[(size_t)k * D + j];
      Lt[(size_t)j * D + i] = t / d;
    }
    __syncthreads();
  }
  return true;
}
// W = cholesky(inv(M⁻¹)).L — hamiltonian.jl:73, restated as in oracle dense_factor():
// C = chol(M⁻¹), Ci = C⁻¹, M = CiᵀCi, W = chol(M); W is stored transposed in wt.
__global__ void k_dense_factor(const double* minv_dense, double* wt, double* tmp, int* status, int D, int B) {
  const int tid = threadIdx.x, nt = blockDim.x;
  const size_t dd = (size_t)D * D;
  double* Ct = tmp + (size_t)blockIdx.x * 3 * dd;
  double* Ci = Ct + dd;
  double* M = Ci + dd;
  for (int c = blockIdx.x; c < B; c += gridDim.x) {
    const double* A = minv_dense + (size_t)c * dd;
    bool ok = chol_lower_t(A, Ct, D);
    if (ok) {
      for (int j = tid; j < D; j += nt) {                 // Ci = C⁻¹, one column per thread
        Ci[(size_t)j * D + j] = 1.0 / Ct[(size_t)j * D + j];
        for (int i = j + 1; i < D; ++i) {
          double sacc = 0.0;
          for (int k = j; k < i; ++k) sacc = sacc - Ct[(size_t)k * D + i] * Ci[(size_t)k * D + j];
          Ci[(size_t)i * D + j] = sacc / Ct[(size_t)i * D + i];
        }
      }
      __syncthreads();
      for (int i = tid; i < D; i += nt)                   // M = Ciᵀ Ci
        for (int j = 0; j <= i; ++j) {
          double sacc = 0.0;
          for (int k = i; k < D; ++k) sacc = sacc + Ci[(size_t)k * D + i] * Ci[(size_t)k * D + j];
          M[(size_t)i * D + j] = sacc; M[(size_t)j * D + i] = sacc;
        }
      __syncthreads();
      ok = chol_lower_t(M, wt + (size_t)c * dd, D);
    }
    if (!ok && tid == 0) atomicOr(status + c, (int)DHMC_CHAIN_NOT_POSDEF);
    __syncthreads();
  }
}
// M⁻¹ = regularize_M⁻¹(Symmetric(cov(X; dims = 2)), λ) — mcmc.jl:211, :218-221, from the
// streamed co-moments (transposed lower) of a window of n draws.
__global__ void k_cov_finish(const double* covt, double* minv_dense, int n, double lambda, int D, int B) {
  const size_t dd = (size_t)D * D;
  const double dn1 = (double)(n - 1);
  for (int c = blockIdx.x; c < B; c += gridDim.x) {
    const double* ct = covt + (size_t)c * dd;
    double* out = minv_dense + (size_t)c * dd;
    for (int i = threadIdx.x; i < D; i += blockDim.x)
      for (int j = 0; j <= i; ++j) {
        const double sij = ct[(size_t)j * D + i] / dn1;
        double v = (1 - lambda) * sij;
        if (i == j) v = v + lambda * sij;
        out[(size_t)i * D + j] = v; out[(size_t)j * D + i] = v;
      }
  }
}
// Pooled metric of every group of 8 chains (DHMC_METRIC_SYMMETRIC_POOLED): the chains' streaming window means and co-moments
// (n draws each) merged in the oracle's fixed order (pooled_regularized_cov), shrunk as regularize_M⁻¹, written to all 8 chains.
__global__ void k_cov_pool(const double* covt, const double* means, double* minv_dense, int n, double lambda, int D, int B) {
  extern __shared__ double gm[];              // group mean [D]
  const size_t dd = (size_t)D * D;
  const double dn = (double)n;
  constexpr int G = 8;
  for (int g = blockIdx.x; g < B / G; g += gridDim.x) {
    const size_t c0 = (size_t)g * G;
    for (int i = threadIdx.x; i < D; i += blockDim.x) {
      double m = means[c0 * D + i];
      for (int c = 1; c < G; ++c) m = m + means[(c0 + c) * D + i];
      gm[i] = m / (double)G;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < D; i += blockDim.x)
      for (int j = 0; j <= i; ++j) {
        double acc = 0.0;
        for (int c = 0; c < G; ++c) {
          const double di = means[(c0 + c) * D + i] - gm[i], dj = means[(c0 + c) * D + j] - gm[j];
          acc = acc + (covt[(c0 + c) * dd + (size_t)j * D + i] + (dn * di) * dj);
        }
        const double sij = acc / ((double)G * dn - 1.0);
        double v = (1 - lambda) * sij;
        if (i == j) v = v + lambda * sij;
        for (int c = 0; c < G; ++c) {
          double* out = minv_dense + (c0 + c) * dd;
          out[(size_t)i * D + j] = v; out[(size_t)j * D + i] = v;
        }
      }
    __syncthreads();
  }
}
// Xp[c][n][j] = X[c][n][j] for n < N, j < D, zero elsewhere: B matrices [N][D] into [B][rows][xs]
// (the rows of X, B = 1; every chain's M⁻¹, N = D)
__global__ void k_pad_rows(const double* X, double* Xp, size_t N, size_t D, size_t rows, size_t xs, size_t B) {
  const size_t per = rows * xs, tot = per * B;
  for (size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x; t < tot; t += (size_t)gridDim.x * blockDim.x) {
    const size_t c = t / per, r = t % per, n = r / xs, j = r % xs;
    Xp[t] = (n < N && j < D) ? X[c * N * D + n * D + j] : 0.0;
  }
}
// Xt[j][n] = X[n][j], rows of Xt padded to ld >= N (pad = 0)
__global__ void k_transpose(const double* X, double* Xt, size_t N, size_t D, size_t ld) {
  const size_t tot = ld * D;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < tot; i += (size_t)gridDim.x * blockDim.x) {
    const size_t j = i / ld, n = i % ld;
    Xt[i] = n < N ? X[n * D + j] : 0.0;
  }
}
// Device-side reduction of tree statistics (Diagnostics.summarize_tree_statistics /
// EBFMI, diagnostics.jl:29-32, 65-106): one warp per chain over its N records.
__global__ void k_tree_summary(const dhmc_tree_stats* stats, int N, int B, unsigned long long* depth_counts /*[33]*/,
                               unsigned long long* term_counts /*[3]: max_depth, divergence, turning*/,
                               double* acc_sum, unsigned long long* step_sum, double* ebfmi /*[B] or null*/) {
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int c = warp; c < B; c += nwarps) {
    const dhmc_tree_stats* s = stats + (size_t)c * N;
    const double pi0 = s[0].pi;   // the mean is taken as π₀ + mean(π − π₀): a chain of constant π gets var = 0 exactly
    double a = 0.0, sp = 0.0, sd2 = 0.0;
    unsigned long long st = 0;
    for (int n = lane; n < N; n += 32) {
      const dhmc_tree_stats r = s[n];
      a += r.acceptance_rate; st += (unsigned long long)r.steps; sp += r.pi - pi0;
      if (n + 1 < N) { const double d = s[n + 1].pi - r.pi; sd2 += d * d; }
      atomicAdd(depth_counts + (r.depth < 32 ? r.depth : 32), 1ull);
      const int k = (r.left == 1 && r.right == 0) ? 0 : (r.left == r.right ? 1 : 2);
      atomicAdd(term_counts + k, 1ull);
    }
    for (int o = 16; o; o >>= 1) {
      a += __shfl_xor_sync(0xffffffffu, a, o); sp += __shfl_xor_sync(0xffffffffu, sp, o);
      sd2 += __shfl_xor_sync(0xffffffffu, sd2, o); st += __shfl_xor_sync(0xffffffffu, st, o);
    }
    const double mean = pi0 + sp / N;
    double ss = 0.0;
    for (int n = lane; n < N; n += 32) { const double d = s[n].pi - mean; ss += d * d; }
    for (int o = 16; o; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    if (lane == 0) {
      atomicAdd(acc_sum, a); atomicAdd(step_sum, st);
      if (ebfmi) ebfmi[c] = (N > 1) ? (sd2 / (N - 1)) / (ss / (N - 1)) : dm_nan();
    }
  }
}

// ---- cross-chain convergence diagnostics on device-resident draws [B][N][D] (§8f-2; the reference's tests use
// MCMCDiagnosticTools.ess_rhat on the same quantities, sample-correctness_utilities.jl:40-43).  Every chain is split in
// two halves of n = N/2 draws (m = 2B sequences).  One warp = 32 consecutive parameters of one sequence: mean, then the
// biased autocovariances at lags 0…L; the per-parameter sums over the sequences of a chain group are accumulated with atomics:
//   acc[g][d][0] = Σ (μ − pilot_gd), [1] = Σ (μ − pilot_gd)², [2 + t] = Σ acov(t)   (pilot_gd = mean of the group's first
//   sequence: a shift that keeps the variance of the means free of cancellation).  The host finishes R̂ and the Geyer sum.
// Chain groups: local chain c belongs to group (off + c) / K — the problems of a batch; K = 0: one group of all chains.
__device__ __forceinline__ int ess_group(long c, long long K, long long off) { return K ? (int)((off + c) / K) : 0; }
// mean of one sequence (stride D) as x₀ + mean(x − x₀): a constant sequence gets its value exactly, so its centred draws,
// W and (for equal constants) the variance of the means are exact zeros
__device__ __forceinline__ double seq_mean(const double* x, int n, int D) {
  const double x0 = x[0];
  double s = 0.0;
  for (int i = 0; i < n; ++i) s += x[(size_t)i * D] - x0;
  return x0 + s / n;
}
__global__ void k_pilot_mean(const double* draws, int n, int N, int D, int B, long long K, long long off, int P, double* pilot) {
  const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long)P * D) return;
  const int g = (int)(t / D), d = (int)(t % D);
  const long long first = (long long)g * K - off;
  const long c0 = (K && first > 0) ? (long)first : 0;                            // the group's first local chain
  if (c0 >= B || ess_group(c0, K, off) != g) return;                            // no local chain: the host reports NaN
  pilot[t] = seq_mean(draws + (size_t)c0 * N * D + d, n, D);
}
__global__ void k_ess_rhat(const double* draws, int N, int n, int D, int B, long long K, long long off, int L, const double* pilot,
                           double* acc) {
  const int lane = threadIdx.x & 31;
  const long warp = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((long)gridDim.x * blockDim.x) >> 5;
  const int tiles = (D + 31) / 32;
  const long work = (long)2 * B * tiles;                    // (sequence, parameter tile)
  for (long w = warp; w < work; w += nwarps) {
    const long seq = w / tiles;
    const int d = (int)(w % tiles) * 32 + lane;
    if (d >= D) continue;
    const double* x = draws + ((size_t)(seq >> 1) * N + (size_t)(seq & 1) * n) * D + d;
    const double mu = seq_mean(x, n, D);
    const size_t gd = (size_t)ess_group(seq >> 1, K, off) * D + d;
    double* a = acc + gd * (L + 3);
    const double dm = mu - pilot[gd];
    atomicAdd(a, dm);
    atomicAdd(a + 1, dm * dm);
    for (int t = 0; t <= L; ++t) {
      double c = 0.0;
      for (int i = 0; i + t < n; ++i) c += (x[(size_t)i * D] - mu) * (x[(size_t)(i + t) * D] - mu);
      atomicAdd(a + 2 + t, c / n);
    }
  }
}
// histogram of the acceptance rates (4096 bins on [0, 1]) of a device statistics buffer
__global__ void k_acceptance_hist(const dhmc_tree_stats* stats, size_t n, unsigned long long* hist, int bins) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    double a = stats[i].acceptance_rate;
    int b = a >= 1.0 ? bins - 1 : a <= 0.0 ? 0 : (int)(a * bins);
    if (!(a == a)) b = bins;                                  // NaN bucket
    atomicAdd(hist + b, 1ull);
  }
}

// broadcast a D-vector (or scalar when D == 1) to all chains
__global__ void k_broadcast(double* dst, const double* src, size_t D, size_t B) {
  const size_t n = D * B;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    dst[i] = src[i % D];
}
__global__ void k_fill(double* dst, double v, size_t n) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    dst[i] = v;
}

// ================================================================== host side
#if defined(DHMC_ALLOC_FAULTS)
// Fault-injection build (make faults, tests/test_device_allocations.py): the k-th next device allocation fails with
// cudaErrorMemoryAllocation without reaching CUDA (k = 0: none fails), and the live allocations are counted.
static int64_t g_fail_alloc_in = 0, g_live_allocations = 0;
extern "C" void dhmc_test_fail_alloc(int64_t k) { g_fail_alloc_in = k; }
extern "C" int64_t dhmc_test_live_allocations(void) { return g_live_allocations; }
#endif

// n elements of T in device memory, freed by the destructor; every device allocation of the host code is one of these.
// alloc(n) frees the current array before it allocates, grow(n) allocates only for an n above the current size, and a
// failed allocation leaves the array empty.
template <class T>
class DeviceArray {
 public:
  DeviceArray() = default;
  DeviceArray(DeviceArray&& o) noexcept : p_(o.p_), n_(o.n_) { o.p_ = nullptr; o.n_ = 0; }
  DeviceArray& operator=(DeviceArray&& o) noexcept {
    if (this != &o) { reset(); std::swap(p_, o.p_); std::swap(n_, o.n_); }
    return *this;
  }
  ~DeviceArray() { reset(); }
  cudaError_t alloc(size_t n) {
    reset();
#if defined(DHMC_ALLOC_FAULTS)
    if (g_fail_alloc_in > 0 && --g_fail_alloc_in == 0) return cudaErrorMemoryAllocation;
#endif
    const cudaError_t e = cudaMalloc(&p_, sizeof(T) * n);
    if (e != cudaSuccess) { p_ = nullptr; return e; }
    n_ = n;
#if defined(DHMC_ALLOC_FAULTS)
    if (p_) ++g_live_allocations;
#endif
    return cudaSuccess;
  }
  cudaError_t grow(size_t n) { return n > n_ ? alloc(n) : cudaSuccess; }
  void reset() {
#if defined(DHMC_ALLOC_FAULTS)
    if (p_) --g_live_allocations;
#endif
    cudaFree(p_); p_ = nullptr; n_ = 0;
  }
  T* get() const { return p_; }
  size_t size() const { return n_; }

 private:
  T* p_ = nullptr;
  size_t n_ = 0;
};

// The handle owns its device arrays, events, streams, page-locked caller buffers and communicator.
struct dhmc_handle {
  dhmc_config cfg;
  int T = 0, W = 0, EPL = 0;
  int G = 1;                        // chains per CTA of the persistent kernels (packed chain groups)
  bool deep = false;                // max_depth > 12: kernels whose slot pool spills past 64 slots (part 3), one chain per CTA
  size_t stride = 0;
  int n_slots = 0, n_sm = 0, grid = 0, sm_count = 0, light_grid = 0;
  int levels = 13, ntab = 64;       // stack entries per warp (max_depth + 1), slot-table entries (>= n_slots)
  size_t smem_bytes = 0;
  size_t scratch_per_cta = 0;
  bool planned = false;             // n_sm, smem_bytes, grid and scratch_per_cta match scratch and lr (plan)
  cudaStream_t stream = nullptr, copy_stream = nullptr, h2d_stream = nullptr;
  cudaEvent_t h2d_ev[16] = {};
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  cudaEvent_t chunk_ev[16] = {};
  cudaEvent_t copy_ev[16] = {};
  bool trace = false;
  DeviceArray<double> tmp_b;        // [B] scratch (phase log densities) and [B·D] momentum override / [D·D] broadcast source,
  DeviceArray<double> tmp_bd;       // allocated once instead of per call
  DeviceArray<unsigned> tmp_dir;
  std::vector<void*> registered;    // caller buffers page-locked on the fly (direct host writes of draws that exceed HBM)
  DeviceArray<char> stage[4];       // grow-only device staging for host outputs
  DeviceArray<double> q, g, lq, p, minv, eps;
  DeviceArray<double> mparams;
  DeviceArray<int> status;
  DeviceArray<double> scratch;
#if defined(DHMC_PHASE_CLOCKS)
  DeviceArray<unsigned long long> phase_clocks;   // leaf profile: kPhCount counters for each of up to 32 CTAs per SM
#endif
  DeviceArray<unsigned> counter;
  DeviceArray<unsigned long long> total_steps;
  uint32_t t = 0;
  int64_t launches = 0;
  double last_ms = 0;
  int64_t last_steps = 0;
  bool has_position = false, has_eps = false;
  bool dense = false;               // κ is a Symmetric (dense) metric
  DeviceArray<double> minv_dense, wt, covt, dense_tmp;
  DeviceArray<double> mean_pool;    // pooled Symmetric stages: window mean of every chain [B][D]
  bool pooled = false;              // the dense metric is shared by every group of 8 chains
  DeviceArray<double> minv_pad;     // packed groups on the tensor cores: zero-padded row blocks of every chain's M⁻¹
  DeviceArray<double> lX, lXt, ly, lr;   // logistic regression
  DeviceArray<double> lXp;          // … zero-padded row blocks of X for the tensor-core likelihood
  int lN = 0, lLd = 0;              // (a batch: lN is the largest N, the row length of the residual scratch lr)
  // problem batch (dhmc_set_problems / _ragged): chains per problem (0 = one problem), problems, and the device table of
  // per-problem descriptors (where each problem's blocks start in mparams, lX, lXt, ly, lXp; its N and leading dimension)
  int64_t batch_k = 0, batch_p = 0;
  DeviceArray<ProblemDesc> problems;
  int reg_ctas[2] = {0, 0};         // occupancy of k_nuts (diag, dense)
  size_t smem_sm = 0, smem_cta_max = 0;
  ncclComm_t comm = nullptr;        // multi-GPU: one communicator per handle (dhmc_comm_init)
  int comm_nranks = 1, comm_rank = 0;
  double last_comm_ms = 0;
  // streaming summary (dhmc_mcmc_summary): grow-only device arena of the SummaryArgs arrays, and the struct itself
  DeviceArray<char> sum_buf;
  DeviceArray<SummaryArgs> sum_args;
  int ngq = 0;                      // generated quantities of a user model (dhmc_generated_count)
  bool gq_random = false;           // ... drawn from the keyed streams (dhmc_generated_random)
  std::string err;

  ~dhmc_handle() {                  // (the device arrays are freed after this body)
    for (void* r : registered) cudaHostUnregister(r);
    if (comm) dhmc_comm_destroy(this);
    for (cudaEvent_t e : {ev0, ev1}) if (e) cudaEventDestroy(e);
    for (cudaEvent_t* evs : {h2d_ev, chunk_ev, copy_ev})
      for (int i = 0; i < 16; ++i) if (evs[i]) cudaEventDestroy(evs[i]);
    for (cudaStream_t s : {copy_stream, h2d_stream, stream}) if (s) cudaStreamDestroy(s);
  }
};

static std::string g_create_err;

#define CK(call)                                                                      \
  do {                                                                                \
    cudaError_t e_ = (call);                                                          \
    if (e_ != cudaSuccess) {                                                          \
      h->err = std::string(#call) + ": " + cudaGetErrorString(e_);                    \
      return e_ == cudaErrorMemoryAllocation ? DHMC_ENOMEM : DHMC_ECUDA;              \
    }                                                                                 \
  } while (0)

// a per-chain staging vector in shared memory: mat-vec input (Symmetric metric), β (logistic), the whole position (USER)
static bool needs_staging(const dhmc_handle* h) {
  return h->minv_dense.get() || h->cfg.family == DHMC_FAMILY_LOGISTIC || h->cfg.family == DHMC_FAMILY_USER;
}
// The instantiation of kernel k for the handle's family, layout and metric kind.  Part 3: the deep persistent kernels;
// part 1: the persistent kernels of packed chain groups (the light kernels run one chain per CTA); part 0: the rest.
static const void* handle_kernel(dhmc_handle* h, KernelId k) {
  const bool heavy = (k == K_NUTS || k == K_SEARCH);
  const int part = heavy && h->deep ? 3 : heavy && h->G > 1 ? 1 : 0;
  const void* fn = lookup_kernel(h->cfg.family, part, h->W, h->EPL, k, h->dense);
  if (!fn) h->err = "kernel not built into this library for this layout (max_depth > 12 needs a user-model library built with its deep part: USER_PARTS=\"0 3\" / deep=True)";
  return fn;
}

// whole blocks of 32 rows: the unit of the bulk copies into the tensor-core rounds (coop_core_tma, coop_matvec_tma)
static size_t tma_rows(size_t n) { return (n + kTmaRows - 1) / kTmaRows * kTmaRows; }

// grid of the dense-metric kernels (factor, window estimate): 4 CTAs per SM, no more than one per chain
static int factor_grid(const dhmc_handle* h) { return (int)std::min<size_t>((size_t)h->sm_count * 4, (size_t)h->cfg.n_chains); }

// rows of N doubles in the logistic scratch (residuals): one per CTA of the light kernels and, with one chain per CTA,
// of the persistent kernels of a plan of `grid` CTAs (packed groups keep theirs in shared memory)
static size_t lr_rows(const dhmc_handle* h, int grid) {
  return std::max<size_t>(h->G > 1 ? 0 : (size_t)grid, (size_t)h->light_grid);
}

// groups of the persistent kernels' reduction buffer (DeviceBackend::kFused): the last leaf of a depth-d adjacent tree carries
// d stack merges and the doubling check, the first two in group 0, so max_depth groups (two at max_depth 1)
static int red_groups(const dhmc_handle* h) {
  return !h->dense && h->G == 1 && h->cfg.family != DHMC_FAMILY_USER ? std::max(2, h->cfg.max_depth) : 1;
}

// Plan the persistent kernels for the current metric kind: CTAs per SM (register
// limited), how many slots fit in shared memory, and the global scratch arena.  The scratch of the current plan is freed
// before the new one is allocated; if that allocation fails, the handle has no plan until the next successful one.
static int plan(dhmc_handle* h) {
  const int T = h->T;
  const size_t B = (size_t)h->cfg.n_chains;
  const size_t slot_doubles = h->stride * (h->dense ? 2 : 1);
  const size_t slot_bytes = sizeof(double) * slot_doubles;
  const size_t xs = needs_staging(h) ? h->stride : 0;
  const int G = h->G;
  auto heavy_smem = [&](int n_sm) -> size_t {
    return G > 1 ? (size_t)G * group_smem_bytes(h->W, n_sm, slot_doubles, xs, h->levels, h->ntab) + tma_smem_bytes(G, (int)h->cfg.dim)
                 : smem_layout(h->W, n_sm, slot_doubles, xs, h->levels, h->ntab, red_groups(h)).total;
  };
  struct { size_t total; } L0{heavy_smem(0)};
  int& reg_ctas = h->reg_ctas[h->dense ? 1 : 0];
  if (reg_ctas == 0) {
    const void* fn = handle_kernel(h, K_NUTS);
    if (!fn) return DHMC_EARG;
    cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)L0.total);
    if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&reg_ctas, fn, T * G, L0.total);
    if (e != cudaSuccess) { h->err = std::string("occupancy query: ") + cudaGetErrorString(e); return DHMC_ECUDA; }
  }
  if (reg_ctas < 1) { h->err = "kernel does not fit on an SM"; return DHMC_ECUDA; }
  const int ctas = h->cfg.ctas_per_sm > 0 ? std::min(h->cfg.ctas_per_sm, reg_ctas) : reg_ctas;
  size_t per_cta = h->smem_sm / ctas - 1024;   // 1 KB system reservation per CTA
  if (per_cta > h->smem_cta_max) per_cta = h->smem_cta_max;
  long n_sm = per_cta > L0.total ? (long)((per_cta - L0.total) / (slot_bytes * (size_t)G)) : 0;
  const int pool = h->n_slots - kWelfordSlots;   // the two highest slots stay in global memory
  if (n_sm > pool) n_sm = pool;
  const int grid = (int)std::min<size_t>((size_t)ctas * h->sm_count, (B + G - 1) / G);
  const size_t scratch_per_cta = (size_t)(h->n_slots - n_sm) * slot_doubles;
  h->planned = false;
  CK(h->scratch.alloc(scratch_per_cta * (size_t)grid * (size_t)G));
  // (an access-policy window over the slot arena was tried and rejected: slower at C2)
  if (h->lN) CK(h->lr.alloc((size_t)h->lN * lr_rows(h, grid)));   // residual scratch of the logistic family follows the grid
  h->n_sm = (int)n_sm;
  h->smem_bytes = heavy_smem(h->n_sm);
  h->grid = grid;
  h->scratch_per_cta = scratch_per_cta;
  h->planned = true;
  return DHMC_OK;
}

static KArgs base_args(dhmc_handle* h) {
  KArgs a;
  std::memset(&a, 0, sizeof(a));
  a.D = (int)h->cfg.dim; a.B = (int)h->cfg.n_chains; a.T = h->T; a.W = h->W;
  a.seed = h->cfg.seed; a.chain_offset = h->cfg.chain_offset;
  a.q = h->q.get(); a.g = h->g.get(); a.lq = h->lq.get(); a.p = h->p.get(); a.minv = h->minv.get(); a.eps = h->eps.get();
  a.mparams = h->mparams.get(); a.status = h->status.get();
  a.max_depth = h->cfg.max_depth; a.min_delta = h->cfg.min_delta;
  a.t0 = h->t;
  a.scratch = h->scratch.get(); a.scratch_per_cta = h->scratch_per_cta;
#if defined(DHMC_PHASE_CLOCKS)
  a.phase_clocks = h->phase_clocks.get();
#endif
  a.n_sm = h->n_sm; a.n_slots = h->n_slots; a.stride = h->stride * (h->dense ? 2 : 1);
  a.levels = h->levels; a.ntab = h->ntab;
  a.red_groups = red_groups(h);
  a.counter = h->counter.get(); a.total_steps = h->total_steps.get();
  a.chain_begin = 0; a.chain_end = (int)h->cfg.n_chains;
  a.minv_dense = h->minv_dense.get(); a.wt = h->wt.get(); a.covt = nullptr; a.minv_pad = h->minv_pad.get(); a.mean_out = nullptr; a.pooled = h->pooled;
  a.xs_doubles = needs_staging(h) ? (int)((size_t)h->T * h->EPL) : 0;
  a.lX = h->lX.get(); a.lXt = h->lXt.get(); a.ly = h->ly.get(); a.lr = h->lr.get(); a.lN = h->lN; a.lLd = h->lLd; a.lXp = h->lXp.get();
  a.batch_k = (int)h->batch_k; a.problems = h->problems.get();
  return a;
}

// dhmc_last_kernel_ms: the time from ev0 to ev1 (synchronises)
static int read_timer(dhmc_handle* h) {
  CK(cudaEventSynchronize(h->ev1));
  float ms = 0;
  CK(cudaEventElapsedTime(&ms, h->ev0, h->ev1));
  h->last_ms = ms;
  return DHMC_OK;
}
// heavy = persistent kernels that use the slot pool (k_nuts, k_search).  before / after (null: none) are recorded right
// before and right after the kernel, so that they time it alone.  reset_steps: zero the Σ steps counter first.
static int launch(dhmc_handle* h, KernelId k, KArgs a, cudaEvent_t before, cudaEvent_t after, bool reset_steps = true) {
  const bool heavy = (k == K_NUTS || k == K_SEARCH);
  if (!h->planned) { h->err = "the handle has no kernel plan: its re-plan failed to allocate the slot scratch; set the metric "
                             "again (dhmc_set_metric, dhmc_set_metric_dense) to re-plan"; return DHMC_ENOMEM; }
  if (!heavy) { a.n_sm = 0; a.red_groups = 1; }
  const size_t smem = heavy ? h->smem_bytes : smem_layout(h->W, 0, a.stride, (size_t)a.xs_doubles).total;
  int grid = heavy ? h->grid : h->light_grid;
  const int G = heavy ? h->G : 1;
  if (heavy) grid = std::max(1, std::min(grid, (a.chain_end - a.chain_begin + G - 1) / G));
  if (heavy) {
    CK(cudaMemsetAsync(h->counter.get(), 0, sizeof(unsigned), h->stream));
    if (reset_steps) CK(cudaMemsetAsync(h->total_steps.get(), 0, sizeof(unsigned long long), h->stream));
  }
  if (before) CK(cudaEventRecord(before, h->stream));
  {
    const void* fn = handle_kernel(h, k);
    if (!fn) return DHMC_EARG;
    cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { h->err = std::string("cudaFuncSetAttribute: ") + cudaGetErrorString(e); return DHMC_ECUDA; }
    void* params[] = {(void*)&a};
    e = cudaLaunchKernel(fn, dim3(grid), dim3(h->T * G), params, smem, h->stream);
    if (e != cudaSuccess) { h->err = std::string("cudaLaunchKernel: ") + cudaGetErrorString(e); return DHMC_ECUDA; }
  }
  h->launches += 1;
  if (after) CK(cudaEventRecord(after, h->stream));
  return DHMC_OK;
}

static int sync_and_check_status(dhmc_handle* h, int mask, const char* what) {
  CK(cudaStreamSynchronize(h->stream));
  const size_t B = (size_t)h->cfg.n_chains;
  std::vector<int> st(B);
  CK(cudaMemcpy(st.data(), h->status.get(), sizeof(int) * B, cudaMemcpyDeviceToHost));
  long bad = 0, first = -1, halted = 0, first_halted = -1;
  for (size_t i = 0; i < B; ++i) {
    if (st[i] & mask) { if (first < 0) first = (long)i; ++bad; }
    // a chain whose first failure is leapfrog's @argcheck (a strict evaluation or a non-finite position fails earlier)
    if ((st[i] & mask & DHMC_CHAIN_LEAPFROG_NONFINITE) && !(st[i] & (DHMC_CHAIN_BAD_INITIAL | DHMC_CHAIN_NONFINITE_Q))) {
      if (first_halted < 0) first_halted = (long)i;
      ++halted;
    }
  }
  if (halted) {      // the ArgumentError of hamiltonian.jl:276 is named first: the shims raise it for these chains
    char buf[320];
    std::snprintf(buf, sizeof buf,
                  "Internal error: leapfrog called from non-finite log density: %ld chain(s) (first: local chain %ld, "
                  "status 0x%x); %ld chain(s) failed in all (%s)", halted, first_halted, st[first_halted], bad, what);
    h->err = buf;
    return DHMC_ENUMERIC;
  }
  if (bad) {
    char buf[256];
    std::snprintf(buf, sizeof buf, "%s: %ld chain(s) failed (first: local chain %ld, status 0x%x)",
                  what, bad, first, st[first]);
    h->err = buf;
    return DHMC_ENUMERIC;
  }
  return DHMC_OK;
}

static void choose_layout(int64_t D, int req_T, int* T, int* EPL) {
  if (req_T > 0) {
    *T = req_T;
    const int W = req_T / 32;
    int e = (int)((D + req_T - 1) / req_T);
    e = e <= 1 ? 1 : e <= 2 ? 2 : e <= 4 ? 4 : e <= 8 ? 8 : e <= 16 ? 16 : e <= 32 ? 32 : 0;
    if (e && !layout_supported(W, e)) e = (e < 4 && layout_supported(W, 4)) ? 4 : (e < 8 && layout_supported(W, 8)) ? 8 : 0;
    *EPL = e;
    return;
  }
  if (D <= 32) { *T = 32; *EPL = 1; }
  else if (D <= 64) { *T = 32; *EPL = 2; }
  else if (D <= 128) { *T = 32; *EPL = 4; }
  else if (D <= 256) { *T = 64; *EPL = 4; }
  else if (D <= 512) { *T = 128; *EPL = 4; }
  else if (D <= 1024) { *T = 128; *EPL = 8; }
  else if (D <= 2048) { *T = 256; *EPL = 8; }
  else if (D <= 4096) { *T = 256; *EPL = 16; }
  else if (D <= 8192) { *T = 256; *EPL = 32; }    // the vectors no longer fit the register file: correct, not fast
  else { *T = 0; *EPL = 0; }
}

extern "C" {

const char* dhmc_last_error(dhmc_handle* h) { return h ? h->err.c_str() : g_create_err.c_str(); }

int dhmc_destroy(dhmc_handle* h) {
  if (!h) return DHMC_OK;
  cudaSetDevice(h->cfg.device);
  delete h;
  return DHMC_OK;
}

// dhmc_create after its argument checks: the device resources of the new handle and its first plan
static int init_handle(dhmc_handle* h, const dhmc_config* cfg) {
  CK(cudaSetDevice(cfg->device));
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, cfg->device));
  h->sm_count = prop.multiProcessorCount;
#if defined(DHMC_PHASE_CLOCKS)
  CK(h->phase_clocks.alloc((size_t)kPhCount * 32 * (size_t)h->sm_count));
  CK(cudaMemset(h->phase_clocks.get(), 0, sizeof(unsigned long long) * kPhCount * 32 * (size_t)h->sm_count));
#endif
  CK(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
  CK(cudaStreamCreateWithFlags(&h->copy_stream, cudaStreamNonBlocking));
  CK(cudaStreamCreateWithFlags(&h->h2d_stream, cudaStreamNonBlocking));
  const bool trace = std::getenv("DHMC_TRACE") != nullptr;      // DHMC_TRACE=1: timeline of the chunk pipeline on stderr
  for (cudaEvent_t* evs : {h->h2d_ev, h->chunk_ev, h->copy_ev})
    for (int i = 0; i < 16; ++i) CK(cudaEventCreateWithFlags(&evs[i], trace ? cudaEventDefault : cudaEventDisableTiming));
  h->trace = trace;
  CK(cudaEventCreate(&h->ev0));
  CK(cudaEventCreate(&h->ev1));
  const size_t B = (size_t)cfg->n_chains, D = (size_t)cfg->dim;
  CK(h->q.alloc(B * D));
  CK(h->g.alloc(B * D));
  CK(h->p.alloc(B * D));
  CK(h->minv.alloc(B * D));
  CK(h->lq.alloc(B));
  CK(h->eps.alloc(B));
  CK(h->status.alloc(B));
  CK(h->counter.alloc(1));
  CK(h->total_steps.alloc(1));
  CK(h->mparams.alloc(2 * D));
  CK(cudaMemsetAsync(h->q.get(), 0, sizeof(double) * B * D, h->stream));
  CK(cudaMemsetAsync(h->g.get(), 0, sizeof(double) * B * D, h->stream));
  CK(cudaMemsetAsync(h->p.get(), 0, sizeof(double) * B * D, h->stream));
  CK(cudaMemsetAsync(h->lq.get(), 0, sizeof(double) * B, h->stream));
  CK(cudaMemsetAsync(h->eps.get(), 0, sizeof(double) * B, h->stream));
  CK(cudaMemsetAsync(h->status.get(), 0, sizeof(int) * B, h->stream));
  CK(cudaMemsetAsync(h->mparams.get(), 0, sizeof(double) * 2 * D, h->stream));
  k_fill<<<1024, 256, 0, h->stream>>>(h->minv.get(), 1.0, B * D);   // κ = GaussianKineticEnergy(D), mcmc.jl:130
  h->launches += 1;

  h->smem_sm = (size_t)prop.sharedMemPerMultiprocessor;          // 228 KB
  h->smem_cta_max = (size_t)prop.sharedMemPerBlockOptin;         // 227 KB
  h->light_grid = (int)std::min<size_t>((size_t)h->sm_count * 16, B);
  if (int rc = plan(h)) return rc;
  CK(cudaStreamSynchronize(h->stream));
  return DHMC_OK;
}

int dhmc_create(const dhmc_config* cfg, dhmc_handle** out) {
  if (!cfg || !out) { g_create_err = "null argument"; return DHMC_EARG; }
  *out = nullptr;
  // @argcheck sites: NUTS.jl:190-191
  if (!(cfg->max_depth > 0 && cfg->max_depth <= kMaxLevels)) { g_create_err = "0 < max_depth <= MAX_DIRECTIONS_DEPTH (32)"; return DHMC_EARG; }   // NUTS.jl:190, trees.jl:10
  if (!(cfg->min_delta < 0)) { g_create_err = "min_delta < 0"; return DHMC_EARG; }
  if (cfg->dim < 1 || cfg->n_chains < 1 || cfg->n_chains > (1ll << 30)) { g_create_err = "dim >= 1, 1 <= n_chains <= 2^30"; return DHMC_EARG; }
  if (cfg->family < 0 || cfg->family >= DHMC_FAMILY_COUNT) { g_create_err = "unknown family"; return DHMC_EARG; }
  if (cfg->family == DHMC_FAMILY_FUNNEL && cfg->dim < 2) { g_create_err = "funnel needs dim >= 2"; return DHMC_EARG; }
  if (cfg->family == DHMC_FAMILY_USER && !family_tu(DHMC_FAMILY_USER, 0)) {
    g_create_err = "this library was built without a user model (make user USER_HEADER=…; api.compile_user_model)";
    return DHMC_EARG;
  }
  if (!family_tu(cfg->family, 0)) { g_create_err = "family not built into this library (a user-model library carries the USER family only)"; return DHMC_EARG; }
  if (cfg->family == DHMC_FAMILY_USER && dhmc_user_family_min_dim && cfg->dim < dhmc_user_family_min_dim()) {
    g_create_err = "dim below the user model's DHMC_USER_MIN_DIM";
    return DHMC_EARG;
  }
  int T = 0, EPL = 0;
  const int rt = cfg->threads_per_chain;
  if (rt != 0 && !(rt == 32 || rt == 64 || rt == 128 || rt == 256)) { g_create_err = "threads_per_chain in {0,32,64,128,256}"; return DHMC_EARG; }
  choose_layout(cfg->dim, rt, &T, &EPL);
  // logistic regression, dim <= 256: kPack chains per CTA, one warp each (8 elements per lane above dim 128: eight
  // warps at 255 registers — the tensor-core rounds need only two warps per sub-partition, and the state machine does
  // not spill), sharing every pass over X (packed chain groups); an explicit threads_per_chain keeps one chain per CTA
  int pack = 1;
  const bool deep = cfg->max_depth > 12;
  if (cfg->family == DHMC_FAMILY_LOGISTIC && rt == 0 && cfg->dim <= 32 * kPack && !deep) {
    if (cfg->dim > 128) { T = 32; EPL = 8; }
    pack = kPack;
  }
  if (T == 0 || EPL == 0) { g_create_err = "dim too large for this build (dim <= 32 * threads_per_chain, 32 only for 256 threads: dim <= 8192)"; return DHMC_EARG; }
  const int ngq = cfg->family == DHMC_FAMILY_USER && dhmc_user_family_ngq ? dhmc_user_family_ngq((int)cfg->dim) : 0;
  if (cfg->family == DHMC_FAMILY_USER && dhmc_user_family_ngq && !(ngq >= 1 && ngq <= DHMC_MAX_GENERATED)) {
    g_create_err = "the user model's dhmc_user_ngq(dim) is outside [1, 8192]";
    return DHMC_EARG;
  }
  int ndev = 0;
  cudaError_t ce = cudaGetDeviceCount(&ndev);
  if (ce != cudaSuccess || ndev == 0) {
    g_create_err = std::string("no CUDA device: ") + (ce != cudaSuccess ? cudaGetErrorString(ce) : "device count 0") +
                   " (libdhmc_b200 has no CPU fallback)";
    return DHMC_ECUDA;
  }
  if (cfg->device < 0 || cfg->device >= ndev) { g_create_err = "bad device ordinal"; return DHMC_EARG; }
  std::unique_ptr<dhmc_handle> h(new dhmc_handle());
  h->cfg = *cfg; h->T = T; h->W = T / 32; h->EPL = EPL; h->stride = (size_t)T * EPL; h->G = pack; h->deep = deep;
  h->ngq = ngq;
  h->gq_random = ngq > 0 && dhmc_user_family_random && dhmc_user_family_random() != 0;
  h->n_slots = slots_needed(cfg->max_depth);
  h->levels = deep ? cfg->max_depth + 1 : kStdLevels;        // deep persistent kernels size their stack / slot table at run time
  h->ntab = deep ? std::max(kStdTab, (h->n_slots + 7) & ~7) : kStdTab;
  if (int rc = init_handle(h.get(), cfg)) { g_create_err = h->err; return rc; }
  *out = h.release();
  return DHMC_OK;
}

int dhmc_get_layout(dhmc_handle* h, int32_t* T, int32_t* epl) {
  if (!h) return DHMC_EARG;
  if (T) *T = h->T;
  if (epl) *epl = h->EPL;
  return DHMC_OK;
}

int dhmc_family_available(int32_t family, int32_t* available) {
  if (!available) return DHMC_EARG;
  *available = (family >= 0 && family < DHMC_FAMILY_COUNT && family_tu(family, 0)) ? 1 : 0;
  return DHMC_OK;
}

int dhmc_user_family_name(char* name, size_t cap) {
  if (!dhmc_user_family_name_str || !name || cap == 0) return DHMC_EARG;
  std::strncpy(name, dhmc_user_family_name_str(), cap - 1);
  name[cap - 1] = 0;
  return DHMC_OK;
}

// Checks one parameter block of the handle's family, blk[0 .. len); `who` names the entry point in the messages.
static int check_block(dhmc_handle* h, const char* who, const double* blk, size_t len) {
  const size_t D = (size_t)h->cfg.dim;
  auto fail = [&](const char* m) { h->err = std::string(who) + ": " + m; return DHMC_EARG; };
  switch (h->cfg.family) {
    case DHMC_FAMILY_USER:                 // any number of doubles, interpreted by the user's formulas
      return len && !blk ? fail("null parameter block") : DHMC_OK;
    case DHMC_FAMILY_DIAG_NORMAL:
      return len != 2 * D || !blk ? fail("DIAG_NORMAL blocks are [mu(D), prec(D)]") : DHMC_OK;
    case DHMC_FAMILY_LOGISTIC: {
      if (!blk || len < 1) return fail("logistic blocks are [N, X (N*D), y (N)]");
      const double v = blk[0];
      if (!(v >= 1.0 && v < 2147483648.0 && v == std::floor(v))) return fail("a logistic block starts with its N, an integer with 1 <= N < 2^31");
      const size_t N = (size_t)v;
      if (len != 1 + N * D + N) return fail("logistic blocks are [N, X (N*D), y (N)]: a block's length disagrees with its N");
      for (size_t i = 0; i < N; ++i) {     // the model is a Bernoulli likelihood: responses (or their means) in [0, 1]
        const double yv = blk[1 + N * D + i];
        if (!(yv >= 0.0 && yv <= 1.0)) return fail("logistic regression needs 0 <= y <= 1");
      }
      return DHMC_OK;
    }
    default:                               // STD_NORMAL, FUNNEL
      return len ? fail("this family has no parameters (n == 0)") : DHMC_OK;
  }
}

// The checks every problem batch shares (dhmc_set_problems, dhmc_set_problems_ragged); `who` names the entry point in the
// messages.
static int check_batch(dhmc_handle* h, const char* who, bool have_blocks, int64_t P, int64_t K) {
  const int fam = h->cfg.family;
  const int64_t off = h->cfg.chain_offset, B = h->cfg.n_chains;
  auto fail = [&](const char* m) { h->err = std::string(who) + ": " + m; return DHMC_EARG; };
  if (fam != DHMC_FAMILY_DIAG_NORMAL && fam != DHMC_FAMILY_LOGISTIC && fam != DHMC_FAMILY_USER)
    return fail("this family has no parameters (a batch of it would be one problem)");
  if (P < 1 || K < 1 || !have_blocks) return fail("n_problems >= 1, chains_per_problem >= 1 and a parameter block per problem");
  if (P > INT32_MAX / K) return fail("n_problems * chains_per_problem < 2^31");
  if (off < 0 || off + B > P * K)
    return fail("the handle's chains [chain_offset, chain_offset + n_chains) lie beyond n_problems * chains_per_problem");
  if (h->G > 1 && (K % 8 != 0 || off % 8 != 0 || B % 8 != 0))
    return fail("packed chain groups (logistic, automatic layout, dim <= 256) run 8 chains of one problem per CTA: "
                "chains_per_problem, chain_offset and n_chains must be multiples of 8 (threads_per_chain=32 runs one chain per CTA without this condition)");
  return DHMC_OK;
}

// Installs P validated blocks (problem p: params[offs[p] .. offs[p+1])), each sampled by K chains; K = 0: one problem
// (P = 1) for every chain, and no descriptor table.  Every problem gets arrays of its own size, back to back, and a
// descriptor that says where they start.  The new arrays are complete before they replace the current ones: on any error
// the previous problem (batch or not) stays in effect.
static int install_problems(dhmc_handle* h, const double* params, const std::vector<size_t>& offs, int64_t P, int64_t K) {
  const int fam = h->cfg.family;
  const size_t D = (size_t)h->cfg.dim, Pz = (size_t)P;
  const size_t xs = fam == DHMC_FAMILY_LOGISTIC ? (size_t)tma_xs((int)D) : 0;
  std::vector<ProblemDesc> desc(Pz);
  size_t tX = 0, tXt = 0, ty = 0, tXp = 0, maxN = 0;
  for (size_t p = 0; p < Pz; ++p) {
    ProblemDesc& d = desc[p];
    d = ProblemDesc{};
    if (fam != DHMC_FAMILY_LOGISTIC) { d.mparams = offs[p]; continue; }
    const size_t N = (size_t)params[offs[p]];
    const size_t ld = (N + 1) & ~(size_t)1;                     // even leading dimension: 16-byte aligned row segments
    d.X = tX; d.Xt = tXt; d.y = ty; d.Xp = h->G > 1 ? tXp : 0; d.N = (int)N; d.ld = (int)ld;
    tX += N * D; tXt += ld * D; ty += N; tXp += tma_rows(N) * xs;
    maxN = std::max(maxN, N);
    if (d.Xt % 2 != 0 || (h->G > 1 && d.Xp % (kTmaRows * xs) != 0)) {
      h->err = "problem batch: misaligned problem base in X^T or padded X (internal error)"; return DHMC_ECUDA;
    }
  }
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaStreamSynchronize(h->stream));
  DeviceArray<double> mp, X, Xt, y, Xp, lr;
  DeviceArray<ProblemDesc> dd;
  const int rc = [&]() -> int {
    if (K) {
      CK(dd.alloc(Pz));
      CK(cudaMemcpyAsync(dd.get(), desc.data(), sizeof(ProblemDesc) * Pz, cudaMemcpyHostToDevice, h->stream));
    }
    if (fam == DHMC_FAMILY_LOGISTIC) {
      // per problem: X [N][D], Xᵀ [D][ld], y [N] and, for packed groups, the zero-padded row blocks [rows][xs]; one residual
      // scratch of rows of the largest N
      CK(X.alloc(tX));
      CK(Xt.alloc(tXt));
      CK(y.alloc(ty));
      CK(lr.alloc(maxN * lr_rows(h, h->grid)));
      if (h->G > 1) CK(Xp.alloc(tXp));
      for (size_t p = 0; p < Pz; ++p) {
        const double* blk = params + offs[p];
        const ProblemDesc& d = desc[p];
        const size_t N = (size_t)d.N;
        CK(cudaMemcpyAsync(X.get() + d.X, blk + 1, sizeof(double) * N * D, cudaMemcpyHostToDevice, h->stream));
        CK(cudaMemcpyAsync(y.get() + d.y, blk + 1 + N * D, sizeof(double) * N, cudaMemcpyHostToDevice, h->stream));
        k_transpose<<<1024, 256, 0, h->stream>>>(X.get() + d.X, Xt.get() + d.Xt, N, D, (size_t)d.ld);
        if (Xp.get()) k_pad_rows<<<1024, 256, 0, h->stream>>>(X.get() + d.X, Xp.get() + d.Xp, N, D, tma_rows(N), xs, 1);
        h->launches += Xp.get() ? 2 : 1;
      }
    } else if (fam == DHMC_FAMILY_DIAG_NORMAL || fam == DHMC_FAMILY_USER) {   // (STD_NORMAL and FUNNEL have no parameters)
      // mparams is never null, also for a USER model without parameters
      CK(mp.alloc(std::max<size_t>(offs[Pz], 1)));
      if (offs[Pz]) CK(cudaMemcpyAsync(mp.get(), params, sizeof(double) * offs[Pz], cudaMemcpyHostToDevice, h->stream));
    }
    CK(cudaGetLastError());
    return DHMC_OK;
  }();
  // the new arrays are freed on an error only after the copies and kernels queued on them
  if (rc != DHMC_OK) { cudaStreamSynchronize(h->stream); return rc; }
  CK(cudaStreamSynchronize(h->stream));
  if (fam == DHMC_FAMILY_LOGISTIC) {
    h->lX = std::move(X); h->lXt = std::move(Xt); h->ly = std::move(y); h->lr = std::move(lr); h->lXp = std::move(Xp);
    h->lN = (int)maxN; h->lLd = desc[0].ld;    // a chain's own N and ld come from its descriptor
  } else if (mp.get()) {
    h->mparams = std::move(mp);
  }
  h->problems = std::move(dd);
  h->batch_k = K; h->batch_p = K ? P : 0;
  return DHMC_OK;
}

int dhmc_set_problem(dhmc_handle* h, const double* params, size_t n) {
  if (!h) return DHMC_EARG;
  if (int rc = check_block(h, "dhmc_set_problem", params, n)) return rc;
  return install_problems(h, params, {0, n}, 1, 0);
}

// P problems of the handle's family and dimension, each with its own parameter block of n doubles; global chain g samples
// problem g / chains_per_problem.  Everything is validated before anything is allocated.
int dhmc_set_problems(dhmc_handle* h, const double* params, size_t n, int64_t P, int64_t K) {
  if (!h) return DHMC_EARG;
  if (int rc = check_batch(h, "dhmc_set_problems", params && n >= 1, P, K)) return rc;
  if (h->cfg.family == DHMC_FAMILY_LOGISTIC)
    for (int64_t p = 1; p < P; ++p)
      if (params[(size_t)p * n] != params[0]) { h->err = "dhmc_set_problems: every logistic problem of a batch needs the same N"; return DHMC_EARG; }
  std::vector<size_t> offs((size_t)P + 1);
  for (size_t p = 0; p <= (size_t)P; ++p) offs[p] = p * n;
  for (int64_t p = 0; p < P; ++p)
    if (int rc = check_block(h, "dhmc_set_problems", params + offs[p], n)) return rc;
  return install_problems(h, params, offs, P, K);
}

// The same with blocks of different lengths: problem p's block is params[block_offsets[p] .. block_offsets[p+1]).
int dhmc_set_problems_ragged(dhmc_handle* h, const double* params, const size_t* offs, int64_t P, int64_t K) {
  if (!h) return DHMC_EARG;
  const char* who = "dhmc_set_problems_ragged";
  if (int rc = check_batch(h, who, params && offs, P, K)) return rc;
  auto fail = [&](const char* m) { h->err = std::string(who) + ": " + m; return DHMC_EARG; };
  if (offs[0] != 0) return fail("block_offsets[0] must be 0");
  for (int64_t p = 0; p < P; ++p)
    if (offs[p + 1] <= offs[p]) return fail("block_offsets must strictly increase (every block holds at least one value)");
  for (int64_t p = 0; p < P; ++p)
    if (int rc = check_block(h, who, params + offs[p], offs[p + 1] - offs[p])) return rc;
  return install_problems(h, params, std::vector<size_t>(offs, offs + P + 1), P, K);
}

static int eval_position(dhmc_handle* h, bool randomize) {
  CK(cudaMemsetAsync(h->status.get(), 0, sizeof(int) * (size_t)h->cfg.n_chains, h->stream));
  KArgs a = base_args(h);
  a.strict = 1; a.randomize = randomize ? 1 : 0;
  int rc = launch(h, K_EVAL, a, nullptr, nullptr);
  if (rc != DHMC_OK) return rc;
  h->has_position = true;
  return sync_and_check_status(h, DHMC_CHAIN_BAD_INITIAL, "initialize_warmup_state: invalid log density or gradient at the initial position");
}

int dhmc_set_position(dhmc_handle* h, const double* q) {
  if (!h || !q) return DHMC_EARG;
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaMemcpyAsync(h->q.get(), q, sizeof(double) * (size_t)h->cfg.n_chains * h->cfg.dim, cudaMemcpyHostToDevice, h->stream));
  return eval_position(h, false);
}
int dhmc_random_position(dhmc_handle* h) {
  if (!h) return DHMC_EARG;
  CK(cudaSetDevice(h->cfg.device));
  return eval_position(h, true);
}

// The arrays of the Symmetric metric, allocated together at the first use.  A handle without a plan re-plans here too.
static int ensure_dense(dhmc_handle* h) {
  if (h->minv_dense.get()) return h->planned ? DHMC_OK : plan(h);
  const size_t B = (size_t)h->cfg.n_chains, dd = (size_t)h->cfg.dim * h->cfg.dim;
  DeviceArray<double> minv_dense, wt, covt, dense_tmp, minv_pad;
  CK(minv_dense.alloc(B * dd));
  CK(wt.alloc(B * dd));
  CK(covt.alloc(B * dd));
  CK(dense_tmp.alloc(3 * dd * (size_t)factor_grid(h)));
  if (h->G > 1)     // [B][⌈D/32⌉·32][XS]: one bulk copy per 32-row block (coop_matvec_tma)
    CK(minv_pad.alloc(B * tma_rows((size_t)h->cfg.dim) * (size_t)tma_xs((int)h->cfg.dim)));
  h->minv_dense = std::move(minv_dense); h->wt = std::move(wt); h->covt = std::move(covt);
  h->dense_tmp = std::move(dense_tmp); h->minv_pad = std::move(minv_pad);
  CK(cudaMemsetAsync(h->wt.get(), 0, sizeof(double) * B * dd, h->stream));
  // re-planned whatever the metric kind: with the dense arrays allocated, the shared-memory layout carries the staging
  // vector (needs_staging) also for the diagonal kernels
  return plan(h);
}
// The metric kind of the handle's kernels: the persistent kernels are re-planned when the slot width (dense) changes, or
// when the handle has no plan.  The kind changes only with a successful plan.
static int set_metric_kind(dhmc_handle* h, bool dense, bool pooled) {
  if (h->planned && h->dense == dense) { h->pooled = pooled; return DHMC_OK; }
  const bool was_dense = h->dense;
  h->dense = dense;
  if (int rc = plan(h)) { h->dense = was_dense; return rc; }
  h->pooled = pooled;
  return DHMC_OK;
}
// κ = GaussianKineticEnergy(Symmetric M⁻¹): W = cholesky(inv(M⁻¹)).L on device, then switch
// the handle to the dense kernels (pooled: M⁻¹ is shared by every group of 8 chains).
static int factor_and_switch(dhmc_handle* h, bool pooled) {
  const size_t B = (size_t)h->cfg.n_chains, D = (size_t)h->cfg.dim;
  CK(cudaMemsetAsync(h->status.get(), 0, sizeof(int) * B, h->stream));
  k_dense_factor<<<factor_grid(h), 128, 0, h->stream>>>(h->minv_dense.get(), h->wt.get(), h->dense_tmp.get(), h->status.get(), (int)D, (int)B);
  h->launches += 1;
  if (h->minv_pad.get()) {
    k_pad_rows<<<2048, 256, 0, h->stream>>>(h->minv_dense.get(), h->minv_pad.get(), D, D, tma_rows(D), (size_t)tma_xs((int)D), B);
    h->launches += 1;
  }
  CK(cudaGetLastError());
  if (int rc = set_metric_kind(h, true, pooled)) return rc;
  return sync_and_check_status(h, DHMC_CHAIN_NOT_POSDEF, "GaussianKineticEnergy: M⁻¹ is not positive definite (PosDefException)");
}

int dhmc_set_metric_dense(dhmc_handle* h, const double* minv, int broadcast) {
  if (!h || !minv) return DHMC_EARG;
  CK(cudaSetDevice(h->cfg.device));
  int rc = ensure_dense(h);
  if (rc != DHMC_OK) return rc;
  const size_t B = (size_t)h->cfg.n_chains, dd = (size_t)h->cfg.dim * h->cfg.dim;
  if (broadcast) {
    CK(h->tmp_bd.grow(dd));
    CK(cudaMemcpyAsync(h->tmp_bd.get(), minv, sizeof(double) * dd, cudaMemcpyHostToDevice, h->stream));
    k_broadcast<<<1024, 256, 0, h->stream>>>(h->minv_dense.get(), h->tmp_bd.get(), dd, B);
    h->launches += 1;
    CK(cudaStreamSynchronize(h->stream));
  } else {
    CK(cudaMemcpyAsync(h->minv_dense.get(), minv, sizeof(double) * B * dd, cudaMemcpyHostToDevice, h->stream));
  }
  return factor_and_switch(h, false);
}
int dhmc_get_metric_dense(dhmc_handle* h, double* minv) {
  if (!h || !minv) return DHMC_EARG;
  if (!h->dense) { h->err = "the current metric is diagonal"; return DHMC_EARG; }
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaMemcpy(minv, h->minv_dense.get(), sizeof(double) * (size_t)h->cfg.n_chains * h->cfg.dim * h->cfg.dim, cudaMemcpyDeviceToHost));
  return DHMC_OK;
}
int dhmc_metric_is_dense(dhmc_handle* h, int32_t* dense) { if (!h || !dense) return DHMC_EARG; *dense = h->dense ? 1 : 0; return DHMC_OK; }

int dhmc_set_metric(dhmc_handle* h, const double* minv, int broadcast) {
  if (!h) return DHMC_EARG;
  CK(cudaSetDevice(h->cfg.device));
  const size_t B = (size_t)h->cfg.n_chains, D = (size_t)h->cfg.dim;
  if (!minv) {
    k_fill<<<1024, 256, 0, h->stream>>>(h->minv.get(), 1.0, B * D);
  } else if (broadcast) {
    CK(h->tmp_bd.grow(D));
    CK(cudaMemcpyAsync(h->tmp_bd.get(), minv, sizeof(double) * D, cudaMemcpyHostToDevice, h->stream));
    k_broadcast<<<1024, 256, 0, h->stream>>>(h->minv.get(), h->tmp_bd.get(), D, B);
    CK(cudaStreamSynchronize(h->stream));
  } else {
    CK(cudaMemcpyAsync(h->minv.get(), minv, sizeof(double) * B * D, cudaMemcpyHostToDevice, h->stream));
  }
  h->launches += 1;
  CK(cudaStreamSynchronize(h->stream));
  return set_metric_kind(h, false, false);
}

int dhmc_set_stepsize(dhmc_handle* h, const double* eps, int broadcast) {
  if (!h || !eps) return DHMC_EARG;
  CK(cudaSetDevice(h->cfg.device));
  const size_t B = (size_t)h->cfg.n_chains;
  if (broadcast) {
    if (!(eps[0] > 0)) { h->err = "ϵ > 0"; return DHMC_EARG; }    // stepsize.jl:135
    k_fill<<<256, 256, 0, h->stream>>>(h->eps.get(), eps[0], B);
    h->launches += 1;
  } else {
    for (size_t i = 0; i < B; ++i) if (!(eps[i] > 0)) { h->err = "ϵ > 0"; return DHMC_EARG; }
    CK(cudaMemcpyAsync(h->eps.get(), eps, sizeof(double) * B, cudaMemcpyHostToDevice, h->stream));
  }
  CK(cudaStreamSynchronize(h->stream));
  h->has_eps = true;
  return DHMC_OK;
}

int dhmc_set_momentum(dhmc_handle* h, const double* p) {
  if (!h || !p) return DHMC_EARG;
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaMemcpyAsync(h->p.get(), p, sizeof(double) * (size_t)h->cfg.n_chains * h->cfg.dim, cudaMemcpyHostToDevice, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return DHMC_OK;
}

int dhmc_get_state(dhmc_handle* h, double* q, double* lq, double* grad, double* minv, double* eps, double* p) {
  if (!h) return DHMC_EARG;
  CK(cudaSetDevice(h->cfg.device));
  const size_t B = (size_t)h->cfg.n_chains, D = (size_t)h->cfg.dim;
  if (q) CK(cudaMemcpyAsync(q, h->q.get(), sizeof(double) * B * D, cudaMemcpyDeviceToHost, h->stream));
  if (grad) CK(cudaMemcpyAsync(grad, h->g.get(), sizeof(double) * B * D, cudaMemcpyDeviceToHost, h->stream));
  if (minv) CK(cudaMemcpyAsync(minv, h->minv.get(), sizeof(double) * B * D, cudaMemcpyDeviceToHost, h->stream));
  if (p) CK(cudaMemcpyAsync(p, h->p.get(), sizeof(double) * B * D, cudaMemcpyDeviceToHost, h->stream));
  if (lq) CK(cudaMemcpyAsync(lq, h->lq.get(), sizeof(double) * B, cudaMemcpyDeviceToHost, h->stream));
  if (eps) CK(cudaMemcpyAsync(eps, h->eps.get(), sizeof(double) * B, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return DHMC_OK;
}

int dhmc_chain_status(dhmc_handle* h, int32_t* status) {
  if (!h || !status) return DHMC_EARG;
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaMemcpy(status, h->status.get(), sizeof(int) * (size_t)h->cfg.n_chains, cudaMemcpyDeviceToHost));
  return DHMC_OK;
}
int dhmc_get_transition_count(dhmc_handle* h, uint32_t* t) { if (!h || !t) return DHMC_EARG; *t = h->t; return DHMC_OK; }
int dhmc_set_transition_count(dhmc_handle* h, uint32_t t) { if (!h) return DHMC_EARG; h->t = t; return DHMC_OK; }

int dhmc_leapfrog(dhmc_handle* h, int32_t n_steps, int32_t sign) {
  if (!h || n_steps < 0) return DHMC_EARG;
  if (!h->has_position || !h->has_eps) { h->err = "dhmc_leapfrog: set position and step size first"; return DHMC_EARG; }
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaMemsetAsync(h->status.get(), 0, sizeof(int) * (size_t)h->cfg.n_chains, h->stream));   // status words describe the current call
  KArgs a = base_args(h);
  a.lf_steps = n_steps; a.lf_sign = sign;
  int rc = launch(h, K_LEAPFROG, a, h->ev0, h->ev1);
  if (rc == DHMC_OK) rc = read_timer(h);
  if (rc != DHMC_OK) return rc;
  return sync_and_check_status(h, DHMC_CHAIN_NONFINITE_Q | DHMC_CHAIN_LEAPFROG_NONFINITE,
                               "leapfrog: position vector has non-finite elements");
}

int dhmc_phase_logdensity(dhmc_handle* h, double* out) {
  if (!h || !out) return DHMC_EARG;
  CK(cudaSetDevice(h->cfg.device));
  const size_t B = (size_t)h->cfg.n_chains;
  CK(h->tmp_b.grow(B));
  KArgs a = base_args(h);
  a.out_phase = h->tmp_b.get();
  const int rc = launch(h, K_PHASE, a, nullptr, nullptr);
  if (rc != DHMC_OK) return rc;
  CK(cudaMemcpyAsync(out, h->tmp_b.get(), sizeof(double) * B, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return DHMC_OK;
}

int dhmc_find_initial_stepsize(dhmc_handle* h, double initial_eps, double log_threshold, int32_t maxiter) {
  if (!h) return DHMC_EARG;
  // InitialStepsizeSearch @argchecks — stepsize.jl:31-33
  if (!(std::isfinite(log_threshold) && log_threshold < 0)) { h->err = "isfinite(log_threshold) && log_threshold < 0"; return DHMC_EARG; }
  if (!(std::isfinite(initial_eps) && 0 < initial_eps)) { h->err = "isfinite(initial_ϵ) && 0 < initial_ϵ"; return DHMC_EARG; }
  if (!(maxiter >= 50)) { h->err = "maxiter_crossing ≥ 50"; return DHMC_EARG; }
  if (!h->has_position) { h->err = "set the position first"; return DHMC_EARG; }
  if (h->has_eps) { h->err = "stepsize ϵ manually specified, won't perform initial search"; return DHMC_EARG; }  // mcmc.jl:137
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaMemsetAsync(h->status.get(), 0, sizeof(int) * (size_t)h->cfg.n_chains, h->stream));   // status words describe the current call
  KArgs a = base_args(h);
  a.s_init = initial_eps; a.s_thresh = log_threshold; a.s_maxiter = maxiter;
  int rc = launch(h, K_SEARCH, a, h->ev0, h->ev1);
  if (rc == DHMC_OK) rc = read_timer(h);
  if (rc != DHMC_OK) return rc;
  // the reference aborts when the search fails (stepsize.jl:58,78): ϵ counts as set only if every chain found one
  rc = sync_and_check_status(h, DHMC_CHAIN_SEARCH_FAILED | DHMC_CHAIN_NONFINITE_Q,
                             "initial stepsize search failed (no crossing, or non-finite starting density)");
  h->has_eps = (rc == DHMC_OK);
  return rc;
}

// Is `p` page-locked host memory that the device can address (cudaHostAlloc / cudaHostRegister)?  Then *dev is its device alias.
static bool host_mapped(const void* p, void** dev) {
  const char* evn = std::getenv("DHMC_NO_DIRECT");        // A/B switch: always stage
  if (evn && std::atoi(evn) == 1) return false;
  cudaPointerAttributes at;
  if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return false; }
  if (at.type != cudaMemoryTypeHost || !at.devicePointer) return false;
  *dev = at.devicePointer;
  return true;
}

// One call of run_nuts: N transitions per chain, every thin-th one kept.  A caller sets the fields it uses.
struct NutsRequest {
  int N = 0, thin = 1;
  AdaptConfig cfg{};                            // warm-up: step-size adaptation and the metric to estimate
  double lambda = 0.0;                          // warm-up: regularisation λ of an estimated Symmetric metric
  bool pool_metric = false;                     // warm-up: pool that estimate over groups of 8 chains
  const double* q_host = nullptr;               // host positions [B][D] to start from (NULL: the handle's)
  const double* p_over_host = nullptr; const uint32_t* dir_over_host = nullptr;   // dhmc_sample_tree: momenta, directions
  // outputs in the order of h->stage: draws, tree statistics, step sizes, log densities (NULL: not kept)
  double* posterior = nullptr; dhmc_tree_stats* stats = nullptr; double* eps_used = nullptr; double* logdens = nullptr;
  bool outputs_on_device = false;               // the outputs are device arrays
  const SummaryArgs* summary = nullptr;         // device SummaryArgs: fold the kept draws into the streaming summary
};

// Common driver of sample_tree / warmup stage / mcmc / mcmc_summary; the transition count advances by N.  Host outputs of
// large runs are pipelined: the chains are cut into chunks, each chunk is one k_nuts launch on the compute stream, and its
// draws/statistics are copied D2H on the copy stream while the next chunk computes (pinned host buffers make the copies
// truly asynchronous; pageable ones still work).
static int run_nuts(dhmc_handle* h, const NutsRequest& r) {
  if ((!h->has_position && !r.q_host) || !h->has_eps) { h->err = "set position and step size (or run the initial search) first"; return DHMC_EARG; }
  const auto tr0 = std::chrono::steady_clock::now();
  auto tr_ms = [&] { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - tr0).count(); };
  double tr_pt[6] = {0, 0, 0, 0, 0, 0};
  CK(cudaSetDevice(h->cfg.device));
  if (r.thin < 1 || r.N % r.thin != 0) { h->err = "thin >= 1 and N a multiple of thin"; return DHMC_EARG; }
  const size_t B = (size_t)h->cfg.n_chains, D = (size_t)h->cfg.dim, n = (size_t)(r.N / r.thin);   // n: kept draws per chain
  double* d_p = nullptr;
  unsigned* d_dir = nullptr;
  int rc = DHMC_OK;
  // Host outputs.  Page-locked (pinned) buffers are written by the kernel itself through their device alias — no staging
  // copy in HBM, no second hop, the PCIe writes overlap the sampling at cache-line granularity and N is not bounded by
  // device memory.  Pageable buffers are staged in HBM (out[i] in stage[i]) and copied chunk by chunk; if the draws would
  // not fit, the buffer is page-locked on the fly (cudaHostRegister) and written directly.
  struct Output { void* host; size_t row; void* dev; bool direct; };       // row: bytes per kept draw of a chain
  Output out[4] = {{r.posterior, sizeof(double) * D, nullptr, false}, {r.stats, sizeof(dhmc_tree_stats), nullptr, false},
                   {r.eps_used, sizeof(double), nullptr, false}, {r.logdens, sizeof(double), nullptr, false}};
  for (int i = 0; i < 4; ++i) {
    Output& o = out[i];
    if (!o.host) continue;
    if (r.outputs_on_device) { o.dev = o.host; continue; }
    const size_t bytes = o.row * B * n;
    if (i == 0) {
      // Draws: staging + DMA copies overlapped chunk by chunk is the faster route when the draws fit in HBM (C2: 21.9 ms per
      // step against 24.1 ms with direct writes — kernel stores reach ~47 GB/s over PCIe, the copy engines 57 GB/s); the
      // kernel writes the host buffer directly when they do not fit (DHMC_DIRECT=1 forces it).
      size_t fr = 0, tot = 0;
      cudaMemGetInfo(&fr, &tot);
      const bool fits = bytes <= h->stage[0].size() || bytes + ((size_t)1 << 30) <= fr;
      const char* evd = std::getenv("DHMC_DIRECT");
      const bool force_direct = evd && std::atoi(evd) == 1;
      if (!fits || force_direct) {
        o.direct = host_mapped(o.host, &o.dev);
        if (!o.direct && !fits) {                                                   // pageable and too large: page-lock the caller's buffer
          if (cudaHostRegister(o.host, bytes, cudaHostRegisterMapped) == cudaSuccess) {
            h->registered.push_back(o.host);
            o.direct = host_mapped(o.host, &o.dev);
          } else {
            cudaGetLastError();
          }
        }
      }
    } else {
      o.direct = host_mapped(o.host, &o.dev);
    }
    if (!o.direct) {
      CK(h->stage[i].grow(bytes));
      o.dev = h->stage[i].get();
    }
  }
  if (r.p_over_host) {
    CK(h->tmp_bd.grow(B * D));
    d_p = h->tmp_bd.get();
    CK(cudaMemcpyAsync(d_p, r.p_over_host, sizeof(double) * B * D, cudaMemcpyHostToDevice, h->stream));
  }
  if (r.dir_over_host) {
    CK(h->tmp_dir.grow(B));
    d_dir = h->tmp_dir.get();
    CK(cudaMemcpyAsync(d_dir, r.dir_over_host, sizeof(unsigned) * B, cudaMemcpyHostToDevice, h->stream));
  }
  tr_pt[0] = tr_ms();
  KArgs a = base_args(h);
  a.N = r.N; a.thin = r.thin; a.N_keep = (int)n; a.cfg = r.cfg; a.p_override = d_p; a.dir_override = d_dir;
  a.out_q = (double*)out[0].dev; a.out_stats = (dhmc_tree_stats*)out[1].dev; a.out_eps = (double*)out[2].dev;
  a.out_lq = (double*)out[3].dev;
  if (r.cfg.metric == DHMC_METRIC_SYMMETRIC) a.covt = h->covt.get();
  if (r.pool_metric) a.mean_out = h->mean_pool.get();
  a.summary = r.summary;
  const size_t out_bytes = r.posterior ? sizeof(double) * B * n * D : 0;
  // chunks must stay many waves long, or the ragged tail of every chunk idles the SMs
  // chunks overlap the staged downloads (and the upload of q_host) with the sampling of the next chunk; with direct
  // host writes only an upload is left to overlap
  const bool staged_big = r.posterior && !out[0].direct && out_bytes >= ((size_t)32 << 20);
  int nchunks = (!r.outputs_on_device && B >= 4096 && (staged_big || r.q_host)) ? 16 : 1;
  while (nchunks > 1 && B / (size_t)nchunks < (size_t)8 * (size_t)h->grid * (size_t)h->G) nchunks /= 2;   // >= 8 waves of chain slots per chunk
  if (const char* ev = std::getenv("DHMC_E2E_CHUNKS")) { const int v = std::atoi(ev); if (v >= 1 && v <= 16 && !r.outputs_on_device) nchunks = v; }
  CK(cudaMemsetAsync(h->status.get(), 0, sizeof(int) * B, h->stream));   // status words describe the current call
  for (int ci = 0; ci < nchunks; ++ci) {
    // (a pooled metric, and a batch on packed groups, keep their groups of 8 chains inside one chunk)
    const size_t unit = (h->pooled || (h->G > 1 && h->batch_k)) ? 8 : 1;
    const size_t c0 = (B / unit) * ci / nchunks * unit, c1 = (B / unit) * (ci + 1) / nchunks * unit, nc = c1 - c0;
    if (nc == 0) continue;
    a.chain_begin = (int)c0; a.chain_end = (int)c1;
    if (r.q_host) {
      // positions of this chunk: H2D on its own stream, then evaluate_ℓ(strict) on the compute
      // stream — overlaps with the previous chunk's sampling and D2H
      if (ci == 0) {   // uploads start after everything already queued on the compute stream
        CK(cudaEventRecord(h->h2d_ev[15], h->stream));
        CK(cudaStreamWaitEvent(h->h2d_stream, h->h2d_ev[15], 0));
      }
      CK(cudaMemcpyAsync(h->q.get() + c0 * D, r.q_host + c0 * D, sizeof(double) * nc * D, cudaMemcpyHostToDevice, h->h2d_stream));
      CK(cudaEventRecord(h->h2d_ev[ci], h->h2d_stream));
      CK(cudaStreamWaitEvent(h->stream, h->h2d_ev[ci], 0));
      KArgs ea = a;
      ea.strict = 1; ea.randomize = 0;
      rc = launch(h, K_EVAL, ea, nullptr, nullptr);
      if (rc != DHMC_OK) return rc;
    }
    // the kernel time of the call: from the first chunk's k_nuts to the end of the last one's
    rc = launch(h, K_NUTS, a, ci == 0 ? h->ev0 : nullptr, ci == nchunks - 1 ? h->ev1 : nullptr, ci == 0);
    if (rc != DHMC_OK) return rc;
    if (!r.outputs_on_device) {
      CK(cudaEventRecord(h->chunk_ev[ci], h->stream));
      CK(cudaStreamWaitEvent(h->copy_stream, h->chunk_ev[ci], 0));
      for (const Output& o : out)
        if (o.host && !o.direct) {
          const size_t at = c0 * n * o.row;
          CK(cudaMemcpyAsync((char*)o.host + at, (const char*)o.dev + at, nc * n * o.row, cudaMemcpyDeviceToHost, h->copy_stream));
        }
      if (h->trace) CK(cudaEventRecord(h->copy_ev[ci], h->copy_stream));
    }
  }
  tr_pt[1] = tr_ms();
  unsigned long long steps = 0;
  CK(cudaMemcpyAsync(&steps, h->total_steps.get(), sizeof steps, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  tr_pt[2] = tr_ms();
  CK(cudaStreamSynchronize(h->copy_stream));
  tr_pt[3] = tr_ms();
  if ((rc = read_timer(h)) != DHMC_OK) return rc;
  if (h->trace && nchunks > 1) {
    float t;
    std::fprintf(stderr, "[dhmc trace] chunks %d:", nchunks);
    for (int ci = 0; ci < nchunks; ++ci) {
      float a = -1, b2 = -1, c = -1;
      if (r.q_host) cudaEventElapsedTime(&a, h->ev0, h->h2d_ev[ci]);
      cudaEventElapsedTime(&b2, h->ev0, h->chunk_ev[ci]);
      if (!r.outputs_on_device) cudaEventElapsedTime(&c, h->ev0, h->copy_ev[ci]);
      std::fprintf(stderr, " [h2d %.2f kern %.2f d2h %.2f]", a, b2, c);
    }
    cudaEventElapsedTime(&t, h->ev0, h->ev1);
    std::fprintf(stderr, " total kernels %.2f ms | host: setup %.2f, enqueued %.2f, compute stream done %.2f, copy stream done %.2f\n", t,
                 tr_pt[0], tr_pt[1], tr_pt[2], tr_pt[3]);
    cudaGetLastError();
  }
  h->last_steps = (int64_t)steps;
  h->t += (uint32_t)r.N;
  if (r.q_host) h->has_position = true;
  if (h->trace) std::fprintf(stderr, "[dhmc trace] host: before status check %.2f ms\n", tr_ms());
  rc = sync_and_check_status(h, DHMC_CHAIN_NONFINITE_Q | DHMC_CHAIN_BAD_ACCEPTANCE | DHMC_CHAIN_BAD_STEPSIZE |
                                    DHMC_CHAIN_LEAPFROG_NONFINITE | (r.q_host ? DHMC_CHAIN_BAD_INITIAL : 0),
                             r.q_host ? "invalid initial position, or non-finite position / acceptance rate / step size while sampling"
                                    : "sampling: non-finite position, acceptance rate or step size");
  if (h->trace) std::fprintf(stderr, "[dhmc trace] host: after status check %.2f ms\n", tr_ms());
  if (rc != DHMC_OK) return rc;
  if (r.cfg.metric == DHMC_METRIC_DIAGONAL) return set_metric_kind(h, false, false);   // κ ← Diagonal: the diagonal kernels
  if (r.cfg.metric == DHMC_METRIC_SYMMETRIC) {
    // κ = GaussianKineticEnergy(regularize_M⁻¹(sample_M⁻¹(Symmetric, X), λ)) — mcmc.jl:282
    const int fgrid = factor_grid(h);
    if (r.pool_metric)
      k_cov_pool<<<fgrid, 128, sizeof(double) * h->cfg.dim, h->stream>>>(h->covt.get(), h->mean_pool.get(), h->minv_dense.get(), r.N, r.lambda, (int)h->cfg.dim, (int)h->cfg.n_chains);
    else
      k_cov_finish<<<fgrid, 128, 0, h->stream>>>(h->covt.get(), h->minv_dense.get(), r.N, r.lambda, (int)h->cfg.dim, (int)h->cfg.n_chains);
    h->launches += 1;
    rc = factor_and_switch(h, r.pool_metric);
  }
  return rc;
}

int dhmc_sample_tree(dhmc_handle* h, const double* p, const uint32_t* directions, dhmc_tree_stats* stats) {
  if (!h) return DHMC_EARG;
  NutsRequest r; r.N = 1; r.p_over_host = p; r.dir_over_host = directions; r.stats = stats;
  return run_nuts(h, r);
}

int dhmc_warmup_stage(dhmc_handle* h, int32_t N, int32_t metric, const dhmc_dual_averaging* da,
                      double lambda, double* posterior, dhmc_tree_stats* stats, double* eps_used,
                      double* logdens) {
  if (!h) return DHMC_EARG;
  // TuningNUTS @argchecks — mcmc.jl:191-192
  if (!(N >= 20)) { h->err = "N ≥ 20"; return DHMC_EARG; }
  if (!(lambda >= 0)) { h->err = "λ ≥ 0"; return DHMC_EARG; }
  if (metric != DHMC_METRIC_NOTHING && metric != DHMC_METRIC_DIAGONAL && metric != DHMC_METRIC_SYMMETRIC &&
      metric != DHMC_METRIC_SYMMETRIC_POOLED) { h->err = "metric: Nothing, Diagonal, Symmetric (or the pooled Symmetric option)"; return DHMC_EARG; }
  const bool pool = metric == DHMC_METRIC_SYMMETRIC_POOLED;
  if (pool && (h->cfg.n_chains % 8 != 0 || h->cfg.chain_offset % 8 != 0)) { h->err = "pooled metric: n_chains and chain_offset must be multiples of 8"; return DHMC_EARG; }
  if (pool && h->batch_k % 8 != 0) { h->err = "pooled metric with a problem batch: chains_per_problem must be a multiple of 8 (a metric group never straddles two problems)"; return DHMC_EARG; }
  NutsRequest r; r.N = N; r.lambda = lambda; r.pool_metric = pool;
  r.posterior = posterior; r.stats = stats; r.eps_used = eps_used; r.logdens = logdens;
  r.cfg.metric = pool ? DHMC_METRIC_SYMMETRIC : metric;
  if (da) {
    // DualAveraging @argchecks — stepsize.jl:108-111
    if (!(0 < da->delta && da->delta < 1) || !(da->gamma > 0) || !(0.5 < da->kappa && da->kappa <= 1) || !(da->t0 >= 0)) {
      h->err = "DualAveraging: 0 < δ < 1, γ > 0, 0.5 < κ ≤ 1, t₀ ≥ 0"; return DHMC_EARG;
    }
    r.cfg.adapt = 1; r.cfg.delta = da->delta; r.cfg.gamma = da->gamma; r.cfg.kappa = da->kappa; r.cfg.t0 = da->t0;
  }
  if (r.cfg.metric == DHMC_METRIC_SYMMETRIC) { int rcd = ensure_dense(h); if (rcd != DHMC_OK) return rcd; }
  if (pool) CK(h->mean_pool.grow((size_t)h->cfg.n_chains * (size_t)h->cfg.dim));
  return run_nuts(h, r);
}

int dhmc_mcmc(dhmc_handle* h, int32_t N, double* posterior, dhmc_tree_stats* stats, double* logdens) {
  if (!h || N < 0) return DHMC_EARG;
  if (N == 0) return DHMC_OK;
  NutsRequest r; r.N = N; r.posterior = posterior; r.stats = stats; r.logdens = logdens;
  return run_nuts(h, r);
}
int dhmc_mcmc_from(dhmc_handle* h, const double* q, int32_t N, double* posterior, dhmc_tree_stats* stats,
                   double* logdens) {
  if (!h || !q || N < 1) return DHMC_EARG;
  NutsRequest r; r.N = N; r.q_host = q; r.posterior = posterior; r.stats = stats; r.logdens = logdens;
  return run_nuts(h, r);
}
int dhmc_mcmc_thinned(dhmc_handle* h, const double* q, int32_t N, int32_t thin, double* posterior,
                      dhmc_tree_stats* stats, double* logdens) {
  if (!h || N < 1 || thin < 1) return DHMC_EARG;
  NutsRequest r; r.N = N; r.thin = thin; r.q_host = q; r.posterior = posterior; r.stats = stats; r.logdens = logdens;
  return run_nuts(h, r);
}
// Page-locked host memory on the NUMA node of the handle's GPU: the calling thread is moved to that node's CPUs while the
// pages are allocated and pinned (first touch), so that the kernel's direct writes / the DMA engines cross one PCIe root
// complex and no inter-socket link.  *node receives the NUMA node (or -1 when unknown).
int dhmc_host_alloc(dhmc_handle* h, size_t bytes, void** out, int32_t* node) {
  if (!h || !out || bytes == 0) return DHMC_EARG;
  CK(cudaSetDevice(h->cfg.device));
  int numa = -1;
  char bus[32] = {0};
  if (cudaDeviceGetPCIBusId(bus, sizeof bus, h->cfg.device) == cudaSuccess) {
    for (char* c = bus; *c; ++c) *c = (char)std::tolower(*c);
    std::ifstream f(std::string("/sys/bus/pci/devices/") + bus + "/numa_node");
    if (f) f >> numa;
  } else {
    cudaGetLastError();
  }
  cpu_set_t old_set, node_set;
  bool moved = false;
  if (numa >= 0 && sched_getaffinity(0, sizeof old_set, &old_set) == 0) {
    std::ifstream f("/sys/devices/system/node/node" + std::to_string(numa) + "/cpulist");
    std::string list;
    if (f && std::getline(f, list)) {
      CPU_ZERO(&node_set);
      size_t pos = 0;
      while (pos < list.size()) {            // "0-31,64-95"
        size_t end = list.find(',', pos);
        if (end == std::string::npos) end = list.size();
        const std::string tok = list.substr(pos, end - pos);
        const size_t dash = tok.find('-');
        const int a = std::atoi(tok.c_str()), b = dash == std::string::npos ? a : std::atoi(tok.c_str() + dash + 1);
        for (int c = a; c <= b && c < CPU_SETSIZE; ++c) if (CPU_ISSET(c, &old_set)) CPU_SET(c, &node_set);
        pos = end + 1;
      }
      if (CPU_COUNT(&node_set) > 0 && sched_setaffinity(0, sizeof node_set, &node_set) == 0) moved = true;
    }
  }
  void* p = nullptr;
  const cudaError_t e = cudaHostAlloc(&p, bytes, cudaHostAllocMapped | cudaHostAllocPortable);
  if (moved) sched_setaffinity(0, sizeof old_set, &old_set);
  if (e != cudaSuccess) { h->err = std::string("cudaHostAlloc: ") + cudaGetErrorString(e); return DHMC_ENOMEM; }
  *out = p;
  if (node) *node = numa;
  return DHMC_OK;
}
int dhmc_host_free(dhmc_handle* h, void* p) {
  if (!h) return DHMC_EARG;
  if (p && cudaFreeHost(p) != cudaSuccess) { h->err = "cudaFreeHost failed"; cudaGetLastError(); return DHMC_ECUDA; }
  return DHMC_OK;
}
int dhmc_mcmc_dev(dhmc_handle* h, int32_t N, double* posterior, dhmc_tree_stats* stats, double* logdens) {
  if (!h || N < 0) return DHMC_EARG;
  if (N == 0) return DHMC_OK;
  NutsRequest r; r.N = N; r.posterior = posterior; r.stats = stats; r.logdens = logdens; r.outputs_on_device = true;
  return run_nuts(h, r);
}

// ------------------------------------------------------------------ streaming posterior summary (DESIGN §4.4)
// The grid of every (d, p) cell of a quantile histogram (include/dhmc.h): nbins in [1, 4096], lo < hi finite, hi − lo and
// nbins / (hi − lo) finite (so that inv_w is a finite number)
static bool valid_grid(const double* lo, const double* hi, int nbins, size_t cells) {
  if (!lo || !hi || nbins < 1 || nbins > 4096) return false;
  for (size_t i = 0; i < cells; ++i) {
    const double w = hi[i] - lo[i];
    if (!(std::isfinite(lo[i]) && std::isfinite(hi[i]) && lo[i] < hi[i] && std::isfinite(w) && std::isfinite((double)nbins / w)))
      return false;
  }
  return true;
}

// rows [r0, r0 + n) of every problem of a host array [P][R] into the device array [P][n]
static cudaError_t upload_rows(double* dst, const double* src, size_t r0, size_t n, size_t R, size_t P, cudaStream_t s) {
  return cudaMemcpy2DAsync(dst, sizeof(double) * n, src + r0, sizeof(double) * R, sizeof(double) * n, P, cudaMemcpyHostToDevice, s);
}

// generated quantities of device points theta [n_problems][n][D] (problem first + j owns points j·n … (j+1)·n − 1) into
// out [n_problems][n][G] on the handle's stream (k_generated, family_tu.cu); random quantities read point pt's key from the
// device arrays chain [pt] and transition [pt] (null for deterministic ones); the caller has checked the arguments
static int launch_generated(dhmc_handle* h, const double* theta, int64_t n, int64_t first, int64_t n_problems, const int64_t* chain,
                            const uint32_t* transition, double* out) {
  const int64_t pts = n * n_problems;
  const int grid = (int)std::min<int64_t>(pts, (int64_t)h->sm_count * 16);
  const int e = dhmc_user_family_generated(theta, n, n_problems, (int)h->cfg.dim, h->ngq, h->mparams.get(),
                                           h->batch_k ? h->problems.get() : nullptr, first, (const long long*)chain, transition,
                                           (unsigned long long)h->cfg.seed, out, h->T, grid, h->stream);
  if (e != cudaSuccess) { h->err = std::string("k_generated: ") + cudaGetErrorString((cudaError_t)e); return DHMC_ECUDA; }
  h->launches += 1;
  return DHMC_OK;
}

// dhmc_generated(_dev) and dhmc_generated_keyed(_dev): DHMC_EARG before anything runs for a handle without generated
// quantities, NULL pointers, n < 1, n_problems < 1, a problem range outside the handle's batch, or a model with random
// quantities called without keys
static int check_generated(dhmc_handle* h, const double* theta, int64_t n, int64_t first, int64_t n_problems, const double* out,
                           bool keyed, const int64_t* chain, const uint32_t* transition) {
  const int64_t P = h->batch_k ? h->batch_p : 1;
  if (h->ngq == 0) { h->err = "dhmc_generated: the handle's model has no generated quantities"; return DHMC_EARG; }
  if (!keyed && h->gq_random) {
    h->err = "dhmc_generated: the model's generated quantities are random (DHMC_USER_GENERATED_RNG); call dhmc_generated_keyed "
             "with the chain id and transition of every point";
    return DHMC_EARG;
  }
  if (!theta || !out) { h->err = "dhmc_generated: theta or out is NULL"; return DHMC_EARG; }
  if (keyed && (!chain || !transition)) { h->err = "dhmc_generated_keyed: chain or transition is NULL"; return DHMC_EARG; }
  if (n < 1 || n_problems < 1 || first < 0 || first > P - n_problems) {
    h->err = "dhmc_generated: n ≥ 1, and problems first … first + n_problems − 1 of the handle's batch";
    return DHMC_EARG;
  }
  return DHMC_OK;
}

int dhmc_user_generated_count(int64_t dim, int32_t* G) {
  if (!dhmc_user_family_name_str || !G || dim < 1 || dim > INT32_MAX) return DHMC_EARG;
  *G = dhmc_user_family_ngq ? dhmc_user_family_ngq((int)dim) : 0;
  return DHMC_OK;
}

int dhmc_user_generated_random(int32_t* random) {
  if (!dhmc_user_family_name_str || !random) return DHMC_EARG;
  *random = dhmc_user_family_random ? dhmc_user_family_random() : 0;
  return DHMC_OK;
}

int dhmc_generated_count(dhmc_handle* h, int32_t* G) {
  if (!h || !G) return DHMC_EARG;
  *G = h->ngq;
  return DHMC_OK;
}

int dhmc_generated_random(dhmc_handle* h, int32_t* random) {
  if (!h || !random) return DHMC_EARG;
  *random = h->gq_random ? 1 : 0;
  return DHMC_OK;
}

// device arrays: check, launch, wait
static int generated_dev(dhmc_handle* h, const double* theta, int64_t n, int64_t first, int64_t n_problems, bool keyed,
                         const int64_t* chain, const uint32_t* transition, double* out) {
  if (!h) return DHMC_EARG;
  const int rc = check_generated(h, theta, n, first, n_problems, out, keyed, chain, transition);
  if (rc != DHMC_OK) return rc;
  CK(cudaSetDevice(h->cfg.device));
  const int rg = launch_generated(h, theta, n, first, n_problems, chain, transition, out);
  if (rg != DHMC_OK) return rg;
  CK(cudaStreamSynchronize(h->stream));
  return DHMC_OK;
}

// host arrays: check (keys: chain ids in [0, 2^56), the key's width), upload points and keys, launch, download
static int generated_host(dhmc_handle* h, const double* theta, int64_t n, int64_t first, int64_t n_problems, bool keyed,
                          const int64_t* chain, const uint32_t* transition, double* out) {
  if (!h) return DHMC_EARG;
  const int rc = check_generated(h, theta, n, first, n_problems, out, keyed, chain, transition);
  if (rc != DHMC_OK) return rc;
  const size_t pts = (size_t)n * (size_t)n_problems, D = (size_t)h->cfg.dim, G = (size_t)h->ngq;
  if (keyed)
    for (size_t i = 0; i < pts; ++i)
      if (chain[i] < 0 || chain[i] >= ((int64_t)1 << 56)) { h->err = "dhmc_generated_keyed: chain ids lie in [0, 2^56)"; return DHMC_EARG; }
  CK(cudaSetDevice(h->cfg.device));
  // one buffer: points [pts][D], out [pts][G], then with keys chain [pts] (8-byte) and transition [pts] (4-byte)
  DeviceArray<char> buf;
  CK(buf.alloc(sizeof(double) * pts * (D + G) + (keyed ? (sizeof(int64_t) + sizeof(uint32_t)) * pts : 0)));
  double* dtheta = (double*)buf.get();
  double* dout = dtheta + pts * D;
  int64_t* dchain = keyed ? (int64_t*)(dout + pts * G) : nullptr;
  uint32_t* dtrans = keyed ? (uint32_t*)(dchain + pts) : nullptr;
  CK(cudaMemcpyAsync(dtheta, theta, sizeof(double) * pts * D, cudaMemcpyHostToDevice, h->stream));
  if (keyed) CK(cudaMemcpyAsync(dchain, chain, sizeof(int64_t) * pts, cudaMemcpyHostToDevice, h->stream));
  if (keyed) CK(cudaMemcpyAsync(dtrans, transition, sizeof(uint32_t) * pts, cudaMemcpyHostToDevice, h->stream));
  if (int rg = launch_generated(h, dtheta, n, first, n_problems, dchain, dtrans, dout)) return rg;
  CK(cudaMemcpyAsync(out, dout, sizeof(double) * pts * G, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return DHMC_OK;
}

int dhmc_generated_dev(dhmc_handle* h, const double* theta, int64_t n, int64_t first_problem, int64_t n_problems, double* out) {
  return generated_dev(h, theta, n, first_problem, n_problems, false, nullptr, nullptr, out);
}

int dhmc_generated(dhmc_handle* h, const double* theta, int64_t n, int64_t first_problem, int64_t n_problems, double* out) {
  return generated_host(h, theta, n, first_problem, n_problems, false, nullptr, nullptr, out);
}

int dhmc_generated_keyed(dhmc_handle* h, const double* theta, int64_t n, int64_t first_problem, int64_t n_problems,
                         const int64_t* chain, const uint32_t* transition, double* out) {
  return generated_host(h, theta, n, first_problem, n_problems, true, chain, transition, out);
}

int dhmc_generated_keyed_dev(dhmc_handle* h, const double* theta, int64_t n, int64_t first_problem, int64_t n_problems,
                             const int64_t* chain, const uint32_t* transition, double* out) {
  return generated_dev(h, theta, n, first_problem, n_problems, true, chain, transition, out);
}

// One block of summary rows: rows r0 … r0 + n − 1 of the [·, R, P] host arrays, and the device arrays the kernels fold them
// into.  width: state per row and resident chain group (3 for parameters, whose moments live in the metric slots; 5 for G).
struct SummaryRows {
  size_t r0, n, width;
  double *acc = nullptr, *shift = nullptr, *ref = nullptr, *row = nullptr, *lo = nullptr, *inv_w = nullptr;
  unsigned long long *below = nullptr, *hist = nullptr;
  unsigned* stage = nullptr;
};

// dhmc_mcmc_summary and, with counts, dhmc_mcmc_summary_histogram (arguments checked by the caller)
static int mcmc_summary(dhmc_handle* h, int32_t N, int32_t thin, const double* reference, const double* lo_host,
                        const double* hi_host, int32_t nbins, double* record, int64_t* counts, dhmc_tree_stats* stats,
                        double* logdens) {
  if (N < 1 || thin < 1 || N % thin != 0) { h->err = "dhmc_mcmc_summary: N ≥ 1, thin ≥ 1 and N a multiple of thin"; return DHMC_EARG; }
  const int n_keep = N / thin;
  if (n_keep < 4) { h->err = "dhmc_mcmc_summary: at least 4 kept draws per chain (N / thin ≥ 4)"; return DHMC_EARG; }
  if (!record) { h->err = "dhmc_mcmc_summary: record is NULL"; return DHMC_EARG; }
  if (!h->has_position || !h->has_eps) { h->err = "set position and step size (or run the initial search) first"; return DHMC_EARG; }
  CK(cudaSetDevice(h->cfg.device));
  // generated quantities: ng rows after the D parameter rows of every host array (R = D + ng); empty with ng = 0
  const size_t D = (size_t)h->cfg.dim, B = (size_t)h->cfg.n_chains, ng = (size_t)h->ngq, R = D + ng;
  const int64_t K = h->batch_k, off = h->cfg.chain_offset;
  // histograms (counts != NULL): cells bins per (row, problem), and staging rows [cells][n] per resident chain group
  const size_t P = K ? (size_t)h->batch_p : 1, groups = (size_t)h->grid * h->G, cells = counts ? (size_t)nbins + 2 : 0;
  SummaryRows blk[2] = {{0, D, 3}, {D, ng, 5}};
  SummaryRows &par = blk[0], &gen = blk[1];
  unsigned long long* chains;                  // completed chains per problem [P]
  int64_t* kchain = nullptr;                   // keys of the generated shift's points, chain [P] and transition [P]
  uint32_t* ktrans = nullptr;
  // one grow-only arena of the arrays below, in this order (8-byte elements, then the 4-byte staging rows, then the 8-aligned
  // keys of random generated quantities): carve(nullptr) measures it, carve(base) places the arrays in it
  auto carve = [&](char* base) {
    size_t at = 0;
    auto take = [&](auto& ptr, size_t n) {
      ptr = base ? reinterpret_cast<std::remove_reference_t<decltype(ptr)>>(base + at) : nullptr;
      at += sizeof(*ptr) * n;
    };
    for (SummaryRows& b : blk) {             // acc, below and hist adjacent: one memset zeroes them
      const size_t pn = P * b.n;
      take(b.acc, 5 * pn); take(b.below, pn); take(b.hist, pn * cells);
      take(b.shift, pn); take(b.ref, pn); take(b.row, groups * b.width * b.n);
      if (counts) { take(b.lo, pn); take(b.inv_w, pn); }
    }
    take(chains, P);
    for (SummaryRows& b : blk) take(b.stage, groups * cells * b.n);
    if (h->gq_random) { at = (at + 7) & ~(size_t)7; take(kchain, P); take(ktrans, P); }
    return at;
  };
  CK(h->sum_buf.grow(carve(nullptr)));
  carve(h->sum_buf.get());
  CK(h->sum_args.grow(1));
  std::vector<double> hinv(counts ? P * R : 0);
  for (size_t i = 0; i < hinv.size(); ++i) hinv[i] = (double)nbins / (hi_host[i] - lo_host[i]);
  for (const SummaryRows& b : blk) {
    if (!b.n) continue;
    CK(cudaMemsetAsync(b.acc, 0, sizeof(double) * P * b.n * (6 + cells), h->stream));
    if (reference) CK(upload_rows(b.ref, reference, b.r0, b.n, R, P, h->stream));
    if (counts) {
      CK(upload_rows(b.lo, lo_host, b.r0, b.n, R, P, h->stream));
      CK(upload_rows(b.inv_w, hinv.data(), b.r0, b.n, R, P, h->stream));
    }
  }
  CK(cudaMemsetAsync(chains, 0, sizeof(unsigned long long) * P, h->stream));
  // shift of problem p: the position of its first local chain, max(p·K − off, 0); problems p0 … p1 have local chains.  Past
  // the first, those chains are K apart: one strided copy (a first problem entered in its middle takes one more).
  const int64_t p0 = K ? off / K : 0, p1 = K ? (off + (int64_t)B - 1) / K : 0;
  const int64_t pa = (K && off % K) ? p0 + 1 : p0;
  if (pa > p0) CK(cudaMemcpyAsync(par.shift + p0 * D, h->q.get(), sizeof(double) * D, cudaMemcpyDeviceToDevice, h->stream));
  if (p1 >= pa)
    CK(cudaMemcpy2DAsync(par.shift + pa * D, sizeof(double) * D, h->q.get() + (size_t)(K ? pa * K - off : 0) * D, sizeof(double) * D * (size_t)(K ? K : 1),
                         sizeof(double) * D, (size_t)(p1 - pa + 1), cudaMemcpyDeviceToDevice, h->stream));
  SummaryArgs sa{par.row, par.shift, reference ? par.ref : nullptr, par.acc, par.below, chains, n_keep / 2, nullptr, nullptr, nullptr, nullptr, 0};
  if (counts) { sa.lo = par.lo; sa.inv_w = par.inv_w; sa.stage = par.stage; sa.hist = par.hist; sa.nbins = nbins; }
  // generated quantities: the shift is g(shift), evaluated on the device
  if (ng) {
    // random quantities: the shift's key is (global id of the problem's first local chain, the call's first transition);
    // it only sets the cancellation shift of the sums
    if (h->gq_random) {
      const size_t np = (size_t)(p1 - p0 + 1);
      std::vector<int64_t> hc(np);
      std::vector<uint32_t> ht(np, h->t);
      for (size_t i = 0; i < np; ++i) hc[i] = K ? std::max((p0 + (int64_t)i) * K, off) : off;
      CK(cudaMemcpyAsync(kchain, hc.data(), sizeof(int64_t) * np, cudaMemcpyHostToDevice, h->stream));
      CK(cudaMemcpyAsync(ktrans, ht.data(), sizeof(uint32_t) * np, cudaMemcpyHostToDevice, h->stream));
    }
    const int rg = launch_generated(h, par.shift + p0 * D, 1, p0, p1 - p0 + 1, kchain, ktrans, gen.shift + p0 * ng);
    if (rg != DHMC_OK) return rg;
    sa.ng = (int)ng; sa.mparams = h->mparams.get(); sa.problems = K ? h->problems.get() : nullptr;
    sa.seed = (unsigned long long)h->cfg.seed; sa.chain_offset = (long long)off; sa.t0 = h->t; sa.thin = thin;
    sa.grow = gen.row; sa.gshift = gen.shift; sa.gref = reference ? gen.ref : nullptr; sa.gacc = gen.acc; sa.gbelow = gen.below;
    if (counts) { sa.glo = gen.lo; sa.ginv_w = gen.inv_w; sa.gstage = gen.stage; sa.ghist = gen.hist; }
  }
  CK(cudaMemcpyAsync(h->sum_args.get(), &sa, sizeof sa, cudaMemcpyHostToDevice, h->stream));
  NutsRequest req; req.N = N; req.thin = thin; req.stats = stats; req.logdens = logdens; req.summary = h->sum_args.get();
  const int rc = run_nuts(h, req);
  if (rc != DHMC_OK && rc != DHMC_ENUMERIC) return rc;    // a chain that failed is left out of its problem's sums
  // host copies: a block's sums [P][5][n], shifts and below-counts [P][n] at P·r0
  std::vector<double> hacc(5 * P * R), hshift(P * R);
  std::vector<unsigned long long> hbelow(P * R), hchains(P);
  for (const SummaryRows& b : blk) {
    if (!b.n) continue;
    const size_t at = P * b.r0, pn = P * b.n, c8 = sizeof(int64_t) * cells;
    CK(cudaMemcpyAsync(&hacc[5 * at], b.acc, sizeof(double) * 5 * pn, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaMemcpyAsync(&hshift[at], b.shift, sizeof(double) * pn, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaMemcpyAsync(&hbelow[at], b.below, sizeof(unsigned long long) * pn, cudaMemcpyDeviceToHost, h->stream));
    // [P][n][cells] into rows r0 … r0 + n − 1 of the column-major [cells, R, P] of the ABI; uint64 counts stay far below 2^63
    if (counts) CK(cudaMemcpy2DAsync(counts + b.r0 * cells, c8 * R, b.hist, c8 * b.n, c8 * b.n, P, cudaMemcpyDeviceToHost, h->stream));
  }
  CK(cudaMemcpyAsync(hchains.data(), chains, sizeof(unsigned long long) * P, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  // record [F, R, P] column-major: the cell of row r0 + k of problem p, from its sums a ([5][n]), shift and below-count
  for (size_t p = 0; p < P; ++p)
    for (const SummaryRows& b : blk)
      for (size_t k = 0, i = P * b.r0 + p * b.n; k < b.n; ++k) {
        const double M = (double)hchains[p], m = 2.0 * M, *a = &hacc[5 * i];
        double* r = record + (p * R + b.r0 + k) * DHMC_SUMMARY_FIELDS;
        r[DHMC_SUMMARY_CHAINS] = M;
        r[DHMC_SUMMARY_NKEEP] = (double)n_keep;
        r[DHMC_SUMMARY_BELOW] = reference ? (double)hbelow[i + k] : dm_nan();
        if (M == 0) { r[DHMC_SUMMARY_MEAN] = r[DHMC_SUMMARY_SS_SEQ] = r[DHMC_SUMMARY_M2] = r[DHMC_SUMMARY_SS_CHAIN] = 0.0; continue; }
        const double s1 = a[k], s2 = a[b.n + k], c1 = a[3 * b.n + k], c2 = a[4 * b.n + k];
        r[DHMC_SUMMARY_MEAN] = hshift[i + k] + s1 / m;
        r[DHMC_SUMMARY_SS_SEQ] = std::max(0.0, s2 - s1 * s1 / m);
        r[DHMC_SUMMARY_M2] = a[2 * b.n + k];
        r[DHMC_SUMMARY_SS_CHAIN] = std::max(0.0, c2 - c1 * c1 / M);
      }
  return rc;
}

int dhmc_mcmc_summary(dhmc_handle* h, int32_t N, int32_t thin, const double* reference, double* record, dhmc_tree_stats* stats,
                      double* logdens) {
  if (!h) return DHMC_EARG;
  return mcmc_summary(h, N, thin, reference, nullptr, nullptr, 0, record, nullptr, stats, logdens);
}

int dhmc_mcmc_summary_histogram(dhmc_handle* h, int32_t N, int32_t thin, const double* reference, const double* lo,
                                const double* hi, int32_t nbins, double* record, int64_t* counts, dhmc_tree_stats* stats,
                                double* logdens) {
  if (!h) return DHMC_EARG;
  if (!counts) { h->err = "dhmc_mcmc_summary_histogram: counts is NULL"; return DHMC_EARG; }
  const size_t cells = ((size_t)h->cfg.dim + (size_t)h->ngq) * (h->batch_k ? (size_t)h->batch_p : 1);
  if (!valid_grid(lo, hi, nbins, cells)) {
    h->err = "dhmc_mcmc_summary_histogram: 1 ≤ nbins ≤ 4096 and, per cell, finite lo < hi with hi − lo and nbins / (hi − lo) finite";
    return DHMC_EARG;
  }
  return mcmc_summary(h, N, thin, reference, lo, hi, nbins, record, counts, stats, logdens);
}

// Type-7 quantile (Julia's default) at α of the values counted in bins 0 … nbins + 1 on the grid (lo, hi, nbins), as
// include/dhmc.h defines it: cum[k] = C_k, the count of bins 0 … k.  Order statistic r lies in the first bin k with r < C_k
// and is placed strictly inside it, at e_{k−1} + ((r − C_{k−1}) + 0.5)/c_k · (e_k − e_{k−1}).  Shared by
// dhmc_histogram_quantiles and dhmc_acceptance_quantiles_dev, whose grid (0, 1, 4096) has exact edges.
static void binned_quantile(const unsigned long long* cum, int nbins, double lo, double hi, double alpha, double* q, double* q_lo,
                            double* q_hi) {
  const unsigned long long n = cum[nbins + 1];
  if (n == 0) { *q = *q_lo = *q_hi = dm_nan(); return; }
  const double w = (hi - lo) / (double)nbins;
  auto edge = [&](int k) { return k < nbins ? lo + (double)k * w : hi; };
  auto bin_of = [&](unsigned long long r) { return (int)(std::upper_bound(cum, cum + nbins + 2, r) - cum); };
  auto place = [&](unsigned long long r, int k) {
    if (k == 0 || k == nbins + 1) return dm_nan();
    const unsigned long long below = cum[k - 1];
    return edge(k - 1) + ((double)(r - below) + 0.5) / (double)(cum[k] - below) * (edge(k) - edge(k - 1));
  };
  const double pos = alpha * (double)(n - 1);
  const unsigned long long j = (unsigned long long)pos;
  const double gamma = pos - (double)j;
  const int kj = bin_of(j), kh = gamma > 0.0 ? bin_of(j + 1) : kj;
  const double xj = place(j, kj);
  *q = gamma > 0.0 ? xj + gamma * (place(j + 1, kh) - xj) : xj;
  *q_lo = kj == 0 ? -dm_inf() : edge(kj - 1);
  *q_hi = kh == nbins + 1 ? dm_inf() : edge(kh);
}

int dhmc_histogram_quantiles(const int64_t* counts, const double* lo, const double* hi, int32_t nbins, int64_t D, int64_t P,
                             const double* probs, int32_t nprobs, double* q, double* q_lo, double* q_hi) {
  if (!counts || !probs || D < 1 || P < 1 || nprobs < 1) return DHMC_EARG;
  const size_t n_cells = (size_t)D * (size_t)P;
  if (!valid_grid(lo, hi, nbins, n_cells)) return DHMC_EARG;
  for (int k = 0; k < nprobs; ++k)
    if (!(probs[k] >= 0.0 && probs[k] <= 1.0)) return DHMC_EARG;
  const size_t nb2 = (size_t)nbins + 2;
  for (size_t i = 0; i < n_cells * nb2; ++i)
    if (counts[i] < 0) return DHMC_EARG;
  std::vector<unsigned long long> cum(nb2);
  for (size_t i = 0; i < n_cells; ++i) {
    unsigned long long c = 0;
    for (size_t b = 0; b < nb2; ++b) cum[b] = c += (unsigned long long)counts[i * nb2 + b];
    for (int k = 0; k < nprobs; ++k) {
      double a, l, u;
      binned_quantile(cum.data(), nbins, lo[i], hi[i], probs[k], &a, &l, &u);
      const size_t o = i * (size_t)nprobs + k;
      if (q) q[o] = a;
      if (q_lo) q_lo[o] = l;
      if (q_hi) q_hi[o] = u;
    }
  }
  return DHMC_OK;
}

int dhmc_summary_merge(double* record, const double* other, int64_t D, int64_t P) {
  if (!record || !other || D < 1 || P < 1) return DHMC_EARG;
  const size_t n = (size_t)D * (size_t)P;
  for (size_t i = 0; i < n; ++i) {      // every count must agree before anything is written
    const double* a = record + i * DHMC_SUMMARY_FIELDS;
    const double* b = other + i * DHMC_SUMMARY_FIELDS;
    if (a[DHMC_SUMMARY_CHAINS] > 0 && b[DHMC_SUMMARY_CHAINS] > 0 && a[DHMC_SUMMARY_NKEEP] != b[DHMC_SUMMARY_NKEEP]) return DHMC_EARG;
  }
  for (size_t i = 0; i < n; ++i) {
    double* a = record + i * DHMC_SUMMARY_FIELDS;
    const double* b = other + i * DHMC_SUMMARY_FIELDS;
    const double ma = a[DHMC_SUMMARY_CHAINS], mb = b[DHMC_SUMMARY_CHAINS], below = a[DHMC_SUMMARY_BELOW] + b[DHMC_SUMMARY_BELOW];
    if (mb == 0) { a[DHMC_SUMMARY_BELOW] = below; continue; }
    if (ma == 0) {
      for (int f = 0; f < DHMC_SUMMARY_FIELDS; ++f) a[f] = b[f];
      a[DHMC_SUMMARY_BELOW] = below;
      continue;
    }
    // Chan, Golub and LeVeque: pooled mean and centred sums of squares of two groups (2 sequences per chain)
    const double M = ma + mb, delta = b[DHMC_SUMMARY_MEAN] - a[DHMC_SUMMARY_MEAN];
    a[DHMC_SUMMARY_MEAN] = a[DHMC_SUMMARY_MEAN] + delta * (mb / M);
    a[DHMC_SUMMARY_SS_SEQ] = a[DHMC_SUMMARY_SS_SEQ] + b[DHMC_SUMMARY_SS_SEQ] + delta * delta * (2.0 * ma * mb / M);
    a[DHMC_SUMMARY_M2] = a[DHMC_SUMMARY_M2] + b[DHMC_SUMMARY_M2];
    a[DHMC_SUMMARY_SS_CHAIN] = a[DHMC_SUMMARY_SS_CHAIN] + b[DHMC_SUMMARY_SS_CHAIN] + delta * delta * (ma * mb / M);
    a[DHMC_SUMMARY_CHAINS] = M;
    a[DHMC_SUMMARY_BELOW] = below;
  }
  return DHMC_OK;
}

int dhmc_summary_finish(const double* record, int64_t D, int64_t P, double* mean, double* sd, double* mcse, double* ess,
                        double* rhat, int64_t* rank, int64_t* draws) {
  if (!record || D < 1 || P < 1) return DHMC_EARG;
  const size_t n_cells = (size_t)D * (size_t)P;
  for (size_t i = 0; i < n_cells; ++i) {
    const double* r = record + i * DHMC_SUMMARY_FIELDS;
    const double M = r[DHMC_SUMMARY_CHAINS], m = 2.0 * M, n = std::floor(r[DHMC_SUMMARY_NKEEP] / 2.0);
    const double below = r[DHMC_SUMMARY_BELOW];
    if (rank) rank[i] = below == below ? (int64_t)below : -1;
    if (draws) draws[i] = (int64_t)(r[DHMC_SUMMARY_NKEEP] * M);
    double o_mean = dm_nan(), o_sd = dm_nan(), o_mcse = dm_nan(), o_ess = dm_nan(), o_rhat = dm_nan();
    if (M > 0) {
      const double ss = r[DHMC_SUMMARY_SS_SEQ], m2 = r[DHMC_SUMMARY_M2];
      const double var = (m2 + n * ss) / (m * n - 1.0);               // pooled variance of the 2n·M draws
      const double W = m2 / (m * (n - 1.0));                          // mean within-sequence variance
      const double var_plus = (n - 1.0) / n * W + ss / (m - 1.0);     // (n−1)/n·W + var(μ_s), as ess_rhat_groups
      o_mean = r[DHMC_SUMMARY_MEAN];
      o_sd = std::sqrt(var);
      o_rhat = std::sqrt(var_plus / W);
      if (M >= 2) {
        const double var_c = r[DHMC_SUMMARY_SS_CHAIN] / (M - 1.0) / M;   // squared standard error of the chain means' mean
        o_mcse = std::sqrt(var_c);
        if (var_plus > 0.0) o_ess = var / var_c;
      }
    }
    if (mean) mean[i] = o_mean;
    if (sd) sd[i] = o_sd;
    if (mcse) mcse[i] = o_mcse;
    if (ess) ess[i] = o_ess;
    if (rhat) rhat[i] = o_rhat;
  }
  return DHMC_OK;
}

int dhmc_tree_summary_dev(dhmc_handle* h, const dhmc_tree_stats* stats_dev, int32_t N, int64_t* depth_counts,
                          int64_t* termination_counts, double* acceptance_sum, int64_t* steps_sum, double* ebfmi) {
  if (!h || !stats_dev || N < 1) return DHMC_EARG;
  CK(cudaSetDevice(h->cfg.device));
  const int B = (int)h->cfg.n_chains;
  DeviceArray<unsigned long long> d_cnt;   // [33 depth][3 term][1 steps]
  DeviceArray<double> d_f;                 // [1 acc][B ebfmi]
  CK(d_cnt.alloc(37));
  CK(d_f.alloc(1 + (size_t)B));
  CK(cudaMemsetAsync(d_cnt.get(), 0, sizeof(unsigned long long) * 37, h->stream));
  CK(cudaMemsetAsync(d_f.get(), 0, sizeof(double), h->stream));
  k_tree_summary<<<h->sm_count * 8, 256, 0, h->stream>>>(stats_dev, N, B, d_cnt.get(), d_cnt.get() + 33, d_f.get(), d_cnt.get() + 36, ebfmi ? d_f.get() + 1 : nullptr);
  h->launches += 1;
  unsigned long long cnt[37];
  double acc = 0;
  CK(cudaMemcpyAsync(cnt, d_cnt.get(), sizeof cnt, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaMemcpyAsync(&acc, d_f.get(), sizeof acc, cudaMemcpyDeviceToHost, h->stream));
  if (ebfmi) CK(cudaMemcpyAsync(ebfmi, d_f.get() + 1, sizeof(double) * B, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  if (depth_counts) for (int i = 0; i < 33; ++i) depth_counts[i] = (int64_t)cnt[i];
  if (termination_counts) for (int i = 0; i < 3; ++i) termination_counts[i] = (int64_t)cnt[33 + i];
  if (steps_sum) *steps_sum = (int64_t)cnt[36];
  if (acceptance_sum) *acceptance_sum = acc;
  return DHMC_OK;
}

// split-R̂ and ESS of every (group, parameter): groups of K chains by global id (K = 0: all local chains form one group),
// outputs rhat / ess [D, P] column-major; a group without local chains gets NaN.
static int ess_rhat_groups(dhmc_handle* h, const double* draws_dev, int32_t N, int32_t max_lag, int64_t K, int P, double* rhat,
                           double* ess) {
  CK(cudaSetDevice(h->cfg.device));
  const int D = (int)h->cfg.dim, B = (int)h->cfg.n_chains, n = N / 2;
  const int64_t off = K ? h->cfg.chain_offset : 0;
  int L = max_lag > 0 ? max_lag : 64;
  if (L > n - 2) L = n - 2;
  if (L < 1) L = 1;
  const size_t PD = (size_t)P * D;
  DeviceArray<double> d_pilot, d_acc;
  CK(d_pilot.alloc(PD));
  CK(d_acc.alloc(PD * (L + 3)));
  CK(cudaMemsetAsync(d_acc.get(), 0, sizeof(double) * PD * (L + 3), h->stream));
  k_pilot_mean<<<(unsigned)((PD + 127) / 128), 128, 0, h->stream>>>(draws_dev, n, N, D, B, K, off, P, d_pilot.get());
  k_ess_rhat<<<h->sm_count * 8, 256, 0, h->stream>>>(draws_dev, N, n, D, B, K, off, L, d_pilot.get(), d_acc.get());
  h->launches += 2;
  std::vector<double> acc(PD * (L + 3));
  CK(cudaMemcpyAsync(acc.data(), d_acc.get(), sizeof(double) * acc.size(), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  const double dn = (double)n;
  for (int g = 0; g < P; ++g) {
    // local chains of group g: [g·K, (g+1)·K) ∩ [off, off + B)
    const int64_t lo = K ? std::max<int64_t>((int64_t)g * K, off) : 0, hi = K ? std::min<int64_t>((int64_t)(g + 1) * K, off + B) : B;
    const double m = 2.0 * (double)std::max<int64_t>(hi - lo, 0);
    for (int d = 0; d < D; ++d) {
      const size_t o = (size_t)g * D + d;
      if (m == 0) { if (rhat) rhat[o] = dm_nan(); if (ess) ess[o] = dm_nan(); continue; }
      const double* a = &acc[o * (L + 3)];
      const double mean_var = a[2] / m * dn / (dn - 1.0);                    // W: mean within-sequence variance (n − 1)
      const double var_means = m > 1 ? (a[1] - a[0] * a[0] / m) / (m - 1.0) : 0.0;
      const double var_plus = mean_var * (dn - 1.0) / dn + var_means;        // (n−1)/n·W + B/n
      if (rhat) rhat[o] = std::sqrt(var_plus / mean_var);
      if (ess && !(var_plus > 0.0)) {
        ess[o] = dm_nan();   // every sequence constant at one value: ρ̂ is 0/0 (MCMCDiagnosticTools returns NaN too)
      } else if (ess) {
        // Geyer's initial monotone sequence on ρ̂_t = 1 − (W − mean acov_t) / var⁺, pairs (ρ̂_2k + ρ̂_2k+1)
        double tau = 0.0, prev = 1e300;
        for (int t = 0; t + 1 <= L; t += 2) {
          const double r0 = 1.0 - (mean_var - a[2 + t] / m) / var_plus, r1 = 1.0 - (mean_var - a[3 + t] / m) / var_plus;
          double pair = r0 + r1;
          if (!(pair > 0.0)) break;
          if (pair > prev) pair = prev;
          prev = pair;
          tau += 2.0 * pair;
        }
        tau -= 1.0;
        if (tau < 1.0 / std::log10(m * dn)) tau = 1.0 / std::log10(m * dn);   // cap of the super-efficient case (Stan: ESS ≤ S·log10 S)
        ess[o] = m * dn / tau;
      }
    }
  }
  return DHMC_OK;
}
int dhmc_ess_rhat_dev(dhmc_handle* h, const double* draws_dev, int32_t N, int32_t max_lag, double* rhat, double* ess) {
  if (!h || !draws_dev || N < 4 || (!rhat && !ess)) return DHMC_EARG;
  return ess_rhat_groups(h, draws_dev, N, max_lag, 0, 1, rhat, ess);
}
int dhmc_ess_rhat_problems_dev(dhmc_handle* h, const double* draws_dev, int32_t N, int32_t max_lag, double* rhat, double* ess) {
  if (!h || !draws_dev || N < 4 || (!rhat && !ess)) return DHMC_EARG;
  if (!h->batch_k) { h->err = "dhmc_ess_rhat_problems_dev: the handle holds no problem batch (dhmc_set_problems)"; return DHMC_EARG; }
  return ess_rhat_groups(h, draws_dev, N, max_lag, h->batch_k, (int)h->batch_p, rhat, ess);
}
int dhmc_acceptance_quantiles_dev(dhmc_handle* h, const dhmc_tree_stats* stats_dev, int32_t N, const double* probs,
                                  int32_t nprobs, double* out) {
  if (!h || !stats_dev || N < 1 || !probs || nprobs < 1 || !out) return DHMC_EARG;
  CK(cudaSetDevice(h->cfg.device));
  constexpr int BINS = 4096;
  DeviceArray<unsigned long long> d_hist;
  CK(d_hist.alloc(BINS + 1));
  CK(cudaMemsetAsync(d_hist.get(), 0, sizeof(unsigned long long) * (BINS + 1), h->stream));
  const size_t n = (size_t)N * (size_t)h->cfg.n_chains;
  k_acceptance_hist<<<h->sm_count * 8, 256, 0, h->stream>>>(stats_dev, n, d_hist.get(), BINS);
  h->launches += 1;
  std::vector<unsigned long long> hist(BINS + 1);
  CK(cudaMemcpyAsync(hist.data(), d_hist.get(), sizeof(unsigned long long) * hist.size(), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  // the non-NaN rates in bins 1 … BINS of the grid (0, 1, BINS), both tails empty: every order statistic is placed
  // strictly inside its bin, so less than one bin width from the true value
  std::vector<unsigned long long> cum(BINS + 2, 0);
  for (int b = 0; b < BINS; ++b) cum[b + 1] = cum[b] + hist[b];
  cum[BINS + 1] = cum[BINS];
  for (int k = 0; k < nprobs; ++k) {
    if (!(probs[k] >= 0.0 && probs[k] <= 1.0)) { h->err = "0 ≤ p ≤ 1"; return DHMC_EARG; }
    double q_lo, q_hi;
    binned_quantile(cum.data(), BINS, 0.0, 1.0, probs[k], out + k, &q_lo, &q_hi);
  }
  return DHMC_OK;
}

int dhmc_last_total_steps(dhmc_handle* h, int64_t* steps) { if (!h || !steps) return DHMC_EARG; *steps = h->last_steps; return DHMC_OK; }
int dhmc_last_kernel_ms(dhmc_handle* h, double* ms) { if (!h || !ms) return DHMC_EARG; *ms = h->last_ms; return DHMC_OK; }
int dhmc_kernel_launches(dhmc_handle* h, int64_t* n) { if (!h || !n) return DHMC_EARG; *n = h->launches; return DHMC_OK; }
#if defined(DHMC_PHASE_CLOCKS)
// Leaf profile of the diagnostic build (benchmarks/leaf_phases.py): out[kPhCount] = the counters summed over all CTAs since the
// last reset (clock cycles of thread 0 of each CTA per phase, and the number of leaves); reset != 0 zeroes them afterwards.
int dhmc_phase_clocks(dhmc_handle* h, uint64_t* out, int reset) {
  if (!h || !out) return DHMC_EARG;
  const size_t n = (size_t)kPhCount * 32 * (size_t)h->sm_count;
  std::vector<unsigned long long> v(n);
  CK(cudaDeviceSynchronize());
  CK(cudaMemcpy(v.data(), h->phase_clocks.get(), sizeof(unsigned long long) * n, cudaMemcpyDeviceToHost));
  for (int k = 0; k < kPhCount; ++k) out[k] = 0;
  for (size_t i = 0; i < n; ++i) out[i % kPhCount] += v[i];
  if (reset) CK(cudaMemset(h->phase_clocks.get(), 0, sizeof(unsigned long long) * n));
  return DHMC_OK;
}
#endif

// ---- multi-GPU (SURVEY §8e): chains are sharded over ranks with no data-path collective; the one exchange is the
// all-gather of (thinned) draws / final positions at the end.  One process per GPU; rank 0 creates the id, the host
// program (Julia: MPI / Distributed; Python: torch.distributed) carries its 128 bytes to the other ranks.
// NCCL is bound with dlopen("libnccl.so.2") at the first dhmc_comm_* call instead of a DT_NEEDED entry: a host process
// that already carries an NCCL (e.g. the copy bundled with PyTorch) must end up with ONE libnccl, and a process that never
// shards pays nothing.  The soname lookup returns the copy that is already loaded, else the system library.
struct nccl_api {
  decltype(&::ncclGetUniqueId) GetUniqueId = nullptr;
  decltype(&::ncclCommInitRank) CommInitRank = nullptr;
  decltype(&::ncclCommDestroy) CommDestroy = nullptr;
  decltype(&::ncclAllGather) AllGather = nullptr;
  decltype(&::ncclGetErrorString) GetErrorString = nullptr;
  decltype(&::ncclGetVersion) GetVersion = nullptr;
  bool ok = false;
  std::string why;
};
static nccl_api& nccl() {
  static nccl_api api;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!lib) lib = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!lib) { api.why = std::string("dlopen(libnccl.so.2): ") + dlerror(); return api; }
#define DHMC_NCCL_SYM(name) api.name = reinterpret_cast<decltype(api.name)>(dlsym(lib, "nccl" #name)); if (!api.name) { api.why = "libnccl lacks nccl" #name; return api; }
    DHMC_NCCL_SYM(GetUniqueId) DHMC_NCCL_SYM(CommInitRank) DHMC_NCCL_SYM(CommDestroy) DHMC_NCCL_SYM(AllGather)
    DHMC_NCCL_SYM(GetErrorString) DHMC_NCCL_SYM(GetVersion)
#undef DHMC_NCCL_SYM
    api.ok = true;
  }
  return api;
}
int dhmc_comm_unique_id(void* id128) {
  if (!id128) return DHMC_EARG;
  static_assert(sizeof(ncclUniqueId) == DHMC_COMM_ID_BYTES, "ncclUniqueId is 128 bytes");
  if (!nccl().ok) { g_create_err = nccl().why; return DHMC_ENCCL; }
  ncclUniqueId id;
  if (nccl().GetUniqueId(&id) != ncclSuccess) { g_create_err = "ncclGetUniqueId failed"; return DHMC_ENCCL; }
  std::memcpy(id128, &id, sizeof id);
  return DHMC_OK;
}
#define CKN(call)                                                                     \
  do {                                                                                \
    if (!nccl().ok) { h->err = nccl().why; return DHMC_ENCCL; }                       \
    ncclResult_t r_ = (call);                                                         \
    if (r_ != ncclSuccess) { h->err = std::string(#call) + ": " + nccl().GetErrorString(r_); return DHMC_ENCCL; } \
  } while (0)
int dhmc_comm_init(dhmc_handle* h, int32_t nranks, int32_t rank, const void* id128) {
  if (!h || !id128 || nranks < 1 || rank < 0 || rank >= nranks) return DHMC_EARG;
  if (h->comm) { h->err = "communicator already initialised"; return DHMC_EARG; }
  CK(cudaSetDevice(h->cfg.device));
  ncclUniqueId id;
  std::memcpy(&id, id128, sizeof id);
  CKN(nccl().CommInitRank(&h->comm, nranks, id, rank));
  h->comm_nranks = nranks; h->comm_rank = rank;
  return DHMC_OK;
}
int dhmc_comm_destroy(dhmc_handle* h) {
  if (!h) return DHMC_EARG;
  if (h->comm) { nccl().CommDestroy(h->comm); h->comm = nullptr; h->comm_nranks = 1; h->comm_rank = 0; }
  return DHMC_OK;
}
// ncclAllGather of `count` doubles per rank, DEVICE pointers (e.g. the draws buffer of dhmc_mcmc_dev): recv is
// [nranks][count]; rank order = global chain order, so recv is the [D, N, B·nranks] column-major draws array.
int dhmc_allgather_dev(dhmc_handle* h, const double* send_dev, double* recv_dev, size_t count) {
  if (!h || !send_dev || !recv_dev) return DHMC_EARG;
  if (!h->comm) { h->err = "dhmc_comm_init first"; return DHMC_EARG; }
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaEventRecord(h->ev0, h->stream));
  CKN(nccl().AllGather(send_dev, recv_dev, count, ncclDouble, h->comm, h->stream));
  CK(cudaEventRecord(h->ev1, h->stream));
  CK(cudaEventSynchronize(h->ev1));
  float ms = 0;
  CK(cudaEventElapsedTime(&ms, h->ev0, h->ev1));
  h->last_comm_ms = ms;
  return DHMC_OK;
}
// The current position of every chain of every rank: recv_dev [D, B·nranks] (DEVICE), one all-gather of D·B doubles per rank.
int dhmc_allgather_positions_dev(dhmc_handle* h, double* recv_dev) {
  if (!h || !recv_dev) return DHMC_EARG;
  return dhmc_allgather_dev(h, h->q.get(), recv_dev, (size_t)h->cfg.n_chains * (size_t)h->cfg.dim);
}
int dhmc_last_comm_ms(dhmc_handle* h, double* ms) { if (!h || !ms) return DHMC_EARG; *ms = h->last_comm_ms; return DHMC_OK; }
#undef CKN

}  // extern "C"
