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
struct dhmc_handle {
  dhmc_config cfg;
  int T = 0, W = 0, EPL = 0;
  int G = 1;                        // chains per CTA of the persistent kernels (packed chain groups)
  bool deep = false;                // max_depth > 12: kernels whose slot pool spills past 64 slots (part 3), one chain per CTA
  size_t stride = 0;
  int n_slots = 0, n_sm = 0, grid = 0, sm_count = 0, light_grid = 0;
  int levels = 13, ntab = 64;       // stack entries per warp (max_depth + 1), slot-table entries (>= n_slots)
  size_t smem_bytes = 0, smem_light = 0;
  size_t scratch_per_cta = 0;
  cudaStream_t stream = nullptr, copy_stream = nullptr, h2d_stream = nullptr;
  cudaEvent_t h2d_ev[16] = {};
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  cudaEvent_t chunk_ev[16] = {};
  cudaEvent_t copy_ev[16] = {};
  bool trace = false;
  double* tmp_b = nullptr;          // [B] scratch (phase log densities) and [B·D] momentum override / [D·D] broadcast source,
  double* tmp_bd = nullptr;         // allocated once instead of per call
  unsigned* tmp_dir = nullptr;
  size_t tmp_bd_doubles = 0;
  std::vector<void*> registered;    // caller buffers page-locked on the fly (direct host writes of draws that exceed HBM)
  void* stage[4] = {nullptr, nullptr, nullptr, nullptr};   // grow-only device staging for host outputs
  size_t stage_bytes[4] = {0, 0, 0, 0};
  double *q = nullptr, *g = nullptr, *lq = nullptr, *p = nullptr, *minv = nullptr, *eps = nullptr;
  double* mparams = nullptr;
  int* status = nullptr;
  double* scratch = nullptr;
#if defined(DHMC_PHASE_CLOCKS)
  unsigned long long* phase_clocks = nullptr;   // leaf profile: kPhCount counters for each of up to 32 CTAs per SM
#endif
  unsigned* counter = nullptr;
  unsigned long long* total_steps = nullptr;
  uint32_t t = 0;
  int64_t launches = 0;
  double last_ms = 0;
  int64_t last_steps = 0;
  bool has_position = false, has_eps = false;
  bool dense = false;               // κ is a Symmetric (dense) metric
  double *minv_dense = nullptr, *wt = nullptr, *covt = nullptr, *dense_tmp = nullptr;
  double* mean_pool = nullptr;      // pooled Symmetric stages: window mean of every chain [B][D]
  bool pooled = false;              // the dense metric is shared by every group of 8 chains
  double* minv_pad = nullptr;       // packed groups on the tensor cores: zero-padded row blocks of every chain's M⁻¹
  double *lX = nullptr, *lXt = nullptr, *ly = nullptr, *lr = nullptr;   // logistic regression
  double* lXp = nullptr;            // … zero-padded row blocks of X for the tensor-core likelihood
  int lN = 0, lLd = 0;              // (a batch: lN is the largest N, the row length of the residual scratch lr)
  // problem batch (dhmc_set_problems / _ragged): chains per problem (0 = one problem), problems, and the device table of
  // per-problem descriptors (where each problem's blocks start in mparams, lX, lXt, ly, lXp; its N and leading dimension)
  int64_t batch_k = 0, batch_p = 0;
  ProblemDesc* problems = nullptr;
  int reg_ctas[2] = {0, 0};         // occupancy of k_nuts (diag, dense)
  size_t smem_sm = 0, smem_cta_max = 0;
  ncclComm_t comm = nullptr;        // multi-GPU: one communicator per handle (dhmc_comm_init)
  int comm_nranks = 1, comm_rank = 0;
  double last_comm_ms = 0;
  // streaming summary (dhmc_mcmc_summary): grow-only device arena of the SummaryArgs arrays, and the struct itself
  void* sum_buf = nullptr;
  size_t sum_bytes = 0;
  SummaryArgs* sum_args = nullptr;
  std::string err;
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
  return h->minv_dense || h->cfg.family == DHMC_FAMILY_LOGISTIC || h->cfg.family == DHMC_FAMILY_USER;
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
// of the persistent kernels (packed groups keep theirs in shared memory)
static size_t lr_rows(const dhmc_handle* h) {
  return std::max<size_t>(h->G > 1 ? 0 : (size_t)h->grid, (size_t)h->light_grid);
}

// groups of the persistent kernels' reduction buffer (DeviceBackend::kFused): the last leaf of a depth-d adjacent tree carries
// d stack merges and the doubling check, the first two in group 0, so max_depth groups (two at max_depth 1)
static int red_groups(const dhmc_handle* h) {
  return !h->dense && h->G == 1 && h->cfg.family != DHMC_FAMILY_USER ? std::max(2, h->cfg.max_depth) : 1;
}

// Plan the persistent kernels for the current metric kind: CTAs per SM (register
// limited), how many slots fit in shared memory, and the global scratch arena.
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
  h->smem_light = smem_layout(h->W, 0, slot_doubles, xs).total;      // light kernels: standard layout
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
  h->n_sm = (int)n_sm;
  h->smem_bytes = heavy_smem(h->n_sm);
  h->grid = (int)std::min<size_t>((size_t)ctas * h->sm_count, (B + G - 1) / G);
  h->light_grid = (int)std::min<size_t>((size_t)h->sm_count * 16, B);
  h->scratch_per_cta = (size_t)(h->n_slots - h->n_sm) * slot_doubles;
  cudaFree(h->scratch); h->scratch = nullptr;
  CK(cudaMalloc(&h->scratch, sizeof(double) * h->scratch_per_cta * (size_t)h->grid * (size_t)G));
  // (an access-policy window over the slot arena was tried and rejected: slower at C2)
  if (h->lN) {   // residual scratch of the logistic family follows the grid
    cudaFree(h->lr); h->lr = nullptr;
    CK(cudaMalloc(&h->lr, sizeof(double) * (size_t)h->lN * lr_rows(h)));
  }
  return DHMC_OK;
}

static int ensure_tmp(dhmc_handle* h, size_t doubles) {      // grow-only device scratch shared by the small entry points
  if (!h->tmp_b) CK(cudaMalloc(&h->tmp_b, sizeof(double) * (size_t)h->cfg.n_chains));
  if (!h->tmp_dir) CK(cudaMalloc(&h->tmp_dir, sizeof(unsigned) * (size_t)h->cfg.n_chains));
  if (doubles > h->tmp_bd_doubles) {
    cudaFree(h->tmp_bd); h->tmp_bd = nullptr; h->tmp_bd_doubles = 0;
    CK(cudaMalloc(&h->tmp_bd, sizeof(double) * doubles));
    h->tmp_bd_doubles = doubles;
  }
  return DHMC_OK;
}

static KArgs base_args(dhmc_handle* h) {
  KArgs a;
  std::memset(&a, 0, sizeof(a));
  a.D = (int)h->cfg.dim; a.B = (int)h->cfg.n_chains; a.T = h->T; a.W = h->W;
  a.seed = h->cfg.seed; a.chain_offset = h->cfg.chain_offset;
  a.q = h->q; a.g = h->g; a.lq = h->lq; a.p = h->p; a.minv = h->minv; a.eps = h->eps;
  a.mparams = h->mparams; a.status = h->status;
  a.max_depth = h->cfg.max_depth; a.min_delta = h->cfg.min_delta;
  a.t0 = h->t;
  a.scratch = h->scratch; a.scratch_per_cta = h->scratch_per_cta;
#if defined(DHMC_PHASE_CLOCKS)
  a.phase_clocks = h->phase_clocks;
#endif
  a.n_sm = h->n_sm; a.n_slots = h->n_slots; a.stride = h->stride * (h->dense ? 2 : 1);
  a.levels = h->levels; a.ntab = h->ntab;
  a.red_groups = red_groups(h);
  a.counter = h->counter; a.total_steps = h->total_steps;
  a.chain_begin = 0; a.chain_end = (int)h->cfg.n_chains;
  a.minv_dense = h->minv_dense; a.wt = h->wt; a.covt = nullptr; a.minv_pad = h->minv_pad; a.mean_out = nullptr; a.pooled = h->pooled ? 1 : 0;
  a.xs_doubles = needs_staging(h) ? (int)((size_t)h->T * h->EPL) : 0;
  a.lX = h->lX; a.lXt = h->lXt; a.ly = h->ly; a.lr = h->lr; a.lN = h->lN; a.lLd = h->lLd; a.lXp = h->lXp;
  a.batch_k = (int)h->batch_k; a.problems = h->problems;
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
  if (!heavy) { a.n_sm = 0; a.red_groups = 1; }
  const size_t smem = heavy ? h->smem_bytes : smem_layout(h->W, 0, a.stride, (size_t)a.xs_doubles).total;
  int grid = heavy ? h->grid : h->light_grid;
  const int G = heavy ? h->G : 1;
  if (heavy) grid = std::max(1, std::min(grid, (a.chain_end - a.chain_begin + G - 1) / G));
  if (heavy) {
    CK(cudaMemsetAsync(h->counter, 0, sizeof(unsigned), h->stream));
    if (reset_steps) CK(cudaMemsetAsync(h->total_steps, 0, sizeof(unsigned long long), h->stream));
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
  CK(cudaMemcpy(st.data(), h->status, sizeof(int) * B, cudaMemcpyDeviceToHost));
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
int dhmc_comm_destroy(dhmc_handle* h);

int dhmc_destroy(dhmc_handle* h) {
  if (!h) return DHMC_OK;
  cudaSetDevice(h->cfg.device);
  cudaFree(h->q); cudaFree(h->g); cudaFree(h->lq); cudaFree(h->p); cudaFree(h->minv); cudaFree(h->eps);
  cudaFree(h->mparams); cudaFree(h->status); cudaFree(h->scratch); cudaFree(h->counter);
#if defined(DHMC_PHASE_CLOCKS)
  cudaFree(h->phase_clocks);
#endif
  cudaFree(h->total_steps);
  cudaFree(h->minv_dense); cudaFree(h->wt); cudaFree(h->covt); cudaFree(h->dense_tmp); cudaFree(h->minv_pad); cudaFree(h->mean_pool);
  cudaFree(h->lX); cudaFree(h->lXt); cudaFree(h->ly); cudaFree(h->lr); cudaFree(h->lXp); cudaFree(h->problems);
  cudaFree(h->tmp_b); cudaFree(h->tmp_bd); cudaFree(h->tmp_dir);
  cudaFree(h->sum_buf); cudaFree(h->sum_args);
  for (void* r : h->registered) cudaHostUnregister(r);
  if (h->comm) dhmc_comm_destroy(h);
  if (h->ev0) cudaEventDestroy(h->ev0);
  if (h->ev1) cudaEventDestroy(h->ev1);
  for (auto& e : h->chunk_ev) if (e) cudaEventDestroy(e);
  for (auto& e : h->copy_ev) if (e) cudaEventDestroy(e);
  for (auto& b : h->stage) cudaFree(b);
  if (h->copy_stream) cudaStreamDestroy(h->copy_stream);
  for (auto& e : h->h2d_ev) if (e) cudaEventDestroy(e);
  if (h->h2d_stream) cudaStreamDestroy(h->h2d_stream);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;
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
  int ndev = 0;
  cudaError_t ce = cudaGetDeviceCount(&ndev);
  if (ce != cudaSuccess || ndev == 0) {
    g_create_err = std::string("no CUDA device: ") + (ce != cudaSuccess ? cudaGetErrorString(ce) : "device count 0") +
                   " (libdhmc_b200 has no CPU fallback)";
    return DHMC_ECUDA;
  }
  if (cfg->device < 0 || cfg->device >= ndev) { g_create_err = "bad device ordinal"; return DHMC_EARG; }
  dhmc_handle* h = new dhmc_handle();
  h->cfg = *cfg; h->T = T; h->W = T / 32; h->EPL = EPL; h->stride = (size_t)T * EPL; h->G = pack; h->deep = deep;
  h->n_slots = slots_needed(cfg->max_depth);
  h->levels = deep ? cfg->max_depth + 1 : kStdLevels;        // deep persistent kernels size their stack / slot table at run time
  h->ntab = deep ? std::max(kStdTab, (h->n_slots + 7) & ~7) : kStdTab;
  auto fail = [&](int rc) { g_create_err = h->err; dhmc_destroy(h); return rc; };
#define CKC(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { h->err = std::string(#call) + ": " + cudaGetErrorString(e_); return fail(e_ == cudaErrorMemoryAllocation ? DHMC_ENOMEM : DHMC_ECUDA); } } while (0)
  CKC(cudaSetDevice(cfg->device));
  cudaDeviceProp prop;
  CKC(cudaGetDeviceProperties(&prop, cfg->device));
  h->sm_count = prop.multiProcessorCount;
#if defined(DHMC_PHASE_CLOCKS)
  CKC(cudaMalloc(&h->phase_clocks, sizeof(unsigned long long) * kPhCount * 32 * (size_t)h->sm_count));
  CKC(cudaMemset(h->phase_clocks, 0, sizeof(unsigned long long) * kPhCount * 32 * (size_t)h->sm_count));
#endif
  CKC(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
  CKC(cudaStreamCreateWithFlags(&h->copy_stream, cudaStreamNonBlocking));
  CKC(cudaStreamCreateWithFlags(&h->h2d_stream, cudaStreamNonBlocking));
  const bool trace = std::getenv("DHMC_TRACE") != nullptr;      // DHMC_TRACE=1: timeline of the chunk pipeline on stderr
  for (auto& e : h->h2d_ev) CKC(cudaEventCreateWithFlags(&e, trace ? cudaEventDefault : cudaEventDisableTiming));
  for (auto& e : h->chunk_ev) CKC(cudaEventCreateWithFlags(&e, trace ? cudaEventDefault : cudaEventDisableTiming));
  for (auto& e : h->copy_ev) CKC(cudaEventCreateWithFlags(&e, trace ? cudaEventDefault : cudaEventDisableTiming));
  h->trace = trace;
  CKC(cudaEventCreate(&h->ev0));
  CKC(cudaEventCreate(&h->ev1));
  const size_t B = (size_t)cfg->n_chains, D = (size_t)cfg->dim;
  CKC(cudaMalloc(&h->q, sizeof(double) * B * D));
  CKC(cudaMalloc(&h->g, sizeof(double) * B * D));
  CKC(cudaMalloc(&h->p, sizeof(double) * B * D));
  CKC(cudaMalloc(&h->minv, sizeof(double) * B * D));
  CKC(cudaMalloc(&h->lq, sizeof(double) * B));
  CKC(cudaMalloc(&h->eps, sizeof(double) * B));
  CKC(cudaMalloc(&h->status, sizeof(int) * B));
  CKC(cudaMalloc(&h->counter, sizeof(unsigned)));
  CKC(cudaMalloc(&h->total_steps, sizeof(unsigned long long)));
  CKC(cudaMalloc(&h->mparams, sizeof(double) * 2 * D));
  CKC(cudaMemsetAsync(h->q, 0, sizeof(double) * B * D, h->stream));
  CKC(cudaMemsetAsync(h->g, 0, sizeof(double) * B * D, h->stream));
  CKC(cudaMemsetAsync(h->p, 0, sizeof(double) * B * D, h->stream));
  CKC(cudaMemsetAsync(h->lq, 0, sizeof(double) * B, h->stream));
  CKC(cudaMemsetAsync(h->eps, 0, sizeof(double) * B, h->stream));
  CKC(cudaMemsetAsync(h->status, 0, sizeof(int) * B, h->stream));
  CKC(cudaMemsetAsync(h->mparams, 0, sizeof(double) * 2 * D, h->stream));
  k_fill<<<1024, 256, 0, h->stream>>>(h->minv, 1.0, B * D);   // κ = GaussianKineticEnergy(D), mcmc.jl:130
  h->launches += 1;

  h->smem_sm = (size_t)prop.sharedMemPerMultiprocessor;          // 228 KB
  h->smem_cta_max = (size_t)prop.sharedMemPerBlockOptin;         // 227 KB
  {
    int rcp = plan(h);
    if (rcp != DHMC_OK) return fail(rcp);
  }
  CKC(cudaStreamSynchronize(h->stream));
#undef CKC
  *out = h;
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
  double *mp = nullptr, *X = nullptr, *Xt = nullptr, *y = nullptr, *Xp = nullptr, *lr = nullptr;
  ProblemDesc* dd = nullptr;
  auto drop = [&] { cudaFree(mp); cudaFree(X); cudaFree(Xt); cudaFree(y); cudaFree(Xp); cudaFree(lr); cudaFree(dd); };
#define CKB(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { h->err = std::string(#call) + ": " + cudaGetErrorString(e_); \
    cudaStreamSynchronize(h->stream); drop(); return e_ == cudaErrorMemoryAllocation ? DHMC_ENOMEM : DHMC_ECUDA; } } while (0)
  if (K) {
    CKB(cudaMalloc(&dd, sizeof(ProblemDesc) * Pz));
    CKB(cudaMemcpyAsync(dd, desc.data(), sizeof(ProblemDesc) * Pz, cudaMemcpyHostToDevice, h->stream));
  }
  if (fam == DHMC_FAMILY_LOGISTIC) {
    // per problem: X [N][D], Xᵀ [D][ld], y [N] and, for packed groups, the zero-padded row blocks [rows][xs]; one residual
    // scratch of rows of the largest N
    CKB(cudaMalloc(&X, sizeof(double) * tX));
    CKB(cudaMalloc(&Xt, sizeof(double) * tXt));
    CKB(cudaMalloc(&y, sizeof(double) * ty));
    CKB(cudaMalloc(&lr, sizeof(double) * maxN * lr_rows(h)));
    if (h->G > 1) CKB(cudaMalloc(&Xp, sizeof(double) * tXp));
    for (size_t p = 0; p < Pz; ++p) {
      const double* blk = params + offs[p];
      const ProblemDesc& d = desc[p];
      const size_t N = (size_t)d.N;
      CKB(cudaMemcpyAsync(X + d.X, blk + 1, sizeof(double) * N * D, cudaMemcpyHostToDevice, h->stream));
      CKB(cudaMemcpyAsync(y + d.y, blk + 1 + N * D, sizeof(double) * N, cudaMemcpyHostToDevice, h->stream));
      k_transpose<<<1024, 256, 0, h->stream>>>(X + d.X, Xt + d.Xt, N, D, (size_t)d.ld);
      if (Xp) k_pad_rows<<<1024, 256, 0, h->stream>>>(X + d.X, Xp + d.Xp, N, D, tma_rows(N), xs, 1);
      h->launches += Xp ? 2 : 1;
    }
  } else if (fam == DHMC_FAMILY_DIAG_NORMAL || fam == DHMC_FAMILY_USER) {   // (STD_NORMAL and FUNNEL have no parameters)
    // mparams is never null, also for a USER model without parameters
    CKB(cudaMalloc(&mp, sizeof(double) * std::max<size_t>(offs[Pz], 1)));
    if (offs[Pz]) CKB(cudaMemcpyAsync(mp, params, sizeof(double) * offs[Pz], cudaMemcpyHostToDevice, h->stream));
  }
  CKB(cudaGetLastError());
  CKB(cudaStreamSynchronize(h->stream));
#undef CKB
  if (fam == DHMC_FAMILY_LOGISTIC) {
    cudaFree(h->lX); cudaFree(h->lXt); cudaFree(h->ly); cudaFree(h->lr); cudaFree(h->lXp);
    h->lX = X; h->lXt = Xt; h->ly = y; h->lr = lr; h->lXp = Xp;
    h->lN = (int)maxN; h->lLd = desc[0].ld;    // a chain's own N and ld come from its descriptor
  } else if (mp) {
    cudaFree(h->mparams);
    h->mparams = mp;
  }
  cudaFree(h->problems);
  h->problems = dd;
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
  CK(cudaMemsetAsync(h->status, 0, sizeof(int) * (size_t)h->cfg.n_chains, h->stream));
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
  CK(cudaMemcpyAsync(h->q, q, sizeof(double) * (size_t)h->cfg.n_chains * h->cfg.dim, cudaMemcpyHostToDevice, h->stream));
  return eval_position(h, false);
}
int dhmc_random_position(dhmc_handle* h) {
  if (!h) return DHMC_EARG;
  CK(cudaSetDevice(h->cfg.device));
  return eval_position(h, true);
}

static int ensure_dense(dhmc_handle* h) {
  if (h->minv_dense) return DHMC_OK;

  const size_t B = (size_t)h->cfg.n_chains, dd = (size_t)h->cfg.dim * h->cfg.dim;
  CK(cudaMalloc(&h->minv_dense, sizeof(double) * B * dd));
  CK(cudaMalloc(&h->wt, sizeof(double) * B * dd));
  CK(cudaMalloc(&h->covt, sizeof(double) * B * dd));
  CK(cudaMalloc(&h->dense_tmp, sizeof(double) * 3 * dd * (size_t)factor_grid(h)));
  CK(cudaMemsetAsync(h->wt, 0, sizeof(double) * B * dd, h->stream));
  if (h->G > 1)     // [B][⌈D/32⌉·32][XS]: one bulk copy per 32-row block (coop_matvec_tma)
    CK(cudaMalloc(&h->minv_pad, sizeof(double) * B * tma_rows((size_t)h->cfg.dim) * (size_t)tma_xs((int)h->cfg.dim)));
  // re-planned whatever the metric kind: with the dense arrays allocated, the shared-memory layout carries the staging
  // vector (needs_staging) also for the diagonal kernels
  return plan(h);
}
// The metric kind of the handle's kernels: the persistent kernels are re-planned when the slot width (dense) changes.
static int set_metric_kind(dhmc_handle* h, bool dense, bool pooled) {
  h->pooled = pooled;
  if (h->dense == dense) return DHMC_OK;
  h->dense = dense;
  return plan(h);
}
// κ = GaussianKineticEnergy(Symmetric M⁻¹): W = cholesky(inv(M⁻¹)).L on device, then switch
// the handle to the dense kernels (pooled: M⁻¹ is shared by every group of 8 chains).
static int factor_and_switch(dhmc_handle* h, bool pooled) {
  const size_t B = (size_t)h->cfg.n_chains, D = (size_t)h->cfg.dim;
  CK(cudaMemsetAsync(h->status, 0, sizeof(int) * B, h->stream));
  k_dense_factor<<<factor_grid(h), 128, 0, h->stream>>>(h->minv_dense, h->wt, h->dense_tmp, h->status, (int)D, (int)B);
  h->launches += 1;
  if (h->minv_pad) {
    k_pad_rows<<<2048, 256, 0, h->stream>>>(h->minv_dense, h->minv_pad, D, D, tma_rows(D), (size_t)tma_xs((int)D), B);
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
    int rct = ensure_tmp(h, dd);
    if (rct != DHMC_OK) return rct;
    CK(cudaMemcpyAsync(h->tmp_bd, minv, sizeof(double) * dd, cudaMemcpyHostToDevice, h->stream));
    k_broadcast<<<1024, 256, 0, h->stream>>>(h->minv_dense, h->tmp_bd, dd, B);
    h->launches += 1;
    CK(cudaStreamSynchronize(h->stream));
  } else {
    CK(cudaMemcpyAsync(h->minv_dense, minv, sizeof(double) * B * dd, cudaMemcpyHostToDevice, h->stream));
  }
  return factor_and_switch(h, false);
}
int dhmc_get_metric_dense(dhmc_handle* h, double* minv) {
  if (!h || !minv) return DHMC_EARG;
  if (!h->dense) { h->err = "the current metric is diagonal"; return DHMC_EARG; }
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaMemcpy(minv, h->minv_dense, sizeof(double) * (size_t)h->cfg.n_chains * h->cfg.dim * h->cfg.dim, cudaMemcpyDeviceToHost));
  return DHMC_OK;
}
int dhmc_metric_is_dense(dhmc_handle* h, int32_t* dense) { if (!h || !dense) return DHMC_EARG; *dense = h->dense ? 1 : 0; return DHMC_OK; }

int dhmc_set_metric(dhmc_handle* h, const double* minv, int broadcast) {
  if (!h) return DHMC_EARG;
  CK(cudaSetDevice(h->cfg.device));
  const size_t B = (size_t)h->cfg.n_chains, D = (size_t)h->cfg.dim;
  if (!minv) {
    k_fill<<<1024, 256, 0, h->stream>>>(h->minv, 1.0, B * D);
  } else if (broadcast) {
    int rct = ensure_tmp(h, D);
    if (rct != DHMC_OK) return rct;
    CK(cudaMemcpyAsync(h->tmp_bd, minv, sizeof(double) * D, cudaMemcpyHostToDevice, h->stream));
    k_broadcast<<<1024, 256, 0, h->stream>>>(h->minv, h->tmp_bd, D, B);
    CK(cudaStreamSynchronize(h->stream));
  } else {
    CK(cudaMemcpyAsync(h->minv, minv, sizeof(double) * B * D, cudaMemcpyHostToDevice, h->stream));
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
    k_fill<<<256, 256, 0, h->stream>>>(h->eps, eps[0], B);
    h->launches += 1;
  } else {
    for (size_t i = 0; i < B; ++i) if (!(eps[i] > 0)) { h->err = "ϵ > 0"; return DHMC_EARG; }
    CK(cudaMemcpyAsync(h->eps, eps, sizeof(double) * B, cudaMemcpyHostToDevice, h->stream));
  }
  CK(cudaStreamSynchronize(h->stream));
  h->has_eps = true;
  return DHMC_OK;
}

int dhmc_set_momentum(dhmc_handle* h, const double* p) {
  if (!h || !p) return DHMC_EARG;
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaMemcpyAsync(h->p, p, sizeof(double) * (size_t)h->cfg.n_chains * h->cfg.dim, cudaMemcpyHostToDevice, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return DHMC_OK;
}

int dhmc_get_state(dhmc_handle* h, double* q, double* lq, double* grad, double* minv, double* eps, double* p) {
  if (!h) return DHMC_EARG;
  CK(cudaSetDevice(h->cfg.device));
  const size_t B = (size_t)h->cfg.n_chains, D = (size_t)h->cfg.dim;
  if (q) CK(cudaMemcpyAsync(q, h->q, sizeof(double) * B * D, cudaMemcpyDeviceToHost, h->stream));
  if (grad) CK(cudaMemcpyAsync(grad, h->g, sizeof(double) * B * D, cudaMemcpyDeviceToHost, h->stream));
  if (minv) CK(cudaMemcpyAsync(minv, h->minv, sizeof(double) * B * D, cudaMemcpyDeviceToHost, h->stream));
  if (p) CK(cudaMemcpyAsync(p, h->p, sizeof(double) * B * D, cudaMemcpyDeviceToHost, h->stream));
  if (lq) CK(cudaMemcpyAsync(lq, h->lq, sizeof(double) * B, cudaMemcpyDeviceToHost, h->stream));
  if (eps) CK(cudaMemcpyAsync(eps, h->eps, sizeof(double) * B, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return DHMC_OK;
}

int dhmc_chain_status(dhmc_handle* h, int32_t* status) {
  if (!h || !status) return DHMC_EARG;
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaMemcpy(status, h->status, sizeof(int) * (size_t)h->cfg.n_chains, cudaMemcpyDeviceToHost));
  return DHMC_OK;
}
int dhmc_get_transition_count(dhmc_handle* h, uint32_t* t) { if (!h || !t) return DHMC_EARG; *t = h->t; return DHMC_OK; }
int dhmc_set_transition_count(dhmc_handle* h, uint32_t t) { if (!h) return DHMC_EARG; h->t = t; return DHMC_OK; }

int dhmc_leapfrog(dhmc_handle* h, int32_t n_steps, int32_t sign) {
  if (!h || n_steps < 0) return DHMC_EARG;
  if (!h->has_position || !h->has_eps) { h->err = "dhmc_leapfrog: set position and step size first"; return DHMC_EARG; }
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaMemsetAsync(h->status, 0, sizeof(int) * (size_t)h->cfg.n_chains, h->stream));   // status words describe the current call
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
  int rc = ensure_tmp(h, 0);
  if (rc != DHMC_OK) return rc;
  KArgs a = base_args(h);
  a.out_phase = h->tmp_b;
  rc = launch(h, K_PHASE, a, nullptr, nullptr);
  if (rc != DHMC_OK) return rc;
  CK(cudaMemcpyAsync(out, h->tmp_b, sizeof(double) * B, cudaMemcpyDeviceToHost, h->stream));
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
  CK(cudaMemsetAsync(h->status, 0, sizeof(int) * (size_t)h->cfg.n_chains, h->stream));   // status words describe the current call
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

// common driver of sample_tree / warmup stage / mcmc.
// Host outputs of large runs are pipelined: the chains are cut into chunks, each
// chunk is one k_nuts launch on the compute stream, and its draws/statistics are
// copied D2H on the copy stream while the next chunk computes (pinned host
// buffers make the copies truly asynchronous; pageable ones still work).
static int ensure_stage(dhmc_handle* h, int i, size_t bytes) {
  if (h->stage_bytes[i] >= bytes) return DHMC_OK;
  cudaFree(h->stage[i]); h->stage[i] = nullptr; h->stage_bytes[i] = 0;
  CK(cudaMalloc(&h->stage[i], bytes));
  h->stage_bytes[i] = bytes;
  return DHMC_OK;
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
static int run_nuts(dhmc_handle* h, int N, const AdaptConfig& cfg, double lambda, const double* p_over_host,
                    const uint32_t* dir_over_host, double* posterior, dhmc_tree_stats* stats,
                    double* eps_used, double* logdens, bool outputs_on_device, bool advance_t,
                    const double* q_host = nullptr, int thin = 1, bool pool_metric = false,
                    const SummaryArgs* summary = nullptr) {
  if ((!h->has_position && !q_host) || !h->has_eps) { h->err = "set position and step size (or run the initial search) first"; return DHMC_EARG; }
  const auto tr0 = std::chrono::steady_clock::now();
  auto tr_ms = [&] { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - tr0).count(); };
  double tr_pt[6] = {0, 0, 0, 0, 0, 0};
  CK(cudaSetDevice(h->cfg.device));
  if (thin < 1 || N % thin != 0) { h->err = "thin >= 1 and N a multiple of thin"; return DHMC_EARG; }
  const size_t B = (size_t)h->cfg.n_chains, D = (size_t)h->cfg.dim, n = (size_t)(N / thin);   // n: kept draws per chain
  double* d_p = nullptr;
  unsigned* d_dir = nullptr;
  int rc = DHMC_OK;
  // Host outputs.  Page-locked (pinned) buffers are written by the kernel itself through their device alias — no staging
  // copy in HBM, no second hop, the PCIe writes overlap the sampling at cache-line granularity and N is not bounded by
  // device memory.  Pageable buffers are staged in HBM (out[i] in stage[i]) and copied chunk by chunk; if the draws would
  // not fit, the buffer is page-locked on the fly (cudaHostRegister) and written directly.
  struct Output { void* host; size_t row; void* dev; bool direct; };       // row: bytes per kept draw of a chain
  Output out[4] = {{posterior, sizeof(double) * D, nullptr, false}, {stats, sizeof(dhmc_tree_stats), nullptr, false},
                   {eps_used, sizeof(double), nullptr, false}, {logdens, sizeof(double), nullptr, false}};
  for (int i = 0; i < 4; ++i) {
    Output& o = out[i];
    if (!o.host) continue;
    if (outputs_on_device) { o.dev = o.host; continue; }
    const size_t bytes = o.row * B * n;
    if (i == 0) {
      // Draws: staging + DMA copies overlapped chunk by chunk is the faster route when the draws fit in HBM (C2: 21.9 ms per
      // step against 24.1 ms with direct writes — kernel stores reach ~47 GB/s over PCIe, the copy engines 57 GB/s); the
      // kernel writes the host buffer directly when they do not fit (DHMC_DIRECT=1 forces it).
      size_t fr = 0, tot = 0;
      cudaMemGetInfo(&fr, &tot);
      const bool fits = bytes <= h->stage_bytes[0] || bytes + ((size_t)1 << 30) <= fr;
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
      if ((rc = ensure_stage(h, i, bytes)) != DHMC_OK) return rc;
      o.dev = h->stage[i];
    }
  }
  if (p_over_host || dir_over_host) {
    if ((rc = ensure_tmp(h, p_over_host ? B * D : 0)) != DHMC_OK) return rc;
  }
  if (p_over_host) {
    d_p = h->tmp_bd;
    CK(cudaMemcpyAsync(d_p, p_over_host, sizeof(double) * B * D, cudaMemcpyHostToDevice, h->stream));
  }
  if (dir_over_host) {
    d_dir = h->tmp_dir;
    CK(cudaMemcpyAsync(d_dir, dir_over_host, sizeof(unsigned) * B, cudaMemcpyHostToDevice, h->stream));
  }
  tr_pt[0] = tr_ms();
  KArgs a = base_args(h);
  a.N = N; a.thin = thin; a.N_keep = (int)n; a.cfg = cfg; a.p_override = d_p; a.dir_override = d_dir;
  a.out_q = (double*)out[0].dev; a.out_stats = (dhmc_tree_stats*)out[1].dev; a.out_eps = (double*)out[2].dev;
  a.out_lq = (double*)out[3].dev;
  if (cfg.metric == DHMC_METRIC_SYMMETRIC) a.covt = h->covt;
  if (pool_metric) a.mean_out = h->mean_pool;
  a.summary = summary;
  const size_t out_bytes = posterior ? sizeof(double) * B * n * D : 0;
  // chunks must stay many waves long, or the ragged tail of every chunk idles the SMs
  // chunks overlap the staged downloads (and the upload of q_host) with the sampling of the next chunk; with direct
  // host writes only an upload is left to overlap
  const bool staged_big = posterior && !out[0].direct && out_bytes >= ((size_t)32 << 20);
  int nchunks = (!outputs_on_device && B >= 4096 && (staged_big || q_host)) ? 16 : 1;
  while (nchunks > 1 && B / (size_t)nchunks < (size_t)8 * (size_t)h->grid * (size_t)h->G) nchunks /= 2;   // >= 8 waves of chain slots per chunk
  if (const char* ev = std::getenv("DHMC_E2E_CHUNKS")) { const int v = std::atoi(ev); if (v >= 1 && v <= 16 && !outputs_on_device) nchunks = v; }
  CK(cudaMemsetAsync(h->status, 0, sizeof(int) * B, h->stream));   // status words describe the current call
  for (int ci = 0; ci < nchunks; ++ci) {
    // (a pooled metric, and a batch on packed groups, keep their groups of 8 chains inside one chunk)
    const size_t unit = (h->pooled || (h->G > 1 && h->batch_k)) ? 8 : 1;
    const size_t c0 = (B / unit) * ci / nchunks * unit, c1 = (B / unit) * (ci + 1) / nchunks * unit, nc = c1 - c0;
    if (nc == 0) continue;
    a.chain_begin = (int)c0; a.chain_end = (int)c1;
    if (q_host) {
      // positions of this chunk: H2D on its own stream, then evaluate_ℓ(strict) on the compute
      // stream — overlaps with the previous chunk's sampling and D2H
      if (ci == 0) {   // uploads start after everything already queued on the compute stream
        CK(cudaEventRecord(h->h2d_ev[15], h->stream));
        CK(cudaStreamWaitEvent(h->h2d_stream, h->h2d_ev[15], 0));
      }
      CK(cudaMemcpyAsync(h->q + c0 * D, q_host + c0 * D, sizeof(double) * nc * D, cudaMemcpyHostToDevice, h->h2d_stream));
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
    if (!outputs_on_device) {
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
  CK(cudaMemcpyAsync(&steps, h->total_steps, sizeof steps, cudaMemcpyDeviceToHost, h->stream));
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
      if (q_host) cudaEventElapsedTime(&a, h->ev0, h->h2d_ev[ci]);
      cudaEventElapsedTime(&b2, h->ev0, h->chunk_ev[ci]);
      if (!outputs_on_device) cudaEventElapsedTime(&c, h->ev0, h->copy_ev[ci]);
      std::fprintf(stderr, " [h2d %.2f kern %.2f d2h %.2f]", a, b2, c);
    }
    cudaEventElapsedTime(&t, h->ev0, h->ev1);
    std::fprintf(stderr, " total kernels %.2f ms | host: setup %.2f, enqueued %.2f, compute stream done %.2f, copy stream done %.2f\n", t,
                 tr_pt[0], tr_pt[1], tr_pt[2], tr_pt[3]);
    cudaGetLastError();
  }
  h->last_steps = (int64_t)steps;
  if (advance_t) h->t += (uint32_t)N;
  if (q_host) h->has_position = true;
  if (h->trace) std::fprintf(stderr, "[dhmc trace] host: before status check %.2f ms\n", tr_ms());
  rc = sync_and_check_status(h, DHMC_CHAIN_NONFINITE_Q | DHMC_CHAIN_BAD_ACCEPTANCE | DHMC_CHAIN_BAD_STEPSIZE |
                                    DHMC_CHAIN_LEAPFROG_NONFINITE | (q_host ? DHMC_CHAIN_BAD_INITIAL : 0),
                             q_host ? "invalid initial position, or non-finite position / acceptance rate / step size while sampling"
                                    : "sampling: non-finite position, acceptance rate or step size");
  if (h->trace) std::fprintf(stderr, "[dhmc trace] host: after status check %.2f ms\n", tr_ms());
  if (rc != DHMC_OK) return rc;
  if (cfg.metric == DHMC_METRIC_DIAGONAL) return set_metric_kind(h, false, false);   // κ ← Diagonal: the diagonal kernels
  if (cfg.metric == DHMC_METRIC_SYMMETRIC) {
    // κ = GaussianKineticEnergy(regularize_M⁻¹(sample_M⁻¹(Symmetric, X), λ)) — mcmc.jl:282
    const int fgrid = factor_grid(h);
    if (pool_metric)
      k_cov_pool<<<fgrid, 128, sizeof(double) * h->cfg.dim, h->stream>>>(h->covt, h->mean_pool, h->minv_dense, N, lambda, (int)h->cfg.dim, (int)h->cfg.n_chains);
    else
      k_cov_finish<<<fgrid, 128, 0, h->stream>>>(h->covt, h->minv_dense, N, lambda, (int)h->cfg.dim, (int)h->cfg.n_chains);
    h->launches += 1;
    rc = factor_and_switch(h, pool_metric);
  }
  return rc;
}

int dhmc_sample_tree(dhmc_handle* h, const double* p, const uint32_t* directions, dhmc_tree_stats* stats) {
  if (!h) return DHMC_EARG;
  AdaptConfig cfg{};
  return run_nuts(h, 1, cfg, 0.0, p, directions, nullptr, stats, nullptr, nullptr, false, true);
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
  AdaptConfig cfg{};
  cfg.metric = pool ? DHMC_METRIC_SYMMETRIC : metric;
  if (da) {
    // DualAveraging @argchecks — stepsize.jl:108-111
    if (!(0 < da->delta && da->delta < 1) || !(da->gamma > 0) || !(0.5 < da->kappa && da->kappa <= 1) || !(da->t0 >= 0)) {
      h->err = "DualAveraging: 0 < δ < 1, γ > 0, 0.5 < κ ≤ 1, t₀ ≥ 0"; return DHMC_EARG;
    }
    cfg.adapt = 1; cfg.delta = da->delta; cfg.gamma = da->gamma; cfg.kappa = da->kappa; cfg.t0 = da->t0;
  }
  if (cfg.metric == DHMC_METRIC_SYMMETRIC) { int rcd = ensure_dense(h); if (rcd != DHMC_OK) return rcd; }
  if (pool && !h->mean_pool) CK(cudaMalloc(&h->mean_pool, sizeof(double) * (size_t)h->cfg.n_chains * (size_t)h->cfg.dim));
  return run_nuts(h, N, cfg, lambda, nullptr, nullptr, posterior, stats, eps_used, logdens, false, true, nullptr, 1, pool);
}

int dhmc_mcmc(dhmc_handle* h, int32_t N, double* posterior, dhmc_tree_stats* stats, double* logdens) {
  if (!h || N < 0) return DHMC_EARG;
  if (N == 0) return DHMC_OK;
  AdaptConfig cfg{};
  return run_nuts(h, N, cfg, 0.0, nullptr, nullptr, posterior, stats, nullptr, logdens, false, true);
}
int dhmc_mcmc_from(dhmc_handle* h, const double* q, int32_t N, double* posterior, dhmc_tree_stats* stats,
                   double* logdens) {
  if (!h || !q || N < 1) return DHMC_EARG;
  AdaptConfig cfg{};
  return run_nuts(h, N, cfg, 0.0, nullptr, nullptr, posterior, stats, nullptr, logdens, false, true, q);
}
int dhmc_mcmc_thinned(dhmc_handle* h, const double* q, int32_t N, int32_t thin, double* posterior,
                      dhmc_tree_stats* stats, double* logdens) {
  if (!h || N < 1 || thin < 1) return DHMC_EARG;
  AdaptConfig cfg{};
  return run_nuts(h, N, cfg, 0.0, nullptr, nullptr, posterior, stats, nullptr, logdens, false, true, q, thin);
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
  AdaptConfig cfg{};
  return run_nuts(h, N, cfg, 0.0, nullptr, nullptr, posterior, stats, nullptr, logdens, true, true);
}

// ------------------------------------------------------------------ streaming posterior summary (DESIGN §4.4)
// record [DHMC_SUMMARY_FIELDS, D, P] column-major: the fields of (parameter d, problem p) at (p·D + d)·F
static double* summary_cell(double* record, int64_t D, int64_t p, int64_t d) { return record + ((size_t)p * D + d) * DHMC_SUMMARY_FIELDS; }

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
  const size_t D = (size_t)h->cfg.dim, B = (size_t)h->cfg.n_chains;
  const int64_t K = h->batch_k, off = h->cfg.chain_offset;
  const size_t P = K ? (size_t)h->batch_p : 1, PD = P * D, rows = (size_t)h->grid * h->G * 3 * D;
  // histograms (counts != NULL): cells bins per (d, p); the staging rows of the resident chain groups
  const size_t cells = counts ? (size_t)nbins + 2 : 0, stage = (size_t)h->grid * h->G * cells * D;
  // one grow-only arena: acc [P][5][D], shift [P][D], ref [P][D], row [grid·G][3][D], below [P][D], chains [P], then with
  // histograms hist [P][D][cells], lo [P][D], inv_w [P][D] (8-byte elements) and stage [grid·G][cells][D] (4-byte)
  const size_t need = sizeof(double) * (8 * PD + rows + P + PD * cells + (counts ? 2 * PD : 0)) + sizeof(unsigned) * stage;
  if (need > h->sum_bytes) {
    cudaFree(h->sum_buf); h->sum_buf = nullptr; h->sum_bytes = 0;
    CK(cudaMalloc(&h->sum_buf, need));
    h->sum_bytes = need;
  }
  if (!h->sum_args) CK(cudaMalloc(&h->sum_args, sizeof(SummaryArgs)));
  double* acc = (double*)h->sum_buf;
  double* shift = acc + 5 * PD;
  double* ref = shift + PD;
  double* row = ref + PD;
  unsigned long long* below = (unsigned long long*)(row + rows);
  unsigned long long* chains = below + PD;
  CK(cudaMemsetAsync(acc, 0, sizeof(double) * 5 * PD, h->stream));
  CK(cudaMemsetAsync(below, 0, sizeof(unsigned long long) * (PD + P), h->stream));
  if (reference) CK(cudaMemcpyAsync(ref, reference, sizeof(double) * PD, cudaMemcpyHostToDevice, h->stream));
  // shift of problem p: the position of its first local chain, max(p·K − off, 0); problems p0 … p1 have local chains.  Past
  // the first, those chains are K apart: one strided copy (a first problem entered in its middle takes one more).
  const int64_t p0 = K ? off / K : 0, p1 = K ? (off + (int64_t)B - 1) / K : 0;
  const int64_t pa = (K && off % K) ? p0 + 1 : p0;
  if (pa > p0) CK(cudaMemcpyAsync(shift + p0 * D, h->q, sizeof(double) * D, cudaMemcpyDeviceToDevice, h->stream));
  if (p1 >= pa)
    CK(cudaMemcpy2DAsync(shift + pa * D, sizeof(double) * D, h->q + (size_t)(K ? pa * K - off : 0) * D, sizeof(double) * D * (size_t)(K ? K : 1),
                         sizeof(double) * D, (size_t)(p1 - pa + 1), cudaMemcpyDeviceToDevice, h->stream));
  SummaryArgs sa{row, shift, reference ? ref : nullptr, acc, below, chains, n_keep / 2, nullptr, nullptr, nullptr, nullptr, 0};
  if (counts) {
    unsigned long long* hist = chains + P;
    double* lo = (double*)(hist + PD * cells);
    double* inv_w = lo + PD;
    std::vector<double> hinv(PD);
    for (size_t i = 0; i < PD; ++i) hinv[i] = (double)nbins / (hi_host[i] - lo_host[i]);
    CK(cudaMemsetAsync(hist, 0, sizeof(unsigned long long) * PD * cells, h->stream));
    CK(cudaMemcpyAsync(lo, lo_host, sizeof(double) * PD, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(inv_w, hinv.data(), sizeof(double) * PD, cudaMemcpyHostToDevice, h->stream));
    sa.lo = lo; sa.inv_w = inv_w; sa.stage = (unsigned*)(inv_w + PD); sa.hist = hist; sa.nbins = nbins;
  }
  CK(cudaMemcpyAsync(h->sum_args, &sa, sizeof sa, cudaMemcpyHostToDevice, h->stream));
  AdaptConfig cfg{};
  const int rc = run_nuts(h, N, cfg, 0.0, nullptr, nullptr, nullptr, stats, nullptr, logdens, false, true, nullptr, thin, false,
                          h->sum_args);
  if (rc != DHMC_OK && rc != DHMC_ENUMERIC) return rc;    // a chain that failed is left out of its problem's sums
  std::vector<double> hacc(5 * PD), hshift(PD);
  std::vector<unsigned long long> hcnt(PD + P);
  CK(cudaMemcpyAsync(hacc.data(), acc, sizeof(double) * hacc.size(), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaMemcpyAsync(hshift.data(), shift, sizeof(double) * PD, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaMemcpyAsync(hcnt.data(), below, sizeof(unsigned long long) * hcnt.size(), cudaMemcpyDeviceToHost, h->stream));
  if (counts)        // [P][D][cells] is the column-major [cells, D, P] of the ABI; uint64 counts stay far below 2^63
    CK(cudaMemcpyAsync(counts, below + PD + P, sizeof(int64_t) * PD * cells, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  for (size_t p = 0; p < P; ++p) {
    const double M = (double)hcnt[PD + p], m = 2.0 * M;
    const double* a = &hacc[p * 5 * D];
    for (size_t d = 0; d < D; ++d) {
      double* r = summary_cell(record, (int64_t)D, (int64_t)p, (int64_t)d);
      r[DHMC_SUMMARY_CHAINS] = M;
      r[DHMC_SUMMARY_NKEEP] = (double)n_keep;
      r[DHMC_SUMMARY_BELOW] = reference ? (double)hcnt[p * D + d] : dm_nan();
      if (M == 0) {
        r[DHMC_SUMMARY_MEAN] = r[DHMC_SUMMARY_SS_SEQ] = r[DHMC_SUMMARY_M2] = r[DHMC_SUMMARY_SS_CHAIN] = 0.0;
        continue;
      }
      const double s1 = a[d], s2 = a[D + d], c1 = a[3 * D + d], c2 = a[4 * D + d];
      r[DHMC_SUMMARY_MEAN] = hshift[p * D + d] + s1 / m;
      r[DHMC_SUMMARY_SS_SEQ] = std::max(0.0, s2 - s1 * s1 / m);
      r[DHMC_SUMMARY_M2] = a[2 * D + d];
      r[DHMC_SUMMARY_SS_CHAIN] = std::max(0.0, c2 - c1 * c1 / M);
    }
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
  const size_t cells = (size_t)h->cfg.dim * (h->batch_k ? (size_t)h->batch_p : 1);
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
  unsigned long long* d_cnt = nullptr;   // [33 depth][3 term][1 steps]
  double* d_f = nullptr;                 // [1 acc][B ebfmi]
  CK(cudaMalloc(&d_cnt, sizeof(unsigned long long) * 37));
  CK(cudaMalloc(&d_f, sizeof(double) * (1 + (size_t)B)));
  CK(cudaMemsetAsync(d_cnt, 0, sizeof(unsigned long long) * 37, h->stream));
  CK(cudaMemsetAsync(d_f, 0, sizeof(double), h->stream));
  k_tree_summary<<<h->sm_count * 8, 256, 0, h->stream>>>(stats_dev, N, B, d_cnt, d_cnt + 33, d_f, d_cnt + 36, ebfmi ? d_f + 1 : nullptr);
  h->launches += 1;
  unsigned long long cnt[37];
  double acc = 0;
  cudaError_t e = cudaMemcpyAsync(cnt, d_cnt, sizeof cnt, cudaMemcpyDeviceToHost, h->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(&acc, d_f, sizeof acc, cudaMemcpyDeviceToHost, h->stream);
  if (e == cudaSuccess && ebfmi) e = cudaMemcpyAsync(ebfmi, d_f + 1, sizeof(double) * B, cudaMemcpyDeviceToHost, h->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
  cudaFree(d_cnt); cudaFree(d_f);
  if (e != cudaSuccess) { h->err = cudaGetErrorString(e); return DHMC_ECUDA; }
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
  double *d_pilot = nullptr, *d_acc = nullptr;
  CK(cudaMalloc(&d_pilot, sizeof(double) * PD));
  CK(cudaMalloc(&d_acc, sizeof(double) * PD * (L + 3)));
  CK(cudaMemsetAsync(d_acc, 0, sizeof(double) * PD * (L + 3), h->stream));
  k_pilot_mean<<<(unsigned)((PD + 127) / 128), 128, 0, h->stream>>>(draws_dev, n, N, D, B, K, off, P, d_pilot);
  k_ess_rhat<<<h->sm_count * 8, 256, 0, h->stream>>>(draws_dev, N, n, D, B, K, off, L, d_pilot, d_acc);
  h->launches += 2;
  std::vector<double> acc(PD * (L + 3));
  cudaError_t e = cudaMemcpyAsync(acc.data(), d_acc, sizeof(double) * acc.size(), cudaMemcpyDeviceToHost, h->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
  cudaFree(d_pilot); cudaFree(d_acc);
  if (e != cudaSuccess) { h->err = cudaGetErrorString(e); return DHMC_ECUDA; }
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
  unsigned long long* d_hist = nullptr;
  CK(cudaMalloc(&d_hist, sizeof(unsigned long long) * (BINS + 1)));
  CK(cudaMemsetAsync(d_hist, 0, sizeof(unsigned long long) * (BINS + 1), h->stream));
  const size_t n = (size_t)N * (size_t)h->cfg.n_chains;
  k_acceptance_hist<<<h->sm_count * 8, 256, 0, h->stream>>>(stats_dev, n, d_hist, BINS);
  h->launches += 1;
  std::vector<unsigned long long> hist(BINS + 1);
  cudaError_t e = cudaMemcpyAsync(hist.data(), d_hist, sizeof(unsigned long long) * hist.size(), cudaMemcpyDeviceToHost, h->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
  cudaFree(d_hist);
  if (e != cudaSuccess) { h->err = cudaGetErrorString(e); return DHMC_ECUDA; }
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
  CK(cudaMemcpy(v.data(), h->phase_clocks, sizeof(unsigned long long) * n, cudaMemcpyDeviceToHost));
  for (int k = 0; k < kPhCount; ++k) out[k] = 0;
  for (size_t i = 0; i < n; ++i) out[i % kPhCount] += v[i];
  if (reset) CK(cudaMemset(h->phase_clocks, 0, sizeof(unsigned long long) * n));
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
  return dhmc_allgather_dev(h, h->q, recv_dev, (size_t)h->cfg.n_chains * (size_t)h->cfg.dim);
}
int dhmc_last_comm_ms(dhmc_handle* h, double* ms) { if (!h || !ms) return DHMC_EARG; *ms = h->last_comm_ms; return DHMC_OK; }
#undef CKN

}  // extern "C"
