// kernels.cuh — the sm_90a kernels of the many-chain NUTS engine (templates; instantiated per
// log-density family in family_tu.cu, looked up by the host side in dhmc_b200.cu).
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
#pragma once
#include <cuda_runtime.h>

#include <type_traits>

#include "../../include/dhmc.h"
#include "device_backend.cuh"

namespace dhmc {

// ------------------------------------------------------------------ kernel args
// One problem of a batch: where its blocks start in the handle's arrays (doubles) and, for logistic regression, its
// observations and the leading dimension of its Xᵀ.  Problems lie back to back, each with arrays of its own size; the
// host keeps every Xᵀ base even and every padded-X base a multiple of 32·tma_xs(D) doubles (16-byte row segments, whole
// row blocks for the bulk copies).
struct ProblemDesc {
  size_t mparams, X, Xt, y, Xp;
  int N, ld;
};

// Streaming posterior summary (dhmc_mcmc_summary, DESIGN §4.4): the kept draws of every chain are folded into Welford
// moments (the metric window's two reserved slots) and, at chain end, into per-problem sums; no draw is written out.
//   row    [grid·G][3][D]  per chain group: sequence 0's mean and M2, and the count of kept draws below the reference
//   shift  [P][D]          the position of the problem's first local chain at call start (keeps the sums free of cancellation)
//   ref    [P][D] or null  the reference of the rank statistic
//   acc    [P][5][D]       Σ(μ_s − s), Σ(μ_s − s)², Σ M2_s over sequences; Σ(μ_c − s), Σ(μ_c − s)² over chains
//   below  [P][D]          Σ #{kept draws with θ < reference} (exact)
//   chains [P]             chains that completed the call
// Histograms for quantiles (dhmc_mcmc_summary_histogram; hist null: off), nbins + 2 bins per cell (include/dhmc.h):
//   lo, inv_w [P][D]                 the grid: lower end and nbins / (hi − lo)
//   stage [grid·G][nbins + 2][D]     per chain group: the counts of the running chain (cleared at its first kept draw)
//   hist  [P][D][nbins + 2]          Σ over the problem's completed chains (the host layout)
// Generated quantities of a user model (include/dhmc_models.h; ng = 0: none), the summary's rows D … D + ng − 1, in arrays
// of their own laid out as those of the parameters with ng in place of D (the parameters' arrays keep their layout):
//   grow   [grid·G][5][ng]  per chain group: the running sequence's mean and M2, sequence 0's mean and M2, the below-count
//   gshift, gref, gbelow, glo, ginv_w [P][ng];  gacc [P][5][ng];  gstage [grid·G][nbins + 2][ng];  ghist [P][ng][nbins + 2]
//   mparams, problems   the problem blocks the quantities read (problems null: one problem)
// Random generated quantities (DHMC_USER_GENERATED_RNG): kept draw j of local chain c has the key (seed, chain_offset + c)
// and transition t0 + (j + 1)·thin − 1, the RNG counter of the transition that produced it (include/dhmc_models.h).
struct SummaryArgs {
  double* row;
  const double* shift;
  const double* ref;
  double* acc;
  unsigned long long* below;
  unsigned long long* chains;
  int n;                        // draws per sequence: ⌊N_keep / 2⌋
  const double* lo;
  const double* inv_w;
  unsigned* stage;
  unsigned long long* hist;
  int nbins;
  int ng;
  const double* mparams;
  const ProblemDesc* problems;
  double* grow;
  const double* gshift;
  const double* gref;
  double* gacc;
  unsigned long long* gbelow;
  const double* glo;
  const double* ginv_w;
  unsigned* gstage;
  unsigned long long* ghist;
  unsigned long long seed;
  long long chain_offset;
  unsigned t0;
  int thin;
};

struct KArgs {
  int D, B, T, W;
  unsigned long long seed;
  long long chain_offset;
  double *q, *g, *lq, *p, *minv, *eps;
  const double* mparams;
  int* status;
  int max_depth;
  double min_delta;
  unsigned t0;
  int N;
  AdaptConfig cfg;
  const double* p_override;
  const unsigned* dir_override;
  double* out_q;
  dhmc_tree_stats* out_stats;
  double* out_lq;
  double* out_eps;
  double* scratch;
  size_t scratch_per_cta;  // doubles
  int n_sm, n_slots;
  size_t stride;
  unsigned* counter;
  unsigned long long* total_steps;
  double s_init, s_thresh;
  int s_maxiter;
  int lf_steps, lf_sign;
  int strict, randomize;
  double* out_phase;
  int chain_begin, chain_end;   // persistent kernels: chains [begin, end) of this launch
  double *minv_dense, *wt, *covt;   // Symmetric metric: M⁻¹, Wᵀ, co-moments, each [B][D][D]
  int xs_doubles;               // shared-memory staging vector (0 unless the dense arrays exist)
  const double *lX, *lXt, *ly;  // logistic regression data
  double* lr;                   // logistic scratch of one chain per CTA: [grid][lN] residuals (packed groups need none)
  int lN, lLd;                  // observations (a batch: the largest N, the scratch row length), leading dimension of Xᵀ (even)
  const double* lXp;            // tensor-core likelihood: zero-padded row blocks of X
  int levels, ntab;             // deep kernels (max_depth > 12) only: stack entries per warp (max_depth + 1), slot-table entries;
                                // all other kernels use the compile-time kStdLevels / kStdTab so that the offsets fold into immediates
  int thin, N_keep;             // draws: every thin-th transition is kept (N_keep = N / thin rows per chain)
  double* mean_out;             // pooled Symmetric stage: the window mean of every chain [B][D] (else null)
  int pooled;                   // the current dense metric is shared by every group of 8 chains (DHMC_METRIC_SYMMETRIC_POOLED)
  const double* minv_pad;       // tensor-core mat-vec: padded M⁻¹ [B][⌈D/32⌉·32][tma_xs(D)]
  // problem batches (dhmc_set_problems / _ragged): global chain g reads problem g / batch_k, described by problems[g / batch_k];
  // batch_k = 0: one problem for every chain (problems is null).  Global ids of a batch stay below 2^31 (host-checked), so
  // the problem index is a 32-bit division.
  int batch_k;
  const ProblemDesc* problems;
  int red_groups;               // groups of the reduction buffer (smem_layout rg) of the kernels with DeviceBackend::kFused
  const SummaryArgs* summary;   // k_nuts: fold the kept draws into a streaming summary (device struct; null: off)
#if defined(DHMC_PHASE_CLOCKS)
  unsigned long long* phase_clocks;   // leaf profile: kPhCount counters per CTA (nuts_machine.cuh)
#endif
};

// Register budget: minimum resident CTAs per SM the compiler must allow for.
__host__ __device__ constexpr int min_ctas(int W, int EPL) {
#ifndef DHMC_MINCTAS_W4E8
#define DHMC_MINCTAS_W4E8 3
#endif
  return W == 1 ? 16 : W == 2 ? 8 : W == 4 ? (EPL >= 8 ? DHMC_MINCTAS_W4E8 : 4) : EPL >= 16 ? 1 : 2;
}

__host__ __device__ inline size_t group_smem_bytes(int W, int n_sm, size_t stride, size_t xs, int levels, int ntab) {
  return (smem_layout(W, n_sm, stride, xs, levels, ntab).total + 127) & ~(size_t)127;   // the CTA-shared area behind the groups stays 128-byte aligned
}

template <int EPL, int FAM, int W, bool DN, int G, bool DP>
__device__ __forceinline__ void setup_backend(DeviceBackend<EPL, FAM, W, DN, G, DP>& b, const KArgs& a,
                                              unsigned char* smem) {
  b.ctid = threadIdx.x; b.grp = 0;
  b.tid = threadIdx.x; b.lane = threadIdx.x & 31; b.warp = threadIdx.x >> 5;
  b.D = a.D;
  using Bk = DeviceBackend<EPL, FAM, W, DN, G, DP>;
  const int rg = Bk::kFused ? a.red_groups : 1;
  const SmemLayout L = smem_layout(W, a.n_sm, b.stride, (size_t)a.xs_doubles, DP ? a.levels : kStdLevels, DP ? a.ntab : kStdTab, rg);
  b.lX = a.lX; b.lXt = a.lXt; b.ly = a.ly; b.lN = a.lN; b.lLd = a.lLd;
  b.lr = a.lr ? a.lr + (size_t)blockIdx.x * a.lN : nullptr;
  b.cb_beta = b.cb_grad = nullptr;
  b.cb_shared = nullptr; b.ring_n = 0; b.lXp = nullptr; b.Mp = a.minv_pad; b.pooled = a.pooled;
  size_t group = blockIdx.x;
  if constexpr (G > 1) {                               // one warp per chain
    b.grp = threadIdx.x >> 5; b.tid = threadIdx.x & 31; b.warp = 0;
    group = (size_t)blockIdx.x * G + b.grp;
    const size_t per = group_smem_bytes(W, a.n_sm, b.stride, (size_t)a.xs_doubles, DP ? a.levels : kStdLevels, DP ? a.ntab : kStdTab);
    unsigned char* shared = smem + per * G;            // the area after the G per-group blocks (128-byte aligned)
    b.cb_shared = shared;
    b.cb_beta = reinterpret_cast<double*>(shared + tma_beta_off());
    b.cb_grad = reinterpret_cast<double*>(shared + tma_ring_off(G));   // Xᵀr [chain][XS] is handed back in stage 0 of the idle ring
    const int nzero = (int)((tma_tabs_off(G) - tma_beta_off()) / sizeof(double));    // β (incl. its zero k-padding), η, residual tiles
    for (int i = threadIdx.x; i < nzero; i += 32 * G) b.cb_beta[i] = 0.0;
    double* tabs = reinterpret_cast<double*>(shared + tma_tabs_off(G));
    for (int i = threadIdx.x; i < DM_TABS_DOUBLES; i += 32 * G) tabs[i] = dm_tabs_entry(i);
    if (threadIdx.x == 0) {
      uint64_t* bars = reinterpret_cast<uint64_t*>(shared + 64);
      for (int s = 0; s < kTmaStages; ++s) { mbar_init(bars + s, 1); mbar_init(bars + kTmaStages + s, G); }
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    b.lXp = a.lXp;
    b.lr = nullptr;
    smem += per * b.grp;
    __syncthreads();
  }
  b.xs = reinterpret_cast<double*>(smem + L.xs_off);
  b.Mrow = nullptr; b.Wt = nullptr; b.covt = nullptr;
  b.red = reinterpret_cast<double*>(smem + L.red_off);
  b.red_buf = 0;
  if constexpr (Bk::kFused) {
    b.red_half_n = (int)red_half_doubles(W, rg); b.red_row = kRedWidth * rg;
    b.m_sp = 0; b.m_c = 0; b.m_dbl = 0; b.m_shift = 0; b.m_buf = b.red;
  }
  b.rexp_cache = 0.0; b.rexp_base = 0xffffffffu; b.rexp_t = 0xffffffffu;
  b.ctl = reinterpret_cast<Entry*>(smem + L.ctl_off) + b.warp * (DP ? a.levels : kStdLevels);
  b.tops = reinterpret_cast<TopState*>(smem + L.top_off + b.warp * ((sizeof(TopState) + 15) & ~(size_t)15));
  b.sm_slots = reinterpret_cast<double*>(smem + L.slots_off);
  b.gl_slots = a.scratch + group * a.scratch_per_cta;
  b.n_sm = a.n_sm; b.n_slots = a.n_slots;
  b.slot_tab = reinterpret_cast<double**>(smem + L.tab_off); b.n_tab = DP ? a.ntab : kStdTab;
  b.build_slot_table();
  b.mparams = a.mparams;
#if defined(DHMC_PHASE_CLOCKS)
  b.ph_acc = a.phase_clocks + (size_t)blockIdx.x * kPhCount;
  b.ph_t = clock64(); b.ph_cur = kPhTrans;
#endif
}

// packed groups: every warp draws its own chains
template <class B>
__device__ __forceinline__ int next_chain_group(B& b, unsigned* counter, int begin) {
  int c = 0;
  if (b.lane == 0) c = begin + (int)atomicAdd(counter, 1u);
  return __shfl_sync(0xffffffffu, c, 0);
}
// pooled metric or problem batch: the whole CTA (8 chains = one metric group / 8 chains of one problem) takes group g; warp w
// runs chain begin + 8·g + w.  All warps arrive here together (they left the previous group through coop_finish), so a CTA
// barrier is safe.
template <class B>
__device__ __forceinline__ int next_pooled_group(B& b, unsigned* counter, int begin) {
  int* slot = reinterpret_cast<int*>(b.cb_shared + 96);
  __syncthreads();
  if (b.ctid == 0) *slot = (int)atomicAdd(counter, 1u);
  __syncthreads();
  return begin + 8 * (*slot) + b.grp;
}
__device__ __forceinline__ int next_chain(unsigned* counter, int* s_misc, int begin) {
  __syncthreads();
  if (threadIdx.x == 0) s_misc[0] = begin + (int)atomicAdd(counter, 1u);
  __syncthreads();
  return s_misc[0];
}

template <int EPL, int FAM, int W, bool DN, int G, bool DP>
__device__ __forceinline__ void load_chain(DeviceBackend<EPL, FAM, W, DN, G, DP>& b, const KArgs& a, long c,
                                           bool with_p) {
  b.chain = c;
  b.rexp_base = 0xffffffffu; b.rexp_t = 0xffffffffu;   // the randexp batch belongs to one chain
  const size_t base = (size_t)c * a.D;
#pragma unroll
  for (int e = 0; e < EPL; ++e) {
    const int i = b.tid + e * b.T;
    const bool ok = i < a.D;
    b.q[e] = ok ? a.q[base + i] : 0.0;
    b.g[e] = ok ? a.g[base + i] : 0.0;
    b.minv[e] = ok ? a.minv[base + i] : 1.0;
    b.p[e] = (ok && with_p) ? a.p[base + i] : 0.0;
    b.rhoL[e] = 0.0;
  }
  b.lq = a.lq[c];
  if (a.batch_k) {       // problem batch: the blocks of this chain's problem (uniform over the chain's threads)
    const ProblemDesc& pd = a.problems[(unsigned)(a.chain_offset + c) / (unsigned)a.batch_k];
    b.mparams = a.mparams + pd.mparams;
    b.lX = a.lX + pd.X; b.lXt = a.lXt + pd.Xt; b.ly = a.ly + pd.y;
    b.lN = pd.N; b.lLd = pd.ld;       // (the per-CTA residual scratch keeps its stride: a.lN, the batch's largest N)
    // packed groups: the CTA's 8 chains are one problem (group fetch, host-checked 8-alignment), so every warp points the
    // shared rounds at the same X and derives the same block count from the same N.  No bulk copy outlives a round —
    // coop_core_tma issues blocks 0, 1 and then b + 2 only while b + 2 < nblk, and waits on every one of them before its
    // closing barrier — so X and N may change between groups.
    if constexpr (G > 1) b.lXp = a.lXp + pd.Xp;
  }
  const size_t dd = (size_t)a.D * a.D;
  if (a.covt) b.covt = a.covt + (size_t)c * dd;
  b.mean_out = a.mean_out ? a.mean_out + (size_t)c * a.D : nullptr;
  if constexpr (DN) {
    b.Mrow = a.minv_dense + (size_t)c * dd;
    b.Wt = a.wt + (size_t)c * dd;
    if (with_p) b.matvec(b.p, b.ps);
  }
}
template <int EPL, int FAM, int W, bool DN, int G, bool DP>
__device__ __forceinline__ void store_vec(const DeviceBackend<EPL, FAM, W, DN, G, DP>& b, double* dst,
                                          const double (&v)[EPL], size_t base, int D) {
#pragma unroll
  for (int e = 0; e < EPL; ++e) {
    const int i = b.tid + e * b.T;
    if (i < D) dst[base + i] = v[e];
  }
}

// ------------------------------------------------------------------ k_nuts
// problem of local chain c (as load_chain)
__device__ __forceinline__ size_t summary_problem(const KArgs& a, long c) {
  return a.batch_k ? (size_t)((unsigned)(a.chain_offset + c) / (unsigned)a.batch_k) : 0;
}
// Random generated quantities key their numbers by the chain: summary_draw takes the local chain c in those builds only, so
// that every other build keeps its code.
#ifdef DHMC_USER_GENERATED_RNG
#define DHMC_GQ_CHAIN_PARAM , long c
#define DHMC_GQ_CHAIN_ARG , c
#else
#define DHMC_GQ_CHAIN_PARAM
#define DHMC_GQ_CHAIN_ARG
#endif
template <class Bk>
__device__ __noinline__ void summary_draw(const SummaryArgs* sp, double** slot_tab, int n_slots, int s_zq, int tid, int grp, int D,
                                         size_t p, int j DHMC_GQ_CHAIN_PARAM);

template <int EPL, int FAM, int W, bool DN, int G, bool DP>
struct DrawSink {
  DeviceBackend<EPL, FAM, W, DN, G, DP>& b;
  const KArgs& a;
  long c;
  __device__ __forceinline__ void operator()(int n, const dhmc_tree_stats& ts, double e) {
    if (a.thin > 1) {                     // thinning: transition n is kept when (n + 1) is a multiple of thin
      if ((n + 1) % a.thin != 0) return;
      n = (n + 1) / a.thin - 1;
    }
    const size_t row = (size_t)c * a.N_keep + n;
    if (a.out_q) {                       // draws are written once and never re-read on the device: streaming stores
#pragma unroll
      for (int e = 0; e < EPL; ++e) {
        const int i = b.tid + e * b.T;
        if (i < a.D) __stcs(a.out_q + row * a.D + i, b.q[e]);
      }
    }
    if (b.tid == 0) {
      if (a.out_stats) a.out_stats[row] = ts;
      if (a.out_lq) a.out_lq[row] = b.lq;
      if (a.out_eps) a.out_eps[row] = e;
    }
    if (a.summary)
      summary_draw<DeviceBackend<EPL, FAM, W, DN, G, DP>>(a.summary, b.slot_tab, b.n_slots, b.top().s_zq, b.tid, b.grp, a.D,
                                                          summary_problem(a, c), n DHMC_GQ_CHAIN_ARG);
  }
};

// ---- streaming summary (DESIGN §4.4), out of line and reached only when KArgs::summary is set, so that its body costs the
// sampling path no registers (ptxas still saves a few bytes around the two calls: benchmarks/streaming_summary_ptxas.md).
// The functions get the chain's slot table, not its backend (whose registers would have to move to memory to be passed); the kept position is read from the slot the transition loaded it from (the proposal ζ),
// and the Welford update is the metric window's own (metric_reset / metric_push on the two reserved slots), run on a view
// that holds only what those read.  Every thread touches its own elements i = tid + e·T, so nothing here synchronises.
template <class Bk>
__device__ __forceinline__ Bk welford_view(double** slot_tab, int n_slots, int tid, int D) {
  Bk w;
  w.slot_tab = slot_tab; w.n_slots = n_slots; w.tid = tid; w.D = D;
  return w;
}
template <class Bk>
__device__ __forceinline__ size_t summary_group(int grp) {
  return Bk::G > 1 ? (size_t)blockIdx.x * Bk::G + grp : (size_t)blockIdx.x;
}
template <class Bk>
__device__ __forceinline__ double* summary_row(const SummaryArgs& s, int grp, int D) {
  return s.row + summary_group<Bk>(grp) * 3 * (size_t)D;
}
template <class Bk>
__device__ __forceinline__ unsigned* summary_stage(const SummaryArgs& s, int grp, int D) {
  return s.stage + summary_group<Bk>(grp) * (size_t)(s.nbins + 2) * (size_t)D;
}
// Quantile histograms (include/dhmc.h): out of line again, with rolled loops that re-read the kept position from its slot
// (zq: the thread's first element, element e at zq[e·T]).  ptxas allocates k_nuts' registers together with these bodies,
// so they stay small, and the summary functions' own element loops are rolled too: with them unrolled, plain sampling in
// some dense-metric kernels slowed by 11 – 12 % (benchmarks/streaming_quantiles_ptxas.md).  Kept draw j: the thread clears its own staging cells at j = 0 and adds
// one count per element; the bin rule rounds the subtract and the multiply apart.
template <class Bk>
__device__ __noinline__ void summary_hist_draw(const SummaryArgs* sp, const double* zq, int tid, int grp, int D, size_t p, int j) {
  constexpr int EPL = sizeof(Bk::q) / sizeof(double), T = Bk::T;
  const SummaryArgs& s = *sp;
  const int nb = s.nbins;
  unsigned* stage = summary_stage<Bk>(s, grp, D);
#pragma unroll 1
  for (int e = 0; e < EPL; ++e) {
    const int i = tid + e * T;
    if (i >= D) break;
    if (j == 0) {
#pragma unroll 1
      for (int k = 0; k < nb + 2; ++k) stage[(size_t)k * D + i] = 0u;
    }
    const double t = __dmul_rn(__dsub_rn(zq[e * T], s.lo[p * D + i]), s.inv_w[p * D + i]);
    const int k = t < 0.0 ? 0 : !(t < (double)nb) ? nb + 1 : 1 + (int)t;
    stage[(size_t)k * D + i] += 1u;
  }
}
// chain end (completed chains only): the non-zero staging cells into the problem's histogram
template <class Bk>
__device__ __noinline__ void summary_hist_fold(const SummaryArgs* sp, int tid, int grp, int D, size_t p) {
  constexpr int EPL = sizeof(Bk::q) / sizeof(double), T = Bk::T;
  const SummaryArgs& s = *sp;
  const size_t cells = (size_t)s.nbins + 2;
  const unsigned* stage = summary_stage<Bk>(s, grp, D);
#pragma unroll 1
  for (int e = 0; e < EPL; ++e) {
    const int i = tid + e * T;
    if (i >= D) break;
    unsigned long long* hist = s.hist + (p * D + i) * cells;
#pragma unroll 1
    for (size_t k = 0; k < cells; ++k) {
      const unsigned c = stage[k * D + i];
      if (c) atomicAdd(hist + k, (unsigned long long)c);
    }
  }
}
#ifdef DHMC_USER_GENERATED
// Generated quantities (include/dhmc_models.h), compiled only into a user library whose model declares them, so that every
// other build keeps its code.  Quantity k reads the whole kept position, elements other threads wrote, so the chain
// synchronises before it reads the slot and again before the next transition may overwrite it (one chain per CTA: the
// USER family has no packed groups).  Thread tid evaluates and folds k = tid + e·T, with the moments, the rank and the bin
// rule of the parameters; its state for k lives in grow, and nothing else reads it.  Random quantities get the draw's key:
// (seed, global chain id) and the counter of the transition that produced kept draw j.
template <class Bk>
__device__ __noinline__ void summary_gq_draw(const SummaryArgs* sp, const double* zq, int tid, int grp, int D, size_t p, int j
                                             DHMC_GQ_CHAIN_PARAM) {
  static_assert(Bk::G == 1, "generated quantities: one chain per CTA");
  constexpr int T = Bk::T;
  const SummaryArgs& s = *sp;
  const int ng = s.ng, n = s.n, nb = s.nbins;
  const double* params = s.mparams + (s.problems ? s.problems[p].mparams : 0);
  double* gr = s.grow + summary_group<Bk>(grp) * 5 * (size_t)ng;
  unsigned* stage = s.ghist ? s.gstage + summary_group<Bk>(grp) * (size_t)(nb + 2) * (size_t)ng : nullptr;
#ifdef DHMC_USER_GENERATED_RNG
  dhmc_gq_rng rng;
  rng.key = dm_make_key(s.seed, (uint64_t)(s.chain_offset + c));
  rng.t = s.t0 + (unsigned)(j + 1) * (unsigned)s.thin - 1u;
#endif
  __syncthreads();
#pragma unroll 1
  for (int k = tid; k < ng; k += T) {
#ifdef DHMC_USER_GENERATED_RNG
    const double v = dhmc_user_generated(k, D, zq, params, &rng);
#else
    const double v = dhmc_user_generated(k, D, zq, params);
#endif
    if (j < 2 * n) {
      const int kk = j < n ? j + 1 : j - n + 1;        // place in its sequence (1-based); metric_reset / metric_push
      const double mean = kk == 1 ? 0.0 : gr[k], m2 = kk == 1 ? 0.0 : gr[ng + k];
      const double dlt = v - mean;
      const double mean1 = mean + dlt / (double)kk;
      const double m21 = m2 + dlt * (v - mean1);
      gr[k] = mean1; gr[ng + k] = m21;
      if (j == n - 1) { gr[2 * ng + k] = mean1; gr[3 * ng + k] = m21; }
    }
    if (s.gref) {
      const double below = v < s.gref[p * ng + k] ? 1.0 : 0.0;
      gr[4 * ng + k] = j == 0 ? below : gr[4 * ng + k] + below;
    }
    if (stage) {
      if (j == 0) {
#pragma unroll 1
        for (int c = 0; c < nb + 2; ++c) stage[(size_t)c * ng + k] = 0u;
      }
      const double t = __dmul_rn(__dsub_rn(v, s.glo[p * ng + k]), s.ginv_w[p * ng + k]);
      const int c = t < 0.0 ? 0 : !(t < (double)nb) ? nb + 1 : 1 + (int)t;
      stage[(size_t)c * ng + k] += 1u;
    }
  }
  __syncthreads();
}
// chain end (completed chains only), as summary_fold
template <class Bk>
__device__ __noinline__ void summary_gq_fold(const SummaryArgs* sp, int tid, int grp, size_t p) {
  constexpr int T = Bk::T;
  const SummaryArgs& s = *sp;
  const int ng = s.ng;
  const size_t cells = (size_t)s.nbins + 2;
  const double* gr = s.grow + summary_group<Bk>(grp) * 5 * (size_t)ng;
  const unsigned* stage = s.ghist ? s.gstage + summary_group<Bk>(grp) * cells * (size_t)ng : nullptr;
  double* acc = s.gacc + p * 5 * (size_t)ng;
#pragma unroll 1
  for (int k = tid; k < ng; k += T) {
    const double sh = s.gshift[p * ng + k];
    const double d0 = gr[2 * ng + k] - sh, d1 = gr[k] - sh, dc = 0.5 * (d0 + d1);
    atomicAdd(acc + k, d0 + d1);
    atomicAdd(acc + ng + k, d0 * d0 + d1 * d1);
    atomicAdd(acc + 2 * ng + k, gr[3 * ng + k] + gr[ng + k]);
    atomicAdd(acc + 3 * ng + k, dc);
    atomicAdd(acc + 4 * ng + k, dc * dc);
    if (s.gref) atomicAdd(s.gbelow + p * ng + k, (unsigned long long)gr[4 * ng + k]);
    if (stage) {
      unsigned long long* hist = s.ghist + (p * ng + k) * cells;
#pragma unroll 1
      for (size_t c = 0; c < cells; ++c) {
        const unsigned cnt = stage[c * ng + k];
        if (cnt) atomicAdd(hist + c, (unsigned long long)cnt);
      }
    }
  }
}
#endif
// kept draw j: sequence 0 is draws [0, n), sequence 1 draws [n, 2n); an odd last draw counts for the rank only
template <class Bk>
__device__ __noinline__ void summary_draw(const SummaryArgs* sp, double** slot_tab, int n_slots, int s_zq, int tid, int grp, int D,
                                         size_t p, int j DHMC_GQ_CHAIN_PARAM) {
  constexpr int EPL = sizeof(Bk::q) / sizeof(double), T = Bk::T;
  const SummaryArgs& s = *sp;
  Bk w = welford_view<Bk>(slot_tab, n_slots, tid, D);
  double* row = summary_row<Bk>(s, grp, D);
  const int n = s.n;
  w.ld_q(s_zq);
  if (j < 2 * n) {
    const int k = j < n ? j + 1 : j - n + 1;          // place in its sequence (1-based)
    if (k == 1) w.metric_reset(DHMC_METRIC_DIAGONAL);
    w.metric_push(DHMC_METRIC_DIAGONAL, k);
    if (j == n - 1) {                                 // sequence 0 is complete: park its mean and M2, free the slots
      const double* m = w.slot(n_slots - 1);
      const double* sv = w.slot(n_slots - 2);
#pragma unroll
      for (int e = 0; e < EPL; ++e) {
        const int i = tid + e * T;
        if (i < D) { row[i] = m[e * T]; row[D + i] = sv[e * T]; }
      }
    }
  }
  if (s.ref) {
    const double* ref = s.ref + p * D;
    const double* zq = slot_tab[s_zq] + tid;
#pragma unroll 1
    for (int e = 0; e < EPL; ++e) {
      const int i = tid + e * T;
      if (i < D) {
        const double below = zq[e * T] < ref[i] ? 1.0 : 0.0;
        row[2 * D + i] = j == 0 ? below : row[2 * D + i] + below;
      }
    }
  }
  if (s.hist) summary_hist_draw<Bk>(sp, slot_tab[s_zq] + tid, tid, grp, D, p, j);
#ifdef DHMC_USER_GENERATED
  if (s.ng) summary_gq_draw<Bk>(sp, slot_tab[s_zq], tid, grp, D, p, j DHMC_GQ_CHAIN_ARG);
#endif
}
// chain end (the chain completed the call): fold its two sequences into its problem's sums
template <class Bk>
__device__ __noinline__ void summary_fold(const SummaryArgs* sp, double** slot_tab, int n_slots, int tid, int grp, int Di, size_t p) {
  constexpr int EPL = sizeof(Bk::q) / sizeof(double), T = Bk::T;
  const SummaryArgs& s = *sp;
  const double* row = summary_row<Bk>(s, grp, Di);
  const double* m = slot_tab[n_slots - 1] + tid;
  const double* sv = slot_tab[n_slots - 2] + tid;
  const size_t D = (size_t)Di;
  double* acc = s.acc + p * 5 * D;
#pragma unroll 1
  for (int e = 0; e < EPL; ++e) {
    const int i = tid + e * T;
    if (i < Di) {
      const double sh = s.shift[p * D + i];
      const double d0 = row[i] - sh, d1 = m[e * T] - sh, dc = 0.5 * (d0 + d1);   // μ_c: the mean of both sequences
      atomicAdd(acc + i, d0 + d1);
      atomicAdd(acc + D + i, d0 * d0 + d1 * d1);
      atomicAdd(acc + 2 * D + i, row[D + i] + sv[e * T]);
      atomicAdd(acc + 3 * D + i, dc);
      atomicAdd(acc + 4 * D + i, dc * dc);
      if (s.ref) atomicAdd(s.below + p * D + i, (unsigned long long)row[2 * D + i]);
    }
  }
  if (s.hist) summary_hist_fold<Bk>(sp, tid, grp, Di, p);
#ifdef DHMC_USER_GENERATED
  if (s.ng) summary_gq_fold<Bk>(sp, tid, grp, p);
#endif
  if (tid == 0) atomicAdd(s.chains + p, 1ull);
}

template <int EPL, int FAM, int W, bool DN, int G = 1, bool DP = false>
__global__ void __launch_bounds__(32 * W * G, G > 1 ? 1 : min_ctas(W, EPL)) k_nuts(const KArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  DeviceBackend<EPL, FAM, W, DN, G, DP> b;
  setup_backend(b, a, smem);
  int* s_misc = reinterpret_cast<int*>(smem + smem_layout(W, a.n_sm, b.stride, (size_t)a.xs_doubles, DP ? a.levels : kStdLevels,
                                                          DP ? a.ntab : kStdTab, decltype(b)::kFused ? a.red_groups : 1).misc_off);   // one chain per CTA: the queue's broadcast slot
  for (;;) {
    int c;
    if constexpr (G > 1) {
      if (a.pooled || a.batch_k) c = next_pooled_group(b, a.counter, a.chain_begin);   // the CTA takes a whole metric group / 8 chains of one problem
      else c = next_chain_group(b, a.counter, a.chain_begin);
    } else {
      c = next_chain(a.counter, s_misc, a.chain_begin);
    }
    if (c >= a.chain_end) break;
    load_chain(b, a, c, false);
    NutsMachine<DeviceBackend<EPL, FAM, W, DN, G, DP>> m(b, dm_make_key(a.seed, (uint64_t)(a.chain_offset + c)),
                                           a.max_depth, a.min_delta, a.n_slots);
    DrawSink<EPL, FAM, W, DN, G, DP> sink{b, a, c};
    const double eps_next = m.run(a.t0, a.N, a.eps[c], a.cfg, a.p_override,
                                  a.dir_override ? a.dir_override + c : nullptr, sink);
    const size_t base = (size_t)c * a.D;
    const bool halted = (m.status & DHMC_CHAIN_LEAPFROG_NONFINITE) != 0;   // the chain keeps the state the call found it in
    if (!halted) {
      store_vec(b, a.q, b.q, base, a.D);
      store_vec(b, a.g, b.g, base, a.D);
      if (a.cfg.metric == DHMC_METRIC_DIAGONAL) store_vec(b, a.minv, b.minv, base, a.D);
    }
    if (b.tid == 0) {
      if (!halted) {
        a.lq[c] = b.lq;
        a.eps[c] = eps_next;
      }
      if (m.status) atomicOr(a.status + c, m.status);
      atomicAdd(a.total_steps, (unsigned long long)m.steps_out);
    }
    if (a.summary && !(m.status & (DHMC_CHAIN_BAD_STEPSIZE | DHMC_CHAIN_LEAPFROG_NONFINITE)))
      summary_fold<DeviceBackend<EPL, FAM, W, DN, G, DP>>(a.summary, b.slot_tab, b.n_slots, b.tid, b.grp, a.D, summary_problem(a, c));
    if constexpr (G > 1) { if (a.pooled || a.batch_k) b.coop_finish(); }     // group fetch: the group leaves together, then the CTA takes the next one
  }
  b.coop_finish();
}

// ------------------------------------------------------------------ k_search
template <int EPL, int FAM, int W, bool DN, int G = 1, bool DP = false>
__global__ void __launch_bounds__(32 * W * G, G > 1 ? 1 : min_ctas(W, EPL)) k_search(const KArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  DeviceBackend<EPL, FAM, W, DN, G, DP> b;
  setup_backend(b, a, smem);
  int* s_misc = reinterpret_cast<int*>(smem + smem_layout(W, a.n_sm, b.stride, (size_t)a.xs_doubles, DP ? a.levels : kStdLevels,
                                                          DP ? a.ntab : kStdTab, decltype(b)::kFused ? a.red_groups : 1).misc_off);   // one chain per CTA: the queue's broadcast slot
  for (;;) {
    int c;
    if constexpr (G > 1) {
      if (a.pooled || a.batch_k) c = next_pooled_group(b, a.counter, a.chain_begin);
      else c = next_chain_group(b, a.counter, a.chain_begin);
    } else {
      c = next_chain(a.counter, s_misc, a.chain_begin);
    }
    if (c >= a.chain_end) break;
    load_chain(b, a, c, false);
    NutsMachine<DeviceBackend<EPL, FAM, W, DN, G, DP>> m(b, dm_make_key(a.seed, (uint64_t)(a.chain_offset + c)),
                                           a.max_depth, a.min_delta, a.n_slots);
    const double eps = m.find_initial_stepsize(a.s_init, a.s_thresh, a.s_maxiter, a.p_override);
    if (b.tid == 0) {
      a.eps[c] = eps;
      if (m.status) atomicOr(a.status + c, m.status);
    }
    if constexpr (G > 1) { if (a.pooled || a.batch_k) b.coop_finish(); }
  }
  b.coop_finish();
}

// ------------------------------------------------------------------ k_leapfrog
// Streaming leapfrog: reads q, p, ∇ℓ, M⁻¹ (32·D B), writes q′, p′, ∇ℓ′ (24·D B).
template <int EPL, int FAM, int W, bool DN>
__global__ void __launch_bounds__(32 * W, min_ctas(W, EPL)) k_leapfrog(const KArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  DeviceBackend<EPL, FAM, W, DN> b;
  setup_backend(b, a, smem);
  for (long c = a.chain_begin + blockIdx.x; c < a.chain_end; c += gridDim.x) {
    load_chain(b, a, c, true);
    const double eps = a.lf_sign >= 0 ? a.eps[c] : -a.eps[c];
    int flags = 0;
    bool halted = false;
    for (int s = 0; s < a.lf_steps; ++s) {
      // @argcheck isfinite(Q.ℓq), hamiltonian.jl:276 (after a non-finite position the reference has raised already)
      if (!dm_isfinite(b.lq) && !(flags & 1)) { halted = true; break; }
      (void)b.leapfrog(eps, &flags);
    }
    const size_t base = (size_t)c * a.D;
    if (!halted) {                         // a halted chain keeps the state the call found it in
      store_vec(b, a.q, b.q, base, a.D);
      store_vec(b, a.p, b.p, base, a.D);
      store_vec(b, a.g, b.g, base, a.D);
    }
    if (b.tid == 0) {
      if (!halted) a.lq[c] = b.lq;
      if (flags & 1) atomicOr(a.status + c, (int)DHMC_CHAIN_NONFINITE_Q);
      if (halted) atomicOr(a.status + c, (int)DHMC_CHAIN_LEAPFROG_NONFINITE);
    }
    if (W > 1) __syncthreads();
  }
}

// ------------------------------------------------------------------ k_eval
template <int EPL, int FAM, int W>
__global__ void __launch_bounds__(32 * W, min_ctas(W, EPL)) k_eval(const KArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  DeviceBackend<EPL, FAM, W> b;
  setup_backend(b, a, smem);
  for (long c = a.chain_begin + blockIdx.x; c < a.chain_end; c += gridDim.x) {
    load_chain(b, a, c, false);
    double qbad = 0.0;
    if (a.randomize) {
      const dm_rng_key key = dm_make_key(a.seed, (uint64_t)(a.chain_offset + c));
#pragma unroll
      for (int e = 0; e < EPL; ++e) {
        const int i = b.tid + e * b.T;
        b.q[e] = i < a.D ? dm_uniform_elem(key, DHMC_STREAM_Q0, 0, (uint32_t)i) * 4 - 2 : 0.0;
      }
    }
#pragma unroll
    for (int e = 0; e < EPL; ++e) if (!dm_isfinite(b.q[e])) qbad = 1.0;
    // raw (unsanitised) validity for the strict check, hamiltonian.jl:205-215
    int flags = 0;
    double ks;
    b.eval_model(false, 0.0, qbad, &ks, &flags);
    const size_t base = (size_t)c * a.D;
    store_vec(b, a.q, b.q, base, a.D);
    store_vec(b, a.g, b.g, base, a.D);
    if (b.tid == 0) {
      a.lq[c] = b.lq;
      if (a.strict && (flags & (1 | 4))) atomicOr(a.status + c, (int)DHMC_CHAIN_BAD_INITIAL);
    }
    if (W > 1) __syncthreads();
  }
}

// ------------------------------------------------------------------ k_phase
template <int EPL, int FAM, int W, bool DN>
__global__ void __launch_bounds__(32 * W, min_ctas(W, EPL)) k_phase(const KArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  DeviceBackend<EPL, FAM, W, DN> b;
  setup_backend(b, a, smem);
  for (long c = a.chain_begin + blockIdx.x; c < a.chain_end; c += gridDim.x) {
    load_chain(b, a, c, true);
    const double H = b.phase_logdensity();
    if (b.tid == 0) a.out_phase[c] = H;
    if (W > 1) __syncthreads();
  }
}


// ------------------------------------------------------------------ kernel lookup
enum KernelId { K_NUTS, K_SEARCH, K_LEAPFROG, K_EVAL, K_PHASE };

// supported (warps per chain, elements per thread) layouts
inline bool layout_supported(int W, int epl) {
  if (W == 1) return epl == 1 || epl == 2 || epl == 4 || epl == 8;
  if (W == 2 || W == 4) return epl == 4 || epl == 8;
  if (W == 8) return epl == 4 || epl == 8 || epl == 16 || epl == 32;       // dim <= 8192
  return false;
}
// dense (Symmetric metric) kernels are instantiated for every layout (D <= 2048; memory: 3·D² doubles per chain)
constexpr bool dense_layout(int W, int EPL) { return W >= 1 && EPL >= 1; }
constexpr int kPack = 8;            // packed chain groups: chains per CTA (logistic family, dim <= 256)
// packed layouts for dim <= 256: one warp per chain, up to 8 elements per lane
constexpr bool packed_layout(int W, int EPL) { return W == 1; }

// which subset of a family's kernels a translation unit instantiates (build parallelism):
//   PART 0: one chain per CTA;  PART 1: packed groups, tensor-core likelihood;
//   PART 3: one chain per CTA, max_depth > 12 (k_nuts / k_search only)
template <int EPL, int FAM, int W, int PART>
const void* kernel_ptr(KernelId k, bool dense) {
  if constexpr (PART == 3) {        // max_depth > 12: one chain per CTA, slot pool with spill words
    if (dense) {
      if constexpr (dense_layout(W, EPL)) {
        if (k == K_NUTS) return (const void*)k_nuts<EPL, FAM, W, true, 1, true>;
        if (k == K_SEARCH) return (const void*)k_search<EPL, FAM, W, true, 1, true>;
      }
      return nullptr;
    }
    if (k == K_NUTS) return (const void*)k_nuts<EPL, FAM, W, false, 1, true>;
    if (k == K_SEARCH) return (const void*)k_search<EPL, FAM, W, false, 1, true>;
    return nullptr;
  } else if constexpr (PART == 1) {
    if constexpr (FAM == DHMC_FAMILY_LOGISTIC && packed_layout(W, EPL)) {
      if (k == K_NUTS) return dense ? (const void*)k_nuts<EPL, FAM, W, true, kPack> : (const void*)k_nuts<EPL, FAM, W, false, kPack>;
      if (k == K_SEARCH) return dense ? (const void*)k_search<EPL, FAM, W, true, kPack> : (const void*)k_search<EPL, FAM, W, false, kPack>;
    }
    return nullptr;
  } else {
    if (dense) {
      if constexpr (dense_layout(W, EPL)) {
        switch (k) {
          case K_NUTS: return (const void*)k_nuts<EPL, FAM, W, true>;
          case K_SEARCH: return (const void*)k_search<EPL, FAM, W, true>;
          case K_LEAPFROG: return (const void*)k_leapfrog<EPL, FAM, W, true>;
          case K_PHASE: return (const void*)k_phase<EPL, FAM, W, true>;
          default: break;
        }
      } else {
        return nullptr;
      }
    }
    switch (k) {
      case K_NUTS: return (const void*)k_nuts<EPL, FAM, W, false>;
      case K_SEARCH: return (const void*)k_search<EPL, FAM, W, false>;
      case K_LEAPFROG: return (const void*)k_leapfrog<EPL, FAM, W, false>;
      case K_EVAL: return (const void*)k_eval<EPL, FAM, W>;
      default: return (const void*)k_phase<EPL, FAM, W, false>;
    }
  }
}
template <int FAM, int PART>
const void* family_kernel_ptr(int W, int epl, KernelId k, bool dense) {
  switch (W * 64 + epl) {
    case 1 * 64 + 1: return kernel_ptr<1, FAM, 1, PART>(k, dense);
    case 1 * 64 + 2: return kernel_ptr<2, FAM, 1, PART>(k, dense);
    case 1 * 64 + 4: return kernel_ptr<4, FAM, 1, PART>(k, dense);
    case 1 * 64 + 8: return kernel_ptr<8, FAM, 1, PART>(k, dense);
    case 2 * 64 + 4: return kernel_ptr<4, FAM, 2, PART>(k, dense);
    case 2 * 64 + 8: return kernel_ptr<8, FAM, 2, PART>(k, dense);
    case 4 * 64 + 4: return kernel_ptr<4, FAM, 4, PART>(k, dense);
    case 4 * 64 + 8: return kernel_ptr<8, FAM, 4, PART>(k, dense);
    case 8 * 64 + 4: return kernel_ptr<4, FAM, 8, PART>(k, dense);
    case 8 * 64 + 8: return kernel_ptr<8, FAM, 8, PART>(k, dense);
    case 8 * 64 + 16: return kernel_ptr<16, FAM, 8, PART>(k, dense);
    case 8 * 64 + 32: return kernel_ptr<32, FAM, 8, PART>(k, dense);
  }
  return nullptr;
}

}  // namespace dhmc
