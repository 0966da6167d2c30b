/* dhmc.h — C ABI of the H100-native many-chain NUTS engine (libdhmc_b200.so).
 *
 * Drop-in boundary for the sampler path of tpapp/DynamicHMC.jl (SURVEY.md §8b):
 * host code (Julia via ccall, or the Python mirror in dynamichmc.jl_b200/)
 * keeps the mcmc_with_warmup / LogDensityProblems surface and calls these entry
 * points; everything numeric runs in hand-written sm_90a CUDA.  Plain pointers
 * and sizes only.  All functions return a status (0 = ok) unless noted.
 *
 * Conventions
 *  - B = n_chains on this handle, D = dim.  Every per-chain vector argument is
 *    [D, B] column-major (chain-major: element i of chain c at c*D + i), which
 *    is Julia's Matrix{Float64}(D, B); draws are [D, N, B] column-major so that
 *    results[k].posterior_matrix (mcmc.jl:230,275) is a zero-copy view.
 *  - dhmc_tree_stats is bit-compatible with TreeStatisticsNUTS (NUTS.jl:208-221).
 *  - Host pointers unless the function name ends in _dev.
 *  - One handle = one device + one stream; calls are synchronous and not
 *    thread-safe per handle (the reference call is single-threaded too).
 *  - Numerical per-chain failures never abort other chains: they set bits in the
 *    per-chain status word and the call returns DHMC_ENUMERIC (the Julia shim
 *    re-throws DynamicHMCError, utilities.jl:17-27, with the chain ids).
 */
#ifndef DHMC_H
#define DHMC_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum {
  DHMC_OK = 0,
  DHMC_EARG = 1,     /* -> ArgumentError (@argcheck sites: NUTS.jl:190-191,
                        stepsize.jl:31-33,108-111, mcmc.jl:191-192) */
  DHMC_ENUMERIC = 2, /* -> DynamicHMCError (hamiltonian.jl:203,213,215;
                        stepsize.jl:58,78) for at least one chain */
  DHMC_ECUDA = 3,
  DHMC_ENOMEM = 4,
  DHMC_ENCCL = 5
};

/* per-chain status bits (dhmc_chain_status) */
enum {
  DHMC_CHAIN_BAD_INITIAL = 1,   /* evaluate_ℓ(strict) failed, hamiltonian.jl:212-215 */
  DHMC_CHAIN_SEARCH_FAILED = 2, /* find_initial_stepsize, stepsize.jl:58 / :78 */
  DHMC_CHAIN_NONFINITE_Q = 4,   /* evaluate_ℓ: non-finite position, hamiltonian.jl:203 */
  DHMC_CHAIN_BAD_ACCEPTANCE = 8, /* adapt_stepsize @argcheck 0 ≤ a ≤ 1, stepsize.jl:148 */
  DHMC_CHAIN_NOT_POSDEF = 16,    /* cholesky(inv(M⁻¹)) failed, hamiltonian.jl:73 (PosDefException) */
  DHMC_CHAIN_BAD_STEPSIZE = 32,  /* initial_adaptation_state @argcheck ϵ > 0, stepsize.jl:135 (chain left untouched) */
  DHMC_CHAIN_LEAPFROG_NONFINITE = 64 /* leapfrog @argcheck isfinite(Q.ℓq), hamiltonian.jl:276 ("leapfrog called from
                                        non-finite log density"; the shims raise ArgumentError): a leapfrog would start
                                        from ℓ = −∞, e.g. after ℓ(q₀) = −∞ or a non-divergent leaf at ℓ = −∞ (min_Δ = −Inf,
                                        or π₀ = −∞ makes Δ NaN).  The chain stops and keeps the state the call found it in. */
};

/* log-density family ids: see include/dhmc_models.h */
enum { DHMC_METRIC_NOTHING = 0, DHMC_METRIC_DIAGONAL = 1, DHMC_METRIC_SYMMETRIC = 2,
       /* NOT reference semantics (the reference adapts every chain on its own window, mcmc.jl:282): the optional exchange of
        * SURVEY.md §8e.  Every group of 8 consecutive GLOBAL chains ends the window with ONE dense metric estimated from the
        * pooled draws of the group (per-chain streaming moments merged in a fixed order, same shrinkage λ).  With a shared
        * metric the packed kernels run M⁻¹·[8 vectors] as a true FP64 tensor-core GEMM and read the metric once per group.
        * Needs n_chains and chain_offset to be multiples of 8. */
       DHMC_METRIC_SYMMETRIC_POOLED = 3 };

typedef struct dhmc_handle dhmc_handle;

/* Flattened NUTS(; max_depth, min_Δ) (NUTS.jl:178-195) + problem shape. */
typedef struct {
  int32_t device;            /* CUDA device ordinal */
  int32_t family;            /* DHMC_FAMILY_* (LogDensityProblems model id) */
  int64_t dim;               /* LogDensityProblems.dimension(ℓ) */
  int64_t n_chains;          /* chains resident on this handle (local shard) */
  int64_t chain_offset;      /* global id of local chain 0 (RNG key), §8e */
  uint64_t seed;             /* RNG seed (stands in for the rng argument) */
  int32_t max_depth;         /* NUTS.max_depth, 0 < . <= 32 (MAX_DIRECTIONS_DEPTH, trees.jl:10) */
  int32_t threads_per_chain; /* 0 = auto; 32..256, power of two.  LOGISTIC, dim <= 256: auto also packs 8 chains
                              * per CTA (shared passes over X, same results); an explicit value keeps one chain per CTA */
  double min_delta;          /* NUTS.min_Δ < 0 */
  int32_t ctas_per_sm;       /* 0 = auto */
  int32_t reserved;
} dhmc_config;

/* TreeStatisticsNUTS — NUTS.jl:208-221 (56 bytes) */
typedef struct {
  double pi;              /* π: logdensity(H, ζ) of the selected point */
  int64_t depth;
  int64_t left, right;    /* termination::InvalidTree, trees.jl:180-202 */
  double acceptance_rate;
  int64_t steps;
  uint32_t directions;    /* Directions.flags, trees.jl:19-21 */
  uint32_t pad;
} dhmc_tree_stats;

/* DualAveraging(; δ, γ, κ, t₀) — stepsize.jl:98-118 */
typedef struct { double delta, gamma, kappa; int32_t t0; int32_t pad; } dhmc_dual_averaging;

/* ---- lifecycle ------------------------------------------------------- */
int dhmc_create(const dhmc_config* cfg, dhmc_handle** out);
int dhmc_destroy(dhmc_handle* h);
/* Message of the last failing call on h (h == NULL: last dhmc_create failure).
 * Valid until the next call. */
const char* dhmc_last_error(dhmc_handle* h);
/* threads per chain (canonical reduction width T) and elements per thread */
int dhmc_get_layout(dhmc_handle* h, int32_t* threads_per_chain, int32_t* elems_per_thread);

/* ---- problem: replaces the ℓ argument (LogDensityProblems object) ------ */
/* params: DIAG_NORMAL [mu(D), prec(D)]; LOGISTIC [N, X row-major (N*D), y (N)] with an integer 1 <= N < 2^31 and
 * 0 <= y <= 1; STD_NORMAL / FUNNEL: n == 0; USER: any block of doubles, handed to the user's formulas as `params`.
 * Everything is checked before anything is allocated; on any error the previous problem (one problem or a batch) stays
 * in effect. */
int dhmc_set_problem(dhmc_handle* h, const double* params, size_t n);
/* Problem batch: n_problems posteriors of the handle's family and dimension, each with its own parameter block, on one
 * handle.  Problem p's block is params + p*n_per_problem, in the format of dhmc_set_problem (LOGISTIC: every block has the
 * same N).  Global chain g samples problem g / chains_per_problem, so chains [p*K, (p+1)*K) of a batch are bit-identical to
 * a single-problem handle that holds problem p with chain_offset = p*K (K = chains_per_problem); every rank of a sharded
 * run holds all blocks.  The handle's global chain ids must all be < n_problems * chains_per_problem.  Packed LOGISTIC
 * handles (automatic layout, dim <= 256) run 8 chains of one problem per CTA: chains_per_problem, chain_offset and
 * n_chains must be multiples of 8 (threads_per_chain = 32 lifts this).  STD_NORMAL and FUNNEL have no parameters and
 * refuse a batch.  Everything is checked before anything is allocated; on any error the previous problem stays in
 * effect.  dhmc_set_problem returns the handle to one problem. */
int dhmc_set_problems(dhmc_handle* h, const double* params, size_t n_per_problem, int64_t n_problems,
                      int64_t chains_per_problem);
/* Ragged problem batch: the same with blocks of different lengths — problem p's block is
 * params[block_offsets[p] .. block_offsets[p+1]), block_offsets[0] == 0 and the offsets strictly increase.  LOGISTIC:
 * every block is [N_p, X_p (N_p*D), y_p (N_p)] with its own integer 1 <= N_p < 2^31 that matches the block's length
 * (per-unit regressions with any number of rows each).  Each problem's data take space of their own size (sum of N_p,
 * not n_problems * max N_p), and a packed CTA streams only its problem's row blocks.  USER: blocks of any positive
 * length (the formulas do not receive the length: a model that needs it stores it in its block).  DIAG_NORMAL: every
 * block is 2*D long.  Every other rule, including the bit-identity to single-problem handles, is that of
 * dhmc_set_problems. */
int dhmc_set_problems_ragged(dhmc_handle* h, const double* params, const size_t* block_offsets, int64_t n_problems,
                             int64_t chains_per_problem);
/* The user's own ℓ (LogDensityProblems.logdensity_and_gradient, call site hamiltonian.jl:204) as device code: a library
 * built from a model header (include/dhmc_models.h "the model header contract"; `make -C dynamichmc.jl_b200/csrc user
 * USER_HEADER=… USER_LIB=…`) carries family DHMC_FAMILY_USER (and only that family).  Copies the model's DHMC_USER_NAME
 * (NUL-terminated, truncated to cap) and returns DHMC_OK, or DHMC_EARG in a library without a user model. */
int dhmc_user_family_name(char* name, size_t cap);
/* Whether this library carries the kernels of `family` (the stock library: the four shipped families; a user-model
 * library: DHMC_FAMILY_USER only).  dhmc_create refuses an absent family with DHMC_EARG. */
int dhmc_family_available(int32_t family, int32_t* available);
/* Generated quantities (include/dhmc_models.h): G = dhmc_user_ngq(dim) functions of a position that a user model may
 * declare (DHMC_USER_GENERATED), e.g. the centred effects of a non-centred model.  dhmc_create refuses a model whose
 * G(dim) lies outside [1, DHMC_MAX_GENERATED].  They never affect sampling.  dhmc_generated_count gives G, 0 for the
 * shipped families and for user models without them. */
#define DHMC_MAX_GENERATED 8192
int dhmc_generated_count(dhmc_handle* h, int32_t* G);
/* The same G for dimension dim without a handle (no device needed): DHMC_EARG in a library without a user model. */
int dhmc_user_generated_count(int64_t dim, int32_t* G);
/* The G quantities of n·n_problems points: theta [D, n, n_problems] and out [G, n, n_problems], column-major; problem
 * first_problem + j of the handle's batch (a handle without a batch is one problem) owns points j·n … (j+1)·n − 1 and
 * lends them its parameter block.  So the draws [D, N, B] of a handle that holds whole problems are an input as they are
 * (n = N·chains per problem), and so are per-problem references [D, P] (n = 1).  Evaluated on the device, one chain width
 * of threads per point.  DHMC_EARG before anything runs for G = 0, NULL pointers, n < 1, n_problems < 1 or a problem
 * range outside the batch.  dhmc_generated takes host arrays, dhmc_generated_dev device arrays. */
int dhmc_generated(dhmc_handle* h, const double* theta, int64_t n, int64_t first_problem, int64_t n_problems, double* out);
int dhmc_generated_dev(dhmc_handle* h, const double* theta, int64_t n, int64_t first_problem, int64_t n_problems,
                       double* out);
/* Random generated quantities (include/dhmc_models.h, DHMC_USER_GENERATED_RNG), e.g. posterior predictive replicates:
 * *random = 1 when the model's quantities draw numbers from the keyed streams, else 0.  dhmc_user_generated_random needs
 * no handle (DHMC_EARG in a library without a user model).  dhmc_generated(_dev) refuses such a model with DHMC_EARG. */
int dhmc_generated_random(dhmc_handle* h, int32_t* random);
int dhmc_user_generated_random(int32_t* random);
/* dhmc_generated with a key per point: chain [n, n_problems] (int64 global chain ids) and transition [n, n_problems] (uint32
 * transition counters), on the same side as theta; point i draws its numbers under (the handle's seed, chain[i]) and
 * transition[i].  The kept draw j of a sampling call that started at transition count t0 with thinning `thin`, of local
 * chain c, has chain = chain_offset + c and transition = t0 + (j + 1)·thin − 1 (uint32 arithmetic): with those keys the
 * quantities equal the summary's.  Layout and problem rules are dhmc_generated's.  DHMC_EARG before anything runs for
 * NULL keys, any argument dhmc_generated rejects, and (host variant) a chain id outside [0, 2^56).  On a model whose
 * quantities are deterministic the keys are ignored and the output is dhmc_generated's, bit for bit. */
int dhmc_generated_keyed(dhmc_handle* h, const double* theta, int64_t n, int64_t first_problem, int64_t n_problems,
                         const int64_t* chain, const uint32_t* transition, double* out);
int dhmc_generated_keyed_dev(dhmc_handle* h, const double* theta, int64_t n, int64_t first_problem, int64_t n_problems,
                             const int64_t* chain, const uint32_t* transition, double* out);

/* ---- state: initialization = (q, κ, ϵ), mcmc.jl:111-132 ---------------- */
/* q: [D,B]; evaluates ℓ, ∇ℓ strictly (initialize_warmup_state, mcmc.jl:129-132). */
int dhmc_set_position(dhmc_handle* h, const double* q);
/* random_position, mcmc.jl:108: q ~ U[-2,2]^D per chain from the handle's RNG. */
int dhmc_random_position(dhmc_handle* h);
/* κ = GaussianKineticEnergy(Diagonal(minv)) (hamiltonian.jl:80); minv [D,B],
 * or [D] broadcast to all chains when broadcast != 0; NULL = identity (:87). */
int dhmc_set_metric(dhmc_handle* h, const double* minv, int broadcast);
/* κ = GaussianKineticEnergy(Symmetric M⁻¹) (hamiltonian.jl:73): minv is [D,D,B], or
 * [D,D] for all chains when broadcast != 0.  W = cholesky(inv(M⁻¹)).L is computed on the
 * device; a matrix that is not positive definite sets DHMC_CHAIN_NOT_POSDEF. */
int dhmc_set_metric_dense(dhmc_handle* h, const double* minv, int broadcast);
int dhmc_get_metric_dense(dhmc_handle* h, double* minv /* [D,D,B] */);
int dhmc_metric_is_dense(dhmc_handle* h, int32_t* dense);
/* ϵ per chain [B], or one value for all chains when broadcast != 0. */
int dhmc_set_stepsize(dhmc_handle* h, const double* eps, int broadcast);
/* Momentum of the phase point used by dhmc_leapfrog / dhmc_phase_logdensity. */
int dhmc_set_momentum(dhmc_handle* h, const double* p);
/* Any output pointer may be NULL.  q, grad, minv, p: [D,B]; lq, eps: [B].  minv is the
 * DIAGONAL metric; with a Symmetric metric use dhmc_get_metric_dense. */
int dhmc_get_state(dhmc_handle* h, double* q, double* lq, double* grad, double* minv,
                   double* eps, double* p);
/* Status words of the most recent state-changing call (they are reset when a call starts). */
int dhmc_chain_status(dhmc_handle* h, int32_t* status /* [B] */);
/* Number of transitions already drawn per chain (RNG counter); get/set make the
 * (q, κ, ϵ, counter) tuple a checkpoint (mcmc_keep_warmup/mcmc_steps, §8f). */
int dhmc_get_transition_count(dhmc_handle* h, uint32_t* t);
int dhmc_set_transition_count(dhmc_handle* h, uint32_t t);

/* ---- fine-grained path (parity tests) --------------------------------- */
/* leapfrog(H, z, ±ϵ) n_steps times on every chain — hamiltonian.jl:273-282.
 * sign = +1 / -1 (NUTS.jl:28-31). */
int dhmc_leapfrog(dhmc_handle* h, int32_t n_steps, int32_t sign);
/* logdensity(H, z) per chain — hamiltonian.jl:251-256.  out: [B]. */
int dhmc_phase_logdensity(dhmc_handle* h, double* out);
/* One NUTS transition per chain at the current (q, κ, ϵ), no adaptation —
 * sample_tree, NUTS.jl:232-241.  p [D,B] and directions [B] override the RNG
 * draws when non-NULL (the reference's p= / directions= keywords). */
int dhmc_sample_tree(dhmc_handle* h, const double* p, const uint32_t* directions,
                     dhmc_tree_stats* stats /* [B] */);

/* ---- coarse path: warmup stages and inference -------------------------- */
/* warmup(::InitialStepsizeSearch) — mcmc.jl:134-148, stepsize.jl:46-85. */
int dhmc_find_initial_stepsize(dhmc_handle* h, double initial_eps, double log_threshold,
                               int32_t maxiter_crossing);
/* warmup(::TuningNUTS{M}) — mcmc.jl:258-286.  da == NULL: FixedStepsize
 * (stepsize.jl:181-189).  metric: DHMC_METRIC_NOTHING | _DIAGONAL | _SYMMETRIC.  lambda is
 * the shrinkage of regularize_M⁻¹ (mcmc.jl:218-221); identity for Diagonal (:223).
 * Outputs may be NULL: posterior [D,N,B], stats/eps_used/logdens [N,B]. */
int dhmc_warmup_stage(dhmc_handle* h, int32_t N, int32_t metric, const dhmc_dual_averaging* da,
                      double lambda, double* posterior, dhmc_tree_stats* stats,
                      double* eps_used, double* logdens);
/* mcmc — mcmc.jl:366-381: N transitions at the adapted (κ, ϵ). */
int dhmc_mcmc(dhmc_handle* h, int32_t N, double* posterior, dhmc_tree_stats* stats,
              double* logdens);
/* mcmc from host positions: WarmupState.Q given by the caller (q: [D,B], evaluated strictly
 * like dhmc_set_position) with the current (κ, ϵ) — mcmc_steps / mcmc_next_step,
 * mcmc.jl:335-351.  Upload, evaluation, sampling and download are pipelined by chain chunks. */
int dhmc_mcmc_from(dhmc_handle* h, const double* q, int32_t N, double* posterior,
                   dhmc_tree_stats* stats, double* logdens);
/* mcmc with a thinned output (§8f-3): N transitions, every thin-th one is kept, outputs are [D, N/thin, B] resp.
 * [N/thin, B].  q == NULL continues from the resident positions, else as dhmc_mcmc_from.
 * All host-output calls: while the kept draws fit in HBM they are staged there and copied chunk by chunk, overlapped with the
 * sampling of the next chunk (page-locked buffers — cudaHostAlloc / cudaHostRegister / dhmc_host_alloc — make the copies
 * asynchronous); when they do not fit, the sampling kernel writes the (page-locked, if need be on the fly) host buffer
 * directly, so N is not bounded by device memory. */
int dhmc_mcmc_thinned(dhmc_handle* h, const double* q, int32_t N, int32_t thin, double* posterior,
                      dhmc_tree_stats* stats, double* logdens);
/* Page-locked, device-mapped host memory on the NUMA node of the handle's GPU (for the output buffers above). */
int dhmc_host_alloc(dhmc_handle* h, size_t bytes, void** out, int32_t* numa_node);
int dhmc_host_free(dhmc_handle* h, void* p);
/* Same with DEVICE output pointers (draws stay in HBM for an NCCL all-gather). */
int dhmc_mcmc_dev(dhmc_handle* h, int32_t N, double* posterior, dhmc_tree_stats* stats,
                  double* logdens);

/* ---- streaming posterior summary (DESIGN.md §4.4): sample without keeping draws ------------------------------------
 * dhmc_mcmc_summary takes N transitions at the adapted (κ, ϵ), exactly as dhmc_mcmc does (same draws, same final state, same
 * transition count, status words, return code), keeps every thin-th one and folds the kept draws into per-(problem,
 * parameter) statistics on the device instead of writing them out.  Definitions: chain c keeps n_keep = N / thin draws;
 * sequence 0 is the first n = ⌊n_keep/2⌋ of them, sequence 1 the next n (an odd n_keep drops its last draw from the
 * moments).  Problem p (a handle without a batch is one problem, P = 1) pools its M local chains that completed the call,
 * m = 2M sequences; a chain whose status has DHMC_CHAIN_BAD_STEPSIZE or DHMC_CHAIN_LEAPFROG_NONFINITE is left out.  Per
 * parameter d:
 *   mean   mean of the 2n·M draws (= the mean of the sequence means μ_s)
 *   sd     √ of their pooled variance (Σ_s M2_s + n·Σ_s (μ_s − μ̄)²) / (m·n − 1)
 *   rhat   split-R̂ as dhmc_ess_rhat_problems_dev: W = Σ_s M2_s / (m(n − 1)), var⁺ = (n − 1)/n·W + var(μ_s), √(var⁺ / W)
 *   mcse   √(var(μ_c) / M), μ_c = chain c's mean over its 2n draws (between-chain batch means; NaN for M < 2)
 *   ess    sd² / mcse² (NaN for M < 2 or var⁺ = 0).  A batch-means estimate that becomes precise with many chains, NOT the
 *          Geyer ESS of dhmc_ess_rhat_dev.
 *   rank   with a reference [D, P]: the number of the problem's kept draws (all n_keep of every local chain) with
 *          θ_d < reference[d, p], an exact integer — the rank statistic of simulation-based calibration (−1 without one)
 *   draws  n_keep·M, the rank's denominator
 * A problem with no local chain gets NaN everywhere (rank 0, draws 0).  Quantiles: dhmc_mcmc_summary_histogram below.
 *
 * Generated quantities: on a handle whose model has G > 0 (dhmc_generated_count), every array below has R = D + G rows
 * in place of D — the D parameters, then the G quantities g(θ) of every kept draw, with the same definitions (the shift
 * of the quantities' sums is g of the position the parameters' shift is).  reference, lo, hi [R, P], record [F, R, P],
 * counts [nbins + 2, R, P]; dhmc_summary_merge, dhmc_summary_finish and dhmc_histogram_quantiles take R as their row
 * count.  A non-finite g(θ) is folded as it is and sets no status bit.  Random quantities (dhmc_generated_random) are
 * ordinary rows: kept draw j of global chain g is evaluated under the key (seed, g) and t = t0 + (j + 1)·thin − 1, those
 * of dhmc_generated_keyed; their shift is g of the shift position under the key (global id of the problem's first local
 * chain, t0), which only keeps the sums free of cancellation.  Their reference cells are given by the caller (a NaN cell
 * counts nothing: v < NaN is false); the arena grows by 2·P doubles for the shift's keys.
 *
 * The record is [DHMC_SUMMARY_FIELDS, D, P] column-major (the fields of (d, p) at (p·D + d)·F) and holds mergeable
 * quantities in absolute terms: the records of shards of one run (handles with different chain_offset, ranks) combine with
 * dhmc_summary_merge into the record one handle holding every chain would produce, up to rounding. */
enum {
  DHMC_SUMMARY_CHAINS = 0,   /* M: chains that contributed */
  DHMC_SUMMARY_NKEEP = 1,    /* n_keep: kept draws per chain */
  DHMC_SUMMARY_MEAN = 2,     /* μ̄: mean of the sequence means */
  DHMC_SUMMARY_SS_SEQ = 3,   /* Σ_s (μ_s − μ̄)² over the 2M sequences */
  DHMC_SUMMARY_M2 = 4,       /* Σ_s M2_s: within-sequence sums of squared deviations */
  DHMC_SUMMARY_SS_CHAIN = 5, /* Σ_c (μ_c − μ̄)² over the M chains */
  DHMC_SUMMARY_BELOW = 6,    /* kept draws below the reference (exact integer; NaN without a reference) */
  DHMC_SUMMARY_FIELDS = 7
};
/* reference: host [D, P] or NULL; record: host [DHMC_SUMMARY_FIELDS, D, P]; stats / logdens: host [N/thin, B] or NULL (the
 * kept transitions, as dhmc_mcmc_thinned).  DHMC_EARG before anything runs for N < 1, thin < 1, N % thin ≠ 0,
 * N / thin < 4 or record == NULL.  Device memory: one grow-only arena of 8·P·D + 3·D·(resident chain groups) + P doubles;
 * with G generated quantities 8·P·R + (3·D + 5·G)·(resident chain groups) + P doubles.
 * On DHMC_ENUMERIC the record is still written, without the chains that failed. */
int dhmc_mcmc_summary(dhmc_handle* h, int32_t N, int32_t thin, const double* reference, double* record,
                      dhmc_tree_stats* stats, double* logdens);
/* record ← record ⊕ other (both [DHMC_SUMMARY_FIELDS, D, P]; pairwise update of Chan, Golub and LeVeque).  DHMC_EARG (and
 * nothing written) when a cell with chains on both sides has two different n_keep.  Pure host code. */
int dhmc_summary_merge(double* record, const double* other, int64_t D, int64_t P);
/* The statistics above from a record; outputs [D, P] column-major, each may be NULL.  Pure host code. */
int dhmc_summary_finish(const double* record, int64_t D, int64_t P, double* mean, double* sd, double* mcse, double* ess,
                        double* rhat, int64_t* rank, int64_t* draws);

/* ---- streaming quantiles: per-(parameter, problem) histograms on a grid the caller fixes (DESIGN.md §4.4) ------------
 * Exact quantiles do not stream in fixed memory; exact bin counts do, and they bracket every quantile.  The grid of
 * (parameter d, problem p) is lo < hi, both finite, with hi − lo and nbins / (hi − lo) finite, 1 ≤ nbins ≤ 4096.  A kept
 * draw θ goes into one of nbins + 2 bins, evaluated on the device and by the numpy mirror with the same IEEE operations
 * (a separate subtract and multiply, no fused multiply-add):
 *   inv_w = nbins / (hi − lo)            (once, on the host)
 *   t     = (θ − lo) · inv_w
 *   bin   = 0              if t < 0         (below lo)
 *           nbins + 1      if !(t < nbins)  (at or above hi; NaN lands here too)
 *           1 + (int)t     otherwise
 * The histogram counts exactly the draws the rank counts: all n_keep kept draws of every local chain of problem p that
 * completed the call (an odd last draw included), so Σ over bins = draws[d, p]; a chain with DHMC_CHAIN_BAD_STEPSIZE or
 * DHMC_CHAIN_LEAPFROG_NONFINITE contributes nothing, even when it halted after keeping draws.  counts [nbins + 2, D, P]
 * column-major (bin fastest) are exact integers: the histograms of shards of one run on one grid add up to the histogram
 * of all their chains, so merging is adding the counts (no merge function is needed).
 *
 * Quantiles from the counts.  Edges e_k = lo + k·((hi − lo)/nbins) for k < nbins, e_nbins = hi.  For α ∈ [0, 1] and
 * n = Σ counts: h = α(n − 1), j = ⌊h⌋, γ = h − j (Julia's type 7).  Order statistic r (0-based) lies in the bin k whose
 * cumulative counts satisfy C_{k−1} ≤ r < C_k.
 *   q_lo  the lower edge of the bin of r = j (−∞ for bin 0)
 *   q_hi  the upper edge of the bin of r = j + 1 (r = j when γ = 0; +∞ for bin nbins + 1)
 *   q     type-7 interpolation of the in-bin placements e_{k−1} + ((r − C_{k−1}) + 0.5)/c_k · (e_k − e_{k−1}) of the order
 *         statistics it needs (dhmc_acceptance_quantiles_dev places its order statistics alike); NaN when one of them
 *         lies in a tail bin
 * n = 0 gives NaN for all three.  Guarantee: the exact type-7 quantile of the counted draws lies in [q_lo, q_hi], up to
 * the rounding of the edges (a few ulps of max(|lo|, |hi|)).
 *
 * dhmc_mcmc_summary_histogram is dhmc_mcmc_summary (same draws, final state, transition count, status words, return code
 * and record) that also writes counts.  lo, hi: host [D, P]; counts: host int64 [nbins + 2, D, P].  DHMC_EARG before
 * anything runs for an invalid grid or nbins, counts == NULL, or any argument dhmc_mcmc_summary rejects.  Device memory
 * on top of dhmc_mcmc_summary's arena: 8·P·D·(nbins + 4) + 4·D·(nbins + 2)·(resident chain groups) bytes (the problem
 * histograms and the grid, and a staging histogram per resident chain group); with G generated quantities R in place of D. */
int dhmc_mcmc_summary_histogram(dhmc_handle* h, int32_t N, int32_t thin, const double* reference, const double* lo,
                                const double* hi, int32_t nbins, double* record, int64_t* counts, dhmc_tree_stats* stats,
                                double* logdens);
/* q, q_lo, q_hi [nprobs, D, P] column-major (each may be NULL) of counts [nbins + 2, D, P] on the grid (lo, hi, nbins), as
 * defined above.  DHMC_EARG for a probability outside [0, 1], an invalid grid, a negative count or a NULL input.  Pure
 * host code. */
int dhmc_histogram_quantiles(const int64_t* counts, const double* lo, const double* hi, int32_t nbins, int64_t D, int64_t P,
                             const double* probs, int32_t nprobs, double* q, double* q_lo, double* q_hi);

/* ---- diagnostics on device-resident statistics (§8f) ------------------------ */
/* Diagnostics.summarize_tree_statistics / EBFMI (diagnostics.jl:29-32, 65-106) reduced on the
 * GPU over stats_dev [N,B] (DEVICE pointer, e.g. the buffer given to dhmc_mcmc_dev): pooled
 * depth counts [33], termination counts [max_depth, divergence, turning], Σ acceptance rate,
 * Σ steps (host outputs, may be NULL) and the per-chain EBFMI [B] (host, may be NULL).  EBFMI is NaN for N = 1 and
 * for a chain whose π is constant (0 / 0: π is centred on its first value, so a constant π has variance exactly 0; Julia's
 * EBFMI returns 0 there when its mean of the constant rounds away from it). */
int dhmc_tree_summary_dev(dhmc_handle* h, const dhmc_tree_stats* stats_dev, int32_t N,
                          int64_t* depth_counts, int64_t* termination_counts,
                          double* acceptance_sum, int64_t* steps_sum, double* ebfmi);

/* Cross-chain convergence diagnostics reduced on the GPU over device-resident draws [D, N, B] (the posterior buffer of
 * dhmc_mcmc_dev): per parameter the split-R̂ and the effective sample size of the pooled sequences (every chain split in two
 * halves; autocorrelations up to max_lag ≤ N/2 − 2, 0 = 64; Geyer's initial monotone sequence) — what the reference's
 * correctness tests compute with MCMCDiagnosticTools.ess_rhat (test/sample-correctness_utilities.jl:40-43).  A parameter
 * whose sequences are all constant at one value (var⁺ = 0) gets ESS = NaN and R̂ = NaN, as in MCMCDiagnosticTools.
 * rhat, ess: host [D], either may be NULL. */
int dhmc_ess_rhat_dev(dhmc_handle* h, const double* draws_dev, int32_t N, int32_t max_lag, double* rhat, double* ess);
/* The same per (problem, parameter) of a problem batch, over each problem's local chains (dhmc_ess_rhat_dev pools all
 * chains, which mixes the problems).  rhat, ess: host [D, n_problems] column-major; a problem without a local chain
 * gets NaN. */
int dhmc_ess_rhat_problems_dev(dhmc_handle* h, const double* draws_dev, int32_t N, int32_t max_lag, double* rhat,
                               double* ess);
/* Quantiles of the acceptance rates (Diagnostics.summarize_tree_statistics: a_quantiles at 0.05 … 0.95,
 * diagnostics.jl:35,100-106) of a device statistics buffer [N, B], from a 4096-bin histogram: the two order statistics
 * Julia's type-7 quantile interpolates between are each placed inside their bin, so every quantile is within 1/4096
 * (2.4e-4) of the type-7 quantile of the records whose rate is not NaN (those are left out; none left: NaN). */
int dhmc_acceptance_quantiles_dev(dhmc_handle* h, const dhmc_tree_stats* stats_dev, int32_t N, const double* probs,
                                  int32_t nprobs, double* out);

/* ---- multi-GPU: chains sharded over ranks, ONE all-gather of draws at the end (SURVEY.md §8e) ------------
 * One process (rank) per GPU; a handle owns the chains [chain_offset, chain_offset + n_chains) and the RNG keys use
 * the global chain id, so results do not depend on the number of ranks.  Nothing is exchanged while sampling.
 * The reference has no counterpart (multi-chain = the user runs mcmc_with_warmup K times,
 * docs/src/worked_example.md:97-103); these entry points replace the user's own gather of the per-chain results
 * (stack_posterior_matrices / pool_posterior_matrices, mcmc.jl:602-617, over all ranks). */
#define DHMC_COMM_ID_BYTES 128
/* rank 0: a fresh ncclUniqueId (128 bytes), to be carried to the other ranks by the host program */
int dhmc_comm_unique_id(void* id128);
/* every rank: ncclCommInitRank on the handle's device */
int dhmc_comm_init(dhmc_handle* h, int32_t nranks, int32_t rank, const void* id128);
int dhmc_comm_destroy(dhmc_handle* h);
/* ncclAllGather of `count` doubles per rank between DEVICE buffers (recv: [nranks][count]); with the draws buffer of
 * dhmc_mcmc_dev as `send`, recv is the [D, N, B·nranks] column-major array of all ranks' draws. */
int dhmc_allgather_dev(dhmc_handle* h, const double* send_dev, double* recv_dev, size_t count);
/* the current position of every chain of every rank, recv_dev: [D, B·nranks] (DEVICE) */
int dhmc_allgather_positions_dev(dhmc_handle* h, double* recv_dev);
/* device time of the last all-gather (CUDA events on the handle's stream) */
int dhmc_last_comm_ms(dhmc_handle* h, double* ms);

/* ---- measurement hooks ------------------------------------------------- */
/* Σ tree_statistics.steps over all chains and draws of the last sampling call. */
int dhmc_last_total_steps(dhmc_handle* h, int64_t* steps);
/* Device time (CUDA events on the handle's stream) of the last sampling /
 * leapfrog kernel, and the number of kernels this handle has launched. */
int dhmc_last_kernel_ms(dhmc_handle* h, double* ms);
int dhmc_kernel_launches(dhmc_handle* h, int64_t* n);

#ifdef __cplusplus
}
#endif
#endif /* DHMC_H */
