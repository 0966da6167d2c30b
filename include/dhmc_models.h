/* dhmc_models.h — scalar formulas of the shipped device log-density family.
 *
 * These play the role of the USER's `LogDensityProblems.logdensity_and_gradient`
 * (reference call site src/hamiltonian.jl:204).  They are inputs to the sampler,
 * not part of it, so the CUDA path and the CPU oracle share the per-element
 * formulas below; every cross-element sum is done by each side's own reduction
 * in the canonical order documented in DESIGN.md §"canonical reduction".
 *
 * Families (SURVEY.md §8d):
 *   STD_NORMAL  l(q) = -1/2 sum q_i^2                      grad = -q
 *   DIAG_NORMAL l(q) = -1/2 sum (q_i-mu_i)^2 * prec_i      grad = -(q_i-mu_i)*prec_i
 *               params = [mu(D), prec(D)]
 *   FUNNEL      Neal's funnel, theta = (v, x_1..x_{D-1}):
 *               l = -v^2/18 - 1/2 e^{-v} sum x_i^2 - (D-1)/2 v
 *   LOGISTIC    logistic regression with a N(0, I) prior (SURVEY.md §8d C4), X [N x p], y in {0,1}:
 *               eta = X beta;  l = sum_n [y_n eta_n - log1pexp(eta_n)] - 1/2 |beta|^2
 *               grad = X' (y - sigma(eta)) - beta      (ll term and sigma share one exponential: dhmc_logit_ll_resid)
 *               params = [N, X row-major (N*p), y (N)];  (X' r)_j is a sequential chain of fused multiply-adds
 *               over n, eta_n a blocked one over j (dhmc_logit_eta), the two scalar sums use the canonical reduction.
 *   USER        a log density supplied by the USER as a header of scalar formulas, compiled into its own copy of the
 *               library (`make -C dynamichmc.jl_b200/csrc user USER_HEADER=…`, `compile_user_model` in api.py): the
 *               device counterpart of handing DynamicHMC an arbitrary LogDensityProblems object (hamiltonian.jl:204).
 *               Contract at the end of this file; examples under include/models/.
 */
#ifndef DHMC_MODELS_H
#define DHMC_MODELS_H
#include "dhmc_math.h"

enum {
  DHMC_FAMILY_STD_NORMAL = 0,
  DHMC_FAMILY_DIAG_NORMAL = 1,
  DHMC_FAMILY_FUNNEL = 2,
  DHMC_FAMILY_LOGISTIC = 3,
  DHMC_FAMILY_USER = 4,      /* present only in a library built with -DDHMC_USER_MODEL_HEADER=… */
  DHMC_FAMILY_COUNT = 5
};

/* --- STD_NORMAL: term of the sum and gradient element */
DHMC_HD double dhmc_std_term(double q) { return q * q; }
DHMC_HD double dhmc_std_grad(double q) { return -q; }
DHMC_HD double dhmc_std_lq(double sum) { return -0.5 * sum; }

/* --- DIAG_NORMAL */
DHMC_HD double dhmc_diag_scaled(double q, double mu, double prec) {
  return prec * (q - mu);
}
DHMC_HD double dhmc_diag_term(double q, double mu, double t) {
  return (q - mu) * t;
}
DHMC_HD double dhmc_diag_grad(double t) { return -t; }
DHMC_HD double dhmc_diag_lq(double sum) { return -0.5 * sum; }

/* --- FUNNEL: S = sum_{i>=1} x_i^2 (element 0 contributes +0.0) */
DHMC_HD double dhmc_funnel_term(int i, double x) { return i == 0 ? 0.0 : x * x; }
DHMC_HD double dhmc_funnel_lq(double v, double ev, double S, int D) {
  double a = (v * v) / 18.0;
  double b = (0.5 * ev) * S;
  double c = (0.5 * (double)(D - 1)) * v;
  return ((-a) - b) - c;
}
DHMC_HD double dhmc_funnel_grad(int i, double x, double v, double ev, double S,
                                int D) {
  if (i == 0) return ((-v) / 9.0 + (0.5 * ev) * S) - 0.5 * (double)(D - 1);
  return -(ev * x);
}

/* --- LOGISTIC */
/* one multiply-accumulate of η_n = Σ_j X_nj β_j and of (Xᵀr)_j = Σ_n X_nj r_n: fused, as a BLAS would */
DHMC_HD double dhmc_logit_mac(double acc, double x, double b) { return dm_fma(x, b, acc); }
/* η_n is a blocked dot product (again as a BLAS would): sequential fused multiply-adds within chunks of
 * DHMC_LOGIT_CHUNK coefficients, the chunk sums added in increasing order:  η = ((s₀ + s₁) + s₂) + …
 * (dim <= 64: one plain sequential sum).  The chunks are independent accumulation chains, which is what lets
 * the tensor-core path spread one row tile over several warps. */
#define DHMC_LOGIT_CHUNK DHMC_DOT_CHUNK
DHMC_HD double dhmc_logit_eta(const double* xrow, const double* beta, int D) { return dm_blocked_dot(xrow, 1, beta, D); }
/* ll term y·η − log(1+e^η) and residual y − σ(η) from ONE exponential t = e^{−|η|}:
 *   log(1+e^η) = max(η,0) + log(1+t)   (table-driven softplus, absolute accuracy, no division)
 *   σ(η) = 1/(1+t) for η >= 0, t/(1+t) for η < 0   (no cancellation; one correctly rounded division) */
DHMC_HD void dhmc_logit_finish(double y, double eta, double sp, double t, double* ll, double* resid) {
  *ll = y * eta - ((eta > 0.0 ? eta : 0.0) + sp);
  /* η = ±∞ (the dot product overflowed): the formula gives ∞ − ∞ or 0·∞ = NaN, the limit is 0 for the outcome the sign
   * predicts (y = 1 at +∞, y = 0 at −∞) and −∞ otherwise.  Finite η keep the formula's value bit for bit. */
  if (eta == dm_inf()) *ll = y == 1.0 ? 0.0 : -dm_inf();
  if (eta == -dm_inf()) *ll = y == 0.0 ? 0.0 : -dm_inf();
  const double u = 1.0 + t;
  const double s = (eta >= 0.0 ? 1.0 : t) / u;
  *resid = y - s;
}
DHMC_HD void dhmc_logit_ll_resid(double y, double eta, double* ll, double* resid) {
  double t;
  const double sp = dm_softplus_neg_exp(dm_fabs(eta), &t);
  dhmc_logit_finish(y, eta, sp, t, ll, resid);
}
/* same values with the math tables behind a pointer (dm_softplus_neg_exp_tabs) */
DHMC_HD void dhmc_logit_ll_resid_tabs(double y, double eta, double* ll, double* resid, const double* tabs) {
  double t;
  const double sp = dm_softplus_neg_exp_tabs(dm_fabs(eta), &t, tabs);
  dhmc_logit_finish(y, eta, sp, t, ll, resid);
}
DHMC_HD double dhmc_logit_ll(double y, double eta) { double l, r; dhmc_logit_ll_resid(y, eta, &l, &r); return l; }
DHMC_HD double dhmc_logit_resid(double y, double eta) { double l, r; dhmc_logit_ll_resid(y, eta, &l, &r); return r; }
DHMC_HD double dhmc_logit_lq(double sum_ll, double sum_b2) { return sum_ll - 0.5 * sum_b2; }
DHMC_HD double dhmc_logit_grad(double xtr, double beta) { return xtr - beta; }

/* --- USER: the model header contract ------------------------------------------------------------------------------
 * A user model is ONE header that defines, with DHMC_HD (host + device, so that the CPU oracle checks the same
 * formulas), a log density of the form "element-wise gradient with the whole position visible, plus up to 4 global
 * sums" — the class that needs no data-parallel pass of its own (separable, neighbour-coupled / banded, hierarchical
 * models; regression likelihoods over large data sets are what the LOGISTIC family's cooperative rounds are for):
 *
 *   #define DHMC_USER_NAME     "my_model"   // reported by dhmc_user_family_name
 *   #define DHMC_USER_NSUMS    K            // 0 <= K <= 4 cross-element sums S[0..K-1]
 *   #define DHMC_USER_NSCALARS M            // 0 <= M <= 4 derived scalars  S[K..K+M-1]   (optional, default 0)
 *   #define DHMC_USER_MIN_DIM  d            // smallest valid dimension                   (optional, default 1)
 *   // contribution of element i to the K sums (t[0..K-1]); q is the WHOLE position vector (read-only)
 *   DHMC_HD void   dhmc_user_terms(int i, int D, const double* q, const double* params, double* t);
 *   // scalars every element needs (e.g. exp(-q[0])), computed once per thread after the sums; writes S[K..K+M-1]
 *   DHMC_HD void   dhmc_user_prepare(int D, const double* q, double* S, const double* params);   // only if M > 0
 *   DHMC_HD double dhmc_user_logdensity(int D, const double* q, const double* S, const double* params);
 *   DHMC_HD double dhmc_user_grad(int i, int D, const double* q, const double* S, const double* params);
 *
 * `params` is the block of doubles handed to dhmc_set_problem (any length) — in a problem batch, the chain's own
 * problem's block.  The formulas never receive the block's length: a model whose blocks differ in length from problem to
 * problem (dhmc_set_problems_ragged: e.g. a different number of observations per unit) stores the length, or whatever
 * it needs to find its data, in the block itself.  The sums are taken in the canonical
 * order (DESIGN.md §3); transcendental functions should come from dhmc_math.h (dm_exp, dm_log, dm_log1p, …) if the
 * device results are to equal the oracle's bit for bit — libm / libdevice calls work, but differ in the last ulp.
 * -Inf / non-finite values are handled by the sampler exactly as for the shipped families (hamiltonian.jl:202-217).
 *
 * Generated quantities (optional): functions of one position that the streaming summary reports beside the parameters
 * (Stan's generated quantities without randomness; e.g. the centred effects of a non-centred model):
 *
 *   #define DHMC_USER_GENERATED 1          // absent: the model has none
 *   DHMC_HD int    dhmc_user_ngq(int D);   // G(D): 1 <= G <= 8192, a function of the dimension only
 *   // quantity k (0 <= k < G) of the WHOLE position q; params as for dhmc_user_terms (the point's own problem block)
 *   DHMC_HD double dhmc_user_generated(int k, int D, const double* q, const double* params);
 *
 * G may depend on D, not on the parameters, so that every problem of a batch has the same G rows.  Generated quantities
 * never affect sampling: the draws, statistics, final state and transition counts are those of the same model without
 * them.  A non-finite value is folded as it is (NaN lands in the top histogram bin and is never below a reference) and
 * sets no chain status bit.  dhmc_generated evaluates them at given points; dhmc_mcmc_summary appends them to the
 * parameters as rows D … D + G − 1 (include/dhmc.h).  Where DHMC_USER_NGQ_CONST is defined as G, the bounds are checked
 * at compile time; otherwise dhmc_create checks G(D).
 *
 * Random generated quantities (optional, with DHMC_USER_GENERATED): Stan's `y_rep = normal_rng(...)`, e.g. posterior
 * predictive replicates and the indicators of a posterior predictive check.  The quantity function takes a fifth argument:
 *
 *   #define DHMC_USER_GENERATED_RNG 1
 *   DHMC_HD double dhmc_user_generated(int k, int D, const double* q, const double* params, const dhmc_gq_rng* rng);
 *
 * and draws its numbers through dhmc_math.h's two helpers, whose definitions are exact (the host reproduces them):
 *   dhmc_gq_uniform(rng, i) = dm_uniform_elem(key, DHMC_STREAM_GQ_U, t, i)   in (0, 1)
 *   dhmc_gq_normal(rng, i)  = dm_normal_elem(key, DHMC_STREAM_GQ_N, t, i)    N(0, 1)
 * The numbers depend only on the key and the index i.  So every quantity of one draw sees the same normal(i), and a test
 * statistic re-derives the replicate rows it summarizes by asking for the same indices (quantity k stays a pure function,
 * evaluated independently of the others).  Different indices are independent; uniforms and normals never share bits; the
 * sampler never reads either stream, so sampling is that of the same model without the part.  Other distributions are
 * built by the header from these two: a Bernoulli(p) is uniform(i) < p; a Poisson by inversion over the indices i·64 + r,
 * r = 0, 1, …; no further helper exists.
 *
 * The key of a kept draw: (the handle's seed, global chain id chain_offset + c) and t, the RNG counter of the transition
 * that produced the draw.  A sampling call that starts at transition count t0 with thinning `thin` keeps, as draw j
 * (0-based), the draw of t = t0 + (j + 1)·thin − 1 (uint32 arithmetic).  So, like the draws, the random quantities do
 * not depend on sharding, chunking or checkpoint / restore.  dhmc_generated_keyed evaluates them at given points and
 * keys; dhmc_generated refuses a model with random quantities. */
#ifdef DHMC_USER_MODEL_HEADER
#include DHMC_USER_MODEL_HEADER
#ifndef DHMC_USER_NSUMS
#error "user model header: define DHMC_USER_NSUMS (0..4)"
#endif
#ifndef DHMC_USER_NSCALARS
#define DHMC_USER_NSCALARS 0
#endif
#ifndef DHMC_USER_MIN_DIM
#define DHMC_USER_MIN_DIM 1
#endif
#ifndef DHMC_USER_NAME
#define DHMC_USER_NAME "user"
#endif
#if DHMC_USER_NSUMS < 0 || DHMC_USER_NSUMS > 4 || DHMC_USER_NSCALARS < 0 || DHMC_USER_NSCALARS > 4
#error "user model header: 0 <= DHMC_USER_NSUMS <= 4 and 0 <= DHMC_USER_NSCALARS <= 4"
#endif
#if defined(DHMC_USER_NGQ_CONST) && (DHMC_USER_NGQ_CONST < 1 || DHMC_USER_NGQ_CONST > 8192)   /* DHMC_MAX_GENERATED */
#error "user model header: 1 <= DHMC_USER_NGQ_CONST <= 8192"
#endif
#if defined(DHMC_USER_NGQ_CONST) && !defined(DHMC_USER_GENERATED)
#error "user model header: DHMC_USER_NGQ_CONST without DHMC_USER_GENERATED"
#endif
#if defined(DHMC_USER_GENERATED_RNG) && !defined(DHMC_USER_GENERATED)
#error "user model header: DHMC_USER_GENERATED_RNG without DHMC_USER_GENERATED"
#endif
#define DHMC_HAVE_USER_FAMILY 1
#endif

#endif
