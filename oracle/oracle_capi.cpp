// oracle_capi.cpp — flat C entry points over oracle.hpp for ctypes
// (oracle/pyoracle.py).  TEST INFRASTRUCTURE ONLY — see the header of oracle.hpp.
#include <malloc.h>
#include <pthread.h>
#include <sched.h>

#include <atomic>
#include <chrono>
#include <cstdlib>
#include <cstring>
#include <thread>

#include "oracle.hpp"

using namespace orc;

namespace {
thread_local std::string g_err;
thread_local int g_dense = 0;   // when set, `minv` pointers are D x D row-major (Symmetric metric)
KineticEnergy make_k(const double* minv, int D) {
  if (g_dense) return KineticEnergy::Dense(vec(minv, minv + (size_t)D * D), D);
  return KineticEnergy(vec(minv, minv + (size_t)D));
}
Model make_model(int family, int D, const double* params, int nparams, int T, int always_div) {
  Model m; m.family = family; m.D = D; m.T = T; m.always_divergent = always_div != 0;
  if (params && nparams > 0) m.params.assign(params, params + nparams);
  return m;
}
thread_local int g_logistic_n = 0;   // N of the logistic-regression family (set by orc_set_logistic_n)
thread_local int g_user_nparams = 0;  // length of the USER family's parameter block (set by orc_set_user_nparams)
int nparams_of(int family, int D) {
  if (family == DHMC_FAMILY_LOGISTIC) return 1 + g_logistic_n * D + g_logistic_n;
  if (family == DHMC_FAMILY_USER) return g_user_nparams;
  return family == DHMC_FAMILY_DIAG_NORMAL ? 2 * D : 0;
}
template <class F>
int guarded(F f) {
  try { f(); return 0; }
  catch (const DynamicHMCError& e) { g_err = e.what(); return 2; }
  catch (const ArgumentError& e) { g_err = e.what(); return 1; }
  catch (const std::exception& e) { g_err = e.what(); return 3; }
}
}  // namespace

extern "C" {

const char* orc_last_error() { return g_err.c_str(); }
void orc_set_dense(int flag) { g_dense = flag; }
void orc_set_logistic_n(int n) { g_logistic_n = n; }
void orc_set_user_nparams(int n) { g_user_nparams = n; }
// name of the user model compiled into this oracle library ("" in the stock liboracle.so)
const char* orc_user_family_name() {
#ifdef DHMC_HAVE_USER_FAMILY
  return DHMC_USER_NAME;
#else
  return "";
#endif
}
// W = cholesky(inv(M⁻¹)).L; returns 0 ok, 2 not positive definite
int orc_dense_factor(int D, const double* minv, double* W) {
  vec w;
  if (!dense_factor(vec(minv, minv + (size_t)D * D), D, w)) return 2;
  std::memcpy(W, w.data(), sizeof(double) * (size_t)D * D);
  return 0;
}
// W of M⁻¹ known to the caller (e.g. assembled from the dense_factor of the blocks of a block-diagonal M⁻¹): later calls
// with this M⁻¹ use it instead of factorising
void orc_seed_dense_factor(int D, const double* minv, const double* W) {
  DenseFactorCache& c = dense_factor_cache();
  c.minv.assign(minv, minv + (size_t)D * D);
  c.w.assign(W, W + (size_t)D * D);
}
void orc_rand_p(uint64_t seed, uint64_t chain, uint32_t stream, uint32_t t, int D, const double* minv, double* out) {
  vec p = rand_p(dm_make_key(seed, chain), stream, t, make_k(minv, D));
  std::memcpy(out, p.data(), sizeof(double) * D);
}

// ------------------------------------------------------------------- math
void orc_math(int fn, int n, const double* x, const double* y, double* out) {
  for (int i = 0; i < n; ++i) {
    switch (fn) {
      case 0: out[i] = dm_exp(x[i]); break;
      case 1: out[i] = dm_log(x[i]); break;
      case 2: out[i] = dm_log1p(x[i]); break;
      case 3: out[i] = dm_logaddexp(x[i], y[i]); break;
      case 4: out[i] = dm_pow(x[i], y[i]); break;
      case 5: out[i] = dm_log1pexp(x[i]); break;
      case 6: { double s, c; dm_sincos2pi(x[i], &s, &c); out[i] = s; break; }
      case 7: { double s, c; dm_sincos2pi(x[i], &s, &c); out[i] = c; break; }
      case 8: out[i] = dm_softplus_neg(x[i]); break;
      default: out[i] = dm_nan();
    }
  }
}
void orc_philox(const uint32_t* ctr, const uint32_t* key, uint32_t* out) {
  dm_u32x4 r = dm_philox4x32_10(ctr[0], ctr[1], ctr[2], ctr[3], key[0], key[1]);
  for (int i = 0; i < 4; ++i) out[i] = r.v[i];
}
void orc_normals(uint64_t seed, uint64_t chain, uint32_t stream, uint32_t t, int D, double* out) {
  dm_rng_key k = dm_make_key(seed, chain);
  for (int i = 0; i < D; ++i) out[i] = dm_normal_elem(k, stream, t, (uint32_t)i);
}
void orc_random_position(uint64_t seed, uint64_t chain, int D, double* out) {
  vec q = random_position(dm_make_key(seed, chain), D);
  std::memcpy(out, q.data(), sizeof(double) * D);
}
double orc_randexp(uint64_t seed, uint64_t chain, uint32_t t, uint32_t j) {
  return dm_randexp(dm_make_key(seed, chain), t, j);
}
uint32_t orc_directions(uint64_t seed, uint64_t chain, uint32_t t) {
  return dm_rand_directions(dm_make_key(seed, chain), t);
}
double orc_canon_dot(int T, int D, const double* a, const double* b) {
  return canon_sum(T, D, [&](int i) { return a[i] * b[i]; });
}

// ------------------------------------------------------------- dummy trees
struct OrcDummyOut {
  int valid; long inv_left, inv_right; long zeta_lo, zeta_hi; int n_lp; double lp[4096];
  double omega; int tau_flag; long tau_lo, tau_hi; long z_last, i_last;
  double v_a; long v_steps; int n_visited; long visited[4096]; int adjacency_ok; int depth;
};
static DummyTrajectory make_dummy(const long* turning, int nt, const long* divergent, int nd) {
  DummyTrajectory tr;
  for (int i = 0; i < nt; ++i) tr.turning.insert(turning[i]);
  for (int i = 0; i < nd; ++i) tr.divergent.insert(divergent[i]);
  return tr;
}
static void dump_visited(const DummyTrajectory& tr, OrcDummyOut* o) {
  o->n_visited = (int)tr.visited.size();
  for (int i = 0; i < o->n_visited && i < 4096; ++i) o->visited[i] = tr.visited[i];
  o->adjacency_ok = tr.adjacency_ok ? 1 : 0;
}
int orc_dummy_adjacent_tree(long z, long i, int depth, int fwd, const long* turning, int nt,
                            const long* divergent, int nd, OrcDummyOut* o) {
  return guarded([&] {
    DummyTrajectory tr = make_dummy(turning, nt, divergent, nd);
    NoRng rng;
    auto [t, v] = adjacent_tree(rng, tr, z, i, depth, fwd != 0);
    std::memset(o, 0, sizeof(*o));
    o->valid = t.valid; o->inv_left = t.invalid.left; o->inv_right = t.invalid.right;
    if (t.valid) {
      o->zeta_lo = t.zeta.lo; o->zeta_hi = t.zeta.hi; o->n_lp = (int)t.zeta.lp.size();
      for (int k = 0; k < o->n_lp; ++k) o->lp[k] = t.zeta.lp[k];
      o->omega = t.omega; o->tau_flag = t.tau.flag; o->tau_lo = t.tau.lo; o->tau_hi = t.tau.hi;
      o->z_last = t.z; o->i_last = t.i;
    }
    o->v_a = v.a; o->v_steps = v.steps;
    dump_visited(tr, o);
  });
}
int orc_dummy_sample_trajectory(long z, int max_depth, uint32_t flags, const long* turning, int nt,
                                const long* divergent, int nd, OrcDummyOut* o) {
  return guarded([&] {
    DummyTrajectory tr = make_dummy(turning, nt, divergent, nd);
    NoRng rng;
    auto r = sample_trajectory(rng, tr, z, max_depth, Directions{flags});
    std::memset(o, 0, sizeof(*o));
    o->valid = 1; o->inv_left = r.termination.left; o->inv_right = r.termination.right;
    o->zeta_lo = r.zeta.lo; o->zeta_hi = r.zeta.hi; o->n_lp = (int)r.zeta.lp.size();
    for (int k = 0; k < o->n_lp; ++k) o->lp[k] = r.zeta.lp[k];
    o->v_a = r.v.a; o->v_steps = r.v.steps; o->depth = r.depth;
    dump_visited(tr, o);
  });
}
void orc_next_directions(uint32_t flags, int n, int* out) {
  Directions d{flags};
  for (int i = 0; i < n; ++i) { auto [f, nd] = next_direction(d); out[i] = f; d = nd; }
}

// ------------------------------------------------------------- hamiltonian
double orc_logdensity_and_gradient(int family, int D, const double* params, int T, const double* q,
                                   double* g_out) {
  Model m = make_model(family, D, params, nparams_of(family, D), T, 0);
  vec g; double lq = m.logdensity_and_gradient(vec(q, q + D), g);
  std::memcpy(g_out, g.data(), sizeof(double) * D);
  return lq;
}
double orc_kinetic_energy(int D, int T, const double* minv, const double* p) {
  Model m = make_model(0, D, nullptr, 0, T, 0);
  Hamiltonian H(make_k(minv, D), m);
  return kinetic_energy(H, vec(p, p + D));
}
// logdensity(H, z) with explicit lq (tests the −Inf fallbacks, test_hamiltonian.jl:196-200)
double orc_phase_logdensity(int D, int T, const double* minv, double lq, const double* p) {
  Model m = make_model(0, D, nullptr, 0, T, 0);
  Hamiltonian H(make_k(minv, D), m);
  PhasePoint z{{vec(D, 0.0), lq, vec(D, 0.0)}, vec(p, p + D)};
  return logdensity(H, z);
}
int orc_evaluate_l(int family, int D, const double* params, int T, const double* q, int strict,
                   double* lq_out, double* g_out) {
  return guarded([&] {
    Model m = make_model(family, D, params, nparams_of(family, D), T, 0);
    auto Q = evaluate_l(m, vec(q, q + D), strict != 0);
    *lq_out = Q.lq; std::memcpy(g_out, Q.g.data(), sizeof(double) * D);
  });
}
// n_steps leapfrog steps of size eps (sign included) from (q, p); g/lq are recomputed at entry.
int orc_leapfrog(int family, int D, const double* params, int T, const double* minv, double* q,
                 double* p, double* g, double* lq, double eps, int n_steps) {
  return guarded([&] {
    Model m = make_model(family, D, params, nparams_of(family, D), T, 0);
    Hamiltonian H(make_k(minv, D), m);
    PhasePoint z{evaluate_l(m, vec(q, q + D)), vec(p, p + D)};
    for (int s = 0; s < n_steps; ++s) z = leapfrog(H, z, eps);
    std::memcpy(q, z.Q.q.data(), sizeof(double) * D);
    std::memcpy(p, z.p.data(), sizeof(double) * D);
    std::memcpy(g, z.Q.g.data(), sizeof(double) * D);
    *lq = z.Q.lq;
  });
}

// -------------------------------------------------------------------- NUTS
// combine_turn_statistics on raw (p₋,p♯₋,p₊,p♯₊,ρ) vectors; returns 1 if turning.
int orc_combine_turn_statistics(int D, int T, const double* x5, const double* y5, double* rho_out) {
  Model m = make_model(0, D, nullptr, 0, T, 0);
  Hamiltonian H(KineticEnergy(D), m);
  TrajectoryNUTS tr{H, 0.0, 1.0, -1000.0};
  auto mk = [&](const double* v) {
    TurnStatistic t;
    t.pm.assign(v, v + D); t.psm.assign(v + D, v + 2 * D); t.pp.assign(v + 2 * D, v + 3 * D);
    t.psp.assign(v + 3 * D, v + 4 * D); t.rho.assign(v + 4 * D, v + 5 * D);
    return t;
  };
  auto r = tr.combine_turn_statistics(mk(x5), mk(y5));
  if (!r.turning) std::memcpy(rho_out, r.rho.data(), sizeof(double) * D);
  return r.turning ? 1 : 0;
}
// acceptance_rate(reduce(combine, leaf statistics)) — test_NUTS.jl:44-55
double orc_acceptance_rate(int n, const double* deltas, const int* is_initial) {
  AcceptanceStatistic a = leaf_acceptance_statistic(deltas[0], is_initial[0] != 0);
  for (int i = 1; i < n; ++i)
    a = combine_acceptance_statistics(a, leaf_acceptance_statistic(deltas[i], is_initial[i] != 0));
  return acceptance_rate(a);
}
// rand_bool_logprob; *consumed reports whether a randexp was drawn
int orc_rand_bool_logprob(uint64_t seed, uint64_t chain, uint32_t t, uint32_t j, double logprob,
                          int* consumed) {
  Rng rng{dm_make_key(seed, chain), t, j};
  bool b = rand_bool_logprob(rng, logprob);
  *consumed = (int)(rng.n_exp - j);
  return b ? 1 : 0;
}

int orc_sample_tree(int family, int D, const double* params, int T, const double* minv,
                    int max_depth, double min_delta, int always_divergent, uint64_t seed,
                    uint64_t chain, uint32_t t, const double* q, double eps,
                    const double* p_override, const uint32_t* dir_override, double* q_out,
                    double* lq_out, double* g_out, TreeStatistics* stats, int* accept_trace,
                    int accept_cap, int* n_accept) {
  return guarded([&] {
    Model m = make_model(family, D, params, nparams_of(family, D), T, always_divergent);
    Hamiltonian H(make_k(minv, D), m);
    NUTS alg{max_depth, min_delta}; alg.check();
    auto Q = evaluate_l(m, vec(q, q + D), true);
    Rng rng{dm_make_key(seed, chain), t, 0};
    vec pv; if (p_override) pv.assign(p_override, p_override + D);
    std::vector<int> trace;
    auto [Q1, ts] = sample_tree(rng, alg, H, Q, eps, p_override ? &pv : nullptr, dir_override, &trace);
    std::memcpy(q_out, Q1.q.data(), sizeof(double) * D);
    std::memcpy(g_out, Q1.g.data(), sizeof(double) * D);
    *lq_out = Q1.lq; *stats = ts;
    if (n_accept) *n_accept = (int)trace.size();
    for (int i = 0; accept_trace && i < (int)trace.size() && i < accept_cap; ++i) accept_trace[i] = trace[i];
  });
}

// ---------------------------------------------------------------- stepsize
// find_initial_stepsize on A(eps) = c*eps + d  (test_stepsize.jl:9-25)
int orc_find_initial_stepsize_affine(double c, double d, double initial_eps, double log_threshold,
                                     int maxiter, double* eps_out) {
  return guarded([&] {
    InitialStepsizeSearch par{initial_eps, log_threshold, maxiter}; par.check();
    *eps_out = find_initial_stepsize(par, [&](double e) { return c * e + d; });
  });
}
int orc_search_params_check(double initial_eps, double log_threshold, int maxiter) {
  return guarded([&] { InitialStepsizeSearch par{initial_eps, log_threshold, maxiter}; par.check(); });
}
int orc_find_initial_stepsize(int family, int D, const double* params, int T, const double* minv,
                              const double* q, const double* p, double initial_eps,
                              double log_threshold, int maxiter, double* eps_out) {
  return guarded([&] {
    Model m = make_model(family, D, params, nparams_of(family, D), T, 0);
    Hamiltonian H(make_k(minv, D), m);
    PhasePoint z{evaluate_l(m, vec(q, q + D), true), vec(p, p + D)};
    InitialStepsizeSearch par{initial_eps, log_threshold, maxiter}; par.check();
    *eps_out = find_initial_stepsize(par, local_log_acceptance_ratio(H, z));
  });
}
double orc_local_log_acceptance_ratio(int family, int D, const double* params, int T,
                                      const double* minv, const double* q, const double* p, double eps) {
  Model m = make_model(family, D, params, nparams_of(family, D), T, 0);
  Hamiltonian H(make_k(minv, D), m);
  PhasePoint z{evaluate_l(m, vec(q, q + D), true), vec(p, p + D)};
  return local_log_acceptance_ratio(H, z)(eps);
}
int orc_da_init(double eps, double* state5) {
  return guarded([&] {
    auto A = initial_adaptation_state(DualAveraging{}, eps);
    state5[0] = A.mu; state5[1] = (double)A.m; state5[2] = A.Hbar; state5[3] = A.logeps; state5[4] = A.logepsbar;
  });
}
int orc_da_adapt(double delta, double gamma, double kappa, int t0, double* state5, double a) {
  return guarded([&] {
    DualAveraging P{delta, gamma, kappa, t0}; P.check();
    DualAveragingState A{state5[0], (int64_t)state5[1], state5[2], state5[3], state5[4]};
    A = adapt_stepsize(P, A, a);
    state5[0] = A.mu; state5[1] = (double)A.m; state5[2] = A.Hbar; state5[3] = A.logeps; state5[4] = A.logepsbar;
  });
}

// -------------------------------------------------------------------- mcmc
// Stages are given as parallel arrays; kind: 0 nothing, 1 search, 2 tuning.
static std::vector<Stage> make_stages(int n, const int* kind, const int* N, const int* metric,
                                      const int* da_on, const double* da4, const double* search3) {
  std::vector<Stage> st(n);
  for (int i = 0; i < n; ++i) {
    st[i].kind = kind[i]; st[i].N = N[i]; st[i].metric = metric[i]; st[i].dual_averaging = da_on[i] != 0;
    st[i].lambda = N[i] > 0 ? 5.0 / N[i] : 0.0;
    if (da4) st[i].da = DualAveraging{da4[0], da4[1], da4[2], (int)da4[3]};
    if (search3) st[i].search = InitialStepsizeSearch{search3[0], search3[1], (int)search3[2]};
  }
  return st;
}

// One chain of mcmc_with_warmup.  Warmup draws of all tuning stages are
// concatenated into *_w outputs when those pointers are non-null.
int orc_mcmc_with_warmup(int family, int D, const double* params, int T, int max_depth,
                         double min_delta, uint64_t seed, uint64_t chain, int N, int n_stages,
                         const int* kind, const int* stN, const int* metric, const int* da_on,
                         const double* da4, const double* search3, const double* q0,
                         const double* minv0, const double* eps0, int welford, double* posterior,
                         TreeStatistics* stats, double* logdens, double* minv_out, double* eps_out,
                         double* posterior_w, TreeStatistics* stats_w, double* eps_w,
                         double* state_q_out) {
  return guarded([&] {
    Sampler S; S.l = make_model(family, D, params, nparams_of(family, D), T, 0);
    S.alg = NUTS{max_depth, min_delta}; S.key = dm_make_key(seed, chain); S.welford = welford != 0;
    auto stages = make_stages(n_stages, kind, stN, metric, da_on, da4, search3);
    vec qv, mv; if (q0) qv.assign(q0, q0 + D);
    if (minv0) mv.assign(minv0, minv0 + (g_dense ? (size_t)D * D : (size_t)D));
    auto r = mcmc_with_warmup(S, N, stages, q0 ? &qv : nullptr, minv0 ? &mv : nullptr, eps0, g_dense != 0);
    for (int i = 0; i < N; ++i) {
      if (posterior) std::memcpy(posterior + (size_t)i * D, r.inference.posterior[i].data(), sizeof(double) * D);
      if (stats) stats[i] = r.inference.stats[i];
      if (logdens) logdens[i] = r.inference.logdensities[i];
    }
    if (minv_out) std::memcpy(minv_out, r.final_state.k.minv.data(), sizeof(double) * r.final_state.k.minv.size());
    if (eps_out) *eps_out = r.final_state.eps;
    if (state_q_out) std::memcpy(state_q_out, r.final_state.Q.q.data(), sizeof(double) * D);
    size_t off = 0;
    for (auto& w : r.warmup) {
      for (size_t i = 0; i < w.posterior.size(); ++i, ++off) {
        if (posterior_w) std::memcpy(posterior_w + off * D, w.posterior[i].data(), sizeof(double) * D);
        if (stats_w) stats_w[off] = w.stats[i];
        if (eps_w) eps_w[off] = w.eps_used[i];
      }
    }
  });
}

// mcmc_with_warmup for the chain group [chain0, chain0 + 8) with pooled Symmetric stages (metric code 3).  Outputs for all
// eight chains: posterior [8][N][D], stats [8][N], logdens [8][N], eps_out [8]; minv_out [D*D] is the (shared) final metric.
int orc_mcmc_with_warmup_pooled(int family, int D, const double* params, int T, int max_depth, double min_delta,
                                uint64_t seed, uint64_t chain0, int N, int n_stages, const int* kind, const int* stN,
                                const int* metric, const int* da_on, const double* da4, const double* search3,
                                double* posterior, TreeStatistics* stats, double* logdens, double* minv_out, double* eps_out) {
  return guarded([&] {
    auto stages = make_stages(n_stages, kind, stN, metric, da_on, da4, search3);
    std::vector<Sampler> S(kPoolGroup);
    for (int c = 0; c < kPoolGroup; ++c) {
      S[c].l = make_model(family, D, params, nparams_of(family, D), T, 0);
      S[c].alg = NUTS{max_depth, min_delta}; S[c].key = dm_make_key(seed, chain0 + (uint64_t)c); S[c].welford = true;
    }
    auto r = mcmc_with_warmup_pooled(S, N, stages);
    for (int c = 0; c < kPoolGroup; ++c) {
      for (int i = 0; i < N; ++i) {
        if (posterior) std::memcpy(posterior + ((size_t)c * N + i) * D, r[c].inference.posterior[i].data(), sizeof(double) * D);
        if (stats) stats[(size_t)c * N + i] = r[c].inference.stats[i];
        if (logdens) logdens[(size_t)c * N + i] = r[c].inference.logdensities[i];
      }
      if (eps_out) eps_out[c] = r[c].final_state.eps;
    }
    if (minv_out) std::memcpy(minv_out, r[0].final_state.k.minv.data(), sizeof(double) * r[0].final_state.k.minv.size());
  });
}

// Multi-threaded CPU baseline: n_chains chains, one per task, n_threads
// std::threads (mirrors OhMyThreads.tcollect over mcmc_with_warmup calls,
// test/sample-correctness_utilities.jl:17).  Fixed eps / fixed minv sampling
// (no warmup) when n_stages == 0.  Returns total leapfrog steps and seconds.
int orc_bench_mcmc(int family, int D, const double* params, int T, int max_depth, double min_delta,
                   uint64_t seed, int n_chains, int n_threads, int N, int n_stages, const int* kind,
                   const int* stN, const int* metric, const int* da_on, const double* minv0,
                   const double* eps0, int64_t* total_steps, double* seconds, double* mean_out) {
  // glibc's per-thread arenas grow/shrink their heaps with mprotect/madvise on this
  // allocate-and-free-8KB-vectors pattern, which serialises threads on the mm lock;
  // keep freed memory in the arenas instead (the reference's GC'd heap behaves likewise).
  mallopt(M_TRIM_THRESHOLD, 1 << 30);
  mallopt(M_TOP_PAD, 64 << 20);
  mallopt(M_MMAP_THRESHOLD, 1 << 30);
  const int nparams = nparams_of(family, D);   // on the calling thread: the logistic N is thread-local state
  std::atomic<int> next{0};
  std::atomic<int64_t> steps{0};
  std::atomic<int> failed{0};
  std::vector<double> mean_acc((size_t)D, 0.0);
  auto stages = make_stages(n_stages, kind, stN, metric, da_on, nullptr, nullptr);
  auto t0 = std::chrono::steady_clock::now();
  // pin worker i to the i-th CPU of the process's affinity mask (stable placement, no migration)
  cpu_set_t allowed;
  CPU_ZERO(&allowed);
  std::vector<int> cpus;
  if (sched_getaffinity(0, sizeof allowed, &allowed) == 0)
    for (int i = 0; i < CPU_SETSIZE; ++i) if (CPU_ISSET(i, &allowed)) cpus.push_back(i);
  auto work = [&](int widx) {
    if (!cpus.empty() && std::getenv("DHMC_ORACLE_NO_PIN") == nullptr) {
      cpu_set_t one;
      CPU_ZERO(&one);
      CPU_SET(cpus[(size_t)widx % cpus.size()], &one);
      pthread_setaffinity_np(pthread_self(), sizeof one, &one);
    }
    for (;;) {
      int c = next.fetch_add(1);
      if (c >= n_chains) break;
      try {
        Sampler S; S.l = make_model(family, D, params, nparams, T, 0);
        S.alg = NUTS{max_depth, min_delta}; S.key = dm_make_key(seed, (uint64_t)c);
        vec mv; if (minv0) mv.assign(minv0, minv0 + D);
        auto r = mcmc_with_warmup(S, N, stages, nullptr, minv0 ? &mv : nullptr, eps0);
        int64_t s = 0;
        for (auto& ts : r.inference.stats) s += ts.steps;
        for (auto& w : r.warmup) for (auto& ts : w.stats) s += ts.steps;
        steps += s;
      } catch (const std::exception& e) { failed += 1; }
    }
  };
  std::vector<std::thread> th;
  for (int i = 0; i < n_threads; ++i) th.emplace_back(work, i);
  for (auto& t : th) t.join();
  auto t1 = std::chrono::steady_clock::now();
  *total_steps = steps.load();
  *seconds = std::chrono::duration<double>(t1 - t0).count();
  (void)mean_out;
  return failed.load() ? 2 : 0;
}

}  // extern "C"
