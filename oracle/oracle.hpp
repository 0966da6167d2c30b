// oracle.hpp — CPU restatement of the DynamicHMC.jl sampler path.
//
// TEST INFRASTRUCTURE ONLY.  Nothing under oracle/ is linked, imported or
// executed by the product path (dynamichmc.jl_b200/); only tests/,
// __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg
// use it, and only as the checker / the CPU baseline.
//
// Every function cites the reference file:line it restates (paths relative to
// the upstream repo, tpapp/DynamicHMC.jl v3.6.0).  The tree code is kept
// RECURSIVE and generic over a trajectory concept exactly like
// src/trees.jl, so the reference's DummyTrajectory known-answer tests
// (test/test_trees.jl) port 1:1 (oracle_capi.cpp, tests/test_oracle_trees.py).
// The CUDA path flattens the same recursion into an explicit stack; agreement
// of the two independent formulations is what the parity tests check.
//
// Parity status: pinned against the reference's own known-answer tests
// (test_trees.jl, test_NUTS.jl, test_stepsize.jl, test_hamiltonian.jl), which
// are property/KAT tests; the reference holds no stored numeric golden files,
// and Julia is not available in this image, so RNG-stream parity with Julia and
// LogExpFunctions.logaddexp last-bit parity are UNPINNED (SURVEY.md §8c).
//
// Arithmetic: every cross-element sum uses the canonical reduction (T virtual
// lanes, lane-strided sequential partials, then a pairwise tree), which is the
// order the GPU uses; all products/sums are separately rounded (compile with
// -ffp-contract=off), mirroring the reference's non-fused vector ops.
#pragma once
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <functional>
#include <set>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "../include/dhmc_math.h"
#include "../include/dhmc_models.h"

namespace orc {

using vec = std::vector<double>;

struct DynamicHMCError : std::runtime_error {  // src/utilities.jl:17-27
  using std::runtime_error::runtime_error;
};
struct ArgumentError : std::invalid_argument {  // @argcheck failures
  using std::invalid_argument::invalid_argument;
};

// ---------------------------------------------------------------- reduction
// Canonical sum (DESIGN.md "canonical reduction"): T virtual lanes; lane v
// accumulates term(i) for i = v, v+T, ... in increasing i starting from +0.0.
// Lanes are combined per group of 32 (a warp) by a pairwise tree with offsets
// 16, 8, 4, 2, 1, then the per-warp sums by a pairwise tree with offsets
// 32, 64, ...  This is exactly the order of the GPU's shuffle reduce-scatter
// followed by its cross-warp exchange.  T == 0 selects plain sequential
// summation (used only for tolerance checks).
template <class F>
double canon_sum(int T, int D, F term) {
  if (T <= 0) {
    double acc = 0.0;
    for (int i = 0; i < D; ++i) acc = acc + term(i);
    return acc;
  }
  double part[1024];
  for (int v = 0; v < T; ++v) {
    double acc = 0.0;
    for (int i = v; i < D; i += T) acc = acc + term(i);
    part[v] = acc;
  }
  for (int base = 0; base < T; base += 32)
    for (int off = 16; off >= 1; off >>= 1)
      for (int v = base; v < base + off; ++v) part[v] = part[v] + part[v + off];
  for (int off = 32; off < T; off <<= 1)
    for (int v = 0; v < T; v += 2 * off) part[v] = part[v] + part[v + off];
  return part[0];
}

// -------------------------------------------------------------------- model
// The user's log density (LogDensityProblems API: dimension,
// logdensity_and_gradient; reference call site src/hamiltonian.jl:204).
struct Model {
  int family = DHMC_FAMILY_STD_NORMAL;
  int D = 0;
  vec params;
  int T = 32;  // canonical reduction width
  // test hook: AlwaysDivergentTest of test/test_NUTS.jl:58-73
  bool always_divergent = false;

  double logdensity_and_gradient(const vec& q, vec& g) const {
    g.resize(D);
    if (always_divergent) {
      bool allzero = true;
      for (int i = 0; i < D; ++i) { g[i] = 1.0; allzero = allzero && q[i] == 0.0; }
      return allzero ? 0.0 : -dm_inf();
    }
    switch (family) {
      case DHMC_FAMILY_STD_NORMAL: {
        double s = canon_sum(T, D, [&](int i) { return dhmc_std_term(q[i]); });
        for (int i = 0; i < D; ++i) g[i] = dhmc_std_grad(q[i]);
        return dhmc_std_lq(s);
      }
      case DHMC_FAMILY_DIAG_NORMAL: {
        const double* mu = params.data();
        const double* pr = params.data() + D;
        vec t(D);
        for (int i = 0; i < D; ++i) t[i] = dhmc_diag_scaled(q[i], mu[i], pr[i]);
        double s = canon_sum(T, D, [&](int i) { return dhmc_diag_term(q[i], mu[i], t[i]); });
        for (int i = 0; i < D; ++i) g[i] = dhmc_diag_grad(t[i]);
        return dhmc_diag_lq(s);
      }
      case DHMC_FAMILY_FUNNEL: {
        double v = q[0];
        double ev = dm_exp(-v);
        double S = canon_sum(T, D, [&](int i) { return dhmc_funnel_term(i, q[i]); });
        for (int i = 0; i < D; ++i) g[i] = dhmc_funnel_grad(i, q[i], v, ev, S, D);
        return dhmc_funnel_lq(v, ev, S, D);
      }
      case DHMC_FAMILY_LOGISTIC: {
        // params = [N, X row-major (N×D), y (N)]
        const int N = (int)params[0];
        const double* X = params.data() + 1;
        const double* y = X + (size_t)N * D;
        vec r(N), ll(N);
        for (int n = 0; n < N; ++n) {
          const double eta = dhmc_logit_eta(X + (size_t)n * D, &q[0], D);
          dhmc_logit_ll_resid(y[n], eta, &ll[n], &r[n]);
        }
        double sll = canon_sum(T, N, [&](int n) { return ll[n]; });
        double sb = canon_sum(T, D, [&](int i) { return q[i] * q[i]; });
        for (int j = 0; j < D; ++j) {
          double acc = 0.0;
          for (int n = 0; n < N; ++n) acc = dhmc_logit_mac(acc, X[(size_t)n * D + j], r[n]);
          g[j] = dhmc_logit_grad(acc, q[j]);
        }
        return dhmc_logit_lq(sll, sb);
      }
#ifdef DHMC_HAVE_USER_FAMILY
      case DHMC_FAMILY_USER: {
        // a user model header (include/dhmc_models.h "the model header contract"): K canonical sums over the elements,
        // derived scalars, then ℓ and the element-wise gradient — what eval_user does on the device
        constexpr int K = DHMC_USER_NSUMS, M = DHMC_USER_NSCALARS;
        double S[K + M > 0 ? K + M : 1] = {0.0};
        const double* qp = q.data();
        const double* pr = params.data();
#if DHMC_USER_NSUMS > 0
        for (int k = 0; k < K; ++k)
          S[k] = canon_sum(T, D, [&](int i) { double t[K]; dhmc_user_terms(i, D, qp, pr, t); return t[k]; });
#endif
#if DHMC_USER_NSCALARS > 0
        dhmc_user_prepare(D, qp, S, pr);
#endif
        for (int i = 0; i < D; ++i) g[i] = dhmc_user_grad(i, D, qp, S, pr);
        return dhmc_user_logdensity(D, qp, S, pr);
      }
#endif
    }
    throw ArgumentError("unknown family");
  }
};

// ------------------------------------------------------------- Hamiltonian
// Deterministic dense linear algebra used by the Symmetric metric.  The reference
// calls LAPACK/BLAS (`cholesky(inv(M⁻¹)).L`, `Symmetric * v`), whose summation order
// is unspecified; these restate the same mathematics with a fixed sequential
// order per output element (what each GPU thread does for its own elements).
inline bool cholesky_lower(const vec& A, int D, vec& L) {   // A = L Lᵀ, row-major
  L.assign((size_t)D * D, 0.0);
  for (int j = 0; j < D; ++j) {
    double s = A[(size_t)j * D + j];
    for (int k = 0; k < j; ++k) s = s - L[(size_t)j * D + k] * L[(size_t)j * D + k];
    if (!(s > 0.0) || !dm_isfinite(s)) return false;          // PosDefException
    const double d = dm_sqrt(s);
    L[(size_t)j * D + j] = d;
    for (int i = j + 1; i < D; ++i) {
      double t = A[(size_t)i * D + j];
      for (int k = 0; k < j; ++k) t = t - L[(size_t)i * D + k] * L[(size_t)j * D + k];
      L[(size_t)i * D + j] = t / d;
    }
  }
  return true;
}
// W = cholesky(inv(M⁻¹)).L — src/hamiltonian.jl:73: C = chol(M⁻¹); Cinv = C⁻¹; M = CinvᵀCinv; W = chol(M)
inline bool dense_factor(const vec& Minv, int D, vec& W) {
  vec C;
  if (!cholesky_lower(Minv, D, C)) return false;
  vec Ci((size_t)D * D, 0.0);
  for (int j = 0; j < D; ++j) {
    Ci[(size_t)j * D + j] = 1.0 / C[(size_t)j * D + j];
    for (int i = j + 1; i < D; ++i) {
      double s = 0.0;
      for (int k = j; k < i; ++k) s = s - C[(size_t)i * D + k] * Ci[(size_t)k * D + j];
      Ci[(size_t)i * D + j] = s / C[(size_t)i * D + i];
    }
  }
  vec M((size_t)D * D, 0.0);
  for (int i = 0; i < D; ++i)
    for (int j = 0; j <= i; ++j) {
      double s = 0.0;
      for (int k = i; k < D; ++k) s = s + Ci[(size_t)k * D + i] * Ci[(size_t)k * D + j];
      M[(size_t)i * D + j] = s; M[(size_t)j * D + i] = s;
    }
  return cholesky_lower(M, D, W);
}

// The last dense factorisation of this thread, or one the caller supplied (orc_seed_dense_factor): every oracle call that
// takes a Symmetric M⁻¹ builds its kinetic energy anew, and dense_factor is O(D³) (11 s at D = 2049), so a call whose M⁻¹
// equals the cached one bit for bit reuses its W.  dense_factor is deterministic, so the cache changes no result.
struct DenseFactorCache {
  vec minv, w;
};
inline DenseFactorCache& dense_factor_cache() {
  static thread_local DenseFactorCache c;
  return c;
}

// GaussianKineticEnergy — src/hamiltonian.jl:56-87: Diagonal M⁻¹ (:80, :87) or dense
// Symmetric M⁻¹ (:73).
struct KineticEnergy {
  bool dense = false;
  int D = 0;
  vec minv;  // diag(M⁻¹) [D]   or M⁻¹ [D*D] row-major (symmetric)
  vec w;     // W = Diagonal(.√inv.(diag(M⁻¹))) [D]   or lower-triangular W [D*D], W Wᵀ = M
  explicit KineticEnergy(const vec& m) : D((int)m.size()), minv(m), w(m.size()) {
    for (size_t i = 0; i < m.size(); ++i) w[i] = dm_sqrt(1.0 / m[i]);
  }
  KineticEnergy(int N, double m = 1.0) : KineticEnergy(vec(N, m)) {}  // :87
  static KineticEnergy Dense(const vec& M, int D_) {                 // :73
    KineticEnergy k(1);
    k.dense = true; k.D = D_; k.minv = M;
    if ((int)M.size() != D_ * D_) throw ArgumentError("checksquare(M⁻¹)");
    DenseFactorCache& c = dense_factor_cache();
    if (c.minv == M) { k.w = c.w; return k; }
    if (!dense_factor(M, D_, k.w)) throw DynamicHMCError("PosDefException: M⁻¹ is not positive definite");
    c.minv = M; c.w = k.w;
    return k;
  }
  int size() const { return D; }                                     // :96
  // M⁻¹ * p
  vec apply_minv(const vec& p) const {
    vec r(D);
    if (!dense) { for (int i = 0; i < D; ++i) r[i] = minv[i] * p[i]; return r; }
    // Symmetric(M⁻¹) * p as a blocked dot product per row (dm_blocked_dot): the order the device uses, on
    // CUDA cores and on the FP64 tensor cores alike
    for (int i = 0; i < D; ++i) r[i] = dm_blocked_dot(&minv[(size_t)i * D], 1, &p[0], D);
    return r;
  }
  // W * z
  vec apply_w(const vec& z) const {
    vec r(D);
    if (!dense) { for (int i = 0; i < D; ++i) r[i] = w[i] * z[i]; return r; }
    for (int i = 0; i < D; ++i) {
      double acc = 0.0;
      for (int j = 0; j <= i; ++j) acc = acc + w[(size_t)i * D + j] * z[j];
      r[i] = acc;
    }
    return r;
  }
};

// EvaluatedLogDensity — src/hamiltonian.jl:165-186
struct EvaluatedLogDensity {
  vec q; double lq; vec g;
};
// PhasePoint — src/hamiltonian.jl:225-234
struct PhasePoint {
  EvaluatedLogDensity Q; vec p;
};

inline bool all_finite(const vec& x) {
  for (double v : x) if (!dm_isfinite(v)) return false;
  return true;
}

// evaluate_ℓ — src/hamiltonian.jl:202-217
inline EvaluatedLogDensity evaluate_l(const Model& l, const vec& q, bool strict = false) {
  if (!all_finite(q)) throw DynamicHMCError("Position vector has non-finite elements.");
  vec g;
  double lq = l.logdensity_and_gradient(q, g);
  if ((dm_isfinite(lq) && all_finite(g)) || lq == -dm_inf()) {
    return {q, lq, g};
  } else if (!strict) {
    return {q, -dm_inf(), g};
  } else if (dm_isfinite(lq)) {
    throw DynamicHMCError("Gradient has non-finite elements.");
  } else {
    throw DynamicHMCError("Invalid log posterior.");
  }
}

struct Hamiltonian {  // src/hamiltonian.jl:130-150
  KineticEnergy k; Model l;
  Hamiltonian(const KineticEnergy& k_, const Model& l_) : k(k_), l(l_) {
    if (l.D != k.size()) throw ArgumentError("dimension(l) == size(k, 1)");
  }
  int T() const { return l.T; }
};

// kinetic_energy — src/hamiltonian.jl:103: dot(p, M⁻¹ * p) / 2
inline double kinetic_energy(const Hamiltonian& H, const vec& p) {
  const vec ps = H.k.apply_minv(p);
  double s = canon_sum(H.T(), (int)p.size(), [&](int i) { return p[i] * ps[i]; });
  return s / 2.0;
}
// calculate_p♯ — src/hamiltonian.jl:110
inline vec calculate_psharp(const Hamiltonian& H, const vec& p) {
  return H.k.apply_minv(p);
}
// logdensity(H, z) — src/hamiltonian.jl:251-256
inline double logdensity(const Hamiltonian& H, const PhasePoint& z) {
  double lq = z.Q.lq;
  if (!dm_isfinite(lq)) return -dm_inf();
  double K = kinetic_energy(H, z.p);
  return lq - (dm_isfinite(K) ? K : dm_inf());
}
// leapfrog — src/hamiltonian.jl:273-282 (operation order preserved)
inline PhasePoint leapfrog(const Hamiltonian& H, const PhasePoint& z, double eps) {
  if (!dm_isfinite(z.Q.lq))
    throw ArgumentError("Internal error: leapfrog called from non-finite log density");
  const int D = (int)z.p.size();
  const double h = eps / 2;
  vec pm(D), q1(D), p1(D);
  for (int i = 0; i < D; ++i) pm[i] = z.p[i] + h * z.Q.g[i];      // :277
  const vec vel = H.k.apply_minv(pm);                             // :117 → :110
  for (int i = 0; i < D; ++i) q1[i] = z.Q.q[i] + eps * vel[i];    // :278
  EvaluatedLogDensity Q1 = evaluate_l(H.l, q1);                   // :279
  for (int i = 0; i < D; ++i) p1[i] = pm[i] + h * Q1.g[i];        // :280
  return {Q1, p1};
}

// -------------------------------------------------------------------- RNG
// Counter-based stream standing in for Julia's rng argument.
struct Rng {
  dm_rng_key key; uint32_t t = 0; uint32_t n_exp = 0;
  std::vector<double>* exp_trace = nullptr;  // records drawn randexp values
  double randexp() {                          // Random.randexp, NUTS.jl:44
    double e = dm_randexp(key, t, n_exp++);
    if (exp_trace) exp_trace->push_back(e);
    return e;
  }
};

// rand_p — src/hamiltonian.jl:124:  κ.W * randn(rng, D)
inline vec rand_p(const dm_rng_key& key, uint32_t stream, uint32_t t, const KineticEnergy& k) {
  int D = k.size();
  vec z(D);
  for (int i = 0; i < D; ++i) z[i] = dm_normal_elem(key, stream, t, (uint32_t)i);
  return k.apply_w(z);
}
// random_position — src/mcmc.jl:108: rand(rng, N) .* 4 .- 2
inline vec random_position(const dm_rng_key& key, int D) {
  vec q(D);
  for (int i = 0; i < D; ++i)
    q[i] = dm_uniform_elem(key, DHMC_STREAM_Q0, 0, (uint32_t)i) * 4 - 2;
  return q;
}

// ===================================================================== trees
// src/trees.jl — generic doubling-tree code.

// Directions — src/trees.jl:19-34
struct Directions { uint32_t flags; };
inline std::pair<bool, Directions> next_direction(Directions d) {
  return {(d.flags & 1u) != 0, Directions{d.flags >> 1}};
}
constexpr int MAX_DIRECTIONS_DEPTH = 32;  // src/trees.jl:10

// InvalidTree — src/trees.jl:180-202
struct InvalidTree { long left, right; };
inline bool is_divergent(InvalidTree t) { return t.left == t.right; }
constexpr InvalidTree REACHED_MAX_DEPTH{1, 0};

// biased_progressive_logprob2 — src/trees.jl:159-161
inline double biased_progressive_logprob2(bool bias, double w1, double w2, double w) {
  return w2 - (bias ? w1 : w);
}

template <class Traj>
struct AdjResult {
  bool valid = false;
  InvalidTree invalid{0, 0};
  typename Traj::Zeta zeta{};
  double omega = 0;
  typename Traj::Tau tau{};
  typename Traj::Z z{};
  long i = 0;
};

// combine_turn_statistics_in_direction — src/trees.jl:135-141
template <class Traj>
typename Traj::Tau combine_turn_statistics_in_direction(Traj& tr, const typename Traj::Tau& t1,
                                                        const typename Traj::Tau& t2, bool fwd) {
  return fwd ? tr.combine_turn_statistics(t1, t2) : tr.combine_turn_statistics(t2, t1);
}

// combine_proposals_and_logweights — src/trees.jl:143-149
template <class Traj, class R>
std::pair<typename Traj::Zeta, double> combine_proposals_and_logweights(
    R& rng, Traj& tr, const typename Traj::Zeta& z1, const typename Traj::Zeta& z2, double w1,
    double w2, bool fwd, bool is_doubling) {
  double w = dm_logaddexp(w1, w2);
  double logprob2 = tr.calculate_logprob2(is_doubling, w1, w2, w);
  auto zeta = tr.combine_proposals(rng, z1, z2, logprob2, fwd);
  return {zeta, w};
}

// adjacent_tree — src/trees.jl:231-262
template <class Traj, class R>
std::pair<AdjResult<Traj>, typename Traj::V> adjacent_tree(R& rng, Traj& tr,
                                                           const typename Traj::Z& z, long i,
                                                           int depth, bool fwd) {
  long i1 = i + (fwd ? 1 : -1);
  if (depth == 0) {
    auto z1 = tr.move(z, fwd);
    auto lf = tr.leaf(z1, false);  // returns {ok, zeta, omega, tau, v}
    AdjResult<Traj> r;
    if (!lf.ok) {
      r.valid = false; r.invalid = InvalidTree{i1, i1};
    } else {
      r.valid = true; r.zeta = lf.zeta; r.omega = lf.omega; r.tau = lf.tau; r.z = z1; r.i = i1;
    }
    return {r, lf.v};
  }
  // "left" tree
  auto [tm, vm] = adjacent_tree(rng, tr, z, i, depth - 1, fwd);
  if (!tm.valid) return {tm, vm};
  // "right" tree — visited information from left is kept even if invalid
  auto [tp, vp] = adjacent_tree(rng, tr, tm.z, tm.i, depth - 1, fwd);
  auto v = tr.combine_visited_statistics(vm, vp);
  if (!tp.valid) return {tp, v};
  // turning invalidates
  auto tau = combine_turn_statistics_in_direction(tr, tm.tau, tp.tau, fwd);
  if (tr.is_turning(tau)) {
    AdjResult<Traj> r; r.valid = false; r.invalid = InvalidTree{i1, tp.i};
    return {r, v};
  }
  // valid subtree, combine proposals
  auto [zeta, omega] =
      combine_proposals_and_logweights(rng, tr, tm.zeta, tp.zeta, tm.omega, tp.omega, fwd, false);
  AdjResult<Traj> r;
  r.valid = true; r.zeta = zeta; r.omega = omega; r.tau = tau; r.z = tp.z; r.i = tp.i;
  return {r, v};
}

template <class Traj>
struct SampleResult {
  typename Traj::Zeta zeta; typename Traj::V v; InvalidTree termination; int depth;
};

// sample_trajectory — src/trees.jl:283-319
template <class Traj, class R>
SampleResult<Traj> sample_trajectory(R& rng, Traj& tr, const typename Traj::Z& z, int max_depth,
                                     Directions directions) {
  if (!(max_depth <= MAX_DIRECTIONS_DEPTH)) throw ArgumentError("max_depth ≤ MAX_DIRECTIONS_DEPTH");
  auto lf = tr.leaf(z, true);
  auto zeta = lf.zeta; double omega = lf.omega; auto tau = lf.tau; auto v = lf.v;
  auto zm = z, zp = z;
  int depth = 0;
  InvalidTree termination = REACHED_MAX_DEPTH;
  long im = 0, ip = 0;
  while (depth < max_depth) {
    auto [fwd, nd] = next_direction(directions);
    directions = nd;
    auto [t1, v1] = adjacent_tree(rng, tr, fwd ? zp : zm, fwd ? ip : im, depth, fwd);
    v = tr.combine_visited_statistics(v, v1);
    // invalid adjacent tree: stop
    if (!t1.valid) { termination = t1.invalid; break; }
    // update edges and combine proposals
    if (fwd) { zp = t1.z; ip = t1.i; } else { zm = t1.z; im = t1.i; }
    // tree has doubled successfully
    auto zw = combine_proposals_and_logweights(rng, tr, zeta, t1.zeta, omega, t1.omega, fwd, true);
    zeta = zw.first; omega = zw.second;
    depth += 1;
    // when the combined tree is turning, stop
    tau = combine_turn_statistics_in_direction(tr, tau, t1.tau, fwd);
    if (tr.is_turning(tau)) { termination = InvalidTree{im, ip}; break; }
  }
  return {zeta, v, termination, depth};
}

// ============================================================ DummyTrajectory
// test/test_trees.jl:28-103 — the reference's fake trajectory for unit tests.
struct DummyTrajectory {
  struct ZetaT { long lo = 0, hi = 0; std::vector<double> lp; };
  struct TauT { bool flag = false; long lo = 0, hi = 0; };
  struct VT { double a = 0; long steps = 0; };
  using Z = long; using Zeta = ZetaT; using Tau = TauT; using V = VT;
  struct Leaf { bool ok; Zeta zeta; double omega; Tau tau; V v; };

  std::set<long> turning, divergent;
  std::function<double(long)> l = [](long z) { return -((double)(z - 3) * (double)(z - 3)) * 0.1; };
  std::vector<long> visited;
  bool adjacency_ok = true;  // mirrors the @test assertions inside the callbacks

  Z move(Z z, bool fwd) { return z + (fwd ? 1 : -1); }            // :45
  bool is_turning(const Tau& t) {                                 // :49-53
    if (!(t.hi - t.lo + 1 > 1)) adjacency_ok = false;
    return t.flag;
  }
  Tau combine_turn_statistics(const Tau& a, const Tau& b) {       // :55-62
    if (a.hi + 1 != b.lo) adjacency_ok = false;
    return {a.flag && b.flag, a.lo, b.hi};
  }
  V combine_visited_statistics(const V& a, const V& b) { return {a.a + b.a, a.steps + b.steps}; }
  double calculate_logprob2(bool dbl, double w1, double w2, double w) {  // :84-86
    return biased_progressive_logprob2(dbl, w1, w2, w);
  }
  template <class R>
  Zeta combine_proposals(R&, Zeta z1, Zeta z2, double logprob2, bool fwd) {  // :70-82
    double lp2 = logprob2 > 0 ? 0.0 : logprob2;
    double lp1 = logprob2 > 0 ? -dm_inf() : std::log1p(-std::exp(lp2));  // log1mexp
    if (!fwd) { std::swap(z1, z2); std::swap(lp1, lp2); }
    if (z1.hi + 1 != z2.lo) adjacency_ok = false;
    Zeta r; r.lo = z1.lo; r.hi = z2.hi;
    for (double x : z1.lp) r.lp.push_back(x + lp1);
    for (double x : z2.lp) r.lp.push_back(x + lp2);
    return r;
  }
  Leaf leaf(Z z, bool is_initial) {                               // :88-103
    bool d = divergent.count(z) > 0;
    if (is_initial && d) throw ArgumentError("don't start with divergent");
    double delta = l(z);
    V v = is_initial ? V{0.0, 0} : V{std::min(std::exp(delta), 1.0), 1};
    if (!is_initial) visited.push_back(z);
    if (d) return {false, {}, 0, {}, v};
    Zeta zt; zt.lo = z; zt.hi = z; zt.lp = {0.0};
    return {true, zt, delta, Tau{turning.count(z) > 0, z, z}, v};
  }
};
struct NoRng {};

// ====================================================================== NUTS
// src/NUTS.jl

// AcceptanceStatistic — src/NUTS.jl:59-89
struct AcceptanceStatistic { double log_sum_a; long steps; };
inline AcceptanceStatistic combine_acceptance_statistics(AcceptanceStatistic A, AcceptanceStatistic B) {
  return {dm_logaddexp(A.log_sum_a, B.log_sum_a), A.steps + B.steps};     // :69-71
}
inline AcceptanceStatistic leaf_acceptance_statistic(double delta, bool is_initial) {  // :78-80
  return is_initial ? AcceptanceStatistic{-dm_inf(), 0}
                    : AcceptanceStatistic{dm_min_nan(delta, 0.0), 1};
}
inline double acceptance_rate(AcceptanceStatistic A) {                    // :87
  return dm_min_nan(dm_exp(A.log_sum_a) / (double)A.steps, 1.0);
}

// GeneralizedTurnStatistic — src/NUTS.jl:107-118 (`turning` stands for `nothing`)
struct TurnStatistic { vec pm, psm, pp, psp, rho; bool turning = false; };

// rand_bool_logprob — src/NUTS.jl:43-45: no draw consumed when logprob ≥ 0
template <class R>
bool rand_bool_logprob(R& rng, double logprob) {
  return logprob >= 0 || (rng.randexp() > -logprob);
}

struct TrajectoryNUTS {  // src/NUTS.jl:15-26
  using Z = PhasePoint;
  struct ZetaT { PhasePoint z; double H = 0; };  // proposal (+ its cached logdensity(H, z))
  using Zeta = ZetaT; using Tau = TurnStatistic; using V = AcceptanceStatistic;
  struct Leaf { bool ok; Zeta zeta; double omega; Tau tau; V v; };

  const Hamiltonian& H; double pi0; double eps; double min_delta;
  std::vector<int>* accept_trace = nullptr;  // one entry per combine_proposals call
  int T() const { return H.T(); }

  Z move(const Z& z, bool fwd) { return leapfrog(H, z, fwd ? eps : -eps); }  // :28-31

  double dot(const vec& a, const vec& b) {
    return canon_sum(T(), (int)a.size(), [&](int i) { return a[i] * b[i]; });
  }
  bool _is_turning(const vec& psm, const vec& psp, const vec& rho) {          // :130
    return dot(psm, rho) < 0 || dot(psp, rho) < 0;
  }
  static vec add(const vec& a, const vec& b) {
    vec r(a.size());
    for (size_t i = 0; i < a.size(); ++i) r[i] = a[i] + b[i];
    return r;
  }
  Tau combine_turn_statistics(const Tau& x, const Tau& y) {                   // :132-139
    Tau out;
    if (_is_turning(x.psm, y.psm, add(x.rho, y.pm))) { out.turning = true; return out; }
    if (_is_turning(x.psp, y.psp, add(x.pp, y.rho))) { out.turning = true; return out; }
    vec rho = add(x.rho, y.rho);
    if (_is_turning(x.psm, y.psp, rho)) { out.turning = true; return out; }
    return Tau{x.pm, x.psm, y.pp, y.psp, rho, false};
  }
  bool is_turning(const Tau& t) { return t.turning; }                         // :141-142
  V combine_visited_statistics(const V& a, const V& b) { return combine_acceptance_statistics(a, b); }
  double calculate_logprob2(bool dbl, double w1, double w2, double w) {       // :47-49
    return biased_progressive_logprob2(dbl, w1, w2, w);
  }
  template <class R>
  Zeta combine_proposals(R& rng, const Zeta& z1, const Zeta& z2, double logprob2, bool) {  // :51-53
    bool b = rand_bool_logprob(rng, logprob2);
    if (accept_trace) accept_trace->push_back(b ? 1 : 0);
    return b ? z2 : z1;
  }
  Leaf leaf(const Z& z, bool is_initial) {                                    // :148-159
    double Hz = logdensity(H, z);
    double delta = is_initial ? 0.0 : Hz - pi0;
    bool isdiv = delta < min_delta;
    V v = leaf_acceptance_statistic(delta, is_initial);
    if (isdiv) return {false, {}, 0, {}, v};
    vec ps = calculate_psharp(H, z.p);                                        // :120-123
    Tau tau{z.p, ps, z.p, ps, z.p, false};
    return {true, Zeta{z, Hz}, delta, tau, v};
  }
};

struct NUTS {  // src/NUTS.jl:178-195
  int max_depth = 10; double min_delta = -1000.0;
  void check() const {
    if (!(0 < max_depth && max_depth <= MAX_DIRECTIONS_DEPTH)) throw ArgumentError("0 < max_depth ≤ 32");
    if (!(min_delta < 0)) throw ArgumentError("min_Δ < 0");
  }
};

// TreeStatisticsNUTS — src/NUTS.jl:208-221 (56 bytes, isbits)
struct TreeStatistics {
  double pi; int64_t depth; int64_t left; int64_t right; double acceptance_rate; int64_t steps;
  uint32_t directions; uint32_t pad;
};

// sample_tree — src/NUTS.jl:232-241.  `p` and `directions` follow the keyword
// defaults: p = rand_p(rng, H.κ) first, directions = rand(rng, Directions) second.
inline std::pair<EvaluatedLogDensity, TreeStatistics> sample_tree(
    Rng& rng, const NUTS& alg, const Hamiltonian& H, const EvaluatedLogDensity& Q, double eps,
    const vec* p_override = nullptr, const uint32_t* dir_override = nullptr,
    std::vector<int>* accept_trace = nullptr) {
  vec p = p_override ? *p_override : rand_p(rng.key, DHMC_STREAM_P, rng.t, H.k);
  uint32_t dirs = dir_override ? *dir_override : dm_rand_directions(rng.key, rng.t);
  rng.n_exp = 0;
  PhasePoint z{Q, p};
  TrajectoryNUTS tr{H, logdensity(H, z), eps, alg.min_delta, accept_trace};
  auto r = sample_trajectory(rng, tr, z, alg.max_depth, Directions{dirs});
  TreeStatistics ts{};
  ts.pi = logdensity(H, r.zeta.z);
  ts.depth = r.depth; ts.left = r.termination.left; ts.right = r.termination.right;
  ts.acceptance_rate = acceptance_rate(r.v); ts.steps = r.v.steps; ts.directions = dirs; ts.pad = 0;
  return {r.zeta.z.Q, ts};
}

// ================================================================== stepsize
// src/stepsize.jl

struct InitialStepsizeSearch {  // :23-36
  double initial_eps = 0.1; double log_threshold = -0.2231435513142097557662950903098345033746;
  int maxiter_crossing = 400;
  void check() const {
    if (!(dm_isfinite(log_threshold) && log_threshold < 0)) throw ArgumentError("log_threshold");
    if (!(dm_isfinite(initial_eps) && 0 < initial_eps)) throw ArgumentError("initial_ϵ");
    if (!(maxiter_crossing >= 50)) throw ArgumentError("maxiter_crossing ≥ 50");
  }
};
// find_initial_stepsize — :46-60
template <class F>
double find_initial_stepsize(const InitialStepsizeSearch& par, F A) {
  double eps = par.initial_eps;
  double Ae = A(eps);
  bool dbl = Ae > par.log_threshold;
  for (int it = 0; it < par.maxiter_crossing; ++it) {
    double eps1 = dbl ? 2 * eps : eps / 2;
    double Ae1 = A(eps1);
    if (dbl ? Ae1 < par.log_threshold : Ae1 > par.log_threshold) return eps1;
    eps = eps1;
  }
  throw DynamicHMCError(std::string("Initial stepsize search reached maximum number of iterations from ") +
                        (dbl ? "below" : "above") + " without crossing.");
}
// local_log_acceptance_ratio — :75-85
inline std::function<double(double)> local_log_acceptance_ratio(const Hamiltonian& H, const PhasePoint& z) {
  double l0 = logdensity(H, z);
  if (!dm_isfinite(l0)) throw DynamicHMCError("Starting point has non-finite density.");
  return [&H, z, l0](double eps) {
    PhasePoint z1 = leapfrog(H, z, eps);
    return logdensity(H, z1) - l0;
  };
}

struct DualAveraging {  // :98-118
  double delta = 0.8, gamma = 0.05, kappa = 0.75; int t0 = 10;
  void check() const {
    if (!(0 < delta && delta < 1)) throw ArgumentError("0 < δ < 1");
    if (!(gamma > 0)) throw ArgumentError("γ > 0");
    if (!(0.5 < kappa && kappa <= 1)) throw ArgumentError("0.5 < κ ≤ 1");
    if (!(t0 >= 0)) throw ArgumentError("t₀ ≥ 0");
  }
};
struct DualAveragingState { double mu; int64_t m; double Hbar, logeps, logepsbar; };  // :121-127
// initial_adaptation_state — :134-138
inline DualAveragingState initial_adaptation_state(const DualAveraging&, double eps) {
  if (!(eps > 0)) throw ArgumentError("ϵ > 0");
  double le = dm_log(eps);
  return {dm_log(10.0) + le, 1, 0.0, le, 0.0};
}
// adapt_stepsize — :147-156
inline DualAveragingState adapt_stepsize(const DualAveraging& P, DualAveragingState A, double a) {
  if (!(0 <= a && a <= 1)) throw ArgumentError("0 ≤ a ≤ 1");
  A.m += 1;
  A.Hbar += (P.delta - a - A.Hbar) / (double)(A.m + P.t0);
  A.logeps = A.mu - dm_sqrt((double)A.m) / P.gamma * A.Hbar;
  A.logepsbar += dm_pow((double)A.m, -P.kappa) * (A.logeps - A.logepsbar);
  return A;
}
inline double current_eps(const DualAveragingState& A) { return dm_exp(A.logeps); }      // :163
inline double final_eps(const DualAveragingState& A) { return dm_exp(A.logepsbar); }     // :170

// ====================================================================== mcmc
// src/mcmc.jl

struct WarmupState { EvaluatedLogDensity Q; KineticEnergy k; double eps; bool has_eps; };  // :72-79

// sample_M⁻¹(Diagonal, X) = Diagonal(vec(var(X; dims = 2))) — mcmc.jl:209.
// Julia's var is two-pass: mean first, then sum of squared deviations / (n-1).
inline vec sample_minv_twopass(const std::vector<vec>& X) {
  size_t n = X.size(), D = X[0].size();
  vec out(D);
  for (size_t i = 0; i < D; ++i) {
    double s = 0; for (size_t j = 0; j < n; ++j) s += X[j][i];
    double mean = s / (double)n;
    double ss = 0; for (size_t j = 0; j < n; ++j) { double d = X[j][i] - mean; ss += d * d; }
    out[i] = ss / (double)(n - 1);
  }
  return out;
}
// Streaming (Welford) variant — what the device accumulates; agrees with the
// two-pass value to rounding (tests/test_oracle_mcmc.py pins the gap).
struct Welford {
  int64_t n = 0; vec mean, m2;
  explicit Welford(int D) : mean(D, 0.0), m2(D, 0.0) {}
  void push(const vec& x) {
    n += 1;
    for (size_t i = 0; i < x.size(); ++i) {
      double d = x[i] - mean[i];
      mean[i] = mean[i] + d / (double)n;
      m2[i] = m2[i] + d * (x[i] - mean[i]);
    }
  }
  vec variance() const {
    vec v(mean.size());
    for (size_t i = 0; i < v.size(); ++i) v[i] = m2[i] / (double)(n - 1);
    return v;
  }
};

// sample_M⁻¹(Symmetric, X) = Symmetric(cov(X; dims = 2)) — mcmc.jl:211 (two-pass)
inline vec sample_cov_twopass(const std::vector<vec>& X) {
  size_t n = X.size(), D = X[0].size();
  vec mean(D), C(D * D);
  for (size_t i = 0; i < D; ++i) { double s = 0; for (size_t k = 0; k < n; ++k) s += X[k][i]; mean[i] = s / (double)n; }
  for (size_t i = 0; i < D; ++i)
    for (size_t j = 0; j <= i; ++j) {
      double ss = 0;
      for (size_t k = 0; k < n; ++k) ss += (X[k][i] - mean[i]) * (X[k][j] - mean[j]);
      C[i * D + j] = C[j * D + i] = ss / (double)(n - 1);
    }
  return C;
}
// streaming co-moments (what the device accumulates): lower triangle, mirrored
struct WelfordCov {
  int64_t n = 0; int D; vec mean, c;
  explicit WelfordCov(int D_) : D(D_), mean(D_, 0.0), c((size_t)D_ * D_, 0.0) {}
  void push(const vec& x) {
    n += 1;
    vec d(D);
    for (int i = 0; i < D; ++i) { d[i] = x[i] - mean[i]; mean[i] = mean[i] + d[i] / (double)n; }
    for (int i = 0; i < D; ++i)
      for (int j = 0; j <= i; ++j) c[(size_t)i * D + j] = c[(size_t)i * D + j] + d[i] * (x[j] - mean[j]);
  }
  vec covariance() const {
    vec C((size_t)D * D);
    for (int i = 0; i < D; ++i)
      for (int j = 0; j <= i; ++j) C[(size_t)i * D + j] = C[(size_t)j * D + i] = c[(size_t)i * D + j] / (double)(n - 1);
    return C;
  }
};
// regularize_M⁻¹(Σ::Symmetric, λ) = (1 - λ) * Σ + λ * Diagonal(diag(Σ)) — mcmc.jl:218-221
inline vec regularize_dense(const vec& S, int D, double lambda) {
  vec R((size_t)D * D);
  for (int i = 0; i < D; ++i)
    for (int j = 0; j < D; ++j) {
      double v = (1 - lambda) * S[(size_t)i * D + j];
      if (i == j) v = v + lambda * S[(size_t)i * D + i];
      R[(size_t)i * D + j] = v;
    }
  return R;
}

enum StageKind { STAGE_NOTHING = 0, STAGE_STEPSIZE_SEARCH = 1, STAGE_TUNING = 2 };
// METRIC_SYMMETRIC_POOLED is NOT in the reference (which adapts every chain on its own draws, mcmc.jl:282): the optional
// exchange of SURVEY.md §8e — the eight chains of a group share one dense metric estimated from their pooled window.
enum MetricKind { METRIC_NOTHING = 0, METRIC_DIAGONAL = 1, METRIC_SYMMETRIC = 2, METRIC_SYMMETRIC_POOLED = 3 };
constexpr int kPoolGroup = 8;
struct Stage {
  int kind = STAGE_TUNING; int N = 0; int metric = METRIC_NOTHING; bool dual_averaging = true;
  double lambda = 0;  // regularisation; identity for Diagonal (mcmc.jl:223)
  InitialStepsizeSearch search; DualAveraging da;
};
// default_warmup_stages — mcmc.jl:415-425
inline std::vector<Stage> default_warmup_stages(int init_steps = 75, int middle_steps = 25,
                                                int doubling_stages = 5, int terminating_steps = 50,
                                                bool search = true, bool dual_averaging = true) {
  std::vector<Stage> st;
  if (search) { Stage s; s.kind = STAGE_STEPSIZE_SEARCH; st.push_back(s); }
  auto tuning = [&](int N, int metric) {
    Stage s; s.kind = STAGE_TUNING; s.N = N; s.metric = metric; s.dual_averaging = dual_averaging;
    s.lambda = 5.0 / N; return s;
  };
  if (dual_averaging) st.push_back(tuning(init_steps, METRIC_NOTHING));
  for (int i = 0; i < doubling_stages; ++i) st.push_back(tuning(middle_steps * (1 << i), METRIC_DIAGONAL));
  if (dual_averaging) st.push_back(tuning(terminating_steps, METRIC_NOTHING));
  return st;
}

struct ChainOutput {
  std::vector<vec> posterior;            // [draw][param]
  std::vector<TreeStatistics> stats;
  std::vector<double> logdensities;
  std::vector<double> eps_used;          // warmup stages only (ϵs, mcmc.jl:273)
};

struct Sampler {  // SamplingLogDensity + the rng counter — mcmc.jl:41-53
  Model l; NUTS alg; dm_rng_key key; uint32_t t = 0;  // t = transitions done so far
  bool welford = false;  // metric estimator: false = two-pass var (reference), true = streaming
};

// warmup(::InitialStepsizeSearch) — mcmc.jl:134-148
inline void warmup_search(Sampler& S, const InitialStepsizeSearch& par, WarmupState& st) {
  if (st.has_eps) throw ArgumentError("stepsize ϵ manually specified, won't perform initial search");
  par.check();
  PhasePoint z{st.Q, rand_p(S.key, DHMC_STREAM_PSEARCH, 0, st.k)};
  Hamiltonian H(st.k, S.l);
  st.eps = find_initial_stepsize(par, local_log_acceptance_ratio(H, z));
  st.has_eps = true;
}

// warmup(::TuningNUTS{M}) — mcmc.jl:258-286
struct WelfordCov;
inline ChainOutput warmup_tuning(Sampler& S, const Stage& stage, WarmupState& st, WelfordCov* pooled_out = nullptr);
// Pooled window covariance of a chain group from the chains' streaming means / co-moments (each over n draws), with the
// reference's shrinkage (regularize_M⁻¹, mcmc.jl:218-221).  Fixed order (chains 0…G−1, sequential) — what k_cov_pool does.
inline vec pooled_regularized_cov(const std::vector<WelfordCov>& w, int D, double lambda);

inline ChainOutput warmup_tuning(Sampler& S, const Stage& stage, WarmupState& st, WelfordCov* pooled_out) {
  if (!(stage.N >= 20)) throw ArgumentError("N ≥ 20");
  if (!(stage.lambda >= 0)) throw ArgumentError("λ ≥ 0");
  ChainOutput out;
  Hamiltonian H(st.k, S.l);
  DualAveragingState da{};
  double fixed_eps = st.eps;
  if (stage.dual_averaging) da = initial_adaptation_state(stage.da, st.eps);
  Welford wf(S.l.D);
  const bool pooled = stage.metric == METRIC_SYMMETRIC_POOLED;
  if (pooled && !pooled_out) throw ArgumentError("the pooled metric needs the whole chain group (mcmc_with_warmup_pooled)");
  WelfordCov wc((stage.metric == METRIC_SYMMETRIC || pooled) ? S.l.D : 1);
  for (int i = 0; i < stage.N; ++i) {
    double eps = stage.dual_averaging ? current_eps(da) : fixed_eps;
    out.eps_used.push_back(eps);
    Rng rng{S.key, S.t, 0};
    auto [Q, stats] = sample_tree(rng, S.alg, H, st.Q, eps);
    S.t += 1;
    st.Q = Q;
    out.posterior.push_back(Q.q); out.logdensities.push_back(Q.lq); out.stats.push_back(stats);
    if (stage.metric == METRIC_DIAGONAL && S.welford) wf.push(Q.q);
    if ((stage.metric == METRIC_SYMMETRIC && S.welford) || pooled) wc.push(Q.q);
    if (stage.dual_averaging) da = adapt_stepsize(stage.da, da, stats.acceptance_rate);
  }
  if (stage.metric == METRIC_DIAGONAL) {
    vec minv = S.welford ? wf.variance() : sample_minv_twopass(out.posterior);
    st.k = KineticEnergy(minv);  // regularize_M⁻¹(::Diagonal) is the identity — mcmc.jl:223
  } else if (stage.metric == METRIC_SYMMETRIC) {
    vec C = S.welford ? wc.covariance() : sample_cov_twopass(out.posterior);
    st.k = KineticEnergy::Dense(regularize_dense(C, S.l.D, stage.lambda), S.l.D);   // mcmc.jl:282
  }
  if (pooled) *pooled_out = wc;            // κ of the whole group is set by the caller from the pooled moments
  st.eps = stage.dual_averaging ? final_eps(da) : fixed_eps;
  return out;
}
inline vec pooled_regularized_cov(const std::vector<WelfordCov>& w, int D, double lambda) {
  const int G = (int)w.size();
  const double n = (double)w[0].n;
  vec mean(D);
  for (int i = 0; i < D; ++i) {
    double m = w[0].mean[i];
    for (int c = 1; c < G; ++c) m = m + w[c].mean[i];
    mean[i] = m / (double)G;
  }
  vec S((size_t)D * D);
  for (int i = 0; i < D; ++i)
    for (int j = 0; j <= i; ++j) {
      double acc = 0.0;
      for (int c = 0; c < G; ++c) {
        const double di = w[c].mean[i] - mean[i], dj = w[c].mean[j] - mean[j];
        acc = acc + (w[c].c[(size_t)i * D + j] + (n * di) * dj);
      }
      S[(size_t)i * D + j] = S[(size_t)j * D + i] = acc / ((double)G * n - 1.0);
    }
  return regularize_dense(S, D, lambda);
}

// mcmc — mcmc.jl:366-381
inline ChainOutput mcmc(Sampler& S, int N, WarmupState& st) {
  ChainOutput out;
  Hamiltonian H(st.k, S.l);
  for (int i = 0; i < N; ++i) {
    Rng rng{S.key, S.t, 0};
    auto [Q, stats] = sample_tree(rng, S.alg, H, st.Q, st.eps);
    S.t += 1;
    st.Q = Q;
    out.posterior.push_back(Q.q); out.logdensities.push_back(Q.lq); out.stats.push_back(stats);
  }
  return out;
}

// initialize_warmup_state — mcmc.jl:129-132 (strict evaluation).  `dense`: minv is a Symmetric M⁻¹ [D*D] (the caller says so:
// at D = 1 the two kinds have the same length)
inline WarmupState initialize_warmup_state(const Sampler& S, const vec* q, const vec* minv, const double* eps,
                                           bool dense = false) {
  vec q0 = q ? *q : random_position(S.key, S.l.D);
  KineticEnergy k = !minv ? KineticEnergy(S.l.D) : dense ? KineticEnergy::Dense(*minv, S.l.D) : KineticEnergy(*minv);
  return WarmupState{evaluate_l(S.l, q0, true), k, eps ? *eps : 0.0, eps != nullptr};
}

// mcmc_keep_warmup / mcmc_with_warmup — mcmc.jl:521-532, :575-584
struct McmcResult { ChainOutput inference; WarmupState final_state; std::vector<ChainOutput> warmup; };
inline McmcResult mcmc_with_warmup(Sampler& S, int N, const std::vector<Stage>& stages,
                                   const vec* q = nullptr, const vec* minv = nullptr,
                                   const double* eps = nullptr, bool dense_minv = false) {
  S.alg.check();
  WarmupState st = initialize_warmup_state(S, q, minv, eps, dense_minv);
  std::vector<ChainOutput> wu;
  for (const Stage& s : stages) {                       // _warmup fold, mcmc.jl:450-457
    if (s.kind == STAGE_NOTHING) { wu.push_back({}); continue; }   // :99-101
    if (s.kind == STAGE_STEPSIZE_SEARCH) { warmup_search(S, s.search, st); wu.push_back({}); continue; }
    if (!st.has_eps) throw ArgumentError("TuningNUTS needs a stepsize");
    wu.push_back(warmup_tuning(S, s, st));
  }
  if (!st.has_eps) throw ArgumentError("mcmc needs a stepsize");
  ChainOutput inf = mcmc(S, N, st);
  return McmcResult{inf, st, wu};
}

// mcmc_with_warmup for a chain group with pooled Symmetric stages: the chains run stage by stage; a pooled stage ends with
// one metric for the whole group.  Everything else is the per-chain reference flow.
inline std::vector<McmcResult> mcmc_with_warmup_pooled(std::vector<Sampler>& S, int N, const std::vector<Stage>& stages) {
  const int G = (int)S.size();
  std::vector<WarmupState> st;
  std::vector<std::vector<ChainOutput>> wu(G);
  for (int c = 0; c < G; ++c) { S[c].alg.check(); st.push_back(initialize_warmup_state(S[c], nullptr, nullptr, nullptr)); }
  for (const Stage& s : stages) {
    if (s.kind == STAGE_NOTHING) { for (int c = 0; c < G; ++c) wu[c].push_back({}); continue; }
    if (s.kind == STAGE_STEPSIZE_SEARCH) {
      for (int c = 0; c < G; ++c) { warmup_search(S[c], s.search, st[c]); wu[c].push_back({}); }
      continue;
    }
    std::vector<WelfordCov> w(G, WelfordCov(1));
    for (int c = 0; c < G; ++c) {
      if (!st[c].has_eps) throw ArgumentError("TuningNUTS needs a stepsize");
      wu[c].push_back(warmup_tuning(S[c], s, st[c], s.metric == METRIC_SYMMETRIC_POOLED ? &w[c] : nullptr));
    }
    if (s.metric == METRIC_SYMMETRIC_POOLED) {
      const vec M = pooled_regularized_cov(w, S[0].l.D, s.lambda);
      const KineticEnergy k = KineticEnergy::Dense(M, S[0].l.D);
      for (int c = 0; c < G; ++c) st[c].k = k;
    }
  }
  std::vector<McmcResult> res;
  for (int c = 0; c < G; ++c) {
    ChainOutput inf = mcmc(S[c], N, st[c]);
    res.push_back(McmcResult{inf, st[c], wu[c]});
  }
  return res;
}

}  // namespace orc
