// nuts_machine.cuh — the NUTS transition of DynamicHMC.jl with the recursive
// doubling tree flattened into an explicit stack (one chain per chain group).
//
// Reference being replaced (paths in tpapp/DynamicHMC.jl v3.6.0):
//   sample_tree           src/NUTS.jl:232-241
//   sample_trajectory     src/trees.jl:283-319   (doubling loop)
//   adjacent_tree         src/trees.jl:231-262   (recursion -> stack, below)
//   leaf / combine_*      src/NUTS.jl:28-159
//   adapt_stepsize        src/stepsize.jl:134-170
//   find_initial_stepsize src/stepsize.jl:46-85
//   warmup(TuningNUTS)    src/mcmc.jl:258-286, mcmc src/mcmc.jl:366-381
//
// This file holds ONLY scalar control flow.  Every D-length vector lives behind
// the Backend (registers + shared/global "slots" on the GPU, see
// device_backend.cuh).  All threads of a chain group execute this code
// redundantly with identical scalars (every scalar is derived from all-reduced
// sums and counter-based RNG), so there is no intra-chain divergence and no
// broadcast step.  tests/hostsim compiles the same control code against a
// plain-loop backend so that the `-m "not gpu"` tests can check the state
// machine against the recursive oracle without a GPU.
//
// Flattening rule (SURVEY.md §3.6 item 4): number the leaves of a depth-d
// adjacent tree k = 1..2^d in build order; after leaf k perform ctz(k) merges,
// each combining the top stack entry E (earlier-built) with the incoming
// subtree L (later-built).  That reproduces the recursion's post-order and
// therefore its randexp consumption order.
//
// Turn statistics are kept in BUILD order (first/last built leaf momentum and
// the momentum sum ρ).  With E earlier and L later the three checks of
// combine_turn_statistics (NUTS.jl:132-139) become, for either direction,
//     (E.ρ + L.first) · {E.first♯, L.first♯},
//     (E.last + L.ρ)  · {E.last♯,  L.last♯},
//     (E.ρ + L.ρ)     · {E.first♯, L.last♯},
// the same six dot products the reference evaluates after
// combine_turn_statistics_in_direction (trees.jl:135-141) has ordered its
// arguments spatially.  p♯ = M⁻¹p is recomputed from p (diagonal metric).
#pragma once
#include "../../include/dhmc.h"
#include "../../include/dhmc_math.h"

#if defined(__CUDACC__)
#define DHMC_M __device__ __forceinline__
#define DHMC_COLD __device__ __noinline__      // rarely taken paths: kept out of line so that they cost the hot loop no registers
#else
#define DHMC_M inline
#define DHMC_COLD inline
#endif

namespace dhmc {

constexpr int kMaxLevels = 32;   // max_depth <= MAX_DIRECTIONS_DEPTH = 32 (trees.jl:10, NUTS.jl:190)
constexpr int kMaskWords = 3;    // slot free-list: 64 slots in a register word + two spill words (max_depth > 12 needs up to 164 slots)
constexpr int kFixedSlots = 7;   // OTHER(q,p,g) NEARP RHOT ZT(q,g)
constexpr int kWelfordSlots = 2; // running mean / M2 of the metric window

DHMC_HD int slots_needed(int max_depth) {
  // stack: one leaf entry (3) + (max_depth-2) inner entries (5) + transient
  int d = max_depth - 1;  // deepest adjacent tree
  int stack = d > 0 ? 3 + 5 * (d - 1) + 2 : 3;
  return kFixedSlots + kWelfordSlots + stack;
}

// One stack entry = a completed subtree, in build order.
struct Entry {
  double omega;   // log weight ω of the subtree
  double vlog;    // visited statistic: log Σ α   (AcceptanceStatistic, NUTS.jl:59-66)
  double zlq;     // proposal ζ: ℓ(q)
  double zH;      //             logdensity(H, ζ)
  int vsteps;     // visited statistic: leapfrog steps
  int ifirst;     // position of the first-built leaf (i′ of adjacent_tree)
  short sfirst, slast, srho;  // slots: p of first / last built leaf, ρ
  short szq, szg;             // slots: proposal q and ∇ℓ
  short leaf;                 // 1: single leaf (sfirst == slast == srho)
};

struct AdaptConfig {
  int adapt;           // 1: DualAveraging, 0: FixedStepsize (stepsize.jl:181-189)
  double delta, gamma, kappa; int t0;
  int metric;          // DHMC_METRIC_*
};

// Transition-level scalars (touched once per doubling or per transition, not per leaf).
// The GPU backend keeps them in shared memory (one copy per warp, every lane writes the same
// values) so that the per-leaf state stays in registers: left to the compiler they are spilled to
// local memory, i.e. to L2 latency, because shared memory takes almost all of the L1 carve-out.
struct TopState {
  double other_lq, zt_lq, zt_H, omega_top, v_log, eps;
  double da_mu, da_Hbar, da_logeps, da_logepsbar;
  long v_steps, term_l, term_r, da_m, total_steps;
  int i_near, i_far, depth, regs_fwd;
  uint32_t flags, dirs;
  int s_oq, s_og, s_zq, s_zg, s_op, s_near, s_rhot;
  uint64_t free_hi[kMaskWords - 1];   // slots 64…: touched only when max_depth > 12
};

template <class B>
struct NutsMachine {
  B& b;
  dm_rng_key key;
  int max_depth;
  double min_delta;
  int n_slots;
  uint64_t freemask = 0;
  uint32_t n_exp = 0;
  uint32_t t = 0;
  int status = 0;

  DHMC_M NutsMachine(B& b_, dm_rng_key k, int md, double mind, int nslots)
      : b(b_), key(k), max_depth(md), min_delta(mind), n_slots(nslots) {}

  // ---- slot pool (bit set = free).  Low indices are the on-chip slots.  Slots 0…63 live in the register word
  // `freemask`; deeper trees (max_depth > 12: up to 164 slots) spill to TopState::free_hi, which the common
  // configurations never touch; the spill paths exist only in backends with kDeep (separate kernel instantiations), so the
  // max_depth <= 12 kernels are exactly the single-word code. ----
  DHMC_M static int ffs64(uint64_t m) {        // index of the lowest set bit (m != 0)
#if defined(__CUDA_ARCH__)
    return __ffsll((long long)m) - 1;
#else
    int s = 0;
    while (!((m >> s) & 1ull)) ++s;
    return s;
#endif
  }
  DHMC_M static int fls64(uint64_t m) {        // index of the highest set bit (m != 0)
#if defined(__CUDA_ARCH__)
    return 63 - __clzll((long long)m);
#else
    int s = 63;
    while (!((m >> s) & 1ull)) --s;
    return s;
#endif
  }
  DHMC_M void init_pool() {
    const int r0 = b.reserved_first();           // slots r0, r0 + 1 are reserved (window statistics)
    freemask = n_slots >= 64 ? ~0ull : ((1ull << n_slots) - 1ull);
    if (r0 < 64) freemask &= ~(1ull << r0);
    if (r0 + 1 < 64) freemask &= ~(1ull << (r0 + 1));
    if constexpr (B::kDeep) { if (n_slots > 64) init_pool_hi(r0); }
  }
  DHMC_COLD void init_pool_hi(int r0) {
    TopState& S = b.top();
    for (int w = 1; w < kMaskWords; ++w) {
      const int lo = 64 * w;
      uint64_t m = n_slots >= lo + 64 ? ~0ull : (n_slots > lo ? ((1ull << (n_slots - lo)) - 1ull) : 0ull);
      if (r0 >= lo && r0 < lo + 64) m &= ~(1ull << (r0 - lo));
      if (r0 + 1 >= lo && r0 + 1 < lo + 64) m &= ~(1ull << (r0 + 1 - lo));
      S.free_hi[w - 1] = m;
    }
    b.top_sync();
  }
  DHMC_M int alloc_lo() {
    const uint64_t m = freemask;
    if constexpr (B::kDeep) {
      if (!m && n_slots > 64) return alloc_lo_hi();
    }
    const int s = m ? ffs64(m) : 63;             // (n_slots <= 64: the pool is sized so that a free slot exists)
    freemask = m & ~(1ull << s);
    return s;
  }
  DHMC_COLD int alloc_lo_hi() {
    TopState& S = b.top();
    for (int w = 0; w < kMaskWords - 1; ++w) {
      const uint64_t mh = S.free_hi[w];
      if (mh) {
        const int s = ffs64(mh);
        b.top_sync();
        S.free_hi[w] = mh & ~(1ull << s);
        b.top_sync();
        return 64 * (w + 1) + s;
      }
    }
    return 63;
  }
  DHMC_M int alloc_hi() {
    if constexpr (B::kDeep) {
      if (n_slots > 64) {
        const int s = alloc_hi_hi();
        if (s >= 0) return s;
      }
    }
    const uint64_t m = freemask;
    const int s = m ? fls64(m) : 0;
    freemask = m & ~(1ull << s);
    return s;
  }
  DHMC_COLD int alloc_hi_hi() {
    TopState& S = b.top();
    for (int w = kMaskWords - 2; w >= 0; --w) {
      const uint64_t mh = S.free_hi[w];
      if (mh) {
        const int s = fls64(mh);
        b.top_sync();
        S.free_hi[w] = mh & ~(1ull << s);
        b.top_sync();
        return 64 * (w + 1) + s;
      }
    }
    return -1;
  }
  DHMC_M void release(int s) {
    if constexpr (B::kDeep) {
      if (s < 64) freemask |= (1ull << s);
      else release_hi(s);
    } else {
      freemask |= (1ull << s);
    }
  }
  DHMC_COLD void release_hi(int s) {
    TopState& S = b.top();
    b.top_sync();
    S.free_hi[(s >> 6) - 1] |= 1ull << (s & 63);
    b.top_sync();
  }

  // rand_bool_logprob — NUTS.jl:43-45 (no draw when logprob ≥ 0)
  DHMC_M bool rand_bool_logprob(double logprob) {
    if (logprob >= 0) return true;
    double e = b.randexp(key, t, n_exp++);
    return e > -logprob;
  }

  // One NUTS transition from the backend's current (q, ℓq, ∇ℓq).
  // On return the backend's current point is the new position ζ.Q — unless a leapfrog would have started from a
  // non-finite ℓ: then DHMC_CHAIN_LEAPFROG_NONFINITE is set, *ts is not written and the backend's point is
  // meaningless (the caller keeps the chain's stored state).
  DHMC_M void transition(uint32_t t_, double eps, const double* p_override,
                          const uint32_t* dir_override, dhmc_tree_stats* ts) {
    t = t_;
    n_exp = 0;
    // p = rand_p(rng, κ) first, directions second — NUTS.jl:233
    b.draw_momentum(key, t, p_override);
    TopState& S = b.top();
    S.dirs = dir_override ? *dir_override : dm_rand_directions(key, t);
    S.flags = S.dirs;
    S.eps = eps;
    uint32_t& flags = S.flags;
    const double pi0 = b.phase_logdensity();  // logdensity(H, z), NUTS.jl:236

    // ---- initial leaf (trees.jl:285, NUTS.jl:148-159 with is_initial) ----
    init_pool();
    S.s_oq = alloc_hi(); S.s_og = alloc_hi();         // other edge q, ∇ℓ (rarely touched)
    S.s_zq = alloc_hi(); S.s_zg = alloc_hi();         // proposal ζ of the whole tree
    S.s_op = alloc_lo();                              // other edge p  (= far-edge momentum)
    S.s_near = alloc_lo();                            // momentum of the near edge before the subtree
    S.s_rhot = alloc_lo();                            // ρ of the whole tree
    const int& s_oq = S.s_oq; const int& s_og = S.s_og; int& s_zq = S.s_zq; int& s_zg = S.s_zg;
    const int& s_op = S.s_op; const int& s_near = S.s_near; const int& s_rhot = S.s_rhot;
    b.st_q(s_oq); b.st_g(s_og); b.st_p(s_op);
    b.st_q(s_zq); b.st_g(s_zg);
    b.st_p(s_rhot);
    double& other_lq = S.other_lq; double& zt_lq = S.zt_lq; double& zt_H = S.zt_H;
    double& omega_top = S.omega_top; double& v_log = S.v_log; long& v_steps = S.v_steps;
    int& i_near = S.i_near; int& i_far = S.i_far; int& regs_fwd = S.regs_fwd; int& depth = S.depth;
    long& term_l = S.term_l; long& term_r = S.term_r;
    other_lq = b.cur_lq();
    zt_lq = b.cur_lq(); zt_H = pi0;
    omega_top = 0.0;                                  // Δ = 0 for the initial leaf
    v_log = -dm_inf(); v_steps = 0;                   // leaf_acceptance_statistic(Δ, true)
    i_near = 0; i_far = 0;
    regs_fwd = 1;
    depth = 0;
    term_l = 1; term_r = 0;                           // REACHED_MAX_DEPTH
    b.top_sync();

    while (depth < max_depth) {
      const bool fwd = (flags & 1u) != 0;             // next_direction, trees.jl:31-34
      flags >>= 1;
      if (depth > 0 && fwd != (regs_fwd != 0)) {
        // continue from the other edge: exchange it with the register-resident point
        double tmp = b.cur_lq(); b.set_cur_lq(other_lq); other_lq = tmp;
        b.swap_cur(s_oq, s_op, s_og);
        int ti = i_near; i_near = i_far; i_far = ti;
      }
      regs_fwd = fwd ? 1 : 0;
      b.st_p(s_near);
      const double eps_s = fwd ? S.eps : -S.eps;      // move, NUTS.jl:28-31

      // ---------------- adjacent_tree(depth) flattened ----------------
      const unsigned nleaves = 1u << depth;
      int sp = 0;
      bool invalid = false;
      long inv_l = 0, inv_r = 0;
      double vacc_log = 0; long vacc_steps = 0;       // v′ of this adjacent tree
      int pos = i_near;
      // incoming subtree L
      double L_omega = 0, L_vlog = 0, L_zlq = 0, L_zH = 0;
      int L_vsteps = 0, L_ifirst = 0, L_sfirst = -1, L_szq = -1, L_szg = -1;
      bool L_leaf = true;
      for (unsigned k = 1; k <= nleaves; ++k) {
        if (!dm_isfinite(b.cur_lq())) {                   // @argcheck isfinite(Q.ℓq), hamiltonian.jl:276
          status |= DHMC_CHAIN_LEAPFROG_NONFINITE;
          break;
        }
        int lf_flags = 0;
        const double Hn = b.leapfrog(eps_s, &lf_flags);   // move + logdensity(H, z′)
        if (lf_flags & 1) status |= DHMC_CHAIN_NONFINITE_Q;
        pos += fwd ? 1 : -1;
        const double delta = Hn - pi0;                    // NUTS.jl:150
        const double leaf_vlog = dm_min_nan(delta, 0.0);  // leaf_acceptance_statistic
        if (delta < min_delta) {                          // divergent leaf, NUTS.jl:151-154
          inv_l = pos; inv_r = pos;
          vacc_log = leaf_vlog; vacc_steps = 1;
          invalid = true;
        } else {
          L_omega = delta; L_vlog = leaf_vlog; L_vsteps = 1; L_ifirst = pos;
          L_zlq = b.cur_lq(); L_zH = Hn; L_szq = -1; L_szg = -1; L_sfirst = -1; L_leaf = true;
          b.rho_from_p();
#if defined(__CUDA_ARCH__)
          const int c = __ffs((int)k) - 1;                // ctz(k): merges after this leaf
#else
          int c = 0;
          while (!((k >> c) & 1u)) ++c;                   // ctz(k): merges after this leaf
#endif
          for (int j = 0; j < c; ++j) {
            const Entry& E = b.get_entry(--sp);
            const bool turning = b.merge_check(E.sfirst, E.slast, E.srho, L_sfirst, L_leaf);
            // v = combine_visited_statistics(v₋, v₊) precedes the checks, trees.jl:249
            // (ω of the merged tree is computed alongside: two independent logaddexp,
            //  evaluated lane-parallel on the GPU)
            double mv_log, om;
            b.logaddexp2(E.vlog, L_vlog, E.omega, L_omega, &mv_log, &om);
            const int mv_steps = E.vsteps + L_vsteps;
            if (turning) {                                // trees.jl:254-255
              inv_l = E.ifirst; inv_r = pos;
              vacc_log = mv_log; vacc_steps = mv_steps;
              invalid = true;
              break;
            }
            // combine_proposals_and_logweights(…, is_doubling = false), trees.jl:258
            const double logprob2 = L_omega - om;         // biased_progressive_logprob2(false,…)
            if (rand_bool_logprob(logprob2)) {            // ζ₂ (later-built) selected
              release(E.szq); release(E.szg);
            } else {
              if (L_szq >= 0) { release(L_szq); release(L_szg); }
              L_szq = E.szq; L_szg = E.szg; L_zlq = E.zlq; L_zH = E.zH;
            }
            if (!L_leaf) release(L_sfirst);
            L_sfirst = E.sfirst;
            if (!E.leaf) { release(E.slast); release(E.srho); }
            b.rho_commit();
            L_omega = om; L_vlog = mv_log; L_vsteps = mv_steps; L_ifirst = E.ifirst;
            L_leaf = false;
          }
        }
        if (invalid) {
          // unwind: every pending ancestor combines its finished left half with
          // the invalid right half's v and passes the InvalidTree up (trees.jl:248-250)
          while (sp > 0) {
            const Entry& E = b.get_entry(--sp);
            vacc_log = dm_logaddexp(E.vlog, vacc_log);
            vacc_steps = E.vsteps + vacc_steps;
          }
          break;
        }
        if (k < nleaves) {
          // push L: materialise what still lives in registers
          Entry N;
          N.omega = L_omega; N.vlog = L_vlog; N.vsteps = L_vsteps; N.ifirst = L_ifirst;
          N.zlq = L_zlq; N.zH = L_zH;
          if (L_leaf) {
            const int sq = alloc_lo(), sg = alloc_lo(), spp = alloc_lo();
            b.st_q(sq); b.st_g(sg); b.st_p(spp);
            N.szq = (short)sq; N.szg = (short)sg;
            N.sfirst = N.slast = N.srho = (short)spp; N.leaf = 1;
          } else {
            const int sl = alloc_lo(), sr = alloc_lo();
            b.st_p(sl); b.st_rho(sr);
            if (L_szq < 0) {
              L_szq = alloc_lo(); L_szg = alloc_lo();
              b.st_q(L_szq); b.st_g(L_szg);
            }
            N.szq = (short)L_szq; N.szg = (short)L_szg;
            N.sfirst = (short)L_sfirst; N.slast = (short)sl; N.srho = (short)sr; N.leaf = 0;
          }
          b.put_entry(sp++, N);
        } else {
          vacc_log = L_vlog; vacc_steps = L_vsteps;
        }
      }
      if (status & DHMC_CHAIN_LEAPFROG_NONFINITE) return;   // the reference raises: no statistics, no new position
      // ---------------- back in sample_trajectory ----------------
      double om_top;
      b.logaddexp2(v_log, vacc_log, omega_top, L_omega, &v_log, &om_top);   // trees.jl:294, :310
      v_steps += vacc_steps;
      if (invalid) { term_l = inv_l; term_r = inv_r; break; }   // trees.jl:297
      i_near = pos;                                       // trees.jl:303-307
      // combine_proposals_and_logweights(…, is_doubling = true), trees.jl:310
      {
        const double om = om_top;
        const double logprob2 = L_omega - omega_top;      // biased: ω₂ − ω₁
        if (rand_bool_logprob(logprob2)) {
          if (L_szq < 0) {
            b.st_q(s_zq); b.st_g(s_zg);                   // overwrite in place
          } else {
            release(s_zq); release(s_zg);
            s_zq = L_szq; s_zg = L_szg;
          }
          zt_lq = L_zlq; zt_H = L_zH;
        } else if (L_szq >= 0) {
          release(L_szq); release(L_szg);
        }
        omega_top = om;
      }
      depth += 1;                                         // trees.jl:312
      // τ = combine_turn_statistics_in_direction(τ, τ′): the tree so far is the
      // earlier entry with first = far-edge p, last = near-edge p before this subtree
      const bool turning = b.merge_check(s_op, s_near, s_rhot, L_sfirst, L_leaf);
      if (!L_leaf) release(L_sfirst);
      if (turning) {                                      // trees.jl:316
        term_l = regs_fwd ? i_far : i_near;
        term_r = regs_fwd ? i_near : i_far;
        break;
      }
      b.rho_commit();
      b.st_rho(s_rhot);
    }

    // TreeStatisticsNUTS — NUTS.jl:238-239
    ts->pi = zt_H;
    ts->depth = depth;
    ts->left = term_l; ts->right = term_r;
    ts->acceptance_rate = dm_min_nan(dm_exp(v_log) / (double)v_steps, 1.0);  // NUTS.jl:87
    ts->steps = v_steps;
    ts->directions = S.dirs;
    ts->pad = 0;
    // new position ζ.Q
    b.ld_q(s_zq); b.ld_g(s_zg); b.set_cur_lq(zt_lq);
  }

  // ---- dual averaging, src/stepsize.jl:121-170 ----
  struct DA { double mu; long m; double Hbar, logeps, logepsbar; };
  DHMC_M static DA da_init(double eps) {                 // initial_adaptation_state :134-138
    DA A; double le = dm_log(eps);
    A.mu = dm_log(10.0) + le; A.m = 1; A.Hbar = 0.0; A.logeps = le; A.logepsbar = 0.0;
    return A;
  }
  DHMC_M static void da_adapt(DA& A, const AdaptConfig& P, double a) {   // adapt_stepsize :147-156
    A.m += 1;
    A.Hbar += (P.delta - a - A.Hbar) / (double)(A.m + P.t0);
    A.logeps = A.mu - dm_sqrt((double)A.m) / P.gamma * A.Hbar;
    A.logepsbar += dm_pow((double)A.m, -P.kappa) * (A.logeps - A.logepsbar);
  }

  // N transitions of one chain: warmup(::TuningNUTS) mcmc.jl:258-286 when
  // cfg.adapt / cfg.metric are set, plain mcmc (mcmc.jl:366-381) otherwise.
  // Returns the step size for the next stage (final_ϵ).  sink(n, stats, eps)
  // is called after each transition with the new position in the backend.
  template <class Sink>
  DHMC_M double run(uint32_t t0, int N, double eps, const AdaptConfig& cfg,
                     const double* p_override, const uint32_t* dir_override, Sink& sink) {
    TopState& S = b.top();
    if (!(eps > 0)) {                      // @argcheck ϵ > 0, stepsize.jl:135 (NaN after a failed search included)
      status |= DHMC_CHAIN_BAD_STEPSIZE;
      steps_out = 0;
      return eps;
    }
    {
      DA A0 = da_init(eps);
      S.da_mu = A0.mu; S.da_m = A0.m; S.da_Hbar = A0.Hbar; S.da_logeps = A0.logeps; S.da_logepsbar = A0.logepsbar;
    }
    if (cfg.metric != DHMC_METRIC_NOTHING) b.metric_reset(cfg.metric);
    S.total_steps = 0;
    for (int n = 0; n < N; ++n) {
      const double e = cfg.adapt ? dm_exp(S.da_logeps) : eps;   // current_ϵ :163
      dhmc_tree_stats ts;
      transition(t0 + (uint32_t)n, e, p_override, dir_override, &ts);
      if (status & DHMC_CHAIN_LEAPFROG_NONFINITE) { steps_out = S.total_steps; return eps; }   // the chain stops here
      S.total_steps += ts.steps;
      sink(n, ts, e);
      if (cfg.adapt) {
        const double a = ts.acceptance_rate;
        if (a >= 0 && a <= 1) {                                // @argcheck 0 ≤ a ≤ 1
          DA A{S.da_mu, S.da_m, S.da_Hbar, S.da_logeps, S.da_logepsbar};
          da_adapt(A, cfg, a);
          S.da_m = A.m; S.da_Hbar = A.Hbar; S.da_logeps = A.logeps; S.da_logepsbar = A.logepsbar;
        } else {
          status |= DHMC_CHAIN_BAD_ACCEPTANCE;
        }
      }
      if (cfg.metric != DHMC_METRIC_NOTHING) b.metric_push(cfg.metric, n + 1);
    }
    if (cfg.metric != DHMC_METRIC_NOTHING) b.metric_finish(cfg.metric, N);   // sample_M⁻¹, mcmc.jl:209-211
    steps_out = S.total_steps;
    return cfg.adapt ? dm_exp(S.da_logepsbar) : eps;             // final_ϵ :170
  }
  long steps_out = 0;

  // find_initial_stepsize — stepsize.jl:46-60 with A = local_log_acceptance_ratio
  // (:75-85) around the current point; momentum from the search stream
  // (mcmc.jl:138).  Returns ϵ, or NaN after setting the status bit.
  DHMC_M double find_initial_stepsize(double initial_eps, double log_threshold, int maxiter,
                                       const double* p_override) {
    b.draw_search_momentum(key, p_override);
    const double l0 = b.phase_logdensity();
    if (!dm_isfinite(l0)) { status |= DHMC_CHAIN_SEARCH_FAILED; return dm_nan(); }
    init_pool();
    const int sq = alloc_lo(), sp = alloc_lo(), sg = alloc_lo();
    b.st_q(sq); b.st_p(sp); b.st_g(sg);
    const double lq0 = b.cur_lq();
    double eps = initial_eps;
    int fl = 0;
    double Ae = b.leapfrog(eps, &fl) - l0;
    const bool dbl = Ae > log_threshold;
    double found = dm_nan();
    for (int it = 0; it < maxiter; ++it) {
      const double eps1 = dbl ? 2 * eps : eps / 2;
      b.ld_q(sq); b.ld_p(sp); b.ld_g(sg); b.set_cur_lq(lq0);
      const double Ae1 = b.leapfrog(eps1, &fl) - l0;
      if (dbl ? (Ae1 < log_threshold) : (Ae1 > log_threshold)) { found = eps1; break; }
      eps = eps1;
    }
    if (fl & 1) status |= DHMC_CHAIN_NONFINITE_Q;
    b.ld_q(sq); b.ld_p(sp); b.ld_g(sg); b.set_cur_lq(lq0);
    if (found != found) status |= DHMC_CHAIN_SEARCH_FAILED;
    return found;
  }
};

}  // namespace dhmc
